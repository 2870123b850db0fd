"""Reshaping per-env wrapper chains (FrameStack, TimeAwareObservation, FlattenObservation) and action stages
(ClipAction, RescaleAction) on the GPU: both backends against the reference fixture, the engine + chain in lockstep
with the chain-less engine + the numpy restatement (oracle/subenv_shapes.py) at launch shapes, device sampling of a
rescaled action space, snapshots / clone / pickle carrying the frame history and t, and the vector-level
NormalizeObservation over a stacked observation."""
import copy
import os
import pickle

import numpy as np
import pytest

from conftest import GOLDEN
from gym_b200 import subenv
from oracle import gen_subenv_shape_fixtures as gen
from oracle.subenv_shapes import SubenvShapeRef, apply_actions

pytestmark = pytest.mark.gpu

FIXTURE = os.path.join(GOLDEN, "reference", "subenv_shape_wrappers.npz")


def _torch():
    import torch
    return torch


def host(x):
    return x.cpu().numpy() if hasattr(x, "cpu") else np.asarray(x)


def bits_equal(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def close(a, b):
    """The CartPole bound of the parity tests: float32 elements within 1e-5 relative (1e-7 absolute floor)."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return a.shape == b.shape and bool(np.all(np.abs(a - b) <= 1e-7 + 1e-5 * np.abs(b)))


def _final_rows(infos, done):
    """(rows of the finishing envs, episode r, episode l) from either backend's infos."""
    if not done.any():
        return None, None, None
    fo = infos["final_observation"]
    if isinstance(fo, np.ndarray) and fo.dtype == object:
        rows = np.stack([fo[i] for i in np.flatnonzero(done)])
        eps = [infos["final_info"][i].get("episode") for i in np.flatnonzero(done)]
        if eps[0] is None:
            return rows, None, None
        return rows, np.array([e["r"] for e in eps]), np.array([e["l"] for e in eps])
    rows = host(fo)[done]
    if "final_info" not in infos:
        return rows, None, None
    ep = infos["final_info"]["episode"]
    return rows, host(ep["r"])[done], host(ep["l"])[done]


@pytest.fixture(scope="module")
def fixture():
    z = np.load(FIXTURE)
    return {k: z[k] for k in z.files}


@pytest.mark.parametrize("backend", ["numpy", "torch"])
@pytest.mark.parametrize("env_id,name,stages", gen.cases(), ids=[f"{e}-{n}" for e, n, _ in gen.cases()])
def test_matches_reference_fixture(fixture, backend, env_id, name, stages):
    import gym_b200
    c = gen.load_case(fixture, env_id, name)
    env = gym_b200.vector.make(env_id, gen.N, wrappers=stages, max_episode_steps=gen.MAX_STEPS, backend=backend)
    assert env.single_observation_space.shape == c["obs"].shape[2:]
    assert bits_equal(env.single_observation_space.low, c["obs_low"])
    assert tuple(env.observation_space.shape) == (gen.N,) + c["obs"].shape[2:]
    if "act_low" in c:
        assert bits_equal(env.single_action_space.low, c["act_low"])
        assert bits_equal(env.single_action_space.high, c["act_high"])
    same = close if env_id.startswith("CartPole") else bits_equal
    obs, _ = env.reset(seed=gen.SEED)
    assert same(host(obs), c["obs0"])
    for t in range(gen.T):
        if t == gen.MID:
            obs, _ = env.reset(seed=gen.SEED_MID)
            assert same(host(obs), c["obs_mid"]), t
        o, r, te, tr, infos = env.step(c["actions"][t])
        te, tr = host(te).astype(bool), host(tr).astype(bool)
        assert bits_equal(te, c["terminated"][t]) and bits_equal(tr, c["truncated"][t]), t
        assert host(o).shape == c["obs"][t].shape and same(host(o), c["obs"][t]), t
        assert bits_equal(host(r), c["reward"][t]), t
        done = te | tr
        rows, ep_r, ep_l = _final_rows(infos, done)
        if rows is not None:
            want = c["final_obs"][t][done]
            if not c["final_f64"][t][done].all():
                want = want.astype(np.float32)
            assert rows.dtype == want.dtype and same(rows, want), t
            if ep_r is not None:
                assert bits_equal(ep_r, c["episode_r"][t][done]) and bits_equal(ep_l, c["episode_l"][t][done]), t
    env.close()


def _lockstep(env_id, n, T, windows, stages, backend="torch", max_episode_steps=30, seed=5):
    """engine + chain vs the chain-less engine + restatement, fed the same actions (the chain-less engine gets them
    through the restatement's action stages); rows `windows` of the batch are checked every step."""
    import gym_b200
    torch = _torch()
    plain = gym_b200.vector.make(env_id, n, max_episode_steps=max_episode_steps, backend=backend)
    env = gym_b200.vector.make(env_id, n, wrappers=stages, max_episode_steps=max_episode_steps, backend=backend)
    desc = [s.describe() for s in stages]
    refs = [SubenvShapeRef(desc, env_id, hi - lo, plain.obs_dim) for lo, hi in windows]
    shape = refs[0].shape
    assert tuple(env.single_observation_space.shape) == shape
    o_raw, _ = plain.reset(seed=seed)
    o, _ = env.reset(seed=seed)
    for (lo, hi), ref in zip(windows, refs):
        assert bits_equal(host(o)[lo:hi], ref.reset(host(o_raw)[lo:hi]).reshape((hi - lo,) + shape))
    rng = np.random.default_rng(seed)
    finished = 0
    for t in range(T):
        if plain.discrete:
            a = a_raw = rng.integers(0, plain.single_action_space.n, size=n)
        else:
            a = rng.uniform(-1.6, 1.6, size=(n, plain.act_dim)).astype(np.float32)
            a_raw = apply_actions(desc, plain.single_action_space.low, plain.single_action_space.high, a)
        if backend == "torch":
            a, a_raw = torch.as_tensor(a, device=env.device), torch.as_tensor(a_raw, device=env.device)
        ro, rr, rte, rtr, rinfo = plain.step(a_raw)
        wo, wr, wte, wtr, winfo = env.step(a)
        rte, rtr = host(rte).astype(bool), host(rtr).astype(bool)
        assert bits_equal(host(wte).astype(bool), rte) and bits_equal(host(wtr).astype(bool), rtr), t
        done = rte | rtr
        finished += int(done.sum())
        raw_fin = host(rinfo["final_observation"]) if backend == "torch" else plain._hio["final_obs"]
        if backend == "torch":
            w_fin = host(winfo["final_observation"])
        else:
            w_fin = env._hio.get("final_obs64", env._hio["final_obs"])
        for (lo, hi), ref in zip(windows, refs):
            o2, r2, f2, er, el = ref.step(host(ro)[lo:hi], host(rr)[lo:hi], rte[lo:hi], rtr[lo:hi], raw_fin[lo:hi])
            d = done[lo:hi]
            assert bits_equal(host(wo)[lo:hi], o2.reshape((hi - lo,) + shape)), (t, lo)
            assert bits_equal(host(wr)[lo:hi], r2), (t, lo)
            assert bits_equal(w_fin[lo:hi][d], f2.reshape((hi - lo,) + shape)[d]), (t, lo)
    assert finished > 0
    env.close()
    plain.close()


RAGGED = (1 << 16) + 77


@pytest.mark.parametrize("stages", [[subenv.FrameStack(4)],
                                    [subenv.FrameStack(4), subenv.TimeAwareObservation()],
                                    [subenv.NormalizeObservation(), subenv.TimeAwareObservation(),
                                     subenv.FrameStack(3), subenv.FlattenObservation()]],
                         ids=["fs4", "fs4_time", "mix"])
def test_lockstep_cartpole_ragged_tile(stages):
    n = RAGGED
    _lockstep("CartPole-v1", n, 40, [(0, 1024), (n // 2 - 300, n // 2 + 500), (n - 1100, n)], stages,
              max_episode_steps=15)


def test_lockstep_lunarlander_continuous_rescale_frame_stack():
    stages = [subenv.RescaleAction(np.float32(-0.5), 0.5), subenv.FrameStack(3), subenv.RecordEpisodeStatistics()]
    _lockstep("LunarLanderContinuous-v2", 2000, 50, [(0, 2000)], stages, max_episode_steps=30)


@pytest.mark.parametrize("backend", ["torch", "numpy"])
def test_lockstep_bipedal_walker_time_aware_frame_stack(backend):
    """24-wide frames, a 4-deep stack of float64 rows (TimeAwareObservation before FrameStack)."""
    stages = [subenv.ClipAction(), subenv.NormalizeObservation(), subenv.TimeAwareObservation(), subenv.FrameStack(4)]
    _lockstep("BipedalWalker-v3", 600, 60, [(0, 600)], stages, backend=backend, max_episode_steps=40)


def test_lockstep_numpy_backend_across_host_chunks():
    """2^19 + 77 envs: the host-buffer path steps, runs the chain into its W-wide HBM rows and copies them back in
    two chunks."""
    n = (1 << 19) + 77
    stages = [subenv.TimeAwareObservation(), subenv.FrameStack(3)]
    _lockstep("CartPole-v1", n, 25, [(0, 1024), (n // 2 - 700, n // 2 + 700), (n - 1024, n)], stages,
              backend="numpy", max_episode_steps=12)


def test_lockstep_pendulum_rescale_and_clip_numpy():
    stages = [subenv.RescaleAction(-1, 1), subenv.ClipAction(), subenv.FrameStack(2)]
    _lockstep("Pendulum-v1", 3000, 40, [(0, 3000)], stages, backend="numpy", max_episode_steps=25)


def test_sample_actions_on_a_rescaled_space():
    import gym_b200
    n = 4099
    env = gym_b200.vector.make("BipedalWalker-v3", n, wrappers=[subenv.RescaleAction(-0.25, np.array(
        [0.5, 0.75, 1.0, 0.125], np.float32))])
    env.action_space.seed(17)
    twin = copy.deepcopy(env.action_space)
    for _ in range(3):
        assert bits_equal(host(env.sample_actions()), twin.sample())
    x = host(env.sample_actions())
    assert x.min() >= np.float32(-0.25) and bool((x <= env.single_action_space.high).all())
    env.close()


def _run(env, acts):
    outs = []
    for a in acts:
        o, r, te, tr, infos = env.step(a)
        done = host(te) | host(tr)
        outs.append([host(o).copy(), host(r).copy(), host(te).copy(), host(tr).copy(),
                     host(infos["final_observation"])[done].copy()])
    return outs


def _same_runs(a, b):
    for x, y in zip(a, b):
        for u, v in zip(x, y):
            assert bits_equal(u, v)


@pytest.mark.parametrize("env_id", ["CartPole-v1", "Pendulum-v1"])
def test_snapshot_restore_clone_pickle_carry_history_and_t(env_id):
    import gym_b200
    n = 300
    stages = [subenv.NormalizeObservation(), subenv.TimeAwareObservation(), subenv.FrameStack(4)]
    if env_id == "Pendulum-v1":
        stages = [subenv.RescaleAction(-1, 1)] + stages
    env = gym_b200.vector.make(env_id, n, wrappers=stages, max_episode_steps=45)
    rng = np.random.default_rng(3)

    def acts(k):
        if env.discrete:
            return [rng.integers(0, 2, size=n) for _ in range(k)]
        return [rng.uniform(-1.2, 1.2, size=(n, 1)).astype(np.float32) for _ in range(k)]

    env.reset(seed=4)
    _run(env, acts(23))
    snap = env.snapshot()
    assert {"history", "head", "t"} <= set(snap.extras["subenv"])
    assert tuple(snap.obs.shape) == (n, 4, env.obs_dim + 1)
    blob = pickle.loads(pickle.dumps(env))
    twin = copy.deepcopy(env)
    fresh = gym_b200.vector.make(env_id, n, wrappers=stages, max_episode_steps=45)
    o, _ = fresh.restore(snap)
    assert bits_equal(host(o), host(snap.obs))
    later = acts(110)
    first = _run(env, later)
    for other in (blob, twin, fresh):
        _same_runs(first, _run(other, later))
    # clone: env i continues as env src[i] did, history and t included
    src = rng.permutation(n)
    twin.restore(snap)
    blob.restore(snap)
    twin.clone(src)
    for a in acts(60):
        b = np.empty_like(a)
        b[src] = a
        o1, r1, *_ = twin.step(a)
        o2, r2, *_ = blob.step(b)
        assert bits_equal(host(o1), host(o2)[src]) and bits_equal(host(r1), host(r2)[src])
    # part of the batch, into the numpy backend
    idx = np.arange(5, 12)
    part = env.snapshot(idx)
    np_env = gym_b200.vector.make(env_id, n, wrappers=stages, max_episode_steps=45, backend="numpy")
    np_env.reset(seed=0)
    o, _ = np_env.restore(part, indices=idx)
    assert bits_equal(o[idx], host(part.obs))
    for e in (env, blob, twin, fresh, np_env):
        e.close()


def test_vector_normalize_observation_over_a_frame_stack():
    """gym_b200.wrappers.NormalizeObservation keeps batch statistics per element of the flattened stacked row (a
    (2, 4) CartPole stack: 8 columns, a width its statistics kernel takes)."""
    import gym_b200
    from gym_b200 import wrappers
    n = 512
    env = wrappers.NormalizeObservation(gym_b200.vector.make("CartPole-v1", n, wrappers=[subenv.FrameStack(2)]))
    assert env.obs_rms.d == 8
    ref = wrappers.NormalizeObservation(gym_b200.vector.make("CartPole-v1", n, wrappers=[
        subenv.FrameStack(2), subenv.FlattenObservation()]))
    o, _ = env.reset(seed=1)
    o2, _ = ref.reset(seed=1)
    assert tuple(o.shape) == (n, 2, 4) and bits_equal(host(o).reshape(n, 8), host(o2))
    rng = np.random.default_rng(0)
    for _ in range(20):
        a = rng.integers(0, 2, size=n)
        o, *_ = env.step(a)
        o2, *_ = ref.step(a)
        assert bits_equal(host(o).reshape(n, 8), host(o2))
    env.close()
    ref.close()
