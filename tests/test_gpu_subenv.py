"""Per-env wrapper chains on the GPU (``vector.make(id, n, wrappers=[...])``): both backends against the reference
fixture, the engine + chain in lockstep with the chain-less engine + the numpy restatement (oracle/subenv_chain.py)
at the batch sizes the kernels are launched with, ClipAction with infinite actions, and snapshots, clone, pickle and
deepcopy of wrapped envs."""
import copy
import os
import pickle

import numpy as np
import pytest

from conftest import GOLDEN
from gym_b200 import error, subenv
from oracle import gen_subenv_fixtures as gen
from oracle.subenv_chain import SubenvChainRef

pytestmark = pytest.mark.gpu

FIXTURE = os.path.join(GOLDEN, "reference", "subenv_wrappers.npz")
ALL_IDS = ["CartPole-v1", "MountainCar-v0", "MountainCarContinuous-v0", "Pendulum-v1", "Acrobot-v1", "LunarLander-v2",
           "LunarLanderContinuous-v2", "BipedalWalker-v3", "BipedalWalkerHardcore-v3"]


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


def ppo_chain(continuous):
    return gen.chains(continuous)["ppo"]


def _final_rows(env, infos, done):
    """(rows of the finishing envs, episode r, episode l) from either backend's infos."""
    if not done.any():
        return None, None, None
    fo = infos["final_observation"]
    if isinstance(fo, np.ndarray) and fo.dtype == object:
        rows = np.stack([fo[i] for i in np.flatnonzero(done)])
        eps = [infos["final_info"][i].get("episode") for i in np.flatnonzero(done)]
        if eps[0] is None:
            return rows, None, None
        assert all(type(e["r"]) is np.float32 and type(e["l"]) is np.int32 for e in eps)
        return rows, np.array([e["r"] for e in eps]), np.array([e["l"] for e in eps])
    assert bits_equal(host(infos["_final_observation"]), done)
    rows = host(fo)[done]
    if "final_info" not in infos:
        return rows, None, None
    assert bits_equal(host(infos["_final_info"]), done)
    ep = infos["final_info"]["episode"]
    return rows, host(ep["r"])[done], host(ep["l"])[done]


@pytest.fixture(scope="module")
def fixture():
    z = np.load(FIXTURE)
    return {k: z[k] for k in z.files}


@pytest.mark.parametrize("backend", ["numpy", "torch"])
@pytest.mark.parametrize("env_id,name", [(e, c) for e in gen.CLASSIC for c in ("ppo", "stats", "reordered")])
def test_matches_reference_fixture(fixture, backend, env_id, name):
    import gym_b200
    p = f"{env_id}/{name}/"
    c = {k[len(p):]: v for k, v in fixture.items() if k.startswith(p)}
    stages = gen.chains(env_id in ("MountainCarContinuous-v0", "Pendulum-v1"))[name]
    env = gym_b200.vector.make(env_id, gen.N, wrappers=stages, max_episode_steps=gen.MAX_STEPS, backend=backend)
    exact = not env_id.startswith("CartPole")
    same = bits_equal if exact else close

    obs, _ = env.reset(seed=gen.SEED)
    assert same(host(obs), c["obs0"])
    for t in range(gen.T):
        if t == gen.MID:
            obs, _ = env.reset(seed=gen.SEED_MID)
            assert same(host(obs), c["obs_mid"]), t
        o, r, te, tr, infos = env.step(c["actions"][t])
        te, tr = host(te).astype(bool), host(tr).astype(bool)
        assert bits_equal(te, c["terminated"][t]) and bits_equal(tr, c["truncated"][t]), t
        assert same(host(o), c["obs"][t]), t
        assert bits_equal(host(r), c["reward"][t]), t    # CartPole's rewards and flags are exact, so is their chain
        done = te | tr
        if backend == "numpy" and not done.any():
            assert infos == {}
        rows, ep_r, ep_l = _final_rows(env, infos, done)
        if rows is not None:
            want = c["final_obs"][t][done]
            if not c["final_f64"][t][done].all():
                want = want.astype(np.float32)
            assert rows.dtype == want.dtype and same(rows, want), t
            assert ep_r is not None   # every fixture chain records episode statistics
            assert bits_equal(ep_r, c["episode_r"][t][done]) and bits_equal(ep_l, c["episode_l"][t][done]), t
    env.close()


def _lockstep(env_id, n, T, windows, backend="torch", max_episode_steps=30, seed=5, stages=None):
    """engine + chain (default: the PPO chain) vs the chain-less engine + restatement, both fed the same actions; rows
    `windows` of the batch are checked every step.  -> number of envs that terminated with reward -100."""
    import gym_b200
    torch = _torch()
    plain = gym_b200.vector.make(env_id, n, max_episode_steps=max_episode_steps, backend=backend)
    continuous = not plain.discrete
    stages = ppo_chain(continuous) if stages is None else stages
    env = gym_b200.vector.make(env_id, n, wrappers=stages, max_episode_steps=max_episode_steps, backend=backend)
    refs = [SubenvChainRef([s.describe() for s in stages], env_id, hi - lo, plain.obs_dim) for lo, hi in windows]
    o_raw, _ = plain.reset(seed=seed)
    o, _ = env.reset(seed=seed)
    for (lo, hi), ref in zip(windows, refs):
        assert bits_equal(host(o)[lo:hi], ref.reset(host(o_raw)[lo:hi]))
    rng = np.random.default_rng(seed)
    finished = falls = 0
    for t in range(T):
        if plain.discrete:
            a = rng.integers(0, plain.single_action_space.n, size=n)
            a_raw = a
        else:
            a = rng.uniform(-1.6, 1.6, size=(n, plain.act_dim)).astype(np.float32) * np.float32(
                plain.single_action_space.high[0])
            a_raw = np.clip(a, plain.single_action_space.low, plain.single_action_space.high)
        if backend == "torch":
            a, a_raw = torch.as_tensor(a, device=env.device), torch.as_tensor(a_raw, device=env.device)
        ro, rr, rte, rtr, rinfo = plain.step(a_raw)
        wo, wr, wte, wtr, winfo = env.step(a)
        rte, rtr = host(rte).astype(bool), host(rtr).astype(bool)
        assert bits_equal(host(wte).astype(bool), rte) and bits_equal(host(wtr).astype(bool), rtr), t
        done = rte | rtr
        finished += int(done.sum())
        falls += int((rte & (host(rr) == -100.0)).sum())
        raw_fin = host(rinfo["final_observation"]) if backend == "torch" else plain._hio["final_obs"]
        w_fin = winfo.get("final_observation")
        w_fin = host(w_fin) if backend == "torch" else env._hio["final_obs64"]
        w_ep = winfo.get("final_info")
        for (lo, hi), ref in zip(windows, refs):
            o2, r2, f2, er, el = ref.step(host(ro)[lo:hi], host(rr)[lo:hi], rte[lo:hi], rtr[lo:hi], raw_fin[lo:hi])
            d = done[lo:hi]
            assert bits_equal(host(wo)[lo:hi], o2) and bits_equal(host(wr)[lo:hi], r2), (t, lo)
            assert bits_equal(w_fin[lo:hi][d], f2[d]), (t, lo)
            if backend == "torch" and d.any():
                assert bits_equal(host(w_ep["episode"]["r"])[lo:hi][d], er[d]), (t, lo)
                assert bits_equal(host(w_ep["episode"]["l"])[lo:hi][d], el[d]), (t, lo)
            if backend == "numpy" and d.any():
                eps = [w_ep[lo + j]["episode"] for j in np.flatnonzero(d)]
                assert bits_equal(np.array([e["r"] for e in eps], np.float32), er[d]), (t, lo)
                assert bits_equal(np.array([e["l"] for e in eps], np.int32), el[d]), (t, lo)
    assert finished > 0
    env.close()
    plain.close()
    return falls


@pytest.mark.parametrize("env_id", ALL_IDS)
@pytest.mark.parametrize("n", [1, 255, 257, 1000])
def test_lockstep_with_restatement_across_cta_boundaries(env_id, n):
    T = 60 if env_id.startswith(("Lunar", "Bipedal")) else 90
    _lockstep(env_id, n, T, [(0, n)], max_episode_steps=40)


@pytest.mark.parametrize("backend", ["torch", "numpy"])
@pytest.mark.parametrize("env_id", ["BipedalWalker-v3", "BipedalWalkerHardcore-v3"])
def test_lockstep_walker_falls_through_inexact_reward_clips(env_id, backend):
    """A fall's reward is the Python int -100: np.clip turns it into an np.float64 with float64 bounds, where the
    walker's other (np.float32) rewards keep float32 and round the bounds."""
    stages = [subenv.ClipReward(-0.7, 0.7), subenv.NormalizeReward(gamma=0.9), subenv.RecordEpisodeStatistics(),
              subenv.NormalizeObservation(), subenv.ClipObservation(-0.3, 0.3)]
    falls = _lockstep(env_id, 500, 200, [(0, 500)], backend=backend, max_episode_steps=400, stages=stages)
    assert falls > 0


def test_lockstep_numpy_backend_across_host_chunks():
    """2^19 + 77 envs: the host-buffer path steps, runs the chain and copies back in two chunks."""
    n = (1 << 19) + 77
    _lockstep("CartPole-v1", n, 30, [(0, 1024), (n // 2 - 700, n // 2 + 700), (n - 1024, n)], backend="numpy",
              max_episode_steps=12)


@pytest.mark.parametrize("env_id", ["Pendulum-v1", "LunarLander-v2", "BipedalWalker-v3"])
def test_lockstep_numpy_backend(env_id):
    _lockstep(env_id, 300, 50, [(0, 300)], backend="numpy", max_episode_steps=35)


def test_lockstep_cartpole_2_20():
    n = 1 << 20
    _lockstep("CartPole-v1", n, 40, [(0, 2048), (n // 2 - 777, n // 2 + 1271), (n - 2048, n)], max_episode_steps=15)


def test_lockstep_lunarlander_2_16():
    n = 1 << 16
    _lockstep("LunarLander-v2", n, 40, [(0, 1024), (n // 2 - 300, n // 2 + 724), (n - 1024, n)], max_episode_steps=25)


@pytest.mark.parametrize("backend", ["torch", "numpy"])
@pytest.mark.parametrize("env_id", ["Pendulum-v1", "MountainCarContinuous-v0", "BipedalWalker-v3"])
def test_clip_action_takes_infinite_actions(env_id, backend):
    import gym_b200
    n = 64
    env = gym_b200.vector.make(env_id, n, wrappers=[subenv.ClipAction()], backend=backend)
    plain = gym_b200.vector.make(env_id, n, backend=backend)
    space = plain.single_action_space
    env.reset(seed=9)
    plain.reset(seed=9)
    rng = np.random.default_rng(0)
    for t in range(20):
        a = rng.choice(np.array([-np.inf, np.inf, 0.25, -3.0], np.float32), size=(n, plain.act_dim))
        out = env.step(a)
        ref = plain.step(np.clip(a, space.low, space.high))
        for k in range(4):
            assert bits_equal(host(out[k]), host(ref[k])), (t, k)
    env.close()
    plain.close()


def _run(env, acts):
    """Outputs of a torch-backend env over `acts`; the episode fields of the finishing envs only."""
    outs = []
    for a in acts:
        o, r, te, tr, infos = env.step(a)
        done = host(te) | host(tr)
        ep = infos["final_info"]["episode"]
        outs.append([host(o).copy(), host(r).copy(), host(te).copy(), host(tr).copy(), host(ep["r"])[done],
                     host(ep["l"])[done]])
    return outs


def _same_runs(a, b):
    for x, y in zip(a, b):
        for u, v in zip(x, y):
            assert bits_equal(u, v)


@pytest.mark.parametrize("env_id", ["CartPole-v1", "Pendulum-v1", "LunarLanderContinuous-v2"])
def test_snapshot_restore_pickle_deepcopy_continue_bit_identically(env_id):
    import gym_b200
    n = 300
    env = gym_b200.vector.make(env_id, n, wrappers=ppo_chain(env_id != "CartPole-v1"), max_episode_steps=20)
    rng = np.random.default_rng(3)

    def acts(k):
        if env.discrete:
            return [rng.integers(0, env.single_action_space.n, size=n) for _ in range(k)]
        return [rng.uniform(-2, 2, size=(n, env.act_dim)).astype(np.float32) for _ in range(k)]

    env.reset(seed=4)
    _run(env, acts(25))
    snap = env.snapshot()
    assert "wrappers" in snap.header["config"] and "subenv" in snap.extras
    twin = copy.deepcopy(env)
    blob = pickle.loads(pickle.dumps(env))
    later = acts(30)
    first = _run(env, later)
    _same_runs(first, _run(twin, later))
    _same_runs(first, _run(blob, later))
    env.restore(snap)
    _same_runs(first, _run(env, later))
    # part of the batch: restoring envs 5..9 brings exactly their rows (and chain state) back
    idx = np.arange(5, 10)
    part = twin.snapshot(idx)
    env.restore(part, indices=idx)
    twin.restore(part, indices=idx)
    nxt = acts(10)
    _same_runs(_run(env, nxt), _run(twin, nxt))
    for e in (env, twin, blob):
        e.close()


def test_clone_copies_the_source_envs_statistics():
    import gym_b200
    n = 257
    env = gym_b200.vector.make("Pendulum-v1", n, wrappers=ppo_chain(True), max_episode_steps=20)
    env.reset(seed=1)
    rng = np.random.default_rng(1)
    for _ in range(13):
        env.step(rng.uniform(-2, 2, size=(n, 1)).astype(np.float32))
    twin = copy.deepcopy(env)
    src = rng.permutation(n)
    env.clone(src)
    for _ in range(30):
        a = rng.uniform(-2, 2, size=(n, 1)).astype(np.float32)
        b = np.empty_like(a)
        b[src] = a
        o, r, te, tr, _ = env.step(a)
        o2, r2, te2, tr2, _ = twin.step(b)
        assert bits_equal(host(o), host(o2)[src]) and bits_equal(host(r), host(r2)[src])
    env.close()
    twin.close()


def test_snapshots_refuse_another_chain_and_chain_less_headers_are_unchanged():
    import gym_b200
    plain = gym_b200.vector.make("Pendulum-v1", 16)
    plain.reset(seed=0)
    snap = plain.snapshot()
    assert set(snap.header["config"]) == {"max_episode_steps", "autoreset", "params", "flags"} and snap.extras == {}
    a = gym_b200.vector.make("Pendulum-v1", 16, wrappers=[subenv.NormalizeObservation()])
    b = gym_b200.vector.make("Pendulum-v1", 16, wrappers=[subenv.NormalizeObservation(epsilon=1e-3)])
    a.reset(seed=0)
    b.reset(seed=0)
    for src, dst in ((snap, a), (a.snapshot(), b), (a.snapshot(), plain)):
        with pytest.raises(error.Error):
            dst.restore(src)
    for e in (plain, a, b):
        e.close()


def test_reset_with_seed_keeps_statistics():
    import gym_b200
    n = 32
    env = gym_b200.vector.make("Acrobot-v1", n, wrappers=[subenv.NormalizeObservation(), subenv.NormalizeReward(),
                                                           subenv.RecordEpisodeStatistics()])
    env.reset(seed=1)
    for _ in range(5):
        env.step(np.ones(n, np.int64))
    st = env._chain.state
    count = st["obs_stats"][-1].clone()
    ret = st["rew_stats"].clone()
    env.reset(seed=2)
    assert bool((st["obs_stats"][-1] == count + 1).all())
    assert bits_equal(host(st["rew_stats"]), host(ret))
    assert int(st["ep_length"].abs().sum()) == 0
    env.close()


def test_reference_wrapper_classes_through_gym_vector_env():
    from oracle.ref_gym import import_reference
    import functools
    try:
        gym = import_reference()
    except ImportError:
        pytest.skip("the reference is not installed in oracle/_ref")
    from gym_b200.gym_compat import GymVectorEnv
    w = gym.wrappers
    env = GymVectorEnv("MountainCarContinuous-v0", 8, backend="numpy", max_episode_steps=gen.MAX_STEPS,
                       wrappers=[w.RecordEpisodeStatistics, w.ClipAction, w.NormalizeObservation,
                                 functools.partial(w.NormalizeReward, gamma=0.99)])
    assert isinstance(env, gym.vector.VectorEnv)
    assert env._chain.stages == [subenv.RecordEpisodeStatistics(), subenv.ClipAction(), subenv.NormalizeObservation(),
                                 subenv.NormalizeReward(0.99)]
    env.reset(seed=0)
    env.step(np.full((8, 1), 5.0, np.float32))
    env.close()


@pytest.mark.parametrize("stages", [[subenv.NormalizeReward()],
                                    [subenv.ClipReward(-0.3, 0.3), subenv.RecordEpisodeStatistics()],
                                    [subenv.NormalizeObservation()]])
def test_vector_episode_statistics_over_a_chain_sum_the_returned_rewards(stages):
    """gym_b200.wrappers.RecordEpisodeStatistics over an env with a chain sums the rewards step() returns, as the
    reference's vector RecordEpisodeStatistics over a SyncVectorEnv of wrapped envs does, whether or not the chain
    changes rewards."""
    import gym_b200
    from gym_b200 import wrappers
    n = 300
    env = wrappers.RecordEpisodeStatistics(gym_b200.vector.make("Pendulum-v1", n, wrappers=stages,
                                                                max_episode_steps=25))
    env.reset(seed=2)
    acc = np.zeros(n, np.float32)
    rng = np.random.default_rng(2)
    checked = 0
    for _ in range(80):
        _, r, te, tr, infos = env.step(rng.uniform(-2, 2, size=(n, 1)).astype(np.float32))
        acc = (acc + host(r)).astype(np.float32)   # `episode_returns += rewards`: float64 add, rounded to float32
        done = host(te) | host(tr)
        mask = host(infos["_episode"]).astype(bool)
        assert bits_equal(mask, done)
        assert bits_equal(host(infos["episode"]["r"])[done], acc[done])
        checked += int(done.sum())
        acc[done] = 0
    assert checked >= 2 * n
    env.close()
