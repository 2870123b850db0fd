"""Env snapshots on the device (B200VectorEnv.snapshot / restore / clone, pickle, deepcopy), every kind.

Batches are ragged (4096 + 77 envs) so the last tile of the snapshot kernels is partial; rollouts are long enough
(K = 300 random steps) that episodes end and autoreset from the env's own PCG64 stream inside them."""
import copy
import pickle

import numpy as np
import pytest

from gym_b200 import error
from gym_b200.wrappers import NormalizeReward, RecordEpisodeStatistics

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

N = 4096 + 77
K = 300
# (id, constructor kwargs); CartPole without autoreset is plain-Env semantics, whose "already terminated" flag must
# travel with the rows
CASES = [
    ("CartPole-v1", {}),
    ("CartPole-v1", {"autoreset": False}),
    ("MountainCar-v0", {}),
    ("MountainCarContinuous-v0", {}),
    ("Pendulum-v1", {}),
    ("Acrobot-v1", {}),
    ("LunarLander-v2", {"enable_wind": True}),
    ("LunarLanderContinuous-v2", {}),
    ("BipedalWalker-v3", {}),
    ("BipedalWalkerHardcore-v3", {}),
]
IDS = [i + ("-plain" if not k.get("autoreset", True) else "") + ("-wind" if k.get("enable_wind") else "")
       for i, k in CASES]


def _make(env_id, kw, seed, n=N, backend="torch"):
    """Reset with `seed`; with wind, the per-env wind counters are drawn from `seed` too, so that two envs made with
    the same seed are twins."""
    from gym_b200.vector_env import B200VectorEnv
    if kw.get("enable_wind"):
        wind, torque = np.random.default_rng(seed).integers(-9999, 9999, (2, n))
        kw = dict(kw, wind_idx=wind, torque_idx=torque)
    env = B200VectorEnv(env_id, n, backend=backend, copy=True, **kw)
    env.reset(seed=seed)
    return env


def _actions(env, k, seed):
    g = torch.Generator(device=env.device)
    g.manual_seed(seed)
    out = []
    for _ in range(k):
        if env.discrete:
            out.append(torch.randint(0, env.single_action_space.n, (env.num_envs,), generator=g, device=env.device))
        else:
            out.append(torch.rand((env.num_envs, env.act_dim), generator=g, device=env.device) * 2 - 1)
    return out


def _run(env, actions):
    """Every output of every step, on the host; final_obs only where an episode ended."""
    rec = []
    for a in actions:
        o, r, te, tr, info = env.step(a)
        done = (te | tr).cpu().numpy()
        fo = info["final_observation"].cpu().numpy()
        fo[~done if env.autoreset else slice(None)] = 0   # written only by an autoreset
        rec.append((o.cpu().numpy(), r.cpu().numpy(), te.cpu().numpy(), tr.cpu().numpy(), fo))
    return rec


def _engine_state(env):
    """Everything the engine exposes about its envs (get_state + Box2D bodies / terrain) as host arrays."""
    st, el, rng = env.get_state()
    out = [st.cpu().numpy(), el.cpu().numpy(), rng.cpu().numpy()]
    if env.kind in (5, 7):
        out += [t.cpu().numpy() for t in env.lunar_bodies()]
    if env.kind in (6, 8):
        out += [t.cpu().numpy() for t in env.walker_bodies()] + [t.cpu().numpy() for t in env.walker_terrain()]
    return out


def _assert_same(a, b, rows_a=None, rows_b=None):
    for x, y in zip(a, b):
        x = x if rows_a is None else x[rows_a]
        y = y if rows_b is None else y[rows_b]
        assert x.shape == y.shape and x.tobytes() == y.tobytes()


def _map(actions, src):
    return [a[src] for a in actions]


@pytest.mark.parametrize("env_id, kw", CASES, ids=IDS)
def test_rewind(env_id, kw):
    env = _make(env_id, kw, seed=11)
    _run(env, _actions(env, 20, 1))
    snap = env.snapshot()
    before = _engine_state(env)
    acts = _actions(env, K, 2)
    first = _run(env, acts)
    obs, info = env.restore(snap)
    assert info == {} and torch.equal(obs, snap.obs)
    _assert_same(_engine_state(env), before)
    second = _run(env, acts)
    for t, (x, y) in enumerate(zip(first, second)):
        _assert_same(x, y)
    ended = sum(int((r[2] | r[3]).sum()) for r in first)
    assert ended > 0 or env_id.startswith("MountainCar")
    env.close()


@pytest.mark.parametrize("env_id, kw", CASES, ids=IDS)
def test_cross_handle(env_id, kw):
    """A snapshot of handle A loaded into handle B (other seed, other history): B continues exactly like A -- any
    per-env word the row forgot would show here."""
    a = _make(env_id, kw, seed=3)
    b = _make(env_id, kw, seed=4)
    _run(a, _actions(a, 25, 5))
    _run(b, _actions(b, 40, 6))
    b.restore(a.snapshot())
    _assert_same(_engine_state(b), _engine_state(a))
    acts = _actions(a, K, 7)
    for x, y in zip(_run(a, acts), _run(b, acts)):
        _assert_same(x, y)
    a.close()
    b.close()


@pytest.mark.parametrize("env_id, kw", CASES, ids=IDS)
def test_clone(env_id, kw):
    env = _make(env_id, kw, seed=21)
    twin = _make(env_id, kw, seed=21)
    hist = _actions(env, 30, 8)
    _run(env, hist)
    _run(twin, hist)
    g = torch.Generator(device=env.device)
    g.manual_seed(9)
    sources = [torch.randint(0, N, (N,), generator=g, device=env.device),       # with duplicates
               torch.arange(N, device=env.device), torch.arange(N - 1, -1, -1, device=env.device)]
    for n_src, src in enumerate(sources):
        obs = env.clone(src)
        srch = src.cpu().numpy()
        assert torch.equal(obs, twin.snapshot().obs[src])
        _assert_same(_engine_state(env), _engine_state(twin), rows_b=srch)
        acts = _actions(env, K if n_src == 0 else 40, 10 + n_src)
        ours, theirs = _run(env, _map(acts, src)), _run(twin, acts)
        for x, y in zip(ours, theirs):
            _assert_same(x, y, rows_b=srch)
        _assert_same(_engine_state(env), _engine_state(twin), rows_b=srch)
        twin.restore(env.snapshot())   # start the next variant from the same state
    env.close()
    twin.close()


@pytest.mark.parametrize("env_id, kw", [CASES[0], CASES[6], CASES[9]], ids=[IDS[0], IDS[6], IDS[9]])
def test_partial_restore_and_bad_indices(env_id, kw):
    env = _make(env_id, kw, seed=31)
    twin = _make(env_id, kw, seed=31)
    sub = np.arange(5, N, 7)
    snap = env.snapshot(sub)
    assert len(snap) == sub.size
    acts = _actions(env, 15, 12)
    _run(env, acts)
    _run(twin, acts)
    obs, _ = env.restore(snap, indices=sub)
    others = np.setdiff1d(np.arange(N), sub)
    _assert_same(_engine_state(env), _engine_state(twin), rows_a=others, rows_b=others)
    assert torch.equal(obs[torch.from_numpy(sub).to(env.device)], snap.obs)
    # the restored envs are where they were when the snapshot was taken: their rows reproduce it
    again = env.snapshot(sub)
    assert torch.equal(again.rows, snap.rows)
    # host indices out of range: refused before anything runs
    twin.restore(env.snapshot())
    with pytest.raises(error.Error, match="out of range"):
        env.clone([0] * (N - 1) + [N])
    with pytest.raises(error.Error, match="out of range"):
        env.restore(snap, indices=np.r_[sub[:-1], -1])
    _assert_same(_engine_state(env), _engine_state(twin))
    # device indices out of range: that entry moves nothing, the error comes with the next call
    src = torch.arange(N - 1, -1, -1, device=env.device)
    src[17] = N + 5
    env.clone(src)
    torch.cuda.synchronize()
    with pytest.raises(error.Error, match="out-of-range"):
        env.step(_actions(env, 1, 13)[0])
    srch = src.cpu().numpy()
    ok = np.arange(N) != 17
    _assert_same(_engine_state(env), _engine_state(twin), rows_a=np.flatnonzero(ok), rows_b=srch[ok])
    _assert_same(_engine_state(env), _engine_state(twin), rows_a=[17], rows_b=[17])
    env.close()
    twin.close()


def test_mismatched_config_raises():
    a = _make("CartPole-v1", {}, seed=1, n=256)
    b = _make("CartPole-v1", {}, seed=1, n=256)
    c = _make("MountainCar-v0", {}, seed=1, n=256)
    from gym_b200.vector_env import B200VectorEnv
    d = B200VectorEnv("CartPole-v1", 256, max_episode_steps=50)
    snap = a.snapshot()
    b.restore(snap)
    with pytest.raises(error.Error, match="kind"):
        c.restore(snap)
    with pytest.raises(error.Error, match="config"):
        d.restore(snap)
    for e in (a, b, c, d):
        e.close()


# ---- pickle / deepcopy -----------------------------------------------------------------------------------------
def _continue_vec(env, acts):
    out = []
    for a in acts:
        o, r, te, tr, _ = env.step(a)
        out.append(tuple(x.cpu().numpy() if hasattr(x, "cpu") else np.array(x) for x in (o, r, te, tr)))
    return out


@pytest.mark.parametrize("backend", ["torch", "numpy"])
@pytest.mark.parametrize("env_id, kw", [CASES[0], CASES[1], CASES[4], CASES[6], CASES[9]],
                         ids=[IDS[0], IDS[1], IDS[4], IDS[6], IDS[9]])
def test_vector_pickle_and_deepcopy_continue_identically(env_id, kw, backend):
    env = _make(env_id, kw, seed=41, n=300, backend=backend)
    _continue_vec(env, [a.cpu().numpy() for a in _actions(env, 30, 14)])
    acts = [a.cpu().numpy() for a in _actions(env, 120, 15)]
    copies = [pickle.loads(pickle.dumps(env)), copy.deepcopy(env)]
    ref = _continue_vec(env, acts)
    for c in copies:
        assert type(c) is type(env) and c.device == env.device and c.backend == backend
        for x, y in zip(ref, _continue_vec(c, acts)):
            _assert_same(x, y)
        c.close()
    env.close()


@pytest.mark.parametrize("env_id, kw", [CASES[0], CASES[5], CASES[6], CASES[8]], ids=[IDS[0], IDS[5], IDS[6], IDS[8]])
def test_single_env_pickle_and_deepcopy(env_id, kw):
    from gym_b200.env import B200Env
    kw = {k: v for k, v in kw.items() if k != "autoreset"}
    env = B200Env(env_id, **kw)
    env.reset(seed=5)
    env.action_space.seed(3)
    for _ in range(25):
        env.step(env.action_space.sample())
    acts = [env.action_space.sample() for _ in range(200)]
    copies = [pickle.loads(pickle.dumps(env)), copy.deepcopy(env)]

    def go(e):
        out = []
        for a in acts:
            o, r, te, tr, _ = e.step(a)
            out.append((np.asarray(o), np.float64(r), te, tr))
            if te or tr:
                out.append(np.asarray(e.reset()[0]))   # later unseeded resets come from the copied stream
        return out

    ref = go(env)
    for c in copies:
        got = go(c)
        assert len(got) == len(ref)
        for x, y in zip(ref, got):
            assert pickle.dumps(x) == pickle.dumps(y)
        c.close()
    env.close()


def test_classic_pickle_matches_the_reference_rollouts():
    """A pickled / deep-copied engine continues the reference's frozen SyncVectorEnv rollouts
    (tests/golden/reference/) under the rules of test_gpu_reference_live.py."""
    from test_oracle_vs_reference import CLASSIC, reference_rollout

    import gym_b200
    for env_id in CLASSIC:
        g = reference_rollout(env_id)
        N_, T, seed, acts = g["N"], g["T"], g["seed"], g["actions"]
        eng = gym_b200.vector.make(env_id, N_, backend="numpy")
        eng.reset(seed=seed)
        half = T // 2
        for t in range(half):
            eng.step(acts[t])
        for c in (pickle.loads(pickle.dumps(eng)), copy.deepcopy(eng)):
            for t in range(half, T):
                o, r, te, tr, _ = c.step(acts[t])
                assert np.array_equal(te, g["terminated"][t]) and np.array_equal(tr, g["truncated"][t]), (env_id, t)
                np.testing.assert_allclose(r, g["reward"][t], rtol=1e-9, atol=1e-9)
                np.testing.assert_allclose(o, g["obs"][t], rtol=1e-5, atol=1e-6, err_msg=f"{env_id} step {t}")
            c.close()
        eng.close()


def test_reference_pickle_pattern_on_gym_make():
    """The reference's test_pickle_env (tests/envs/test_envs.py:192-200) on gym.make("B200/<id>")."""
    from oracle import ref_gym
    if ref_gym.reference_path() is None:
        pytest.skip("the reference is not installed in oracle/_ref")
    gym = ref_gym.import_reference()
    import gym_b200.plugin  # noqa: F401  (registers the B200/ ids)
    for env_id in ("CartPole-v1", "Pendulum-v1", "LunarLander-v2"):
        env = gym.make(f"B200/{env_id}", disable_env_checker=True)
        env.reset(seed=0)
        pickled = pickle.loads(pickle.dumps(env))
        a, b = env.reset(), pickled.reset()
        assert np.array_equal(a[0], b[0])
        action = env.action_space.sample()
        x, y = env.step(action), pickled.step(action)
        assert all(np.array_equal(u, v) for u, v in zip(x[:4], y[:4]))
        env.close()
        pickled.close()


# ---- wrappers --------------------------------------------------------------------------------------------------
def test_wrappers_follow_clone_and_restore():
    def wrapped(seed):
        return RecordEpisodeStatistics(NormalizeReward(_make("CartPole-v1", {}, seed=seed)))

    w, twin = wrapped(51), wrapped(51)
    hist = _actions(w.unwrapped, 60, 16)
    for a in hist:
        w.step(a)
        twin.step(a)
    src = torch.randint(0, N, (N,), device=w.unwrapped.device)
    before = [t.clone() for t in (w.episode_returns, w.episode_lengths, w.env.returns, w.env.return_rms.stats)]
    w.clone(src)
    assert torch.equal(w.episode_returns, before[0][src])
    assert torch.equal(w.episode_lengths, before[1][src])
    assert torch.equal(w.env.returns, before[2][src])
    assert torch.equal(w.env.return_rms.stats, before[3])   # statistics left alone
    acts = _actions(w.unwrapped, 40, 17)
    for a in acts:
        w.step(a[src])
        twin.step(a)
    assert torch.equal(w.episode_lengths, twin.episode_lengths[src])
    # rewind of the whole stack: running statistics, ring and counter restored whole; the replay is bit for bit
    snap = w.snapshot()
    first = [tuple(x.clone() for x in w.step(a)[:4]) for a in acts]
    state1 = (w.episode_returns.clone(), w.env.returns.clone(), w.env.return_rms.stats.clone(), w.episode_count)
    w.restore(snap)
    second = [tuple(x.clone() for x in w.step(a)[:4]) for a in acts]
    for x, y in zip(first, second):
        assert all(torch.equal(u, v) for u, v in zip(x, y))
    assert torch.equal(state1[0], w.episode_returns) and torch.equal(state1[1], w.env.returns)
    assert torch.equal(state1[2], w.env.return_rms.stats) and state1[3] == w.episode_count
    w.close()
    twin.close()


def test_sharded_env_refuses_snapshots():
    from gym_b200.distributed import ShardedVectorEnv
    env = ShardedVectorEnv("CartPole-v1", 256, gather=None)
    for call in (lambda: env.snapshot(), lambda: env.restore(None), lambda: env.clone(None)):
        with pytest.raises(error.Error, match="ShardedVectorEnv"):
            call()
    env.close()
