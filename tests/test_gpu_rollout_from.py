"""``B200VectorEnv.rollout_from(snap, actions, rows=, states=)`` on the GPU, against its definition: a fresh twin env
of B envs restored from the gathered rows, rolled out with ``rollout(actions)``, its rewards and flags folded over the
first episode end, and its ``snapshot()`` for the end states.

Every comparison is bitwise.  Each case also checks that the env the call runs on is left exactly as it was, and that a
second call from the returned end states equals the twin continuing.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

CLASSIC = ["CartPole-v0", "CartPole-v1", "MountainCar-v0", "MountainCarContinuous-v0", "Pendulum-v1", "Acrobot-v1"]
BOX2D = [("LunarLander-v2", {}), ("LunarLanderContinuous-v2", dict(enable_wind=True, wind_idx=11, torque_idx=-7)),
         ("BipedalWalker-v3", {}), ("BipedalWalkerHardcore-v3", {})]
NS = [1, 31, 256, 257, 33 * 256 + 5, (1 << 16) + 3]
TS = [1, 2, 37, 300]
BOX2D_TS = [1, 3]


def _torch():
    import torch
    return torch


def _bits(t):
    torch = _torch()
    if t.dtype == torch.float32:
        return t.view(torch.int32)
    if t.dtype == torch.float64:
        return t.view(torch.int64)
    return t


def _eq(a, b, what):
    torch = _torch()
    assert a.dtype == b.dtype and a.shape == b.shape, (what, a.dtype, b.dtype, a.shape, b.shape)
    if not torch.equal(_bits(a), _bits(b)):
        bad = (_bits(a) != _bits(b)).nonzero()
        raise AssertionError(f"{what}: {len(bad)} entries differ, first at {bad[0].tolist()}")


def _make(env_id, n, seed, warm=0, **kw):
    """An env of n envs reset with `seed` and stepped `warm` times with seeded random actions."""
    import gym_b200
    env = gym_b200.vector.make(env_id, n, **kw)
    env.reset(seed=seed)
    for t in range(warm):
        env.step(_actions(env, 1, n, seed * 1000 + t)[0])
    return env


def _actions(env, T, B, seed):
    torch = _torch()
    g = torch.Generator(device=env.device).manual_seed(seed)
    if env.discrete:
        return torch.randint(0, int(env.single_action_space.n), (T, B), generator=g, device=env.device)
    lo = float(env.single_action_space.low[0])
    hi = float(env.single_action_space.high[0])
    return (lo + (hi - lo) * torch.rand((T, B, env.act_dim), generator=g, device=env.device)).float()


def _fold(rew, te, tr):
    """(returns, lengths, ended) of rollout_linear(summary=True), restated in torch float64 from full outputs."""
    torch = _torch()
    T, B = rew.shape
    done = te | tr
    ended = done.any(dim=0)
    first = done.to(torch.int32).argmax(dim=0)
    t_end = torch.where(ended, first, torch.full_like(first, T - 1))
    returns = torch.zeros(B, dtype=torch.float64, device=rew.device)
    for t in range(T):
        returns = torch.where(t <= t_end, returns + rew[t], returns)
    return returns, (t_end + 1).to(torch.int32), ended


def _twin(env_id, snap, rows, B, **kw):
    """A fresh env of B envs restored from the rows `rows` of `snap` (all of them in order if rows is None)."""
    import gym_b200
    from gym_b200.snapshot import EnvSnapshot
    twin = gym_b200.vector.make(env_id, B, **kw)
    if rows is not None:
        torch = _torch()
        r = torch.as_tensor(rows, device=snap.rows.device)
        snap = EnvSnapshot(snap.header, snap.rows[r], snap.obs[r])
    twin.restore(snap)
    return twin


def _state_of(env):
    """Everything of `env` that rollout_from must leave alone, as host copies."""
    torch = _torch()
    torch.cuda.synchronize()
    snap = env.snapshot()
    outs = [{k: v.clone() for k, v in o.items()} for o in env._out]
    return (snap.rows.clone(), snap.obs.clone(), [x.clone() for x in env.get_state()], outs, env._flip,
            env.action_space.np_random.bit_generator.state)


def _assert_untouched(env, before, what):
    after = _state_of(env)
    _eq(after[0], before[0], f"{what}: snapshot rows")
    _eq(after[1], before[1], f"{what}: snapshot observations")
    for x, y in zip(after[2], before[2]):
        _eq(x, y, f"{what}: get_state()")
    for o, p in zip(after[3], before[3]):
        for k in p:
            _eq(o[k], p[k], f"{what}: output buffer {k}")
    assert after[4] == before[4], f"{what}: _flip"
    assert after[5] == before[5], f"{what}: action-space generator"


def _check(env, snap, acts, rows, env_id, kw, what=""):
    """rollout_from with and without end states against the twin -> (the end snapshot, the twin)."""
    B = acts.shape[1]
    got = env.rollout_from(snap, acts, rows=rows, states=True)
    plain = env.rollout_from(snap, acts, rows=rows)
    assert len(plain) == 3
    twin = _twin(env_id, snap, rows, B, **kw)
    o, r, te, tr, _ = twin.rollout(acts)
    for name, x, y, z in zip(("returns", "lengths", "ended"), got, plain, _fold(r, te, tr)):
        _eq(x, z, f"{what}{name}")
        _eq(y, z, f"{what}{name} (states=False)")
    end = twin.snapshot()
    _eq(got[3].rows, end.rows, f"{what}end rows")
    _eq(got[3].obs, end.obs, f"{what}end observations")
    assert got[3].header == snap.header
    return got[3], twin


def _continue(env, end, twin, seed, env_id, kw):
    """A second rollout_from from the end states equals the twin continuing."""
    B = twin.num_envs
    acts = _actions(env, 5, B, seed)
    got = env.rollout_from(end, acts, states=True)
    o, r, te, tr, _ = twin.rollout(acts)
    for name, x, y in zip(("returns", "lengths", "ended"), got, _fold(r, te, tr)):
        _eq(x, y, f"continued {name}")
    again = twin.snapshot()
    _eq(got[3].rows, again.rows, "continued end rows")
    _eq(got[3].obs, again.obs, "continued end observations")


@pytest.mark.parametrize("T", TS)
@pytest.mark.parametrize("n", NS)
@pytest.mark.parametrize("env_id", CLASSIC)
def test_rollout_from_equals_restored_twin(env_id, n, T):
    env = _make(env_id, n, seed=100 + n, warm=3, max_episode_steps=40)
    kw = dict(max_episode_steps=40)
    snap = env.snapshot()
    before = _state_of(env)
    end, twin = _check(env, snap, _actions(env, T, n, T), None, env_id, kw)
    _assert_untouched(env, before, "rollout_from")
    _continue(env, end, twin, 7 * T + 1, env_id, kw)
    _assert_untouched(env, before, "second rollout_from")


@pytest.mark.parametrize("T", BOX2D_TS)
@pytest.mark.parametrize("n", NS)
@pytest.mark.parametrize("env_id,kwargs", BOX2D, ids=[b[0] for b in BOX2D])
def test_box2d_rollout_from_equals_restored_twin(env_id, kwargs, n, T):
    env = _make(env_id, n, seed=200 + n, warm=2, **kwargs)
    snap = env.snapshot()
    before = _state_of(env)
    end, twin = _check(env, snap, _actions(env, T, n, T), None, env_id, kwargs)
    _assert_untouched(env, before, "rollout_from")
    _continue(env, end, twin, 3 * T + 1, env_id, kwargs)
    # R roots x K branches through rows, on the same scratch batch
    R, K = min(n, 5), 3
    rows = _torch().arange(R, device=env.device).repeat_interleave(K)
    _check(env, snap, _actions(env, T, R * K, 11), rows, env_id, kwargs, "roots x branches: ")
    _assert_untouched(env, before, "box2d rollout_from")


@pytest.mark.parametrize("env_id", CLASSIC)
def test_roots_times_branches(env_id):
    """R roots x K branches, as a CUDA tensor and as a host list; short episodes so that autoresets happen."""
    torch = _torch()
    env = _make(env_id, 64, seed=5, warm=4, max_episode_steps=8)
    kw = dict(max_episode_steps=8)
    snap = env.snapshot(list(range(0, 64, 4)))   # 16 roots
    R, K, T = 16, 32, 20
    rows = torch.arange(R, device=env.device).repeat_interleave(K)
    acts = _actions(env, T, R * K, 3)
    end, _ = _check(env, snap, acts, rows, env_id, kw)
    host = env.rollout_from(snap, acts, rows=rows.tolist(), states=True)
    _eq(host[3].rows, end.rows, "host rows")
    # branches of one root that take the same actions draw the same resets
    same = acts.view(T, R, K, *acts.shape[2:])[:, :, :1].expand(T, R, K, *acts.shape[2:]).reshape(acts.shape)
    end2, _ = _check(env, snap, same.contiguous(), rows, env_id, kw, "same actions: ")
    r = end2.rows.view(R, K, -1)
    _eq(r, r[:, :1].expand_as(r).contiguous(), "branches of one root")


@pytest.mark.parametrize("env_id", CLASSIC)
def test_without_autoreset(env_id):
    """autoreset=False: roots stepped until some have ended (CartPole's flag byte set in their rows)."""
    kw = dict(autoreset=False, max_episode_steps=0)
    env = _make(env_id, 300, seed=9, warm=60, **kw)
    snap = env.snapshot()
    rows = _torch().randint(0, 300, (500,), device=env.device)
    _check(env, snap, _actions(env, 30, 500, 4), rows, env_id, kw)


def test_snapshot_of_another_handle():
    """A snapshot taken from a different handle, with another seed and history, and a long TimeLimit."""
    a = _make("Acrobot-v1", 1000, seed=1, warm=9)
    b = _make("Acrobot-v1", 77, seed=99, warm=2)
    snap = a.snapshot()
    before = _state_of(b)
    rows = _torch().randint(0, 1000, (4000,), device=b.device)
    end, twin = _check(b, snap, _actions(b, 50, 4000, 6), rows, "Acrobot-v1", {})
    _assert_untouched(b, before, "other handle")
    _continue(b, end, twin, 8, "Acrobot-v1", {})


def test_out_of_range_device_rows_skip_and_raise_next():
    from gym_b200 import error
    torch = _torch()
    env = _make("CartPole-v1", 100, seed=3, warm=2)
    snap = env.snapshot()
    rows = torch.randint(0, 100, (300,), device=env.device)
    bad = torch.tensor([0, 150, 299])
    rows[bad] = torch.tensor([-1, 100, 1 << 40], device=env.device)
    acts = _actions(env, 12, 300, 2)
    got = env.rollout_from(snap, acts, rows=rows, states=True)
    torch.cuda.synchronize()
    ok = torch.ones(300, dtype=torch.bool)
    ok[bad] = False
    ok = ok.to(env.device)
    assert (got[0][~ok] == 0).all() and (got[1][~ok] == 0).all() and not got[2][~ok].any()
    assert (got[3].rows[~ok] == 0).all() and (got[3].obs[~ok] == 0).all()
    twin = _twin("CartPole-v1", snap, torch.where(ok, rows, 0), 300)
    o, r, te, tr, _ = twin.rollout(acts)
    for name, x, y in zip(("returns", "lengths", "ended"), got, _fold(r, te, tr)):
        _eq(x[ok], y[ok], name)
    _eq(got[3].rows[ok], twin.snapshot().rows[ok], "end rows")
    with pytest.raises(error.Error, match="out-of-range"):
        env.rollout_from(snap, acts, rows=rows)
    env.rollout_from(snap, acts[:, :100])   # the flag is cleared by the raise
    with pytest.raises(error.Error, match="out of range"):
        env.rollout_from(snap, acts[:, :2], rows=[0, 100])


def test_invalid_actions_count_on_this_env():
    from gym_b200 import error
    env = _make("CartPole-v1", 50, seed=4, warm=1)
    snap = env.snapshot()
    acts = _actions(env, 6, 50, 1)
    acts[2, ::5] = 7
    acts[4, 1] = -3
    got = env.rollout_from(snap, acts)
    assert _torch().isnan(got[0][::5]).all()
    with pytest.raises(error.InvalidAction, match="^11 out-of-range"):
        env.check_actions()


@pytest.mark.parametrize("env_id", ["CartPole-v1", "MountainCar-v0", "MountainCarContinuous-v0", "Pendulum-v1",
                                    "Acrobot-v1"])
def test_captured_rollout_from_replays_equal_eager_calls(env_id):
    """Replays read the current snap.rows, rows and actions and rewrite the outputs allocated at capture."""
    torch = _torch()
    env = _make(env_id, 200, seed=6, warm=3)
    other = _make(env_id, 200, seed=60, warm=11)
    snap = env.snapshot()
    B, T = 700, 16
    rows = torch.randint(0, 200, (B,), device=env.device)
    acts = _actions(env, T, B, 0)
    env.rollout_from(snap, acts, rows=rows)   # outside the capture: allocates the index-error flag
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = env.rollout_from(snap, acts, rows=rows, states=True)
    for r in range(3):
        snap.rows.copy_((env if r % 2 else other).snapshot().rows)
        acts.copy_(_actions(env, T, B, 10 + r))
        rows.copy_(torch.randint(0, 200, (B,), device=env.device))
        g.replay()
        want = env.rollout_from(snap, acts, rows=rows, states=True)
        for name, x, y in zip(("returns", "lengths", "ended"), out[:3], want[:3]):
            _eq(x, y, f"replay {r} {name}")
        _eq(out[3].rows, want[3].rows, f"replay {r} end rows")
        _eq(out[3].obs, want[3].obs, f"replay {r} end observations")


@pytest.mark.parametrize("env_id,kwargs", BOX2D, ids=[b[0] for b in BOX2D])
def test_box2d_capture_is_refused(env_id, kwargs):
    from gym_b200 import error
    torch = _torch()
    env = _make(env_id, 33, seed=7, **kwargs)
    snap = env.snapshot()
    acts = _actions(env, 2, 33, 0)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with pytest.raises(error.Error, match="Box2D"):
        with torch.cuda.graph(g):
            env.rollout_from(snap, acts)
    del g
    end, _ = _check(env, snap, acts, None, env_id, kwargs, "after the refused capture: ")


def test_guards_and_refusals():
    import gym_b200
    from gym_b200 import error, subenv, wrappers
    from gym_b200.distributed import ShardedVectorEnv
    from gym_b200.env import B200Env
    from gym_b200.snapshot import EnvSnapshot
    torch = _torch()

    env = gym_b200.vector.make("CartPole-v1", 64)
    src = _make("CartPole-v1", 64, seed=1, warm=1)
    snap = src.snapshot()
    acts = _actions(src, 3, 64, 0)
    env.rollout_from(snap, acts)   # no reset() needed
    env.reset(seed=2)
    before = _state_of(env)
    dev = env.device
    bad_calls = [
        lambda: env.rollout_from(snap.rows, acts),                                          # not a snapshot
        lambda: env.rollout_from(_make("CartPole-v1", 4, seed=0, max_episode_steps=9).snapshot(), acts[:, :4]),
        lambda: env.rollout_from(_make("Acrobot-v1", 4, seed=0).snapshot(), acts[:, :4]),    # another kind
        lambda: env.rollout_from(EnvSnapshot(snap.header, snap.rows.cpu(), snap.obs), acts),
        lambda: env.rollout_from(EnvSnapshot(snap.header, snap.rows[:, :32].contiguous(), snap.obs), acts),
        lambda: env.rollout_from(EnvSnapshot(snap.header, snap.rows.view(torch.int32), snap.obs), acts),
        lambda: env.rollout_from(snap, acts[:, :63]),                                        # B mismatch
        lambda: env.rollout_from(snap, acts[0]),                                             # no T axis
        lambda: env.rollout_from(snap, acts[:0]),                                            # T = 0
        lambda: env.rollout_from(snap, acts.float()),                                        # float Discrete actions
        lambda: env.rollout_from(snap, acts[:, :0], rows=torch.zeros(0, dtype=torch.int64, device=dev)),   # B = 0
        lambda: env.rollout_from(snap, acts[:, :0], rows=[]),                                # B = 0, host rows
        lambda: env.rollout_from(EnvSnapshot(snap.header, snap.rows[:0], snap.obs[:0]), acts[:, :0]),
        lambda: env.rollout_from(snap, acts, rows=torch.zeros(64, device=dev)),              # float rows
        lambda: env.rollout_from(snap, acts, rows=torch.zeros((64, 1), dtype=torch.int64, device=dev)),
        lambda: env.rollout_from(snap, acts, rows=[64] * 64),                                # host rows out of range
    ]
    for k, call in enumerate(bad_calls):
        with pytest.raises(error.Error):
            call()
        _assert_untouched(env, before, f"refusal {k}")
    env.step_async(torch.zeros(64, dtype=torch.int64, device=dev))
    with pytest.raises(error.AlreadyPendingCallError):
        env.rollout_from(snap, acts)
    env.step_wait()
    before = _state_of(env)
    for wr in (wrappers.RecordEpisodeStatistics(env), wrappers.NormalizeObservation(env),
               wrappers.NormalizeReward(env), wrappers.VectorListInfo(env)):
        with pytest.raises(error.Error, match="rollout_from"):
            wr.rollout_from(snap, acts)
    _assert_untouched(env, before, "wrappers")
    env.close()
    with pytest.raises(error.ClosedEnvironmentError):
        env.rollout_from(snap, acts)

    host = gym_b200.vector.make("CartPole-v1", 64, backend="numpy")
    host.reset(seed=3)
    with pytest.raises(error.Error, match="backend"):
        host.rollout_from(snap, acts)
    host.close()
    chain = gym_b200.vector.make("CartPole-v1", 64, wrappers=[subenv.RecordEpisodeStatistics()])
    chain.reset(seed=4)
    with pytest.raises(error.Error, match="wrappers"):
        chain.rollout_from(chain.snapshot(), acts)
    chain.close()
    assert not hasattr(ShardedVectorEnv, "rollout_from")
    assert not hasattr(B200Env, "rollout_from")
