"""``B200VectorEnv.rollout_from_mlp(snap, params, hidden, T, noise=, rows=, states=, ...)`` on the GPU, against its
definition: a fresh twin env of B envs restored from the gathered rows, rolled out by ``rollout_mlp`` (no noise) or
``rollout_mlp_noisy`` with the same policy, noise and statistics, its rewards and flags folded over the first episode
end, its first actions, and its ``snapshot()`` for the end states.

Every comparison is bitwise.  Each case also checks that the env the call runs on is left exactly as it was.
"""
import ctypes
import math

import pytest

from test_gpu_rollout_from import _assert_untouched, _eq, _fold, _make, _state_of, _twin

pytestmark = pytest.mark.gpu

CLASSIC = ["CartPole-v0", "CartPole-v1", "MountainCar-v0", "MountainCarContinuous-v0", "Pendulum-v1", "Acrobot-v1"]
BOX2D = [("LunarLander-v2", {}), ("LunarLanderContinuous-v2", dict(enable_wind=True, wind_idx=11, torque_idx=-7)),
         ("BipedalWalker-v3", {})]
HIDDEN = [(64, 64), (6, 5), (8,)]
# (per-branch rows, noise, obs_norm): every combination but noise with per-branch rows and obs_norm, which is refused
POLICIES = [(pb, noisy, norm) for pb in (False, True) for noisy in (False, True) for norm in (False, True)
            if not (pb and noisy and norm)]


def _torch():
    import torch
    return torch


def _K(env):
    return int(env.single_action_space.n) if env.discrete else int(env.act_dim)


def _params(env, hidden, B, seed):
    """One policy (B None) or B per-branch rows, float32, seeded."""
    torch = _torch()
    sizes = [env.obs_dim] + list(hidden) + [_K(env)]
    P = sum(o * i + o for i, o in zip(sizes[:-1], sizes[1:]))
    g = torch.Generator(device=env.device).manual_seed(seed)
    shape = (P,) if B is None else (B, P)
    return (0.5 * torch.randn(shape, generator=g, device=env.device)).float()


def _noise(env, T, B, seed):
    torch = _torch()
    g = torch.Generator(device=env.device).manual_seed(seed)
    if env.discrete:
        u = torch.rand((T, B, _K(env)), generator=g, device=env.device).clamp_(min=torch.finfo(torch.float32).tiny)
        return -torch.log(-torch.log(u))
    return 0.3 * torch.randn((T, B, _K(env)), generator=g, device=env.device)


def _stats(env, seed):
    torch = _torch()
    g = torch.Generator(device=env.device).manual_seed(seed)
    mean = torch.randn(env.obs_dim, generator=g, device=env.device, dtype=torch.float64)
    var = 0.05 + 2.0 * torch.rand(env.obs_dim, generator=g, device=env.device, dtype=torch.float64)
    return mean, var


def _check(env, snap, rows, params, hidden, T, env_id, kw, noise=None, act="relu", norm=None, clip=None, what=""):
    """rollout_from_mlp with and without end states against the twin -> (the end snapshot, the twin)."""
    B = int(snap.rows.shape[0]) if rows is None else len(rows)
    pol = dict(activation=act, obs_norm=norm, clip_obs=clip)
    got = env.rollout_from_mlp(snap, params, hidden, T, noise=noise, rows=rows, states=True, **pol)
    plain = env.rollout_from_mlp(snap, params, hidden, T, noise=noise, rows=rows, **pol)
    assert len(plain) == 4
    twin = _twin(env_id, snap, rows, B, **kw)
    if noise is None:
        a, o, r, te, tr, _ = twin.rollout_mlp(params, hidden, T, **pol)
    else:
        a, z, o, r, te, tr, _ = twin.rollout_mlp_noisy(params, hidden, noise, **pol)
    for name, x, y, w in zip(("returns", "lengths", "ended", "first actions"), got, plain, _fold(r, te, tr) + (a[0],)):
        _eq(x, w, f"{what}{name}")
        _eq(y, w, f"{what}{name} (states=False)")
    end = twin.snapshot()
    _eq(got[4].rows, end.rows, f"{what}end rows")
    _eq(got[4].obs, end.obs, f"{what}end observations")
    assert got[4].header == snap.header
    return got[4], twin


@pytest.mark.parametrize("per_branch,noisy,norm", POLICIES)
@pytest.mark.parametrize("hidden", HIDDEN)
@pytest.mark.parametrize("act", ["relu", "tanh"])
@pytest.mark.parametrize("env_id", CLASSIC)
def test_classic_equals_restored_twin(env_id, act, hidden, per_branch, noisy, norm):
    """Random rows with duplicates, B = 777; then a second call from the end states equals the twin continuing."""
    torch = _torch()
    kw = dict(max_episode_steps=40)
    env = _make(env_id, 100, seed=11, warm=3, **kw)
    snap = env.snapshot()
    before = _state_of(env)
    B, T = 777, 37
    rows = torch.randint(0, 100, (B,), device=env.device, generator=torch.Generator(device=env.device).manual_seed(1))
    params = _params(env, hidden, B if per_branch else None, 2)
    stats = _stats(env, 3) if norm else None
    clip = 3.0 if norm else None
    noise = _noise(env, T, B, 4) if noisy else None
    end, twin = _check(env, snap, rows, params, hidden, T, env_id, kw, noise, act, stats, clip)
    _assert_untouched(env, before, "rollout_from_mlp")
    noise = _noise(env, 5, B, 5) if noisy else None
    _check(env, end, None, params, hidden, 5, env_id, kw, noise, act, stats, clip, "continued: ")
    _assert_untouched(env, before, "second rollout_from_mlp")


@pytest.mark.parametrize("env_id,kwargs", BOX2D, ids=[b[0] for b in BOX2D])
def test_box2d_equals_restored_twin(env_id, kwargs):
    """Shared and per-branch policies, noise, normalised inputs; R x K rows; a continuation."""
    torch = _torch()
    env = _make(env_id, 24, seed=21, warm=2, **kwargs)
    snap = env.snapshot()
    before = _state_of(env)
    R, K, T = 6, 4, 3
    rows = torch.arange(R, device=env.device).repeat_interleave(K)
    hid = (16, 16)
    end, twin = _check(env, snap, rows, _params(env, hid, None, 1), hid, T, env_id, kwargs, what="shared: ")
    _check(env, snap, rows, _params(env, hid, R * K, 2), hid, T, env_id, kwargs, act="tanh", what="per-branch: ")
    _check(env, snap, rows, _params(env, hid, None, 3), hid, T, env_id, kwargs, _noise(env, T, R * K, 4), "tanh",
           _stats(env, 5), 2.0, "noisy normalised: ")
    _check(env, snap, None, _params(env, (6,), 24, 6), (6,), 2, env_id, kwargs, _noise(env, 2, 24, 7),
           what="per-branch noisy: ")
    _assert_untouched(env, before, "box2d rollout_from_mlp")
    _check(env, end, None, _params(env, hid, None, 1), hid, 2, env_id, kwargs, what="continued: ")
    _assert_untouched(env, before, "box2d second call")


def test_snapshot_of_another_handle_and_roots_times_branches():
    """A snapshot of a different handle; R roots x K Gumbel samples of a tanh actor, rows as a CUDA tensor and as a
    host list."""
    torch = _torch()
    a = _make("CartPole-v1", 1000, seed=1, warm=9)
    b = _make("CartPole-v1", 77, seed=99, warm=2)
    snap = a.snapshot(list(range(0, 1000, 10)))   # 100 roots
    before = _state_of(b)
    R, K, T = 100, 64, 32
    rows = torch.arange(R, device=b.device).repeat_interleave(K)
    params = _params(b, (64, 64), None, 8)
    noise = _noise(b, T, R * K, 9)
    end, _ = _check(b, snap, rows, params, (64, 64), T, "CartPole-v1", {}, noise, "tanh")
    host = b.rollout_from_mlp(snap, params, (64, 64), T, noise=noise, rows=rows.tolist(), states=True,
                              activation="tanh")
    _eq(host[4].rows, end.rows, "host rows")
    _assert_untouched(b, before, "other handle")


def test_out_of_range_device_rows_skip_and_raise_next():
    from gym_b200 import error
    torch = _torch()
    for env_id in ("CartPole-v1", "Pendulum-v1", "LunarLanderContinuous-v2"):
        env = _make(env_id, 40, seed=3, warm=2)
        snap = env.snapshot()
        B, T = 60, 6
        rows = torch.randint(0, 40, (B,), device=env.device)
        bad = torch.tensor([0, 31, 59])
        rows[bad] = torch.tensor([-1, 40, 1 << 40], device=env.device)
        params = _params(env, (8, 8), None, 1)
        noise = _noise(env, T, B, 2)
        got = env.rollout_from_mlp(snap, params, (8, 8), T, noise=noise, rows=rows, states=True)
        torch.cuda.synchronize()
        ok = torch.ones(B, dtype=torch.bool)
        ok[bad] = False
        ok = ok.to(env.device)
        assert (got[0][~ok] == 0).all() and (got[1][~ok] == 0).all() and not got[2][~ok].any()
        assert (got[3][~ok] == 0).all()
        assert (got[4].rows[~ok] == 0).all() and (got[4].obs[~ok] == 0).all()
        twin = _twin(env_id, snap, torch.where(ok, rows, 0), B)
        a, z, o, r, te, tr, _ = twin.rollout_mlp_noisy(params, (8, 8), noise)
        for name, x, y in zip(("returns", "lengths", "ended", "first actions"), got, _fold(r, te, tr) + (a[0],)):
            _eq(x[ok], y[ok], name)
        _eq(got[4].rows[ok], twin.snapshot().rows[ok], "end rows")
        with pytest.raises(error.Error, match="out-of-range"):
            env.rollout_from_mlp(snap, params, (8, 8), T, rows=rows)
        env.rollout_from_mlp(snap, params, (8, 8), T)   # the flag is cleared by the raise
        with pytest.raises(error.Error, match="out of range"):
            env.rollout_from_mlp(snap, params, (8, 8), T, rows=[0, 40])
        env.close()


@pytest.mark.parametrize("env_id", ["CartPole-v1", "MountainCar-v0", "MountainCarContinuous-v0", "Pendulum-v1",
                                    "Acrobot-v1"])
def test_captured_replays_read_current_inputs(env_id):
    """Replays read the current snap.rows, rows, params, noise, mean and var, and rewrite the outputs allocated at
    capture, for a shared noisy normalised policy and per-branch deterministic ones."""
    torch = _torch()
    env = _make(env_id, 200, seed=6, warm=3)
    other = _make(env_id, 200, seed=60, warm=11)
    snap = env.snapshot()
    B, T = 700, 16
    rows = torch.randint(0, 200, (B,), device=env.device)
    for per_branch in (False, True):
        params = _params(env, (32, 32), B if per_branch else None, 0)
        noise = None if per_branch else _noise(env, T, B, 1)
        mean, var = _stats(env, 2)
        kw = dict(noise=noise, rows=rows, states=True, activation="tanh", obs_norm=(mean, var), clip_obs=5.0)
        env.rollout_from_mlp(snap, params, (32, 32), T, **kw)   # outside the capture: allocates the index-error flag
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            out = env.rollout_from_mlp(snap, params, (32, 32), T, **kw)
        for r in range(3):
            snap.rows.copy_((env if r % 2 else other).snapshot().rows)
            rows.copy_(torch.randint(0, 200, (B,), device=env.device))
            params.copy_(_params(env, (32, 32), B if per_branch else None, 10 + r))
            if noise is not None:
                noise.copy_(_noise(env, T, B, 20 + r))
            m2, v2 = _stats(env, 30 + r)
            mean.copy_(m2)
            var.copy_(v2)
            g.replay()
            want = env.rollout_from_mlp(snap, params, (32, 32), T, **kw)
            for name, x, y in zip(("returns", "lengths", "ended", "first actions"), out[:4], want[:4]):
                _eq(x, y, f"replay {r} {name}")
            _eq(out[4].rows, want[4].rows, f"replay {r} end rows")
            _eq(out[4].obs, want[4].obs, f"replay {r} end observations")


@pytest.mark.parametrize("env_id,kwargs", BOX2D, ids=[b[0] for b in BOX2D])
def test_box2d_capture_is_refused(env_id, kwargs):
    from gym_b200 import error
    torch = _torch()
    env = _make(env_id, 9, seed=7, **kwargs)
    snap = env.snapshot()
    params = _params(env, (8,), None, 0)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with pytest.raises(error.Error, match="Box2D"):
        with torch.cuda.graph(g):
            env.rollout_from_mlp(snap, params, (8,), 2)
    del g
    _check(env, snap, None, params, (8,), 2, env_id, kwargs, what="after the refused capture: ")


def test_refusals_come_before_any_cuda_call(monkeypatch):
    """Every refusal, with the C entry point replaced by a stub that raises: none of them reaches it."""
    import gym_b200
    from gym_b200 import _lib, error, subenv, wrappers
    from gym_b200.distributed import ShardedVectorEnv
    from gym_b200.env import B200Env
    from gym_b200.snapshot import EnvSnapshot
    torch = _torch()

    def stub(*args):
        raise AssertionError("b200gym_rollout_from_mlp was called")
    monkeypatch.setattr(_lib.load(), "b200gym_rollout_from_mlp", stub)
    env = gym_b200.vector.make("CartPole-v1", 64)
    src = _make("CartPole-v1", 64, seed=1, warm=1)
    snap = src.snapshot()
    dev = env.device
    p = _params(env, (8,), None, 0)
    pb = _params(env, (8,), 64, 0)
    e = _noise(env, 3, 64, 0)
    m, v = _stats(env, 0)
    env.reset(seed=2)
    before = _state_of(env)
    bad_calls = [
        (error.Error, lambda: env.rollout_from_mlp(snap.rows, p, (8,), 3)),                        # not a snapshot
        (error.Error, lambda: env.rollout_from_mlp(_make("Acrobot-v1", 4, seed=0).snapshot(), p, (8,), 3)),
        (error.Error, lambda: env.rollout_from_mlp(EnvSnapshot(snap.header, snap.rows.cpu(), snap.obs), p, (8,), 3)),
        (error.Error, lambda: env.rollout_from_mlp(snap, p, (8,), 3, rows=[])),                    # B = 0
        (error.Error, lambda: env.rollout_from_mlp(snap, p, (8,), 3, rows=[64])),                  # host row range
        (error.Error, lambda: env.rollout_from_mlp(snap, p, (8,), 3, rows=torch.zeros(4, device=dev))),
        (ValueError, lambda: env.rollout_from_mlp(snap, p, (8,), 0)),                              # T = 0
        (ValueError, lambda: env.rollout_from_mlp(snap, p, (8,), 2 ** 31)),
        (ValueError, lambda: env.rollout_from_mlp(snap, p, (8,), 3.0)),
        (ValueError, lambda: env.rollout_from_mlp(snap, p, (65,), 3)),                             # width
        (ValueError, lambda: env.rollout_from_mlp(snap, p, (8, 8, 8), 3)),
        (ValueError, lambda: env.rollout_from_mlp(snap, p, (8,), 3, activation="gelu")),
        (ValueError, lambda: env.rollout_from_mlp(snap, p.double(), (8,), 3)),
        (ValueError, lambda: env.rollout_from_mlp(snap, p.cpu(), (8,), 3)),
        (ValueError, lambda: env.rollout_from_mlp(snap, p[:-1], (8,), 3)),
        (ValueError, lambda: env.rollout_from_mlp(snap, pb[:63], (8,), 3)),                       # rows != B
        (ValueError, lambda: env.rollout_from_mlp(snap, pb, (8,), 3, rows=list(range(32)))),
        (ValueError, lambda: env.rollout_from_mlp(snap, p, (8,), 4, noise=e)),                     # T mismatch
        (ValueError, lambda: env.rollout_from_mlp(snap, p, (8,), 3, noise=e[:, :63].contiguous())),   # B mismatch
        (ValueError, lambda: env.rollout_from_mlp(snap, p, (8,), 3, noise=e.double())),
        (ValueError, lambda: env.rollout_from_mlp(snap, p, (8,), 3, noise=e.transpose(0, 1))),
        (ValueError, lambda: env.rollout_from_mlp(snap, p, (8,), 3, clip_obs=5.0)),                # clip, no stats
        (ValueError, lambda: env.rollout_from_mlp(snap, p, (8,), 3, obs_norm=(m.float(), v))),
        (ValueError, lambda: env.rollout_from_mlp(snap, p, (8,), 3, obs_norm=(m, v[:3].contiguous()))),
        (ValueError, lambda: env.rollout_from_mlp(snap, p, (8,), 3, obs_norm=(m, v), norm_epsilon=-1.0)),
        (ValueError, lambda: env.rollout_from_mlp(snap, p, (8,), 3, obs_norm=(m, v), clip_obs=0.0)),
        (ValueError, lambda: env.rollout_from_mlp(snap, p, (8,), 3, obs_norm=(m,))),
        (ValueError, lambda: env.rollout_from_mlp(snap, pb, (8,), 3, noise=e, obs_norm=(m, v))),   # noisy rows + norm
    ]
    for k, (exc, call) in enumerate(bad_calls):
        with pytest.raises(exc):
            call()
        _assert_untouched(env, before, f"refusal {k}")
    with pytest.raises(ValueError, match="with obs_norm needs one policy shared by every env, not per-env rows"):
        env.rollout_from_mlp(snap, pb, (8,), 3, noise=e, obs_norm=(m, v))
    env.step_async(torch.zeros(64, dtype=torch.int64, device=dev))
    with pytest.raises(error.AlreadyPendingCallError):
        env.rollout_from_mlp(snap, p, (8,), 3)
    env.step_wait()
    for wr in (wrappers.RecordEpisodeStatistics(env), wrappers.NormalizeObservation(env)):
        with pytest.raises(error.Error, match="rollout_from_mlp"):
            wr.rollout_from_mlp(snap, p, (8,), 3)
    env.close()
    with pytest.raises(error.ClosedEnvironmentError):
        env.rollout_from_mlp(snap, p, (8,), 3)
    host = gym_b200.vector.make("CartPole-v1", 64, backend="numpy")
    host.reset(seed=3)
    with pytest.raises(error.Error, match="backend"):
        host.rollout_from_mlp(snap, p, (8,), 3)
    host.close()
    chain = gym_b200.vector.make("CartPole-v1", 64, wrappers=[subenv.RecordEpisodeStatistics()])
    chain.reset(seed=4)
    with pytest.raises(error.Error, match="wrappers"):
        chain.rollout_from_mlp(chain.snapshot(), p, (8,), 3)
    chain.close()
    lunar = _make("LunarLander-v2", 8, seed=5)
    ls = lunar.snapshot()
    with pytest.raises(error.Error, match="observations"):
        lunar.rollout_from_mlp(EnvSnapshot(ls.header, ls.rows, ls.obs[:4]), _params(lunar, (8,), None, 0), (8,), 2)
    lunar.close()
    assert not hasattr(ShardedVectorEnv, "rollout_from_mlp")
    assert not hasattr(B200Env, "rollout_from_mlp")


def test_c_entry_point_validates_its_arguments():
    """The C entry point re-checks B, T, the layer count, widths, activation, statistics and noise, the buffers and
    the end-state pair, and launches nothing when they are wrong."""
    torch = _torch()
    env = _make("CartPole-v1", 8, seed=2)
    snap = env.snapshot()
    before = _state_of(env)
    buf = torch.zeros(4096, device=env.device)
    st = torch.ones(64, dtype=torch.float64, device=env.device)
    vp = ctypes.c_void_p
    ok, s = vp(buf.data_ptr()), vp(st.data_ptr())
    good = dict(rows=vp(snap.rows.data_ptr()), n_rows=8, idx=None, B=8, per_branch=0, layers=1, h1=4, h2=0, T=3,
                noise=None, act=0, mean=None, var=None, eps=1e-8, clip=math.inf, first=ok, end_rows=None, end_obs=None)
    bad = [dict(B=0), dict(T=0), dict(n_rows=4), dict(layers=3), dict(h1=0), dict(h1=65), dict(layers=2, h2=0),
           dict(act=2), dict(mean=s), dict(var=s), dict(eps=-1.0), dict(clip=0.0), dict(clip=10.0),
           dict(mean=s, var=s, noise=ok, per_branch=1), dict(first=None), dict(end_rows=ok),
           dict(rows=None), dict(rows=vp(snap.rows.data_ptr() + 4))]
    for change in bad:
        c = {**good, **change}
        rc = env._lib.b200gym_rollout_from_mlp(env._handle, c["rows"], None, c["n_rows"], c["idx"], c["B"], ok,
                                               c["per_branch"], c["layers"], c["h1"], c["h2"], c["T"], c["noise"],
                                               c["act"], c["mean"], c["var"], c["eps"], c["clip"], ok, ok, ok,
                                               c["first"], c["end_rows"], c["end_obs"], env._stream())
        assert rc != 0, change
        assert b"b200gym_rollout_from_mlp" in env._lib.b200gym_last_error(env._handle), change
    lunar = _make("LunarLander-v2", 4, seed=1)
    ls = lunar.snapshot()
    rc = lunar._lib.b200gym_rollout_from_mlp(lunar._handle, vp(ls.rows.data_ptr()), None, 4, None, 4, ok, 0, 1, 4, 0,
                                             2, None, 0, None, None, 1e-8, math.inf, ok, ok, ok, ok, None, None,
                                             lunar._stream())
    assert rc != 0 and b"snap_obs_dev" in lunar._lib.b200gym_last_error(lunar._handle)
    torch.cuda.synchronize()
    _assert_untouched(env, before, "C-side refusals")
