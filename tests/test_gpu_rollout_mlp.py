"""``B200VectorEnv.rollout_mlp(params, hidden, T)`` on the GPU: bit for bit what ``a = mlp(obs); obs, ... = step(a)``
T times returns, with the MLP restated in torch elementwise ops in the documented order (each unit its bias plus one
rounded product at a time, left to right; ReLU ``z if z > 0 or z is NaN else +0.0``).

Every comparison is against an eager twin, as in test_gpu_rollout_linear.py: the actions, the outputs, the final
observations on the rows the mask selects, ``get_state()``, ``snapshot()`` rows and observations, and the step after.
"""
import pytest

from test_gpu_rollout_linear import (BOX2D, CLASSIC, NAMES, Twin, _assert_equals_loop, _assert_same_env,
                                     _assert_untouched, _eq, _untouched, summary_of)

pytestmark = pytest.mark.gpu

HIDDEN = [(1,), (5,), (64,), (3, 7), (64, 64)]


def _torch():
    import torch
    return torch


def _sizes(env, hidden):
    K = env.single_action_space.n if env.discrete else env.act_dim
    return [env.obs_dim] + list(hidden) + [int(K)]


class MlpTwin(Twin):
    """Twin with ``policy(params, hidden)``: the torch restatement of the MLP."""

    def outputs(self, params, hidden):
        torch = _torch()
        n = self.env.num_envs
        P = params.shape[-1]
        W = params.expand(n, P)
        x, off = self.obs, 0
        sizes = _sizes(self.env, hidden)
        for layer, (fan_in, fan_out) in enumerate(zip(sizes[:-1], sizes[1:])):
            w = W[:, off:off + fan_out * fan_in].reshape(n, fan_out, fan_in)
            off += fan_out * fan_in
            z = W[:, off:off + fan_out].clone()
            off += fan_out
            for k in range(fan_in):
                z = z + w[:, :, k] * x[:, None, k]
            if layer < len(hidden):
                z = torch.where((z > 0) | torch.isnan(z), z, torch.zeros_like(z))
            x = z
        assert off == P
        return x

    def policy(self, params, hidden):
        torch = _torch()
        z = self.outputs(params, hidden)
        if not self.env.discrete:
            return z
        n = z.shape[0]
        m, best = z[:, 0], torch.zeros(n, dtype=torch.int64, device=z.device)
        for j in range(1, z.shape[1]):   # np.argmax: the first NaN, else the first maximum
            take = ~torch.isnan(m) & (torch.isnan(z[:, j]) | (z[:, j] > m))
            m = torch.where(take, z[:, j], m)
            best = torch.where(take, torch.full_like(best, j), best)
        return best


def _pair(env_id, n, seed=3, **kwargs):
    import gym_b200
    envs = [gym_b200.vector.make(env_id, n, **kwargs) for _ in range(2)]
    obs = [e.reset(seed=seed)[0] for e in envs]
    return envs[0], MlpTwin(envs[1], obs[1])


def _params(env, hidden, per_env, seed, scale=0.5):
    torch = _torch()
    g = torch.Generator(device="cpu").manual_seed(seed)
    sizes = _sizes(env, hidden)
    P = sum(o * i + o for i, o in zip(sizes[:-1], sizes[1:]))
    lead = (env.num_envs,) if per_env else ()
    return (scale * torch.randn(lead + (P,), generator=g)).to(env.device)


def _twin_check(env_id, n, T, hidden, per_env, seed=3, **kwargs):
    a, b = _pair(env_id, n, seed=seed, **kwargs)
    p = _params(a, hidden, per_env, seed + T)
    got = a.rollout_mlp(p, hidden, T)
    _assert_equals_loop(got, b.loop(p, hidden, T))
    _eq(a.snapshot().obs, got[1][-1], "snapshot().obs vs obs[T-1]")
    _assert_same_env(a, b.env)
    nxt = b.policy(p, hidden)
    for name, x, y in zip(NAMES, a.step(nxt)[:4], b.env.step(nxt)[:4]):
        _eq(x, y, f"next step {name}")
    a.close()
    b.env.close()
    return got


# ---------------------------------------------------------------------------------------------- the eager twin
@pytest.mark.parametrize("per_env", [False, True], ids=["shared", "per_env"])
@pytest.mark.parametrize("n,T", [(1, 1), (257, 37), (33 * 256 + 5, 2), (4099, 300)])
@pytest.mark.parametrize("hidden", HIDDEN, ids=str)
@pytest.mark.parametrize("env_id", CLASSIC)
def test_rollout_mlp_equals_eager_loop(env_id, hidden, n, T, per_env):
    got = _twin_check(env_id, n, T, hidden, per_env)
    assert tuple(got[0].shape[:2]) == (T, n)


def test_unaligned_per_env_rows():
    """h1 % 4 == 0, but the per-env rows are not 16-byte aligned, so the second layer is read a float at a time: P % 4
    != 0, or P % 4 == 0 with params starting 4 bytes into their allocation."""
    _twin_check("MountainCar-v0", 515, 9, (4, 3), True)   # P = 8 + 4 + 12 + 3 + 9 + 3 = 39
    a, b = _pair("CartPole-v1", 515)
    p = _params(a, (8, 6), True, 4)                        # P = 32 + 8 + 48 + 6 + 12 + 2 = 108
    big = _torch().zeros(1 + p.numel(), device=p.device)
    big[1:] = p.reshape(-1)
    q = big[1:].view(p.shape)
    _assert_equals_loop(a.rollout_mlp(q, (8, 6), 9), b.loop(p, (8, 6), 9))


@pytest.mark.parametrize("per_env", [False, True], ids=["shared", "per_env"])
@pytest.mark.parametrize("hidden", [(5,), (64, 64)], ids=str)
@pytest.mark.parametrize("env_id,kwargs", BOX2D, ids=[b[0] for b in BOX2D])
def test_box2d_rollout_mlp_equals_eager_loop(env_id, kwargs, hidden, per_env):
    _twin_check(env_id, 67, 5, hidden, per_env, seed=7, **kwargs)


@pytest.mark.parametrize("env_id", CLASSIC)
def test_rollout_mlp_short_time_limit_and_without_autoreset(env_id):
    got = _twin_check(env_id, 4099, 25, (16, 8), True, max_episode_steps=4)
    assert bool(got[4][3].any())
    _twin_check(env_id, 2053, 40, (6,), False, autoreset=False)
    _twin_check(env_id, 2053, 40, (6, 6), True, autoreset=False, max_episode_steps=4)


def test_rollout_mlp_offsets_past_two_to_the_31():
    """CartPole, n = 2^20, T = 520: T * n * D > 2^31; compared slice by slice with the eager loop."""
    n, T, hidden = 1 << 20, 520, (8, 8)
    assert T * n * 4 > 1 << 31
    a, b = _pair("CartPole-v1", n, seed=5)
    p = _params(a, hidden, False, 5, scale=0.3)
    acts, obs, rew, term, trunc, infos = a.rollout_mlp(p, hidden, T)
    fin, mask = infos["final_observation"], infos["_final_observation"]
    for t in range(T):
        act = b.policy(p, hidden)
        o, r, te, tr, inf = b.env.step(act)
        b.obs = o.clone()
        _eq(acts[t], act, f"actions[{t}]")
        _eq(obs[t], o, f"obs[{t}]")
        _eq(rew[t], r, f"reward[{t}]")
        _eq(term[t], te, f"terminated[{t}]")
        _eq(trunc[t], tr, f"truncated[{t}]")
        m = inf["_final_observation"]
        _eq(mask[t], m, f"mask[{t}]")
        _eq(fin[t][m], inf["final_observation"][m], f"final_observation[{t}]")
    _assert_same_env(a, b.env)


# ------------------------------------------------------------------------------------------------- summary mode
def _summary_check(env_id, n, T, hidden, per_env, seed=9, **kwargs):
    a, b = _pair(env_id, n, seed=seed, **kwargs)
    p = _params(a, hidden, per_env, seed)
    full = b.env.rollout_mlp(p, hidden, T)
    got = a.rollout_mlp(p, hidden, T, summary=True)
    for name, x, y in zip(("returns", "lengths", "ended"), got, summary_of(*full[2:5])):
        _eq(x, y, name)
    _eq(a.snapshot().obs, full[1][-1], "snapshot().obs vs obs[T-1]")
    _assert_same_env(a, b.env)
    a.close()
    b.env.close()
    return got


@pytest.mark.parametrize("per_env", [False, True], ids=["shared", "per_env"])
@pytest.mark.parametrize("hidden", [(5,), (64, 64)], ids=str)
@pytest.mark.parametrize("env_id", CLASSIC)
def test_summary_equals_restatement(env_id, hidden, per_env):
    got = _summary_check(env_id, 33 * 256 + 5, 300, hidden, per_env)
    torch = _torch()
    assert got[0].dtype == torch.float64 and got[1].dtype == torch.int32 and got[2].dtype == torch.bool
    ended = _summary_check(env_id, 1000, 30, hidden, per_env, max_episode_steps=7)[2]
    assert bool(ended.all())


@pytest.mark.parametrize("env_id,kwargs", BOX2D, ids=[b[0] for b in BOX2D])
def test_box2d_summary_equals_restatement(env_id, kwargs):
    _summary_check(env_id, 67, 5, (16, 16), True, seed=7, **kwargs)


# -------------------------------------------------------------------------------------------- interleaving
@pytest.mark.parametrize("env_id", ["CartPole-v1", "MountainCarContinuous-v0", "Acrobot-v1", "LunarLander-v2"])
def test_rollout_mlp_interleaved(env_id):
    """step(), rollout(), rollout_sampled(), rollout_linear(), reset(seed=), restore and clone between calls, mirrored
    on the twin."""
    torch = _torch()
    n, T, hidden = (300, 3, (8,)) if env_id.startswith("Lunar") else (1000, 17, (12, 9))
    a, b = _pair(env_id, n)
    p = _params(a, hidden, True, 1)
    _assert_equals_loop(a.rollout_mlp(p, hidden, T), b.loop(p, hidden, T), "first ")
    act = b.policy(p, hidden)
    o = a.step(act)
    b.obs = b.env.step(act)[0].clone()
    _eq(o[0], b.obs, "step")
    _assert_equals_loop(a.rollout_mlp(p, hidden, T), b.loop(p, hidden, T), "after step ")
    acts = b.policy(p, hidden)[None].repeat(4, *([1] * (1 + (not a.discrete))))
    ra, rb = a.rollout(acts), b.env.rollout(acts)
    b.obs = rb[0][-1].clone()
    _eq(ra[0], rb[0], "rollout obs")
    _assert_equals_loop(a.rollout_mlp(p, hidden, T), b.loop(p, hidden, T), "after rollout ")
    for e in (a, b.env):
        e.action_space.seed(4)
    sa, sb = a.rollout_sampled(3), b.env.rollout_sampled(3)
    b.obs = sb[1][-1].clone()
    _eq(sa[1], sb[1], "rollout_sampled obs")
    _assert_equals_loop(a.rollout_mlp(p, hidden, T), b.loop(p, hidden, T), "after rollout_sampled ")
    K = a.single_action_space.n if a.discrete else a.act_dim
    w = torch.randn(n, K, a.obs_dim, device="cuda:0")
    bias = torch.randn(n, K, device="cuda:0")
    la, lb = a.rollout_linear(w, bias, 3), b.env.rollout_linear(w, bias, 3)
    b.obs = lb[1][-1].clone()
    _eq(la[1], lb[1], "rollout_linear obs")
    _assert_equals_loop(a.rollout_mlp(p, hidden, T), b.loop(p, hidden, T), "after rollout_linear ")
    snap_a, snap_b = a.snapshot(), b.env.snapshot()
    _assert_equals_loop(a.rollout_mlp(p, hidden, T), b.loop(p, hidden, T), "before restore ")
    ra = a.reset(seed=77)[0]
    b.obs = b.env.reset(seed=77)[0].clone()
    _eq(ra, b.obs, "reset")
    _assert_equals_loop(a.rollout_mlp(p, hidden, T), b.loop(p, hidden, T), "after reset ")
    ro = a.restore(snap_a)[0]
    b.obs = b.env.restore(snap_b)[0].clone()
    _eq(ro, b.obs, "restore")
    _assert_equals_loop(a.rollout_mlp(p, hidden, T), b.loop(p, hidden, T), "after restore ")
    src = torch.randint(0, n, (n,), device="cuda:0")
    co = a.clone(src)
    b.obs = b.env.clone(src).clone()
    _eq(co, b.obs, "clone")
    _assert_equals_loop(a.rollout_mlp(p, hidden, T), b.loop(p, hidden, T), "after clone ")
    _assert_same_env(a, b.env)


def test_set_state_then_rollout_mlp_starts_from_the_state():
    """After set_state() the first input is the observation of that state; a step with an out-of-range action returns
    exactly that, so a probe env gives the twin its first input."""
    import gym_b200
    torch = _torch()
    a, b = _pair("Acrobot-v1", 300, seed=4)
    state, elapsed, rng = b.env.get_state()
    state = state.clone()
    state[:, 0] += 0.25
    probe = gym_b200.vector.make("Acrobot-v1", 300)
    probe.reset(seed=4)
    for e in (a, b.env, probe):
        e.set_state(state, elapsed, rng)
    b.obs = probe.step(torch.full((300,), 7, dtype=torch.int64, device="cuda:0"))[0].clone()
    p = _params(a, (64, 64), True, 6)
    _assert_equals_loop(a.rollout_mlp(p, (64, 64), 9), b.loop(p, (64, 64), 9))
    _assert_same_env(a, b.env)


# ------------------------------------------------------------------------------------------------ CUDA graphs
@pytest.mark.parametrize("summary", [False, True], ids=["full", "summary"])
@pytest.mark.parametrize("per_env", [False, True], ids=["shared", "per_env"])
@pytest.mark.parametrize("env_id", ["CartPole-v1", "Pendulum-v1", "Acrobot-v1"])
def test_captured_rollout_mlp_replays_equal_eager_calls(env_id, per_env, summary):
    """Replay k equals eager call k with the parameters copied in place between replays, after a captured step()."""
    torch = _torch()
    n, T, k, hidden = 515, 24, 3, (16, 12)
    a, b = _pair(env_id, n)
    p = _params(a, hidden, per_env, 2)
    step_act = b.policy(p, hidden)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        st = a.step(step_act)
        out = a.rollout_mlp(p, hidden, T, summary=summary)
    for r in range(k):
        p2 = _params(a, hidden, per_env, 100 + r)
        p.copy_(p2)
        g.replay()
        o = b.env.step(step_act)
        b.obs = o[0].clone()
        for name, x, y in zip(NAMES, st[:4], o[:4]):
            _eq(x, y, f"replay {r} step {name}")
        if summary:
            full = b.env.rollout_mlp(p2, hidden, T)
            b.obs = full[1][-1].clone()
            for name, x, y in zip(("returns", "lengths", "ended"), out, summary_of(*full[2:5])):
                _eq(x, y, f"replay {r} {name}")
        else:
            _assert_equals_loop(out, b.loop(p2, hidden, T), f"replay {r} ")
    _assert_same_env(a, b.env)


@pytest.mark.parametrize("env_id,kwargs", BOX2D[:2], ids=[b[0] for b in BOX2D[:2]])
def test_box2d_capture_is_refused(env_id, kwargs):
    from gym_b200 import error
    torch = _torch()
    a, b = _pair(env_id, 33, seed=7, **kwargs)
    p = _params(a, (8,), False, 3)
    before = _untouched(a)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with pytest.raises(error.Error, match="double|alternate|stale"):
        with torch.cuda.graph(g):
            a.rollout_mlp(p, (8,), 2)
    del g
    _assert_untouched(a, before, "capture")
    _assert_equals_loop(a.rollout_mlp(p, (8,), 2), b.loop(p, (8,), 2), "after the refused capture ")


# ------------------------------------------------------------------------------------- the module's packing
@pytest.mark.parametrize("hidden", [(32,), (64, 64)], ids=str)
@pytest.mark.parametrize("env_id", ["CartPole-v1", "Pendulum-v1", "Acrobot-v1"])
def test_packing_is_the_modules(env_id, hidden):
    """parameters_to_vector(nn.Sequential(...)) is the packing: step 0's actions agree with the module's forward, which
    runs through cuBLAS with another summation order (and possibly TF32 off or on), so only within a float32
    tolerance, not bit for bit."""
    torch = _torch()
    a, b = _pair(env_id, 4096, seed=11)
    sizes = _sizes(a, hidden)
    torch.manual_seed(1)
    mods = []
    for i, (fan_in, fan_out) in enumerate(zip(sizes[:-1], sizes[1:])):
        mods += [torch.nn.Linear(fan_in, fan_out)] + ([torch.nn.ReLU()] if i < len(hidden) else [])
    net = torch.nn.Sequential(*mods).to("cuda:0")
    p = torch.nn.utils.parameters_to_vector(net.parameters()).detach().contiguous()
    torch.backends.cuda.matmul.allow_tf32 = False
    with torch.no_grad():
        want = net(b.obs)
    got = a.rollout_mlp(p, hidden, 1)[0][0]
    torch.testing.assert_close(b.outputs(p, hidden), want, rtol=1e-4, atol=1e-4)
    if a.discrete:
        z = want.sort(dim=1).values
        clear = z[:, -1] - z[:, -2] > 1e-3   # no near-tie that rounding could flip
        assert torch.equal(got[clear], want.argmax(dim=1)[clear])
    else:
        torch.testing.assert_close(got.reshape(want.shape), want, rtol=1e-4, atol=1e-4)


# ------------------------------------------------------------------------------------------ refusals and guards
def test_rollout_mlp_guards_and_refusals():
    import gym_b200
    from gym_b200 import error, wrappers
    from gym_b200.distributed import ShardedVectorEnv
    from gym_b200.env import B200Env
    torch = _torch()

    env = gym_b200.vector.make("CartPole-v1", 64)
    p = _params(env, (8, 4), False, 0)
    with pytest.raises(error.ResetNeeded):
        env.rollout_mlp(p, (8, 4), 3)
    env.reset(seed=1)
    before = _untouched(env)
    for bad in (0, -1, 2 ** 31, 2.0, True, "3"):
        with pytest.raises(ValueError):
            env.rollout_mlp(p, (8, 4), bad)
        _assert_untouched(env, before, repr(bad))
    pp = _params(env, (8, 4), True, 0)
    bad_args = [
        (p.double(), (8, 4)), (p.half(), (8, 4)), (p.cpu(), (8, 4)),                 # dtype, device
        (p[:-1], (8, 4)), (p[None], (8, 4)), (pp[:-1], (8, 4)), (pp[:, :-1], (8, 4)),  # shapes
        (p, (8,)), (p, (4, 8)), (pp, (8, 5)),                                           # the wrong widths
        (torch.stack([pp, pp], 2)[:, :, 0], (8, 4)),                                     # not contiguous
        (p.tolist(), (8, 4)),
        (p, ()), (p, (8, 4, 4)), (p, (0,)), (p, (65,)), (p, (8, 0)), (p, (8, 65)),      # layers, widths
        (p, (8.0, 4)), (p, (True, 4)), (p, 8), (p, None),
    ]
    for k, (x, h) in enumerate(bad_args):
        with pytest.raises(ValueError):
            env.rollout_mlp(x, h, 3)
        _assert_untouched(env, before, f"bad arguments {k}")
    env.step_async(torch.zeros(64, dtype=torch.int64, device="cuda:0"))
    with pytest.raises(error.AlreadyPendingCallError):
        env.rollout_mlp(p, (8, 4), 3)
    env.step_wait()
    before = _untouched(env)
    for wr in (wrappers.RecordEpisodeStatistics(env), wrappers.NormalizeObservation(env),
               wrappers.NormalizeReward(env), wrappers.VectorListInfo(env)):
        with pytest.raises(error.Error, match="rollout_mlp"):
            wr.rollout_mlp(p, (8, 4), 3)
        with pytest.raises(error.Error, match="rollout_mlp"):
            wr.rollout_mlp(p, (8, 4), 3, summary=True)
    _assert_untouched(env, before, "wrappers")
    env.close()
    with pytest.raises(error.ClosedEnvironmentError):
        env.rollout_mlp(p, (8, 4), 3)

    host = gym_b200.vector.make("CartPole-v1", 16, backend="numpy")
    host.reset(seed=3)
    rows = host.snapshot().rows.clone()
    with pytest.raises(error.Error, match="backend"):
        host.rollout_mlp(p, (8, 4), 3)
    assert torch.equal(host.snapshot().rows, rows)
    host.close()

    from gym_b200 import subenv
    chain = gym_b200.vector.make("CartPole-v1", 16, wrappers=[subenv.RecordEpisodeStatistics()])
    chain.reset(seed=4)
    before = _untouched(chain)
    with pytest.raises(error.Error, match="wrappers"):
        chain.rollout_mlp(p, (8, 4), 3)
    _assert_untouched(chain, before, "per-env wrappers")
    chain.close()

    assert not hasattr(ShardedVectorEnv, "rollout_mlp")
    assert not hasattr(B200Env, "rollout_mlp")


def test_c_entry_point_validates_widths():
    """The C entry point checks the layer count and widths itself, for callers other than the Python layer."""
    import ctypes

    import gym_b200
    env = gym_b200.vector.make("CartPole-v1", 8)
    env.reset(seed=2)
    p = _params(env, (4,), False, 0)
    last = _torch().empty(8, 4, device="cuda:0")
    vp = ctypes.c_void_p
    for layers, h1, h2 in ((0, 4, 0), (3, 4, 4), (1, 0, 0), (1, 65, 0), (2, 4, 0), (2, 4, 65)):
        rc = env._lib.b200gym_rollout_mlp(env._handle, vp(p.data_ptr()), 0, layers, h1, h2, 3, *([None] * 6),
                                          vp(last.data_ptr()), vp(last.data_ptr()), vp(last.data_ptr()),
                                          vp(last.data_ptr()), None, env._stream())
        assert rc != 0, (layers, h1, h2)
        assert b"b200gym_rollout_mlp" in env._lib.b200gym_last_error(env._handle)
    env.close()
