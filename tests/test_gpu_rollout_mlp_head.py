"""``rollout_mlp(..., head=...)`` and ``rollout_mlp_noisy(..., head=...)`` on the GPU: the tanh-squashed TD3 / DDPG and
SAC actors.

The SAC head's exp is CUDA's ``expf``.  The first test runs it on every float32 bit pattern through
``b200gym_selftest_exp`` and compares it with ``torch.exp`` on the same device, bit for bit; with the tanh of
test_gpu_rollout_mlp_tanh.py, that is what makes the torch restatement of the head below bit-exact for the torch build
the tests run.  The rest compare both calls with eager twins built on test_gpu_rollout_mlp.py's and
test_gpu_rollout_mlp_noisy.py's: the MLP and the documented head in torch elementwise ops, then ``step()``.  Compared
are the actions, the outputs, the env outputs, the final observations on the rows the mask selects, the summary,
``get_state()``, ``snapshot()`` rows and observations, and the step after.
"""
import ctypes

import pytest

from test_gpu_rollout_linear import (NAMES, _assert_equals_loop, _assert_same_env, _assert_untouched, _eq, _untouched,
                                     summary_of)
from test_gpu_rollout_mlp_noisy import NoisyTwin, _assert_equals_noisy

pytestmark = pytest.mark.gpu

CLASSIC_BOX = ["Pendulum-v1", "MountainCarContinuous-v0"]
BOX2D_BOX = [("LunarLanderContinuous-v2", {}), ("BipedalWalker-v3", {}), ("BipedalWalkerHardcore-v3", {})]
HEADS = ["tanh", "tanh_normal"]
HIDDEN = [(1,), (3, 7), (64, 64)]


def _torch():
    import torch
    return torch


class HeadTwin(NoisyTwin):
    """NoisyTwin with the hidden layers' `activation` and the head `head`: ``policy`` is the deterministic head,
    ``noisy_policy`` the head with noise, both in torch elementwise ops in the documented order."""

    def __init__(self, env, obs, activation, head):
        super().__init__(env, obs)
        torch = _torch()
        single = env.single_action_space
        self.activation, self.head, self.A = activation, head, int(env.act_dim)
        self.K = self.A * (2 if head == "tanh_normal" else 1)
        f32 = dict(dtype=torch.float32, device=env.device)
        # CleanRL's action_scale and action_bias
        self.scale = torch.tensor((single.high - single.low) / 2.0, **f32)
        self.bias = torch.tensor((single.high + single.low) / 2.0, **f32)
        self.low, self.high = torch.tensor(single.low, **f32), torch.tensor(single.high, **f32)

    def outputs(self, params, hidden):
        torch = _torch()
        n = self.env.num_envs
        P = params.shape[-1]
        W = params.expand(n, P)
        x, off = self.obs, 0
        sizes = [self.env.obs_dim] + list(hidden) + [self.K]
        for layer, (fan_in, fan_out) in enumerate(zip(sizes[:-1], sizes[1:])):
            w = W[:, off:off + fan_out * fan_in].reshape(n, fan_out, fan_in)
            off += fan_out * fan_in
            z = W[:, off:off + fan_out].clone()
            off += fan_out
            for k in range(fan_in):
                z = z + w[:, :, k] * x[:, None, k]
            if layer < len(hidden):
                z = torch.tanh(z) if self.activation == "tanh" else torch.where((z > 0) | torch.isnan(z), z,
                                                                                torch.zeros_like(z))
            x = z
        assert off == P
        return x

    def policy(self, params, hidden):
        return _torch().tanh(self.outputs(params, hidden)[:, :self.A]) * self.scale + self.bias

    def noisy_policy(self, params, hidden, e):
        torch = _torch()
        z = self.outputs(params, hidden)
        A = self.A
        if self.head == "tanh":
            v = (torch.tanh(z) * self.scale + self.bias) + e
            return z, torch.where(v < self.low, self.low, torch.where(v > self.high, self.high, v))
        ls = -5 + 3.5 * (torch.tanh(z[:, A:]) + 1)
        x = z[:, :A] + e * ls.exp()
        return z, torch.tanh(x) * self.scale + self.bias


def _pair(env_id, n, activation, head, seed=3, **kwargs):
    import gym_b200
    envs = [gym_b200.vector.make(env_id, n, **kwargs) for _ in range(2)]
    obs = [e.reset(seed=seed)[0] for e in envs]
    return envs[0], HeadTwin(envs[1], obs[1], activation, head)


def _params(b, hidden, per_env, seed, scale=1.0):
    torch = _torch()
    g = torch.Generator(device="cpu").manual_seed(seed)
    sizes = [b.env.obs_dim] + list(hidden) + [b.K]
    P = sum(o * i + o for i, o in zip(sizes[:-1], sizes[1:]))
    lead = (b.env.num_envs,) if per_env else ()
    return (scale * torch.randn(lead + (P,), generator=g)).to(b.env.device)


def _noise(b, T, seed, scale=1.0):
    torch = _torch()
    g = torch.Generator(device=b.env.device).manual_seed(seed)
    return scale * torch.randn((T, b.env.num_envs, b.A), generator=g, device=b.env.device)


def _next_step(a, b, p, hidden):
    _assert_same_env(a, b.env)
    nxt = b.policy(p, hidden)
    o = b.env.step(nxt)
    for name, x, y in zip(NAMES, a.step(nxt)[:4], o[:4]):
        _eq(x, y, f"next step {name}")
    b.obs = o[0].clone()


def _check(env_id, n, T, hidden, per_env, activation, head, seed=3, **kwargs):
    """Full, noisy and summary calls in a row on one env and its twin, each against the eager loop."""
    a, b = _pair(env_id, n, activation, head, seed=seed, **kwargs)
    kw = dict(activation=activation, head=head)
    p = _params(b, hidden, per_env, seed + T)
    got = a.rollout_mlp(p, hidden, T, **kw)
    assert tuple(got[0].shape) == (T, n, b.A)
    _assert_equals_loop(got, b.loop(p, hidden, T))
    _eq(a.snapshot().obs, got[1][-1], "snapshot().obs vs obs[T-1]")
    _next_step(a, b, p, hidden)
    e = _noise(b, T, seed + 1)
    got = a.rollout_mlp_noisy(p, hidden, e, **kw)
    assert tuple(got[1].shape) == (T, n, b.K)
    _assert_equals_noisy(got, b.noisy_loop(p, hidden, e))
    _eq(a.snapshot().obs, got[2][-1], "snapshot().obs vs obs[T-1]")
    _next_step(a, b, p, hidden)
    got = a.rollout_mlp(p, hidden, T, summary=True, **kw)
    full = b.loop(p, hidden, T)
    for name, x, y in zip(("returns", "lengths", "ended"), got, summary_of(*full[1][1:4])):
        _eq(x, y, name)
    _eq(a.snapshot().obs, full[1][0][-1], "summary: snapshot().obs vs obs[T-1]")
    _next_step(a, b, p, hidden)
    a.close()
    b.env.close()


# ------------------------------------------------------------------------------------------------- expf itself
def test_exp_equals_torch_exp_for_every_float32():
    """All 2^32 bit patterns, 2^28 at a time: b200gym_selftest_exp against torch.exp of the same tensor on the same
    device, compared as int32 so that signed zeros and NaN payloads count."""
    import gym_b200  # noqa: F401
    from gym_b200 import _lib
    torch = _torch()
    lib = _lib.load()
    chunk = 1 << 28
    x = torch.empty(chunk, dtype=torch.int32, device="cuda:0")
    y = torch.empty(chunk, dtype=torch.float32, device="cuda:0")
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    bad, first = 0, []
    for lo in range(-(1 << 31), 1 << 31, chunk):
        x.copy_(torch.arange(lo, lo + chunk, dtype=torch.int64, device="cuda:0"))   # every value fits in int32
        xf = x.view(torch.float32)
        assert lib.b200gym_selftest_exp(ctypes.c_void_p(xf.data_ptr()), chunk, ctypes.c_void_p(y.data_ptr()),
                                        stream) == 0
        want = torch.exp(xf)
        diff = y.view(torch.int32) != want.view(torch.int32)
        k = int(diff.sum())
        if k:
            bad += k
            idx = diff.nonzero()[:4, 0]
            first += [(hex(int(x[i]) & 0xffffffff), hex(int(y.view(torch.int32)[i]) & 0xffffffff),
                       hex(int(want.view(torch.int32)[i]) & 0xffffffff)) for i in idx]
    assert bad == 0, f"{bad} of 2^32 inputs differ from torch.exp; first (x, engine, torch): {first[:8]}"


# ---------------------------------------------------------------------------------------------- the eager twins
@pytest.mark.parametrize("per_env", [False, True], ids=["shared", "per_env"])
@pytest.mark.parametrize("n,T", [(1, 1), (257, 37), (33 * 256 + 5, 2), (4099, 60)])
@pytest.mark.parametrize("hidden", HIDDEN, ids=str)
@pytest.mark.parametrize("activation", ["relu", "tanh"])
@pytest.mark.parametrize("head", HEADS)
@pytest.mark.parametrize("env_id", CLASSIC_BOX)
def test_head_rollouts_equal_eager_loop(env_id, head, activation, hidden, n, T, per_env):
    _check(env_id, n, T, hidden, per_env, activation, head)


@pytest.mark.parametrize("head", HEADS)
@pytest.mark.parametrize("env_id", CLASSIC_BOX)
def test_head_short_time_limit_and_without_autoreset(env_id, head):
    _check(env_id, 2053, 13, (16, 8), True, "tanh", head, max_episode_steps=1)
    _check(env_id, 2053, 13, (16, 8), False, "relu", head, max_episode_steps=13)
    _check(env_id, 2053, 20, (6,), False, "tanh", head, autoreset=False, max_episode_steps=4)


@pytest.mark.parametrize("per_env", [False, True], ids=["shared", "per_env"])
@pytest.mark.parametrize("head", HEADS)
@pytest.mark.parametrize("env_id,kwargs", BOX2D_BOX, ids=[b[0] for b in BOX2D_BOX])
def test_box2d_head_rollouts_equal_eager_loop(env_id, kwargs, head, per_env):
    _check(env_id, 67, 5, (64, 64), per_env, "relu", head, seed=7, **kwargs)


def _special():
    torch = _torch()
    f = torch.finfo(torch.float32)
    return torch.tensor([0.0, -0.0, 1e-45, -1e-45, f.tiny, -f.tiny, float("inf"), float("-inf"), float("nan"), 1.0,
                         -1.0, 20.0, -20.0, 2.0, -2.0, f.max, -f.max], dtype=torch.float32)


@pytest.mark.parametrize("head", HEADS)
@pytest.mark.parametrize("env_id", CLASSIC_BOX)
def test_special_outputs_noise_and_bounds(env_id, head):
    """Per-env hidden (1,) policies whose outputs are exactly chosen values (zero first layer, output weights -0.0, so
    z = the output bias): z, m and s at +-0, subnormals, +-tiny, +-inf, NaN, +-1, +-2, +-20 and +-FLT_MAX against noise
    at the same values, every pair once.  That covers saturated log-stds (ls = 2 and -5 exactly), actions at and beyond
    the bounds, and NaN through the clamp; the TD3 clamp also equals torch.clamp on them."""
    torch = _torch()
    v = _special().to("cuda:0")
    m, e = torch.meshgrid(v, v, indexing="ij")
    m, e = m.reshape(-1), e.reshape(-1)
    n = m.numel()
    for noisy in (False, True):
        a, b = _pair(env_id, n, "relu", head, seed=8)
        D, K = a.obs_dim, b.K
        p = torch.zeros(n, D + 1 + 2 * K, device="cuda:0")
        p[:, D + 1:D + 1 + K] = -0.0
        p[:, D + 1 + K:] = torch.stack([m, m.roll(5)], dim=1)[:, :K]
        if noisy:
            got = a.rollout_mlp_noisy(p, (1,), e.reshape(1, n, 1), head=head)
            _assert_equals_noisy(got, b.noisy_loop(p, (1,), e.reshape(1, n, 1)))
            chosen, nan = p[:, D + 1 + K:], torch.isnan(p[:, D + 1 + K:])
            assert torch.equal(torch.isnan(got[1][0]), nan)   # the add makes any NaN the canonical one
            _eq(got[1][0][~nan], chosen[~nan], "outputs are the chosen values")
            if head == "tanh":
                z = got[1][0, :, 0]
                _eq(got[0][0, :, 0], torch.clamp(torch.tanh(z) * b.scale + b.bias + e, float(b.low), float(b.high)),
                    "torch.clamp")
            else:
                ls = -5 + 3.5 * (torch.tanh(torch.tensor([20.0, -20.0], device="cuda:0")) + 1)
                assert ls.tolist() == [2.0, -5.0]
        else:
            got = a.rollout_mlp(p, (1,), 1, head=head)
            _assert_equals_loop(got, b.loop(p, (1,), 1))
        _assert_same_env(a, b.env)
        a.close()
        b.env.close()


# ------------------------------------------------------------------------------------------- CleanRL's actors
def _cleanrl_actors(D, A, H, scale, bias):
    """The actors of CleanRL's td3_continuous_action.py and sac_continuous_action.py at hidden (H, H), on cuda:0."""
    torch = _torch()
    nn, F = torch.nn, torch.nn.functional

    class TD3Actor(nn.Module):
        def __init__(self):
            super().__init__()
            self.fc1, self.fc2, self.fc_mu = nn.Linear(D, H), nn.Linear(H, H), nn.Linear(H, A)
            self.register_buffer("action_scale", scale)
            self.register_buffer("action_bias", bias)

        def forward(self, x):
            x = F.relu(self.fc2(F.relu(self.fc1(x))))
            return torch.tanh(self.fc_mu(x)) * self.action_scale + self.action_bias

    class SACActor(nn.Module):
        def __init__(self):
            super().__init__()
            self.fc1, self.fc2 = nn.Linear(D, H), nn.Linear(H, H)
            self.fc_mean, self.fc_logstd = nn.Linear(H, A), nn.Linear(H, A)
            self.register_buffer("action_scale", scale)
            self.register_buffer("action_bias", bias)

        def trunk(self, x):
            return F.relu(self.fc2(F.relu(self.fc1(x))))

        def forward(self, x):
            x = self.trunk(x)
            log_std = torch.tanh(self.fc_logstd(x))
            return self.fc_mean(x), -5 + 0.5 * (2 - -5) * (log_std + 1)

        def get_action(self, x, eps):
            """(sampled action, deterministic action); Normal(mean, std).rsample() is mean + eps * std"""
            mean, log_std = self(x)
            x_t = mean + eps * log_std.exp()
            squash = lambda y: torch.tanh(y) * self.action_scale + self.action_bias  # noqa: E731
            return squash(x_t), squash(mean)

    torch.manual_seed(0)
    return TD3Actor().cuda(), SACActor().cuda()


@pytest.mark.parametrize("env_id", CLASSIC_BOX + ["BipedalWalker-v3"])
def test_cleanrl_actor_packings(env_id):
    """parameters_to_vector of CleanRL's TD3 actor, and the documented torch.cat line for its two-head SAC actor, give
    the modules' own actions (nn.Linear sums in another order, so within float32 rounding)."""
    import gym_b200
    torch = _torch()
    n = 515
    env = gym_b200.vector.make(env_id, n)
    obs = env.reset(seed=4)[0].clone()
    single = env.single_action_space
    f32 = dict(dtype=torch.float32, device="cuda:0")
    scale = torch.tensor((single.high - single.low) / 2.0, **f32)
    bias = torch.tensor((single.high + single.low) / 2.0, **f32)
    td3, sac = _cleanrl_actors(env.obs_dim, env.act_dim, 64, scale, bias)
    close = dict(rtol=1e-5, atol=1e-5)
    with torch.no_grad():
        p = torch.nn.utils.parameters_to_vector(td3.parameters()).detach()
        noise = torch.randn(1, n, env.act_dim, **f32) * (scale * 0.1)
        s = env.snapshot()
        a = env.rollout_mlp(p, (64, 64), 1, head="tanh")[0][0]
        torch.testing.assert_close(a, td3(obs), **close)
        env.restore(s)
        a = env.rollout_mlp_noisy(p, (64, 64), noise, head="tanh")[0][0]
        want = (td3(obs) + noise[0]).clamp(float(single.low[0]), float(single.high[0]))
        torch.testing.assert_close(a, want, **close)
        env.restore(s)
        p = torch.cat([q.reshape(-1) for q in (sac.fc1.weight, sac.fc1.bias, sac.fc2.weight, sac.fc2.bias,
                                               sac.fc_mean.weight, sac.fc_logstd.weight, sac.fc_mean.bias,
                                               sac.fc_logstd.bias)]).detach()
        eps = torch.randn(1, n, env.act_dim, **f32)
        sampled, mean = sac.get_action(obs, eps[0])
        torch.testing.assert_close(env.rollout_mlp(p, (64, 64), 1, head="tanh_normal")[0][0], mean, **close)
        env.restore(s)
        got = env.rollout_mlp_noisy(p, (64, 64), eps, head="tanh_normal")
        torch.testing.assert_close(got[0][0], sampled, **close)
        h = sac.trunk(obs)
        torch.testing.assert_close(got[1][0], torch.cat([sac.fc_mean(h), sac.fc_logstd(h)], dim=1), **close)
    env.close()


# ------------------------------------------------------------------------------------------------ CUDA graphs
@pytest.mark.parametrize("head", HEADS)
@pytest.mark.parametrize("per_env", [False, True], ids=["shared", "per_env"])
@pytest.mark.parametrize("env_id", CLASSIC_BOX)
def test_captured_head_rollouts_replay_equal_eager_calls(env_id, per_env, head):
    """One graph holds a head rollout_mlp(), a noise draw and a head rollout_mlp_noisy(); replay k equals eager call k
    with the parameters copied in place between replays and new noise drawn inside the graph."""
    torch = _torch()
    n, T, k, hidden = 515, 24, 3, (16, 12)
    a, b = _pair(env_id, n, "tanh", head)
    kw = dict(activation="tanh", head=head)
    p = _params(b, hidden, per_env, 2)
    e = _noise(b, T, 2)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = a.rollout_mlp(p, hidden, T, **kw)
        e.copy_(torch.randn(e.shape, device=e.device))
        noisy = a.rollout_mlp_noisy(p, hidden, e, **kw)
    e_prev = None
    for r in range(k):
        p.copy_(_params(b, hidden, per_env, 100 + r))
        g.replay()
        _assert_equals_loop(out, b.loop(p, hidden, T), f"replay {r} ")
        e_now = e.clone()
        _assert_equals_noisy(noisy, b.noisy_loop(p, hidden, e_now), f"replay {r} noisy ")
        if e_prev is not None:
            assert not torch.equal(e_now, e_prev), "each replay draws new noise"
        e_prev = e_now
    _assert_same_env(a, b.env)
    a.close()
    b.env.close()


@pytest.mark.parametrize("env_id,kwargs", BOX2D_BOX[:1], ids=[b[0] for b in BOX2D_BOX[:1]])
def test_box2d_capture_is_refused(env_id, kwargs):
    from gym_b200 import error
    torch = _torch()
    a, b = _pair(env_id, 64, "relu", "tanh_normal", **kwargs)
    p = _params(b, (8,), False, 1)
    e = _noise(b, 3, 1)
    before = _untouched(a)
    for call in (lambda: a.rollout_mlp(p, (8,), 3, head="tanh_normal"),
                 lambda: a.rollout_mlp_noisy(p, (8,), e, head="tanh_normal")):
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with pytest.raises(error.Error, match="double|alternate|stale"):
            with torch.cuda.graph(g):
                call()
        del g
        _assert_untouched(a, before, "refused capture")
    a.close()
    b.env.close()


# ------------------------------------------------------------------------------------- unchanged default path
@pytest.mark.parametrize("env_id", ["CartPole-v1", "Pendulum-v1", "LunarLanderContinuous-v2"])
def test_head_none_never_reaches_the_head_entry_points(monkeypatch, env_id):
    """With the head entry points replaced by a stub that raises, head=None calls run the existing entry points and
    return what a twin returns without the keyword."""
    import gym_b200
    from gym_b200 import _lib

    def stub(*args):
        raise AssertionError("a head entry point was called")
    lib = _lib.load()
    for name in ("b200gym_rollout_mlp_head", "b200gym_rollout_mlp_noisy_head"):
        monkeypatch.setattr(lib, name, stub)
    envs = [gym_b200.vector.make(env_id, 300, max_episode_steps=9) for _ in range(2)]
    for env in envs:
        env.reset(seed=6)
    from test_gpu_rollout_mlp import _params as mlp_params
    from test_gpu_rollout_mlp_noisy import _noise as mlp_noise
    p = mlp_params(envs[0], (8, 8), False, 6)
    e = mlp_noise(envs[0], 12, 6)
    x, y = envs[0].rollout_mlp(p, (8, 8), 12, head=None), envs[1].rollout_mlp(p, (8, 8), 12)
    for name, s, t in zip(("actions",) + NAMES, x[:5], y[:5]):
        _eq(s, t, name)
    x, y = envs[0].rollout_mlp_noisy(p, (8, 8), e, head=None), envs[1].rollout_mlp_noisy(p, (8, 8), e)
    for name, s, t in zip(("actions", "outputs") + NAMES, x[:6], y[:6]):
        _eq(s, t, name)
    x, y = envs[0].rollout_mlp(p, (8, 8), 5, summary=True, head=None), envs[1].rollout_mlp(p, (8, 8), 5, summary=True)
    for name, s, t in zip(("returns", "lengths", "ended"), x, y):
        _eq(s, t, name)
    _assert_same_env(envs[0], envs[1])
    if not envs[0].discrete:
        with pytest.raises(AssertionError, match="head entry point"):   # the stub is what head= reaches
            envs[0].rollout_mlp(_params(HeadTwin(envs[0], envs[0]._out[envs[0]._flip]["obs"], "relu", "tanh"),
                                        (8, 8), False, 1), (8, 8), 3, head="tanh")
    monkeypatch.undo()
    for env in envs:
        env.close()


# ------------------------------------------------------------------------------------------- argument checks
def test_refusals_leave_the_env_untouched():
    import gym_b200
    from gym_b200 import error, wrappers
    torch = _torch()
    env = gym_b200.vector.make("Pendulum-v1", 64)
    env.reset(seed=1)
    b = HeadTwin(env, env._out[env._flip]["obs"], "relu", "tanh_normal")
    p2 = _params(b, (8, 4), False, 0)                        # K = 2: the SAC actor
    p1 = _params(HeadTwin(env, b.obs, "relu", "tanh"), (8, 4), False, 0)   # K = 1
    e = _noise(b, 3, 0)
    f64 = dict(dtype=torch.float64, device="cuda:0")
    stats = (torch.zeros(env.obs_dim, **f64), torch.ones(env.obs_dim, **f64))
    before = _untouched(env)
    for bad in ("TANH", "", "normal", "tanh ", "squash", 0, 1, 2, True, b"tanh", ["tanh"], torch.tanh):
        for call in (lambda: env.rollout_mlp(p1, (8, 4), 3, head=bad),
                     lambda: env.rollout_mlp(p1, (8, 4), 3, summary=True, head=bad),
                     lambda: env.rollout_mlp_noisy(p1, (8, 4), e, head=bad)):
            with pytest.raises(ValueError, match="head"):
                call()
            _assert_untouched(env, before, f"head {bad!r}")
    wrong = [lambda: env.rollout_mlp(p1, (8, 4), 3, head="tanh_normal"),          # params of the other head
             lambda: env.rollout_mlp(p2, (8, 4), 3, head="tanh"),
             lambda: env.rollout_mlp_noisy(p1, (8, 4), e, head="tanh_normal"),
             lambda: env.rollout_mlp_noisy(p2, (8, 4), torch.zeros(3, 64, 2, device="cuda:0"), head="tanh_normal"),
             lambda: env.rollout_mlp(p2, (8, 4), 3, head="tanh_normal", obs_norm=stats),
             lambda: env.rollout_mlp(p2, (8, 4), 3, summary=True, head="tanh_normal", obs_moments=True),
             lambda: env.rollout_mlp(p2, (8, 4), 3, head="tanh_normal", clip_obs=5.0),
             lambda: env.rollout_mlp_noisy(p2, (8, 4), e, head="tanh_normal", obs_norm=stats),
             lambda: env.rollout_mlp_noisy(p2, (8, 4), e, head="tanh_normal", clip_obs=5.0)]
    for k, call in enumerate(wrong):
        with pytest.raises(ValueError):
            call()
        _assert_untouched(env, before, f"refusal {k}")
    with pytest.raises(TypeError):
        env.rollout_mlp_noisy(p2, (8, 4), e, "relu", "tanh_normal")   # keyword only
    for wr in (wrappers.RecordEpisodeStatistics(env), wrappers.NormalizeObservation(env)):
        with pytest.raises(error.Error, match="rollout_mlp"):
            wr.rollout_mlp(p2, (8, 4), 3, head="tanh_normal")
        with pytest.raises(error.Error, match="rollout_mlp_noisy"):
            wr.rollout_mlp_noisy(p2, (8, 4), e, head="tanh_normal")
    _assert_untouched(env, before, "wrappers")
    env.close()
    cp = gym_b200.vector.make("CartPole-v1", 64)
    cp.reset(seed=1)
    from test_gpu_rollout_mlp import _params as mlp_params
    q = mlp_params(cp, (8,), False, 0)
    before = _untouched(cp)
    for head in HEADS:
        with pytest.raises(ValueError, match="Box"):
            cp.rollout_mlp(q, (8,), 3, head=head)
        with pytest.raises(ValueError, match="Box"):
            cp.rollout_mlp_noisy(q, (8,), torch.zeros(3, 64, 2, device="cuda:0"), head=head)
    _assert_untouched(cp, before, "Discrete")
    cp.close()


def test_c_entry_points_check_the_head_code_and_kind():
    """The head entry points check the code, the kind, the layers and the widths themselves, for callers other than
    the Python layer."""
    import gym_b200
    torch = _torch()
    vp = ctypes.c_void_p
    for env_id in ("Pendulum-v1", "CartPole-v1"):
        env = gym_b200.vector.make(env_id, 8)
        env.reset(seed=2)
        p = torch.zeros(4096, device="cuda:0")
        e = torch.zeros(3, 8, 2, device="cuda:0")
        outputs = torch.empty(3, 8, 2, device="cuda:0")
        actions = torch.empty(3, 8, 2, device="cuda:0")
        obs = torch.empty(3, 8, env.obs_dim, device="cuda:0")
        reward = torch.empty(3, 8, dtype=torch.float64, device="cuda:0")
        flags = torch.empty(2, 3, 8, dtype=torch.uint8, device="cuda:0")
        last = torch.empty(8, env.obs_dim, device="cuda:0")
        first = env._out[env._flip]["obs"]
        outs = [vp(actions.data_ptr()), vp(obs.data_ptr()), vp(reward.data_ptr()), vp(flags[0].data_ptr()),
                vp(flags[1].data_ptr()), None]
        before = _untouched(env)
        cases = [(0, 1, 4, 0, 1, "head"), (3, 1, 4, 0, 1, "head"), (-1, 1, 4, 0, 1, "head"),
                 (1, 3, 4, 0, 1, "n_layers"), (2, 1, 65, 0, 1, "widths"), (2, 2, 4, 0, 1, "widths"), (1, 1, 4, 0, 2, "activation")]
        if env.discrete:
            cases = [(1, 1, 4, 0, 0, "Box"), (2, 1, 4, 0, 1, "Box")]
        for head, layers, h1, h2, act, what in cases:
            rc = env._lib.b200gym_rollout_mlp_head(env._handle, vp(p.data_ptr()), 0, layers, h1, h2, 3, *outs, None,
                                                   None, None, vp(last.data_ptr()), vp(first.data_ptr()),
                                                   env._stream(), act, head)
            assert rc != 0 and what.encode() in env._lib.b200gym_last_error(env._handle), (env_id, head, what)
            rc = env._lib.b200gym_rollout_mlp_noisy_head(env._handle, vp(p.data_ptr()), 0, layers, h1, h2, 3,
                                                         vp(e.data_ptr()), vp(outputs.data_ptr()), *outs,
                                                         vp(last.data_ptr()), vp(first.data_ptr()), env._stream(), act,
                                                         head)
            assert rc != 0 and what.encode() in env._lib.b200gym_last_error(env._handle), (env_id, head, what)
        _assert_untouched(env, before, f"{env_id}: refused codes")
        env.close()
