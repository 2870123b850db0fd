"""``rollout_mlp(..., activation="tanh")`` and ``rollout_mlp_noisy(..., activation="tanh")`` on the GPU.

The engine's tanh is CUDA's ``tanhf``.  The first test runs it on every float32 bit pattern through
``b200gym_selftest_tanh`` and compares it with ``torch.tanh`` on the same device, bit for bit; that is what makes
``torch.tanh`` / ``nn.Tanh`` a bit-exact restatement of the activation for the torch build the tests run.  The second
sends chosen pre-activations through the rollout kernels themselves.  The rest compare the rollouts with the eager
twins of test_gpu_rollout_mlp.py and test_gpu_rollout_mlp_noisy.py, their activation swapped for ``torch.tanh``: the
actions, the outputs, the env outputs, the final observations on the rows the mask selects, ``get_state()``,
``snapshot()`` rows and observations, and the step after.
"""
import ctypes

import pytest

from test_gpu_rollout_linear import (BOX2D, CLASSIC, NAMES, _assert_equals_loop, _assert_same_env, _assert_untouched,
                                     _eq, _untouched, summary_of)
from test_gpu_rollout_mlp import _params, _sizes
from test_gpu_rollout_mlp_noisy import NoisyTwin, _assert_equals_noisy, _noise

pytestmark = pytest.mark.gpu

HIDDEN = [(1,), (64,), (3, 7), (64, 64)]
TANH = {"activation": "tanh"}


def _torch():
    import torch
    return torch


class TanhTwin(NoisyTwin):
    """NoisyTwin (so also MlpTwin's ``policy`` and ``loop``) with ``torch.tanh`` after every hidden layer."""

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
                z = torch.tanh(z)
            x = z
        assert off == P
        return x


def _pair(env_id, n, seed=3, **kwargs):
    import gym_b200
    envs = [gym_b200.vector.make(env_id, n, **kwargs) for _ in range(2)]
    obs = [e.reset(seed=seed)[0] for e in envs]
    return envs[0], TanhTwin(envs[1], obs[1])


def _close(a, b):
    a.close()
    b.env.close()


def _check_next_step(a, b, p, hidden):
    _assert_same_env(a, b.env)
    nxt = b.policy(p, hidden)
    for name, x, y in zip(NAMES, a.step(nxt)[:4], b.env.step(nxt)[:4]):
        _eq(x, y, f"next step {name}")


def _twin_check(env_id, n, T, hidden, per_env, seed=3, **kwargs):
    a, b = _pair(env_id, n, seed=seed, **kwargs)
    p = _params(a, hidden, per_env, seed + T)
    got = a.rollout_mlp(p, hidden, T, **TANH)
    _assert_equals_loop(got, b.loop(p, hidden, T))
    _eq(a.snapshot().obs, got[1][-1], "snapshot().obs vs obs[T-1]")
    _check_next_step(a, b, p, hidden)
    _close(a, b)


def _noisy_twin_check(env_id, n, T, hidden, per_env, seed=3, **kwargs):
    a, b = _pair(env_id, n, seed=seed, **kwargs)
    p = _params(a, hidden, per_env, seed + T)
    e = _noise(a, T, seed + 1)
    got = a.rollout_mlp_noisy(p, hidden, e, **TANH)
    _assert_equals_noisy(got, b.noisy_loop(p, hidden, e))
    _eq(a.snapshot().obs, got[2][-1], "snapshot().obs vs obs[T-1]")
    _check_next_step(a, b, p, hidden)
    _close(a, b)


def _summary_check(env_id, n, T, hidden, per_env, seed=9, **kwargs):
    a, b = _pair(env_id, n, seed=seed, **kwargs)
    p = _params(a, hidden, per_env, seed)
    got = a.rollout_mlp(p, hidden, T, summary=True, **TANH)
    full = b.loop(p, hidden, T)
    for name, x, y in zip(("returns", "lengths", "ended"), got, summary_of(*full[1][1:4])):
        _eq(x, y, name)
    _eq(a.snapshot().obs, full[1][0][-1], "snapshot().obs vs obs[T-1]")
    _check_next_step(a, b, p, hidden)
    _close(a, b)
    return got


# ------------------------------------------------------------------------------------------- tanhf itself
def test_tanh_equals_torch_tanh_for_every_float32():
    """All 2^32 bit patterns, 2^28 at a time: b200gym_selftest_tanh against torch.tanh of the same tensor on the same
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
        assert lib.b200gym_selftest_tanh(ctypes.c_void_p(xf.data_ptr()), chunk, ctypes.c_void_p(y.data_ptr()),
                                         stream) == 0
        want = torch.tanh(xf)
        diff = y.view(torch.int32) != want.view(torch.int32)
        k = int(diff.sum())
        if k:
            bad += k
            idx = diff.nonzero()[:4, 0]
            first += [(hex(int(x[i]) & 0xffffffff), hex(int(y.view(torch.int32)[i]) & 0xffffffff),
                       hex(int(want.view(torch.int32)[i]) & 0xffffffff)) for i in idx]
    assert bad == 0, f"{bad} of 2^32 inputs differ from torch.tanh; first (x, engine, torch): {first[:8]}"


def _edge_values():
    """Pre-activations across tanhf's branch points (|x| = 0.6, 9.0109138), +-0, subnormals, +-inf, NaN, +-FLT_MAX and a
    sweep of [-10, 10]."""
    torch = _torch()
    f32 = torch.float32
    v = [0.0, -0.0, float("inf"), float("-inf"), float("nan"), 1e-45, -1e-45, 1.17549421e-38, 1.1754942e-38,
         torch.finfo(f32).max, -torch.finfo(f32).max, torch.finfo(f32).tiny, 1e-20, -1e-3]
    vals = torch.tensor(v, dtype=f32)
    edges = torch.tensor([0.6, 9.0109138], dtype=f32)
    below = torch.nextafter(edges, torch.zeros_like(edges))
    above = torch.nextafter(edges, torch.full_like(edges, float("inf")))
    near = torch.cat([edges, below, above, torch.nextafter(below, torch.zeros_like(below)),
                      torch.nextafter(above, torch.full_like(above, float("inf")))])
    return torch.cat([vals, near, -near, torch.linspace(-10, 10, 4001, dtype=f32)])


@pytest.mark.parametrize("env_id", ["Pendulum-v1", "MountainCarContinuous-v0"])
def test_kernel_tanh_equals_torch_tanh(env_id):
    """Per-env policies with hidden (1,): first-layer weights 0 and bias v, output weight 1 and bias -0.0, so action 0
    is tanh of the unit's sum u, which is v itself unless v is -0.0 (or NaN, whose payload the float32 adds may
    change).  Both entry points, against torch.tanh(u) bit for bit and against the twin's step (which also
    follows a NaN action into the env)."""
    torch = _torch()
    v = _edge_values().to("cuda:0")
    n = v.numel()
    for noisy in (False, True):
        a, b = _pair(env_id, n, seed=8)
        D = a.obs_dim
        p = torch.zeros(n, D + 3, device="cuda:0")
        p[:, D] = v
        p[:, D + 1] = 1.0
        p[:, D + 2] = -0.0
        u = v.clone()
        for k in range(D):
            u = u + 0.0 * b.obs[:, k]
        same = (v != 0) & ~torch.isnan(v)
        _eq(u[same], v[same], "pre-activations")
        assert torch.equal(torch.isnan(u), torch.isnan(v))
        if noisy:
            e = torch.full((1, n, 1), -0.0, device="cuda:0")
            got = a.rollout_mlp_noisy(p, (1,), e, **TANH)
            _assert_equals_noisy(got, b.noisy_loop(p, (1,), e))
            _eq(got[1][0, :, 0], torch.tanh(u), "outputs[0]")
        else:
            got = a.rollout_mlp(p, (1,), 1, **TANH)
            _assert_equals_loop(got, b.loop(p, (1,), 1))
        _eq(got[0][0, :, 0], torch.tanh(u), "actions[0]")
        _assert_same_env(a, b.env)
        _close(a, b)


# ---------------------------------------------------------------------------------------------- the eager twins
@pytest.mark.parametrize("per_env", [False, True], ids=["shared", "per_env"])
@pytest.mark.parametrize("n,T", [(1, 1), (257, 37), (33 * 256 + 5, 2), (4099, 300)])
@pytest.mark.parametrize("hidden", HIDDEN, ids=str)
@pytest.mark.parametrize("env_id", CLASSIC)
def test_tanh_rollout_mlp_equals_eager_loop(env_id, hidden, n, T, per_env):
    _twin_check(env_id, n, T, hidden, per_env)


@pytest.mark.parametrize("per_env", [False, True], ids=["shared", "per_env"])
@pytest.mark.parametrize("n,T", [(1, 1), (257, 37), (33 * 256 + 5, 2), (4099, 300)])
@pytest.mark.parametrize("hidden", HIDDEN, ids=str)
@pytest.mark.parametrize("env_id", CLASSIC)
def test_tanh_rollout_mlp_noisy_equals_eager_loop(env_id, hidden, n, T, per_env):
    _noisy_twin_check(env_id, n, T, hidden, per_env)


@pytest.mark.parametrize("per_env", [False, True], ids=["shared", "per_env"])
@pytest.mark.parametrize("hidden", [(5,), (64, 64)], ids=str)
@pytest.mark.parametrize("env_id", CLASSIC)
def test_tanh_summary_equals_restatement(env_id, hidden, per_env):
    _summary_check(env_id, 33 * 256 + 5, 300, hidden, per_env)
    ended = _summary_check(env_id, 1000, 30, hidden, per_env, max_episode_steps=7)[2]
    assert bool(ended.all())


@pytest.mark.parametrize("env_id", CLASSIC)
def test_tanh_short_time_limit_and_without_autoreset(env_id):
    _twin_check(env_id, 4099, 25, (16, 8), True, max_episode_steps=4)
    _noisy_twin_check(env_id, 2053, 40, (6, 6), True, autoreset=False, max_episode_steps=4)


@pytest.mark.parametrize("per_env", [False, True], ids=["shared", "per_env"])
@pytest.mark.parametrize("hidden", [(5,), (64, 64)], ids=str)
@pytest.mark.parametrize("env_id,kwargs", BOX2D[:3], ids=[b[0] for b in BOX2D[:3]])
def test_box2d_tanh_rollouts_equal_eager_loop(env_id, kwargs, hidden, per_env):
    _twin_check(env_id, 67, 5, hidden, per_env, seed=7, **kwargs)
    _noisy_twin_check(env_id, 67, 5, hidden, per_env, seed=7, **kwargs)
    _summary_check(env_id, 67, 5, hidden, per_env, seed=7, **kwargs)


# ------------------------------------------------------------------------------------------------ CUDA graphs
@pytest.mark.parametrize("per_env", [False, True], ids=["shared", "per_env"])
@pytest.mark.parametrize("env_id", ["CartPole-v1", "Pendulum-v1", "Acrobot-v1"])
def test_captured_tanh_rollouts_replay_equal_eager_calls(env_id, per_env):
    """One graph holds a step(), a tanh rollout_mlp(), a noise draw and a tanh rollout_mlp_noisy(); replay k equals
    eager call k with the parameters copied in place between replays.  The step's outputs are copied inside the graph:
    the second rollout writes its last observations into the buffer the step returned."""
    torch = _torch()
    n, T, k, hidden = 515, 24, 3, (16, 12)
    a, b = _pair(env_id, n)
    p = _params(a, hidden, per_env, 2)
    e = _noise(a, T, 2)
    step_act = b.policy(p, hidden)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        st = [x.clone() for x in a.step(step_act)[:4]]
        out = a.rollout_mlp(p, hidden, T, **TANH)
        if a.discrete:
            u = torch.rand(e.shape, device=e.device).clamp_(min=torch.finfo(torch.float32).tiny)
            e.copy_(-torch.log(-torch.log(u)))
        else:
            e.copy_(0.3 * torch.randn(e.shape, device=e.device))
        noisy = a.rollout_mlp_noisy(p, hidden, e, **TANH)
    e_prev = None
    for r in range(k):
        p2 = _params(a, hidden, per_env, 100 + r)
        p.copy_(p2)
        g.replay()
        o = b.env.step(step_act)
        b.obs = o[0].clone()
        for name, x, y in zip(NAMES, st, o[:4]):
            _eq(x, y, f"replay {r} step {name}")
        _assert_equals_loop(out, b.loop(p2, hidden, T), f"replay {r} ")
        e_now = e.clone()
        _assert_equals_noisy(noisy, b.noisy_loop(p2, hidden, e_now), f"replay {r} noisy ")
        if e_prev is not None:
            assert not torch.equal(e_now, e_prev), "each replay draws new noise"
        e_prev = e_now
    _assert_same_env(a, b.env)
    _close(a, b)


# ------------------------------------------------------------------------------------- the default is ReLU
@pytest.mark.parametrize("per_env", [False, True], ids=["shared", "per_env"])
def test_relu_is_the_default(per_env):
    """activation="relu" gives the bits of a call without the argument, for both entry points."""
    import gym_b200
    n, T, hidden = 4099, 40, (64, 64)
    envs = [gym_b200.vector.make("Acrobot-v1", n) for _ in range(2)]
    for env in envs:
        env.reset(seed=12)
    p = _params(envs[0], hidden, per_env, 12)
    e = _noise(envs[0], T, 12)
    x, y = envs[0].rollout_mlp(p, hidden, T), envs[1].rollout_mlp(p, hidden, T, activation="relu")
    for name, s, t in zip(("actions",) + NAMES, x[:5], y[:5]):
        _eq(s, t, name)
    _eq(x[5]["_final_observation"], y[5]["_final_observation"], "_final_observation")
    x, y = envs[0].rollout_mlp_noisy(p, hidden, e), envs[1].rollout_mlp_noisy(p, hidden, e, activation="relu")
    for name, s, t in zip(("actions", "outputs") + NAMES, x[:6], y[:6]):
        _eq(s, t, name)
    x, y = envs[0].rollout_mlp(p, hidden, T, summary=True), envs[1].rollout_mlp(p, hidden, T, summary=True,
                                                                                  activation="relu")
    for name, s, t in zip(("returns", "lengths", "ended"), x, y):
        _eq(s, t, name)
    _assert_same_env(envs[0], envs[1])
    z = envs[0].rollout_mlp(p, hidden, T, **TANH)[0]
    assert not _torch().equal(z, envs[1].rollout_mlp(p, hidden, T)[0]), "tanh and relu policies act alike"
    for env in envs:
        env.close()


# ------------------------------------------------------------------------------------------- argument checks
def test_bad_activation_is_refused_untouched():
    import gym_b200
    from gym_b200 import error, wrappers
    torch = _torch()
    env = gym_b200.vector.make("CartPole-v1", 64)
    env.reset(seed=1)
    p = _params(env, (8, 4), False, 0)
    e = _noise(env, 3, 0)
    before = _untouched(env)
    for bad in ("Tanh", "TANH", "relu ", "", "sigmoid", None, torch.nn.Tanh, torch.nn.Tanh(), torch.tanh, 0, 1, True,
                b"tanh", ["tanh"]):
        with pytest.raises(ValueError, match="activation"):
            env.rollout_mlp(p, (8, 4), 3, activation=bad)
        _assert_untouched(env, before, f"rollout_mlp {bad!r}")
        with pytest.raises(ValueError, match="activation"):
            env.rollout_mlp(p, (8, 4), 3, summary=True, activation=bad)
        _assert_untouched(env, before, f"rollout_mlp summary {bad!r}")
        with pytest.raises(ValueError, match="activation"):
            env.rollout_mlp_noisy(p, (8, 4), e, activation=bad)
        _assert_untouched(env, before, f"rollout_mlp_noisy {bad!r}")
    with pytest.raises(TypeError):
        env.rollout_mlp(p, (8, 4), 3, False, "tanh")   # keyword only
    with pytest.raises(TypeError):
        env.rollout_mlp_noisy(p, (8, 4), e, "tanh")
    _assert_untouched(env, before, "positional activation")
    for wr in (wrappers.RecordEpisodeStatistics(env), wrappers.NormalizeObservation(env)):
        with pytest.raises(error.Error, match="rollout_mlp"):
            wr.rollout_mlp(p, (8, 4), 3, activation="tanh")
        with pytest.raises(error.Error, match="rollout_mlp_noisy"):
            wr.rollout_mlp_noisy(p, (8, 4), e, activation="tanh")
    _assert_untouched(env, before, "wrappers")
    env.close()


def test_c_entry_points_refuse_unknown_activation_codes():
    """The _act entry points check the activation code themselves, for callers other than the Python layer; the codes
    the header names are accepted."""
    import gym_b200
    torch = _torch()
    env = gym_b200.vector.make("CartPole-v1", 8)
    env.reset(seed=2)
    p = _params(env, (4,), False, 0)
    e = _noise(env, 3, 0)
    vp = ctypes.c_void_p
    outputs = torch.empty_like(e)
    actions = torch.empty(3, 8, dtype=torch.int64, device="cuda:0")
    obs = torch.empty(3, 8, 4, device="cuda:0")
    reward = torch.empty(3, 8, dtype=torch.float64, device="cuda:0")
    flags = torch.empty(2, 3, 8, dtype=torch.uint8, device="cuda:0")
    last = torch.empty(8, 4, device="cuda:0")
    first = env._out[env._flip]["obs"]
    outs = [vp(actions.data_ptr()), vp(obs.data_ptr()), vp(reward.data_ptr()), vp(flags[0].data_ptr()),
            vp(flags[1].data_ptr()), None]
    before = _untouched(env)
    for code in (-1, 2, 7):
        rc = env._lib.b200gym_rollout_mlp_act(env._handle, vp(p.data_ptr()), 0, 1, 4, 0, 3, *outs, None, None, None,
                                              vp(last.data_ptr()), vp(first.data_ptr()), env._stream(), code)
        assert rc != 0, code
        assert b"activation" in env._lib.b200gym_last_error(env._handle)
        rc = env._lib.b200gym_rollout_mlp_noisy_act(env._handle, vp(p.data_ptr()), 0, 1, 4, 0, 3, vp(e.data_ptr()),
                                                    vp(outputs.data_ptr()), *outs, vp(last.data_ptr()),
                                                    vp(first.data_ptr()), env._stream(), code)
        assert rc != 0, code
        assert b"activation" in env._lib.b200gym_last_error(env._handle)
    _assert_untouched(env, before, "refused codes")
    env.close()


# ----------------------------------------------------------------------------------------------- large shapes
@pytest.mark.parametrize("noisy", [False, True], ids=["rollout_mlp", "rollout_mlp_noisy"])
def test_tanh_cartpole_two_to_the_20(noisy):
    """CartPole at 2^20 envs, T = 64, one (64, 64) policy: the shape the benchmark times."""
    torch = _torch()
    n, T, hidden = 1 << 20, 64, (64, 64)
    a, b = _pair("CartPole-v1", n, seed=6)
    p = _params(a, hidden, False, 6, scale=0.3)
    if noisy:
        e = _noise(a, T, 6)
        _assert_equals_noisy(a.rollout_mlp_noisy(p, hidden, e, **TANH), b.noisy_loop(p, hidden, e))
    else:
        _assert_equals_loop(a.rollout_mlp(p, hidden, T, **TANH), b.loop(p, hidden, T))
    _assert_same_env(a, b.env)
    _close(a, b)
    torch.cuda.empty_cache()


def test_tanh_rollout_mlp_noisy_offsets_past_two_to_the_31():
    """CartPole, n = 2^20, T = 520: the noise and outputs pass 2^31 bytes; compared slice by slice with the eager
    loop."""
    torch = _torch()
    n, T, hidden = 1 << 20, 520, (8, 8)
    assert T * n * 2 * 4 > 1 << 31   # K = 2
    a, b = _pair("CartPole-v1", n, seed=5)
    p = _params(a, hidden, False, 5, scale=0.3)
    e = _noise(a, T, 5)
    acts, outputs, obs, rew, term, trunc, infos = a.rollout_mlp_noisy(p, hidden, e, **TANH)
    fin, mask = infos["final_observation"], infos["_final_observation"]
    for t in range(T):
        z, act = b.noisy_policy(p, hidden, e[t])
        o, r, te, tr, inf = b.env.step(act)
        b.obs = o.clone()
        _eq(outputs[t], z, f"outputs[{t}]")
        _eq(acts[t], act, f"actions[{t}]")
        for name, x, y in zip(NAMES, (obs[t], rew[t], term[t], trunc[t]), (o, r, te, tr)):
            _eq(x, y, f"{name}[{t}]")
        m = inf["_final_observation"]
        _eq(mask[t], m, f"mask[{t}]")
        _eq(fin[t][m], inf["final_observation"][m], f"final_observation[{t}]")
    _assert_same_env(a, b.env)
    del acts, outputs, obs, rew, term, trunc, infos, fin, mask, e
    _close(a, b)
    torch.cuda.empty_cache()

