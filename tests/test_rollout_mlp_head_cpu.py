"""rollout_mlp_head_kernel's and rollout_mlp_noisy_head_kernel's device source on the CPU
(tests/hostsim/rollout_mlp_head.cpp), against a numpy restatement of the MLP, the squashing head and T launches of
kernel A's driver.

For both classic Box kinds, both heads, both activations, shared and per-env policies, full and summary mode: the
outputs must be the numpy float32 MLP (test_rollout_mlp_cpu.mlp_outputs) of the observation stream; the actions the
documented head, every product and sum one rounded float32 operation; the env outputs and the float64 state, TimeLimit
counters and PCG64 records bit for bit those of T kernel-A steps fed those actions; the summary the float64 fold of the
full outputs.  The host build's tanh and exp are the C library's ``tanhf`` and ``expf``, so the restatement calls those
same functions through ctypes.  The device's ``expf`` is pinned against ``torch.exp`` by
tests/test_gpu_rollout_mlp_head.py, as its ``tanhf`` is by tests/test_gpu_rollout_mlp_tanh.py.
"""
import ctypes
import ctypes.util

import numpy as np
import pytest

import test_rollout_mlp_cpu as mlp_cpu
from hostsim.rollout_mlp_head_sim import MlpHeadRolloutSim
from test_rollout_linear_cpu import _assert_same, _config, summary_of
from test_rollout_mlp_tanh_cpu import libm_tanhf

ENV_IDS = ["Pendulum-v1", "MountainCarContinuous-v0"]
HEADS = ["tanh", "tanh_normal"]
HIDDEN = [(1,), (3, 7), (64, 64)]
# (N, T): one env, N not a multiple of 256 over several CTAs with short rollouts, a long rollout at a small N
SHAPES = [(1, 1), (257, 9), (513, 2), (67, 60)]

f32 = np.float32
_libm = ctypes.CDLL(ctypes.util.find_library("m"))
_libm.expf.restype = ctypes.c_float
_libm.expf.argtypes = [ctypes.c_float]


def libm_expf(x):
    """The C library's expf, elementwise over a float32 array."""
    x = np.asarray(x, dtype=np.float32)
    return np.fromiter(map(_libm.expf, x.ravel().tolist()), dtype=np.float32, count=x.size).reshape(x.shape)


def bounds_of(env_id):
    """float32 (low, high, scale, bias) of the action space, scale and bias as CleanRL computes them."""
    single = _config(env_id)[3]
    low, high = f32(single.low[0]), f32(single.high[0])
    return np.array([low, high, f32(f32(high - low) / f32(2)), f32(f32(high + low) / f32(2))], dtype=np.float32)


def outputs(params, hidden, obs, K, activation):
    """test_rollout_mlp_cpu.mlp_outputs with the hidden layers' activation `activation`."""
    if activation == "relu":
        return mlp_cpu.mlp_outputs(params, hidden, obs, K)
    relu = mlp_cpu.relu
    mlp_cpu.relu = libm_tanhf
    try:
        return mlp_cpu.mlp_outputs(params, hidden, obs, K)
    finally:
        mlp_cpu.relu = relu


def log_std(s):
    """The SAC head's ls = -5 + 3.5 * (tanh(s) + 1), one rounded float32 operation at a time."""
    return f32(-5) + f32(3.5) * (libm_tanhf(s) + f32(1))


def head_action(z, e, head, bounds):
    """The documented head in numpy float32: z (n, K), e (n, A) or None for the deterministic action -> (n, A)."""
    low, high, scale, bias = bounds
    A = z.shape[1] // (2 if head == "tanh_normal" else 1)
    with np.errstate(all="ignore"):
        if head == "tanh_normal" and e is not None:
            x = z[:, :A] + e * libm_expf(log_std(z[:, A:]))
            return libm_tanhf(x) * scale + bias
        v = libm_tanhf(z[:, :A]) * scale + bias
        if e is None:
            return v
        v = v + e
        return np.where(v < low, low, np.where(v > high, high, v))   # NaN stays NaN


def _assert_same_nan(got, want, what):
    """Bit for bit, except that a NaN need only be NaN: numpy and the host build may return either NaN operand of a sum
    of two NaNs, and so may two compilations of one step once a NaN action has made the state NaN."""
    got, want = np.asarray(got), np.asarray(want)
    if got.dtype.kind != "f":
        return _assert_same(got, want, what)
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan), f"{what}: NaN positions differ"
    _assert_same(np.where(nan, 0, got).astype(got.dtype), np.where(nan, 0, want).astype(want.dtype), what)


_assert_actions = _assert_same_nan


class _Case:
    """A head-rollout batch, a kernel-A twin and a summary-mode twin, reset alike."""

    def __init__(self, env_id, N, seed, head, activation, **kw):
        self.kind, mes, param0, single = _config(env_id)
        mes = kw.pop("max_episode_steps", mes)
        self.head, self.activation, self.bounds = head, activation, bounds_of(env_id)
        self.ro, self.step, self.summ = [MlpHeadRolloutSim(self.kind, N, max_episode_steps=mes, param0=param0, **kw)
                                         for _ in range(3)]
        self.obs = self.ro.reset(seed)
        for sim in (self.step, self.summ):
            _assert_same(sim.reset(seed), self.obs, "reset")
        self.A = int(single.shape[0])
        self.K = self.A * (2 if head == "tanh_normal" else 1)

    def params(self, rng, hidden, per_env, scale=0.5):
        lead = (self.ro.n,) if per_env else ()
        P = mlp_cpu.param_count(self.ro.obs_dim, hidden, self.K)
        return (scale * rng.standard_normal(lead + (P,))).astype(np.float32)

    def noise(self, rng, T, scale=1.0):
        return (scale * rng.standard_normal((T, self.ro.n, self.A))).astype(np.float32)

    def _check_env(self, got, outs, last, k0):
        for k, name in enumerate(("obs", "reward", "terminated", "truncated", "final_obs")):
            _assert_same_nan(got[k0 + k], np.stack([o[k] for o in outs]), name)
        _assert_same(last, got[k0][-1], "last observation buffer")
        for x, y, name in zip(self.ro.get_state(), self.step.get_state(), ("state", "elapsed", "flags", "rng")):
            _assert_same_nan(x, y, name)

    def check(self, params, hidden, T):
        """The deterministic head, full mode against the restatement and kernel A, summary mode against the fold."""
        ro = self.ro
        last = np.zeros((ro.n, ro.obs_dim), dtype=np.float32)
        got = ro.rollout_mlp_head(params, hidden, T, self.activation, self.head, self.bounds, last_obs=last)
        outs = []
        for t in range(T):
            z = outputs(params, hidden, self.obs, self.K, self.activation)
            _assert_actions(got[0][t], head_action(z, None, self.head, self.bounds), f"actions[{t}]")
            outs.append(self.step.step(got[0][t]))
            self.obs = outs[-1][0]
        self._check_env(got, outs, last, 1)
        last_s = np.zeros_like(last)
        summ = self.summ.rollout_mlp_head(params, hidden, T, self.activation, self.head, self.bounds, summary=True,
                                          last_obs=last_s)
        for x, y, name in zip(summ, summary_of(got[2], got[3], got[4]), ("returns", "lengths", "ended")):
            _assert_same_nan(x, y, name)
        _assert_same_nan(last_s, last, "summary: last observation buffer")
        for x, y, name in zip(self.summ.get_state(), ro.get_state(), ("state", "elapsed", "flags", "rng")):
            _assert_same_nan(x, y, f"summary: {name}")
        return got

    def check_noisy(self, params, hidden, noise):
        """The head with noise: outputs, actions, env outputs and state; the summary twin is stepped alike so that
        check() can follow."""
        ro = self.ro
        T = noise.shape[0]
        last = np.zeros((ro.n, ro.obs_dim), dtype=np.float32)
        got = ro.rollout_mlp_noisy_head(params, hidden, noise, self.activation, self.head, self.bounds, last_obs=last)
        assert got[1].shape == (T, ro.n, self.K) and got[0].shape == (T, ro.n, self.A)
        outs = []
        for t in range(T):
            z = outputs(params, hidden, self.obs, self.K, self.activation)
            _assert_same(got[1][t], z, f"outputs[{t}]")
            _assert_actions(got[0][t], head_action(z, noise[t], self.head, self.bounds), f"actions[{t}]")
            outs.append(self.step.step(got[0][t]))
            self.summ.step(got[0][t])
            self.obs = outs[-1][0]
        self._check_env(got, outs, last, 2)
        return got


def test_libm_expf_is_not_numpys():
    """The restatement's exp is the C library's: numpy's float32 exp differs from it on some inputs, so a test that
    passed with either would not pin which one the host build calls."""
    x = np.random.default_rng(0).uniform(-10, 10, 1 << 18).astype(np.float32)
    assert not np.array_equal(libm_expf(x).view(np.int32), np.exp(x).view(np.int32))


def test_bounds_are_cleanrls():
    assert bounds_of("Pendulum-v1").tolist() == [-2.0, 2.0, 2.0, 0.0]
    assert bounds_of("MountainCarContinuous-v0").tolist() == [-1.0, 1.0, 1.0, 0.0]


@pytest.mark.parametrize("per_env", [False, True])
@pytest.mark.parametrize("N,T", SHAPES)
@pytest.mark.parametrize("hidden", HIDDEN)
@pytest.mark.parametrize("activation", ["relu", "tanh"])
@pytest.mark.parametrize("head", HEADS)
@pytest.mark.parametrize("env_id", ENV_IDS)
def test_head_rollouts_equal_policy_and_steps(env_id, head, activation, hidden, N, T, per_env):
    """Deterministic (full and summary), then noisy, then deterministic again: each call starts from the state the one
    before left."""
    c = _Case(env_id, N, 8000 + T + N, head, activation)
    rng = np.random.default_rng(T * 7919 + N + len(hidden))
    c.check(c.params(rng, hidden, per_env, scale=1.0), hidden, T)
    c.check_noisy(c.params(rng, hidden, per_env, scale=1.0), hidden, c.noise(rng, T))
    c.check(c.params(rng, hidden, per_env, scale=1.0), hidden, T)


def _special():
    f = np.finfo(np.float32)
    return np.array([0.0, -0.0, f.smallest_subnormal, -f.smallest_subnormal, f.tiny, -f.tiny, np.inf, -np.inf,
                     np.nan, -np.nan, 1.0, -1.0, 20.0, -20.0, f.max, -f.max], dtype=np.float32)


def _output_params(n, D, K, bias):
    """Per-env hidden (1,) policies whose K outputs are exactly bias[i] (n, K): the hidden unit is +0.0 under either
    activation, and its output weights -0.0, so z = bias + (-0.0 * +0.0) = bias, signed zeros included."""
    P = mlp_cpu.param_count(D, (1,), K)
    params = np.zeros((n, P), dtype=np.float32)
    params[:, D + 1:D + 1 + K] = -0.0     # W2 (K, 1)
    params[:, D + 1 + K:] = bias          # b2 (K,)
    return params


@pytest.mark.parametrize("activation", ["relu", "tanh"])
@pytest.mark.parametrize("head", HEADS)
@pytest.mark.parametrize("env_id", ENV_IDS)
def test_special_outputs_and_noise(env_id, head, activation):
    """z (and for SAC m and s) at +-0, subnormals, +-tiny, +-inf, NaN, +-1, +-20 and +-FLT_MAX, against noise at the
    same values, every pair once: the outputs keep their bits and the head's actions follow the restatement."""
    v = _special()
    A = 1
    K = A * (2 if head == "tanh_normal" else 1)
    m, e = np.meshgrid(v, v, indexing="ij")
    m, e = m.ravel(), e.ravel()
    n = m.size
    bias = np.stack([m, np.roll(m, 7)], axis=1)[:, :K]   # s walks the same values against other m
    kind, mes, param0, _ = _config(env_id)
    c = _Case(env_id, n, 21, head, activation)
    params = _output_params(n, c.ro.obs_dim, K, bias)
    got = c.check_noisy(params, (1,), e.reshape(1, n, A))
    _assert_same(got[1][0], bias, "outputs")
    got = c.check(params, (1,), 1)


@pytest.mark.parametrize("env_id", ENV_IDS)
def test_td3_actions_at_and_beyond_the_bounds(env_id):
    """tanh(z) * scale + bias + e lands exactly on low / high, just inside and beyond them: the clamp gives the bound
    itself for everything beyond and keeps the rest; the +0.0 bias has already made a -0.0 tanh +0.0."""
    b = bounds_of(env_id)
    low, high = b[0], b[1]
    z = np.array([0.0, 0.0, 0.0, 0.0, 20.0, -20.0, 20.0, -20.0, 0.0, 0.0, -0.0, 0.0], dtype=np.float32)
    e = np.array([high, low, np.nextafter(high, f32(0)), np.nextafter(high, f32(np.inf)), 0.0, -0.0, 1e-7, -1e-7,
                  np.inf, -np.inf, -0.0, np.nan], dtype=np.float32)
    n = z.size
    c = _Case(env_id, n, 23, "tanh", "relu")
    got = c.check_noisy(_output_params(n, c.ro.obs_dim, 1, z[:, None]), (1,), e.reshape(1, n, 1))
    a = got[0][0, :, 0]
    want = np.array([high, low, np.nextafter(high, f32(0)), high, high, low, high, low, high, low, 0.0, np.nan],
                    dtype=np.float32)
    assert np.array_equal(np.isnan(a), np.isnan(want))
    _assert_same(a[:-1], want[:-1], "clamped actions")


@pytest.mark.parametrize("env_id", ENV_IDS)
def test_sac_log_std_saturates_at_its_bounds(env_id):
    """tanh(s) = +-1 gives ls = 2 and -5 exactly, so the standard deviation is expf(2) and expf(-5)."""
    s = np.array([20.0, -20.0, np.inf, -np.inf], dtype=np.float32)
    _assert_same(log_std(s), np.array([2.0, -5.0, 2.0, -5.0], dtype=np.float32), "ls")
    n = s.size
    eps = np.array([1.0, 1.0, -0.5, 3.0], dtype=np.float32)
    c = _Case(env_id, n, 25, "tanh_normal", "tanh")
    bias = np.stack([np.full(n, 0.25, dtype=np.float32), s], axis=1)
    got = c.check_noisy(_output_params(n, c.ro.obs_dim, 2, bias), (1,), eps.reshape(1, n, 1))
    std = libm_expf(np.array([2.0, -5.0, 2.0, -5.0], dtype=np.float32))
    want = libm_tanhf(f32(0.25) + eps * std) * bounds_of(env_id)[2] + bounds_of(env_id)[3]
    _assert_same(got[0][0, :, 0], want, "actions")


@pytest.mark.parametrize("head", HEADS)
@pytest.mark.parametrize("env_id", ENV_IDS)
def test_episodes_ending_at_the_first_and_last_step(env_id, head):
    """max_episode_steps = 1: every episode ends at t = 0 and the policy goes on from the reset observation; a limit
    of T: every episode ends at t = T - 1."""
    rng = np.random.default_rng(5)
    c = _Case(env_id, 257, 27, head, "tanh", max_episode_steps=1)
    got = c.check(c.params(rng, (4, 12), True), (4, 12), 5)
    assert got[4].all()
    c.check_noisy(c.params(rng, (4, 12), False), (4, 12), c.noise(rng, 5))
    T = 6
    c = _Case(env_id, 257, 29, head, "relu", max_episode_steps=T)
    got = c.check(c.params(rng, (8,), False), (8,), T)
    assert got[4][T - 1].all() and not got[4][:T - 1].any()
