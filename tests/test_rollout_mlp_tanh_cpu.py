"""The tanh instantiations of rollout_mlp_kernel's and rollout_mlp_noisy_kernel's device source on the CPU
(tests/hostsim/rollout_mlp_tanh.cpp), against the numpy restatements of test_rollout_mlp_cpu.py and
test_rollout_mlp_noisy_cpu.py with tanh in place of their ReLU.

The host build's activation is the C library's ``tanhf``, so the restatement calls that same function through ctypes,
not ``np.tanh`` (numpy has a float32 tanh of its own).  This checks the wiring: every hidden unit, and only the hidden
units, goes through the activation the template selects, in every driver and mode.  The device's ``tanhf`` is checked
against ``torch.tanh`` by tests/test_gpu_rollout_mlp_tanh.py.
"""
import ctypes
import ctypes.util

import numpy as np
import pytest

import test_rollout_mlp_cpu as mlp_cpu
import test_rollout_mlp_noisy_cpu as noisy_cpu
from hostsim.rollout_mlp_tanh_sim import MlpTanhRolloutSim
from test_rollout_linear_cpu import ENV_IDS, _assert_same, _config

HIDDEN = [(1,), (64,), (3, 7), (64, 64)]
# (N, T): one env, N not a multiple of 256 over several CTAs with short rollouts, a long rollout at a small N
SHAPES = [(1, 1), (257, 9), (513, 2), (67, 60)]

_libm = ctypes.CDLL(ctypes.util.find_library("m"))
_libm.tanhf.restype = ctypes.c_float
_libm.tanhf.argtypes = [ctypes.c_float]


def libm_tanhf(z):
    """The C library's tanhf, elementwise over a float32 array."""
    z = np.asarray(z, dtype=np.float32)
    return np.fromiter(map(_libm.tanhf, z.ravel().tolist()), dtype=np.float32, count=z.size).reshape(z.shape)


@pytest.fixture
def tanh(monkeypatch):
    """The ReLU restatements and host builds of the existing tests, switched to tanh: their activation becomes
    libm_tanhf, and their rollout simulators the tanh launches."""
    monkeypatch.setattr(mlp_cpu, "relu", libm_tanhf)
    monkeypatch.setattr(mlp_cpu, "MlpRolloutSim", MlpTanhRolloutSim)
    monkeypatch.setattr(noisy_cpu, "MlpNoisyRolloutSim", MlpTanhRolloutSim)


def test_libm_tanhf_is_not_numpys():
    """The restatement's tanh is the C library's: it differs from np.tanh's float32 on some inputs, so a test that
    passed with either would not pin which one the host build calls."""
    x = np.random.default_rng(0).uniform(-10, 10, 1 << 16).astype(np.float32)
    assert not np.array_equal(libm_tanhf(x).view(np.int32), np.tanh(x).view(np.int32))


@pytest.mark.parametrize("per_env", [False, True])
@pytest.mark.parametrize("N,T", SHAPES)
@pytest.mark.parametrize("hidden", HIDDEN)
@pytest.mark.parametrize("env_id", ENV_IDS)
def test_tanh_mlp_rollout_equals_policy_and_steps(tanh, env_id, hidden, N, T, per_env):
    """Full and summary mode, two calls in a row."""
    c = mlp_cpu._Case(env_id, N, seed=6000 + T + N)
    assert isinstance(c.ro, MlpTanhRolloutSim)
    rng = np.random.default_rng(T * 7919 + N + len(hidden))
    for _ in range(2):
        c.check(c.params(rng, hidden, per_env), hidden, T)


@pytest.mark.parametrize("per_env", [False, True])
@pytest.mark.parametrize("N,T", SHAPES)
@pytest.mark.parametrize("hidden", HIDDEN)
@pytest.mark.parametrize("env_id", ENV_IDS)
def test_tanh_noisy_rollout_equals_policy_and_steps(tanh, env_id, hidden, N, T, per_env):
    c = noisy_cpu._Case(env_id, N, seed=7000 + T + N)
    assert isinstance(c.ro, MlpTanhRolloutSim)
    rng = np.random.default_rng(T * 7919 + N + len(hidden))
    for _ in range(2):
        c.check(c.params(rng, hidden, per_env), hidden, c.noise(rng, T))


@pytest.mark.parametrize("env_id", ["CartPole-v1", "Pendulum-v1"])
def test_tanh_rollout_truncates_and_resets(tanh, env_id):
    c = mlp_cpu._Case(env_id, 257, seed=15, max_episode_steps=4)
    got = c.check(c.params(np.random.default_rng(3), (4, 12), True), (4, 12), 37)
    assert (got[3] | got[4]).any(axis=0).all()


def _special_inputs():
    f = np.float32
    edges = [f(0.6), f(9.0109138)]
    v = [f(0.0), -f(0.0), f(np.inf), -f(np.inf), f(np.nan), np.finfo(f).max, -np.finfo(f).max,
         np.finfo(f).smallest_subnormal, -np.finfo(f).smallest_subnormal, np.finfo(f).tiny, f(1e-20), f(-1e-3)]
    for e in edges:
        for x in (e, np.nextafter(e, f(0)), np.nextafter(e, f(np.inf))):
            v += [f(x), -f(x)]
    return np.array(v, dtype=np.float32)


def test_tanh_of_special_pre_activations():
    """hidden (1,), first-layer weights 0 and bias v, output weight 1 and bias -0.0: the action is tanhf of the unit's
    sum (v itself unless v is -0.0), for v at tanhf's branch points, +-0, subnormals, +-inf, NaN and +-FLT_MAX."""
    v = _special_inputs()
    n = len(v)
    kind, mes, param0, _ = _config("MountainCarContinuous-v0")
    sim = MlpTanhRolloutSim(kind, n, max_episode_steps=mes, param0=param0)
    obs = sim.reset(5)
    D = sim.obs_dim
    params = np.zeros((n, D + 3), dtype=np.float32)
    params[:, D] = v                 # b1
    params[:, D + 1] = 1.0           # W2
    params[:, D + 2] = -0.0          # b2
    acts = sim.rollout_mlp(params, (1,), 1)[0]
    u = v.copy()
    for k in range(D):
        u = u + np.float32(0.0) * obs[:, k]
    nonzero = v != 0
    assert np.array_equal(u[nonzero].view(np.int32), v[nonzero].view(np.int32))
    _assert_same(acts[0, :, 0], libm_tanhf(u), "actions")

