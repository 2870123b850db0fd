"""Host-side logic and the C-ABI boundary, without a GPU."""
import ctypes
import os
import re

import numpy as np
import pytest

import gym_b200
from conftest import ROOT, have_cuda
from gym_b200 import _lib, envs, error, registration, spaces


# ---------------------------------------------------------------- C ABI -----
def _declared_symbols():
    text = open(os.path.join(ROOT, "include", "b200gym.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(b200gym_[a-z_0-9]+)\s*\(", text)))


def test_library_builds_and_exports_every_declared_symbol():
    from gym_b200 import build
    path = build.build()
    assert os.path.exists(path)
    lib = ctypes.CDLL(path)
    declared = _declared_symbols()
    assert len(declared) >= 18
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in include/b200gym.h but not exported"
    # and the Python binding types exactly that set
    assert sorted(_lib.SIGNATURES) == declared


def test_abi_version_4_and_shape_queries_need_no_device():
    lib = _lib.load()
    assert lib.b200gym_version() == 4   # 4: the moments launches take a work buffer (fixed-order sums)
    assert [lib.b200gym_obs_dim(k) for k in range(9)] == [4, 2, 2, 3, 6, 8, 24, 8, 24]
    assert [lib.b200gym_act_dim(k) for k in range(9)] == [0, 0, 1, 1, 0, 0, 4, 2, 4]
    assert [lib.b200gym_num_actions(k) for k in range(9)] == [2, 3, 0, 0, 3, 4, 0, 0, 0]
    assert [lib.b200gym_state_dim(k) for k in range(9)] == [4, 2, 2, 2, 4, 0, 0, 0, 0]
    assert lib.b200gym_obs_dim(99) == -1


@pytest.mark.skipif(have_cuda(), reason="checks the no-GPU failure mode")
def test_no_cpu_fallback_create_fails_loudly():
    lib = _lib.load()
    cfg = _lib.Config(kind=0, max_episode_steps=500, autoreset=1)
    h = ctypes.c_void_p()
    rc = lib.b200gym_create(ctypes.byref(cfg), 8, 0, ctypes.byref(h))
    assert rc != 0 and not h.value
    assert "no CUDA device" in _lib.last_error(None) or "CPU fallback" in _lib.last_error(None)
    with pytest.raises(error.DependencyNotInstalled):
        gym_b200.vector.make("CartPole-v1", 4)
    with pytest.raises(error.DependencyNotInstalled):
        gym_b200.make("CartPole-v1")


def test_create_rejects_bad_arguments_without_touching_a_device():
    lib = _lib.load()
    h = ctypes.c_void_p()
    cfg = _lib.Config(kind=42)
    assert lib.b200gym_create(ctypes.byref(cfg), 8, 0, ctypes.byref(h)) != 0
    assert "kind" in _lib.last_error(None)
    cfg = _lib.Config(kind=0)
    assert lib.b200gym_create(ctypes.byref(cfg), 0, 0, ctypes.byref(h)) != 0
    assert "num_envs" in _lib.last_error(None)


def test_product_code_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "gym_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                text = open(os.path.join(dirpath, f)).read()
                assert "oracle" not in text.lower(), f"{f} mentions the oracle"


# ---------------------------------------------------------------- registry --
def test_registry_matches_reference_table():
    # gym/envs/__init__.py:11-60
    want = {"CartPole-v0": (200, 195.0), "CartPole-v1": (500, 475.0), "MountainCar-v0": (200, -110.0),
            "MountainCarContinuous-v0": (999, 90.0), "Pendulum-v1": (200, None), "Acrobot-v1": (500, -100.0),
            "LunarLander-v2": (1000, 200), "LunarLanderContinuous-v2": (1000, 200), "BipedalWalker-v3": (1600, 300),
            "BipedalWalkerHardcore-v3": (2000, 300)}
    for env_id, (steps, thr) in want.items():
        s = gym_b200.spec(env_id)
        assert s.max_episode_steps == steps and s.reward_threshold == thr
    assert gym_b200.spec("LunarLanderContinuous-v2").kwargs == {"continuous": True}   # gym/envs/__init__.py:62-68
    assert gym_b200.spec("BipedalWalkerHardcore-v3").kwargs == {"hardcore": True}     # gym/envs/__init__.py:79-85
    assert gym_b200.spec("CartPole").id == "CartPole-v1"  # unversioned -> latest (registration.py:548-570)
    with pytest.raises(error.VersionNotFound):
        gym_b200.spec("CartPole-v7")
    with pytest.raises(error.NameNotFound):
        gym_b200.spec("Nope-v0")
    with pytest.raises(error.Error):
        gym_b200.spec("“bad id”")


def test_lunar_lander_constructor_variants_resolve_like_the_reference():
    """LunarLander.__init__ (lunar_lander.py:191-233): continuous -> Box(2) actions, gravity asserted in (-12, 0),
    wind powers outside the recommended range only warn."""
    from gym_b200 import envs
    K = _lib.KIND_LUNARLANDER
    assert envs.resolve_variant(K, {}) == (K, 0)
    assert envs.resolve_variant(K, {"continuous": True}) == (_lib.KIND_LUNARLANDER_CONT, 0)
    assert envs.resolve_variant(_lib.KIND_LUNARLANDER_CONT, {"continuous": False, "enable_wind": True}) == (K, 1)
    assert envs.resolve_params(K, {}) == [-10.0, 15.0, 1.5, 0.0]
    assert envs.resolve_params(K, {"gravity": -3.0, "wind_power": 4.0, "turbulence_power": 0.25})[:3] == [-3.0, 4.0, 0.25]
    for bad in (-12.0, 0.0, 1.0):
        with pytest.raises(AssertionError):
            envs.resolve_params(K, {"gravity": bad})
    with pytest.warns(UserWarning, match="wind_power"):
        envs.resolve_params(K, {"wind_power": 25.0})
    with pytest.warns(UserWarning, match="turbulence_power"):
        envs.resolve_params(K, {"turbulence_power": 2.5})
    with pytest.raises(TypeError):
        envs.resolve_params(K, {"hardcore": True})
    W = _lib.KIND_BIPEDALWALKER
    assert envs.resolve_variant(W, {"hardcore": True}) == (_lib.KIND_BIPEDALWALKER_HARDCORE, 0)
    assert envs.resolve_variant(_lib.KIND_BIPEDALWALKER_HARDCORE, {"hardcore": False}) == (W, 0)
    assert envs.resolve_variant(_lib.KIND_BIPEDALWALKER_HARDCORE, {}) == (_lib.KIND_BIPEDALWALKER_HARDCORE, 0)
    with pytest.raises(TypeError):
        envs.resolve_params(W, {"gravity": -5.0})
    obs_space, act_space = envs.KINDS[_lib.KIND_LUNARLANDER_CONT].spaces(None)
    assert act_space.shape == (2,) and act_space.dtype == np.float32
    assert float(act_space.low.min()) == -1.0 and float(act_space.high.max()) == 1.0 and obs_space.shape == (8,)


def test_reset_option_parsing_follows_reference():
    # classic_control/utils.py:17-46 and tests/envs/test_env_implementation.py:150-215
    k = _lib.KIND_CARTPOLE
    assert envs.parse_reset_bounds(k, None) is None
    assert envs.parse_reset_bounds(k, {}) == (-0.05, 0.05)
    assert envs.parse_reset_bounds(k, {"low": -0.1}) == (-0.1, 0.05)
    assert envs.parse_reset_bounds(k, {"low": "0.01", "high": 0.02}) == (0.01, 0.02)
    with pytest.raises(ValueError):
        envs.parse_reset_bounds(k, {"low": 0.1, "high": 0.0})
    with pytest.raises(ValueError):
        envs.parse_reset_bounds(k, {"low": "x"})
    p = _lib.KIND_PENDULUM
    assert envs.parse_reset_bounds(p, {"x_init": 0.5}) == (0.5, 1.0)
    with pytest.raises(ValueError):
        envs.parse_reset_bounds(p, {"y_init": None})
    assert envs.resolve_params(p, {"g": 9.81})[0] == 9.81
    assert envs.resolve_params(p, {})[0] == 10.0
    with pytest.raises(TypeError):
        envs.resolve_params(k, {"g": 1.0})
    with pytest.raises(ValueError):
        envs.resolve_params(k, {"render_mode": "human"})


# ---------------------------------------------------------------- spaces ----
def test_spaces_shapes_dtypes_and_batching():
    obs, act = envs.KINDS[_lib.KIND_CARTPOLE].spaces(None)
    assert obs.shape == (4,) and obs.dtype == np.float32 and act.n == 2
    np.testing.assert_allclose(obs.high[[0, 2]], [4.8, 0.41887903], rtol=1e-6)
    b = spaces.batch_space(act, 5)
    assert isinstance(b, spaces.MultiDiscrete) and b.shape == (5,) and b.dtype == np.int64
    bo = spaces.batch_space(obs, 5)
    assert bo.shape == (5, 4) and bo.dtype == np.float32
    _, pact = envs.KINDS[_lib.KIND_PENDULUM].spaces(None)
    assert pact.shape == (1,) and pact.low[0] == -2.0 and pact.high[0] == 2.0
    assert spaces.batch_space(pact, 3).shape == (3, 1)


def test_space_sampling_reproduces_numpy_generator_streams():
    # Space.seed -> seeding.np_random; Discrete.sample (discrete.py:81), MultiDiscrete.sample
    # (multi_discrete.py:123), Box.sample (box.py:171-222)
    d = spaces.Discrete(3, seed=7)
    g = np.random.Generator(np.random.PCG64(np.random.SeedSequence(7)))
    assert [d.sample() for _ in range(10)] == [int(g.integers(3)) for _ in range(10)]
    m = spaces.MultiDiscrete([2] * 6, seed=11)
    g = np.random.Generator(np.random.PCG64(np.random.SeedSequence(11)))
    assert np.array_equal(m.sample(), (g.random((6,)) * np.array([2] * 6)).astype(np.int64))
    b = spaces.Box(-2.0, 2.0, shape=(1,), dtype=np.float32, seed=3)
    g = np.random.Generator(np.random.PCG64(np.random.SeedSequence(3)))
    g.normal(size=(0,)); g.exponential(size=(0,)); g.exponential(size=(0,))
    want = g.uniform(low=np.float32(-2.0), high=np.float32(2.0), size=(1,)).astype(np.float32)
    assert np.array_equal(b.sample(), want)


def test_space_membership():
    d = spaces.Discrete(2)
    assert 0 in d and np.int64(1) in d and 2 not in d and -1 not in d and 0.5 not in d
    b = spaces.Box(-1.0, 1.0, shape=(1,), dtype=np.float32)
    assert np.array([0.5], dtype=np.float32) in b
    assert np.array([1.5], dtype=np.float32) not in b
    assert np.array([0.5, 0.1], dtype=np.float32) not in b
    md = spaces.MultiDiscrete([3, 3])
    assert np.array([0, 2]) in md and np.array([0, 3]) not in md and [1, 1] in md


def test_seed_words_validation():
    from gym_b200.vector_env import seed_words
    assert list(seed_words(2**40 + 7)) == [7, 256, 0, 0]
    with pytest.raises(error.Error):
        seed_words(-1)
    with pytest.raises(error.Error):
        seed_words(2**128)
