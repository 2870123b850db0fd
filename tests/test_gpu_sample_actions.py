"""``B200VectorEnv.sample_actions()``: ``envs.action_space.sample()`` drawn on the device (space_sample_kernel), bit for
bit, with the space's generator left where the host ``sample()`` leaves it."""
import copy
import os

import numpy as np
import pytest

from conftest import GOLDEN
from oracle import ref_gym

pytestmark = pytest.mark.gpu
needs_reference = pytest.mark.skipif(ref_gym.reference_path() is None,
                                     reason="the reference is not installed in oracle/_ref")

IDS = ["CartPole-v0", "CartPole-v1", "MountainCar-v0", "MountainCarContinuous-v0", "Pendulum-v1", "Acrobot-v1",
       "LunarLander-v2", "LunarLanderContinuous-v2", "BipedalWalker-v3", "BipedalWalkerHardcore-v3"]
CLASSIC = ["CartPole-v1", "MountainCar-v0", "MountainCarContinuous-v0", "Pendulum-v1", "Acrobot-v1"]
BASE_SIZES = [1, 7, 31, 32, 33, 255, 256, 257, 4097, (1 << 16) + 77]
ACT_DIM = {"MountainCarContinuous-v0": 1, "Pendulum-v1": 1, "LunarLanderContinuous-v2": 2, "BipedalWalker-v3": 4,
           "BipedalWalkerHardcore-v3": 4}


def _boundaries(env_id):
    """Batch sizes on each side of the kernel's boundaries (space_sample.cuh): a thread's 16-byte vector (2 int64 /
    4 float32), a CTA's 256 vectors, and the grid b200gym_sample_space picks -- one vector per thread up to 264 CTAs
    (67584 vectors), then 264 CTAs with several rounds, then ~8 rounds per thread (beyond 2112 * 256 vectors)."""
    cols = ACT_DIM.get(env_id, 0)
    per_vec = 2 if cols == 0 else 4
    rows_per = lambda vectors: vectors * per_vec // max(cols, 1)   # noqa: E731
    sizes = {rows_per(1) - 1, rows_per(1) + 1, rows_per(256) - 1, rows_per(256) + 1}
    if env_id in ("CartPole-v1", "Pendulum-v1", "BipedalWalker-v3"):
        sizes |= {rows_per(67584) - 1, rows_per(67584) + 1}
    if env_id == "CartPole-v1":
        sizes |= {rows_per(2112 * 256) - 1, rows_per(2112 * 256) + 3, 1 << 20}
    if env_id.startswith(("LunarLander", "BipedalWalker")):
        sizes.add(1 << 16)   # the size bench.py times
    return sorted(s for s in sizes if s > 0)


def _assert_same(got, want, what=""):
    import torch
    assert isinstance(got, torch.Tensor) and got.is_cuda
    got = got.cpu().numpy()
    want = np.asarray(want)
    assert got.dtype == want.dtype and got.shape == want.shape, (what, got.dtype, got.shape, want.dtype, want.shape)
    if got.dtype == np.float32:
        got, want = got.view(np.uint32), want.view(np.uint32)
    if not np.array_equal(got, want):
        bad = np.argwhere(got != want)
        raise AssertionError(f"{what}: {len(bad)} elements differ, first at {bad[0]}")


def _check_rounds(envs, seed, rounds=3, what=""):
    envs.action_space.seed(seed)
    twin = copy.deepcopy(envs.action_space)
    for r in range(rounds):
        _assert_same(envs.sample_actions(), twin.sample(), f"{what} round {r}")
    assert envs.action_space.np_random.bit_generator.state == twin.np_random.bit_generator.state


@pytest.mark.parametrize("env_id", IDS)
def test_sample_actions_equals_host_sample(env_id):
    import gym_b200
    for n in sorted(set(BASE_SIZES) | set(_boundaries(env_id))):
        envs = gym_b200.vector.make(env_id, n)
        _check_rounds(envs, seed=n, what=f"{env_id} n={n}")
        envs.close()


@pytest.mark.parametrize("env_id", ["CartPole-v1", "Pendulum-v1", "BipedalWalker-v3"])
def test_interleaved_host_and_device_sampling(env_id):
    import gym_b200
    envs = gym_b200.vector.make(env_id, 1000)
    envs.action_space.seed(3)
    twin = copy.deepcopy(envs.action_space)
    for r in range(8):
        got = envs.sample_actions() if r % 3 != 1 else envs.action_space.sample()
        want = twin.sample()
        if r % 3 == 1:
            assert np.array_equal(np.asarray(got), np.asarray(want))
        else:
            _assert_same(got, want, f"round {r}")
    assert envs.action_space.np_random.bit_generator.state == twin.np_random.bit_generator.state
    envs.close()


@pytest.mark.parametrize("env_id", ["Acrobot-v1", "LunarLanderContinuous-v2"])
def test_buffered_uint32_is_kept(env_id):
    import gym_b200
    envs = gym_b200.vector.make(env_id, 513)
    envs.action_space.seed(4)
    envs.action_space.np_random.integers(7)   # leaves has_uint32 = 1
    assert envs.action_space.np_random.bit_generator.state["has_uint32"] == 1
    twin = copy.deepcopy(envs.action_space)
    _assert_same(envs.sample_actions(), twin.sample())
    assert envs.action_space.np_random.bit_generator.state == twin.np_random.bit_generator.state
    assert envs.action_space.np_random.integers(100, size=5).tolist() == twin.np_random.integers(100, size=5).tolist()
    envs.close()


@pytest.mark.parametrize("env_id", CLASSIC)
def test_against_the_references_batch_sample(env_id):
    """tests/golden/reference/spaces.npz: batch_space(action_space, 7) seeded with 9 and sampled by the reference."""
    import gym_b200
    z = np.load(os.path.join(GOLDEN, "reference", "spaces.npz"))
    envs = gym_b200.vector.make(env_id, 7)
    envs.action_space.seed(9)
    _assert_same(envs.sample_actions(), z[f"{env_id}/batch_sample"], env_id)
    envs.close()


def _random_loop(env_id, n, steps, device):
    """The reference's seeded random-action loop: reset(seed=0), action_space.seed(0), `steps` x
    step(action_space.sample()) -- with the actions drawn on the device or on the host."""
    import gym_b200
    import torch
    envs = gym_b200.vector.make(env_id, n)
    obs, _ = envs.reset(seed=0)
    envs.action_space.seed(0)
    trace = [obs.clone()]
    for _ in range(steps):
        a = envs.sample_actions() if device else envs.action_space.sample()
        o, r, te, tr, info = envs.step(a)
        trace += [torch.as_tensor(a, device=envs.device).clone(), o.clone(), r.clone(), te.clone(), tr.clone()]
    state = envs.action_space.np_random.bit_generator.state
    envs.close()
    return trace, state


@pytest.mark.parametrize("env_id, n, steps", [("CartPole-v1", 4, 1000), ("Pendulum-v1", 4096, 1000),
                                              ("LunarLanderContinuous-v2", 1024, 300)])
def test_seeded_random_action_loop(env_id, n, steps):
    import torch
    dev, dev_state = _random_loop(env_id, n, steps, device=True)
    host, host_state = _random_loop(env_id, n, steps, device=False)
    assert dev_state == host_state
    for k, (a, b) in enumerate(zip(dev, host)):
        assert a.dtype == b.dtype and a.shape == b.shape and torch.equal(a, b), f"entry {k} differs"


def test_non_default_stream_feeds_step():
    import gym_b200
    import torch
    n = 1 << 14
    a_env, b_env = gym_b200.vector.make("Pendulum-v1", n), gym_b200.vector.make("Pendulum-v1", n)
    a_env.reset(seed=5)
    b_env.reset(seed=5)
    a_env.action_space.seed(6)
    b_env.action_space.seed(6)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(5):
            act = a_env.sample_actions()
            obs_a, rew_a, *_ = a_env.step(act)
        obs_a, rew_a = obs_a.clone(), rew_a.clone()
    for _ in range(5):
        obs_b, rew_b, *_ = b_env.step(b_env.action_space.sample())
    torch.cuda.current_stream().wait_stream(side)
    assert torch.equal(obs_a, obs_b) and torch.equal(rew_a, rew_b)
    a_env.close()
    b_env.close()


def test_through_record_episode_statistics():
    import gym_b200
    from gym_b200.wrappers import RecordEpisodeStatistics
    env = RecordEpisodeStatistics(gym_b200.vector.make("CartPole-v1", 300))
    env.reset(seed=0)
    env.action_space.seed(2)
    twin = copy.deepcopy(env.action_space)
    for _ in range(40):
        a = env.sample_actions()
        _assert_same(a, twin.sample())
        env.step(a)
    env.close()


def test_numpy_backend_returns_the_host_sample():
    import gym_b200
    envs = gym_b200.vector.make("Acrobot-v1", 33, backend="numpy")
    envs.reset(seed=0)
    envs.action_space.seed(1)
    twin = copy.deepcopy(envs.action_space)
    a = envs.sample_actions()
    assert isinstance(a, np.ndarray) and np.array_equal(a, twin.sample())
    envs.step(a)
    envs.close()


def test_errors_on_a_real_env():
    import gym_b200
    from gym_b200 import error, spaces
    envs = gym_b200.vector.make("CartPole-v1", 64)
    envs.action_space = spaces.MultiDiscrete(np.full(64, 2), seed=np.random.Generator(np.random.Philox(1)))
    twin = copy.deepcopy(envs.action_space)
    with pytest.raises(error.Error):
        envs.sample_actions()
    assert np.array_equal(envs.action_space.sample(), twin.sample())   # the refused call drew nothing
    envs.action_space = spaces.MultiDiscrete(np.full(65, 2))   # not the batch of this env's space any more
    with pytest.raises(error.Error):
        envs.sample_actions()
    envs.action_space = spaces.Box(-1.0, 1.0, shape=(64,), dtype=np.float32)
    with pytest.raises(error.Error):
        envs.sample_actions()
    envs.close()
    with pytest.raises(error.ClosedEnvironmentError):
        envs.sample_actions()
    p = gym_b200.vector.make("Pendulum-v1", 8)
    p.single_action_space = spaces.Box(-np.inf, np.inf, shape=(1,), dtype=np.float32)   # not a bounded Box
    with pytest.raises(error.Error):
        p.sample_actions()
    p.close()


@needs_reference
@pytest.mark.parametrize("env_id", IDS)
def test_gym_vector_env_with_the_references_spaces(env_id):
    """GymVectorEnv's spaces are the reference's gym.spaces classes; only .np_random.bit_generator is used."""
    gym = ref_gym.import_reference()
    from gym_b200.gym_compat import GymVectorEnv
    for n in (1, 33, 257, 4097):
        envs = GymVectorEnv(env_id, n)
        assert type(envs.action_space).__module__.startswith("gym.spaces")
        assert isinstance(envs.action_space, gym.spaces.Space)
        _check_rounds(envs, seed=n + 1, what=f"{env_id} n={n}")
        envs.close()
    # an unseeded space is seeded lazily by the first sample, as sample() would seed it
    envs = GymVectorEnv(env_id, 16)
    a = envs.sample_actions()
    assert tuple(a.shape) == tuple(envs.action_space.shape)
    envs.close()
