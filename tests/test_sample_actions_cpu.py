"""Device sampling of the batched action spaces, without a GPU: the generator bookkeeping on the host and the device
source of space_sample_kernel (gym_b200/csrc/space_sample.cuh, rng.cuh), run on the CPU through
tests/hostsim/sample_space.cpp, both against numpy itself."""
import copy

import numpy as np
import pytest

from gym_b200 import error
from gym_b200.spaces import Box, Discrete, MultiDiscrete, batch_space, pcg64_jump, pcg64_skip, pcg64_state
from hostsim import sample_sim as sim

DELTAS = [0, 1, 2, 255, 2 ** 20, 2 ** 40 + 7, 2 ** 64 - 1, 2 ** 64, 2 ** 127 + 5]
SEEDS = [0, 1, 9, 2 ** 40 + 3, 123456789123456789]


def _advanced(seed, delta):
    bg = np.random.PCG64(seed)
    bg.advance(delta)
    return bg.state["state"]["state"]


@pytest.mark.parametrize("seed", SEEDS)
def test_pcg64_jump_equals_numpy_advance(seed):
    words = np.random.PCG64(seed).state["state"]
    for delta in DELTAS:
        want = _advanced(seed, delta)
        assert pcg64_jump(words["state"], words["inc"], delta) == want, delta
        # the device source: square-and-multiply, and the sampling kernel's table walk (64-bit offsets)
        assert sim.pcg64_jump(words["state"], words["inc"], delta) == want, delta
        if delta < 2 ** 64:
            assert sim.pcg64_jump(words["state"], words["inc"], delta, table=True) == want, delta


def test_pcg64_jump_equals_draws():
    g = np.random.Generator(np.random.PCG64(4))
    words = g.bit_generator.state["state"]
    g.random(1000)
    assert pcg64_jump(words["state"], words["inc"], 1000) == g.bit_generator.state["state"]["state"]


def _primed(space, seed, prime):
    space.seed(seed)
    if prime:
        space.np_random.integers(3)   # leaves a buffered 32-bit draw: has_uint32 = 1
    return space


@pytest.mark.parametrize("prime", [False, True])
def test_skip_keeps_the_buffered_uint32(prime):
    space = _primed(MultiDiscrete(np.full(37, 3)), 2, prime)
    twin = copy.deepcopy(space)
    bg = space.np_random.bit_generator
    assert bg.state["has_uint32"] == int(prime)
    pcg64_skip(bg, pcg64_state(bg), 37)
    twin.sample()
    assert bg.state == twin.np_random.bit_generator.state
    # and the next bounded-integer draw (which consumes the buffered word) agrees too
    assert space.np_random.integers(5, size=9).tolist() == twin.np_random.integers(5, size=9).tolist()


def _device_sample(space, rows, cols, n_choices, low=None, high=None, blocks=0):
    """What sample_actions() does, with the kernel replaced by its host build: read the state, sample, skip."""
    bg = space.np_random.bit_generator
    state = pcg64_state(bg)
    out = sim.sample_space(state["state"]["state"], state["state"]["inc"], rows, cols, n_choices, low, high, blocks)
    pcg64_skip(bg, state, out.size)
    return out


# batch sizes around the per-thread vector (2 int64 / 4 float32), the warp (32 vectors), the CTA (256 vectors) and the
# grid sizes b200gym_sample_space picks (one vector per thread up to 264 CTAs, ~8 rounds per thread beyond)
ROWS = [1, 2, 3, 5, 7, 31, 32, 33, 255, 256, 257, 511, 513, 4097, 67583, 67585, 135167, 135169, (1 << 16) + 77]


@pytest.mark.parametrize("n", [2, 3, 4])
@pytest.mark.parametrize("prime", [False, True])
def test_hostsim_multidiscrete_equals_numpy(n, prime):
    for rows in ROWS:
        space = _primed(batch_space(Discrete(n), rows), 17 + rows, prime)
        twin = copy.deepcopy(space)
        got = _device_sample(space, rows, 1, n)
        want = twin.sample()
        assert got.dtype == want.dtype and got.shape == want.shape
        assert np.array_equal(got, want), (n, rows)
        assert space.np_random.bit_generator.state == twin.np_random.bit_generator.state


BOXES = {
    "pm1": (np.full(4, -1.0, np.float32), np.full(4, 1.0, np.float32)),
    "pm2": (np.full(1, -2.0, np.float32), np.full(1, 2.0, np.float32)),
    "mixed2": (np.array([-1.0, 0.25], np.float32), np.array([1.0, 0.3], np.float32)),
    "mixed3": (np.array([-1.0, -2.5, 0.1], np.float32), np.array([1.0, 3.0, 0.7], np.float32)),
    "mixed5": (np.array([-1.0, -2.0, 0.0, -0.3, 5.0], np.float32), np.array([1.0, 2.0, 1e-3, 0.3, 7.5], np.float32)),
}


@pytest.mark.parametrize("bounds", list(BOXES))
@pytest.mark.parametrize("prime", [False, True])
def test_hostsim_box_equals_numpy(bounds, prime):
    low, high = BOXES[bounds]
    single = Box(low, high, dtype=np.float32)
    cols = low.shape[0]
    for rows in ROWS:
        space = _primed(batch_space(single, rows), 3 + rows, prime)
        twin = copy.deepcopy(space)
        got = _device_sample(space, rows, cols, 0, low.astype(np.float64), high.astype(np.float64))
        want = twin.sample()
        assert got.dtype == want.dtype == np.float32 and got.shape == want.shape
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (bounds, rows)
        assert space.np_random.bit_generator.state == twin.np_random.bit_generator.state


@pytest.mark.parametrize("blocks", [1, 2, 3, 7])
def test_hostsim_many_rounds_per_thread(blocks):
    """Small grids: every thread strides over many vectors, the last one ragged."""
    rows = 3 * 256 * 4 * blocks + 5
    low, high = BOXES["mixed3"]
    box = batch_space(Box(low, high, dtype=np.float32), rows)
    box.seed(8)
    twin = copy.deepcopy(box)
    got = _device_sample(box, rows, 3, 0, low.astype(np.float64), high.astype(np.float64), blocks=blocks)
    assert np.array_equal(got.view(np.uint32), twin.sample().view(np.uint32))
    md = batch_space(Discrete(3), rows)
    md.seed(8)
    twin = copy.deepcopy(md)
    assert np.array_equal(_device_sample(md, rows, 1, 3, blocks=blocks), twin.sample())


def test_interleaved_host_and_device_sampling_reproduce_the_host_sequence():
    space = batch_space(Discrete(3), 1000)
    space.seed(0)
    twin = copy.deepcopy(space)
    for r in range(6):
        got = _device_sample(space, 1000, 1, 3) if r % 2 else space.sample()
        assert np.array_equal(got, twin.sample()), r


def test_non_pcg64_generator_is_refused():
    space = MultiDiscrete(np.full(8, 2), seed=np.random.Generator(np.random.Philox(1)))
    with pytest.raises(error.Error):
        pcg64_state(space.np_random.bit_generator)
    space = MultiDiscrete(np.full(8, 2), seed=np.random.Generator(np.random.PCG64DXSM(1)))
    with pytest.raises(error.Error):
        pcg64_state(space.np_random.bit_generator)


def test_unsupported_action_spaces_are_refused():
    """sample_actions' plan is made from the single action space alone; it needs no device."""
    from gym_b200.vector_env import B200VectorEnv

    def plan(single, n=4):
        env = B200VectorEnv.__new__(B200VectorEnv)
        env.single_action_space, env.num_envs, env._sample_cache = single, n, None
        return env._sample_plan()

    assert plan(Discrete(3))[:2] == (3, 1)
    assert plan(Box(-1.0, 1.0, shape=(4,), dtype=np.float32))[:2] == (0, 4)
    for bad in (Discrete(3, start=1), Box(-np.inf, 1.0, shape=(2,), dtype=np.float32),
                Box(-1.0, 1.0, shape=(2,), dtype=np.float64), Box(0, 5, shape=(2,), dtype=np.int64),
                Box(-1.0, 1.0, shape=(2, 2), dtype=np.float32), Box(-1.0, 1.0, shape=(33,), dtype=np.float32)):
        with pytest.raises(error.Error):
            plan(bad)
