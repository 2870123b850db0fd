"""The action-space stream of captured sample_actions() calls, without a GPU: the device source of
space_sample_stream_kernel (gym_b200/csrc/space_sample.cuh) run on the CPU through tests/hostsim/sample_stream.cpp,
consecutive calls on one record against numpy's Generator, element for element and state for state."""
import numpy as np
import pytest

from gym_b200.spaces import Box, Discrete, batch_space
from hostsim import sample_stream_sim as sim

# (rows, single space): MultiDiscrete and Box batches from one CTA to grids of several hundred CTAs, ragged tails
CASES = [
    (1, Discrete(2)), (3, Discrete(3)), (1000, Discrete(4)), (70001, Discrete(2)),
    (1, Box(-2.0, 2.0, (1,), np.float32)), (777, Box(-1.0, 1.0, (2,), np.float32)),
    (20001, Box(-1.0, 1.0, (4,), np.float32)), (301, Box(-3.5, 0.25, (3,), np.float32)),
]


def _plan(single):
    if isinstance(single, Discrete):
        return 1, int(single.n), None, None
    return single.shape[0], 0, single.low.astype(np.float64), single.high.astype(np.float64)


def _state(space):
    st = space.np_random.bit_generator.state["state"]
    return st["state"], st["inc"]


def _record_state(record):
    w = [int(x) for x in record[:4]]
    return (w[0] << 64) | w[1], (w[2] << 64) | w[3]


@pytest.mark.parametrize("rows,single", CASES, ids=[f"{r}x{s}" for r, s in CASES])
def test_consecutive_calls_continue_the_stream(rows, single):
    """The first call takes the host generator as its override, the next ones read the record the previous call left:
    each batch is the next `space.sample()`, and the record ends where the generator does."""
    cols, n_choices, low, high = _plan(single)
    space = batch_space(single, n=rows)
    space.seed(11)
    record = sim.new_record()
    for call in range(4):
        before = _state(space)
        want = space.sample()
        got = sim.sample_space_stream(record, rows, cols, n_choices, low, high, override=before if call == 0 else None)
        assert np.array_equal(got.reshape(want.shape), want), call
        # numpy has advanced already: record == generator, and the ticket is back at 0
        assert _record_state(record) == _state(space), call
        assert int(record[4]) == 0


@pytest.mark.parametrize("rows,single", [CASES[2], CASES[6]], ids=["discrete", "box"])
def test_override_restarts_the_stream(rows, single):
    """A reseed (new state AND new inc) passed as the override: that call and the record-driven ones after it follow
    the new generator, whatever the record held."""
    cols, n_choices, low, high = _plan(single)
    space = batch_space(single, n=rows)
    space.seed(3)
    record = sim.new_record()
    sim.sample_space_stream(record, rows, cols, n_choices, low, high, override=_state(space))
    space.seed(2 ** 70 + 5)      # another SeedSequence: another inc
    assert _state(space)[1] != _record_state(record)[1]
    want = space.sample()
    got = sim.sample_space_stream(record, rows, cols, n_choices, low, high, override=None)   # stale record
    assert not np.array_equal(got.reshape(want.shape), want)
    space.seed(2 ** 70 + 5)
    for call in range(3):
        before = _state(space)
        want = space.sample()
        got = sim.sample_space_stream(record, rows, cols, n_choices, low, high, override=before if call == 0 else None)
        assert np.array_equal(got.reshape(want.shape), want), call
        assert _record_state(record) == _state(space), call


def test_host_draws_between_calls():
    """Host draws move the numpy generator past the record; passing its state as the override puts the device back on
    it, which is what sample_actions() does when the host generator differs from what it last left in the record."""
    single, rows = Discrete(3), 4099
    cols, n_choices, low, high = _plan(single)
    space = batch_space(single, n=rows)
    space.seed(0)
    record = sim.new_record()
    got0 = sim.sample_space_stream(record, rows, cols, n_choices, low, high, override=_state(space))
    assert np.array_equal(got0, space.sample())
    twin = batch_space(single, n=rows)
    twin.seed(0)
    twin.sample()
    space.np_random.random(17)     # a host draw
    # the record has not seen the host draw: without the override it continues where the first call left it
    assert np.array_equal(sim.sample_space_stream(record.copy(), rows, cols, n_choices, low, high), twin.sample())
    # with the override it follows the host
    before = _state(space)
    want = space.sample()
    assert np.array_equal(sim.sample_space_stream(record, rows, cols, n_choices, low, high, override=before), want)
    assert _record_state(record) == _state(space)
