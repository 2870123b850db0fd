"""rollout_sampled_kernel's device source on the CPU (tests/hostsim/rollout_sampled.cpp), against numpy's Generator and
T launches of kernel A's driver.

For every classic-control id: the actions drawn must be T consecutive ``batch_space(single, N).sample()`` calls of a
generator with the same seed; the outputs, the float64 state, TimeLimit counters, CartPole flags and PCG64 records must
be bit for bit those of T kernel-A steps fed those actions; and the record must end where the numpy generator does,
with the ticket back at 0.  The grids cover one CTA, a ragged last CTA and many CTAs.
"""
import numpy as np
import pytest

from gym_b200 import envs as _envs
from gym_b200.registration import spec as _spec
from gym_b200.spaces import batch_space
from hostsim.rollout_sampled_sim import SampledRolloutSim, new_record, record_state

ENV_IDS = ["CartPole-v0", "CartPole-v1", "MountainCar-v0", "MountainCarContinuous-v0", "Pendulum-v1", "Acrobot-v1"]
NS = [1, 31, 256, 257, 33 * 256 + 5]
TS = [1, 2, 37]


def _config(env_id):
    """(kind, registry max_episode_steps, param0, single action space) as B200VectorEnv resolves them"""
    s = _spec(env_id)
    ctor = dict(s.kwargs)
    kind, _ = _envs.resolve_variant(s.kind, ctor)
    params = _envs.resolve_params(kind, ctor)
    return kind, s.max_episode_steps, params[0], _envs.KINDS[kind].spaces(params)[1]


def _plan(single):
    """(n_choices, low, high) of b200gym_rollout_sampled"""
    if hasattr(single, "n"):
        return int(single.n), 0.0, 0.0
    return 0, float(single.low[0]), float(single.high[0])


def _gen_state(space):
    st = space.np_random.bit_generator.state["state"]
    return st["state"], st["inc"]


def _bits(x):
    return np.ascontiguousarray(x).view(np.uint8)


def _assert_same(a, b, what):
    assert a.shape == b.shape and a.dtype == b.dtype, what
    assert np.array_equal(_bits(a), _bits(b)), f"{what}: {np.count_nonzero(np.asarray(a) != np.asarray(b))} differ"


class _Case:
    """A sampled-rollout batch, a kernel-A twin and the batched action space both follow, reset alike."""

    def __init__(self, env_id, N, seed, space_seed, **kw):
        self.kind, mes, param0, self.single = _config(env_id)
        mes = kw.pop("max_episode_steps", mes)
        self.ro, self.step = [SampledRolloutSim(self.kind, N, max_episode_steps=mes, param0=param0, **kw)
                              for _ in range(2)]
        _assert_same(self.ro.reset(seed), self.step.reset(seed), "reset")
        self.space = batch_space(self.single, n=N)
        self.space.seed(space_seed)
        self.plan = _plan(self.single)
        self.record = new_record()

    def check(self, T, override):
        """One sampled rollout (from `override`, or from the record) against T host samples and T kernel-A steps."""
        ro, step = self.ro, self.step
        last = np.zeros((ro.n, ro.obs_dim), dtype=np.float32)
        got = ro.rollout_sampled(self.record, T, *self.plan, override=override, last_obs=last)
        want_actions = np.stack([self.space.sample() for _ in range(T)])
        _assert_same(got[0].reshape(want_actions.shape), want_actions, "actions")
        outs = [step.step(a) for a in got[0]]
        names = ("obs", "reward", "terminated", "truncated", "final_obs")
        for k, name in enumerate(names):
            _assert_same(got[k + 1], np.stack([o[k] for o in outs]), name)
        assert got[6] == 0 == sum(o[5] for o in outs), "invalid actions"
        _assert_same(last, got[1][-1], "last observation buffer")
        for x, y, name in zip(ro.get_state(), step.get_state(), ("state", "elapsed", "flags", "rng")):
            _assert_same(x, y, name)
        assert record_state(self.record) == _gen_state(self.space), "record after the rollout"
        assert int(self.record[4]) == 0, "ticket"
        return got


@pytest.mark.parametrize("N", NS)
@pytest.mark.parametrize("T", TS)
@pytest.mark.parametrize("env_id", ENV_IDS)
def test_sampled_rollout_equals_samples_and_steps(env_id, T, N):
    """The first call starts from the override (the host generator), the second from the record the first left."""
    c = _Case(env_id, N, seed=2000 + T + N, space_seed=T * 7919 + N)
    c.check(T, override=_gen_state(c.space))
    c.check(T, override=None)


@pytest.mark.parametrize("env_id", ENV_IDS)
def test_override_restarts_the_stream(env_id):
    """A reseeded space (new state and inc) passed as the override wins over a stale record, and the record-driven
    call after it continues the new stream."""
    c = _Case(env_id, 300, seed=5, space_seed=3)
    c.check(4, override=_gen_state(c.space))
    c.space.seed(2 ** 70 + 5)
    assert _gen_state(c.space)[1] != record_state(c.record)[1]
    c.check(6, override=_gen_state(c.space))
    c.check(5, override=None)


@pytest.mark.parametrize("env_id", ENV_IDS)
def test_host_draws_between_calls(env_id):
    """Host draws between calls move the generator past the record; passing its state as the override follows it."""
    c = _Case(env_id, 129, seed=8, space_seed=0)
    c.check(3, override=_gen_state(c.space))
    c.space.sample()
    c.space.np_random.random(17)
    c.check(3, override=_gen_state(c.space))


@pytest.mark.parametrize("limit", [None, 4])
@pytest.mark.parametrize("env_id", ENV_IDS)
def test_sampled_rollout_without_autoreset(env_id, limit):
    """autoreset=False, with and without a short TimeLimit: no resets, CartPole's flag byte in memory."""
    kw = {"autoreset": False} if limit is None else {"autoreset": False, "max_episode_steps": limit}
    c = _Case(env_id, 50, seed=11, space_seed=12, **kw)
    c.check(60, override=_gen_state(c.space))


@pytest.mark.parametrize("env_id", ENV_IDS)
def test_sampled_rollout_truncates_and_resets(env_id):
    """max_episode_steps=4: every env ends an episode inside the rollout and is reset inline."""
    c = _Case(env_id, 257, seed=13, space_seed=14, max_episode_steps=4)
    got = c.check(37, override=_gen_state(c.space))
    assert (got[3] | got[4]).any(axis=0).all()
