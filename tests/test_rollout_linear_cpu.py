"""rollout_linear_kernel's device source on the CPU (tests/hostsim/rollout_linear.cpp), against a numpy restatement of
the linear policy and T launches of kernel A's driver.

For every classic-control id, with one shared policy and with one per env: the actions must be the numpy float32
policy (each product and sum rounded separately, ``np.argmax``) applied to the observation stream; the outputs and the
float64 state, TimeLimit counters, CartPole flags and PCG64 records must be bit for bit those of T kernel-A steps fed
those actions; and the summary mode must equal a float64 restatement over the full outputs and leave the same state.
Step 0 starts from ``observe(state)``, so the observation every path returns must be that function of the state.
"""
import numpy as np
import pytest

from gym_b200 import envs as _envs
from gym_b200.registration import spec as _spec
from hostsim.rollout_linear_sim import LinearRolloutSim

ENV_IDS = ["CartPole-v0", "CartPole-v1", "MountainCar-v0", "MountainCarContinuous-v0", "Pendulum-v1", "Acrobot-v1"]
NS = [1, 31, 257, 33 * 256 + 5]
TS = [1, 2, 37]


def _config(env_id):
    """(kind, registry max_episode_steps, param0, single action space) as B200VectorEnv resolves them"""
    s = _spec(env_id)
    ctor = dict(s.kwargs)
    kind, _ = _envs.resolve_variant(s.kind, ctor)
    params = _envs.resolve_params(kind, ctor)
    return kind, s.max_episode_steps, params[0], _envs.KINDS[kind].spaces(params)[1]


def _bits(x):
    return np.ascontiguousarray(x).view(np.uint8)


def _assert_same(a, b, what):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape and a.dtype == b.dtype, f"{what}: {a.shape} {a.dtype} vs {b.shape} {b.dtype}"
    assert np.array_equal(_bits(a), _bits(b)), f"{what}: {np.count_nonzero(a != b)} differ"


def policy(weight, bias, obs, discrete):
    """The documented arithmetic in numpy float32: z = bias, then z = z + weight[:, k] * o[k] for k in order; argmax
    (first NaN, else first maximum) for Discrete, z for Box.  weight (K, D) or (n, K, D), obs (n, D)."""
    n, D = obs.shape
    W = np.broadcast_to(weight, (n,) + weight.shape[-2:])
    z = np.array(np.broadcast_to(bias, (n, bias.shape[-1])), dtype=np.float32)
    for k in range(D):
        z = z + W[:, :, k] * obs[:, None, k]
    assert z.dtype == np.float32
    return np.argmax(z, axis=1).astype(np.int64) if discrete else z


def summary_of(rew, te, tr):
    """(returns, lengths, ended) over each env's first episode end, restated in float64 from the full outputs."""
    T, n = rew.shape
    done = te | tr
    ended = done.any(axis=0)
    t_end = np.where(ended, np.argmax(done, axis=0), T - 1)
    returns = np.zeros(n)
    for t in range(T):
        returns = np.where(t <= t_end, returns + rew[t], returns)
    return returns, (t_end + 1).astype(np.int32), ended


class _Case:
    """A linear-rollout batch, a kernel-A twin and a summary-mode twin, reset alike."""

    def __init__(self, env_id, N, seed, **kw):
        self.kind, mes, param0, single = _config(env_id)
        mes = kw.pop("max_episode_steps", mes)
        self.discrete = hasattr(single, "n")
        self.ro, self.step, self.summ = [LinearRolloutSim(self.kind, N, max_episode_steps=mes, param0=param0, **kw)
                                         for _ in range(3)]
        self.obs = self.ro.reset(seed)
        for sim in (self.step, self.summ):
            _assert_same(sim.reset(seed), self.obs, "reset")
        self.K = int(single.n) if self.discrete else int(single.shape[0])

    def params(self, rng, per_env, scale=1.0):
        lead = (self.ro.n,) if per_env else ()
        w = (scale * rng.standard_normal(lead + (self.K, self.ro.obs_dim))).astype(np.float32)
        b = (scale * rng.standard_normal(lead + (self.K,))).astype(np.float32)
        return w, b

    def check(self, weight, bias, T):
        ro, step = self.ro, self.step
        last = np.zeros((ro.n, ro.obs_dim), dtype=np.float32)
        got = ro.rollout_linear(weight, bias, T, last_obs=last)
        outs = []
        for t in range(T):
            want = policy(weight, bias, self.obs, self.discrete)
            _assert_same(got[0][t], want if self.discrete else want.reshape(got[0][t].shape), f"actions[{t}]")
            outs.append(step.step(got[0][t]))
            assert outs[-1][5] == 0, "invalid actions"
            self.obs = outs[-1][0]
        for k, name in enumerate(("obs", "reward", "terminated", "truncated", "final_obs")):
            _assert_same(got[k + 1], np.stack([o[k] for o in outs]), name)
        _assert_same(last, got[1][-1], "last observation buffer")
        for x, y, name in zip(ro.get_state(), step.get_state(), ("state", "elapsed", "flags", "rng")):
            _assert_same(x, y, name)
        # the summary twin takes the same T steps and folds them
        last_s = np.zeros_like(last)
        summ = self.summ.rollout_linear(weight, bias, T, summary=True, last_obs=last_s)
        for x, y, name in zip(summ, summary_of(got[2], got[3], got[4]), ("returns", "lengths", "ended")):
            _assert_same(x, y, name)
        _assert_same(last_s, last, "summary: last observation buffer")
        for x, y, name in zip(self.summ.get_state(), ro.get_state(), ("state", "elapsed", "flags", "rng")):
            _assert_same(x, y, f"summary: {name}")
        return got


@pytest.mark.parametrize("per_env", [False, True])
@pytest.mark.parametrize("N", NS)
@pytest.mark.parametrize("T", TS)
@pytest.mark.parametrize("env_id", ENV_IDS)
def test_linear_rollout_equals_policy_and_steps(env_id, T, N, per_env):
    """Two calls in a row: the second starts from the state the first left."""
    c = _Case(env_id, N, seed=3000 + T + N)
    rng = np.random.default_rng(T * 7919 + N)
    for _ in range(2):
        c.check(*c.params(rng, per_env), T)


@pytest.mark.parametrize("limit", [None, 4])
@pytest.mark.parametrize("env_id", ENV_IDS)
def test_linear_rollout_without_autoreset(env_id, limit):
    """autoreset=False, with and without a short TimeLimit: no resets, CartPole's flag byte in memory."""
    kw = {"autoreset": False} if limit is None else {"autoreset": False, "max_episode_steps": limit}
    c = _Case(env_id, 50, seed=11, **kw)
    c.check(*c.params(np.random.default_rng(1), True), 60)


@pytest.mark.parametrize("env_id", ENV_IDS)
def test_linear_rollout_truncates_and_resets(env_id):
    """max_episode_steps=4: every env ends an episode inside the rollout, is reset inline, and its policy goes on
    from the reset observation; the summary stops at the first end."""
    c = _Case(env_id, 257, seed=13, max_episode_steps=4)
    got = c.check(*c.params(np.random.default_rng(2), False), 37)
    assert (got[3] | got[4]).any(axis=0).all()


@pytest.mark.parametrize("env_id", ["CartPole-v1", "MountainCar-v0", "Acrobot-v1"])
def test_tied_and_nan_logits(env_id):
    """Zero parameters tie every logit: action 0.  A NaN logit wins from its index on, even behind a larger one."""
    c = _Case(env_id, 64, seed=17)
    K, D, n = c.K, c.ro.obs_dim, c.ro.n
    got = c.check(np.zeros((K, D), np.float32), np.zeros(K, np.float32), 3)
    assert (got[0] == 0).all()
    b = np.zeros((n, K), np.float32)
    b[:, 0] = 5.0
    b[0::2, K - 1] = np.nan      # NaN in the last logit only
    b[1::4, 1:] = np.nan         # NaN from index 1 on: the first NaN is 1
    w = np.zeros((n, K, D), np.float32)
    w[3::4, 0, 0] = np.nan       # logit 0 NaN through the weight
    got = c.check(w, b, 3)
    want = np.where(np.arange(n) % 4 == 3, 0, np.where(np.arange(n) % 4 == 1, 1, np.where(np.arange(n) % 2 == 0, K - 1, 0)))
    assert (got[0] == want).all()


@pytest.mark.parametrize("env_id", ENV_IDS)
def test_observe_is_the_last_returned_observation(env_id):
    """Step 0's input is observe(state): it must equal the observation the env last returned after reset(seed=),
    reset(options=), steps, autoresets, autoreset=False, and after a restore or clone (state copied with its
    observation)."""
    kind, mes, param0, single = _config(env_id)
    rng = np.random.default_rng(5)
    discrete = hasattr(single, "n")

    def actions(n):
        if discrete:
            return rng.integers(0, single.n, size=n)
        return rng.uniform(-3.0, 3.0, size=(n, 1)).astype(np.float32)

    for kw in ({"max_episode_steps": 5}, {"autoreset": False}, {"autoreset": False, "max_episode_steps": 3}):
        sim = LinearRolloutSim(kind, 300, param0=param0, **{"max_episode_steps": mes, **kw})
        obs = sim.reset(21)
        _assert_same(sim.observe(), obs, "reset(seed=)")
        obs = sim.reset(22, bounds=(-0.03, 0.04))
        _assert_same(sim.observe(), obs, "reset(options=)")
        saved, saved_obs = None, None
        for t in range(40):
            obs = sim.step(actions(sim.n))[0]
            _assert_same(sim.observe(), obs, f"step {t} ({kw})")
            if t == 9:
                saved, saved_obs = [x.copy() for x in (sim.state, sim.elapsed, sim.flags, sim.rng)], obs.copy()
        if kw.get("max_episode_steps") == 5:
            assert sim.elapsed.max() < 5   # autoresets happened along the way
        # restore (and clone, which is a restore from another batch): the saved rows with their observation
        other = LinearRolloutSim(kind, 300, param0=param0, **{"max_episode_steps": mes, **kw})
        for dst in (sim, other):
            for x, y in zip((dst.state, dst.elapsed, dst.flags, dst.rng), saved):
                x[...] = y
            _assert_same(dst.observe(), saved_obs, "restore / clone")
