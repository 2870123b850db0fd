"""rollout_linear_norm_kernel's and rollout_mlp_norm_kernel's device source on the CPU
(tests/hostsim/rollout_policy_norm.cpp), against a numpy restatement: the observations normalised in float64,
``float32((float64(o) - mean) / sqrt(var + eps))`` clamped to [-c, c], then test_rollout_linear_cpu's logits or
test_rollout_mlp_cpu's float32 MLP on them.

The env outputs stay raw: obs, rewards and final observations must be those of T kernel-A steps of a twin batch fed
the same actions.  Summary mode on a third twin must give the fold of the full outputs, and the observation moments the
sequential float64 fold of the raw inputs of each env's first episode.  Identity statistics (mean 0, var 1, eps 0, no
clip) must give the drivers without normalisation byte for byte.  The per-element edges of test_rollout_norm_cpu.py
(var = -eps, NaN through the clip, -0.0, clip bounds hit exactly) are run through the whole drivers.
"""
import numpy as np
import pytest

import test_rollout_mlp_cpu as mlp_cpu
from hostsim.rollout_policy_norm_sim import RELU, TANH, PolicyNormRolloutSim
from test_rollout_linear_cpu import ENV_IDS, _assert_same, _config, summary_of
from test_rollout_linear_cpu import policy as linear_policy
from test_rollout_mlp_cpu import param_count
from test_rollout_norm_cpu import norm_restated

HIDDEN = [(16,), (64,), (64, 64)]
SHAPES = [(1, 1), (257, 37), (33 * 256 + 5, 2), (67, 120)]


def moments_restated(inputs, lengths):
    """The sequential fold of the raw inputs (T, n, D) over t < lengths: s = +0.0; s = s + o, q = q + o * o."""
    o = inputs.astype(np.float64)
    s = np.zeros(o.shape[1:])
    q = np.zeros(o.shape[1:])
    for t in range(o.shape[0]):
        keep = (t < lengths)[:, None]
        s = np.where(keep, s + o[t], s)
        q = np.where(keep, q + o[t] * o[t], q)
    return s, q


class _Case:
    """A batch for the normalised drivers, a kernel-A twin and a summary-mode twin, reset alike."""

    def __init__(self, env_id, N, seed, **kw):
        self.kind, mes, param0, single = _config(env_id)
        mes = kw.pop("max_episode_steps", mes)
        self.discrete = hasattr(single, "n")
        self.ro, self.step, self.summ = [PolicyNormRolloutSim(self.kind, N, max_episode_steps=mes, param0=param0, **kw)
                                         for _ in range(3)]
        self.obs = self.ro.reset(seed)
        for sim in (self.step, self.summ):
            _assert_same(sim.reset(seed), self.obs, "reset")
        self.K = int(single.n) if self.discrete else int(single.shape[0])
        self.D = self.ro.obs_dim
        self.n = N

    def stats(self, rng):
        return rng.standard_normal(self.D) * 0.3, rng.random(self.D) * 2.0 + 0.01

    def linear(self, rng, per_env, scale=1.0):
        lead = (self.n,) if per_env else ()
        return ((scale * rng.standard_normal(lead + (self.K, self.D))).astype(np.float32),
                (scale * rng.standard_normal(lead + (self.K,))).astype(np.float32))

    def mlp(self, rng, hidden, per_env, scale=0.5):
        lead = (self.n,) if per_env else ()
        return (scale * rng.standard_normal(lead + (param_count(self.D, hidden, self.K),))).astype(np.float32)

    def check(self, net, T, mean, var, eps, clip, hidden=None, act=RELU, nan_returns=False):
        """net: (weight, bias) for the linear driver, params with `hidden` for the MLP one.  mean None: raw inputs.
        nan_returns: NaN rewards are expected, and numpy's fold of them need not give the driver's NaN bits, so the
        returns are compared as values (NaN equal to NaN)."""
        if hidden is None:
            run = lambda sim, **kw: sim.rollout_linear_norm(*net, T, mean, var, eps, clip, **kw)  # noqa: E731
            want = lambda x: linear_policy(*net, x, self.discrete)  # noqa: E731
        else:
            run = lambda sim, **kw: sim.rollout_mlp_norm(net, hidden, T, mean, var, eps, clip, act, **kw)  # noqa: E731
            want = lambda x: mlp_cpu.policy(net, hidden, x, self.K, self.discrete)  # noqa: E731
        last = np.zeros((self.n, self.D), dtype=np.float32)
        got = run(self.ro, last_obs=last)
        outs, inputs = [], []
        for t in range(T):
            inputs.append(self.obs)
            x = self.obs if mean is None else norm_restated(self.obs, mean, var, eps, clip)
            w = want(x)
            _assert_same(got[0][t], w if self.discrete else w.reshape(got[0][t].shape), f"actions[{t}]")
            outs.append(self.step.step(got[0][t]))
            assert outs[-1][5] == 0, "invalid actions"
            self.obs = outs[-1][0]
        for k, name in enumerate(("obs", "reward", "terminated", "truncated", "final_obs")):
            _assert_same(got[k + 1], np.stack([o[k] for o in outs]), name)
        _assert_same(last, got[1][-1], "last observation buffer")
        for x, y, name in zip(self.ro.get_state(), self.step.get_state(), ("state", "elapsed", "flags", "rng")):
            _assert_same(x, y, name)
        # the summary twin takes the same T steps, folds them, and folds the raw inputs of the first episode
        last_s = np.zeros_like(last)
        summ = run(self.summ, summary=True, moments=True, last_obs=last_s)
        ret, lengths, ended = summary_of(got[2], got[3], got[4])
        for x, y, name in zip(summ, (ret, lengths, ended) + moments_restated(np.stack(inputs), lengths),
                              ("returns", "lengths", "ended", "obs_sum", "obs_sumsq")):
            if nan_returns and name == "returns":
                np.testing.assert_array_equal(x, y, err_msg=name)
            else:
                _assert_same(x, y, name)
        _assert_same(last_s, last, "summary: last observation buffer")
        for x, y, name in zip(self.summ.get_state(), self.ro.get_state(), ("state", "elapsed", "flags", "rng")):
            _assert_same(x, y, f"summary: {name}")
        return got, summ


@pytest.fixture
def tanh(monkeypatch):
    """The numpy MLP with the C library's tanhf, which the host build's tanh instantiation calls."""
    from test_rollout_mlp_tanh_cpu import libm_tanhf
    monkeypatch.setattr(mlp_cpu, "relu", libm_tanhf)


@pytest.mark.parametrize("clip", [None, 0.75])
@pytest.mark.parametrize("per_env", [False, True])
@pytest.mark.parametrize("N,T", SHAPES)
@pytest.mark.parametrize("env_id", ENV_IDS)
def test_linear_norm_equals_restatement(env_id, N, T, per_env, clip):
    c = _Case(env_id, N, seed=300 + N + T)
    rng = np.random.default_rng(N * 7 + T + per_env)
    mean, var = c.stats(rng)
    net = c.linear(rng, per_env)
    c.check(net, T, mean, var, 1e-8, clip)
    c.check(net, 2, mean, var, 1e-8, clip)            # continues from the state left


@pytest.mark.parametrize("per_env", [False, True])
@pytest.mark.parametrize("N,T", SHAPES)
@pytest.mark.parametrize("hidden", HIDDEN)
@pytest.mark.parametrize("env_id", ENV_IDS)
def test_mlp_norm_equals_restatement(env_id, hidden, N, T, per_env):
    c = _Case(env_id, N, seed=700 + N + T)
    rng = np.random.default_rng(N * 13 + T + len(hidden) + per_env)
    mean, var = c.stats(rng)
    c.check(c.mlp(rng, hidden, per_env), T, mean, var, 1e-8, 1.5, hidden)


@pytest.mark.parametrize("per_env", [False, True])
@pytest.mark.parametrize("hidden", [(5,), (64, 64)])
@pytest.mark.parametrize("env_id", ENV_IDS)
def test_tanh_norm_equals_restatement(tanh, env_id, hidden, per_env):
    c = _Case(env_id, 67, seed=81, max_episode_steps=6)
    rng = np.random.default_rng(9)
    mean, var = c.stats(rng)
    c.check(c.mlp(rng, hidden, per_env), 20, mean, var, 1e-5, 0.9, hidden, act=TANH)


@pytest.mark.parametrize("net", ["linear", "mlp"])
@pytest.mark.parametrize("env_id", ENV_IDS)
def test_moments_without_normalisation(env_id, net):
    """obs_moments with raw inputs (mean null): the policy reads o itself."""
    c = _Case(env_id, 300, seed=5, max_episode_steps=9)
    rng = np.random.default_rng(1)
    if net == "linear":
        c.check(c.linear(rng, True), 25, None, None, 1e-8, None)
    else:
        c.check(c.mlp(rng, (8, 8), True), 25, None, None, 1e-8, None, (8, 8))


@pytest.mark.parametrize("env_id", ENV_IDS)
def test_moments_at_the_edges_of_the_first_episode(env_id):
    """max_episode_steps=1: every env ends at t = 0, so the moments are one input each; a long limit with T = 3 leaves
    most envs running to the end (lengths = T); and T = 1."""
    for mes, T in ((1, 4), (10 ** 6, 3), (10 ** 6, 1)):
        c = _Case(env_id, 129, seed=mes + T, max_episode_steps=mes)
        rng = np.random.default_rng(T)
        mean, var = c.stats(rng)
        _, summ = c.check(c.linear(rng, True), T, mean, var, 1e-8, None)
        if mes == 1:
            assert (summ[1] == 1).all() and summ[2].all()
        elif T == 3:
            assert (summ[1] == 3).any()


@pytest.mark.parametrize("per_env", [False, True])
@pytest.mark.parametrize("hidden", [None, (16,), (64, 64)])
@pytest.mark.parametrize("env_id", ENV_IDS)
def test_identity_statistics_give_the_drivers_without_normalisation(env_id, hidden, per_env):
    """mean 0, var 1, eps 0, no clip: x = float32(float64(o) / 1) = o, so every output, full and summary, is byte for
    byte that of rollout_linear_env / rollout_mlp_env."""
    kind, mes, param0, single = _config(env_id)
    sims = [PolicyNormRolloutSim(kind, 300, max_episode_steps=7, param0=param0) for _ in range(4)]
    for s in sims:
        s.reset(33)
    D = sims[0].obs_dim
    K = int(single.n) if hasattr(single, "n") else int(single.shape[0])
    rng = np.random.default_rng(4)
    lead = (300,) if per_env else ()
    mean, var = np.zeros(D), np.ones(D)
    for summary in (False, True):
        if hidden is None:
            w = rng.standard_normal(lead + (K, D)).astype(np.float32)
            b = rng.standard_normal(lead + (K,)).astype(np.float32)
            got = sims[0 + 2 * summary].rollout_linear_norm(w, b, 25, mean, var, 0.0, None, summary=summary)
            want = sims[1 + 2 * summary].rollout_linear(w, b, 25, summary=summary)
        else:
            p = (0.5 * rng.standard_normal(lead + (param_count(D, hidden, K),))).astype(np.float32)
            got = sims[0 + 2 * summary].rollout_mlp_norm(p, hidden, 25, mean, var, 0.0, None, summary=summary)
            want = sims[1 + 2 * summary].rollout_mlp(p, hidden, 25, summary=summary)
        assert len(got) == len(want)
        for k, (x, y) in enumerate(zip(got, want)):
            _assert_same(x, y, f"summary={summary} output {k}")
        for x, y in zip(sims[0 + 2 * summary].get_state(), sims[1 + 2 * summary].get_state()):
            _assert_same(x, y, "state")


@pytest.mark.parametrize("case", ["zero_sd", "nan_clip", "minus_zero", "clip_bounds"])
@pytest.mark.parametrize("env_id", ENV_IDS)
def test_edges_through_the_drivers(env_id, case):
    """The per-element edges, with the statistics chosen against the env's first observations: var = -eps (sd = 0:
    infinite and NaN inputs), the same through a clip (NaN stays NaN), mean -0.0 / +0.0 with var 1 and eps 0 (x keeps
    o's sign bits), and a clip equal to an input exactly."""
    c = _Case(env_id, 257, seed=17, max_episode_steps=5)
    rng = np.random.default_rng(3)
    D = c.D
    mean, var, eps, clip = np.zeros(D), np.ones(D), 0.0, None
    if case in ("zero_sd", "nan_clip"):
        mean = c.obs[0].astype(np.float64)      # env 0's inputs are NaN at step 0, the others' +-inf
        var, eps = np.full(D, -1e-8), 1e-8
        clip = 10.0 if case == "nan_clip" else None
    elif case == "minus_zero":
        mean = np.where(np.arange(D) % 2 == 0, -0.0, 0.0)
    else:
        clip = float(abs(c.obs[1, 0])) or 0.5  # env 1's first input hits the bound exactly
    for hidden in (None, (8,)):
        net = c.linear(rng, True) if hidden is None else c.mlp(rng, hidden, True)
        c.check(net, 6, mean, var, eps, clip, hidden, nan_returns=True)
