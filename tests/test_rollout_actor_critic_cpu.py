"""rollout_actor_critic_kernel's and gae_kernel's device source on the CPU (tests/hostsim/rollout_actor_critic.cpp),
against a numpy float32 restatement.

The driver: for every classic-control id, the actor's outputs, the actions and the env outputs, state, TimeLimit
counters and PCG64 records must be those of test_rollout_mlp_noisy_cpu's restatement (the numpy MLP plus the noise, and
T kernel-A steps of the same batch); ``values[t]`` the numpy critic (the same MLP code with one output) of the
observation step t acts on and ``values[T]`` of the last one; and the advantages the documented recursion in numpy
float32, with the critic of the final observation where a step truncated without terminating.

``gae_env`` alone, on hand-made rows: terminated, truncated and both on one step, a done on the last step, T = 1, a NaN
reward, gamma = 0, gae_lambda 0 and 1, rewards that round when cast to float32, and -0.0 deltas.
"""
import numpy as np
import pytest

import test_rollout_mlp_cpu as mlp_cpu
from hostsim.rollout_actor_critic_sim import RELU, TANH, ActorCriticRolloutSim, gae
from test_rollout_linear_cpu import ENV_IDS, _assert_same, _config
from test_rollout_mlp_cpu import mlp_outputs, param_count
from test_rollout_mlp_noisy_cpu import _assert_actions, noisy_action

HIDDEN = [(1,), (64,), (3, 7), (64, 64)]
# (N, T): one env, N not a multiple of 256 and a multi-CTA N with short rollouts, a long rollout at a small N
SHAPES = [(1, 1), (257, 37), (33 * 256 + 5, 2), (67, 300)]


def coefficients(gamma, gae_lambda):
    """The Python layer's rounding: float32(gamma), float32(gamma * gae_lambda) with the product in float64."""
    return np.float32(gamma), np.float32(float(gamma) * float(gae_lambda))


def gae_restated(g, gl, rew, te, tr, values, vf):
    """The documented recursion in numpy float32, one rounded operation at a time."""
    g, gl = np.float32(g), np.float32(gl)
    T, n = rew.shape
    adv = np.empty((T, n), np.float32)
    nxt = np.zeros(n, np.float32)
    with np.errstate(all="ignore"):
        for t in reversed(range(T)):
            r = rew[t].astype(np.float32)
            d_term = r - values[t]
            d_trunc = (r + g * vf[t]) - values[t]
            d_cont = (r + g * values[t + 1]) - values[t]
            delta = np.where(te[t], d_term, np.where(tr[t], d_trunc, d_cont))
            nxt = np.where(te[t] | tr[t], delta, delta + gl * nxt)
            assert nxt.dtype == np.float32
            adv[t] = nxt
    return adv


def _assert_same_nan(got, want, what):
    """Bit for bit where want is a number; NaN where want is NaN (numpy and the host build may keep either NaN
    operand's payload)."""
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan), f"{what}: NaN positions differ"
    _assert_same(np.where(nan, 0, got).astype(got.dtype), np.where(nan, 0, want).astype(want.dtype), what)


class _Case:
    """An actor-critic batch and a kernel-A twin, reset alike."""

    def __init__(self, env_id, N, seed, **kw):
        self.kind, mes, param0, single = _config(env_id)
        mes = kw.pop("max_episode_steps", mes)
        self.discrete = hasattr(single, "n")
        self.ro, self.step = [ActorCriticRolloutSim(self.kind, N, max_episode_steps=mes, param0=param0, **kw)
                              for _ in range(2)]
        self.obs = self.ro.reset(seed)
        _assert_same(self.step.reset(seed), self.obs, "reset")
        self.K = int(single.n) if self.discrete else int(single.shape[0])

    def nets(self, rng, hidden, scale=0.5):
        D = self.ro.obs_dim
        return ((scale * rng.standard_normal(param_count(D, hidden, self.K))).astype(np.float32),
                (scale * rng.standard_normal(param_count(D, hidden, 1))).astype(np.float32))

    def noise(self, rng, T, scale=1.0):
        return (scale * rng.standard_normal((T, self.ro.n, self.K))).astype(np.float32)

    def check(self, actor, critic, hidden, noise, gamma=0.99, gae_lambda=0.95, act=RELU):
        ro, step = self.ro, self.step
        T = noise.shape[0]
        g, gl = coefficients(gamma, gae_lambda)
        last = np.zeros((ro.n, ro.obs_dim), dtype=np.float32)
        got = ro.rollout_actor_critic(actor, critic, hidden, noise, g, gl, act, last_obs=last)
        acts, outs_z, values, adv = got[:4]
        assert values.shape == (T + 1, ro.n) and adv.shape == (T, ro.n)
        outs, vf = [], np.full((T, ro.n), np.nan, np.float32)
        for t in range(T):
            z = mlp_outputs(actor, hidden, self.obs, self.K)
            _assert_same(outs_z[t], z, f"outputs[{t}]")
            _assert_same(values[t], mlp_outputs(critic, hidden, self.obs, 1)[:, 0], f"values[{t}]")
            _assert_actions(acts[t], noisy_action(z, noise[t], self.discrete), f"actions[{t}]")
            outs.append(step.step(acts[t]))
            assert outs[-1][5] == 0, "invalid actions"
            o, _, te, tr, fo = outs[-1][:5]
            held = tr.astype(bool) & ~te.astype(bool)
            vf[t, held] = mlp_outputs(critic, hidden, fo[held], 1)[:, 0]
            self.obs = o
        _assert_same(values[T], mlp_outputs(critic, hidden, self.obs, 1)[:, 0], "values[T]")
        for k, name in enumerate(("obs", "reward", "terminated", "truncated", "final_obs")):
            _assert_same(got[k + 4], np.stack([o[k] for o in outs]), name)
        _assert_same(last, got[4][-1], "last observation buffer")
        for x, y, name in zip(ro.get_state(), step.get_state(), ("state", "elapsed", "flags", "rng")):
            _assert_same(x, y, name)
        want = gae_restated(g, gl, got[5], got[6], got[7], values, vf)
        _assert_same_nan(adv, want, "advantages")
        return got


@pytest.mark.parametrize("N,T", SHAPES)
@pytest.mark.parametrize("hidden", HIDDEN)
@pytest.mark.parametrize("env_id", ENV_IDS)
def test_actor_critic_rollout_equals_restatement(env_id, hidden, N, T):
    """Two calls in a row: the second starts from the state the first left, and its values[0] is the first's
    values[T]."""
    c = _Case(env_id, N, seed=8000 + T + N)
    rng = np.random.default_rng(T * 7919 + N + len(hidden))
    a, v = c.nets(rng, hidden)
    first = c.check(a, v, hidden, c.noise(rng, T))
    second = c.check(a, v, hidden, c.noise(rng, T))
    _assert_same(second[2][0], first[2][-1], "values[0] of the next call")


@pytest.fixture
def tanh(monkeypatch):
    """The numpy MLP with the C library's tanhf, which the host build's tanh instantiation calls."""
    from test_rollout_mlp_tanh_cpu import libm_tanhf
    monkeypatch.setattr(mlp_cpu, "relu", libm_tanhf)


@pytest.mark.parametrize("hidden", [(5,), (64, 64)])
@pytest.mark.parametrize("env_id", ENV_IDS)
def test_tanh_actor_critic_rollout_equals_restatement(tanh, env_id, hidden):
    c = _Case(env_id, 67, seed=81, max_episode_steps=6)
    rng = np.random.default_rng(9)
    a, v = c.nets(rng, hidden)
    c.check(a, v, hidden, c.noise(rng, 20), act=TANH)


@pytest.mark.parametrize("gamma,gae_lambda", [(0.99, 0.95), (0.0, 0.95), (0.9, 0.0), (0.97, 1.0), (1.0, 1.0)])
@pytest.mark.parametrize("env_id", ENV_IDS)
def test_truncations_bootstrap_from_the_final_observation(env_id, gamma, gae_lambda):
    """max_episode_steps=4: every env truncates inside the call, most without terminating, and the bootstrap of those
    steps is the critic of the final observation, not of the reset observation that follows."""
    c = _Case(env_id, 257, seed=14, max_episode_steps=4)
    rng = np.random.default_rng(2)
    a, v = c.nets(rng, (8, 6))
    got = c.check(a, v, (8, 6), c.noise(rng, 37), gamma, gae_lambda)
    te, tr = got[6], got[7]
    assert (tr & ~te).any(axis=0).all()


def test_termination_on_the_time_limit():
    """CartPole pushed one way only (-0.0 noise, an actor that always picks action 0) terminates after 8 to 10 steps;
    with max_episode_steps=9 some envs terminate on the step that also truncates, which bootstraps nothing."""
    c = _Case("CartPole-v1", 1000, seed=3, max_episode_steps=9)
    hidden = (1,)
    a = np.zeros(param_count(4, hidden, 2), np.float32)
    a[-2] = 1.0                                                  # output bias: logit 0 is 1, logit 1 is 0
    v = np.random.default_rng(4).standard_normal(param_count(4, hidden, 1)).astype(np.float32)
    got = c.check(a, v, hidden, np.full((40, 1000, 2), -0.0, np.float32))
    te, tr = got[6], got[7]
    assert (te & tr).any() and (tr & ~te).any() and (te & ~tr).any()


# ----------------------------------------------------------------------------------------- gae_env on its own
def _gae_both(g, gl, rew, te, tr, values, vf):
    held = np.where(tr & ~te, vf, np.float32(np.nan)).astype(np.float32)
    got = gae(g, gl, rew, te, tr, values, held)
    _assert_same_nan(got, gae_restated(g, gl, rew, te, tr, values, vf), "advantages")
    return got


def test_gae_flags_by_hand():
    """One env, T = 4: step 1 truncated (bootstrap from Vf), step 2 terminated and truncated (no bootstrap), step 3
    (the last) terminated; g = 0.5 and gl = 0.25 keep every value exact, so the expected numbers are written out."""
    rew = np.array([[1.0], [2.0], [3.0], [4.0]])
    te = np.array([[0], [0], [1], [1]], bool)
    tr = np.array([[0], [1], [1], [0]], bool)
    values = np.array([[0.5], [1.0], [2.0], [3.0], [100.0]], np.float32)
    vf = np.array([[0.0], [8.0], [0.0], [0.0]], np.float32)
    got = _gae_both(np.float32(0.5), np.float32(0.25), rew, te, tr, values, vf)
    # t=3: 4-3 = 1; t=2: 3-2 = 1; t=1: (2 + 0.5*8) - 1 = 5; t=0: (1 + 0.5*1) - 0.5 = 1, + 0.25*5 = 2.25
    assert got[:, 0].tolist() == [2.25, 5.0, 1.0, 1.0]


def test_gae_done_on_the_last_step_and_t_equals_one():
    """T = 1: no done bootstraps from values[1]; a done on the last step ignores values[T] and Vf, but a truncation
    without termination uses Vf."""
    rew = np.array([[1.0, 1.0, 1.0, 1.0]])
    te = np.array([[0, 1, 0, 1]], bool)
    tr = np.array([[0, 0, 1, 1]], bool)
    values = np.array([[0.25] * 4, [2.0] * 4], np.float32)
    vf = np.array([[16.0] * 4], np.float32)
    got = _gae_both(np.float32(0.5), np.float32(0.5), rew, te, tr, values, vf)
    assert got[0].tolist() == [1.75, 0.75, 8.75, 0.75]


@pytest.mark.parametrize("gamma,gae_lambda", [(0.0, 0.3), (0.99, 0.0), (0.99, 1.0), (1.0, 1.0), (0.95, 0.9)])
def test_gae_random_rows(gamma, gae_lambda):
    """Random flags (about 1 in 8 done), rewards and values over (T, n) = (50, 300); gamma = 0 gives delta = r - v."""
    rng = np.random.default_rng(int(gamma * 100 + gae_lambda * 10))
    T, n = 50, 300
    rew = rng.standard_normal((T, n)) * 3
    te, tr = rng.random((T, n)) < 0.07, rng.random((T, n)) < 0.07
    values = rng.standard_normal((T + 1, n)).astype(np.float32)
    vf = rng.standard_normal((T, n)).astype(np.float32)
    g, gl = coefficients(gamma, gae_lambda)
    got = _gae_both(g, gl, rew, te, tr, values, vf)
    if gamma == 0.0:
        last = (te | tr)
        with np.errstate(all="ignore"):
            want = np.where(last, rew.astype(np.float32) - values[:-1], np.float32(0) + rew.astype(np.float32) - values[:-1])
        assert np.array_equal(got[-1][last[-1]], want[-1][last[-1]])


def test_gae_nan_reward():
    """An invalid Discrete action returns a NaN reward: that step's advantage is NaN, and so is every earlier one up
    to the previous done; steps after it and before that done are untouched."""
    rew = np.array([[1.0], [np.nan], [1.0], [1.0], [1.0]])
    te = np.array([[0], [0], [0], [1], [0]], bool)
    tr = np.zeros((5, 1), bool)
    values = np.zeros((6, 1), np.float32)
    got = _gae_both(np.float32(0.9), np.float32(0.9), rew, te, tr, values, np.zeros((5, 1), np.float32))
    assert np.isnan(got[:2, 0]).all() and not np.isnan(got[2:, 0]).any()


def test_gae_rewards_round_to_float32_first():
    """r is float32(reward) before any arithmetic: 1 + 2^-30 rounds to 1.0f, so r - V with V = 1 is +0.0 (in float64
    it would be 2^-30), and 0.1 becomes 0.1f."""
    rew = np.array([[1.0 + 2.0 ** -30, 0.1]])
    te = np.ones((1, 2), bool)
    values = np.array([[1.0, 0.0], [0.0, 0.0]], np.float32)
    got = _gae_both(np.float32(0.9), np.float32(0.9), rew, te, np.zeros((1, 2), bool), values,
                    np.zeros((1, 2), np.float32))
    assert got[0].view(np.uint32).tolist() == [0, np.float32(0.1).view(np.uint32)]


def test_gae_minus_zero_deltas():
    """-0.0 deltas keep their sign: a terminated step with reward -0.0 and value +0.0 has delta -0.0 - +0.0 = -0.0;
    a step that is not done, with reward -0.0, value +0.0 and next value -0.0, has (-0.0 + g * -0.0) - +0.0 = -0.0,
    and with gl = 0 its advantage adds 0 * adv[t+1] = -0.0 for a negative adv[t+1], staying -0.0."""
    got = _gae_both(np.float32(0.5), np.float32(0.5), np.array([[-0.0]]), np.ones((1, 1), bool), np.zeros((1, 1), bool),
                    np.array([[0.0], [7.0]], np.float32), np.zeros((1, 1), np.float32))
    assert got.view(np.uint32).tolist() == [[0x80000000]]
    rew = np.array([[-0.0], [-1.0]])
    te = np.array([[0], [1]], bool)
    values = np.array([[0.0], [-0.0], [5.0]], np.float32)
    got = _gae_both(np.float32(0.5), np.float32(0.0), rew, te, np.zeros((2, 1), bool), values,
                    np.zeros((2, 1), np.float32))
    assert got.view(np.uint32)[:, 0].tolist() == [0x80000000, np.float32(-1.0).view(np.uint32)]
