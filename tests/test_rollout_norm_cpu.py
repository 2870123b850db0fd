"""rollout_mlp_noisy_norm_kernel's, rollout_actor_critic_norm_kernel's and gae_scaled_kernel's device source on the
CPU (tests/hostsim/rollout_norm.cpp), against a numpy restatement: the observations normalised in float64,
``float32((float64(o) - mean) / sqrt(var + eps))`` clamped to [-c, c], then test_rollout_mlp_cpu's float32 MLP on
them, and the rewards the advantages read scaled as ``float32(reward / sqrt(var + eps))`` clamped to [-c_r, c_r].

The env outputs stay raw: obs, rewards and final observations must be those of T kernel-A steps of a twin batch fed
the same actions.  The identity statistics (mean 0, var 1, eps 0, no clip) must give the drivers without
normalisation byte for byte.  The edges are pinned on hand-made inputs: var = -eps (sd = 0: infinite and NaN inputs),
NaN through the clip, -0.0, clip bounds hit exactly, and rewards scaled to +-inf.
"""
import numpy as np
import pytest

import test_rollout_mlp_cpu as mlp_cpu
from hostsim.rollout_norm_sim import RELU, TANH, NormRolloutSim, gae_scaled, norm_elems
from test_rollout_actor_critic_cpu import _assert_same_nan, coefficients, gae_restated
from test_rollout_linear_cpu import ENV_IDS, _assert_same, _config
from test_rollout_mlp_cpu import mlp_outputs, param_count
from test_rollout_mlp_noisy_cpu import _assert_actions, noisy_action

HIDDEN = [(16,), (64,), (64, 64)]
SHAPES = [(1, 1), (257, 37), (33 * 256 + 5, 2), (67, 120)]
CLIPS = [None, 0.75]


def norm_restated(o, mean, var, eps, clip):
    """float32((float64(o) - mean) / sqrt(var + eps)), clamped with torch.clamp's rule (NaN stays NaN)."""
    with np.errstate(all="ignore"):
        x = ((o.astype(np.float64) - mean) / np.sqrt(var + eps)).astype(np.float32)
        if clip is not None:
            c = np.float32(clip)
            x = np.where(x < -c, -c, np.where(x > c, c, x)).astype(np.float32)
    return x


def scale_rewards(rew, ret_var, eps, clip):
    """float32(reward / sqrt(var + eps)) in float64, clamped as the observations."""
    with np.errstate(all="ignore"):
        r = (rew / np.sqrt(np.float64(ret_var) + eps)).astype(np.float32)
        if clip is not None:
            c = np.float32(clip)
            r = np.where(r < -c, -c, np.where(r > c, c, r)).astype(np.float32)
    return r


class _Case:
    """A batch for the normalised drivers and a kernel-A twin, reset alike, with statistics near the observations'."""

    def __init__(self, env_id, N, seed, **kw):
        self.kind, mes, param0, single = _config(env_id)
        mes = kw.pop("max_episode_steps", mes)
        self.discrete = hasattr(single, "n")
        self.ro, self.step = [NormRolloutSim(self.kind, N, max_episode_steps=mes, param0=param0, **kw)
                              for _ in range(2)]
        self.obs = self.ro.reset(seed)
        _assert_same(self.step.reset(seed), self.obs, "reset")
        self.K = int(single.n) if self.discrete else int(single.shape[0])
        self.D = self.ro.obs_dim

    def stats(self, rng):
        return rng.standard_normal(self.D) * 0.3, rng.random(self.D) * 2.0 + 0.01

    def nets(self, rng, hidden, scale=0.5):
        return ((scale * rng.standard_normal(param_count(self.D, hidden, self.K))).astype(np.float32),
                (scale * rng.standard_normal(param_count(self.D, hidden, 1))).astype(np.float32))

    def noise(self, rng, T):
        return rng.standard_normal((T, self.ro.n, self.K)).astype(np.float32)

    def _env_outputs(self, got, outs, last):
        for k, name in enumerate(("obs", "reward", "terminated", "truncated", "final_obs")):
            _assert_same(got[k], np.stack([o[k] for o in outs]), name)
        _assert_same(last, got[0][-1], "last observation buffer")
        for x, y, name in zip(self.ro.get_state(), self.step.get_state(), ("state", "elapsed", "flags", "rng")):
            _assert_same(x, y, name)

    def check_noisy(self, params, hidden, noise, mean, var, eps, clip, act=RELU):
        T = noise.shape[0]
        last = np.zeros((self.ro.n, self.D), dtype=np.float32)
        got = self.ro.rollout_mlp_noisy_norm(params, hidden, noise, mean, var, eps, clip, act, last_obs=last)
        outs = []
        for t in range(T):
            z = mlp_outputs(params, hidden, norm_restated(self.obs, mean, var, eps, clip), self.K)
            _assert_same(got[1][t], z, f"outputs[{t}]")
            _assert_actions(got[0][t], noisy_action(z, noise[t], self.discrete), f"actions[{t}]")
            outs.append(self.step.step(got[0][t]))
            assert outs[-1][5] == 0, "invalid actions"
            self.obs = outs[-1][0]
        self._env_outputs(got[2:], outs, last)
        return got

    def check_ac(self, actor, critic, hidden, noise, mean, var, eps, clip, ret_var=None, clip_r=None, gamma=0.99,
                 gae_lambda=0.95, act=RELU):
        T = noise.shape[0]
        g, gl = coefficients(gamma, gae_lambda)
        last = np.zeros((self.ro.n, self.D), dtype=np.float32)
        got = self.ro.rollout_actor_critic_norm(actor, critic, hidden, noise, g, gl, mean, var, eps, clip, ret_var,
                                                clip_r, act, last_obs=last)
        acts, outs_z, values, adv = got[:4]
        outs, vf = [], np.full((T, self.ro.n), np.nan, np.float32)
        V = lambda o: mlp_outputs(critic, hidden, norm_restated(o, mean, var, eps, clip), 1)[:, 0]  # noqa: E731
        for t in range(T):
            z = mlp_outputs(actor, hidden, norm_restated(self.obs, mean, var, eps, clip), self.K)
            _assert_same(outs_z[t], z, f"outputs[{t}]")
            _assert_same(values[t], V(self.obs), f"values[{t}]")
            _assert_actions(acts[t], noisy_action(z, noise[t], self.discrete), f"actions[{t}]")
            outs.append(self.step.step(acts[t]))
            assert outs[-1][5] == 0, "invalid actions"
            o, _, te, tr, fo = outs[-1][:5]
            held = tr.astype(bool) & ~te.astype(bool)
            if held.any():
                vf[t, held] = V(fo[held])
            self.obs = o
        _assert_same(values[T], V(self.obs), "values[T]")
        self._env_outputs(got[4:], outs, last)
        rew = got[5] if ret_var is None else scale_rewards(got[5], ret_var, eps, clip_r)
        _assert_same_nan(adv, gae_restated(g, gl, rew, got[6], got[7], values, vf), "advantages")
        return got


@pytest.fixture
def tanh(monkeypatch):
    """The numpy MLP with the C library's tanhf, which the host build's tanh instantiation calls."""
    from test_rollout_mlp_tanh_cpu import libm_tanhf
    monkeypatch.setattr(mlp_cpu, "relu", libm_tanhf)


@pytest.mark.parametrize("clip", CLIPS)
@pytest.mark.parametrize("N,T", SHAPES)
@pytest.mark.parametrize("hidden", HIDDEN)
@pytest.mark.parametrize("env_id", ENV_IDS)
def test_noisy_norm_equals_restatement(env_id, hidden, N, T, clip):
    c = _Case(env_id, N, seed=500 + N + T)
    rng = np.random.default_rng(N * 31 + T + len(hidden))
    mean, var = c.stats(rng)
    a, _ = c.nets(rng, hidden)
    c.check_noisy(a, hidden, c.noise(rng, T), mean, var, 1e-8, clip)
    c.check_noisy(a, hidden, c.noise(rng, 2), mean, var, 1e-8, clip)          # continues from the state left


@pytest.mark.parametrize("clips", [(None, None), (0.75, None), (None, 0.4), (1.5, 0.4)])
@pytest.mark.parametrize("N,T", SHAPES)
@pytest.mark.parametrize("hidden", HIDDEN)
@pytest.mark.parametrize("env_id", ENV_IDS)
def test_actor_critic_norm_equals_restatement(env_id, hidden, N, T, clips):
    """Two calls in a row; the second's values[0] is the first's values[T]."""
    c = _Case(env_id, N, seed=900 + N + T)
    rng = np.random.default_rng(N * 17 + T + len(hidden))
    mean, var = c.stats(rng)
    a, v = c.nets(rng, hidden)
    first = c.check_ac(a, v, hidden, c.noise(rng, T), mean, var, 1e-8, clips[0], 2.5, clips[1])
    second = c.check_ac(a, v, hidden, c.noise(rng, T), mean, var, 1e-8, clips[0], 2.5, clips[1])
    _assert_same(second[2][0], first[2][-1], "values[0] of the next call")


@pytest.mark.parametrize("hidden", [(5,), (64, 64)])
@pytest.mark.parametrize("env_id", ENV_IDS)
def test_tanh_norm_equals_restatement(tanh, env_id, hidden):
    c = _Case(env_id, 67, seed=81, max_episode_steps=6)
    rng = np.random.default_rng(9)
    mean, var = c.stats(rng)
    a, v = c.nets(rng, hidden)
    c.check_noisy(a, hidden, c.noise(rng, 20), mean, var, 1e-8, 0.9, act=TANH)
    c.check_ac(a, v, hidden, c.noise(rng, 20), mean, var, 1e-5, 0.9, 0.7, 3.0, act=TANH)


@pytest.mark.parametrize("env_id", ENV_IDS)
def test_truncations_bootstrap_from_the_normalised_final_observation(env_id):
    """max_episode_steps=4: most envs truncate inside the call without terminating, and their bootstrap is the critic
    of the normalised final observation."""
    c = _Case(env_id, 257, seed=14, max_episode_steps=4)
    rng = np.random.default_rng(2)
    mean, var = c.stats(rng)
    a, v = c.nets(rng, (8, 6))
    got = c.check_ac(a, v, (8, 6), c.noise(rng, 37), mean, var, 1e-8, 0.5, 0.3, 1.0)
    assert (got[7] & ~got[6]).any(axis=0).all()


@pytest.mark.parametrize("hidden", [(16,), (64, 64)])
@pytest.mark.parametrize("env_id", ENV_IDS)
def test_identity_statistics_give_the_drivers_without_normalisation(env_id, hidden):
    """mean 0, var 1, eps 0, no clip: x = float32(float64(o) / 1) = o, and float32(reward / 1) = float32(reward), so
    every output is byte for byte that of rollout_mlp_noisy_env / rollout_actor_critic_env and gae_env."""
    kind, mes, param0, single = _config(env_id)
    sims = [NormRolloutSim(kind, 300, max_episode_steps=7, param0=param0) for _ in range(4)]
    for s in sims:
        s.reset(33)
    D = sims[0].obs_dim
    K = int(single.n) if hasattr(single, "n") else int(single.shape[0])
    rng = np.random.default_rng(4)
    a = (0.5 * rng.standard_normal(param_count(D, hidden, K))).astype(np.float32)
    v = (0.5 * rng.standard_normal(param_count(D, hidden, 1))).astype(np.float32)
    e = rng.standard_normal((25, 300, K)).astype(np.float32)
    mean, var = np.zeros(D), np.ones(D)
    g, gl = coefficients(0.99, 0.95)
    for got, want, name in (
            (sims[0].rollout_mlp_noisy_norm(a, hidden, e, mean, var, 0.0, None), sims[1].rollout_mlp_noisy(a, hidden, e),
             "rollout_mlp_noisy"),
            (sims[2].rollout_actor_critic_norm(a, v, hidden, e, g, gl, mean, var, 0.0, None, 1.0, None),
             sims[3].rollout_actor_critic(a, v, hidden, e, g, gl), "rollout_actor_critic")):
        assert len(got) == len(want)
        for k, (x, y) in enumerate(zip(got, want)):
            _assert_same(x, y, f"{name} output {k}")
    for x, y in zip(sims[0].get_state(), sims[1].get_state()):
        _assert_same(x, y, "state")


# ----------------------------------------------------------------------------------------------- edges by hand
def _bits(x):
    return np.asarray(x, np.float32).view(np.uint32).tolist()


def test_zero_sd_gives_infinite_and_nan_inputs():
    """var = -eps: sd = 0, so o > mean gives +inf, o < mean -inf and o = mean NaN (0 / 0); the clip takes the
    infinities to +-c and leaves NaN."""
    o = np.array([1.0, -1.0, 0.5], np.float32)
    x = norm_elems(o, 0.5, -1e-8, 1e-8, None)
    assert x[0] == np.inf and x[1] == -np.inf and np.isnan(x[2])
    x = norm_elems(o, 0.5, -1e-8, 1e-8, 10.0)
    assert x[0] == np.float32(10.0) and x[1] == np.float32(-10.0) and np.isnan(x[2])
    _assert_same_nan(x, norm_restated(o, 0.5, -1e-8, 1e-8, 10.0), "restated")


def test_nan_passes_through_the_clip():
    o = np.array([np.nan, -np.nan, np.inf, -np.inf], np.float32)
    x = norm_elems(o, 0.0, 1.0, 0.0, 2.0)
    assert np.isnan(x[:2]).all() and x[2] == np.float32(2.0) and x[3] == np.float32(-2.0)


def test_minus_zero_keeps_its_sign():
    """-0.0 - (+0.0) = -0.0, / 1 = -0.0, not clamped; +0.0 stays +0.0; and -0.0 - (-0.0) = +0.0."""
    o = np.array([-0.0, 0.0], np.float32)
    assert _bits(norm_elems(o, 0.0, 1.0, 0.0, 1.0)) == [0x80000000, 0]
    assert _bits(norm_elems(o, -0.0, 1.0, 0.0, None)) == [0, 0]


def test_clip_bounds_hit_exactly():
    """x equal to +-c is returned as is; the nearest float32 values beyond it are clamped, those inside are not; and
    the clamp compares the float32 x with float32(c), so a value that rounds to c in float32 is not clamped below
    it."""
    c = np.float32(0.1)
    o = np.array([c, -c, np.nextafter(c, np.float32(1)), -np.nextafter(c, np.float32(1)),
                  np.nextafter(c, np.float32(0))], np.float32)
    x = norm_elems(o, 0.0, 1.0, 0.0, 0.1)
    assert _bits(x) == _bits([c, -c, c, -c, o[4]])
    _assert_same(x, norm_restated(o, 0.0, 1.0, 0.0, 0.1), "restated")


def test_rewards_scaled_to_infinity():
    """A return variance of -eps makes sd = 0: rewards of +-1 scale to +-inf (0 to NaN).  Clipped they become +-c_r;
    unclipped the advantages follow IEEE arithmetic."""
    rew = np.array([[1.0, -1.0, 0.0, 2.0]])
    te = np.ones((1, 4), bool)
    tr = np.zeros((1, 4), bool)
    values = np.array([[0.5] * 4, [0.0] * 4], np.float32)
    held = np.zeros((1, 4), np.float32)
    g, gl = np.float32(0.9), np.float32(0.9)
    got = gae_scaled(g, gl, -1e-8, 1e-8, 5.0, rew, te, tr, values, held)
    assert got[0, :2].tolist() == [4.5, -5.5] and np.isnan(got[0, 2]) and got[0, 3] == np.float32(4.5)
    got = gae_scaled(g, gl, -1e-8, 1e-8, None, rew, te, tr, values, held)
    assert got[0, 0] == np.inf and got[0, 1] == -np.inf and np.isnan(got[0, 2])


@pytest.mark.parametrize("clip_r", [None, 0.3])
@pytest.mark.parametrize("gamma,gae_lambda", [(0.99, 0.95), (0.0, 0.5), (1.0, 1.0)])
def test_gae_scaled_random_rows(gamma, gae_lambda, clip_r):
    rng = np.random.default_rng(int(gamma * 100 + gae_lambda * 10))
    T, n = 50, 300
    rew = rng.standard_normal((T, n)) * 3
    te, tr = rng.random((T, n)) < 0.07, rng.random((T, n)) < 0.07
    values = rng.standard_normal((T + 1, n)).astype(np.float32)
    vf = rng.standard_normal((T, n)).astype(np.float32)
    held = np.where(tr & ~te, vf, np.float32(np.nan)).astype(np.float32)
    g, gl = coefficients(gamma, gae_lambda)
    got = gae_scaled(g, gl, 7.3, 1e-8, clip_r, rew, te, tr, values, held)
    want = gae_restated(g, gl, scale_rewards(rew, 7.3, 1e-8, clip_r), te, tr, values, vf)
    _assert_same_nan(got, want, "advantages")
