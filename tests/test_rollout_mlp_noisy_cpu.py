"""rollout_mlp_noisy_kernel's device source on the CPU (tests/hostsim/rollout_mlp_noisy.cpp), against a numpy
restatement of the ReLU MLP policy plus the caller's noise and T launches of kernel A's driver.

For every classic-control id, with one shared policy and with one per env: the outputs must be the numpy float32 MLP
(test_rollout_mlp_cpu.mlp_outputs) of the observation stream; the actions ``np.argmax(z + noise[t])`` (Discrete) or
``z + noise[t]`` (Box), each sum one rounded float32 add; the env outputs and the float64 state, TimeLimit counters,
CartPole flags and PCG64 records bit for bit those of T kernel-A steps fed those actions.  NaN and infinite noise
follow IEEE float32, and noise of -0.0 everywhere reproduces rollout_mlp bit for bit.
"""
import numpy as np
import pytest

from hostsim.rollout_mlp_noisy_sim import MlpNoisyRolloutSim
from test_rollout_linear_cpu import ENV_IDS, _assert_same, _config
from test_rollout_mlp_cpu import _pack, mlp_outputs, param_count

HIDDEN = [(1,), (64,), (3, 7), (64, 64)]
# (N, T): N not a multiple of 256 and a multi-CTA N with short rollouts, a long rollout at a small N
SHAPES = [(1, 1), (257, 37), (33 * 256 + 5, 2), (67, 300)]


def noisy_action(z, e, discrete):
    """The documented rule: y = z + noise, one float32 add per element; np.argmax(y) (first NaN, else first maximum)
    for Discrete, y for Box."""
    with np.errstate(all="ignore"):
        y = z + e
    assert y.dtype == np.float32
    return np.argmax(y, axis=1).astype(np.int64) if discrete else y


def _assert_actions(got, want, what):
    """Bit for bit, except that a NaN Box action need only be NaN: numpy and the host build may return either NaN
    operand of a sum of two NaNs."""
    want = want.reshape(got.shape)
    if got.dtype == np.float32:
        nan = np.isnan(want)
        assert np.array_equal(np.isnan(got), nan), f"{what}: NaN positions differ"
        got, want = np.where(nan, 0.0, got).astype(np.float32), np.where(nan, 0.0, want).astype(np.float32)
    _assert_same(got, want, what)


class _Case:
    """A noisy MLP-rollout batch and a kernel-A twin, reset alike."""

    def __init__(self, env_id, N, seed, **kw):
        self.kind, mes, param0, single = _config(env_id)
        mes = kw.pop("max_episode_steps", mes)
        self.discrete = hasattr(single, "n")
        self.ro, self.step, self.plain = [MlpNoisyRolloutSim(self.kind, N, max_episode_steps=mes, param0=param0, **kw)
                                          for _ in range(3)]
        self.obs = self.ro.reset(seed)
        for sim in (self.step, self.plain):
            _assert_same(sim.reset(seed), self.obs, "reset")
        self.K = int(single.n) if self.discrete else int(single.shape[0])

    def params(self, rng, hidden, per_env, scale=0.5):
        lead = (self.ro.n,) if per_env else ()
        P = param_count(self.ro.obs_dim, hidden, self.K)
        return (scale * rng.standard_normal(lead + (P,))).astype(np.float32)

    def noise(self, rng, T, scale=1.0):
        return (scale * rng.standard_normal((T, self.ro.n, self.K))).astype(np.float32)

    def check(self, params, hidden, noise):
        ro, step = self.ro, self.step
        T = noise.shape[0]
        last = np.zeros((ro.n, ro.obs_dim), dtype=np.float32)
        got = ro.rollout_mlp_noisy(params, hidden, noise, last_obs=last)
        acts, outs_z = got[0], got[1]
        assert outs_z.shape == (T, ro.n, self.K) and outs_z.dtype == np.float32
        outs = []
        for t in range(T):
            z = mlp_outputs(params, hidden, self.obs, self.K)
            _assert_same(outs_z[t], z, f"outputs[{t}]")
            _assert_actions(acts[t], noisy_action(z, noise[t], self.discrete), f"actions[{t}]")
            outs.append(step.step(acts[t]))
            assert outs[-1][5] == 0, "invalid actions"
            self.obs = outs[-1][0]
        for k, name in enumerate(("obs", "reward", "terminated", "truncated", "final_obs")):
            _assert_same(got[k + 2], np.stack([o[k] for o in outs]), name)
        _assert_same(last, got[2][-1], "last observation buffer")
        for x, y, name in zip(ro.get_state(), step.get_state(), ("state", "elapsed", "flags", "rng")):
            _assert_same(x, y, name)
        return got


@pytest.mark.parametrize("per_env", [False, True])
@pytest.mark.parametrize("N,T", SHAPES)
@pytest.mark.parametrize("hidden", HIDDEN)
@pytest.mark.parametrize("env_id", ENV_IDS)
def test_noisy_rollout_equals_policy_and_steps(env_id, hidden, N, T, per_env):
    """Two calls in a row: the second starts from the state the first left."""
    c = _Case(env_id, N, seed=5000 + T + N)
    rng = np.random.default_rng(T * 7919 + N + len(hidden))
    for _ in range(2):
        c.check(c.params(rng, hidden, per_env), hidden, c.noise(rng, T))


@pytest.mark.parametrize("hidden", [(5,), (64, 64)])
@pytest.mark.parametrize("limit", [None, 4])
@pytest.mark.parametrize("env_id", ENV_IDS)
def test_noisy_rollout_without_autoreset(env_id, limit, hidden):
    """autoreset=False, with and without a short TimeLimit: no resets, CartPole's flag byte in memory."""
    kw = {"autoreset": False} if limit is None else {"autoreset": False, "max_episode_steps": limit}
    c = _Case(env_id, 50, seed=12, **kw)
    rng = np.random.default_rng(1)
    c.check(c.params(rng, hidden, True), hidden, c.noise(rng, 60))


@pytest.mark.parametrize("hidden", [(8,), (4, 12)])
@pytest.mark.parametrize("env_id", ENV_IDS)
def test_noisy_rollout_truncates_and_resets(env_id, hidden):
    """max_episode_steps=4: every env ends an episode inside the rollout, is reset inline, and its policy goes on
    from the reset observation."""
    c = _Case(env_id, 257, seed=14, max_episode_steps=4)
    rng = np.random.default_rng(2)
    got = c.check(c.params(rng, hidden, False), hidden, c.noise(rng, 37))
    assert (got[4] | got[5]).any(axis=0).all()


@pytest.mark.parametrize("per_env", [False, True])
@pytest.mark.parametrize("hidden", [(5,), (3, 7), (64, 64)])
@pytest.mark.parametrize("env_id", ENV_IDS)
def test_minus_zero_noise_is_rollout_mlp(env_id, hidden, per_env):
    """Noise of -0.0 everywhere: z + (-0.0) is z for every float32 z, -0.0 and NaN included, so actions, env outputs
    and state are rollout_mlp's bit for bit, and the outputs are its actions' source."""
    c = _Case(env_id, 300, seed=31)
    rng = np.random.default_rng(3)
    p = c.params(rng, hidden, per_env)
    T = 40
    noise = np.full((T, c.ro.n, c.K), -0.0, np.float32)
    got = c.ro.rollout_mlp_noisy(p, hidden, noise)
    want = c.plain.rollout_mlp(p, hidden, T)
    _assert_same(got[0], want[0], "actions")
    for k, name in enumerate(("obs", "reward", "terminated", "truncated", "final_obs")):
        _assert_same(got[k + 2], want[k + 1], name)
    for x, y, name in zip(c.ro.get_state(), c.plain.get_state(), ("state", "elapsed", "flags", "rng")):
        _assert_same(x, y, name)
    if c.discrete:
        _assert_same(got[0], np.argmax(got[1], axis=2).astype(np.int64), "argmax of the outputs")
    else:
        _assert_same(got[0], got[1], "Box actions are the outputs")


def test_minus_zero_output_keeps_its_sign_only_under_minus_zero_noise():
    """A Pendulum output of exactly -0.0 (bias -0.0 plus -1 * relu(...) = -0.0): -0.0 noise keeps the torque -0.0, as
    rollout_mlp gives it, while +0.0 noise makes it +0.0."""
    D = 3
    layers = [(np.zeros((2, D), np.float32), np.full(2, -1e30, np.float32)),   # relu(-1e30) = +0.0
              (np.full((1, 2), -1.0, np.float32), np.full(1, -0.0, np.float32))]   # -0.0 + -1 * +0.0 = -0.0
    p = _pack(layers)
    for fill, bits in ((-0.0, 0x80000000), (0.0, 0)):
        c = _Case("Pendulum-v1", 33, seed=19)
        noise = np.full((4, 33, 1), fill, np.float32)
        got = c.check(p, (2,), noise)
        assert (got[1].view(np.uint32) == 0x80000000).all(), "every output must be -0.0"
        assert (got[0].view(np.uint32) == bits).all(), f"noise {fill}: every torque must have bits {bits:#x}"
    want = c.plain.rollout_mlp(p, (2,), 4)[0]
    assert (want.view(np.uint32) == 0x80000000).all()


@pytest.mark.parametrize("env_id", ["CartPole-v1", "MountainCar-v0", "Acrobot-v1"])
def test_discrete_nan_inf_noise_and_ties(env_id):
    """Zero parameters make every output +0.0, so the action is np.argmax of the noise row itself:
    - -inf on choice 0 and finite elsewhere: 0 is never picked;
    - +inf on the last choice: picked, unless a NaN comes first;
    - NaN anywhere: the first NaN is picked;
    - equal noise on every choice, or a tie at the maximum: the first of the tied choices.
    With an output of +inf on choice 0, -inf noise there makes NaN, which is then picked."""
    c = _Case(env_id, 600, seed=37)
    K, D, n = c.K, c.ro.obs_dim, c.ro.n
    rng = np.random.default_rng(5)
    T = 6
    noise = c.noise(rng, T)
    kind = np.arange(n) % 6
    noise[:, kind == 0, 0] = -np.inf
    noise[:, kind == 1, K - 1] = np.inf
    noise[:, kind == 2, K - 1] = np.nan
    noise[:, kind == 3] = 0.5
    noise[:, kind == 4, 1:] = 2.0                     # ties between choices 1 .. K-1 at the maximum
    noise[:, kind == 4, 0] = 1.0
    noise[:, kind == 5, K - 1] = np.inf
    noise[:, kind == 5, 1] = np.nan                   # the first NaN, before an +inf (CartPole: in its place)
    hidden = (3,)
    got = c.check(np.zeros(param_count(D, hidden, K), np.float32), hidden, noise)
    a = got[0]
    assert (a[:, kind == 0] != 0).all()
    assert (a[:, kind == 1] == K - 1).all() and (a[:, kind == 2] == K - 1).all()
    assert (a[:, kind == 3] == 0).all() and (a[:, kind == 4] == 1).all() and (a[:, kind == 5] == 1).all()
    # an output of +inf on choice 0: -inf noise there gives NaN, the first NaN is choice 0
    b3 = np.zeros(K, np.float32)
    b3[0] = np.inf
    p = _pack([(np.zeros((3, D), np.float32), np.zeros(3, np.float32)), (np.zeros((K, 3), np.float32), b3)])
    noise = c.noise(rng, T)
    noise[:, :, 0] = -np.inf
    got = c.check(p, hidden, noise)
    assert np.isnan(got[1][:, :, 0]).sum() == 0 and (got[0] == 0).all()


@pytest.mark.parametrize("env_id", ["MountainCarContinuous-v0", "Pendulum-v1"])
def test_box_nan_inf_noise(env_id):
    """Box kinds: the action is z + noise, so +-inf and NaN noise reach the step as +-inf and NaN torques, which the
    step then takes exactly as kernel A takes them."""
    c = _Case(env_id, 300, seed=41)
    rng = np.random.default_rng(6)
    T = 8
    noise = c.noise(rng, T)
    kind = np.arange(c.ro.n) % 4
    noise[:, kind == 0] = np.inf
    noise[:, kind == 1] = -np.inf
    noise[:, kind == 2] = np.nan
    got = c.check(c.params(rng, (6,), True), (6,), noise)
    a = got[0][..., 0]
    assert np.isposinf(a[:, kind == 0]).all() and np.isneginf(a[:, kind == 1]).all()
    assert np.isnan(a[:, kind == 2]).all() and np.isfinite(a[:, kind == 3]).all()
