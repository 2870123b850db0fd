"""rollout_mlp_kernel's device source on the CPU (tests/hostsim/rollout_mlp.cpp), against a numpy restatement of the
ReLU MLP policy and T launches of kernel A's driver.

For every classic-control id, with one shared policy and with one per env, one and two hidden layers of several
widths: the actions must be the numpy float32 policy (each unit its bias plus one rounded product at a time, left to
right; ReLU ``z if z > 0 or z is NaN else +0.0``; ``np.argmax``) applied to the observation stream; the outputs and the
float64 state, TimeLimit counters, CartPole flags and PCG64 records must be bit for bit those of T kernel-A steps fed
those actions; and the summary mode must equal a float64 restatement over the full outputs and leave the same state.
"""
import numpy as np
import pytest

from hostsim.rollout_mlp_sim import MlpRolloutSim
from test_rollout_linear_cpu import ENV_IDS, _assert_same, _config, summary_of

HIDDEN = [(1,), (5,), (64,), (3, 7), (64, 64)]
# (N, T): N not a multiple of 256 and a multi-CTA N with short rollouts, a long rollout at a small N
SHAPES = [(1, 1), (31, 2), (257, 37), (33 * 256 + 5, 2), (67, 300)]


def layer_sizes(D, hidden, K):
    return [D] + list(hidden) + [K]


def param_count(D, hidden, K):
    sizes = layer_sizes(D, hidden, K)
    return sum(o * i + o for i, o in zip(sizes[:-1], sizes[1:]))


def relu(z):
    """The documented activation: z if z > 0 or z is NaN, else +0.0."""
    return np.where((z > 0) | np.isnan(z), z, np.float32(0.0))


def mlp_outputs(params, hidden, obs, K):
    """The documented arithmetic in numpy float32, left to right with separate multiply and add.  params (P,) or
    (n, P), obs (n, D) -> (n, K)."""
    n, D = obs.shape
    sizes = layer_sizes(D, hidden, K)
    W = np.broadcast_to(params, (n, params.shape[-1]))
    x, off = obs, 0
    with np.errstate(all="ignore"):
        for layer, (fan_in, fan_out) in enumerate(zip(sizes[:-1], sizes[1:])):
            w = W[:, off:off + fan_out * fan_in].reshape(n, fan_out, fan_in)
            off += fan_out * fan_in
            z = np.array(W[:, off:off + fan_out], dtype=np.float32)
            off += fan_out
            for k in range(fan_in):
                z = z + w[:, :, k] * x[:, None, k]
            x = relu(z) if layer < len(hidden) else z
    assert off == W.shape[1] and x.dtype == np.float32
    return x


def policy(params, hidden, obs, K, discrete):
    z = mlp_outputs(params, hidden, obs, K)
    return np.argmax(z, axis=1).astype(np.int64) if discrete else z


class _Case:
    """An MLP-rollout batch, a kernel-A twin and a summary-mode twin, reset alike."""

    def __init__(self, env_id, N, seed, **kw):
        self.kind, mes, param0, single = _config(env_id)
        mes = kw.pop("max_episode_steps", mes)
        self.discrete = hasattr(single, "n")
        self.ro, self.step, self.summ = [MlpRolloutSim(self.kind, N, max_episode_steps=mes, param0=param0, **kw)
                                         for _ in range(3)]
        self.obs = self.ro.reset(seed)
        for sim in (self.step, self.summ):
            _assert_same(sim.reset(seed), self.obs, "reset")
        self.K = int(single.n) if self.discrete else int(single.shape[0])

    def params(self, rng, hidden, per_env, scale=0.5):
        lead = (self.ro.n,) if per_env else ()
        P = param_count(self.ro.obs_dim, hidden, self.K)
        return (scale * rng.standard_normal(lead + (P,))).astype(np.float32)

    def check(self, params, hidden, T, nan_returns=False):
        """nan_returns: compare NaN returns as NaN, without their sign bit.  numpy and the host build may add a NaN
        reward (a Box kind fed a NaN action) with the operands in either order, which picks either NaN's sign."""
        ro, step = self.ro, self.step
        last = np.zeros((ro.n, ro.obs_dim), dtype=np.float32)
        got = ro.rollout_mlp(params, hidden, T, last_obs=last)
        outs = []
        for t in range(T):
            want = policy(params, hidden, self.obs, self.K, self.discrete)
            _assert_same(got[0][t], want if self.discrete else want.reshape(got[0][t].shape), f"actions[{t}]")
            outs.append(step.step(got[0][t]))
            assert outs[-1][5] == 0, "invalid actions"
            self.obs = outs[-1][0]
        for k, name in enumerate(("obs", "reward", "terminated", "truncated", "final_obs")):
            _assert_same(got[k + 1], np.stack([o[k] for o in outs]), name)
        _assert_same(last, got[1][-1], "last observation buffer")
        for x, y, name in zip(ro.get_state(), step.get_state(), ("state", "elapsed", "flags", "rng")):
            _assert_same(x, y, name)
        last_s = np.zeros_like(last)
        summ = self.summ.rollout_mlp(params, hidden, T, summary=True, last_obs=last_s)
        for x, y, name in zip(summ, summary_of(got[2], got[3], got[4]), ("returns", "lengths", "ended")):
            if nan_returns and name == "returns":
                assert np.array_equal(x, y, equal_nan=True), name
                x, y = np.where(np.isnan(x), 0.0, x), np.where(np.isnan(y), 0.0, y)
            _assert_same(x, y, name)
        _assert_same(last_s, last, "summary: last observation buffer")
        for x, y, name in zip(self.summ.get_state(), ro.get_state(), ("state", "elapsed", "flags", "rng")):
            _assert_same(x, y, f"summary: {name}")
        return got


@pytest.mark.parametrize("per_env", [False, True])
@pytest.mark.parametrize("N,T", SHAPES)
@pytest.mark.parametrize("hidden", HIDDEN)
@pytest.mark.parametrize("env_id", ENV_IDS)
def test_mlp_rollout_equals_policy_and_steps(env_id, hidden, N, T, per_env):
    """Two calls in a row: the second starts from the state the first left."""
    c = _Case(env_id, N, seed=4000 + T + N)
    rng = np.random.default_rng(T * 7919 + N + len(hidden))
    for _ in range(2):
        c.check(c.params(rng, hidden, per_env), hidden, T)


@pytest.mark.parametrize("hidden", [(5,), (64, 64)])
@pytest.mark.parametrize("limit", [None, 4])
@pytest.mark.parametrize("env_id", ENV_IDS)
def test_mlp_rollout_without_autoreset(env_id, limit, hidden):
    """autoreset=False, with and without a short TimeLimit: no resets, CartPole's flag byte in memory."""
    kw = {"autoreset": False} if limit is None else {"autoreset": False, "max_episode_steps": limit}
    c = _Case(env_id, 50, seed=11, **kw)
    c.check(c.params(np.random.default_rng(1), hidden, True), hidden, 60)


@pytest.mark.parametrize("hidden", [(8,), (4, 12)])
@pytest.mark.parametrize("env_id", ENV_IDS)
def test_mlp_rollout_truncates_and_resets(env_id, hidden):
    """max_episode_steps=4: every env ends an episode inside the rollout, is reset inline, and its policy goes on
    from the reset observation; the summary stops at the first end."""
    c = _Case(env_id, 257, seed=13, max_episode_steps=4)
    got = c.check(c.params(np.random.default_rng(2), hidden, False), hidden, 37)
    assert (got[3] | got[4]).any(axis=0).all()


def _pack(layers):
    """[(W (out, in), b (out,)), ...] -> the packed float32 vector."""
    return np.concatenate([np.concatenate([w.ravel(), b]) for w, b in layers]).astype(np.float32)


@pytest.mark.parametrize("env_id", ["CartPole-v1", "MountainCar-v0", "Acrobot-v1"])
def test_tied_and_nan_outputs(env_id):
    """Zero parameters tie every output: action 0.  A NaN hidden unit propagates to every output (the ReLU keeps it),
    so the action is 0, the first NaN, where the finite outputs would choose K - 1."""
    c = _Case(env_id, 64, seed=17)
    K, D, n = c.K, c.ro.obs_dim, c.ro.n
    for hidden in [(3,), (3, 5)]:
        got = c.check(np.zeros(param_count(D, hidden, K), np.float32), hidden, 3)
        assert (got[0] == 0).all()
    hidden = (3,)
    b1 = np.zeros(3, np.float32)
    b3 = np.zeros(K, np.float32)
    b3[K - 1] = 5.0
    ok = _pack([(np.zeros((3, D), np.float32), b1), (np.full((K, 3), 0.25, np.float32), b3)])
    nan = _pack([(np.zeros((3, D), np.float32), np.array([0.0, np.nan, 0.0], np.float32)),
                 (np.full((K, 3), 0.25, np.float32), b3)])
    params = np.stack([nan if i % 2 else ok for i in range(n)])
    got = c.check(params, hidden, 3)
    assert (got[0] == np.where(np.arange(n) % 2 == 1, 0, K - 1)).all()


def test_relu_of_minus_zero_is_plus_zero():
    """A second-layer pre-activation of exactly -0.0 (bias -0.0 plus -1 * +0.0) goes out of the ReLU as +0.0, so the
    Pendulum torque -0.0 + 1 * relu(-0.0) is +0.0; passing -0.0 through would give -0.0."""
    c = _Case("Pendulum-v1", 33, seed=19)
    D = c.ro.obs_dim
    layers = [(np.zeros((2, D), np.float32), np.full(2, -1e30, np.float32)),   # relu(-1e30) = +0.0
              (np.full((1, 2), -1.0, np.float32), np.full(1, -0.0, np.float32)),   # -0.0 + -1 * +0.0 = -0.0
              (np.ones((1, 1), np.float32), np.full(1, -0.0, np.float32))]
    got = c.check(_pack(layers), (2, 1), 4)
    assert (got[0].view(np.uint32) == 0).all(), "every torque must be +0.0"
    r = relu(np.array([-0.0, np.nan, -1.0, 2.0], np.float32))
    assert np.isnan(r[1]) and r[[0, 2, 3]].tobytes() == np.array([0.0, 0.0, 2.0], np.float32).tobytes()


@pytest.mark.parametrize("env_id", ["CartPole-v1", "Pendulum-v1", "Acrobot-v1"])
def test_infinite_weights(env_id):
    """Infinite weights make infinite and NaN (inf * 0, inf - inf) units; the kernel must still be the restatement."""
    c = _Case(env_id, 97, seed=23)
    rng = np.random.default_rng(7)
    for hidden in [(6,), (8, 5)]:
        params = c.params(rng, hidden, True)
        params[rng.random(params.shape) < 0.05] = np.inf
        params[rng.random(params.shape) < 0.05] = -np.inf
        c.check(params, hidden, 5, nan_returns=True)


@pytest.mark.parametrize("hidden", [(5,), (64,), (3, 7), (64, 64)])
@pytest.mark.parametrize("env_id", ["CartPole-v1", "Pendulum-v1", "Acrobot-v1"])
def test_packing_is_parameters_to_vector(env_id, hidden):
    """The packing is torch's: parameters_to_vector of nn.Sequential(Linear, ReLU, ..., Linear) has P entries, and
    the restatement and the host build evaluated on it agree with the module's forward to float32 rounding (the module
    sums in another order, so not bit for bit)."""
    torch = pytest.importorskip("torch")
    c = _Case(env_id, 40, seed=29)
    D, K = c.ro.obs_dim, c.K
    torch.manual_seed(len(hidden) * 100 + hidden[0])
    sizes = layer_sizes(D, hidden, K)
    mods = []
    for i, (fan_in, fan_out) in enumerate(zip(sizes[:-1], sizes[1:])):
        mods += [torch.nn.Linear(fan_in, fan_out)] + ([torch.nn.ReLU()] if i < len(hidden) else [])
    net = torch.nn.Sequential(*mods)
    vec = torch.nn.utils.parameters_to_vector(net.parameters()).detach().numpy().astype(np.float32)
    assert vec.shape == (param_count(D, hidden, K),)
    with torch.no_grad():
        want = net(torch.as_tensor(c.obs)).numpy()
    np.testing.assert_allclose(mlp_outputs(vec, hidden, c.obs, K), want, rtol=1e-5, atol=1e-5)
    acts = c.check(vec, hidden, 1)[0][0]
    if c.discrete:
        z = np.sort(want, axis=1)
        clear = z[:, -1] - z[:, -2] > 1e-4   # no near-tie that float32 rounding could flip
        assert (acts[clear] == np.argmax(want, axis=1)[clear]).all()
    else:
        np.testing.assert_allclose(acts.reshape(want.shape), want, rtol=1e-5, atol=1e-5)
