"""rollout_from_mlp_kernel's device source on the CPU (tests/hostsim/rollout_from_mlp.cpp), against the existing MLP
rollout drivers run on a batch restored from the same snapshot rows.

A root batch is reset and stepped, and its state is packed into snapshot rows (test_rollout_from_cpu's restatement of
the row layout).  Each rollout_from_mlp call is compared with its twin: a batch of B envs restored from the gathered
rows and rolled out in full mode by rollout_mlp_env (no noise, raw inputs), rollout_mlp_norm_env (no noise,
normalised inputs), rollout_mlp_noisy_env (noise, raw inputs) or rollout_mlp_noisy_norm_env (noise, normalised
inputs), its rewards and flags folded over the first episode end.  Returns, lengths, end flags, the step-0 actions and
the end observations must match bit for bit and the end rows byte for byte.
"""
import numpy as np
import pytest

from hostsim.rollout_from_mlp_sim import RELU, TANH, RolloutFromMlpSim
from hostsim.rollout_mlp_noisy_sim import MlpNoisyRolloutSim
from hostsim.rollout_mlp_tanh_sim import MlpTanhRolloutSim
from hostsim.rollout_norm_sim import NormRolloutSim
from hostsim.rollout_policy_norm_sim import PolicyNormRolloutSim
from test_rollout_from_cpu import _assert_same, _config, load_rows, pack_rows, row_layout, summary_of

ENV_IDS = ["CartPole-v0", "CartPole-v1", "MountainCar-v0", "MountainCarContinuous-v0", "Pendulum-v1", "Acrobot-v1"]
# one hidden layer with h1 % 4 == 0, two without, two with
HIDDEN = [(8,), (6, 5), (16, 12)]


def _param_count(D, hidden, K):
    sizes = [D] + list(hidden) + [K]
    return sum(o * i + o for i, o in zip(sizes[:-1], sizes[1:]))


# (per-branch rows, noise, obs_norm): every combination but noise with per-branch rows and obs_norm, which is refused
POLICIES = [(pb, noisy, norm) for pb in (False, True) for noisy in (False, True) for norm in (False, True)
            if not (pb and noisy and norm)]


class _Case:
    """A root batch of N envs, reset and stepped `warm` times, its snapshot rows, and a policy generator."""

    def __init__(self, env_id, N, seed, warm=3, **kw):
        self.kind, mes, self.param0, self.single = _config(env_id)
        self.kw = {"max_episode_steps": mes, **kw}
        self.discrete = hasattr(self.single, "n")
        self.K = int(self.single.n) if self.discrete else 1
        self.root = RolloutFromMlpSim(self.kind, N, param0=self.param0, **self.kw)
        self.root.reset(seed)
        self.D = self.root.obs_dim
        self.rng = np.random.default_rng(seed)
        for _ in range(warm):
            if self.discrete:
                a = self.rng.integers(0, self.K, size=N).astype(np.int64)
            else:
                a = self.rng.uniform(-2.0, 2.0, size=(N, 1)).astype(np.float32)
            self.root.step(a)
        self.rows = pack_rows(self.root)

    def params(self, hidden, B=None):
        P = _param_count(self.D, hidden, self.K)
        shape = (P,) if B is None else (B, P)
        return (0.6 * self.rng.standard_normal(shape)).astype(np.float32)

    def noise(self, T, B):
        if self.discrete:
            u = np.maximum(self.rng.random((T, B, self.K)), np.finfo(np.float32).tiny)
            return (-np.log(-np.log(u))).astype(np.float32)
        return (0.5 * self.rng.standard_normal((T, B, self.K))).astype(np.float32)

    def stats(self):
        mean = self.rng.standard_normal(self.D)
        var = self.rng.uniform(0.05, 3.0, self.D)
        return mean, var

    def twin(self, rows, params, hidden, T, noise, act, mean, var, eps, clip):
        """The restored twin's full rollout -> (actions, rewards, terminated, truncated, last obs, twin)."""
        B = rows.shape[0]
        if noise is None and mean is None:
            t = (MlpTanhRolloutSim if act == TANH else MlpNoisyRolloutSim)(self.kind, B, param0=self.param0, **self.kw)
        elif noise is None:
            t = PolicyNormRolloutSim(self.kind, B, param0=self.param0, **self.kw)
        elif mean is None:
            t = (MlpTanhRolloutSim if act == TANH else MlpNoisyRolloutSim)(self.kind, B, param0=self.param0, **self.kw)
        else:
            t = NormRolloutSim(self.kind, B, param0=self.param0, **self.kw)
        load_rows(t, rows)
        last = np.zeros((B, self.D), dtype=np.float32)
        if noise is None and mean is None:
            acts, _, rew, te, tr, _ = t.rollout_mlp(params, hidden, T, last_obs=last)
        elif noise is None:
            acts, _, rew, te, tr, _ = t.rollout_mlp_norm(params, hidden, T, mean, var, eps, clip, act=act, last_obs=last)
        elif mean is None:
            acts, _, _, rew, te, tr, _ = t.rollout_mlp_noisy(params, hidden, noise, last_obs=last)
        else:
            acts, _, _, rew, te, tr, _ = t.rollout_mlp_noisy_norm(params, hidden, noise, mean, var, eps, clip, act=act,
                                                                 last_obs=last)
        return acts, rew, te, tr, last, t

    def check(self, hidden, T, row_idx=None, rows=None, per_branch=False, noisy=False, act=RELU, norm=False,
              clip=None, eps=1e-8):
        """rollout_from_mlp against its twin, with and without end states -> (the twin's summary, the outputs)."""
        rows = self.rows if rows is None else rows
        idx = np.arange(rows.shape[0]) if row_idx is None else np.asarray(row_idx)
        B = idx.shape[0]
        params = self.params(hidden, B if per_branch else None)
        noise = self.noise(T, B) if noisy else None
        mean, var = self.stats() if norm else (None, None)
        kw = dict(row_idx=row_idx, noise=noise, act=act, mean=mean, var=var, eps=eps, clip=clip)
        before = [x.copy() for x in self.root.get_state()]
        got = self.root.rollout_from_mlp(rows, params, hidden, T, states=True, **kw)
        plain = self.root.rollout_from_mlp(rows, params, hidden, T, states=False, **kw)
        for x, y, name in zip(plain[:4], got[:4], ("returns", "lengths", "ended", "first actions")):
            _assert_same(x, y, f"states=False: {name}")
        for x, y, name in zip(self.root.get_state(), before, ("state", "elapsed", "flags", "rng")):
            _assert_same(x, y, f"root batch {name} moved")
        ok = (idx >= 0) & (idx < rows.shape[0])
        assert got[7] == int(not ok.all()), "index-error flag"
        assert got[6] == 0, "a policy's actions are always valid"
        acts, rew, te, tr, last, twin = self.twin(rows[np.where(ok, idx, 0)], params, hidden, T, noise, act, mean,
                                                  var, eps, clip)
        want = summary_of(rew, te, tr)
        end_rows, end_obs, first = pack_rows(twin), last, acts[0].copy()
        # a skipped branch: zero summary, action, end row and observation
        want = (np.where(ok, want[0], 0.0), np.where(ok, want[1], 0).astype(np.int32), want[2] & ok)
        first[~ok] = 0
        end_rows[~ok] = 0
        end_obs[~ok] = 0.0
        for x, y, name in zip(got[:3], want, ("returns", "lengths", "ended")):
            _assert_same(x, y, name)
        _assert_same(got[3], first, "first actions")
        _assert_same(got[4], end_rows, "end rows")
        _assert_same(got[5], end_obs, "end observations")
        return want, got


@pytest.mark.parametrize("per_branch,noisy,norm", POLICIES)
@pytest.mark.parametrize("hidden", HIDDEN)
@pytest.mark.parametrize("act", [RELU, TANH])
@pytest.mark.parametrize("env_id", ENV_IDS)
def test_matches_restored_twin(env_id, act, hidden, per_branch, noisy, norm):
    """Every classic id, both activations, three widths, shared and per-branch policies, with and without noise and
    normalised inputs (noise with per-branch rows and obs_norm has no twin and is refused), from random rows with
    duplicates, B = 300 (not a multiple of 256)."""
    c = _Case(env_id, 64, seed=100 + 7 * act + len(hidden) + hidden[0])
    idx = c.rng.integers(0, 64, size=300)
    c.check(hidden, 23, idx, per_branch=per_branch, noisy=noisy, act=act, norm=norm)


@pytest.mark.parametrize("noisy", [False, True])
@pytest.mark.parametrize("env_id", ENV_IDS)
def test_clip_obs(env_id, noisy):
    """clip_obs small enough to clamp most inputs, and a zero epsilon."""
    c = _Case(env_id, 40, seed=21)
    c.check((8, 8), 17, per_branch=not noisy, noisy=noisy, act=TANH, norm=True, clip=0.25, eps=0.0)


@pytest.mark.parametrize("env_id", ENV_IDS)
def test_continuation_from_end_rows(env_id):
    """Branch b from row b, then from the first call's end rows: the twin continuing."""
    c = _Case(env_id, 50, seed=31)
    _, got = c.check((16, 12), 9, noisy=True)
    c.check((16, 12), 9, rows=got[4], noisy=True)


@pytest.mark.parametrize("T", [1, 2])
@pytest.mark.parametrize("env_id", ENV_IDS)
def test_short_horizons(env_id, T):
    c = _Case(env_id, 33, seed=41 + T)
    c.check((6, 5), T, c.rng.integers(0, 33, size=257), per_branch=True)


@pytest.mark.parametrize("env_id", ENV_IDS)
def test_without_autoreset(env_id):
    """autoreset=False: roots stepped far enough that some have already ended (CartPole's flag byte set in the row)."""
    c = _Case(env_id, 200, seed=7, warm=60, autoreset=False)
    if c.kind == 0:
        assert c.root.flags.any(), "some CartPole roots must have fallen"
    c.check((8,), 30, c.rng.integers(0, 200, size=260), noisy=True)
    c.check((8,), 30, c.rng.integers(0, 200, size=260), act=TANH)


@pytest.mark.parametrize("noisy", [False, True])
@pytest.mark.parametrize("env_id", ENV_IDS)
def test_episode_ends_at_first_and_last_step(env_id, noisy):
    """TimeLimit of 10 with the rows' counters set to 9 (truncation at step 0), 10 - T (at step T - 1) and values in
    between: every branch ends an episode inside the horizon, at both edges."""
    T, N = 5, 64
    c = _Case(env_id, N, seed=9, warm=0, max_episode_steps=10)
    _, off = row_layout(c.root.state_dim)
    el = np.array([9, 10 - T] + list(c.rng.integers(10 - T, 10, size=N - 2)), dtype=np.int32)
    c.rows[:, off:off + 4] = el.view(np.uint8).reshape(N, 4)
    want, _ = c.check((8, 8), T, noisy=noisy, act=TANH)
    assert want[1][0] == 1 and want[2][0], "truncated at step 0"
    assert want[1][1] <= T and want[2][1], "ended by step T - 1"
    assert want[2].all()


@pytest.mark.parametrize("env_id", ["CartPole-v1", "MountainCarContinuous-v0", "Pendulum-v1", "Acrobot-v1"])
def test_out_of_range_rows_skip_their_branch(env_id):
    c = _Case(env_id, 40, seed=11)
    idx = c.rng.integers(0, 40, size=50)
    idx[[3, 17, 49]] = [-1, 40, 1 << 40]
    c.check((8,), 7, idx, per_branch=True, noisy=True)
    c.check((8,), 7, idx, norm=True)


@pytest.mark.parametrize("env_id", ["CartPole-v1", "Pendulum-v1"])
def test_signed_zero_actions(env_id):
    """A policy whose outputs are all -0.0: without noise the Box action keeps the sign (z itself, not z + 0); with
    noise of -0.0 too, and with +0.0 noise the Box action becomes +0.0, as in the twin."""
    c = _Case(env_id, 20, seed=51)
    P = _param_count(c.D, (8,), c.K)
    params = np.zeros(P, dtype=np.float32)
    params[-(8 * c.K + c.K):] = -0.0          # the output layer: -0.0 + -0.0 * relu(u) = -0.0
    out = c.root.rollout_from_mlp(c.rows, params, (8,), 3)
    acts, _, _, _, _, _ = c.twin(c.rows, params, (8,), 3, None, RELU, None, None, 1e-8, None)
    _assert_same(out[3], acts[0], "first actions, no noise")
    if not c.discrete:
        assert np.signbit(out[3]).all()
    for z in (-0.0, 0.0):
        noise = np.full((3, 20, c.K), z, dtype=np.float32)
        got = c.root.rollout_from_mlp(c.rows, params, (8,), 3, noise=noise)
        acts, rew, te, tr, _, _ = c.twin(c.rows, params, (8,), 3, noise, RELU, None, None, 1e-8, None)
        _assert_same(got[3], acts[0], f"first actions, noise {z}")
        for x, y, name in zip(got[:3], summary_of(rew, te, tr), ("returns", "lengths", "ended")):
            _assert_same(x, y, name)
