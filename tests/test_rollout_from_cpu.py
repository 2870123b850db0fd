"""rollout_from_kernel's device source on the CPU (tests/hostsim/rollout_from.cpp), against rollout_kernel's driver run
on a batch restored from the same snapshot rows.

A root batch is reset and stepped, and its state is packed into snapshot rows by a numpy restatement of the row
layout (PCG64 record, float64 state, TimeLimit counter, flag byte, zero padding).  Each rollout_from call is compared
with its twin: a batch of B envs restored from the gathered rows, rolled out with the same actions by rollout_env, its
rewards and flags folded in float64 over the first episode end, and its end state packed the same way.  Returns,
lengths, end flags, end observations and the invalid-action count must match bit for bit and the end rows byte for
byte.
"""
import numpy as np
import pytest

from gym_b200 import envs as _envs
from gym_b200.registration import spec as _spec
from hostsim.rollout_from_sim import RolloutFromSim

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
    assert np.array_equal(_bits(a), _bits(b)), f"{what}: {np.count_nonzero(_bits(a) != _bits(b))} bytes differ"


def row_layout(S):
    """(row bytes, offset of the TimeLimit counter) of a classic kind with S state words"""
    return (32 + 8 * S + 5 + 31) // 32 * 32, 32 + 8 * S


def pack_rows(sim):
    """The snapshot rows of every env of `sim`: the numpy restatement of snapshot_save_kernel's layout."""
    n, S = sim.n, sim.state_dim
    R, off = row_layout(S)
    rows = np.zeros((n, R), dtype=np.uint8)
    rows[:, :32] = sim.rng.view(np.uint8).reshape(n, 32)
    rows[:, 32:off] = np.ascontiguousarray(sim.state.T).view(np.uint8).reshape(n, 8 * S)
    rows[:, off:off + 4] = sim.elapsed.view(np.uint8).reshape(n, 4)
    rows[:, off + 4] = sim.flags
    return rows


def load_rows(sim, rows):
    """restore(): every env of `sim` from one row, in place (the batch holds pointers to its arrays)."""
    n, S = sim.n, sim.state_dim
    _, off = row_layout(S)
    rows = np.ascontiguousarray(rows)
    sim.rng[...] = rows[:, :32].copy().view(np.uint64).reshape(n, 4)
    sim.state[...] = rows[:, 32:off].copy().view(np.float64).reshape(n, S).T
    sim.elapsed[...] = rows[:, off:off + 4].copy().view(np.int32).reshape(n)
    sim.flags[...] = rows[:, off + 4]


def summary_of(rew, te, tr):
    """(returns, lengths, ended) over each branch's first episode end, restated in float64 from the full outputs."""
    T, n = rew.shape
    done = te | tr
    ended = done.any(axis=0)
    t_end = np.where(ended, np.argmax(done, axis=0), T - 1)
    returns = np.zeros(n)
    for t in range(T):
        returns = np.where(t <= t_end, returns + rew[t], returns)
    return returns, (t_end + 1).astype(np.int32), ended


class _Case:
    """A root batch of N envs, reset and stepped `warm` times, and its snapshot rows."""

    def __init__(self, env_id, N, seed, warm=3, **kw):
        self.kind, mes, self.param0, self.single = _config(env_id)
        self.kw = {"max_episode_steps": mes, **kw}
        self.discrete = hasattr(self.single, "n")
        self.root = RolloutFromSim(self.kind, N, param0=self.param0, **self.kw)
        self.root.reset(seed)
        self.rng = np.random.default_rng(seed)
        for _ in range(warm):
            self.root.step(self.actions(1, N)[0])
        self.rows = pack_rows(self.root)
        assert self.rows.shape[1] == self.root.row_bytes

    def actions(self, T, B):
        if self.discrete:
            return self.rng.integers(0, self.single.n, size=(T, B)).astype(np.int64)
        return self.rng.uniform(-3.0, 3.0, size=(T, B, 1)).astype(np.float32)

    def check(self, actions, row_idx=None, rows=None):
        """rollout_from against its twin, with and without end states -> the twin's summary."""
        rows = self.rows if rows is None else rows
        B = actions.shape[1]
        before = [x.copy() for x in self.root.get_state()]
        got = self.root.rollout_from(rows, actions, row_idx, states=True)
        plain = self.root.rollout_from(rows, actions, row_idx, states=False)
        for x, y, name in zip(plain[:3], got[:3], ("returns", "lengths", "ended")):
            _assert_same(x, y, f"states=False: {name}")
        assert plain[5] == got[5]
        for x, y, name in zip(self.root.get_state(), before, ("state", "elapsed", "flags", "rng")):
            _assert_same(x, y, f"root batch {name} moved")
        idx = np.arange(B) if row_idx is None else np.asarray(row_idx)
        ok = (idx >= 0) & (idx < rows.shape[0])
        assert got[6] == int(not ok.all()), "index-error flag"
        twin = RolloutFromSim(self.kind, B, param0=self.param0, **self.kw)
        load_rows(twin, rows[np.where(ok, idx, 0)])
        last = np.zeros((B, twin.obs_dim), dtype=np.float32)
        obs, rew, te, tr, fo, invalid = twin.rollout(actions, last_obs=last)
        want = summary_of(rew, te, tr)
        end_rows, end_obs = pack_rows(twin), last
        # a skipped branch: zero summary, zero end row and observation; it does not step
        want = (np.where(ok, want[0], 0.0), np.where(ok, want[1], 0).astype(np.int32), want[2] & ok)
        end_rows[~ok] = 0
        end_obs[~ok] = 0.0
        for x, y, name in zip(got[:3], want, ("returns", "lengths", "ended")):
            _assert_same(x, y, name)
        _assert_same(got[3], end_rows, "end rows")
        _assert_same(got[4], end_obs, "end observations")
        if ok.all():
            assert got[5] == invalid, "invalid-action count"
        return want, got


@pytest.mark.parametrize("N", NS)
@pytest.mark.parametrize("T", TS)
@pytest.mark.parametrize("env_id", ENV_IDS)
def test_rollout_from_equals_restored_rollout(env_id, T, N):
    """Branch b from row b, then N branches from random rows (duplicates), then a second call from the end rows of the
    first, which must equal the twin continuing."""
    c = _Case(env_id, N, seed=4000 + T + N)
    c.check(c.actions(T, N))
    idx = c.rng.integers(0, N, size=N)
    _, got = c.check(c.actions(T, N), idx)
    c.check(c.actions(T, N), rows=got[3])


@pytest.mark.parametrize("env_id", ENV_IDS)
def test_roots_times_branches(env_id):
    """R roots x K branches: branches of one root that take the same actions end alike, autoresets included."""
    c = _Case(env_id, 16, seed=5, max_episode_steps=6)
    R, K, T = 16, 8, 20
    idx = np.repeat(np.arange(R), K)
    acts = np.repeat(c.actions(T, R), K, axis=1)
    want, got = c.check(acts, idx)
    for k in range(1, K):
        _assert_same(got[3][k::K], got[3][0::K], f"branch {k} end rows")
    assert (want[2]).any(), "some branches must end an episode"


@pytest.mark.parametrize("env_id", ENV_IDS)
def test_without_autoreset(env_id):
    """autoreset=False: roots stepped far enough that some have already ended (CartPole's flag byte set in the row),
    and the flag moves with the branch, not the root."""
    c = _Case(env_id, 200, seed=7, warm=60, autoreset=False)
    if c.kind == 0:
        assert c.root.flags.any(), "some CartPole roots must have fallen"
    c.check(c.actions(30, 200))
    c.check(c.actions(30, 300), c.rng.integers(0, 200, size=300))


@pytest.mark.parametrize("env_id", ENV_IDS)
def test_episode_ends_at_first_and_last_step(env_id):
    """TimeLimit of 10 with the rows' counters set to 9 (truncation at step 0), 10 - T (at step T - 1) and values in
    between: every branch ends an episode inside the horizon, at both edges."""
    T, N = 5, 64
    c = _Case(env_id, N, seed=9, warm=0, max_episode_steps=10)
    _, off = row_layout(c.root.state_dim)
    el = np.array([9, 10 - T] + list(c.rng.integers(10 - T, 10, size=N - 2)), dtype=np.int32)
    c.rows[:, off:off + 4] = el.view(np.uint8).reshape(N, 4)
    want, got = c.check(c.actions(T, N))
    assert want[1][0] == 1 and want[2][0], "truncated at step 0"
    assert want[1][1] <= T and want[2][1], "ended by step T - 1"
    assert want[2].all()


@pytest.mark.parametrize("env_id", ["CartPole-v1", "MountainCar-v0", "Pendulum-v1", "Acrobot-v1"])
def test_out_of_range_rows_skip_their_branch(env_id):
    c = _Case(env_id, 40, seed=11)
    idx = c.rng.integers(0, 40, size=50)
    idx[[3, 17, 49]] = [-1, 40, 1 << 40]
    c.check(c.actions(7, 50), idx)


@pytest.mark.parametrize("env_id", ["CartPole-v1", "MountainCar-v0", "Acrobot-v1"])
def test_invalid_actions(env_id):
    """An out-of-range Discrete action: NaN reward, counted, the branch untouched for that step."""
    c = _Case(env_id, 33, seed=13)
    acts = c.actions(6, 33)
    acts[2, ::4] = -1
    acts[4, 1::5] = 99
    want, got = c.check(acts)
    assert np.isnan(got[0][::4]).all() and got[5] > 0
