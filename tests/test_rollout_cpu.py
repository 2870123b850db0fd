"""rollout_kernel's per-env driver (per_env.cuh: rollout_env) on the CPU against T launches of kernel A's driver.

Both run through tests/hostsim/rollout.cpp, the device source compiled with g++: the rollout must give every output
slice, the final observations, the handle's last-observation buffer, the float64 state, TimeLimit counters, CartPole
flags and PCG64 records bit for bit as the T steps do, and the step after it must agree too.  The same driver replays
the reference fixtures of tests/golden under the bars of test_gpu_parity.py.
"""
import numpy as np
import pytest

from conftest import golden_names, load_golden
from gym_b200 import envs as _envs
from gym_b200.registration import spec as _spec
from hostsim.rollout_sim import DIMS, RolloutSim

ENV_IDS = ["CartPole-v0", "CartPole-v1", "MountainCar-v0", "MountainCarContinuous-v0", "Pendulum-v1", "Acrobot-v1"]
DISCRETE_DTYPES = [np.int64, np.int32, np.uint8]


def _config(env_id, **kwargs):
    """(kind, registry max_episode_steps, param0) as B200VectorEnv resolves them"""
    spec = _spec(env_id)
    ctor = dict(spec.kwargs)
    ctor.update(kwargs)
    kind, _ = _envs.resolve_variant(spec.kind, ctor)
    return kind, spec.max_episode_steps, _envs.resolve_params(kind, ctor)[0]


def _actions(kind, rng, T, N, dtype=np.int64, invalid=False):
    if DIMS[kind][1] == 0:
        nact = 2 if kind == 0 else 3
        a = rng.integers(0, nact, size=(T, N))
        if invalid:   # a few out-of-range actions (the step kernels leave those envs untouched for that step)
            bad = rng.random((T, N)) < 0.05
            a = np.where(bad, nact + rng.integers(0, 3, size=(T, N)), a)
        return a.astype(dtype)
    hi = 2.0 if kind == 3 else 1.0
    return rng.uniform(-3 * hi, 3 * hi, size=(T, N, 1)).astype(np.float32)   # out-of-bounds values included


def _bits(x):
    return np.ascontiguousarray(x).view(np.uint8)


def _assert_same(a, b, what):
    assert a.shape == b.shape and a.dtype == b.dtype, what
    assert np.array_equal(_bits(a), _bits(b)), f"{what}: {np.count_nonzero(np.asarray(a) != np.asarray(b))} differ"


def _twin(env_id, N, seed=7, **kw):
    kind, mes, param0 = _config(env_id)
    mes = kw.pop("max_episode_steps", mes)
    sims = [RolloutSim(kind, N, max_episode_steps=mes, param0=param0, **kw) for _ in range(2)]
    o0 = [s.reset(seed) for s in sims]
    _assert_same(o0[0], o0[1], "reset")
    return kind, sims


def _check(kind, sims, acts):
    """sims[0].rollout(acts) == [sims[1].step(a) for a in acts], stacked; then one more step on both."""
    ro, step = sims
    last = np.zeros((ro.n, ro.obs_dim), dtype=np.float32)
    got = ro.rollout(acts, last)
    outs = [step.step(a) for a in acts]
    names = ("obs", "reward", "terminated", "truncated", "final_obs")
    for k, name in enumerate(names):
        _assert_same(got[k], np.stack([o[k] for o in outs]), name)
    assert got[5] == sum(o[5] for o in outs), "invalid-action count"
    _assert_same(last, got[0][-1], "last observation buffer")
    for x, y, name in zip(ro.get_state(), step.get_state(), ("state", "elapsed", "flags", "rng")):
        _assert_same(x, y, name)
    nxt = _actions(kind, np.random.default_rng(99), 1, ro.n, acts.dtype)[0]
    for k, (x, y) in enumerate(zip(ro.step(nxt)[:5], step.step(nxt)[:5])):
        _assert_same(x, y, f"next step {names[k]}")
    return got


def _cases():
    for env_id in ENV_IDS:
        kind = _config(env_id)[0]
        for dt in (DISCRETE_DTYPES if DIMS[kind][1] == 0 else [np.float32]):
            yield env_id, dt


@pytest.mark.parametrize("N", [1, 7, 300])
@pytest.mark.parametrize("T", [1, 2, 37, 300])
@pytest.mark.parametrize("env_id,dtype", list(_cases()), ids=lambda v: getattr(v, "__name__", v))
def test_rollout_equals_steps(env_id, dtype, T, N):
    kind, sims = _twin(env_id, N, seed=1000 + T + N)
    got = _check(kind, sims, _actions(kind, np.random.default_rng(T * 1000 + N), T, N, dtype))
    if T == 300 and N == 300 and env_id.startswith("CartPole"):
        assert (got[2] | got[3]).any(), "the episodes should have ended inside the rollout"


@pytest.mark.parametrize("env_id", ENV_IDS)
def test_rollout_every_env_truncates_on_the_same_step(env_id):
    """max_episode_steps=3: every env that has not terminated truncates at steps 3, 6, 9, ... of the rollout."""
    kind, sims = _twin(env_id, 64, max_episode_steps=3)
    got = _check(kind, sims, _actions(kind, np.random.default_rng(5), 20, 64))
    assert got[3][2].sum() + got[2][:3].any(axis=0).sum() >= 64


@pytest.mark.parametrize("limit", [None, 4])
@pytest.mark.parametrize("env_id", ENV_IDS)
def test_rollout_without_autoreset(env_id, limit):
    """autoreset=False: no resets, CartPole's post-termination reward of 0.0 through the flag byte in memory."""
    kind, sims = _twin(env_id, 50, autoreset=False, **({} if limit is None else {"max_episode_steps": limit}))
    _check(kind, sims, _actions(kind, np.random.default_rng(11), 60, 50))


@pytest.mark.parametrize("env_id", ["CartPole-v1", "MountainCar-v0", "Acrobot-v1"])
@pytest.mark.parametrize("dtype", DISCRETE_DTYPES, ids=lambda d: d.__name__)
def test_rollout_invalid_actions(env_id, dtype):
    """An out-of-range action leaves the env untouched for that step (NaN reward, current observation); the env
    carries on with the next row, as T step launches do."""
    kind, sims = _twin(env_id, 40)
    got = _check(kind, sims, _actions(kind, np.random.default_rng(3), 30, 40, dtype, invalid=True))
    assert got[5] > 0 and np.isnan(got[1]).sum() == got[5]


@pytest.mark.parametrize("name", golden_names())
def test_rollout_reproduces_reference_fixture(name):
    """One rollout over a fixture's whole action sequence, under test_gpu_parity.py's bars: flags exact,
    observations within 1e-5 relative (+1e-7), rewards within 1e-9."""
    g = load_golden(name)
    kw = {}
    if g["param0"] is not None:
        kw["g" if g["env_id"].startswith("Pendulum") else "goal_velocity"] = g["param0"]
    kind, mes, param0 = _config(g["env_id"], **kw)
    if g["max_episode_steps"] is not None:
        mes = g["max_episode_steps"]
    sim = RolloutSim(kind, g["N"], max_episode_steps=mes, param0=param0)
    obs0 = sim.reset(g["seed"], g["bounds"])

    def close(a, b, what):
        a64, b64 = a.astype(np.float64), b.astype(np.float64)
        assert (np.abs(a64 - b64) <= 1e-7 + 1e-5 * np.abs(b64)).all(), what

    close(obs0, g["obs0"], "reset obs")
    acts = g["actions"]
    if DIMS[kind][1]:
        acts = acts.reshape(g["T"], g["N"], 1).astype(np.float32)
    obs, rew, te, tr, fo, bad = sim.rollout(acts)
    assert bad == 0
    assert np.array_equal(te, g["terminated"]) and np.array_equal(tr, g["truncated"])
    close(obs, g["obs"], "obs")
    np.testing.assert_allclose(rew, g["reward"], rtol=1e-9, atol=1e-9)
    m = g["final_mask"]
    assert np.array_equal(te | tr, m)
    close(fo[m], g["final_obs"][m], "final obs")
