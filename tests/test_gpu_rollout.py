"""``B200VectorEnv.rollout(actions)`` on the GPU: T steps in one call, bit for bit what T ``step()`` calls return.

Every comparison is against an eager twin -- a second env built and reset the same way that takes the T steps one
``step()`` at a time -- and covers the outputs, the final observations on the rows the mask selects, the engine state
(``get_state()``, ``snapshot()`` rows and observations) and the step after the rollout.
"""
import numpy as np
import pytest

from conftest import golden_names, load_golden

pytestmark = pytest.mark.gpu

CLASSIC = ["CartPole-v0", "CartPole-v1", "MountainCar-v0", "MountainCarContinuous-v0", "Pendulum-v1", "Acrobot-v1"]
NS = [1, 31, 256, 257, 33 * 256 + 5, (1 << 16) + 3]
TS = [1, 2, 37, 300]
NAMES = ("obs", "reward", "terminated", "truncated")


def _torch():
    import torch
    return torch


def _make(env_id, n, kernel=None, **kwargs):
    import gym_b200
    with pytest.MonkeyPatch.context() as mp:
        mp.delenv("B200GYM_KERNEL", raising=False)
        if kernel is not None:
            mp.setenv("B200GYM_KERNEL", kernel)
        return gym_b200.vector.make(env_id, n, **kwargs)


def _pair(env_id, n, seed=3, kernel=None, **kwargs):
    """(env that rolls out, eager twin), both reset with `seed`."""
    a, b = _make(env_id, n, **kwargs), _make(env_id, n, kernel=kernel, **kwargs)
    a.reset(seed=seed)
    b.reset(seed=seed)
    return a, b


def _actions(env, T, seed=0, dtype=None, wild=True):
    """(T, N) Discrete actions or (T, N, A) float32 actions reaching 20 % past each bound."""
    torch = _torch()
    g = torch.Generator(device="cuda:0")
    g.manual_seed(seed)
    if env.discrete:
        a = torch.randint(0, int(env.single_action_space.n), (T, env.num_envs), generator=g, device="cuda:0")
        return a if dtype is None else a.to(dtype)
    lo = torch.as_tensor(env.single_action_space.low, device="cuda:0")
    hi = torch.as_tensor(env.single_action_space.high, device="cuda:0")
    u = torch.rand((T, env.num_envs, env.act_dim), generator=g, device="cuda:0", dtype=torch.float32)
    return (lo - 0.2 * (hi - lo) + 1.4 * (hi - lo) * u) if wild else (lo + (hi - lo) * u)


def _bits(t):
    torch = _torch()
    if t.dtype == torch.float32:
        return t.view(torch.int32)
    if t.dtype == torch.float64:
        return t.view(torch.int64)
    return t


def _eq(a, b, what):
    torch = _torch()
    assert a.dtype == b.dtype and a.shape == b.shape, (what, a.dtype, b.dtype, a.shape, b.shape)
    if not torch.equal(_bits(a), _bits(b)):
        bad = (_bits(a) != _bits(b)).nonzero()
        raise AssertionError(f"{what}: {len(bad)} entries differ, first at {bad[0].tolist()}")


def _eager(env, acts, catch=False):
    """[env.step(a) for a in acts], stacked, with the final observations (masked rows only meaningful).  catch=True:
    an InvalidAction raised by a step (for an earlier step's invalid action) is caught and the step repeated."""
    from gym_b200 import error
    torch = _torch()
    outs, fin, masks = [], [], []
    for a in acts:
        try:
            o = env.step(a)
        except error.InvalidAction:
            if not catch:
                raise
            o = env.step(a)
        outs.append([x.clone() for x in o[:4]])
        fin.append(o[4]["final_observation"].clone())
        masks.append(o[4]["_final_observation"].clone())
    stacked = [torch.stack([o[k] for o in outs]) for k in range(4)]
    return stacked, torch.stack(fin), torch.stack(masks)


def _assert_rollout_equals(got, want, what=""):
    obs, rew, term, trunc, infos = got
    (wo, wr, wte, wtr), wfin, wmask = want
    for name, g, w in zip(NAMES, (obs, rew, term, trunc), (wo, wr, wte, wtr)):
        _eq(g, w, f"{what}{name}")
    _eq(infos["_final_observation"], wmask, f"{what}_final_observation")
    _eq(infos["final_observation"][wmask], wfin[wmask], f"{what}final_observation")


def _assert_same_env(a, b, what=""):
    torch = _torch()
    for name, x, y in zip(("state", "elapsed", "rng"), a.get_state(), b.get_state()):
        _eq(x, y, f"{what}{name}")
    sa, sb = a.snapshot(), b.snapshot()
    assert torch.equal(sa.rows, sb.rows), f"{what}snapshot rows"
    _eq(sa.obs, sb.obs, f"{what}snapshot obs")


def _twin_check(env_id, n, T, dtype=None, kernel=None, seed=3, **kwargs):
    a, b = _pair(env_id, n, seed=seed, kernel=kernel, **kwargs)
    acts = _actions(a, T, seed=seed + T, dtype=dtype)
    got = a.rollout(acts)
    _assert_rollout_equals(got, _eager(b, acts))
    _eq(a.snapshot().obs, got[0][-1], "snapshot().obs vs obs[T-1]")
    _assert_same_env(a, b)
    nxt = _actions(a, 1, seed=seed + 999, dtype=dtype)[0]
    for name, x, y in zip(NAMES, a.step(nxt)[:4], b.step(nxt)[:4]):
        _eq(x, y, f"next step {name}")
    a.close()
    b.close()
    return got


# ------------------------------------------------------------------------------------------- reference fixtures
@pytest.mark.parametrize("name", golden_names())
def test_rollout_reproduces_reference_fixture(name):
    """reset(seed, options) then ONE rollout over the fixture's actions: the parity bars, and bitwise the twin."""
    from test_gpu_parity import REW_TOL, _assert_obs
    torch = _torch()
    g = load_golden(name)
    kwargs = {"max_episode_steps": g["max_episode_steps"]}
    if g["param0"] is not None:
        kwargs["g" if g["env_id"].startswith("Pendulum") else "goal_velocity"] = g["param0"]
    options = None
    if g["bounds"] is not None:
        keys = ("x_init", "y_init") if g["env_id"].startswith("Pendulum") else ("low", "high")
        options = dict(zip(keys, g["bounds"]))
    a, b = _make(g["env_id"], g["N"], **kwargs), _make(g["env_id"], g["N"], **kwargs)
    a.reset(seed=g["seed"], options=options)
    b.reset(seed=g["seed"], options=options)
    acts = torch.as_tensor(g["actions"], device=a.device)
    if not a.discrete:
        acts = acts.reshape(g["T"], g["N"], a.act_dim).to(torch.float32)
    obs, rew, te, tr, infos = got = a.rollout(acts)
    assert np.array_equal(te.cpu().numpy(), g["terminated"]) and np.array_equal(tr.cpu().numpy(), g["truncated"])
    _assert_obs(obs.cpu().numpy(), g["obs"], "rollout obs")
    np.testing.assert_allclose(rew.cpu().numpy(), g["reward"], rtol=REW_TOL, atol=REW_TOL)
    m = g["final_mask"]
    assert np.array_equal(infos["_final_observation"].cpu().numpy(), m)
    if m.any():
        _assert_obs(infos["final_observation"].cpu().numpy()[m], g["final_obs"][m], "final obs")
    _assert_rollout_equals(got, _eager(b, acts))
    _assert_same_env(a, b)


# ---------------------------------------------------------------------------------------------- the eager twin
@pytest.mark.parametrize("T", TS)
@pytest.mark.parametrize("n", NS)
@pytest.mark.parametrize("env_id", CLASSIC)
def test_rollout_equals_eager_steps(env_id, n, T):
    _twin_check(env_id, n, T)


@pytest.mark.parametrize("n", [257, (1 << 16) + 3])
@pytest.mark.parametrize("dtype", ["int32", "uint8"])
@pytest.mark.parametrize("env_id", ["CartPole-v1", "MountainCar-v0", "Acrobot-v1"])
def test_rollout_narrow_action_dtypes(env_id, dtype, n):
    _twin_check(env_id, n, 37, dtype=getattr(_torch(), dtype))


@pytest.mark.parametrize("env_id", CLASSIC)
def test_rollout_every_env_truncates_on_the_same_step(env_id):
    got = _twin_check(env_id, 4099, 25, max_episode_steps=4)
    assert bool(got[3][3].any())


@pytest.mark.parametrize("limit", [None, 5])
@pytest.mark.parametrize("env_id", CLASSIC)
def test_rollout_without_autoreset(env_id, limit):
    _twin_check(env_id, 2053, 40, autoreset=False, max_episode_steps=limit)


@pytest.mark.parametrize("kernel", ["a", "p", "b"])
@pytest.mark.parametrize("n", [33 * 256 + 5, (1 << 16) + 3])
@pytest.mark.parametrize("env_id", CLASSIC)
def test_rollout_equals_every_step_kernel(env_id, n, kernel):
    """The twin steps on kernel A, P or B (B200GYM_KERNEL); the rollout is the same whichever the step path is."""
    _twin_check(env_id, n, 37, kernel=kernel)


# -------------------------------------------------------------------------------------------- interleaving
@pytest.mark.parametrize("env_id", ["CartPole-v1", "MountainCarContinuous-v0", "Acrobot-v1"])
def test_rollout_interleaved_with_step_reset_and_clone(env_id):
    """step, rollout, reset(seed=), rollout, clone, rollout == the same sequence stepped eagerly."""
    torch = _torch()
    n = 1000
    a, b = _pair(env_id, n)
    s0 = _actions(a, 1, seed=1)[0]
    for name, x, y in zip(NAMES, a.step(s0)[:4], b.step(s0)[:4]):
        _eq(x, y, f"step {name}")
    acts = _actions(a, 50, seed=2)
    _assert_rollout_equals(a.rollout(acts), _eager(b, acts), "first rollout ")
    _eq(a.reset(seed=77)[0], b.reset(seed=77)[0], "reset")
    acts = _actions(a, 20, seed=3)
    _assert_rollout_equals(a.rollout(acts), _eager(b, acts), "second rollout ")
    src = torch.randint(0, n, (n,), device="cuda:0")
    _eq(a.clone(src), b.clone(src), "clone")
    acts = _actions(a, 33, seed=4)
    _assert_rollout_equals(a.rollout(acts), _eager(b, acts), "third rollout ")
    _assert_same_env(a, b)


# ------------------------------------------------------------------------------------------------ large offsets
def test_rollout_offsets_past_two_to_the_31():
    """CartPole, n = 2^20 + 3, T = 520: T * n * D > 2^31, so slices past the 32-bit range must land right."""
    torch = _torch()
    n, T = (1 << 20) + 3, 520
    assert T * n * 4 > 1 << 31
    a, b = _pair("CartPole-v1", n, seed=5)
    acts = _actions(a, T, seed=6, dtype=torch.uint8)
    obs, rew, term, trunc, infos = a.rollout(acts)
    fin, mask = infos["final_observation"], infos["_final_observation"]
    for t in range(T):
        o, r, te, tr, inf = b.step(acts[t])
        _eq(obs[t], o, f"obs[{t}]")
        _eq(rew[t], r, f"reward[{t}]")
        _eq(term[t], te, f"terminated[{t}]")
        _eq(trunc[t], tr, f"truncated[{t}]")
        m = inf["_final_observation"]
        _eq(mask[t], m, f"mask[{t}]")
        _eq(fin[t][m], inf["final_observation"][m], f"final_observation[{t}]")
    _assert_same_env(a, b)


# ------------------------------------------------------------------------------------------------ CUDA graphs
@pytest.mark.parametrize("env_id", ["CartPole-v1", "Pendulum-v1", "LunarLander-v2"])
def test_captured_rollout_replays_equal_eager_rollouts(env_id):
    torch = _torch()
    n, T, k = 515, 24, 4
    a, b = _pair(env_id, n)
    buf = _actions(a, T, seed=10).clone()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = a.rollout(buf)
    mask = out[4]["_final_observation"]
    for r in range(k):
        acts = _actions(a, T, seed=20 + r)
        buf.copy_(acts)
        g.replay()
        want = _eager(b, acts)
        obs, rew, term, trunc, infos = out
        for name, x, y in zip(NAMES, (obs, rew, term, trunc), want[0]):
            _eq(x, y, f"replay {r} {name}")
        _eq(mask, want[2], f"replay {r} mask")
        _eq(infos["final_observation"][mask], want[1][mask], f"replay {r} final_observation")
        _assert_same_env(a, b, f"replay {r} ")


# ------------------------------------------------------------------------------------------------ Box2D tasks
@pytest.mark.parametrize("env_id,kwargs", [
    ("LunarLander-v2", {}),
    ("LunarLanderContinuous-v2", dict(enable_wind=True, wind_idx=11, torque_idx=-7)),
    ("BipedalWalker-v3", {}),
    ("BipedalWalkerHardcore-v3", {}),
])
def test_box2d_rollout_equals_eager_steps(env_id, kwargs):
    _twin_check(env_id, 256, 30, seed=7, **kwargs)


# --------------------------------------------------------------------------------------------- invalid actions
@pytest.mark.parametrize("env_id", ["CartPole-v1", "MountainCar-v0", "Acrobot-v1"])
def test_rollout_with_invalid_actions(env_id):
    """Out-of-range actions at some (t, i): that env is left untouched for step t (NaN reward, current observation)
    and carries on; the twin catches the InvalidAction each next step raises and repeats it.  The next call after
    the rollout raises."""
    from gym_b200 import error
    torch = _torch()
    a, b = _pair(env_id, 300)
    acts = _actions(a, 40, seed=8)
    g = torch.Generator(device="cuda:0")
    g.manual_seed(9)
    bad = torch.rand(acts.shape, generator=g, device="cuda:0") < 0.03
    acts = torch.where(bad, acts + int(a.single_action_space.n) + 1, acts)
    got = a.rollout(acts)
    _assert_rollout_equals(got, _eager(b, acts, catch=True))
    assert int(torch.isnan(got[1]).sum()) == int(bad.sum())
    with pytest.raises(error.InvalidAction):
        a.rollout(acts[:1])
    with pytest.raises(error.InvalidAction):
        b.step(acts[0])
    _assert_same_env(a, b)


# ------------------------------------------------------------------------------------------ refusals and guards
def _rows(env):
    _torch().cuda.synchronize()
    return env.snapshot().rows.clone()


def test_rollout_guards_and_refusals():
    import gym_b200
    from gym_b200 import error, wrappers
    torch = _torch()

    env = gym_b200.vector.make("CartPole-v1", 64)
    with pytest.raises(error.ResetNeeded):
        env.rollout(torch.zeros((3, 64), dtype=torch.int64, device="cuda:0"))
    env.reset(seed=1)
    rows = _rows(env)
    for bad in (torch.zeros((3, 63), dtype=torch.int64), torch.zeros((0, 64), dtype=torch.int64),
                torch.zeros((64,), dtype=torch.int64), torch.zeros((3, 64, 1), dtype=torch.int64),
                torch.zeros((3, 64), dtype=torch.float32)):
        with pytest.raises(error.Error):
            env.rollout(bad.to("cuda:0"))
        assert torch.equal(_rows(env), rows), tuple(bad.shape)
    env.step_async(torch.zeros(64, dtype=torch.int64, device="cuda:0"))
    with pytest.raises(error.AlreadyPendingCallError):
        env.rollout(torch.zeros((3, 64), dtype=torch.int64, device="cuda:0"))
    env.step_wait()
    rows = _rows(env)
    for w in (wrappers.RecordEpisodeStatistics(env), wrappers.NormalizeObservation(env),
              wrappers.NormalizeReward(env), wrappers.VectorListInfo(env)):
        with pytest.raises(error.Error, match="rollout"):
            w.rollout(torch.zeros((3, 64), dtype=torch.int64, device="cuda:0"))
    assert torch.equal(_rows(env), rows)
    env.close()
    with pytest.raises(error.ClosedEnvironmentError):
        env.rollout(torch.zeros((3, 64), dtype=torch.int64, device="cuda:0"))

    pend = gym_b200.vector.make("Pendulum-v1", 32)
    pend.reset(seed=2)
    rows = _rows(pend)
    for bad in (torch.zeros((3, 32, 2)), torch.zeros((3, 31, 1)), torch.zeros((3, 32)), torch.zeros((0, 32, 1))):
        with pytest.raises(error.Error):
            pend.rollout(bad.to("cuda:0"))
        assert torch.equal(_rows(pend), rows), tuple(bad.shape)
    pend.close()

    host = gym_b200.vector.make("CartPole-v1", 16, backend="numpy")
    host.reset(seed=3)
    rows = _rows(host)
    with pytest.raises(error.Error, match="backend"):
        host.rollout(np.zeros((3, 16), dtype=np.int64))
    assert torch.equal(_rows(host), rows)
    host.close()

    from gym_b200 import subenv
    chain = gym_b200.vector.make("CartPole-v1", 16, wrappers=[subenv.RecordEpisodeStatistics()])
    chain.reset(seed=4)
    rows = _rows(chain)
    with pytest.raises(error.Error, match="wrappers"):
        chain.rollout(torch.zeros((3, 16), dtype=torch.int64, device="cuda:0"))
    assert torch.equal(_rows(chain), rows)
    chain.close()

    from gym_b200.distributed import ShardedVectorEnv
    assert not hasattr(ShardedVectorEnv, "rollout")


def test_rollout_outputs_are_fresh_and_host_actions_are_accepted():
    """Each call returns new tensors; numpy actions of any accepted dtype are converted as step() converts them."""
    torch = _torch()
    a, b = _pair("CartPole-v1", 100)
    acts = np.random.default_rng(0).integers(0, 2, size=(6, 100)).astype(np.int16)
    first = a.rollout(acts)
    kept = first[0].clone()
    second = a.rollout(acts)
    assert first[0].data_ptr() != second[0].data_ptr()
    _eq(first[0], kept, "first rollout's obs after a second call")
    want1, want2 = _eager(b, torch.as_tensor(acts)), _eager(b, torch.as_tensor(acts))
    _assert_rollout_equals(first, want1)
    _assert_rollout_equals(second, want2)
