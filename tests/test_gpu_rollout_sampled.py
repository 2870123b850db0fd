"""``B200VectorEnv.rollout_sampled(T)`` on the GPU: bit for bit what ``a = sample_actions(); step(a)`` T times returns.

Every comparison is against an eager twin -- a second env built, reset and seeded the same way that runs that loop --
and covers the actions, the outputs, the final observations on the rows the mask selects, the engine state
(``get_state()``, ``snapshot()`` rows and observations), the step after the rollout and the host generator of the
action space.
"""
import pytest

pytestmark = pytest.mark.gpu

CLASSIC = ["CartPole-v0", "CartPole-v1", "MountainCar-v0", "MountainCarContinuous-v0", "Pendulum-v1", "Acrobot-v1"]
BOX2D = [("LunarLander-v2", {}), ("LunarLanderContinuous-v2", dict(enable_wind=True, wind_idx=11, torque_idx=-7)),
         ("BipedalWalker-v3", {}), ("BipedalWalkerHardcore-v3", {})]
NS = [1, 31, 256, 257, 33 * 256 + 5, (1 << 16) + 3]
TS = [1, 2, 37, 300]
NAMES = ("obs", "reward", "terminated", "truncated")


def _torch():
    import torch
    return torch


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


def _pair(env_id, n, seed=3, space_seed=11, **kwargs):
    """(env that rolls out, eager twin), both reset with `seed` and their action spaces seeded with `space_seed`."""
    import gym_b200
    envs = [gym_b200.vector.make(env_id, n, **kwargs) for _ in range(2)]
    for e in envs:
        e.reset(seed=seed)
        e.action_space.seed(space_seed)
    return envs


def _loop(env, T):
    """``a = env.sample_actions(); env.step(a)`` T times -> (actions, [obs, reward, term, trunc], final obs, masks)."""
    torch = _torch()
    acts, outs, fin, masks = [], [], [], []
    for _ in range(T):
        a = env.sample_actions()
        o = env.step(a)
        acts.append(a.clone())
        outs.append([x.clone() for x in o[:4]])
        fin.append(o[4]["final_observation"].clone())
        masks.append(o[4]["_final_observation"].clone())
    return torch.stack(acts), [torch.stack([o[k] for o in outs]) for k in range(4)], torch.stack(fin), torch.stack(masks)


def _as_rollout(loop):
    """A _loop result shaped as rollout_sampled() returns it."""
    acts, (o, r, te, tr), fin, masks = loop
    return acts, o, r, te, tr, {"final_observation": fin, "_final_observation": masks}


def _assert_equals_loop(got, want, what=""):
    acts, obs, rew, term, trunc, infos = got
    wa, (wo, wr, wte, wtr), wfin, wmask = want
    _eq(acts, wa, f"{what}actions")
    for name, g, w in zip(NAMES, (obs, rew, term, trunc), (wo, wr, wte, wtr)):
        _eq(g, w, f"{what}{name}")
    _eq(infos["_final_observation"], wmask, f"{what}_final_observation")
    _eq(infos["final_observation"][wmask], wfin[wmask], f"{what}final_observation")


def _generator(env):
    return env.action_space.np_random.bit_generator.state


def _assert_same_env(a, b, what=""):
    torch = _torch()
    for name, x, y in zip(("state", "elapsed", "rng"), a.get_state(), b.get_state()):
        _eq(x, y, f"{what}{name}")
    sa, sb = a.snapshot(), b.snapshot()
    assert torch.equal(sa.rows, sb.rows), f"{what}snapshot rows"
    _eq(sa.obs, sb.obs, f"{what}snapshot obs")
    assert _generator(a) == _generator(b), f"{what}host generator"


def _twin_check(env_id, n, T, seed=3, **kwargs):
    a, b = _pair(env_id, n, seed=seed, space_seed=seed + 100 * T, **kwargs)
    got = a.rollout_sampled(T)
    _assert_equals_loop(got, _loop(b, T))
    _eq(a.snapshot().obs, got[1][-1], "snapshot().obs vs obs[T-1]")
    _assert_same_env(a, b)
    _assert_equals_loop(_as_rollout(_loop(a, 1)), _loop(b, 1), "next step ")
    a.close()
    b.close()
    return got


# ---------------------------------------------------------------------------------------------- the eager twin
@pytest.mark.parametrize("T", TS)
@pytest.mark.parametrize("n", NS)
@pytest.mark.parametrize("env_id", CLASSIC)
def test_rollout_sampled_equals_eager_loop(env_id, n, T):
    got = _twin_check(env_id, n, T)
    torch = _torch()
    assert got[0].dtype == (torch.float32 if "Continuous" in env_id or "Pendulum" in env_id else torch.int64)
    assert tuple(got[0].shape[:2]) == (T, n)


@pytest.mark.parametrize("env_id,kwargs", BOX2D, ids=[b[0] for b in BOX2D])
def test_box2d_rollout_sampled_equals_eager_loop(env_id, kwargs):
    _twin_check(env_id, 67, 5, seed=7, **kwargs)


@pytest.mark.parametrize("env_id", CLASSIC)
def test_rollout_sampled_every_env_truncates(env_id):
    got = _twin_check(env_id, 4099, 25, max_episode_steps=4)
    assert bool(got[4][3].any())


@pytest.mark.parametrize("limit", [None, 4])
@pytest.mark.parametrize("env_id", CLASSIC)
def test_rollout_sampled_without_autoreset(env_id, limit):
    _twin_check(env_id, 2053, 40, autoreset=False, max_episode_steps=limit)


def test_rollout_sampled_offsets_past_two_to_the_31():
    """CartPole, n = 2^20, T = 520: T * n * D > 2^31, so slices and stream positions past the 32-bit range must land
    right; compared slice by slice with the eager loop."""
    n, T = 1 << 20, 520
    assert T * n * 4 > 1 << 31
    a, b = _pair("CartPole-v1", n, seed=5)
    acts, obs, rew, term, trunc, infos = a.rollout_sampled(T)
    fin, mask = infos["final_observation"], infos["_final_observation"]
    for t in range(T):
        act = b.sample_actions()
        o, r, te, tr, inf = b.step(act)
        _eq(acts[t], act, f"actions[{t}]")
        _eq(obs[t], o, f"obs[{t}]")
        _eq(rew[t], r, f"reward[{t}]")
        _eq(term[t], te, f"terminated[{t}]")
        _eq(trunc[t], tr, f"truncated[{t}]")
        m = inf["_final_observation"]
        _eq(mask[t], m, f"mask[{t}]")
        _eq(fin[t][m], inf["final_observation"][m], f"final_observation[{t}]")
    _assert_same_env(a, b)


# -------------------------------------------------------------------------------------------- interleaving
@pytest.mark.parametrize("env_id", ["CartPole-v1", "MountainCarContinuous-v0", "Acrobot-v1", "LunarLander-v2"])
def test_rollout_sampled_interleaved(env_id):
    """Host draws, action_space.seed() (the override path), sample_actions(), rollout(), reset(seed=) and clone
    between calls, mirrored on the twin with the eager loop."""
    torch = _torch()
    n, T = (300, 3) if env_id.startswith("Lunar") else (1000, 17)
    a, b = _pair(env_id, n)
    _assert_equals_loop(a.rollout_sampled(T), _loop(b, T), "first ")
    for e in (a, b):
        e.action_space.sample()      # a host draw: the next call starts from the override
    _assert_equals_loop(a.rollout_sampled(T), _loop(b, T), "after a host draw ")
    for e in (a, b):
        e.action_space.seed(2 ** 70 + 9)   # another inc
    _assert_equals_loop(a.rollout_sampled(T), _loop(b, T), "after a reseed ")
    _assert_equals_loop(_as_rollout(_loop(a, 2)), _loop(b, 2), "sample_actions ")
    acts = b.sample_actions()[None].repeat(4, *([1] * (1 + (not a.discrete))))
    a.action_space.sample()          # keep the two generators together: b drew once on the device
    eager = [[y.clone() for y in b.step(x)[:4]] for x in acts]
    for name, x, y in zip(NAMES, a.rollout(acts)[:4], [torch.stack(v) for v in zip(*eager)]):
        _eq(x, y, f"rollout {name}")
    _eq(a.reset(seed=77)[0], b.reset(seed=77)[0], "reset")
    _assert_equals_loop(a.rollout_sampled(T), _loop(b, T), "after reset ")
    src = torch.randint(0, n, (n,), device="cuda:0")
    _eq(a.clone(src), b.clone(src), "clone")
    _assert_equals_loop(a.rollout_sampled(T), _loop(b, T), "after clone ")
    _assert_same_env(a, b)


# ------------------------------------------------------------------------------------------------ CUDA graphs
@pytest.mark.parametrize("env_id", ["CartPole-v1", "Pendulum-v1", "LunarLander-v2"])
def test_captured_rollout_sampled_replays_equal_eager_calls(env_id):
    """Replay k equals eager call k: the replays move the record only, and sync_action_space() brings the host there."""
    torch = _torch()
    n, T, k = 515, 24 if not env_id.startswith("Lunar") else 4, 3
    a, b = _pair(env_id, n)
    _assert_equals_loop(a.rollout_sampled(T), _loop(b, T), "eager ")   # puts the generator on the device
    before = _generator(a)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = a.rollout_sampled(T)
    assert _generator(a) == before, "a capture leaves the host generator alone"
    for r in range(k):
        g.replay()
        _assert_equals_loop(out, _loop(b, T), f"replay {r} ")
    assert _generator(a) == before
    a.sync_action_space()
    _assert_same_env(a, b)


def test_two_rollouts_and_sample_actions_in_one_graph_continue_one_stream():
    torch = _torch()
    n, T1, T2 = 777, 5, 9
    a, b = _pair("Acrobot-v1", n)
    a.sample_actions()
    b.sample_actions()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        first = a.rollout_sampled(T1)
        act = a.sample_actions()
        step = a.step(act)
        second = a.rollout_sampled(T2)
    for r in range(2):
        g.replay()
        _assert_equals_loop(first, _loop(b, T1), f"replay {r} first ")
        wa, wstep = _loop(b, 1)[:2]
        _eq(act, wa[0], f"replay {r} sample_actions")
        for name, x, y in zip(NAMES, step[:4], wstep):
            _eq(x, y[0], f"replay {r} step {name}")
        _assert_equals_loop(second, _loop(b, T2), f"replay {r} second ")
    a.sync_action_space()
    _assert_same_env(a, b)


# ------------------------------------------------------------------------------------------ refusals and guards
def _untouched(env):
    """What a refused call must leave alone: the engine rows, the device record and the host generator."""
    _torch().cuda.synchronize()
    rec = None if env._sample_record is None else env._sample_record.clone()
    return env.snapshot().rows.clone(), rec, _generator(env)


def _assert_untouched(env, before, what):
    torch = _torch()
    rows, rec, gen = _untouched(env)
    assert torch.equal(rows, before[0]), what
    assert (rec is None and before[1] is None) or torch.equal(rec, before[1]), what
    assert gen == before[2], what


def test_rollout_sampled_guards_and_refusals():
    import gym_b200
    from gym_b200 import error, wrappers
    from gym_b200.distributed import ShardedVectorEnv
    from gym_b200.env import B200Env
    torch = _torch()

    env = gym_b200.vector.make("CartPole-v1", 64)
    with pytest.raises(error.ResetNeeded):
        env.rollout_sampled(3)
    env.reset(seed=1)
    env.action_space.seed(2)
    before = _untouched(env)
    for bad in (0, -1, 2 ** 31, 2.0, True, "3"):
        with pytest.raises((ValueError, TypeError)):
            env.rollout_sampled(bad)
        _assert_untouched(env, before, repr(bad))
    # capture before the device holds the generator
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with pytest.raises(error.Error, match="captured"):
        with torch.cuda.graph(g):
            env.rollout_sampled(3)
    del g
    _assert_untouched(env, before, "capture")
    env.step_async(torch.zeros(64, dtype=torch.int64, device="cuda:0"))
    with pytest.raises(error.AlreadyPendingCallError):
        env.rollout_sampled(3)
    env.step_wait()
    before = _untouched(env)
    for w in (wrappers.RecordEpisodeStatistics(env), wrappers.NormalizeObservation(env),
              wrappers.NormalizeReward(env), wrappers.VectorListInfo(env)):
        with pytest.raises(error.Error, match="rollout_sampled"):
            w.rollout_sampled(3)
    _assert_untouched(env, before, "wrappers")
    # an invalid action of an earlier call is reported by the next one, before it launches anything
    bad = torch.full((2, 64), 5, dtype=torch.int64, device="cuda:0")
    env.rollout(bad)
    torch.cuda.synchronize()
    before = _untouched(env)
    with pytest.raises(error.InvalidAction):
        env.rollout_sampled(3)
    _assert_untouched(env, before, "invalid-action poll")
    env.close()
    with pytest.raises(error.ClosedEnvironmentError):
        env.rollout_sampled(3)

    host = gym_b200.vector.make("CartPole-v1", 16, backend="numpy")
    host.reset(seed=3)
    host.action_space.seed(4)
    before = _untouched(host)
    with pytest.raises(error.Error, match="backend"):
        host.rollout_sampled(3)
    _assert_untouched(host, before, "numpy backend")
    host.close()

    from gym_b200 import subenv
    chain = gym_b200.vector.make("CartPole-v1", 16, wrappers=[subenv.RecordEpisodeStatistics()])
    chain.reset(seed=4)
    chain.action_space.seed(5)
    before = _untouched(chain)
    with pytest.raises(error.Error, match="wrappers"):
        chain.rollout_sampled(3)
    _assert_untouched(chain, before, "per-env wrappers")
    chain.close()

    assert not hasattr(ShardedVectorEnv, "rollout_sampled")
    assert not hasattr(B200Env, "rollout_sampled")


def test_rollout_sampled_outputs_are_fresh():
    a, b = _pair("Pendulum-v1", 100)
    first = a.rollout_sampled(6)
    kept = [x.clone() for x in first[:5]]
    second = a.rollout_sampled(6)
    for x, y in zip(first[:5], second[:5]):
        assert x.data_ptr() != y.data_ptr()
    for k, (x, y) in enumerate(zip(first[:5], kept)):
        _eq(x, y, f"first call's output {k} after a second call")
    _assert_equals_loop(first, _loop(b, 6), "first ")
    _assert_equals_loop(second, _loop(b, 6), "second ")
