"""``B200VectorEnv.rollout_linear(weight, bias, T)`` on the GPU: bit for bit what ``a = policy(obs); obs, ... = step(a)``
T times returns, with the policy restated in torch elementwise ops in the documented order.

Every comparison is against an eager twin -- a second env built and reset the same way that runs that loop -- and
covers the actions, the outputs, the final observations on the rows the mask selects, the engine state (``get_state()``,
``snapshot()`` rows and observations) and the step after the rollout.  The summary mode is compared with a float64
restatement over a full-output call of a twin.
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


class Twin:
    """An env and the observation it last returned, stepped eagerly by the torch restatement of the policy."""

    def __init__(self, env, obs):
        self.env, self.obs = env, obs.clone()

    def policy(self, w, b):
        torch = _torch()
        n = self.env.num_envs
        z = b.expand(n, b.shape[-1]).clone()
        for k in range(self.env.obs_dim):
            z = z + w[..., k] * self.obs[:, None, k]
        if not self.env.discrete:
            return z
        m, best = z[:, 0], torch.zeros(n, dtype=torch.int64, device=z.device)
        for j in range(1, z.shape[1]):   # np.argmax: the first NaN, else the first maximum
            take = ~torch.isnan(m) & (torch.isnan(z[:, j]) | (z[:, j] > m))
            m = torch.where(take, z[:, j], m)
            best = torch.where(take, torch.full_like(best, j), best)
        return best

    def loop(self, w, b, T):
        """T steps -> (actions, [obs, reward, term, trunc], final obs, masks), stacked."""
        torch = _torch()
        acts, outs, fin, masks = [], [], [], []
        for _ in range(T):
            a = self.policy(w, b)
            o = self.env.step(a)
            self.obs = o[0].clone()
            acts.append(a)
            outs.append([x.clone() for x in o[:4]])
            fin.append(o[4]["final_observation"].clone())
            masks.append(o[4]["_final_observation"].clone())
        return torch.stack(acts), [torch.stack([o[k] for o in outs]) for k in range(4)], torch.stack(fin), torch.stack(masks)


def _pair(env_id, n, seed=3, **kwargs):
    """(env that rolls out, eager Twin), both reset with `seed`."""
    import gym_b200
    envs = [gym_b200.vector.make(env_id, n, **kwargs) for _ in range(2)]
    obs = [e.reset(seed=seed)[0] for e in envs]
    return envs[0], Twin(envs[1], obs[1])


def _params(env, per_env, seed, scale=1.0):
    torch = _torch()
    g = torch.Generator(device="cpu").manual_seed(seed)
    K = env.single_action_space.n if env.discrete else env.act_dim
    lead = (env.num_envs,) if per_env else ()
    w = (scale * torch.randn(lead + (K, env.obs_dim), generator=g)).to(env.device)
    b = (scale * torch.randn(lead + (K,), generator=g)).to(env.device)
    return w, b


def _assert_equals_loop(got, want, what=""):
    acts, obs, rew, term, trunc, infos = got
    wa, (wo, wr, wte, wtr), wfin, wmask = want
    _eq(acts, wa, f"{what}actions")
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


def summary_of(rew, te, tr):
    """(returns, lengths, ended) over each env's first episode end, restated in float64 from the full outputs."""
    torch = _torch()
    T = rew.shape[0]
    done = te | tr
    ended = done.any(dim=0)
    t_end = torch.where(ended, done.to(torch.int8).argmax(dim=0), torch.full_like(ended, T - 1, dtype=torch.int64))
    returns = torch.zeros(rew.shape[1], dtype=torch.float64, device=rew.device)
    for t in range(T):
        returns = torch.where(t <= t_end, returns + rew[t], returns)
    return returns, (t_end + 1).to(torch.int32), ended


def _twin_check(env_id, n, T, per_env, seed=3, **kwargs):
    a, b = _pair(env_id, n, seed=seed, **kwargs)
    w, bias = _params(a, per_env, seed + T)
    got = a.rollout_linear(w, bias, T)
    _assert_equals_loop(got, b.loop(w, bias, T))
    _eq(a.snapshot().obs, got[1][-1], "snapshot().obs vs obs[T-1]")
    _assert_same_env(a, b.env)
    nxt = b.policy(w, bias)
    for name, x, y in zip(NAMES, a.step(nxt)[:4], b.env.step(nxt)[:4]):
        _eq(x, y, f"next step {name}")
    a.close()
    b.env.close()
    return got


# ---------------------------------------------------------------------------------------------- the eager twin
@pytest.mark.parametrize("per_env", [False, True], ids=["shared", "per_env"])
@pytest.mark.parametrize("T", TS)
@pytest.mark.parametrize("n", NS)
@pytest.mark.parametrize("env_id", CLASSIC)
def test_rollout_linear_equals_eager_loop(env_id, n, T, per_env):
    got = _twin_check(env_id, n, T, per_env)
    torch = _torch()
    assert got[0].dtype == (torch.float32 if "Continuous" in env_id or "Pendulum" in env_id else torch.int64)
    assert tuple(got[0].shape[:2]) == (T, n)


@pytest.mark.parametrize("per_env", [False, True], ids=["shared", "per_env"])
@pytest.mark.parametrize("env_id,kwargs", BOX2D, ids=[b[0] for b in BOX2D])
def test_box2d_rollout_linear_equals_eager_loop(env_id, kwargs, per_env):
    _twin_check(env_id, 67, 5, per_env, seed=7, **kwargs)


@pytest.mark.parametrize("env_id", CLASSIC)
def test_rollout_linear_every_env_truncates(env_id):
    got = _twin_check(env_id, 4099, 25, True, max_episode_steps=4)
    assert bool(got[4][3].any())


@pytest.mark.parametrize("limit", [None, 4])
@pytest.mark.parametrize("env_id", CLASSIC)
def test_rollout_linear_without_autoreset(env_id, limit):
    _twin_check(env_id, 2053, 40, False, autoreset=False, max_episode_steps=limit)


def test_rollout_linear_offsets_past_two_to_the_31():
    """CartPole, n = 2^20, T = 520: T * n * D > 2^31, so slices past the 32-bit range must land right; compared slice
    by slice with the eager loop."""
    n, T = 1 << 20, 520
    assert T * n * 4 > 1 << 31
    a, b = _pair("CartPole-v1", n, seed=5)
    w, bias = _params(a, True, 5, scale=0.3)
    acts, obs, rew, term, trunc, infos = a.rollout_linear(w, bias, T)
    fin, mask = infos["final_observation"], infos["_final_observation"]
    for t in range(T):
        act = b.policy(w, bias)
        o, r, te, tr, inf = b.env.step(act)
        b.obs = o.clone()
        _eq(acts[t], act, f"actions[{t}]")
        _eq(obs[t], o, f"obs[{t}]")
        _eq(rew[t], r, f"reward[{t}]")
        _eq(term[t], te, f"terminated[{t}]")
        _eq(trunc[t], tr, f"truncated[{t}]")
        m = inf["_final_observation"]
        _eq(mask[t], m, f"mask[{t}]")
        _eq(fin[t][m], inf["final_observation"][m], f"final_observation[{t}]")
    _assert_same_env(a, b.env)


# ------------------------------------------------------------------------------------------------- summary mode
def _summary_check(env_id, n, T, per_env, seed=9, **kwargs):
    """summary=True against the restatement over a full-output call of a twin; both leave the same env."""
    a, b = _pair(env_id, n, seed=seed, **kwargs)
    w, bias = _params(a, per_env, seed)
    full = b.env.rollout_linear(w, bias, T)
    got = a.rollout_linear(w, bias, T, summary=True)
    for name, x, y in zip(("returns", "lengths", "ended"), got, summary_of(*full[2:5])):
        _eq(x, y, name)
    _eq(a.snapshot().obs, full[1][-1], "snapshot().obs vs obs[T-1]")
    _assert_same_env(a, b.env)
    a.close()
    b.env.close()
    return got


@pytest.mark.parametrize("per_env", [False, True], ids=["shared", "per_env"])
@pytest.mark.parametrize("T", [1, 37, 300])
@pytest.mark.parametrize("env_id", CLASSIC)
def test_summary_equals_restatement(env_id, T, per_env):
    got = _summary_check(env_id, 33 * 256 + 5, T, per_env)
    torch = _torch()
    assert got[0].dtype == torch.float64 and got[1].dtype == torch.int32 and got[2].dtype == torch.bool


@pytest.mark.parametrize("env_id", CLASSIC)
def test_summary_with_short_episodes_and_without_autoreset(env_id):
    ended = _summary_check(env_id, 1000, 30, True, max_episode_steps=7)[2]
    assert bool(ended.all())
    _summary_check(env_id, 1000, 30, False, autoreset=False, max_episode_steps=5)


@pytest.mark.parametrize("env_id,kwargs", BOX2D, ids=[b[0] for b in BOX2D])
def test_box2d_summary_equals_restatement(env_id, kwargs):
    _summary_check(env_id, 67, 5, True, seed=7, **kwargs)


# -------------------------------------------------------------------------------------------- interleaving
@pytest.mark.parametrize("env_id", ["CartPole-v1", "MountainCarContinuous-v0", "Acrobot-v1", "LunarLander-v2"])
def test_rollout_linear_interleaved(env_id):
    """step(), rollout(), rollout_sampled(), reset(seed=), restore and clone between calls, mirrored on the twin."""
    torch = _torch()
    n, T = (300, 3) if env_id.startswith("Lunar") else (1000, 17)
    a, b = _pair(env_id, n)
    w, bias = _params(a, True, 1)
    _assert_equals_loop(a.rollout_linear(w, bias, T), b.loop(w, bias, T), "first ")
    act = b.policy(w, bias)
    o = a.step(act)
    b.obs = b.env.step(act)[0].clone()
    _eq(o[0], b.obs, "step")
    _assert_equals_loop(a.rollout_linear(w, bias, T), b.loop(w, bias, T), "after step ")
    acts = b.policy(w, bias)[None].repeat(4, *([1] * (1 + (not a.discrete))))
    ra = a.rollout(acts)
    rb = b.env.rollout(acts)
    b.obs = rb[0][-1].clone()
    _eq(ra[0], rb[0], "rollout obs")
    _assert_equals_loop(a.rollout_linear(w, bias, T), b.loop(w, bias, T), "after rollout ")
    for e in (a, b.env):
        e.action_space.seed(4)
    sa, sb = a.rollout_sampled(3), b.env.rollout_sampled(3)
    b.obs = sb[1][-1].clone()
    _eq(sa[1], sb[1], "rollout_sampled obs")
    _assert_equals_loop(a.rollout_linear(w, bias, T), b.loop(w, bias, T), "after rollout_sampled ")
    snap_a, snap_b = a.snapshot(), b.env.snapshot()
    _assert_equals_loop(a.rollout_linear(w, bias, T), b.loop(w, bias, T), "before restore ")
    ra = a.reset(seed=77)[0]
    b.obs = b.env.reset(seed=77)[0].clone()
    _eq(ra, b.obs, "reset")
    _assert_equals_loop(a.rollout_linear(w, bias, T), b.loop(w, bias, T), "after reset ")
    ro = a.restore(snap_a)[0]
    b.obs = b.env.restore(snap_b)[0].clone()
    _eq(ro, b.obs, "restore")
    _assert_equals_loop(a.rollout_linear(w, bias, T), b.loop(w, bias, T), "after restore ")
    src = torch.randint(0, n, (n,), device="cuda:0")
    co = a.clone(src)
    b.obs = b.env.clone(src).clone()
    _eq(co, b.obs, "clone")
    _assert_equals_loop(a.rollout_linear(w, bias, T), b.loop(w, bias, T), "after clone ")
    _assert_same_env(a, b.env)


# ------------------------------------------------------------------------------------------------ CUDA graphs
@pytest.mark.parametrize("summary", [False, True], ids=["full", "summary"])
@pytest.mark.parametrize("env_id", ["CartPole-v1", "Pendulum-v1", "Acrobot-v1", "MountainCarContinuous-v0"])
def test_captured_rollout_linear_replays_equal_eager_calls(env_id, summary):
    """Replay k equals eager call k with the parameters copied in place between replays, and with a step() captured
    before the rollout."""
    torch = _torch()
    n, T, k = 515, 24, 3
    a, b = _pair(env_id, n)
    w, bias = _params(a, True, 2)
    step_act = b.policy(w, bias)   # a fixed action for the captured step
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        st = a.step(step_act)
        out = a.rollout_linear(w, bias, T, summary=summary)
    for r in range(k):
        w2, b2 = _params(a, True, 100 + r)
        w.copy_(w2)
        bias.copy_(b2)
        g.replay()
        o = b.env.step(step_act)
        b.obs = o[0].clone()
        for name, x, y in zip(NAMES, st[:4], o[:4]):
            _eq(x, y, f"replay {r} step {name}")
        if summary:
            # the twin's full-output call is checked against its own eager loop elsewhere
            full = b.env.rollout_linear(w2, b2, T)
            b.obs = full[1][-1].clone()
            for name, x, y in zip(("returns", "lengths", "ended"), out, summary_of(*full[2:5])):
                _eq(x, y, f"replay {r} {name}")
        else:
            _assert_equals_loop(out, b.loop(w2, b2, T), f"replay {r} ")
    _assert_same_env(a, b.env)


@pytest.mark.parametrize("env_id,kwargs", BOX2D, ids=[b[0] for b in BOX2D])
def test_box2d_capture_is_refused(env_id, kwargs):
    from gym_b200 import error
    torch = _torch()
    a, b = _pair(env_id, 33, seed=7, **kwargs)
    w, bias = _params(a, False, 3)
    before = _untouched(a)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with pytest.raises(error.Error, match="double|alternate|stale"):
        with torch.cuda.graph(g):
            a.rollout_linear(w, bias, 2)
    del g
    _assert_untouched(a, before, "capture")
    _assert_equals_loop(a.rollout_linear(w, bias, 2), b.loop(w, bias, 2), "after the refused capture ")


# ------------------------------------------------------------------------------------------ refusals and guards
def _untouched(env):
    _torch().cuda.synchronize()
    return env.snapshot().rows.clone(), env._flip


def _assert_untouched(env, before, what):
    torch = _torch()
    rows, flip = _untouched(env)
    assert torch.equal(rows, before[0]), what
    assert flip == before[1], what


def test_rollout_linear_guards_and_refusals():
    import gym_b200
    from gym_b200 import error, wrappers
    from gym_b200.distributed import ShardedVectorEnv
    from gym_b200.env import B200Env
    torch = _torch()

    env = gym_b200.vector.make("CartPole-v1", 64)
    w, b = _params(env, False, 0)
    with pytest.raises(error.ResetNeeded):
        env.rollout_linear(w, b, 3)
    env.reset(seed=1)
    before = _untouched(env)
    for bad in (0, -1, 2 ** 31, 2.0, True, "3"):
        with pytest.raises(ValueError):
            env.rollout_linear(w, b, bad)
        _assert_untouched(env, before, repr(bad))
    wp, bp = _params(env, True, 0)
    bad_params = [
        (w.double(), b), (w, b.half()), (w.cpu(), b), (w, b.cpu()),                 # dtype, device
        (w[:, :3], b), (w, b[:1]), (w[None], b), (w.t(), b),                        # shapes
        (wp, b), (w, bp), (wp[:-1], bp[:-1]),                                        # a mix, the wrong N
        (wp.transpose(1, 2).contiguous().transpose(1, 2), bp),                      # not contiguous
        (w.tolist(), b),
    ]
    for k, (x, y) in enumerate(bad_params):
        with pytest.raises(ValueError):
            env.rollout_linear(x, y, 3)
        _assert_untouched(env, before, f"bad parameters {k}")
    env.step_async(torch.zeros(64, dtype=torch.int64, device="cuda:0"))
    with pytest.raises(error.AlreadyPendingCallError):
        env.rollout_linear(w, b, 3)
    env.step_wait()
    before = _untouched(env)
    for wr in (wrappers.RecordEpisodeStatistics(env), wrappers.NormalizeObservation(env),
               wrappers.NormalizeReward(env), wrappers.VectorListInfo(env)):
        with pytest.raises(error.Error, match="rollout_linear"):
            wr.rollout_linear(w, b, 3)
        with pytest.raises(error.Error, match="rollout_linear"):
            wr.rollout_linear(w, b, 3, summary=True)
    _assert_untouched(env, before, "wrappers")
    env.close()
    with pytest.raises(error.ClosedEnvironmentError):
        env.rollout_linear(w, b, 3)

    host = gym_b200.vector.make("CartPole-v1", 16, backend="numpy")
    host.reset(seed=3)
    rows = host.snapshot().rows.clone()
    with pytest.raises(error.Error, match="backend"):
        host.rollout_linear(w, b, 3)
    assert torch.equal(host.snapshot().rows, rows)
    host.close()

    from gym_b200 import subenv
    chain = gym_b200.vector.make("CartPole-v1", 16, wrappers=[subenv.RecordEpisodeStatistics()])
    chain.reset(seed=4)
    before = _untouched(chain)
    with pytest.raises(error.Error, match="wrappers"):
        chain.rollout_linear(w, b, 3)
    _assert_untouched(chain, before, "per-env wrappers")
    chain.close()

    assert not hasattr(ShardedVectorEnv, "rollout_linear")
    assert not hasattr(B200Env, "rollout_linear")


def test_set_state_then_rollout_linear_starts_from_the_state():
    """After set_state(), which sets a state without an observation, the first input is the observation of that state.
    A step with an out-of-range action returns exactly that (the env's current observation), so a probe env gives the
    twin its first input."""
    import gym_b200
    torch = _torch()
    a, b = _pair("Acrobot-v1", 300, seed=4)
    state, elapsed, rng = b.env.get_state()
    state = state.clone()
    state[:, 0] += 0.25
    probe = gym_b200.vector.make("Acrobot-v1", 300)
    probe.reset(seed=4)
    for e in (a, b.env, probe):
        e.set_state(state, elapsed, rng)
    b.obs = probe.step(torch.full((300,), 7, dtype=torch.int64, device="cuda:0"))[0].clone()
    w, bias = _params(a, True, 6)
    _assert_equals_loop(a.rollout_linear(w, bias, 9), b.loop(w, bias, 9))
    _assert_same_env(a, b.env)
