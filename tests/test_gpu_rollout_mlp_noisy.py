"""``B200VectorEnv.rollout_mlp_noisy(params, hidden, noise)`` on the GPU: bit for bit what
``z = mlp(obs); a = rule(z + noise[t]); obs, ... = step(a)`` T times returns, with the MLP restated in torch elementwise
ops as in test_gpu_rollout_mlp.py, ``z + noise[t]`` one torch float32 add, and ``rule`` ``np.argmax`` (Discrete) or
the identity (Box).

Every comparison is against an eager twin, as in test_gpu_rollout_linear.py: the actions, the outputs z, the env
outputs, the final observations on the rows the mask selects, ``get_state()``, ``snapshot()`` rows and observations, and
the step after.
"""
import math

import pytest

from test_gpu_rollout_linear import (BOX2D, CLASSIC, NAMES, _assert_equals_loop, _assert_same_env, _assert_untouched,
                                     _eq, _untouched)
from test_gpu_rollout_mlp import MlpTwin, _params

pytestmark = pytest.mark.gpu

HIDDEN = [(1,), (64,), (3, 7), (64, 64)]


def _torch():
    import torch
    return torch


def _argmax_first(y):
    """np.argmax over dim 1: the first NaN, else the first maximum."""
    torch = _torch()
    n = y.shape[0]
    m, best = y[:, 0], torch.zeros(n, dtype=torch.int64, device=y.device)
    for j in range(1, y.shape[1]):
        take = ~torch.isnan(m) & (torch.isnan(y[:, j]) | (y[:, j] > m))
        m = torch.where(take, y[:, j], m)
        best = torch.where(take, torch.full_like(best, j), best)
    return best


class NoisyTwin(MlpTwin):
    """MlpTwin with ``noisy_policy`` and ``noisy_loop``: the MLP's outputs plus the noise, then the action rule."""

    def noisy_policy(self, params, hidden, e):
        """-> (outputs z, action)"""
        z = self.outputs(params, hidden)
        y = z + e
        return z, (_argmax_first(y) if self.env.discrete else y)

    def noisy_loop(self, params, hidden, noise):
        """T = len(noise) steps -> (actions, outputs, [obs, reward, term, trunc], final obs, masks), stacked."""
        torch = _torch()
        acts, zs, outs, fin, masks = [], [], [], [], []
        for t in range(noise.shape[0]):
            z, a = self.noisy_policy(params, hidden, noise[t])
            o = self.env.step(a)
            self.obs = o[0].clone()
            acts.append(a)
            zs.append(z)
            outs.append([x.clone() for x in o[:4]])
            fin.append(o[4]["final_observation"].clone())
            masks.append(o[4]["_final_observation"].clone())
        return (torch.stack(acts), torch.stack(zs), [torch.stack([o[k] for o in outs]) for k in range(4)],
                torch.stack(fin), torch.stack(masks))


def _assert_equals_noisy(got, want, what=""):
    acts, outputs, obs, rew, term, trunc, infos = got
    wa, wz, wouts, wfin, wmask = want
    _eq(outputs, wz, f"{what}outputs")
    _assert_equals_loop((acts, obs, rew, term, trunc, infos), (wa, wouts, wfin, wmask), what)


def _pair(env_id, n, seed=3, **kwargs):
    import gym_b200
    envs = [gym_b200.vector.make(env_id, n, **kwargs) for _ in range(2)]
    obs = [e.reset(seed=seed)[0] for e in envs]
    return envs[0], NoisyTwin(envs[1], obs[1])


def _K(env):
    return int(env.single_action_space.n if env.discrete else env.act_dim)


def _noise(env, T, seed, scale=1.0):
    """Gumbel noise for a Discrete kind, scale * N(0, 1) for a Box kind, (T, N, K) on the env's device."""
    torch = _torch()
    g = torch.Generator(device=env.device).manual_seed(seed)
    shape = (T, env.num_envs, _K(env))
    if env.discrete:
        u = torch.rand(shape, generator=g, device=env.device).clamp_(min=torch.finfo(torch.float32).tiny)
        return -torch.log(-torch.log(u))
    return scale * torch.randn(shape, generator=g, device=env.device)


def _twin_check(env_id, n, T, hidden, per_env, seed=3, **kwargs):
    a, b = _pair(env_id, n, seed=seed, **kwargs)
    p = _params(a, hidden, per_env, seed + T)
    e = _noise(a, T, seed + 1)
    got = a.rollout_mlp_noisy(p, hidden, e)
    _assert_equals_noisy(got, b.noisy_loop(p, hidden, e))
    _eq(a.snapshot().obs, got[2][-1], "snapshot().obs vs obs[T-1]")
    _assert_same_env(a, b.env)
    nxt = b.policy(p, hidden)
    for name, x, y in zip(NAMES, a.step(nxt)[:4], b.env.step(nxt)[:4]):
        _eq(x, y, f"next step {name}")
    a.close()
    b.env.close()
    return got


# ---------------------------------------------------------------------------------------------- the eager twin
@pytest.mark.parametrize("per_env", [False, True], ids=["shared", "per_env"])
@pytest.mark.parametrize("n,T", [(1, 1), (257, 37), (33 * 256 + 5, 2), (4099, 300)])
@pytest.mark.parametrize("hidden", HIDDEN, ids=str)
@pytest.mark.parametrize("env_id", CLASSIC)
def test_rollout_mlp_noisy_equals_eager_loop(env_id, hidden, n, T, per_env):
    got = _twin_check(env_id, n, T, hidden, per_env)
    torch = _torch()
    box = env_id in ("MountainCarContinuous-v0", "Pendulum-v1")
    assert tuple(got[0].shape) == ((T, n, 1) if box else (T, n))
    assert got[0].dtype == (torch.float32 if box else torch.int64)
    K = 1 if box else 2 if env_id.startswith("CartPole") else 3
    assert got[1].dtype == torch.float32 and tuple(got[1].shape) == (T, n, K)


def test_unaligned_per_env_rows():
    """h1 % 4 == 0, but the per-env rows are not 16-byte aligned, so the second layer is read a float at a time: P % 4
    != 0, or P % 4 == 0 with params starting 4 bytes into their allocation."""
    _twin_check("MountainCar-v0", 515, 9, (4, 3), True)   # P = 39
    a, b = _pair("CartPole-v1", 515)
    p = _params(a, (8, 6), True, 4)                        # P = 108
    big = _torch().zeros(1 + p.numel(), device=p.device)
    big[1:] = p.reshape(-1)
    q = big[1:].view(p.shape)
    e = _noise(a, 9, 4)
    _assert_equals_noisy(a.rollout_mlp_noisy(q, (8, 6), e), b.noisy_loop(p, (8, 6), e))


@pytest.mark.parametrize("per_env", [False, True], ids=["shared", "per_env"])
@pytest.mark.parametrize("hidden", [(5,), (64, 64)], ids=str)
@pytest.mark.parametrize("env_id,kwargs", BOX2D, ids=[b[0] for b in BOX2D])
def test_box2d_rollout_mlp_noisy_equals_eager_loop(env_id, kwargs, hidden, per_env):
    _twin_check(env_id, 67, 5, hidden, per_env, seed=7, **kwargs)


@pytest.mark.parametrize("env_id", CLASSIC)
def test_rollout_mlp_noisy_short_time_limit_and_without_autoreset(env_id):
    got = _twin_check(env_id, 4099, 25, (16, 8), True, max_episode_steps=4)
    assert bool(got[5][3].any())
    _twin_check(env_id, 2053, 40, (6,), False, autoreset=False)
    _twin_check(env_id, 2053, 40, (6, 6), True, autoreset=False, max_episode_steps=4)


def test_rollout_mlp_noisy_offsets_past_two_to_the_31():
    """CartPole, n = 2^20, T = 520: the noise and outputs pass 2^31 bytes (4.4 GB each) and the observations 2^31
    elements; compared slice by slice with the eager loop."""
    torch = _torch()
    n, T, hidden = 1 << 20, 520, (8, 8)
    assert T * n * 2 * 4 > 1 << 31 and T * n * 4 > 1 << 31
    a, b = _pair("CartPole-v1", n, seed=5)
    p = _params(a, hidden, False, 5, scale=0.3)
    e = _noise(a, T, 5)
    acts, outputs, obs, rew, term, trunc, infos = a.rollout_mlp_noisy(p, hidden, e)
    fin, mask = infos["final_observation"], infos["_final_observation"]
    for t in range(T):
        z, act = b.noisy_policy(p, hidden, e[t])
        o, r, te, tr, inf = b.env.step(act)
        b.obs = o.clone()
        _eq(outputs[t], z, f"outputs[{t}]")
        _eq(acts[t], act, f"actions[{t}]")
        _eq(obs[t], o, f"obs[{t}]")
        _eq(rew[t], r, f"reward[{t}]")
        _eq(term[t], te, f"terminated[{t}]")
        _eq(trunc[t], tr, f"truncated[{t}]")
        m = inf["_final_observation"]
        _eq(mask[t], m, f"mask[{t}]")
        _eq(fin[t][m], inf["final_observation"][m], f"final_observation[{t}]")
    _assert_same_env(a, b.env)
    del acts, outputs, obs, rew, term, trunc, infos, fin, mask, e
    a.close()
    b.env.close()
    torch.cuda.empty_cache()


# --------------------------------------------------------------------------------------- -0.0 noise, IEEE sums
@pytest.mark.parametrize("per_env", [False, True], ids=["shared", "per_env"])
@pytest.mark.parametrize("env_id", CLASSIC + ["LunarLanderContinuous-v2"])
def test_minus_zero_noise_equals_rollout_mlp(env_id, per_env):
    """z + (-0.0) is z for every float32 z, so noise of -0.0 everywhere gives rollout_mlp()'s results bit for bit."""
    torch = _torch()
    n, T, hidden = (67, 5, (16, 16)) if env_id.startswith("Lunar") else (4099, 50, (64, 64))
    import gym_b200
    a, c = [gym_b200.vector.make(env_id, n) for _ in range(2)]
    for e in (a, c):
        e.reset(seed=21)
    p = _params(a, hidden, per_env, 21)
    got = a.rollout_mlp_noisy(p, hidden, torch.full((T, n, _K(a)), -0.0, device=a.device))
    want = c.rollout_mlp(p, hidden, T)
    _eq(got[0], want[0], "actions")
    for name, x, y in zip(NAMES, got[2:6], want[1:5]):
        _eq(x, y, name)
    _eq(got[6]["_final_observation"], want[5]["_final_observation"], "_final_observation")
    _assert_same_env(a, c)
    if a.discrete:
        _eq(got[0], torch.stack([_argmax_first(z) for z in got[1]]), "argmax of the outputs")
    else:
        _eq(got[0], got[1], "Box actions are the outputs")


def test_discrete_infinite_and_nan_noise():
    """-inf noise on a choice: never picked while its output is finite; NaN noise: the first NaN is picked; an output
    of +inf under -inf noise is NaN, and so picked."""
    torch = _torch()
    a, b = _pair("Acrobot-v1", 3000, seed=8)
    n, K, T = 3000, 3, 12
    p = _params(a, (8,), True, 8)
    e = _noise(a, T, 8)
    kind = torch.arange(n, device="cuda:0") % 3
    e[:, kind == 0, 0] = -math.inf
    e[:, kind == 1, 2] = math.nan
    got = a.rollout_mlp_noisy(p, (8,), e)
    _assert_equals_noisy(got, b.noisy_loop(p, (8,), e))
    assert bool((got[0][:, kind == 0] != 0).all()) and bool((got[0][:, kind == 1] == 2).all())
    # output 0 is +inf (its bias), and -inf noise there: NaN, the first NaN
    P = p.shape[1]
    q = torch.zeros(n, P, device="cuda:0")
    q[:, P - K] = math.inf
    e[:, :, 0] = -math.inf
    got = a.rollout_mlp_noisy(q, (8,), e)
    _assert_equals_noisy(got, b.noisy_loop(q, (8,), e))
    assert bool(torch.isposinf(got[1][:, :, 0]).all()) and bool((got[0] == 0).all())


# -------------------------------------------------------------------------------------------- interleaving
@pytest.mark.parametrize("env_id", ["CartPole-v1", "MountainCarContinuous-v0", "Acrobot-v1", "LunarLander-v2"])
def test_rollout_mlp_noisy_interleaved(env_id):
    """step(), rollout(), rollout_sampled(), rollout_linear(), rollout_mlp(), reset(seed=), restore and clone between
    calls, mirrored on the twin."""
    torch = _torch()
    n, T, hidden = (300, 3, (8,)) if env_id.startswith("Lunar") else (1000, 17, (12, 9))
    a, b = _pair(env_id, n)
    p = _params(a, hidden, True, 1)
    seeds = iter(range(100, 200))

    def check(what):
        e = _noise(a, T, next(seeds))
        _assert_equals_noisy(a.rollout_mlp_noisy(p, hidden, e), b.noisy_loop(p, hidden, e), what)

    check("first ")
    act = b.policy(p, hidden)
    o = a.step(act)
    b.obs = b.env.step(act)[0].clone()
    _eq(o[0], b.obs, "step")
    check("after step ")
    acts = b.policy(p, hidden)[None].repeat(4, *([1] * (1 + (not a.discrete))))
    ra, rb = a.rollout(acts), b.env.rollout(acts)
    b.obs = rb[0][-1].clone()
    _eq(ra[0], rb[0], "rollout obs")
    check("after rollout ")
    for e in (a, b.env):
        e.action_space.seed(4)
    sa, sb = a.rollout_sampled(3), b.env.rollout_sampled(3)
    b.obs = sb[1][-1].clone()
    _eq(sa[1], sb[1], "rollout_sampled obs")
    check("after rollout_sampled ")
    K = _K(a)
    w = torch.randn(n, K, a.obs_dim, device="cuda:0")
    bias = torch.randn(n, K, device="cuda:0")
    la, lb = a.rollout_linear(w, bias, 3), b.env.rollout_linear(w, bias, 3)
    b.obs = lb[1][-1].clone()
    _eq(la[1], lb[1], "rollout_linear obs")
    check("after rollout_linear ")
    ma, mb = a.rollout_mlp(p, hidden, 3), b.env.rollout_mlp(p, hidden, 3)
    b.obs = mb[1][-1].clone()
    _eq(ma[1], mb[1], "rollout_mlp obs")
    check("after rollout_mlp ")
    snap_a, snap_b = a.snapshot(), b.env.snapshot()
    check("before restore ")
    ra = a.reset(seed=77)[0]
    b.obs = b.env.reset(seed=77)[0].clone()
    _eq(ra, b.obs, "reset")
    check("after reset ")
    ro = a.restore(snap_a)[0]
    b.obs = b.env.restore(snap_b)[0].clone()
    _eq(ro, b.obs, "restore")
    check("after restore ")
    src = torch.randint(0, n, (n,), device="cuda:0")
    co = a.clone(src)
    b.obs = b.env.clone(src).clone()
    _eq(co, b.obs, "clone")
    check("after clone ")
    _assert_same_env(a, b.env)


def test_set_state_then_rollout_mlp_noisy_starts_from_the_state():
    """After set_state() the first input is the observation of that state; a step with an out-of-range action returns
    exactly that, so a probe env gives the twin its first input."""
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
    p = _params(a, (64, 64), True, 6)
    e = _noise(a, 9, 6)
    _assert_equals_noisy(a.rollout_mlp_noisy(p, (64, 64), e), b.noisy_loop(p, (64, 64), e))
    _assert_same_env(a, b.env)


# ------------------------------------------------------------------------------------------------ CUDA graphs
@pytest.mark.parametrize("fill", ["in_place", "in_graph"])
@pytest.mark.parametrize("per_env", [False, True], ids=["shared", "per_env"])
@pytest.mark.parametrize("env_id", ["CartPole-v1", "Pendulum-v1", "Acrobot-v1"])
def test_captured_rollout_mlp_noisy_replays_equal_eager_calls(env_id, per_env, fill):
    """Replay k equals eager call k, after a captured step(), with the parameters copied in place between replays and
    the noise either copied in place too (in_place) or drawn inside the graph (in_graph: the whole collection, noise
    included, is one graph; the twin reads what the replay drew)."""
    torch = _torch()
    n, T, k, hidden = 515, 24, 3, (16, 12)
    a, b = _pair(env_id, n)
    p = _params(a, hidden, per_env, 2)
    e = _noise(a, T, 2)
    step_act = b.policy(p, hidden)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        st = a.step(step_act)
        if fill == "in_graph":
            if a.discrete:
                u = torch.rand(e.shape, device=e.device).clamp_(min=torch.finfo(torch.float32).tiny)
                e.copy_(-torch.log(-torch.log(u)))
            else:
                e.copy_(0.3 * torch.randn(e.shape, device=e.device))
        out = a.rollout_mlp_noisy(p, hidden, e)
    for r in range(k):
        p2 = _params(a, hidden, per_env, 100 + r)
        p.copy_(p2)
        if fill == "in_place":
            e.copy_(_noise(a, T, 200 + r))
        g.replay()
        o = b.env.step(step_act)
        b.obs = o[0].clone()
        for name, x, y in zip(NAMES, st[:4], o[:4]):
            _eq(x, y, f"replay {r} step {name}")
        e_now = e.clone()
        _assert_equals_noisy(out, b.noisy_loop(p2, hidden, e_now), f"replay {r} ")
        if fill == "in_graph" and r > 0:
            assert not torch.equal(e_now, e_prev), "each replay draws new noise"
        e_prev = e_now
    _assert_same_env(a, b.env)


@pytest.mark.parametrize("env_id,kwargs", BOX2D[:2], ids=[b[0] for b in BOX2D[:2]])
def test_box2d_capture_is_refused(env_id, kwargs):
    from gym_b200 import error
    torch = _torch()
    a, b = _pair(env_id, 33, seed=7, **kwargs)
    p = _params(a, (8,), False, 3)
    e = _noise(a, 2, 3)
    before = _untouched(a)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with pytest.raises(error.Error, match="double|alternate|stale"):
        with torch.cuda.graph(g):
            a.rollout_mlp_noisy(p, (8,), e)
    del g
    _assert_untouched(a, before, "capture")
    _assert_equals_noisy(a.rollout_mlp_noisy(p, (8,), e), b.noisy_loop(p, (8,), e), "after the refused capture ")


# ------------------------------------------------------------------------------------------ the docstring's recipes
def test_gumbel_recipe_samples_softmax():
    """CartPole, zero weights and output bias (log 0.3, log 0.7): with the docstring's Gumbel noise the frequency of
    action 1 over 2^20 env-steps is within 5 sigma of 0.7, and Categorical(logits=outputs) gives log 0.3 / log 0.7."""
    torch = _torch()
    import gym_b200
    n, T = 1 << 14, 64
    env = gym_b200.vector.make("CartPole-v1", n)
    env.reset(seed=1)
    P = 4 * 1 + 1 + 2 * 1 + 2
    params = torch.zeros(P, device="cuda:0")
    params[-2:] = torch.tensor([math.log(0.3), math.log(0.7)])
    torch.manual_seed(1234)
    u = torch.rand(T, n, 2, device="cuda:0").clamp_(min=torch.finfo(torch.float32).tiny)
    g = -torch.log(-torch.log(u))
    a, logits, *_ = env.rollout_mlp_noisy(params, (1,), g)
    freq = a.double().mean().item()
    sigma = math.sqrt(0.7 * 0.3 / (n * T))
    assert abs(freq - 0.7) < 5 * sigma, (freq, sigma)
    logp = torch.distributions.Categorical(logits=logits).log_prob(a)
    want = torch.where(a == 1, math.log(0.7), math.log(0.3)).float()
    torch.testing.assert_close(logp, want, rtol=0, atol=1e-6)
    env.close()


def test_gaussian_recipe_on_pendulum():
    """Pendulum with the docstring's Gaussian noise: the actions are outputs + noise, one float32 add, so
    Normal(outputs, std).log_prob(actions) is Normal(0, std).log_prob(noise) to float32 rounding.  Noise on a grid of
    2^-12 with outputs on it too (zero weights, bias 0.25) makes every sum exact, and then actions - outputs == noise."""
    torch = _torch()
    import gym_b200
    n, T, hidden = 4096, 32, (64, 64)
    env = gym_b200.vector.make("Pendulum-v1", n)
    env.reset(seed=2)
    std = torch.tensor(0.6, device="cuda:0")
    p = _params(env, hidden, False, 3)
    torch.manual_seed(5)
    noise = std * torch.randn(T, n, 1, device="cuda:0")
    a, mean, *_ = env.rollout_mlp_noisy(p, hidden, noise)
    _eq(a, mean + noise, "actions == outputs + noise")
    lp = torch.distributions.Normal(mean, std).log_prob(a)
    torch.testing.assert_close(lp, torch.distributions.Normal(0.0, std).log_prob(noise), rtol=1e-4, atol=1e-4)
    q = torch.zeros_like(p)
    q[-1] = 0.25
    grid = torch.round(noise * 4096) / 4096
    a, mean, *_ = env.rollout_mlp_noisy(q, hidden, grid)
    assert bool((mean == 0.25).all())
    assert torch.equal(a - mean, grid), "actions - outputs == noise"   # as values: 0.25 - 0.25 is +0.0 for noise -0.0
    env.close()


# ------------------------------------------------------------------------------------------ refusals and guards
def test_rollout_mlp_noisy_guards_and_refusals():
    import gym_b200
    from gym_b200 import error, wrappers
    from gym_b200.distributed import ShardedVectorEnv
    from gym_b200.env import B200Env
    torch = _torch()

    env = gym_b200.vector.make("CartPole-v1", 64)
    p = _params(env, (8, 4), False, 0)
    e = torch.zeros(3, 64, 2, device="cuda:0")
    with pytest.raises(error.ResetNeeded):
        env.rollout_mlp_noisy(p, (8, 4), e)
    env.reset(seed=1)
    before = _untouched(env)
    pp = _params(env, (8, 4), True, 0)
    bad_args = [
        (p.double(), (8, 4), e), (p.cpu(), (8, 4), e), (p[:-1], (8, 4), e), (pp[:, :-1], (8, 4), e),
        (p, (8,), e), (p, (8, 65), e), (p, (), e), (p, (8, 4, 4), e), (p, (True, 4), e), (p.tolist(), (8, 4), e),
        (p, (8, 4), e.double()), (p, (8, 4), e.half()), (p, (8, 4), e.cpu()),            # noise dtype, device
        (p, (8, 4), e[:, :, :1]), (p, (8, 4), torch.zeros(3, 64, 3, device="cuda:0")),   # the wrong K
        (p, (8, 4), e[:, :63]), (p, (8, 4), e[0]), (p, (8, 4), e[None]),                 # the wrong N, rank
        (p, (8, 4), e[:0]),                                                               # T = 0
        (p, (8, 4), e.transpose(0, 1).contiguous().transpose(0, 1)),                      # not contiguous
        (p, (8, 4), e.tolist()), (p, (8, 4), None),
    ]
    for k, (x, h, y) in enumerate(bad_args):
        with pytest.raises(ValueError):
            env.rollout_mlp_noisy(x, h, y)
        _assert_untouched(env, before, f"bad arguments {k}")
    env.step_async(torch.zeros(64, dtype=torch.int64, device="cuda:0"))
    with pytest.raises(error.AlreadyPendingCallError):
        env.rollout_mlp_noisy(p, (8, 4), e)
    env.step_wait()
    before = _untouched(env)
    for wr in (wrappers.RecordEpisodeStatistics(env), wrappers.NormalizeObservation(env),
               wrappers.NormalizeReward(env), wrappers.VectorListInfo(env)):
        with pytest.raises(error.Error, match="rollout_mlp_noisy"):
            wr.rollout_mlp_noisy(p, (8, 4), e)
    _assert_untouched(env, before, "wrappers")
    env.close()
    with pytest.raises(error.ClosedEnvironmentError):
        env.rollout_mlp_noisy(p, (8, 4), e)

    host = gym_b200.vector.make("CartPole-v1", 16, backend="numpy")
    host.reset(seed=3)
    rows = host.snapshot().rows.clone()
    with pytest.raises(error.Error, match="backend"):
        host.rollout_mlp_noisy(p, (8, 4), e[:, :16])
    assert torch.equal(host.snapshot().rows, rows)
    host.close()

    from gym_b200 import subenv
    chain = gym_b200.vector.make("CartPole-v1", 16, wrappers=[subenv.RecordEpisodeStatistics()])
    chain.reset(seed=4)
    before = _untouched(chain)
    with pytest.raises(error.Error, match="wrappers"):
        chain.rollout_mlp_noisy(p, (8, 4), e[:, :16].contiguous())
    _assert_untouched(chain, before, "per-env wrappers")
    chain.close()

    assert not hasattr(ShardedVectorEnv, "rollout_mlp_noisy")
    assert not hasattr(B200Env, "rollout_mlp_noisy")


def test_c_entry_point_validates_its_arguments():
    """The C entry point checks the layer count, the widths, T and the buffers itself, for callers other than the
    Python layer, and launches nothing when they are wrong."""
    import ctypes

    import gym_b200
    torch = _torch()
    env = gym_b200.vector.make("CartPole-v1", 8)
    env.reset(seed=2)
    p = _params(env, (4,), False, 0)
    buf = torch.zeros(64, 8, 4, device="cuda:0")
    before = _untouched(env)
    vp = ctypes.c_void_p
    ok = vp(buf.data_ptr())
    good = dict(layers=1, h1=4, h2=0, T=3, noise=ok, outputs=ok, actions=ok, obs=ok, reward=ok, term=ok, trunc=ok,
                last=ok)
    bad = [dict(layers=0), dict(layers=3, h2=4), dict(h1=0), dict(h1=65), dict(layers=2, h2=0), dict(layers=2, h2=65),
           dict(T=0), dict(T=-1), dict(noise=None), dict(outputs=None), dict(actions=None), dict(obs=None),
           dict(reward=None), dict(term=None), dict(trunc=None), dict(last=None)]
    for change in bad:
        c = {**good, **change}
        rc = env._lib.b200gym_rollout_mlp_noisy(env._handle, vp(p.data_ptr()), 0, c["layers"], c["h1"], c["h2"],
                                                c["T"], c["noise"], c["outputs"], c["actions"], c["obs"], c["reward"],
                                                c["term"], c["trunc"], None, c["last"], ok, env._stream())
        assert rc != 0, change
        assert b"b200gym_rollout_mlp_noisy" in env._lib.b200gym_last_error(env._handle)
    _assert_untouched(env, before, "C-side refusals")
    env.close()
