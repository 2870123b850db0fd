"""``rollout_mlp_noisy(..., obs_norm=, clip_obs=)`` and ``rollout_actor_critic(..., obs_norm=, reward_norm=, ...)`` on
the GPU, against an eager twin: test_gpu_rollout_actor_critic.py's twin (the MLP restated in torch elementwise ops),
with every network input normalised by the torch expression of the contract,
``((o.double() - mean) / torch.sqrt(var + eps)).float().clamp(-c, c)``, and the rewards the GAE reads scaled by
``(r / torch.sqrt(var + eps)).float().clamp(-c_r, c_r)``.  Every output is compared bit for bit (float32 as int32
views), and the env afterwards.
"""
import numpy as np
import pytest

from test_gpu_rollout_actor_critic import _nets, coefficients, gae_restated, mlp
from test_gpu_rollout_linear import BOX2D, CLASSIC, NAMES, _assert_same_env, _assert_untouched, _eq, _untouched
from test_gpu_rollout_mlp_noisy import _K, _argmax_first, _noise

pytestmark = pytest.mark.gpu

HIDDEN = [(1,), (64,), (3, 7), (64, 64)]
ACTS = ["relu", "tanh"]
SHAPES = [(1, 1), (257, 37), (33 * 256 + 5, 37), (4099, 300)]


def _torch():
    import torch
    return torch


def normalize(o, mean, var, eps, clip):
    x = ((o.double() - mean) / _torch().sqrt(var + eps)).float()
    return x if clip is None else x.clamp(-float(np.float32(clip)), float(np.float32(clip)))


def scale_rewards(r, rvar, eps, clip):
    x = (r / _torch().sqrt(rvar + eps)).float()
    return x if clip is None else x.clamp(-float(np.float32(clip)), float(np.float32(clip)))


class NormTwin:
    """An env stepped eagerly with the restated nets reading normalised inputs."""

    def __init__(self, env, obs, activation):
        self.env, self.obs, self.activation = env, obs.clone(), activation
        self.K = _K(env)

    def loop(self, actor, critic, hidden, noise, norm, gamma=0.99, gae_lambda=0.95):
        """norm: dict(mean, var, eps, clip, rvar, clip_r); critic None: the noisy rollout only ->
        (actions, outputs, values, advantages, [obs, reward, term, trunc], final obs, masks), stacked."""
        torch = _torch()
        x = lambda o: o if norm["mean"] is None else normalize(o, norm["mean"], norm["var"], norm["eps"],  # noqa: E731
                                                               norm["clip"])
        V = lambda o: mlp(critic, hidden, x(o), 1, self.activation)[:, 0]  # noqa: E731
        acts, zs, vals, vfs, outs, fin, masks = [], [], [], [], [], [], []
        for t in range(noise.shape[0]):
            if critic is not None:
                vals.append(V(self.obs))
            z = mlp(actor, hidden, x(self.obs), self.K, self.activation)
            y = z + noise[t]
            a = _argmax_first(y) if self.env.discrete else y
            o = self.env.step(a)
            self.obs = o[0].clone()
            acts.append(a)
            zs.append(z)
            outs.append([v.clone() for v in o[:4]])
            fin.append(o[4]["final_observation"].clone())
            masks.append(o[4]["_final_observation"].clone())
            if critic is not None:
                vfs.append(V(fin[-1]))
        o4 = [torch.stack([o[k] for o in outs]) for k in range(4)]
        values = adv = None
        if critic is not None:
            vals.append(V(self.obs))
            values = torch.stack(vals)
            r = o4[1] if norm.get("rvar") is None else scale_rewards(o4[1], norm["rvar"], norm["eps"], norm["clip_r"])
            adv = gae_restated(*coefficients(gamma, gae_lambda), r, o4[2], o4[3], values, torch.stack(vfs))
        return torch.stack(acts), torch.stack(zs), values, adv, o4, torch.stack(fin), torch.stack(masks)


def _assert_equals(got, want, what=""):
    if len(got) == 7:                                   # rollout_mlp_noisy
        got = (got[0], got[1], None, None) + tuple(got[2:])
    acts, outputs, values, adv, obs, rew, term, trunc, infos = got
    wa, wz, wv, wadv, (wo, wr, wte, wtr), wfin, wmask = want
    _eq(acts, wa, f"{what}actions")
    _eq(outputs, wz, f"{what}outputs")
    if wv is not None:
        _eq(values, wv, f"{what}values")
        _eq(adv, wadv, f"{what}advantages")
    for name, x, y in zip(NAMES, (obs, rew, term, trunc), (wo, wr, wte, wtr)):
        _eq(x, y, f"{what}{name}")
    m = infos["_final_observation"]
    _eq(m, wmask, f"{what}_final_observation")
    _eq(infos["final_observation"][m], wfin[wmask], f"{what}final_observation")


def _pair(env_id, n, activation="relu", seed=3, **kwargs):
    import gym_b200
    envs = [gym_b200.vector.make(env_id, n, **kwargs) for _ in range(2)]
    obs = [e.reset(seed=seed)[0] for e in envs]
    return envs[0], NormTwin(envs[1], obs[1], activation)


def _stats(env, seed, clip=10.0, clip_r=10.0, eps=1e-8):
    torch = _torch()
    g = torch.Generator(device="cpu").manual_seed(seed)
    D = env.obs_dim
    mean = (0.3 * torch.randn(D, generator=g, dtype=torch.float64)).to(env.device)
    var = (2.0 * torch.rand(D, generator=g, dtype=torch.float64) + 0.01).to(env.device)
    rvar = (5.0 * torch.rand(1, generator=g, dtype=torch.float64) + 0.1).to(env.device)
    return dict(mean=mean, var=var, eps=eps, clip=clip, rvar=rvar, clip_r=clip_r)


def _kw(norm, rewards=True):
    kw = dict(obs_norm=(norm["mean"], norm["var"]), norm_epsilon=norm["eps"], clip_obs=norm["clip"])
    if rewards:
        kw.update(reward_norm=norm["rvar"], clip_reward=norm["clip_r"])
    return kw


def _twin_check(env_id, n, T, hidden, activation="relu", seed=3, clip=10.0, clip_r=10.0, **kwargs):
    a, b = _pair(env_id, n, activation, seed=seed, **kwargs)
    pa, pc = _nets(a, hidden, seed + T)
    norm = _stats(a, seed, clip, clip_r)
    e = _noise(a, T, seed + 1)
    kw = dict(gamma=0.99, gae_lambda=0.95, activation=activation, **_kw(norm))
    got = a.rollout_actor_critic(pa, pc, hidden, e, **kw)
    _assert_equals(got, b.loop(pa, pc, hidden, e, norm))
    _assert_same_env(a, b.env)
    e2 = _noise(a, 2, seed + 2)
    nxt = a.rollout_actor_critic(pa, pc, hidden, e2, **kw)
    _assert_equals(nxt, b.loop(pa, pc, hidden, e2, norm), "next call ")
    _eq(nxt[2][0], got[2][-1], "next call's values[0] vs values[T]")
    # the noisy rollout with the same statistics continues from there
    e3 = _noise(a, 3, seed + 3)
    noisy = a.rollout_mlp_noisy(pa, hidden, e3, activation=activation, **_kw(norm, rewards=False))
    _assert_equals(noisy, b.loop(pa, None, hidden, e3, norm), "rollout_mlp_noisy ")
    _assert_same_env(a, b.env)
    a.close()
    b.env.close()
    return got


# ---------------------------------------------------------------------------------------------- the eager twin
@pytest.mark.parametrize("activation", ACTS)
@pytest.mark.parametrize("n,T", SHAPES)
@pytest.mark.parametrize("hidden", HIDDEN, ids=str)
@pytest.mark.parametrize("env_id", CLASSIC)
def test_normalised_rollouts_equal_eager_loop(env_id, hidden, n, T, activation):
    """Tight clips (0.8 for the observations, 0.5 for the rewards) with ReLU, so the clamps act often; the usual 10
    with tanh."""
    clips = (0.8, 0.5) if activation == "relu" else (10.0, 10.0)
    _twin_check(env_id, n, T, hidden, activation, clip=clips[0], clip_r=clips[1])


@pytest.mark.parametrize("clips", [(None, None), (None, 1.0), (2.0, None)])
@pytest.mark.parametrize("env_id", CLASSIC)
def test_truncations_and_optional_clips(env_id, clips):
    """max_episode_steps=5: the bootstrap of a truncation reads the normalised final observation; each clip may be
    left out."""
    got = _twin_check(env_id, 4099, 23, (16, 8), "tanh", clip=clips[0], clip_r=clips[1], max_episode_steps=5)
    assert bool((got[7] & ~got[6]).any())


@pytest.mark.parametrize("env_id", CLASSIC)
def test_only_one_of_the_normalisations(env_id):
    """obs_norm alone leaves the GAE on raw rewards; reward_norm alone leaves the nets on raw observations."""
    torch = _torch()
    a, b = _pair(env_id, 515, "tanh", seed=6, max_episode_steps=9)
    pa, pc = _nets(a, (16,), 6)
    norm = _stats(a, 6)
    e = _noise(a, 20, 6)
    got = a.rollout_actor_critic(pa, pc, (16,), e, gamma=0.99, gae_lambda=0.95, activation="tanh",
                                 obs_norm=(norm["mean"], norm["var"]))
    _assert_equals(got, b.loop(pa, pc, (16,), e, dict(norm, clip=None, rvar=None)))
    got = a.rollout_actor_critic(pa, pc, (16,), e, gamma=0.99, gae_lambda=0.95, activation="tanh",
                                 reward_norm=norm["rvar"], clip_reward=3.0)
    _assert_equals(got, b.loop(pa, pc, (16,), e, dict(norm, mean=None, clip_r=3.0)))
    _assert_same_env(a, b.env)
    torch.cuda.synchronize()


@pytest.mark.parametrize("env_id", CLASSIC)
def test_identity_statistics_give_the_calls_without_normalisation(env_id):
    """mean 0, var 1, eps 0, no clip: bit for bit the calls without the keywords, on a twin env."""
    import gym_b200
    torch = _torch()
    n, T, hidden = 1000, 40, (64, 64)
    envs = [gym_b200.vector.make(env_id, n, max_episode_steps=13) for _ in range(2)]
    for e in envs:
        e.reset(seed=11)
    pa, pc = _nets(envs[0], hidden, 11)
    D = envs[0].obs_dim
    mean = torch.zeros(D, dtype=torch.float64, device="cuda:0")
    var = torch.ones(D, dtype=torch.float64, device="cuda:0")
    rvar = torch.ones(1, dtype=torch.float64, device="cuda:0")
    for act in ACTS:
        e = _noise(envs[0], T, 12)
        got = envs[0].rollout_actor_critic(pa, pc, hidden, e, gamma=0.99, gae_lambda=0.95, activation=act,
                                           obs_norm=(mean, var), norm_epsilon=0.0, reward_norm=rvar)
        want = envs[1].rollout_actor_critic(pa, pc, hidden, e, gamma=0.99, gae_lambda=0.95, activation=act)
        for k in range(8):
            _eq(got[k], want[k], f"{act} rollout_actor_critic output {k}")
        got = envs[0].rollout_mlp_noisy(pa, hidden, e, activation=act, obs_norm=(mean, var), norm_epsilon=0)
        want = envs[1].rollout_mlp_noisy(pa, hidden, e, activation=act)
        for k in range(6):
            _eq(got[k], want[k], f"{act} rollout_mlp_noisy output {k}")
    _assert_same_env(envs[0], envs[1])


@pytest.mark.parametrize("env_id", ["CartPole-v1", "MountainCar-v0", "Pendulum-v1", "Acrobot-v1"])
def test_normalised_input_equals_rms_apply_obs(env_id):
    """A critic with hidden (2,) whose output is relu(x[k]) - relu(-x[k]) = x[k] exactly (for x[k] != -0.0) reads one
    normalised input; values[t] must be column k of b200gym_rms_apply_obs (no update) on the step's input rows, with
    the same statistics in its [mean, var, count] layout."""
    import ctypes
    torch = _torch()
    n, T = 2000, 6
    a, b = _pair(env_id, n, seed=4)
    D = a.obs_dim
    norm = _stats(a, 4)
    pa = _nets(a, (2,), 4)[0]
    stats = torch.cat([norm["mean"], norm["var"], torch.ones(1, dtype=torch.float64, device="cuda:0")])
    spare = torch.zeros_like(stats)
    scratch = torch.zeros(2 * D, dtype=torch.float64, device="cuda:0")
    vp = ctypes.c_void_p
    first = b.obs                                          # the observations the env last returned
    for k in range(D):
        pc = torch.zeros(2 * D + 2 + 2 + 1, device="cuda:0")
        pc[k], pc[D + k] = 1.0, -1.0                      # W1 rows e_k and -e_k, b1 = 0
        pc[2 * D + 2], pc[2 * D + 3] = 1.0, -1.0           # W2 = [1, -1], b2 = 0
        e = _noise(a, T, 20 + k)
        got = a.rollout_actor_critic(pa, pc, (2,), e, gamma=0.99, gae_lambda=0.95, obs_norm=(norm["mean"], norm["var"]))
        inputs = torch.cat([first[None], got[4]]).contiguous()     # T + 1 rows: values[t] reads row t
        ref = torch.empty_like(inputs)
        for t in range(T + 1):
            assert a._lib.b200gym_rms_apply_obs(vp(inputs[t].data_ptr()), vp(ref[t].data_ptr()), n, D,
                                                vp(stats.data_ptr()), vp(spare.data_ptr()), vp(scratch.data_ptr()),
                                                vp(scratch.data_ptr()), float(n), norm["eps"], 0, a._stream()) == 0
        torch.cuda.synchronize()
        _eq(got[2], ref[:, :, k].contiguous(), f"column {k}")
        first = got[4][-1].clone()
    a.close()
    b.env.close()


# ------------------------------------------------------------------------------------------------ CUDA graphs
@pytest.mark.parametrize("env_id", ["CartPole-v1", "Pendulum-v1", "Acrobot-v1", "MountainCarContinuous-v0"])
def test_captured_replays_read_the_current_statistics(env_id):
    """One graph draws the noise and runs both calls; between replays the statistics are rewritten in place, and
    replay k equals eager calls of the twin with the statistics of replay k."""
    torch = _torch()
    n, T, hidden = 515, 16, (16, 12)
    a, b = _pair(env_id, n, "tanh")
    pa, pc = _nets(a, hidden, 2)
    norm = _stats(a, 2, clip=1.5, clip_r=2.0)
    e = _noise(a, T, 2)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        if a.discrete:
            u = torch.rand(e.shape, device=e.device).clamp_(min=torch.finfo(torch.float32).tiny)
            e.copy_(-torch.log(-torch.log(u)))
        else:
            e.copy_(0.3 * torch.randn(e.shape, device=e.device))
        out = a.rollout_actor_critic(pa, pc, hidden, e, gamma=0.98, gae_lambda=0.9, activation="tanh", **_kw(norm))
        out2 = a.rollout_mlp_noisy(pa, hidden, e, activation="tanh", **_kw(norm, rewards=False))
    for r in range(3):
        new = _stats(a, 100 + r, clip=1.5, clip_r=2.0)
        for key in ("mean", "var", "rvar"):
            norm[key].copy_(new[key])
        g.replay()
        e_now = e.clone()
        snap = dict(norm, mean=norm["mean"].clone(), var=norm["var"].clone(), rvar=norm["rvar"].clone())
        _assert_equals(out, b.loop(pa, pc, hidden, e_now, snap, 0.98, 0.9), f"replay {r} ")
        _assert_equals(out2, b.loop(pa, None, hidden, e_now, snap), f"replay {r} noisy ")
    _assert_same_env(a, b.env)


# ---------------------------------------------------------------------------------------------------- Box2D
@pytest.mark.parametrize("hidden", [(5,), (64, 64)], ids=str)
@pytest.mark.parametrize("env_id,kwargs", BOX2D[:3], ids=[b[0] for b in BOX2D[:3]])
def test_box2d_equals_eager_loop(env_id, kwargs, hidden):
    _twin_check(env_id, 67, 5, hidden, "tanh", seed=7, clip=1.0, clip_r=0.5, **kwargs)


def test_box2d_truncations_bootstrap():
    got = _twin_check("LunarLanderContinuous-v2", 33, 7, (8,), seed=9, max_episode_steps=3)
    assert bool((got[7] & ~got[6]).any())


@pytest.mark.parametrize("env_id,kwargs", BOX2D[:3], ids=[b[0] for b in BOX2D[:3]])
def test_box2d_capture_is_refused(env_id, kwargs):
    from gym_b200 import error
    torch = _torch()
    a, b = _pair(env_id, 33, seed=7, **kwargs)
    pa, pc = _nets(a, (8,), 3)
    norm = _stats(a, 3)
    e = _noise(a, 2, 3)
    before = _untouched(a)
    for call in (lambda: a.rollout_actor_critic(pa, pc, (8,), e, gamma=0.99, gae_lambda=0.95, **_kw(norm)),
                 lambda: a.rollout_mlp_noisy(pa, (8,), e, **_kw(norm, rewards=False))):
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with pytest.raises(error.Error, match="double|alternate|stale"):
            with torch.cuda.graph(g):
                call()
        del g
        _assert_untouched(a, before, "capture")
    _assert_equals(a.rollout_actor_critic(pa, pc, (8,), e, gamma=0.99, gae_lambda=0.95, **_kw(norm)),
                   b.loop(pa, pc, (8,), e, norm), "after the refused capture ")


# ------------------------------------------------------------------------------------------ refusals and guards
def test_refusals_leave_the_env_untouched():
    import gym_b200
    from gym_b200 import error, wrappers
    torch = _torch()

    env = gym_b200.vector.make("CartPole-v1", 64)
    env.reset(seed=1)
    pa, pc = _nets(env, (8, 4), 0)
    e = torch.zeros(3, 64, 2, device="cuda:0")
    m = torch.zeros(4, dtype=torch.float64, device="cuda:0")
    v = torch.ones(4, dtype=torch.float64, device="cuda:0")
    rv = torch.ones(1, dtype=torch.float64, device="cuda:0")
    ac = dict(gamma=0.99, gae_lambda=0.95)
    bad_stats = [m.float(), m.cpu(), m[:3], torch.zeros(4, 2, dtype=torch.float64, device="cuda:0")[:, 0],
                 torch.zeros(5, dtype=torch.float64, device="cuda:0"), m.tolist(), None]
    bad_obs_norm = [(x, v) for x in bad_stats] + [(m, x) for x in bad_stats] + [m, (m,), (m, v, v), "mv"]
    bad_scalar = [float("nan"), float("inf"), -1.0, 0, 0.0, 1e-50, 1e39, True, False, np.bool_(True), "10",
                  torch.tensor(10.0), 1j]
    bad_eps = [float("nan"), float("inf"), -1e-8, True, None, "1e-8", torch.tensor(1e-8), 1j]
    cases = []
    for on in bad_obs_norm:
        cases.append(("noisy", dict(obs_norm=on)))
        cases.append(("ac", dict(obs_norm=on)))
    for x in bad_eps:
        cases.append(("noisy", dict(obs_norm=(m, v), norm_epsilon=x)))
        cases.append(("ac", dict(norm_epsilon=x)))
    for x in bad_scalar:
        cases.append(("noisy", dict(obs_norm=(m, v), clip_obs=x)))
        cases.append(("ac", dict(obs_norm=(m, v), clip_obs=x)))
        cases.append(("ac", dict(reward_norm=rv, clip_reward=x)))
    for x in (rv.float(), rv.cpu(), torch.ones(2, dtype=torch.float64, device="cuda:0"),
              torch.ones((), dtype=torch.float64, device="cuda:0"), 1.0):
        cases.append(("ac", dict(reward_norm=x)))
    cases += [("noisy", dict(clip_obs=10.0)), ("ac", dict(clip_obs=10.0)), ("ac", dict(clip_reward=10.0)),
              ("ac", dict(obs_norm=(m, v), clip_reward=10.0)), ("ac", dict(reward_norm=rv, clip_obs=10.0)),
              ("noisy_per_env", dict(obs_norm=(m, v)))]
    before = _untouched(env)
    for k, (which, kw) in enumerate(cases):
        with pytest.raises(ValueError):
            if which == "noisy":
                env.rollout_mlp_noisy(pa, (8, 4), e, **kw)
            elif which == "noisy_per_env":
                env.rollout_mlp_noisy(pa.expand(64, -1).contiguous(), (8, 4), e, **kw)
            else:
                env.rollout_actor_critic(pa, pc, (8, 4), e, **ac, **kw)
        _assert_untouched(env, before, f"bad arguments {k}: {which} {kw}")
    with pytest.raises(TypeError):
        env.rollout_mlp_noisy(pa, (8, 4), e, reward_norm=rv)        # rollout_mlp_noisy has no reward keywords
    # per-env rows without obs_norm still run, as before
    env.rollout_mlp_noisy(pa.expand(64, -1).contiguous(), (8, 4), e)
    before = _untouched(env)
    for wr in (wrappers.NormalizeObservation(env), wrappers.NormalizeReward(env)):
        with pytest.raises(error.Error, match="rollout"):
            wr.rollout_actor_critic(pa, pc, (8, 4), e, **ac)
        with pytest.raises(error.Error, match="rollout"):
            wr.rollout_mlp_noisy(pa, (8, 4), e)
    _assert_untouched(env, before, "wrappers")
    env.close()

    no_reset = gym_b200.vector.make("CartPole-v1", 64, autoreset=False)
    no_reset.reset(seed=2)
    before = _untouched(no_reset)
    with pytest.raises(error.Error, match="autoreset"):
        no_reset.rollout_actor_critic(pa, pc, (8, 4), e, **ac, obs_norm=(m, v), reward_norm=rv)
    _assert_untouched(no_reset, before, "autoreset=False")
    no_reset.close()


def test_c_entry_points_validate_their_arguments():
    """The C entry points check the statistics pointers, eps and the clips themselves, and launch nothing when they
    are wrong; a null mean / var is 'not normalised' and a clip of +inf 'no clip'."""
    import ctypes
    import math

    import gym_b200
    torch = _torch()
    env = gym_b200.vector.make("CartPole-v1", 8)
    env.reset(seed=2)
    pa, pc = _nets(env, (4,), 0)
    buf = torch.zeros(64, 8, 4, device="cuda:0")
    st = torch.ones(8, dtype=torch.float64, device="cuda:0")
    before = _untouched(env)
    vp = ctypes.c_void_p
    ok, s = vp(buf.data_ptr()), vp(st.data_ptr())
    inf = math.inf
    good = dict(per_env=0, mean=s, var=s, eps=1e-8, clip=inf, rvar=s, clip_r=inf, h1=4, act=0)
    bad = [dict(mean=None), dict(var=None), dict(eps=-1.0), dict(eps=float("nan")), dict(eps=inf), dict(clip=0.0),
           dict(clip=-1.0), dict(clip=float("nan")), dict(clip=-inf), dict(mean=None, var=None, clip=10.0),
           dict(per_env=1), dict(h1=0), dict(act=2)]
    bad_ac = [dict(clip_r=0.0), dict(clip_r=float("nan")), dict(rvar=None, clip_r=10.0)]
    for change in bad + bad_ac:
        c = {**good, **change}
        if change in bad:
            rc = env._lib.b200gym_rollout_mlp_noisy_norm(
                env._handle, vp(pa.data_ptr()), c["per_env"], 1, c["h1"], 0, 3, ok, ok, ok, ok, ok, ok, ok, ok, ok,
                ok, env._stream(), c["act"], c["mean"], c["var"], c["eps"], c["clip"])
            assert rc != 0, change
            assert b"b200gym_rollout_mlp_noisy" in env._lib.b200gym_last_error(env._handle)
        if "per_env" in change:
            continue
        rc = env._lib.b200gym_rollout_actor_critic_norm(
            env._handle, vp(pa.data_ptr()), vp(pc.data_ptr()), 1, c["h1"], 0, 3, ok, ok, ok, ok, ok, ok, ok, ok, ok,
            ok, 0.99, 0.9, ok, ok, env._stream(), c["act"], c["mean"], c["var"], c["eps"], c["clip"], c["rvar"],
            c["clip_r"])
        assert rc != 0, change
        assert b"b200gym_rollout_actor_critic_norm" in env._lib.b200gym_last_error(env._handle)
    _assert_untouched(env, before, "C-side refusals")
    env.close()
