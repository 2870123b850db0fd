"""``B200VectorEnv.rollout_actor_critic(actor, critic, hidden, noise, gamma=, gae_lambda=)`` on the GPU, against an
eager twin: the noisy actor's loop of test_gpu_rollout_mlp_noisy.py (the MLP restated in torch elementwise ops, ReLU or
``torch.tanh``), the critic restated the same way with one output, on every input observation, on the last one and on
``infos["final_observation"]`` where a step truncated without terminating, and the GAE recursion restated in torch
float32 with ``torch.where``.  Every output is compared bit for bit (float32 as int32 views), and the env afterwards:
``get_state()``, ``snapshot()`` and the step after.
"""
import pytest

from test_gpu_rollout_linear import BOX2D, CLASSIC, NAMES, _assert_same_env, _assert_untouched, _eq, _untouched
from test_gpu_rollout_mlp_noisy import _K, _argmax_first, _noise

pytestmark = pytest.mark.gpu

HIDDEN = [(1,), (64,), (3, 7), (64, 64)]
ACTS = ["relu", "tanh"]


def _torch():
    import torch
    return torch


def mlp(params, hidden, x, K, activation):
    """The documented MLP in torch elementwise ops: each unit its bias plus one rounded product at a time, in order;
    ReLU (``z if z > 0 or z is NaN else +0.0``) or ``torch.tanh`` after every hidden layer.  params (P,), x (n, D)."""
    torch = _torch()
    n, D = x.shape
    sizes = [D] + list(hidden) + [K]
    off = 0
    for layer, (fan_in, fan_out) in enumerate(zip(sizes[:-1], sizes[1:])):
        w = params[off:off + fan_out * fan_in].reshape(fan_out, fan_in)
        off += fan_out * fan_in
        z = params[off:off + fan_out].expand(n, fan_out).clone()
        off += fan_out
        for k in range(fan_in):
            z = z + w[None, :, k] * x[:, None, k]
        if layer < len(hidden):
            z = torch.tanh(z) if activation == "tanh" else torch.where((z > 0) | torch.isnan(z), z, torch.zeros_like(z))
        x = z
    assert off == params.numel()
    return x


def coefficients(gamma, gae_lambda):
    import numpy as np
    return float(np.float32(gamma)), float(np.float32(float(gamma) * float(gae_lambda)))


def gae_restated(g, gl, rew, te, tr, values, vf):
    """The documented recursion in torch float32, one rounded operation per op."""
    torch = _torch()
    T, n = rew.shape
    g = torch.tensor(g, dtype=torch.float32, device=rew.device)
    gl = torch.tensor(gl, dtype=torch.float32, device=rew.device)
    adv = torch.empty((T, n), dtype=torch.float32, device=rew.device)
    nxt = torch.zeros(n, dtype=torch.float32, device=rew.device)
    for t in reversed(range(T)):
        r = rew[t].float()
        d_term = r - values[t]
        d_trunc = (r + g * vf[t]) - values[t]
        d_cont = (r + g * values[t + 1]) - values[t]
        delta = torch.where(te[t], d_term, torch.where(tr[t], d_trunc, d_cont))
        nxt = torch.where(te[t] | tr[t], delta, delta + gl * nxt)
        adv[t] = nxt
    return adv


class AcTwin:
    """An env stepped eagerly with the restated actor, noise and critic."""

    def __init__(self, env, obs, activation):
        self.env, self.obs, self.activation = env, obs.clone(), activation
        self.K = _K(env)

    def actor(self, actor, hidden, e):
        z = mlp(actor, hidden, self.obs, self.K, self.activation)
        y = z + e
        return z, (_argmax_first(y) if self.env.discrete else y)

    def value(self, critic, hidden, x):
        return mlp(critic, hidden, x, 1, self.activation)[:, 0]

    def loop(self, actor, critic, hidden, noise, gamma, gae_lambda):
        """-> (actions, outputs, values, advantages, [obs, reward, term, trunc], final obs, masks), stacked."""
        torch = _torch()
        acts, zs, vals, vfs, outs, fin, masks = [], [], [], [], [], [], []
        for t in range(noise.shape[0]):
            vals.append(self.value(critic, hidden, self.obs))
            z, a = self.actor(actor, hidden, noise[t])
            o = self.env.step(a)
            self.obs = o[0].clone()
            acts.append(a)
            zs.append(z)
            outs.append([x.clone() for x in o[:4]])
            fin.append(o[4]["final_observation"].clone())
            masks.append(o[4]["_final_observation"].clone())
            vfs.append(self.value(critic, hidden, fin[-1]))
        vals.append(self.value(critic, hidden, self.obs))
        values = torch.stack(vals)
        o4 = [torch.stack([o[k] for o in outs]) for k in range(4)]
        adv = gae_restated(*coefficients(gamma, gae_lambda), o4[1], o4[2], o4[3], values, torch.stack(vfs))
        return torch.stack(acts), torch.stack(zs), values, adv, o4, torch.stack(fin), torch.stack(masks)


def _assert_equals(got, want, what=""):
    acts, outputs, values, adv, obs, rew, term, trunc, infos = got
    wa, wz, wv, wadv, (wo, wr, wte, wtr), wfin, wmask = want
    _eq(acts, wa, f"{what}actions")
    _eq(outputs, wz, f"{what}outputs")
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
    return envs[0], AcTwin(envs[1], obs[1], activation)


def _nets(env, hidden, seed, scale=0.5):
    torch = _torch()
    g = torch.Generator(device="cpu").manual_seed(seed)
    out = []
    for K in (_K(env), 1):
        sizes = [env.obs_dim] + list(hidden) + [K]
        P = sum(o * i + o for i, o in zip(sizes[:-1], sizes[1:]))
        out.append((scale * torch.randn(P, generator=g)).to(env.device))
    return out


def _twin_check(env_id, n, T, hidden, activation="relu", seed=3, gamma=0.99, gae_lambda=0.95, **kwargs):
    a, b = _pair(env_id, n, activation, seed=seed, **kwargs)
    pa, pc = _nets(a, hidden, seed + T)
    e = _noise(a, T, seed + 1)
    kw = dict(gamma=gamma, gae_lambda=gae_lambda, activation=activation)
    got = a.rollout_actor_critic(pa, pc, hidden, e, **kw)
    _assert_equals(got, b.loop(pa, pc, hidden, e, gamma, gae_lambda))
    _eq(a.snapshot().obs, got[4][-1], "snapshot().obs vs obs[T-1]")
    _assert_same_env(a, b.env)
    # continuity: the next call starts where this one ended, and its values[0] is this call's values[T]
    e2 = _noise(a, 2, seed + 2)
    nxt = a.rollout_actor_critic(pa, pc, hidden, e2, **kw)
    _assert_equals(nxt, b.loop(pa, pc, hidden, e2, gamma, gae_lambda), "next call ")
    _eq(nxt[2][0], got[2][-1], "next call's values[0] vs values[T]")
    _assert_same_env(a, b.env)
    act = b.actor(pa, hidden, _noise(a, 1, seed + 3)[0])[1]
    for name, x, y in zip(NAMES, a.step(act)[:4], b.env.step(act)[:4]):
        _eq(x, y, f"next step {name}")
    a.close()
    b.env.close()
    return got


# ---------------------------------------------------------------------------------------------- the eager twin
@pytest.mark.parametrize("activation", ACTS)
@pytest.mark.parametrize("n,T", [(1, 1), (257, 37), (33 * 256 + 5, 37), (4099, 300)])
@pytest.mark.parametrize("hidden", HIDDEN, ids=str)
@pytest.mark.parametrize("env_id", CLASSIC)
def test_rollout_actor_critic_equals_eager_loop(env_id, hidden, n, T, activation):
    got = _twin_check(env_id, n, T, hidden, activation)
    torch = _torch()
    assert got[2].dtype == torch.float32 and tuple(got[2].shape) == (T + 1, n)
    assert got[3].dtype == torch.float32 and tuple(got[3].shape) == (T, n)


@pytest.mark.parametrize("gamma,gae_lambda", [(0.99, 0.95), (0.0, 0.5), (0.9, 0.0), (1.0, 1.0)])
@pytest.mark.parametrize("env_id", CLASSIC)
def test_truncations_bootstrap_from_the_final_observation(env_id, gamma, gae_lambda):
    """max_episode_steps=5: truncations without termination happen inside the call, and their bootstrap is the critic
    of the final observation."""
    got = _twin_check(env_id, 4099, 23, (16, 8), "tanh", gamma=gamma, gae_lambda=gae_lambda, max_episode_steps=5)
    te, tr = got[6], got[7]
    assert bool((tr & ~te).any())


def test_termination_on_the_time_limit():
    """CartPole pushed one way only (-0.0 noise, an actor that always picks action 0) terminates after 8 to 10 steps;
    with max_episode_steps=9 some envs terminate on the step that also truncates, which bootstraps nothing."""
    torch = _torch()
    n, T, hidden = 1000, 40, (1,)
    a, b = _pair("CartPole-v1", n, max_episode_steps=9)
    pa = torch.zeros(4 + 1 + 2 + 2, device="cuda:0")
    pa[-2] = 1.0
    pc = _nets(a, hidden, 4)[1]
    e = torch.full((T, n, 2), -0.0, device="cuda:0")
    got = a.rollout_actor_critic(pa, pc, hidden, e, gamma=0.99, gae_lambda=0.95)
    _assert_equals(got, b.loop(pa, pc, hidden, e, 0.99, 0.95))
    te, tr = got[6], got[7]
    assert bool((te & tr).any()) and bool((tr & ~te).any()) and bool((te & ~tr).any())


def test_offsets_past_two_to_the_31():
    """CartPole, n = 2^20, T = 520: values and advantages pass 2^31 bytes (2.2 GB each), compared slice by slice with
    the eager loop."""
    torch = _torch()
    n, T, hidden = 1 << 20, 520, (8, 8)
    assert T * n * 4 > 1 << 31
    a, b = _pair("CartPole-v1", n, seed=5)
    pa, pc = _nets(a, hidden, 5, scale=0.3)
    e = _noise(a, T, 5)
    acts, outputs, values, adv, obs, rew, term, trunc, infos = a.rollout_actor_critic(pa, pc, hidden, e, gamma=0.99,
                                                                                      gae_lambda=0.95)
    fin, mask = infos["final_observation"], infos["_final_observation"]
    vfs = torch.empty((T, n), device="cuda:0")
    for t in range(T):
        _eq(values[t], b.value(pc, hidden, b.obs), f"values[{t}]")
        z, act = b.actor(pa, hidden, e[t])
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
        vfs[t] = b.value(pc, hidden, inf["final_observation"])
    _eq(values[T], b.value(pc, hidden, b.obs), "values[T]")
    want = gae_restated(*coefficients(0.99, 0.95), rew, term, trunc, values, vfs)
    for t in range(T):
        _eq(adv[t], want[t], f"advantages[{t}]")
    _assert_same_env(a, b.env)
    del acts, outputs, values, adv, obs, rew, term, trunc, infos, fin, mask, e, vfs, want
    a.close()
    b.env.close()
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ CUDA graphs
@pytest.mark.parametrize("env_id", ["CartPole-v1", "Pendulum-v1", "Acrobot-v1"])
def test_captured_replays_equal_eager_calls(env_id):
    """One graph draws the noise and runs rollout_actor_critic; replay k equals eager call k of the twin, with the
    actor and the critic rewritten in place between replays, and gamma / gae_lambda those of the capture."""
    torch = _torch()
    n, T, k, hidden = 515, 24, 3, (16, 12)
    a, b = _pair(env_id, n, "tanh")
    pa, pc = _nets(a, hidden, 2)
    e = _noise(a, T, 2)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        if a.discrete:
            u = torch.rand(e.shape, device=e.device).clamp_(min=torch.finfo(torch.float32).tiny)
            e.copy_(-torch.log(-torch.log(u)))
        else:
            e.copy_(0.3 * torch.randn(e.shape, device=e.device))
        out = a.rollout_actor_critic(pa, pc, hidden, e, gamma=0.98, gae_lambda=0.9, activation="tanh")
    prev = None
    for r in range(k):
        qa, qc = _nets(a, hidden, 100 + r)
        pa.copy_(qa)
        pc.copy_(qc)
        g.replay()
        e_now = e.clone()
        _assert_equals(out, b.loop(qa, qc, hidden, e_now, 0.98, 0.9), f"replay {r} ")
        if prev is not None:
            assert not torch.equal(e_now, prev), "each replay draws new noise"
        prev = e_now
    _assert_same_env(a, b.env)


# ---------------------------------------------------------------------------------------------------- Box2D
@pytest.mark.parametrize("hidden", [(5,), (64, 64)], ids=str)
@pytest.mark.parametrize("env_id,kwargs", [BOX2D[0], BOX2D[1], BOX2D[2]], ids=[b[0] for b in BOX2D[:3]])
def test_box2d_equals_eager_loop(env_id, kwargs, hidden):
    _twin_check(env_id, 67, 5, hidden, "tanh", seed=7, **kwargs)


@pytest.mark.parametrize("env_id", ["LunarLander-v2", "BipedalWalker-v3"])
def test_box2d_truncations_bootstrap(env_id):
    got = _twin_check(env_id, 33, 7, (8,), seed=9, max_episode_steps=3)
    assert bool((got[7] & ~got[6]).any())


@pytest.mark.parametrize("env_id,kwargs", BOX2D[:2], ids=[b[0] for b in BOX2D[:2]])
def test_box2d_capture_is_refused(env_id, kwargs):
    from gym_b200 import error
    torch = _torch()
    a, b = _pair(env_id, 33, seed=7, **kwargs)
    pa, pc = _nets(a, (8,), 3)
    e = _noise(a, 2, 3)
    before = _untouched(a)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with pytest.raises(error.Error, match="double|alternate|stale"):
        with torch.cuda.graph(g):
            a.rollout_actor_critic(pa, pc, (8,), e, gamma=0.99, gae_lambda=0.95)
    del g
    _assert_untouched(a, before, "capture")
    _assert_equals(a.rollout_actor_critic(pa, pc, (8,), e, gamma=0.99, gae_lambda=0.95),
                   b.loop(pa, pc, (8,), e, 0.99, 0.95), "after the refused capture ")


# ------------------------------------------------------------------------------------------ refusals and guards
def test_refusals_leave_the_env_untouched():
    import numpy as np

    import gym_b200
    from gym_b200 import error, wrappers
    from gym_b200.distributed import ShardedVectorEnv
    from gym_b200.env import B200Env
    torch = _torch()

    env = gym_b200.vector.make("CartPole-v1", 64)
    pa, pc = _nets(env, (8, 4), 0)
    e = torch.zeros(3, 64, 2, device="cuda:0")
    kw = dict(gamma=0.99, gae_lambda=0.95)
    with pytest.raises(error.ResetNeeded):
        env.rollout_actor_critic(pa, pc, (8, 4), e, **kw)
    env.reset(seed=1)
    before = _untouched(env)
    bad_args = [
        (pa.expand(64, -1).contiguous(), pc, (8, 4), e, kw),                       # per-env actor rows
        (pa, pc.expand(64, -1).contiguous(), (8, 4), e, kw),                       # per-env critic rows
        (pa, pc[:-1], (8, 4), e, kw), (pa, torch.cat([pc, pc[:1]]), (8, 4), e, kw),  # the wrong critic length
        (pa, pc.double(), (8, 4), e, kw), (pa, pc.cpu(), (8, 4), e, kw), (pa, pc.tolist(), (8, 4), e, kw),
        (pa[:-1], pc, (8, 4), e, kw), (pa, pc, (8,), e, kw), (pa, pc, (8, 4), e[:, :63], kw),
        (pa, pc, (8, 4), e, dict(kw, activation="Tanh")),
    ]
    for name in ("gamma", "gae_lambda"):
        for x in (float("nan"), float("inf"), -0.01, 1.01, -1, 2, True, False, np.bool_(True), None, "0.9",
                  torch.tensor(0.9), 1j):
            bad_args.append((pa, pc, (8, 4), e, dict(kw, **{name: x})))
    for k, (x, c, h, y, kk) in enumerate(bad_args):
        with pytest.raises(ValueError):
            env.rollout_actor_critic(x, c, h, y, **kk)
        _assert_untouched(env, before, f"bad arguments {k}")
    with pytest.raises(TypeError):
        env.rollout_actor_critic(pa, pc, (8, 4), e)                                # gamma, gae_lambda required
    env.step_async(torch.zeros(64, dtype=torch.int64, device="cuda:0"))
    with pytest.raises(error.AlreadyPendingCallError):
        env.rollout_actor_critic(pa, pc, (8, 4), e, **kw)
    env.step_wait()
    before = _untouched(env)
    for wr in (wrappers.RecordEpisodeStatistics(env), wrappers.NormalizeObservation(env),
               wrappers.NormalizeReward(env), wrappers.VectorListInfo(env)):
        with pytest.raises(error.Error, match="rollout_actor_critic"):
            wr.rollout_actor_critic(pa, pc, (8, 4), e, **kw)
    _assert_untouched(env, before, "wrappers")
    env.close()

    no_reset = gym_b200.vector.make("CartPole-v1", 64, autoreset=False)
    no_reset.reset(seed=2)
    before = _untouched(no_reset)
    with pytest.raises(error.Error, match="autoreset"):
        no_reset.rollout_actor_critic(pa, pc, (8, 4), e, **kw)
    _assert_untouched(no_reset, before, "autoreset=False")
    no_reset.close()

    host = gym_b200.vector.make("CartPole-v1", 16, backend="numpy")
    host.reset(seed=3)
    rows = host.snapshot().rows.clone()
    with pytest.raises(error.Error, match="backend"):
        host.rollout_actor_critic(pa, pc, (8, 4), e[:, :16].contiguous(), **kw)
    assert torch.equal(host.snapshot().rows, rows)
    host.close()

    from gym_b200 import subenv
    chain = gym_b200.vector.make("CartPole-v1", 16, wrappers=[subenv.RecordEpisodeStatistics()])
    chain.reset(seed=4)
    before = _untouched(chain)
    with pytest.raises(error.Error, match="wrappers"):
        chain.rollout_actor_critic(pa, pc, (8, 4), e[:, :16].contiguous(), **kw)
    _assert_untouched(chain, before, "per-env wrappers")
    chain.close()

    assert not hasattr(ShardedVectorEnv, "rollout_actor_critic")
    assert not hasattr(B200Env, "rollout_actor_critic")


def test_c_entry_point_validates_its_arguments():
    """The C entry point checks the activation, layer count, widths, T, the GAE coefficients and the buffers itself,
    final_obs_dev included, and launches nothing when they are wrong."""
    import ctypes

    import gym_b200
    torch = _torch()
    env = gym_b200.vector.make("CartPole-v1", 8)
    env.reset(seed=2)
    pa, pc = _nets(env, (4,), 0)
    buf = torch.zeros(64, 8, 4, device="cuda:0")
    before = _untouched(env)
    vp = ctypes.c_void_p
    ok = vp(buf.data_ptr())
    good = dict(layers=1, h1=4, h2=0, T=3, critic=ok, noise=ok, outputs=ok, actions=ok, obs=ok, reward=ok, term=ok,
                trunc=ok, final=ok, values=ok, adv=ok, g=0.99, gl=0.9, last=ok, act=0)
    bad = [dict(layers=0), dict(layers=3, h2=4), dict(h1=0), dict(h1=65), dict(layers=2, h2=0), dict(layers=2, h2=65),
           dict(T=0), dict(T=-1), dict(act=2), dict(act=-1), dict(g=float("nan")), dict(g=1.5), dict(gl=-0.5),
           dict(critic=None), dict(noise=None), dict(outputs=None), dict(actions=None), dict(obs=None),
           dict(reward=None), dict(term=None), dict(trunc=None), dict(final=None), dict(values=None), dict(adv=None),
           dict(last=None)]
    for change in bad:
        c = {**good, **change}
        rc = env._lib.b200gym_rollout_actor_critic(
            env._handle, vp(pa.data_ptr()), c["critic"], c["layers"], c["h1"], c["h2"], c["T"], c["noise"],
            c["outputs"], c["actions"], c["obs"], c["reward"], c["term"], c["trunc"], c["final"], c["values"],
            c["adv"], c["g"], c["gl"], c["last"], ok, env._stream(), c["act"])
        assert rc != 0, change
        assert b"b200gym_rollout_actor_critic" in env._lib.b200gym_last_error(env._handle)
    _assert_untouched(env, before, "C-side refusals")
    env.close()
