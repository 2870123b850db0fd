"""``rollout_linear(..., obs_norm=, clip_obs=, obs_moments=)`` and ``rollout_mlp(...)`` with the same keywords on the
GPU, against an eager twin: the torch normalisation of the contract,
``((o.double() - mean) / torch.sqrt(var + eps)).float().clamp(-c, c)``, the policy restated in torch elementwise ops
(test_gpu_rollout_linear's logits, test_gpu_rollout_mlp's MLP with either activation, shared or per-env rows), then
``step()``.  Every output is compared bit for bit (float32 as int32 views), and the env afterwards.  Summary mode runs
on a third env reset alike: its returns, lengths and ended must be the fold of the full outputs, and ``obs_sum`` /
``obs_sumsq`` the masked sequential float64 fold of the raw inputs.
"""
import ctypes
import math

import pytest

from test_gpu_rollout_linear import BOX2D, CLASSIC, _assert_same_env, _assert_untouched, _eq, _untouched, summary_of
from test_gpu_rollout_mlp_noisy import _K, _argmax_first
from test_gpu_rollout_norm import normalize

pytestmark = pytest.mark.gpu

SHAPES = [(1, 1), (257, 37), (33 * 256 + 5, 37), (4099, 300)]
NETS = ["linear", "linear_per_env", "mlp64x64_tanh", "mlp16_relu_per_env"]


def _torch():
    import torch
    return torch


def linear_policy(w, b, discrete):
    def pol(x):
        n = x.shape[0]
        z = b.expand(n, b.shape[-1]).clone()
        for k in range(x.shape[1]):
            z = z + w[..., k] * x[:, None, k]
        return _argmax_first(z) if discrete else z
    return pol


def mlp_policy(params, hidden, K, activation, discrete):
    """The documented MLP in torch elementwise ops, params (P,) or (n, P) (row i for env i)."""
    torch = _torch()

    def pol(x):
        n, D = x.shape
        W = params.expand(n, params.shape[-1])
        sizes = [D] + list(hidden) + [K]
        off = 0
        for layer, (fan_in, fan_out) in enumerate(zip(sizes[:-1], sizes[1:])):
            w = W[:, off:off + fan_out * fan_in].reshape(n, fan_out, fan_in)
            off += fan_out * fan_in
            z = W[:, off:off + fan_out].clone()
            off += fan_out
            for k in range(fan_in):
                z = z + w[:, :, k] * x[:, None, k]
            if layer < len(hidden):
                z = torch.tanh(z) if activation == "tanh" else torch.where((z > 0) | torch.isnan(z), z,
                                                                            torch.zeros_like(z))
            x = z
        assert off == W.shape[1]
        return _argmax_first(x) if discrete else x
    return pol


class Twin:
    """An env stepped eagerly, the policy reading the torch normalisation of the observation it last returned."""

    def __init__(self, env, obs):
        self.env, self.obs = env, obs.clone()

    def loop(self, pol, T, norm):
        """-> (actions, [obs, reward, term, trunc], final obs, masks, raw inputs), stacked."""
        torch = _torch()
        acts, outs, fin, masks, inputs = [], [], [], [], []
        for _ in range(T):
            inputs.append(self.obs)
            x = self.obs if norm is None else normalize(self.obs, norm["mean"], norm["var"], norm["eps"], norm["clip"])
            a = pol(x)
            o = self.env.step(a)
            self.obs = o[0].clone()
            acts.append(a)
            outs.append([v.clone() for v in o[:4]])
            fin.append(o[4]["final_observation"].clone())
            masks.append(o[4]["_final_observation"].clone())
        return (torch.stack(acts), [torch.stack([o[k] for o in outs]) for k in range(4)], torch.stack(fin),
                torch.stack(masks), torch.stack(inputs))


def moments_of(inputs, lengths):
    """The masked sequential fold: s = +0.0; s = s + o[t] where t < lengths; q likewise with o[t] * o[t]."""
    torch = _torch()
    o = inputs.double()
    s = torch.zeros(o.shape[1:], dtype=torch.float64, device=o.device)
    q = torch.zeros_like(s)
    for t in range(o.shape[0]):
        keep = (t < lengths)[:, None]
        s = torch.where(keep, s + o[t], s)
        q = torch.where(keep, q + o[t] * o[t], q)
    return s, q


def _envs(env_id, n, seed, count=3, **kwargs):
    import gym_b200
    envs = [gym_b200.vector.make(env_id, n, **kwargs) for _ in range(count)]
    obs = [e.reset(seed=seed)[0] for e in envs]
    return envs, obs


def _stats(env, seed, clip=1.5, eps=1e-8):
    torch = _torch()
    g = torch.Generator(device="cpu").manual_seed(seed)
    D = env.obs_dim
    mean = (0.3 * torch.randn(D, generator=g, dtype=torch.float64)).to(env.device)
    var = (2.0 * torch.rand(D, generator=g, dtype=torch.float64) + 0.01).to(env.device)
    return dict(mean=mean, var=var, eps=eps, clip=clip)


def _kw(norm):
    return {} if norm is None else dict(obs_norm=(norm["mean"], norm["var"]), norm_epsilon=norm["eps"],
                                        clip_obs=norm["clip"])


def _net(env, name, seed):
    """-> (call(env, T, **kw), eager policy, the parameter tensors the call reads) for one of NETS."""
    torch = _torch()
    g = torch.Generator(device="cpu").manual_seed(seed)
    K, D, n = _K(env), env.obs_dim, env.num_envs
    per_env = name.endswith("per_env")
    lead = (n,) if per_env else ()
    if name.startswith("linear"):
        w = torch.randn(lead + (K, D), generator=g).to(env.device)
        b = torch.randn(lead + (K,), generator=g).to(env.device)
        return (lambda e, T, **kw: e.rollout_linear(w, b, T, **kw)), linear_policy(w, b, env.discrete), (w, b)
    hidden = (64, 64) if "64x64" in name else (16,)
    act = "tanh" if name.endswith("tanh") else "relu"
    sizes = [D] + list(hidden) + [K]
    P = sum(o * i + o for i, o in zip(sizes[:-1], sizes[1:]))
    p = (0.5 * torch.randn(lead + (P,), generator=g)).to(env.device)
    return ((lambda e, T, **kw: e.rollout_mlp(p, hidden, T, activation=act, **kw)),
            mlp_policy(p, hidden, K, act, env.discrete), (p,))


def _check(env_id, n, T, net, norm_seed=5, clip=1.5, seed=3, **kwargs):
    """Full mode against the twin, summary mode with moments against the fold; with obs_norm unless norm_seed is
    None.  Returns the full outputs and the summary."""
    (a, b, c), (_, ob, _) = _envs(env_id, n, seed, **kwargs)
    call, pol, _ = _net(a, net, seed + T)
    norm = None if norm_seed is None else _stats(a, norm_seed, clip)
    got = call(a, T, **_kw(norm))
    wa, (wo, wr, wte, wtr), wfin, wmask, inputs = Twin(b, ob).loop(pol, T, norm)
    _eq(got[0], wa, "actions")
    for name, x, y in zip(("obs", "reward", "terminated", "truncated"), got[1:5], (wo, wr, wte, wtr)):
        _eq(x, y, name)
    _eq(got[5]["_final_observation"], wmask, "_final_observation")
    _eq(got[5]["final_observation"][wmask], wfin[wmask], "final_observation")
    _assert_same_env(a, b)
    summ = call(c, T, summary=True, obs_moments=True, **_kw(norm))
    ret, lengths, ended = summary_of(wr, wte, wtr)
    s, q = moments_of(inputs, lengths)
    for name, x, y in zip(("returns", "lengths", "ended", "obs_sum", "obs_sumsq"), summ, (ret, lengths, ended, s, q)):
        _eq(x, y, f"summary {name}")
    _assert_same_env(c, a, "summary ")
    for e in (a, b, c):
        e.close()
    return got, summ


# ---------------------------------------------------------------------------------------------- the eager twin
@pytest.mark.parametrize("n,T", SHAPES)
@pytest.mark.parametrize("net", NETS)
@pytest.mark.parametrize("env_id", CLASSIC)
def test_normalised_policy_rollouts_equal_eager_loop(env_id, net, n, T):
    if n * T > 1 << 20 and net.startswith("mlp"):
        T = 37                                                # the elementwise MLP twin is slow at 300 steps
    _check(env_id, n, T, net)


@pytest.mark.parametrize("net", ["linear_per_env", "mlp64x64_tanh"])
@pytest.mark.parametrize("env_id", CLASSIC)
def test_moments_without_obs_norm(env_id, net):
    """obs_moments alone: the policy reads the raw observations, the call still runs the moment-folding kernel."""
    _check(env_id, 4099, 40, net, norm_seed=None, max_episode_steps=17)


@pytest.mark.parametrize("env_id", CLASSIC)
def test_short_episodes_and_no_clip(env_id):
    """max_episode_steps=3: every env's first episode ends inside the call; clip_obs left out."""
    got, summ = _check(env_id, 515, 11, "linear_per_env", clip=None, max_episode_steps=3)
    assert bool(summ[2].all()) and int(summ[1].max()) <= 3


@pytest.mark.parametrize("net", ["linear_per_env", "mlp16_relu_per_env", "mlp64x64_tanh"])
@pytest.mark.parametrize("env_id,kwargs", BOX2D[:3], ids=[b[0] for b in BOX2D[:3]])
def test_box2d_equals_eager_loop(env_id, kwargs, net):
    _check(env_id, 67, 6, net, seed=7, clip=1.0, **kwargs)
    _check(env_id, 67, 9, net, norm_seed=None, seed=8, max_episode_steps=4, **kwargs)


# --------------------------------------------------------------------------------------------- unchanged paths
@pytest.mark.parametrize("net", NETS)
@pytest.mark.parametrize("env_id", CLASSIC + ["LunarLander-v2"])
def test_defaults_run_the_existing_entry_points(monkeypatch, env_id, net):
    """With the new entry points replaced by a stub that raises, calls with the keywords at their defaults still run
    and return what a twin env returns, full and summary."""
    from gym_b200 import _lib
    (a, b), (_, ob) = _envs(env_id, 300, 4, count=2, max_episode_steps=9)

    def stub(*args):
        raise AssertionError("a _norm entry point was called")
    lib = _lib.load()
    for name in ("b200gym_rollout_linear_norm", "b200gym_rollout_mlp_norm"):
        monkeypatch.setattr(lib, name, stub)
    call, pol, _ = _net(a, net, 1)
    twin = Twin(b, ob)
    got = call(a, 12)
    want = twin.loop(pol, 12, None)
    _eq(got[0], want[0], "actions")
    for x, y, name in zip(got[1:5], want[1], ("obs", "reward", "terminated", "truncated")):
        _eq(x, y, name)
    got = call(a, 5, summary=True)
    wr = twin.loop(pol, 5, None)[1]
    for x, y, name in zip(got, summary_of(*wr[1:]), ("returns", "lengths", "ended")):
        _eq(x, y, name)
    _assert_same_env(a, b)
    with pytest.raises(AssertionError, match="_norm entry point"):   # the stub is what the keywords reach
        call(a, 3, summary=True, obs_moments=True)
    monkeypatch.undo()
    a.close()
    b.close()


@pytest.mark.parametrize("net", ["linear", "mlp64x64_tanh"])
@pytest.mark.parametrize("env_id", CLASSIC)
def test_identity_statistics_give_the_calls_without_normalisation(env_id, net):
    """mean 0, var 1, eps 0, no clip: bit for bit the calls without the keywords, full and summary."""
    torch = _torch()
    (a, b), _ = _envs(env_id, 1000, 11, count=2, max_episode_steps=13)
    call = _net(a, net, 11)[0]
    D = a.obs_dim
    ident = (torch.zeros(D, dtype=torch.float64, device="cuda:0"), torch.ones(D, dtype=torch.float64, device="cuda:0"))
    got, want = call(a, 40, obs_norm=ident, norm_epsilon=0.0), call(b, 40)
    for k in range(5):
        _eq(got[k], want[k], f"output {k}")
    got, want = call(a, 20, summary=True, obs_norm=ident, norm_epsilon=0.0), call(b, 20, summary=True)
    for k in range(3):
        _eq(got[k], want[k], f"summary output {k}")
    _assert_same_env(a, b)


# ------------------------------------------------------------------------------------------------ CUDA graphs
@pytest.mark.parametrize("net", NETS)
@pytest.mark.parametrize("env_id", CLASSIC)
def test_captured_replays_read_the_current_statistics_and_parameters(env_id, net):
    """One graph per call: between replays the statistics and the parameters are rewritten in place with copy_, and
    replay k equals eager call k on a twin env with the values of replay k."""
    torch = _torch()
    n, T = 515, 16
    (a, b), _ = _envs(env_id, n, 2, count=2, max_episode_steps=40)
    call_a, _, params = _net(a, net, 2)
    norm = _stats(a, 2, clip=1.5)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = call_a(a, T, summary=True, obs_moments=True, **_kw(norm))
    for r in range(3):
        new = _stats(a, 100 + r)
        norm["mean"].copy_(new["mean"])
        norm["var"].copy_(new["var"])
        for p in params:
            p.copy_(p * 0.9 + 0.05 * r)
        g.replay()
        want = call_a(b, T, summary=True, obs_moments=True, obs_norm=(norm["mean"].clone(), norm["var"].clone()),
                      norm_epsilon=norm["eps"], clip_obs=norm["clip"])
        for k, name in enumerate(("returns", "lengths", "ended", "obs_sum", "obs_sumsq")):
            _eq(out[k], want[k], f"replay {r} {name}")
        _assert_same_env(a, b, f"replay {r} ")


@pytest.mark.parametrize("env_id,kwargs", BOX2D[:3], ids=[b[0] for b in BOX2D[:3]])
def test_box2d_capture_is_refused(env_id, kwargs):
    from gym_b200 import error
    torch = _torch()
    (a,), _ = _envs(env_id, 33, 7, count=1, **kwargs)
    norm = _stats(a, 3)
    before = _untouched(a)
    for net in ("linear_per_env", "mlp16_relu_per_env"):
        call = _net(a, net, 3)[0]
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with pytest.raises(error.Error, match="double|alternate|stale"):
            with torch.cuda.graph(g):
                call(a, 2, summary=True, obs_moments=True, **_kw(norm))
        del g
        _assert_untouched(a, before, "capture")
    a.close()


# ------------------------------------------------------------------------------------------ refusals and guards
def test_refusals_are_raised_before_any_cuda_call():
    import gym_b200
    torch = _torch()
    env = gym_b200.vector.make("CartPole-v1", 64)
    env.reset(seed=1)
    w, b = torch.zeros(2, 4, device="cuda:0"), torch.zeros(2, device="cuda:0")
    p = torch.zeros(4 * 8 + 8 + 2 * 8 + 2, device="cuda:0")
    m = torch.zeros(4, dtype=torch.float64, device="cuda:0")
    v = torch.ones(4, dtype=torch.float64, device="cuda:0")
    calls = {"linear": lambda **kw: env.rollout_linear(w, b, 3, **kw),
             "mlp": lambda **kw: env.rollout_mlp(p, (8,), 3, **kw)}
    bad_stats = [m.float(), m.cpu(), m[:3], torch.zeros(4, 2, dtype=torch.float64, device="cuda:0")[:, 0], None]
    cases = [dict(obs_norm=(x, v)) for x in bad_stats] + [dict(obs_norm=(m, x)) for x in bad_stats]
    cases += [dict(obs_norm=m), dict(obs_norm=(m, v), norm_epsilon=-1.0), dict(obs_norm=(m, v), norm_epsilon=math.nan),
              dict(obs_norm=(m, v), clip_obs=0.0), dict(obs_norm=(m, v), clip_obs=math.inf), dict(clip_obs=10.0),
              dict(obs_moments=True), dict(obs_moments=True, obs_norm=(m, v)), dict(summary=True, obs_moments=1),
              dict(summary=True, obs_moments="yes")]
    before = _untouched(env)
    for which, call in calls.items():
        for k, kw in enumerate(cases):
            with pytest.raises(ValueError):
                call(**kw)
            _assert_untouched(env, before, f"{which} bad arguments {k}: {kw}")
    # per-env rows with obs_norm are refused by the noisy and actor-critic rollouts, as before
    e = torch.zeros(3, 64, 2, device="cuda:0")
    with pytest.raises(ValueError, match="with obs_norm needs one policy shared by every env, not per-env rows"):
        env.rollout_mlp_noisy(p.expand(64, -1).contiguous(), (8,), e, obs_norm=(m, v))
    env.close()


def test_c_entry_points_validate_their_arguments():
    """The C entry points re-check the statistics, the moment buffers (both or neither, summary mode only) and the
    existing outputs, widths and T, and launch nothing when they are wrong."""
    import gym_b200
    torch = _torch()
    env = gym_b200.vector.make("CartPole-v1", 8)
    env.reset(seed=2)
    buf = torch.zeros(64, 8, 4, device="cuda:0")
    st = torch.ones(64, dtype=torch.float64, device="cuda:0")
    before = _untouched(env)
    vp = ctypes.c_void_p
    ok, s = vp(buf.data_ptr()), vp(st.data_ptr())
    inf = math.inf
    good = dict(mean=s, var=s, eps=1e-8, clip=inf, sum=s, sumsq=s, summary=True, T=3, h1=4, act=0)
    bad = [dict(mean=None), dict(var=None), dict(eps=-1.0), dict(eps=math.nan), dict(clip=0.0), dict(clip=math.nan),
           dict(mean=None, var=None, clip=10.0), dict(sum=None), dict(sumsq=None), dict(summary=False), dict(T=0),
           dict(h1=0), dict(act=2)]
    for change in bad:
        c = {**good, **change}
        outs = [None] * 6 + [ok, ok, ok] if c["summary"] else [ok] * 6 + [None] * 3
        tail = (c["mean"], c["var"], c["eps"], c["clip"], c["sum"], c["sumsq"])
        if "h1" not in change and "act" not in change:
            rc = env._lib.b200gym_rollout_linear_norm(env._handle, ok, ok, 0, c["T"], *outs, ok, ok, env._stream(),
                                                      *tail)
            assert rc != 0, change
            assert b"b200gym_rollout_linear_norm" in env._lib.b200gym_last_error(env._handle)
        rc = env._lib.b200gym_rollout_mlp_norm(env._handle, ok, 0, 1, c["h1"], 0, c["T"], *outs, ok, ok,
                                               env._stream(), c["act"], *tail)
        assert rc != 0, change
        assert b"b200gym_rollout_mlp_norm" in env._lib.b200gym_last_error(env._handle)
    _assert_untouched(env, before, "C-side refusals")
    env.close()
