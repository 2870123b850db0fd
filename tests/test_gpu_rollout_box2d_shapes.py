"""The Box2D rollouts at the shapes their benchmarks time (scripts/rollout*_bench.py): 2^16 LunarLander(-Continuous)
envs and 2^14 BipedalWalker envs with T = 8, 2^16 + 77 hardcore walkers with T = 16, and rollout_from(_mlp) with
2^4 rows x 2^10 branches.  For the Box2D kinds every rollout is composed launch by launch (DESIGN.md §4.12): per step
a policy launch (which in summary mode also folds the step before), the step sequence of test_gpu_box2d_launch_shapes.py
(step kernel -> TOI kernel over the parked envs -> compacted reset-list kernel) and the caller's hooks (the critic on
the final observations, the normalised input rows, the observation moments); then the GAE.  rollout_from(_mlp) step a
scratch batch the env creates on first use and grows when B grows.

At these sizes, after bench.py's 250 warm-up steps of random play, episodes end naturally inside a call, so the
first-episode folds (summary, obs_moments, rollout_from) and the GAE meet terminations, not only time limits; the TOI
warps carry several parked envs and go round twice; and whole-batch truncations and forced falls queue more resets
than the reset-list kernel has threads.

Every case warms one engine up, copies its state into the other three DEVICE_CONFIGS settings and an eager twin with
snapshot() / restore(), and then runs a sequence of rollouts.  Every output of every call is bit for bit the same in
the four settings and equals the twin, which computes the policy with the torch restatements of the other rollout
tests and steps with step().  Three windows of the batch (the first, the middle and the last envs) are stepped by the
CPU oracle with the actions of the rollout and checked bit for bit.  The twin reads box2d_list_counts() after every
step; each case asserts the branches its docstring names and prints the counts (pytest -rP).  The advantages are also
checked against a float64 recursion written from the definition, within a rounding bound.
"""
import concurrent.futures

import numpy as np
import pytest

from test_gpu_box2d_launch_shapes import (DEVICE_CONFIGS, FALL_VY, RESET_CTAS_PER_SM, RESET_THREADS, TOI_CTAS_PER_SM,
                                          WARMUP, _bits, _Engine, _force_falls, _lanes, _make_oracle,
                                          _random_actions, _sms, _Windows)
from test_gpu_rollout_actor_critic import mlp
from test_gpu_rollout_from import _fold
from test_gpu_rollout_from_mlp import _noise as _branch_noise
from test_gpu_rollout_linear import summary_of
from test_gpu_rollout_mlp_head import HeadTwin
from test_gpu_rollout_mlp_noisy import _K, _noise
from test_gpu_rollout_norm import NormTwin, normalize
from test_gpu_rollout_policy_norm import Twin as PolicyTwin
from test_gpu_rollout_policy_norm import linear_policy, mlp_policy, moments_of

pytestmark = pytest.mark.gpu

WIND = dict(enable_wind=True, wind_idx=11, torque_idx=-7)
U32 = 2.0 ** -24          # unit roundoff of float32


def _torch():
    import torch
    return torch


class _Counting:
    """The twin's env as the restatements see it: every step() also reads box2d_list_counts() (parked, resets)."""

    def __init__(self, env):
        self._env, self.counts = env, []

    def __getattr__(self, name):
        return getattr(self._env, name)

    def step(self, actions):
        out = self._env.step(actions)
        parked, resets = self._env.box2d_list_counts()
        self.counts.append((int(parked[0]), int(resets[0])))
        return out


def _flat(out):
    """A rollout's outputs as (name, tensor) pairs: the final observations under their mask, snapshots as rows and
    observations."""
    torch = _torch()
    items = []
    for k, x in enumerate(out):
        if isinstance(x, torch.Tensor):
            items.append((f"output {k}", x))
        elif hasattr(x, "rows"):
            items += [(f"output {k} rows", x.rows), (f"output {k} obs", x.obs)]
        else:
            m = x["_final_observation"]
            items += [("_final_observation", m), ("final_observation", x["final_observation"][m])]
    return items


def _assert_outputs(ref, got, what):
    torch = _torch()
    a, b = _flat(ref), _flat(got)
    assert [n for n, _ in a] == [n for n, _ in b], what
    for (name, x), (_, y) in zip(a, b):
        assert x.dtype == y.dtype and x.shape == y.shape, (what, name, x.dtype, y.dtype, x.shape, y.shape)
        if not torch.equal(_bits(x), _bits(y)):
            bad = (_bits(x) != _bits(y)).nonzero()
            raise AssertionError(f"{what}: {name}: {len(bad)} entries differ, first at {bad[0].tolist()}")


def _first_terminations(te, tr, lengths, ended):
    """how many envs' first episode in the call ended by termination (the step a summary fold stops at)"""
    torch = _torch()
    t_end = (lengths.long() - 1).clamp(min=0)
    return int((ended & te.gather(0, t_end[None])[0]).sum())


def _eager_steps(env, acts):
    """env.step(a) for each a of acts -> (obs, reward, terminated, truncated, final observations, masks), stacked"""
    torch = _torch()
    outs, fin, masks = [], [], []
    for a in acts:
        o = env.step(a)
        outs.append([x.clone() for x in o[:4]])
        fin.append(o[4]["final_observation"].clone())
        masks.append(o[4]["_final_observation"].clone())
    return tuple(torch.stack([x[k] for x in outs]) for k in range(4)) + (torch.stack(fin), torch.stack(masks))


def gae_float64(rew, te, tr, values, vf, gamma, gae_lambda):
    """CleanRL's GAE recursion with Stable-Baselines3's bootstrap of a truncation (the reward plus gamma times the
    value of the final observation), in float64 from the definition, with exact gamma and lambda -> (advantages, bound).
    bound[t] is 4 u times the magnitudes that go into adv[t] (rewards, values, bootstraps, advantages, down the
    discounted chain), u = 2^-24: the float32 recursion rounds each of them at most about three times."""
    torch = _torch()
    T, n = rew.shape
    v = values.double()
    zero = torch.zeros(n, dtype=torch.float64, device=rew.device)
    adv = torch.zeros(T, n, dtype=torch.float64, device=rew.device)
    mag = torch.zeros_like(adv)
    nxt, nmag = zero, zero
    for t in reversed(range(T)):
        nonterminal = 1.0 - (te[t] | tr[t]).double()
        # the final observation is only defined where the step ended: select, do not multiply by 0
        boot = torch.where(tr[t] & ~te[t], gamma * vf[t].double(), zero)
        delta = rew[t] + boot + gamma * v[t + 1] * nonterminal - v[t]
        nxt = delta + gamma * gae_lambda * nonterminal * nxt
        nmag = (rew[t].abs() + boot.abs() + gamma * v[t + 1].abs() * nonterminal + v[t].abs() + nxt.abs()
                + gamma * gae_lambda * nonterminal * nmag)
        adv[t], mag[t] = nxt, nmag
    return adv, 4 * U32 * mag


class _Batch:
    """A warmed batch: the four DEVICE_CONFIGS engines, an eager twin with the default configuration, and three oracle
    windows of m envs, all in lockstep from reset(seed) + `warmup` steps of bench.py's cycled random pool (played on the
    first engine and the oracles, copied into the other engines with snapshot() / restore()).  The oracles run on a
    thread of their own, one queued job after another; finish() waits for them."""

    def __init__(self, env_id, n, m, seed=0, oracle=None, warmup=WARMUP, **kw):
        torch = _torch()
        self.dev = torch.device("cuda", 0)
        self.env_id, self.n, self.kw = env_id, n, kw
        self.engines = [_Engine(name, env_id, n, knobs, **kw) for name, knobs in DEVICE_CONFIGS]
        self.twin = _Engine("eager", env_id, n, {}, **kw)
        self.eager = _Counting(self.twin.env)
        self.windows = _Windows(oracle or _make_oracle(env_id, self.engines[0].env.max_episode_steps), n, m)
        self.thread = concurrent.futures.ThreadPoolExecutor(max_workers=1)
        self.jobs, self.counts, self.terms = [], {}, {}
        e0 = self.engines[0]
        obs = e0.call(e0.env.reset, seed=seed)[0].cpu().numpy()
        for lo, ro in zip(self.windows.los, self.windows.reset(seed)):
            assert np.array_equal(obs[lo:lo + m], ro), f"window {lo}: reset obs"
        rng = np.random.default_rng(1234)
        pool = [_random_actions(env_id, n, rng) for _ in range(8)]
        pool_dev = [torch.as_tensor(a, device=self.dev) for a in pool]

        def replay():
            refs = []
            for t in range(warmup):
                refs = self.windows.step(pool[t % len(pool)])
            return refs
        warm = self.thread.submit(replay)
        for t in range(warmup):
            e0.call(e0.env.step, pool_dev[t % len(pool)])
        snap = e0.env.snapshot()
        for e in self.engines[1:] + [self.twin]:
            e.call(e.env.restore, snap)
        self.obs = snap.obs.clone()     # what the envs last returned: the first input of the next call
        last = snap.obs.cpu().numpy()

        def check_warm():
            for lo, ref in zip(self.windows.los, warm.result()):
                assert np.array_equal(last[lo:lo + m], ref[0]), f"window {lo}: observations after the warm-up"
        self.jobs.append(self.thread.submit(check_warm))

    def sync(self):
        for j in self.jobs:
            j.result()
        self.jobs = []

    def oracle(self, what, acts, obs, rew, te, tr, masks, fin):
        """Queue the windows' T steps with `acts` and the check of the T steps of outputs."""
        host = [x.cpu().numpy() for x in (acts, obs, rew, te, tr, masks, fin)]

        def run():
            for t in range(host[0].shape[0]):
                refs = self.windows.step(host[0][t])
                self.windows.check(tuple(x[t] for x in host[1:]), refs, f"{what}, step {t}")
        self.jobs.append(self.thread.submit(run))

    def rollout(self, what, call, eager):
        """call(env) on every engine (its knobs set), the four bit for bit the same and equal to eager() on the twin,
        which returns (the outputs, the per-step tensors for the oracle).  -> the outputs."""
        outs = [e.call(call, e.env) for e in self.engines]
        for e, o in zip(self.engines[1:], outs[1:]):
            _assert_outputs(outs[0], o, f"{what}, {e.name}")
        start = len(self.eager.counts)
        want, steps = eager()
        _assert_outputs(outs[0], want, f"{what}, eager twin")
        self.counts[what] = self.eager.counts[start:]
        acts, o, r, te, tr, masks, fin = steps
        ret, lengths, ended = summary_of(r, te, tr)
        self.terms[what] = _first_terminations(te, tr, lengths, ended)
        self.oracle(what, *steps)
        return outs[0]

    # ------------------------------------------------------------------------------------------- the entry points
    def actions(self, what, acts):
        """rollout(acts)"""

        def eager():
            o, r, te, tr, fin, masks = _eager_steps(self.eager, acts)
            self.obs = o[-1].clone()
            infos = {"final_observation": fin, "_final_observation": masks}
            return (o, r, te, tr, infos), (acts, o, r, te, tr, masks, fin)
        return self.rollout(what, lambda env: env.rollout(acts), eager)

    def sampled(self, what, T, space_seed):
        """rollout_sampled(T) from action spaces seeded with space_seed"""
        torch = _torch()

        def call(env):
            env.action_space.seed(space_seed)
            return env.rollout_sampled(T)

        def eager():
            self.eager.action_space.seed(space_seed)
            acts, outs, fin, masks = [], [], [], []
            for _ in range(T):
                a = self.eager.sample_actions().clone()
                o = self.eager.step(a)
                acts.append(a)
                outs.append([x.clone() for x in o[:4]])
                fin.append(o[4]["final_observation"].clone())
                masks.append(o[4]["_final_observation"].clone())
            acts = torch.stack(acts)
            o, r, te, tr = (torch.stack([x[k] for x in outs]) for k in range(4))
            fin, masks = torch.stack(fin), torch.stack(masks)
            self.obs = o[-1].clone()
            infos = {"final_observation": fin, "_final_observation": masks}
            return (acts, o, r, te, tr, infos), (acts, o, r, te, tr, masks, fin)
        return self.rollout(what, call, eager)

    def policy(self, what, call, pol, T, summary=False, norm=None, moments=False):
        """rollout_linear / rollout_mlp: call(env) against test_gpu_rollout_policy_norm's Twin with policy `pol`"""

        def eager():
            tw = PolicyTwin(self.eager, self.obs)
            acts, (o, r, te, tr), fin, masks, inputs = tw.loop(pol, T, norm)
            self.obs = tw.obs
            steps = (acts, o, r, te, tr, masks, fin)
            if not summary:
                return (acts, o, r, te, tr, {"final_observation": fin, "_final_observation": masks}), steps
            ret, lengths, ended = summary_of(r, te, tr)
            return ((ret, lengths, ended) + (moments_of(inputs, lengths) if moments else ())), steps
        return self.rollout(what, call, eager)

    def head(self, what, call, params, hidden, activation, head, noise=None, T=None):
        """rollout_mlp / rollout_mlp_noisy with head=: against test_gpu_rollout_mlp_head's HeadTwin"""

        def eager():
            tw = HeadTwin(self.eager, self.obs, activation, head)
            if noise is None:
                acts, (o, r, te, tr), fin, masks = tw.loop(params, hidden, T)
                lead = (acts,)
            else:
                acts, zs, (o, r, te, tr), fin, masks = tw.noisy_loop(params, hidden, noise)
                lead = (acts, zs)
            self.obs = tw.obs
            infos = {"final_observation": fin, "_final_observation": masks}
            return lead + (o, r, te, tr, infos), (acts, o, r, te, tr, masks, fin)
        return self.rollout(what, call, eager)

    def noisy(self, what, call, actor, critic, hidden, noise, activation, norm=None, gamma=0.99, gae_lambda=0.95):
        """rollout_mlp_noisy (critic None) / rollout_actor_critic: against test_gpu_rollout_norm's NormTwin; the
        advantages also against gae_float64"""
        norm = norm or dict(mean=None)
        torch = _torch()

        def eager():
            tw = NormTwin(self.eager, self.obs, activation)
            acts, zs, values, adv, (o, r, te, tr), fin, masks = tw.loop(actor, critic, hidden, noise, norm, gamma,
                                                                        gae_lambda)
            self.obs = tw.obs
            infos = {"final_observation": fin, "_final_observation": masks}
            lead = (acts, zs) if critic is None else (acts, zs, values, adv)
            return lead + (o, r, te, tr, infos), (acts, o, r, te, tr, masks, fin)
        out = self.rollout(what, call, eager)
        if critic is not None:
            acts, zs, values, adv, o, r, te, tr, infos = out
            fin = infos["final_observation"]
            T, n, D = fin.shape
            x = fin.reshape(T * n, D)
            if norm["mean"] is not None:
                x = normalize(x, norm["mean"], norm["var"], norm["eps"], norm["clip"])
            vf = mlp(critic, hidden, x, 1, activation)[:, 0].reshape(T, n)
            if norm.get("rvar") is not None:
                c = float(np.float32(norm["clip_r"]))
                r = (r / torch.sqrt(norm["rvar"] + norm["eps"])).clamp(-c, c)
            want, bound = gae_float64(r, te, tr, values, vf, gamma, gae_lambda)
            err = (adv.double() - want).abs()
            worst = int((err - bound).flatten().argmax())
            assert bool((err <= bound).all()), (f"{what}: advantages off the float64 recursion by "
                                                f"{float(err.flatten()[worst]):.3g} at {divmod(worst, n)}, bound "
                                                f"{float(bound.flatten()[worst]):.3g}")
        return out

    def branches(self, what, call, snap, rows, loop, blocks=()):
        """rollout_from / rollout_from_mlp: call(env) on every engine, bit for bit the same and equal to the restored
        twin of their contract (a fresh env of B envs, default configuration, restored from snap's `rows`), stepped by
        loop(env, first observations) through _Counting, which returns (the outputs before the end states, the per-step
        tensors).  Branches [bo, bo + m) of `blocks` hold the rows of the windows' envs in order and are checked
        against the oracles."""
        import gym_b200
        from gym_b200.snapshot import EnvSnapshot
        torch = _torch()
        outs = [e.call(call, e.env) for e in self.engines]
        for e, o in zip(self.engines[1:], outs[1:]):
            _assert_outputs(outs[0], o, f"{what}, {e.name}")
        twin = gym_b200.vector.make(self.env_id, len(rows), **self.kw)
        try:
            twin.restore(EnvSnapshot(snap.header, snap.rows[rows], snap.obs[rows]))
            tw = _Counting(twin)
            lead, steps = loop(tw, snap.obs[rows])
            _assert_outputs(outs[0], lead + (twin.snapshot(),), f"{what}, restored twin")
        finally:
            twin.close()
        self.counts[what] = tw.counts
        acts, o, r, te, tr, masks, fin = steps
        self.terms[what] = _first_terminations(te, tr, *_fold(r, te, tr)[1:])
        if blocks:
            m = self.windows.m
            src = torch.cat([torch.arange(bo, bo + m) for bo in blocks]).to(self.dev)
            dst = torch.cat([torch.arange(lo, lo + m) for lo in self.windows.los]).to(self.dev)

            def spread(x):   # branch bo + k -> env lo + k of the windows
                y = torch.zeros((x.shape[0], self.n) + tuple(x.shape[2:]), dtype=x.dtype, device=x.device)
                y[:, dst] = x[:, src]
                return y
            self.oracle(what, *(spread(x) for x in steps))
        return outs[0]

    # ---------------------------------------------------------------------------------------------------- the end
    def finish(self, case):
        """Wait for the oracles, compare every engine's end state with the twin's, print the counts -> all the
        twin's per-step counts."""
        torch = _torch()
        try:
            self.sync()
            ref = self.twin.env.snapshot()
            for e in self.engines:
                s = e.env.snapshot()
                assert torch.equal(s.rows, ref.rows), f"{e.name}: end state"
                assert torch.equal(_bits(s.obs), _bits(ref.obs)), f"{e.name}: end observations"
        finally:
            self.close()
        return _report(case, self.n, self.counts, self.terms)

    def close(self):
        self.thread.shutdown(wait=True)
        for e in self.engines + [self.twin]:
            e.env.close()
        self.windows.close()


def _report(case, n, counts, terms):
    """Print the counts the docstrings quote -> every step's (parked, resets)."""
    sms = _sms()
    grid = min(n, TOI_CTAS_PER_SM * sms)
    steps = [c for v in counts.values() for c in v]
    p = max(c[0] for c in steps)
    r = max(c[1] for c in steps)
    print(f"{case}: {sms} SMs, TOI grid {grid}: largest parked {p} (L = {_lanes(p, grid)}), largest resets {r} "
          f"({RESET_CTAS_PER_SM * sms * RESET_THREADS} reset-list threads); first episodes ended by termination: "
          f"{terms}")
    return steps


def _grid(n):
    return min(n, TOI_CTAS_PER_SM * _sms())


def _reset_threads():
    return RESET_CTAS_PER_SM * _sms() * RESET_THREADS


def _mlp_params(env, hidden, K, seed, lead=(), scale=0.5):
    torch = _torch()
    sizes = [env.obs_dim] + list(hidden) + [K]
    P = sum(o * i + o for i, o in zip(sizes[:-1], sizes[1:]))
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (scale * torch.randn(tuple(lead) + (P,), generator=g)).to(env.device)


def _linear_params(env, seed, scale=0.5):
    torch = _torch()
    g = torch.Generator(device="cpu").manual_seed(seed)
    n, K, D = env.num_envs, _K(env), env.obs_dim
    w = (scale * torch.randn((n, K, D), generator=g)).to(env.device)
    b = (scale * torch.randn((n, K), generator=g)).to(env.device)
    return w, b


def _obs_stats(env, seed, clip=5.0, eps=1e-8):
    torch = _torch()
    g = torch.Generator(device="cpu").manual_seed(seed)
    D = env.obs_dim
    mean = (0.3 * torch.randn(D, generator=g, dtype=torch.float64)).to(env.device)
    var = (2.0 * torch.rand(D, generator=g, dtype=torch.float64) + 0.01).to(env.device)
    rvar = (5.0 * torch.rand(1, generator=g, dtype=torch.float64) + 0.1).to(env.device)
    return dict(mean=mean, var=var, eps=eps, clip=clip, rvar=rvar, clip_r=3.0)


def _norm_kw(norm, rewards=False):
    kw = dict(obs_norm=(norm["mean"], norm["var"]), norm_epsilon=norm["eps"], clip_obs=norm["clip"])
    if rewards:
        kw.update(reward_norm=norm["rvar"], clip_reward=norm["clip_r"])
    return kw


def _assert_multi_lane(n, steps):
    assert max(c[0] for c in steps) > _grid(n), "a step that parks more envs than the TOI grid has warps"


def _assert_second_round(n, steps):
    assert max(c[0] for c in steps) > 32 * _grid(n), "a step that parks more than 32 envs per TOI warp"


# --------------------------------------------------------------------------------------------------------- the cases
def test_bench_lunar():
    """LunarLander-v2 as the rollout benchmarks time it: 2^16 envs, T = 8, ten calls in a row after bench.py's warm-up.
    Episodes end by crash or rest inside the first episode of every call, so every fold meets terminations; the TOI
    warps carry several envs; several reset-list CTAs run.  On an H100 (132 SMs, TOI grid 1 584): up to 2 623 envs
    parked in a step (L = 2), up to 1 013 resets; 5 760 to 7 836 first episodes per call end by termination.  Random
    play never resets more envs in a step than the reset-list kernel has threads (33 792); the whole-batch truncation
    and the forced falls below do."""
    n, T, H = 1 << 16, 8, (64, 64)
    b = _Batch("LunarLander-v2", n, m=1024)
    try:
        env = b.twin.env
        rng = np.random.default_rng(7)
        acts = _torch().as_tensor(np.stack([_random_actions("LunarLander-v2", n, rng) for _ in range(T)]), device=b.dev)
        b.actions("rollout", acts)
        b.sampled("rollout_sampled", T, space_seed=5)
        w, bias = _linear_params(env, 1)
        pol = linear_policy(w, bias, True)
        b.policy("rollout_linear per-env", lambda e: e.rollout_linear(w, bias, T), pol, T)
        b.policy("rollout_linear per-env summary", lambda e: e.rollout_linear(w, bias, T, summary=True), pol, T,
                 summary=True)
        for act in ("relu", "tanh"):
            p = _mlp_params(env, H, 4, 2)
            pol = mlp_policy(p, H, 4, act, True)
            b.policy(f"rollout_mlp {act}", lambda e: e.rollout_mlp(p, H, T, activation=act), pol, T)
            b.policy(f"rollout_mlp {act} summary", lambda e: e.rollout_mlp(p, H, T, summary=True, activation=act),
                     pol, T, summary=True)
        p = _mlp_params(env, H, 4, 3)
        e = _noise(env, T, 4)
        b.noisy("rollout_mlp_noisy", lambda x: x.rollout_mlp_noisy(p, H, e), p, None, H, e, "relu")
        pa, pc = _mlp_params(env, H, 4, 5), _mlp_params(env, H, 1, 6)
        e = _noise(env, T, 7)
        b.noisy("rollout_actor_critic", lambda x: x.rollout_actor_critic(pa, pc, H, e, gamma=0.99, gae_lambda=0.95,
                                                                          activation="tanh"), pa, pc, H, e, "tanh")
    except BaseException:
        b.close()
        raise
    steps = b.finish("bench_lunar")
    _assert_multi_lane(n, steps)
    assert max(c[1] for c in steps) > RESET_THREADS, "a step with more resets than one reset-list CTA has threads"
    for what in ("rollout_linear per-env summary", "rollout_mlp relu summary", "rollout_mlp tanh summary",
                 "rollout_actor_critic"):
        assert b.terms[what] > 0, f"{what}: a first episode that ends by termination"


def test_continuous_wind_lunar():
    """LunarLanderContinuous-v2 with wind at 2^16 envs, T = 8: the normalised-input paths (norm_rows_kernel before
    every policy launch, obs_moments_kernel in summary mode), the TD3 and SAC heads, and PPO collection with
    normalised observations and rewards (the critic on normalised final observations, gae_scaled_kernel).  On an H100:
    up to 1 932 envs parked in a step (L = 2), up to 780 resets; 5 390 to 5 849 first episodes per call end by
    termination."""
    from oracle.oracle import OracleLunar
    n, T, H = 1 << 16, 8, (64, 64)
    b = _Batch("LunarLanderContinuous-v2", n, m=1024, oracle=lambda m: OracleLunar(
        m, max_episode_steps=1000, continuous=True, enable_wind=True, wind_idx=11, torque_idx=-7), **WIND)
    try:
        env = b.twin.env
        norm = _obs_stats(env, 1)
        kw = _norm_kw(norm)
        w, bias = _linear_params(env, 2)
        pol = linear_policy(w, bias, False)
        b.policy("rollout_linear per-env obs_norm", lambda e: e.rollout_linear(w, bias, T, **kw), pol, T, norm=norm)
        b.policy("rollout_linear per-env obs_norm obs_moments",
                 lambda e: e.rollout_linear(w, bias, T, summary=True, obs_moments=True, **kw), pol, T, summary=True,
                 norm=norm, moments=True)
        p = _mlp_params(env, H, 2, 3)
        pol = mlp_policy(p, H, 2, "tanh", False)
        b.policy("rollout_mlp tanh obs_norm", lambda e: e.rollout_mlp(p, H, T, activation="tanh", **kw), pol, T,
                 norm=norm)
        b.policy("rollout_mlp tanh obs_norm obs_moments",
                 lambda e: e.rollout_mlp(p, H, T, summary=True, activation="tanh", obs_moments=True, **kw), pol, T,
                 summary=True, norm=norm, moments=True)
        for head, K in (("tanh", 2), ("tanh_normal", 4)):
            p = _mlp_params(env, H, K, 4)
            e = _noise(env, T, 5, scale=0.1 if head == "tanh" else 1.0)
            b.head(f"rollout_mlp_noisy head={head}", lambda x: x.rollout_mlp_noisy(p, H, e, head=head), p, H, "relu",
                   head, noise=e)
        pa, pc = _mlp_params(env, H, 2, 6), _mlp_params(env, H, 1, 7)
        e = _noise(env, T, 8, scale=0.5)
        b.noisy("rollout_actor_critic obs_norm reward_norm", lambda x: x.rollout_actor_critic(
            pa, pc, H, e, gamma=0.99, gae_lambda=0.95, activation="tanh", **_norm_kw(norm, rewards=True)),
            pa, pc, H, e, "tanh", norm=norm)
    except BaseException:
        b.close()
        raise
    steps = b.finish("continuous_wind_lunar")
    _assert_multi_lane(n, steps)
    for what in ("rollout_linear per-env obs_norm obs_moments", "rollout_mlp tanh obs_norm obs_moments",
                 "rollout_actor_critic obs_norm reward_norm"):
        assert b.terms[what] > 0, f"{what}: a first episode that ends by termination"


def test_walker_sac():
    """BipedalWalker-v3 at 2^14 envs, T = 8, as rollout_mlp_head_bench.py times CleanRL's SAC actor: (64, 64) ReLU
    and the tanh_normal head, sampled and deterministic.  On an H100: up to 6 243 envs parked in a step (L = 4), up
    to 121 resets; about 850 first episodes per call end by termination (a fall)."""
    n, T, H = 1 << 14, 8, (64, 64)
    b = _Batch("BipedalWalker-v3", n, m=512)
    try:
        env = b.twin.env
        p = _mlp_params(env, H, 8, 1)
        e = _noise(env, T, 2)
        b.head("rollout_mlp_noisy head=tanh_normal", lambda x: x.rollout_mlp_noisy(p, H, e, head="tanh_normal"),
               p, H, "relu", "tanh_normal", noise=e)
        b.head("rollout_mlp head=tanh_normal", lambda x: x.rollout_mlp(p, H, T, head="tanh_normal"), p, H, "relu",
               "tanh_normal", T=T)
    except BaseException:
        b.close()
        raise
    steps = b.finish("walker_sac")
    _assert_multi_lane(n, steps)


def test_hardcore_ragged():
    """BipedalWalkerHardcore-v3 at 2^16 + 77 envs, T = 16: the step kernel's last CTA is partial and the TOI warps
    carry many envs.  On an H100: up to 26 495 envs parked in a step (L = 17), up to 510 resets; 6 326 and 6 359
    first episodes end by termination.  Random play after the warm-up does not park more than 32 envs per warp; the
    whole-batch truncation below does (the warps go round twice)."""
    n, T, H = (1 << 16) + 77, 16, (64, 64)
    b = _Batch("BipedalWalkerHardcore-v3", n, m=512)
    try:
        env = b.twin.env
        rng = np.random.default_rng(3)
        acts = _torch().as_tensor(np.stack([_random_actions("BipedalWalker", n, rng) for _ in range(T)]),
                                  device=b.dev)
        b.actions("rollout", acts)
        p = _mlp_params(env, H, 4, 4)
        b.policy("rollout_mlp relu", lambda e: e.rollout_mlp(p, H, T), mlp_policy(p, H, 4, "relu", False), T)
    except BaseException:
        b.close()
        raise
    steps = b.finish("hardcore_ragged")
    _assert_multi_lane(n, steps)


def test_walker_whole_batch_truncation():
    """BipedalWalker-v3 at 2^16 envs with a TimeLimit of 8 steps: no walker falls that fast, so the whole batch stays
    in phase through the warm-up (250 = 31 x 8 + 2) and truncates at step 5 of each call.  rollout_actor_critic
    bootstraps 2^16 final observations at once, then rollout_mlp(summary=True) folds first episodes that all end on
    the same step.  On an H100: 65 536 envs parked in a step (L = 32, two rounds) and 65 536 resets in one step,
    more than the reset-list kernel has threads."""
    n, T, H = 1 << 16, 8, (64, 64)
    b = _Batch("BipedalWalker-v3", n, m=512, max_episode_steps=8)
    try:
        env = b.twin.env
        pa, pc = _mlp_params(env, H, 4, 1), _mlp_params(env, H, 1, 2)
        e = _noise(env, T, 3, scale=0.3)
        out = b.noisy("rollout_actor_critic", lambda x: x.rollout_actor_critic(pa, pc, H, e, gamma=0.99,
                                                                                gae_lambda=0.95), pa, pc, H, e, "relu")
        te, tr = out[6], out[7]
        assert bool(tr[5].all()) and not bool(te.any()), "every env truncates at step 5, none terminates"
        p = _mlp_params(env, H, 4, 4)
        got = b.policy("rollout_mlp summary", lambda x: x.rollout_mlp(p, H, T, summary=True),
                       mlp_policy(p, H, 4, "relu", False), T, summary=True)
        assert bool(got[2].all()) and bool((got[1] == 6).all()), "every first episode ends at step 5"
    except BaseException:
        b.close()
        raise
    steps = b.finish("walker_whole_batch_truncation")
    assert max(c[1] for c in steps) == n > _reset_threads()
    _assert_second_round(n, steps)


@pytest.mark.parametrize("pattern,warmup", [("all", 0), ("every_4th", WARMUP)])
def test_forced_falls_lunar(pattern, warmup):
    """LunarLander-v2 at 2^16 envs: the pattern's landers are thrown down at 95 m/s (as in
    test_gpu_box2d_launch_shapes.py), then rollout_mlp and rollout_actor_critic run, so the crashes, their TOI
    sub-steps and the mass resets happen inside the composed sequence.  "all", right after reset, where every lander
    starts at the same height and so hits the ground in the same step: more than 32 parked envs per TOI warp and more
    resets in a step than the reset-list kernel has threads.  "every_4th", after the warm-up, at the heights random
    play left: between 2 and 32 per warp.  On an H100: 65 536 parked (L = 32, two rounds) and 65 536 resets in one
    step ("all"); up to 7 493 parked (L = 5) and 5 193 resets ("every_4th")."""
    n, T, H = 1 << 16, 8, (64, 64)
    b = _Batch("LunarLander-v2", n, m=1024, seed=3, warmup=warmup)
    try:
        b.sync()
        mask = np.ones(n, dtype=bool) if pattern == "all" else np.arange(n) % 4 == 0
        _force_falls(b.engines + [b.twin], b.windows, mask, FALL_VY)
        b.obs = b.twin.env.snapshot().obs.clone()
        env = b.twin.env
        p = _mlp_params(env, H, 4, 1)
        b.policy("rollout_mlp", lambda e: e.rollout_mlp(p, H, T), mlp_policy(p, H, 4, "relu", True), T)
        pa, pc = _mlp_params(env, H, 4, 2), _mlp_params(env, H, 1, 3)
        e = _noise(env, T, 4)
        b.noisy("rollout_actor_critic", lambda x: x.rollout_actor_critic(pa, pc, H, e, gamma=0.99, gae_lambda=0.95),
                pa, pc, H, e, "relu")
    except BaseException:
        b.close()
        raise
    steps = b.finish(f"forced_falls_lunar[{pattern}]")
    grid = _grid(n)
    if pattern == "all":
        _assert_second_round(n, steps)
        assert max(c[1] for c in steps) > _reset_threads()
    else:
        assert any(grid < c[0] <= 32 * grid for c in steps)
    assert b.terms["rollout_mlp"] > 0


@pytest.mark.parametrize("entry", ["rollout_from", "rollout_from_mlp"])
def test_rollout_from_bench_shape(entry):
    """LunarLander-v2 as rollout_from_bench.py / rollout_from_mlp_bench.py time it: 2^4 rows x 2^10 branches, T = 8,
    from a snapshot of 2^16 warmed envs (rollout_from_mlp: the (64, 64) tanh policy).  Of the B = 2^14 branches,
    3 x 1 024 hold the windows' envs in order and are checked against the oracles; the others are 16 roots, 832
    branches each.  Then B = 3 000 (the scratch batch reused, stepped over fewer envs than it holds; Gumbel noise),
    B = 2^17 + 77 (the batch grown, a ragged last CTA, several envs per TOI warp; per-branch ReLU policies) and B = 1,
    each against its own restored twin.  On an H100: at B = 2^14 about 285 branches end their first episode by
    termination and at most 1 127 envs park in a step (L = 1); at B = 2^17 + 77 up to 4 453 park (L = 3)."""
    torch = _torch()
    n, m, T, H = 1 << 16, 1024, 8, (64, 64)
    b = _Batch("LunarLander-v2", n, m=m)
    try:
        snap = b.twin.env.snapshot()
        env = b.twin.env
        g = torch.Generator(device="cpu").manual_seed(11)
        B = 1 << 14
        rows = torch.randint(0, n, (16,), generator=g).repeat_interleave(B // 16)
        blocks = [0, (B - m) // 2, B - m]
        for bo, lo in zip(blocks, b.windows.los):
            rows[bo:bo + m] = torch.arange(lo, lo + m)
        calls = [(rows, blocks), (torch.randint(0, n, (3000,), generator=g), ()),
                 (torch.randint(0, n, ((1 << 17) + 77,), generator=g), ()), (torch.tensor([n - 1]), ())]
        for k, (rows, blocks) in enumerate(calls):
            rows = rows.to(b.dev)
            B = len(rows)
            what = f"{entry} B={B}"
            if entry == "rollout_from":
                acts = torch.randint(0, 4, (T, B), generator=g).to(b.dev)

                def loop(tw, obs0):
                    o, r, te, tr, fin, masks = _eager_steps(tw, acts)
                    return _fold(r, te, tr), (acts, o, r, te, tr, masks, fin)
                b.branches(what, lambda e: e.rollout_from(snap, acts, rows=rows, states=True), snap, rows, loop,
                           blocks)
                continue
            act = "relu" if k == 2 else "tanh"
            p = _mlp_params(env, H, 4, 20 + k, lead=(B,) if k == 2 else ())
            noise = _branch_noise(env, T, B, 30) if k == 1 else None

            def loop(tw, obs0):
                if noise is None:
                    acts, (o, r, te, tr), fin, masks, _ = PolicyTwin(tw, obs0).loop(mlp_policy(p, H, 4, act, True),
                                                                                    T, None)
                else:
                    acts, _, _, _, (o, r, te, tr), fin, masks = NormTwin(tw, obs0, act).loop(p, None, H, noise,
                                                                                          dict(mean=None))
                return _fold(r, te, tr) + (acts[0],), (acts, o, r, te, tr, masks, fin)
            b.branches(what, lambda e: e.rollout_from_mlp(snap, p, H, T, noise=noise, rows=rows, states=True,
                                                          activation=act), snap, rows, loop, blocks)
    except BaseException:
        b.close()
        raise
    b.finish(f"{entry}_bench_shape")
    _assert_multi_lane((1 << 17) + 77, b.counts[f"{entry} B={(1 << 17) + 77}"])
    assert b.terms[f"{entry} B={1 << 14}"] > 0, "a branch whose first episode ends by termination"
