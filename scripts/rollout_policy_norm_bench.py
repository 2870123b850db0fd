"""Time per batch step of population-search rollouts on normalised observations with the observation moments
(DESIGN §4.19): ``rollout_linear`` / ``rollout_mlp`` with ``obs_norm``, ``clip_obs`` and ``obs_moments``.

1. ``graph_replay``: one replay of a graph of T eager steps (the observation normalised in torch, the policy in torch
   -- ``addmm`` / ``nn.Sequential`` for a shared policy, ``baddbmm`` over the per-env rows otherwise -- ``step()``),
   with the returns, lengths, ended flags and the observation moments folded in torch: what such a user runs without
   the keywords.  Eager for the Box2D kinds, which cannot be captured;
2. ``summary_norm``: the summary call with ``obs_norm``, ``clip_obs`` and ``obs_moments``;
3. ``summary_raw``: today's summary call without them;
4. ``full_norm``: the full-mode call with ``obs_norm`` and ``clip_obs``.

The torch arm runs through cuBLAS, so its values are not bit for bit those of the rollout; it is what a user would
otherwise write.  Timing follows rollout_norm_bench.py's rules: every shape is warmed up, L2 is flushed before each
timed call (bench.py's L2Flush), each timed call gets one CUDA-event pair, and the arms alternate, round by round, in a
rotating order.  Each line gives the median over the rounds and the spread (min, max) per arm, in µs per batch step
(one step of all N envs), and the bytes per env-step each call moves, from the shapes.  Prints the card (name, power
limit, max SM clock) before and after.
Usage: python scripts/rollout_policy_norm_bench.py [--rounds R] [--out FILE]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import gym_b200  # noqa: E402
from bench import L2Flush  # noqa: E402
from rollout_bench import timed  # noqa: E402
from sample_bench import card  # noqa: E402

EPS, CLIP = 1e-8, 10.0
ARMS = ("summary_norm", "summary_raw", "full_norm")
# (env_id, log2 envs, T, net, per_env, first arm); net: "linear" or hidden widths of a tanh MLP
WORKLOADS = [
    ("CartPole-v1", 20, 500, "linear", False, "graph_replay"),
    ("CartPole-v1", 20, 500, "linear", True, "graph_replay"),
    ("CartPole-v1", 20, 500, (64, 64), False, "graph_replay"),
    ("Pendulum-v1", 18, 200, "linear", True, "graph_replay"),
    ("Pendulum-v1", 14, 200, (64, 64), True, "graph_replay"),
    ("Pendulum-v1", 16, 200, (64, 64), True, "graph_replay"),
    ("LunarLanderContinuous-v2", 16, 8, "linear", True, "eager"),
]


def torch_policy(net, per_env, w, b, p, sizes, discrete):
    """The torch policy of arm 1: logits or tanh MLP outputs of x, then argmax (Discrete) or the outputs (Box)."""
    layers = []
    if net != "linear":
        off = 0
        for fi, fo in zip(sizes[:-1], sizes[1:]):
            W = p[..., off:off + fo * fi].reshape(p.shape[:-1] + (fo, fi))
            off += fo * fi
            layers.append((W, p[..., off:off + fo]))
            off += fo

    def pol(x):
        if net == "linear":
            z = torch.baddbmm(b[:, :, None], w, x[:, :, None])[:, :, 0] if per_env else torch.addmm(b, x, w.t())
        else:
            z = x
            for j, (W, bb) in enumerate(layers):
                z = torch.baddbmm(bb[:, :, None], W, z[:, :, None])[:, :, 0] if per_env else torch.addmm(bb, z, W.t())
                if j < len(layers) - 1:
                    z = torch.tanh(z)
        return z.argmax(dim=1) if discrete else z
    return pol


def bytes_per_env_step(arm, D, A, K, net, per_env, P):
    """HBM bytes per env-step from the shapes: the per-step outputs of full mode (obs and final obs float32, reward
    float64, two flags, the action), and for per-env rows the parameters read each step (an MLP row) or once (a
    linear row, held in registers; amortised over T, not counted)."""
    b = 0
    if arm == "full_norm":
        b += 2 * 4 * D + 8 + 2 + (8 if A == 0 else 4 * A)
    if per_env and net != "linear":
        b += 4 * P
    return b


def run(env_id, log2n, T, net, per_env, first_arm, rounds, flush):
    n = 1 << log2n
    names = (first_arm,) + ARMS
    envs = {k: gym_b200.vector.make(env_id, n, device=0) for k in names}
    obs = {k: e.reset(seed=i)[0] for i, (k, e) in enumerate(envs.items())}
    e0 = envs[first_arm]
    K, D = int(e0.single_action_space.n if e0.discrete else e0.act_dim), e0.obs_dim
    torch.manual_seed(0)
    lead = (n,) if per_env else ()
    w = b = p = None
    sizes, P = [], 0
    if net == "linear":
        w, b = 0.1 * torch.randn(lead + (K, D), device="cuda:0"), torch.zeros(lead + (K,), device="cuda:0")
        P = K * D + K
    else:
        sizes = [D] + list(net) + [K]
        P = sum(o * i + o for i, o in zip(sizes[:-1], sizes[1:]))
        p = 0.3 * torch.randn(lead + (P,), device="cuda:0")
    f64 = dict(dtype=torch.float64, device="cuda:0")
    mean, var = 0.1 * torch.randn(D, **f64), torch.rand(D, **f64) + 0.5
    pol = torch_policy(net, per_env, w, b, p, sizes, e0.discrete)

    def norm(o):
        return ((o.double() - mean) / torch.sqrt(var + EPS)).float().clamp(-CLIP, CLIP)

    def eager(k):
        e, o = envs[k], obs[k]
        ret = torch.zeros(n, **f64)
        length = torch.zeros(n, dtype=torch.int32, device="cuda:0")
        ended = torch.zeros(n, dtype=torch.bool, device="cuda:0")
        s, q = torch.zeros(n, D, **f64), torch.zeros(n, D, **f64)
        with torch.no_grad():
            for _ in range(T):
                a = pol(norm(o))
                alive = ~ended
                o64 = o.double()
                s = torch.where(alive[:, None], s + o64, s)
                q = torch.where(alive[:, None], q + o64 * o64, q)
                o, r, te, tr, _ = e.step(a)
                ret = torch.where(alive, ret + r, ret)
                length += alive.to(torch.int32)
                ended = ended | te | tr
        obs[k] = o
        return ret, length, ended, s, q

    if net == "linear":
        call = lambda e, **kw: e.rollout_linear(w, b, T, **kw)  # noqa: E731
    else:
        call = lambda e, **kw: e.rollout_mlp(p, net, T, activation="tanh", **kw)  # noqa: E731
    arms = {}
    if first_arm == "eager":
        arms["eager"] = lambda: eager("eager")
    else:
        eager("graph_replay")   # warm the step path and cuBLAS before the capture
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            eager("graph_replay")
        arms["graph_replay"] = g.replay
    obs_kw = dict(obs_norm=(mean, var), norm_epsilon=EPS, clip_obs=CLIP)
    arms["summary_norm"] = lambda: call(envs["summary_norm"], summary=True, obs_moments=True, **obs_kw)
    arms["summary_raw"] = lambda: call(envs["summary_raw"], summary=True)
    arms["full_norm"] = lambda: call(envs["full_norm"], **obs_kw)
    for fn in arms.values():   # warm-up
        fn()
    torch.cuda.synchronize()
    ms = {k: [] for k in arms}
    order = list(arms)
    for r in range(rounds):
        for j in range(len(order)):
            k = order[(r + j) % len(order)]
            ms[k].append(timed(arms[k], flush, r * len(order) + j))
    out = {"env_id": env_id, "log2_envs": log2n, "T": T, "net": net if net == "linear" else list(net),
           "activation": None if net == "linear" else "tanh", "per_env": per_env, "clip_obs": CLIP, "rounds": rounds,
           "bytes_per_env_step": {a: bytes_per_env_step(a, D, e0.act_dim if not e0.discrete else 0, K, net, per_env, P)
                                  for a in ARMS}}
    for k, v in ms.items():
        v = np.asarray(v) * 1e3 / T   # µs per batch step
        out[k + "_us_per_batch_step"] = {"median": round(float(np.median(v)), 2), "min": round(float(v.min()), 2),
                                         "max": round(float(v.max()), 2)}
    med = {k: out[k + "_us_per_batch_step"]["median"] for k in ms}
    out["summary_norm_speedup_vs_" + first_arm] = round(med[first_arm] / med["summary_norm"], 3)
    out["summary_norm_over_summary_raw"] = round(med["summary_norm"] / med["summary_raw"], 3)
    out["full_norm_over_summary_norm"] = round(med["full_norm"] / med["summary_norm"], 3)
    for e in envs.values():
        e.close()
    arms.clear()
    torch.cuda.empty_cache()
    return out


def main():
    p = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    p.add_argument("--rounds", type=int, default=5)
    p.add_argument("--out", default=None, help="also write the lines to this JSON-lines file")
    args = p.parse_args()
    assert torch.cuda.is_available(), "rollout_policy_norm_bench.py measures on the GPU"
    assert args.rounds >= 3
    flush = L2Flush(torch, torch.device("cuda:0"))
    lines = [{"card": card()}]
    print(json.dumps(lines[0]), flush=True)
    for w in WORKLOADS:
        lines.append(run(*w, args.rounds, flush))
        print(json.dumps(lines[-1]), flush=True)
    lines.append({"card": card()})
    print(json.dumps(lines[-1]), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            f.writelines(json.dumps(x) + "\n" for x in lines)


if __name__ == "__main__":
    main()
