"""Time per batch step of closed-loop evaluation of a ReLU MLP policy, four ways (DESIGN §4.13): T eager steps
(``nn.Sequential`` forward, or ``torch.baddbmm`` per layer for per-env parameters, then ``step()``), one replay of a
graph of those T steps, ``rollout_mlp(summary=False)`` and ``rollout_mlp(summary=True)``.  The eager arms run through
cuBLAS, so their actions are not bit for bit those of ``rollout_mlp``; they are what a user would otherwise write.

Timing follows rollout_bench.py's rules: every shape is warmed up, L2 is flushed before each timed call (bench.py's
L2Flush), each timed call gets one CUDA-event pair, and the arms alternate, round by round, in a rotating order.  Each
line gives the median over the rounds and the spread (min, max) per arm, in µs per batch step (one step of all N envs),
and, from shapes (``flops`` and ``mlp_bytes``, not measured), the float32 FLOP/s and HBM bytes/s ``rollout_mlp``
achieves.  The policy is unfused multiply and add, so its FLOP/s compare with half of the data sheet's 67 TFLOP/s
FP32.  Prints the card (name, power limit, max SM clock) before and after.
Usage: python scripts/rollout_mlp_bench.py [--rounds R] [--out FILE]
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
from rollout_linear_bench import linear_bytes  # noqa: E402
from sample_bench import card  # noqa: E402

FP32_UNFUSED_PEAK = 67e12 / 2   # H100 SXM data sheet FP32 (FMA counted as 2), halved: no fused multiply-add
HBM_PEAK = 3.35e12

# (env_id, log2 envs, T, hidden, per-env parameters, arms); LunarLander is not captured (rollout_mlp refuses capture,
# and the graph arm would time the same launches as the eager one)
ALL = ("eager", "graph_replay", "rollout_mlp", "rollout_mlp_summary")
WORKLOADS = [
    ("CartPole-v1", 20, 64, (32, 32), False, ALL), ("CartPole-v1", 20, 500, (32, 32), False, ALL),
    ("Pendulum-v1", 18, 64, (64, 64), False, ALL), ("Acrobot-v1", 18, 64, (64, 64), False, ALL),
    ("CartPole-v1", 14, 64, (64, 64), True, ALL), ("CartPole-v1", 16, 64, (64, 64), True, ALL),
    ("Pendulum-v1", 14, 64, (64, 64), True, ALL), ("Pendulum-v1", 16, 64, (64, 64), True, ALL),
    ("LunarLander-v2", 16, 8, (64, 64), True, ("eager", "rollout_mlp", "rollout_mlp_summary")),
]


def layers(env, hidden):
    K = env.single_action_space.n if env.discrete else env.act_dim
    sizes = [env.obs_dim] + list(hidden) + [int(K)]
    return list(zip(sizes[:-1], sizes[1:]))


def param_count(env, hidden):
    return sum(o * i + o for i, o in layers(env, hidden))


def flops(env, hidden):
    """float32 operations per env-step of the policy: one multiply and one add per weight."""
    return sum(2 * o * i for i, o in layers(env, hidden))


def mlp_bytes(env, T, hidden, per_env, summary):
    """HBM bytes per env-step of one rollout_mlp call, from shapes: rollout_linear's (linear_bytes, without its
    per-env linear parameters) plus, with per-env parameters, the env's P floats read at every step.  A shared policy
    is read from HBM once per call (each CTA's copy comes from L2), which rounds to 0 per env-step."""
    base = linear_bytes(env, T, False, summary)
    return base + (4 * param_count(env, hidden) if per_env else 0)


def unpack(env, params, hidden):
    """[(W (N, out, in), b (N, out, 1))] views of per-env params (N, P)."""
    out, off, n = [], 0, env.num_envs
    for i, o in layers(env, hidden):
        w = params[:, off:off + o * i].view(n, o, i)
        off += o * i
        out.append((w, params[:, off:off + o].view(n, o, 1)))
        off += o
    return out


def run(env_id, log2n, T, hidden, per_env, arms_wanted, rounds, flush):
    n = 1 << log2n
    envs = {k: gym_b200.vector.make(env_id, n, device=0) for k in arms_wanted}
    obs = {}
    for i, (k, e) in enumerate(envs.items()):
        obs[k] = e.reset(seed=i)[0]
    e0 = next(iter(envs.values()))
    torch.manual_seed(0)
    mods = []
    for j, (i, o) in enumerate(layers(e0, hidden)):
        mods += [torch.nn.Linear(i, o)] + ([torch.nn.ReLU()] if j < len(hidden) else [])
    net = torch.nn.Sequential(*mods).to("cuda:0")
    vec = torch.nn.utils.parameters_to_vector(net.parameters()).detach()
    params = (vec + 0.05 * torch.randn(n, vec.numel(), device="cuda:0")).contiguous() if per_env else vec.contiguous()
    views = unpack(e0, params, hidden) if per_env else None

    def forward(x):
        if not per_env:
            return net(x)
        x = x.unsqueeze(2)
        for j, (w, b) in enumerate(views):
            x = torch.baddbmm(b, w, x)
            if j < len(hidden):
                x = torch.relu(x)
        return x.squeeze(2)

    def loop(k):
        e = envs[k]
        o = obs[k]
        with torch.no_grad():
            for _ in range(T):
                z = forward(o)
                o = e.step(z.argmax(dim=1) if e.discrete else z)[0]
        obs[k] = o

    arms = {}
    if "eager" in envs:
        arms["eager"] = lambda: loop("eager")
    if "graph_replay" in envs:
        loop("graph_replay")   # warm the step path and cuBLAS before the capture
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            loop("graph_replay")
        arms["graph_replay"] = graph.replay
    if "rollout_mlp" in envs:
        arms["rollout_mlp"] = lambda: envs["rollout_mlp"].rollout_mlp(params, hidden, T)
    if "rollout_mlp_summary" in envs:
        arms["rollout_mlp_summary"] = lambda: envs["rollout_mlp_summary"].rollout_mlp(params, hidden, T, summary=True)
    for fn in arms.values():   # warm-up
        fn()
    torch.cuda.synchronize()
    ms = {k: [] for k in arms}
    names = list(arms)
    for r in range(rounds):
        for j in range(len(names)):
            k = names[(r + j) % len(names)]
            ms[k].append(timed(arms[k], flush, r * len(names) + j))
    out = {"env_id": env_id, "log2_envs": log2n, "T": T, "hidden": list(hidden),
           "params": "per_env" if per_env else "shared", "P": param_count(e0, hidden), "rounds": rounds}
    for k, v in ms.items():
        v = np.asarray(v) * 1e3 / T   # µs per batch step
        out[k + "_us_per_batch_step"] = {"median": round(float(np.median(v)), 2), "min": round(float(v.min()), 2),
                                         "max": round(float(v.max()), 2)}
    out["flops_per_env_step_from_shapes"] = flops(e0, hidden)
    for a, summary in (("rollout_mlp", False), ("rollout_mlp_summary", True)):
        nbytes = mlp_bytes(e0, T, hidden, per_env, summary)
        sec = out[a + "_us_per_batch_step"]["median"] * 1e-6
        out[a + "_bytes_per_env_step_from_shapes"] = round(nbytes, 2)
        out[a + "_tflops"] = round(n * flops(e0, hidden) / sec / 1e12, 3)
        out[a + "_tflops_share_of_unfused_fp32_peak"] = round(n * flops(e0, hidden) / sec / FP32_UNFUSED_PEAK, 4)
        out[a + "_tb_per_s"] = round(n * nbytes / sec / 1e12, 3)
        out[a + "_share_of_hbm_peak"] = round(n * nbytes / sec / HBM_PEAK, 4)
    for k in ("eager", "graph_replay"):
        if k in ms:
            for a in ("rollout_mlp", "rollout_mlp_summary"):
                out[f"{a}_speedup_vs_{k}"] = round(out[k + "_us_per_batch_step"]["median"] /
                                                   out[a + "_us_per_batch_step"]["median"], 3)
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
    assert torch.cuda.is_available(), "rollout_mlp_bench.py measures on the GPU"
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
