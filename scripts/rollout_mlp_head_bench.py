"""Time per batch step of off-policy collection with a tanh-squashed actor, three ways (DESIGN §4.21): one replay of a
graph of T eager steps (a CleanRL-shaped actor module, its head and its exploration noise in torch, then ``step()``),
``rollout_mlp_noisy(head=...)`` and ``rollout_mlp_noisy`` without a head on the same trunk (the head's own cost is the
ratio of the two).  Every arm draws its noise in the timed call: the graph inside it as CleanRL does at each step, the
rollouts into a buffer just before the launch.  BipedalWalker cannot be captured, so its first arm runs the T eager
steps instead.  The eager arms run through cuBLAS, so their actions are not bit for bit those of the rollouts; they
are what a user would otherwise write.

The actors, at hidden (64, 64) with ReLU, as in CleanRL's td3_continuous_action.py and sac_continuous_action.py:
``td3``: ``fc1``, ``fc2``, ``fc_mu``, action ``clamp(tanh(fc_mu(x)) * scale + bias + N(0, (0.1 * scale)^2), low,
high)``; ``sac``: ``fc1``, ``fc2``, ``fc_mean``, ``fc_logstd``, action ``tanh(m + eps * exp(ls)) * scale + bias``.
The arm without a head runs the TD3 actor's trunk and ``fc_mu`` (for SAC, ``fc_mean``) with the same noise added.

Timing follows rollout_bench.py's rules: every shape is warmed up, L2 is flushed before each timed call (bench.py's
L2Flush), each timed call gets one CUDA-event pair, and the arms alternate, round by round, in a rotating order.  Each
line gives the median over the rounds and the spread (min, max) per arm, in µs per batch step (one step of all N
envs), and, from shapes (not measured), the policy's float32 operations and the HBM bytes per env-step of the fused
call and the rate it achieves.  Prints the card (name, power limit, max SM clock) before and after.
Usage: python scripts/rollout_mlp_head_bench.py [--rounds R] [--out FILE]
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
from rollout_mlp_bench import HBM_PEAK, mlp_bytes  # noqa: E402
from sample_bench import card  # noqa: E402

HIDDEN = (64, 64)
# (env_id, log2 envs, T, actor, arms)
WORKLOADS = [
    ("Pendulum-v1", 18, 64, "td3", ("graph_replay", "head", "no_head")),
    ("Pendulum-v1", 18, 64, "sac", ("graph_replay", "head", "no_head")),
    ("MountainCarContinuous-v0", 18, 64, "td3", ("graph_replay", "head", "no_head")),
    ("MountainCarContinuous-v0", 18, 64, "sac", ("graph_replay", "head", "no_head")),
    ("BipedalWalker-v3", 14, 8, "sac", ("eager", "head", "no_head")),
]


def head_flops(D, A, K):
    """float32 operations per env-step of the policy, from shapes: one multiply and one add per weight of
    D -> 64 -> 64 -> K."""
    sizes = [D] + list(HIDDEN) + [K]
    return sum(2 * o * i for i, o in zip(sizes[:-1], sizes[1:]))


def head_bytes(env, T, K):
    """HBM bytes per env-step of one rollout_mlp_noisy(head=...) call, from shapes: rollout_mlp's with a shared policy,
    plus A floats of noise read and K floats of outputs written."""
    return mlp_bytes(env, T, HIDDEN, False, False) + 4 * (int(env.act_dim) + K)


def run(env_id, log2n, T, kind, arms_wanted, rounds, flush):
    n = 1 << log2n
    envs = {k: gym_b200.vector.make(env_id, n, device=0) for k in arms_wanted}
    obs = {}
    for i, (k, e) in enumerate(envs.items()):
        obs[k] = e.reset(seed=i)[0]
    e0 = next(iter(envs.values()))
    D, A = e0.obs_dim, int(e0.act_dim)
    single = e0.single_action_space
    f32 = dict(dtype=torch.float32, device="cuda:0")
    scale = torch.tensor((single.high - single.low) / 2.0, **f32)
    bias = torch.tensor((single.high + single.low) / 2.0, **f32)
    low, high = float(single.low[0]), float(single.high[0])
    torch.manual_seed(0)
    fc1, fc2 = torch.nn.Linear(D, 64).cuda(), torch.nn.Linear(64, 64).cuda()
    mu, logstd = torch.nn.Linear(64, A).cuda(), torch.nn.Linear(64, A).cuda()
    trunk = [fc1.weight, fc1.bias, fc2.weight, fc2.bias]
    if kind == "td3":
        params = torch.cat([p.reshape(-1) for p in trunk + [mu.weight, mu.bias]]).detach().contiguous()
        no_head = params
    else:   # CleanRL's two-head packing
        params = torch.cat([p.reshape(-1) for p in trunk + [mu.weight, logstd.weight, mu.bias, logstd.bias]])
        params = params.detach().contiguous()
        no_head = torch.cat([p.reshape(-1) for p in trunk + [mu.weight, mu.bias]]).detach().contiguous()
    K = A * (2 if kind == "sac" else 1)
    noise = {k: torch.empty(T, n, A, **f32) for k in ("head", "no_head")}

    def draw(k):
        e = noise[k].normal_()
        return e.mul_(scale * 0.1) if kind == "td3" else e

    def act(o):
        h = torch.relu(fc2(torch.relu(fc1(o))))
        if kind == "td3":
            x = torch.tanh(mu(h)) * scale + bias
            return (x + torch.randn_like(x) * (scale * 0.1)).clamp(low, high)
        m = mu(h)
        ls = -5 + 3.5 * (torch.tanh(logstd(h)) + 1)
        return torch.tanh(m + torch.randn_like(m) * ls.exp()) * scale + bias

    def loop(k):
        e = envs[k]
        o = obs[k]
        with torch.no_grad():
            for _ in range(T):
                o = e.step(act(o))[0]
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
    head = "tanh" if kind == "td3" else "tanh_normal"
    arms["head"] = lambda: envs["head"].rollout_mlp_noisy(params, HIDDEN, draw("head"), head=head)
    arms["no_head"] = lambda: envs["no_head"].rollout_mlp_noisy(no_head, HIDDEN, draw("no_head"))
    for fn in arms.values():   # warm-up
        fn()
    torch.cuda.synchronize()
    ms = {k: [] for k in arms}
    names = list(arms)
    for r in range(rounds):
        for j in range(len(names)):
            k = names[(r + j) % len(names)]
            ms[k].append(timed(arms[k], flush, r * len(names) + j))
    out = {"env_id": env_id, "log2_envs": log2n, "T": T, "hidden": list(HIDDEN), "actor": kind, "head": head,
           "P": int(params.numel()), "K": K, "rounds": rounds}
    for k, v in ms.items():
        v = np.asarray(v) * 1e3 / T   # µs per batch step
        out[k + "_us_per_batch_step"] = {"median": round(float(np.median(v)), 2), "min": round(float(v.min()), 2),
                                         "max": round(float(v.max()), 2)}
    out["flops_per_env_step_from_shapes"] = head_flops(D, A, K)
    nbytes = head_bytes(e0, T, K)
    sec = out["head_us_per_batch_step"]["median"] * 1e-6
    out["head_bytes_per_env_step_from_shapes"] = round(nbytes, 2)
    out["head_tflop_per_s"] = round(n * head_flops(D, A, K) / sec / 1e12, 2)
    out["head_share_of_hbm_peak"] = round(n * nbytes / sec / HBM_PEAK, 4)
    base = "graph_replay" if "graph_replay" in ms else "eager"
    out[f"head_speedup_vs_{base}"] = round(out[base + "_us_per_batch_step"]["median"] /
                                           out["head_us_per_batch_step"]["median"], 3)
    out["head_over_no_head"] = round(out["head_us_per_batch_step"]["median"] /
                                     out["no_head_us_per_batch_step"]["median"], 3)
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
    assert torch.cuda.is_available(), "rollout_mlp_head_bench.py measures on the GPU"
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
