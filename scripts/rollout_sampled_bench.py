"""Per-env-step time of random-action collection, four ways (DESIGN §4.11): T eager ``step(sample_actions())`` calls,
one replay of a graph of those T calls, T ``sample_actions()`` + ``torch.stack`` + ``rollout()``, and
``rollout_sampled(T)``.  All four draw the action space's stream bit for bit as ``action_space.sample()`` does.

Timing follows rollout_bench.py's rules: every shape is warmed up, L2 is flushed before each timed call (bench.py's
L2Flush), each timed call gets one CUDA-event pair, and the arms alternate, round by round, in a rotating order.  Each
line gives the median over the rounds and the spread (min, max) per arm, in ns per env-step, plus the bytes per
env-step ``rollout_sampled`` must move (computed from shapes, not measured) and the bandwidth that implies against the
H100 SXM data sheet's 3.35 TB/s.  Prints the card (name, power limit, max SM clock) before and after.
Usage: python scripts/rollout_sampled_bench.py [--rounds R] [--out FILE]
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
from rollout_bench import DATASHEET_TBPS, timed  # noqa: E402
from sample_bench import card  # noqa: E402

# (env_id, log2 envs, T)
WORKLOADS = [
    ("CartPole-v1", 20, 8), ("CartPole-v1", 20, 64),
    ("Pendulum-v1", 18, 64), ("MountainCar-v0", 18, 64), ("MountainCarContinuous-v0", 18, 64),
    ("Acrobot-v1", 18, 64), ("LunarLander-v2", 16, 8),
]


def sampled_bytes(env, T):
    """HBM bytes per env-step of one rollout_sampled call, from shapes: the action written (int64, or float32 per
    element), the observation, the reward and both flags every step; the float64 state and the TimeLimit counter
    loaded and stored once per call.  Not counted: final observations and PCG64 records of the envs that finish, and
    the action-space record (80 bytes per call)."""
    S = env._lib.b200gym_state_dim(env.kind)
    act = 8 if env.discrete else 4 * env.act_dim
    return act + 4 * env.obs_dim + 8 + 2 + 2 * (8 * S + 4) / T


def run(env_id, log2n, T, rounds, flush):
    n = 1 << log2n
    eager, graphed, stacked, sampled = envs = [gym_b200.vector.make(env_id, n, device=0) for _ in range(4)]
    for i, e in enumerate(envs):
        e.reset(seed=i)
        e.action_space.seed(100 + i)

    def eager_arm():
        for _ in range(T):
            eager.step(eager.sample_actions())

    def stacked_arm():
        stacked.rollout(torch.stack([stacked.sample_actions() for _ in range(T)]))

    for _ in range(T):   # warm the step path and put the generator on the device before the capture
        graphed.step(graphed.sample_actions())
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(T):
            graphed.step(graphed.sample_actions())
    arms = {"eager_sample_step": eager_arm, "graph_replay": g.replay, "sample_stack_rollout": stacked_arm,
            "rollout_sampled": lambda: sampled.rollout_sampled(T)}
    for fn in arms.values():   # warm-up
        fn()
    torch.cuda.synchronize()
    ms = {k: [] for k in arms}
    names = list(arms)
    for r in range(rounds):
        for j in range(len(names)):
            k = names[(r + j) % len(names)]
            ms[k].append(timed(arms[k], flush, r * len(names) + j))
    per = T * n
    out = {"env_id": env_id, "log2_envs": log2n, "T": T, "rounds": rounds}
    for k, v in ms.items():
        v = np.asarray(v) * 1e6 / per   # ns per env-step
        out[k + "_ns_per_env_step"] = {"median": float(np.median(v)), "min": float(v.min()), "max": float(v.max())}
    b = sampled_bytes(sampled, T)
    med = out["rollout_sampled_ns_per_env_step"]["median"]
    out["rollout_sampled_bytes_per_env_step_from_shapes"] = round(b, 2)
    out["rollout_sampled_implied_TBps"] = round(b / med / 1e3, 3)
    out["rollout_sampled_implied_share_of_datasheet_3.35TBps"] = round(b / med / 1e3 / DATASHEET_TBPS, 3)
    for k in ("graph_replay", "sample_stack_rollout"):
        out[f"rollout_sampled_speedup_vs_{k}"] = round(out[k + "_ns_per_env_step"]["median"] / med, 3)
    for e in envs:
        e.close()
    del g
    torch.cuda.empty_cache()
    return out


def main():
    p = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    p.add_argument("--rounds", type=int, default=5)
    p.add_argument("--out", default=None, help="also write the lines to this JSON-lines file")
    args = p.parse_args()
    assert torch.cuda.is_available(), "rollout_sampled_bench.py measures on the GPU"
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
