"""Per-env-step time of `rollout(actions)` against T eager `step()` calls and one replay of a graph of those T steps
(DESIGN §4.10).

Timing follows bench.py's rules: every shape is warmed up, L2 is flushed before each timed call (bench.py's L2Flush),
each timed call -- T eager steps, one graph replay, one rollout -- gets one CUDA-event pair, and the three arms
alternate, round by round, in a rotating order.  Each line gives the median over the rounds and the spread (min, max)
per arm, in ns per env-step, plus the bytes per env-step the rollout must move (computed from shapes, not measured)
and the bandwidth that implies against the H100 SXM data sheet's 3.35 TB/s.  Prints the card (name, power limit, max
SM clock) before and after.  Usage: python scripts/rollout_bench.py [--rounds R] [--out FILE]
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
from sample_bench import card  # noqa: E402

DATASHEET_TBPS = 3.35
# (env_id, log2 envs, T, action dtype)
WORKLOADS = [
    ("CartPole-v1", 20, 8, "uint8"), ("CartPole-v1", 20, 64, "uint8"),
    ("CartPole-v1", 20, 8, "int64"), ("CartPole-v1", 20, 64, "int64"),
    ("Pendulum-v1", 18, 64, "float32"), ("MountainCar-v0", 18, 64, "int64"),
    ("MountainCarContinuous-v0", 18, 64, "float32"), ("Acrobot-v1", 18, 64, "int64"),
    ("LunarLander-v2", 16, 8, "int64"),
]


def rollout_bytes(env, T, act_bytes):
    """HBM bytes per env-step of one rollout, from shapes: the action, the observation, the reward and both flags
    every step; the float64 state and the TimeLimit counter loaded and stored once per call.  Not counted: final
    observations and PCG64 records of the envs that finish (a few percent of the env-steps)."""
    S = env._lib.b200gym_state_dim(env.kind)
    return act_bytes + 4 * env.obs_dim + 8 + 2 + 2 * (8 * S + 4) / T


def actions(env, T, dtype, gen):
    n = env.num_envs
    if env.discrete:
        return torch.randint(0, int(env.single_action_space.n), (T, n), device="cuda:0", generator=gen).to(dtype)
    lo = torch.as_tensor(env.single_action_space.low, device="cuda:0")
    hi = torch.as_tensor(env.single_action_space.high, device="cuda:0")
    return lo + (hi - lo) * torch.rand((T, n, env.act_dim), device="cuda:0", generator=gen)


def timed(fn, flush, k):
    flush(k)
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e)


def run(env_id, log2n, T, dtype, rounds, flush):
    n = 1 << log2n
    dt = getattr(torch, dtype)
    eager, graphed, rolled = (gym_b200.vector.make(env_id, n, device=0) for _ in range(3))
    for i, e in enumerate((eager, graphed, rolled)):
        e.reset(seed=i)
    gen = torch.Generator(device="cuda:0")
    gen.manual_seed(0)
    acts = actions(eager, T, dt, gen)

    def eager_arm():
        for t in range(T):
            eager.step(acts[t])

    for t in range(T):   # warm the step path before the capture, as a user would
        graphed.step(acts[t])
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for t in range(T):
            graphed.step(acts[t])
    arms = {"eager_steps": eager_arm, "graph_replay": g.replay, "rollout": lambda: rolled.rollout(acts)}
    for fn in arms.values():   # warm-up
        fn()
    torch.cuda.synchronize()
    ms = {k: [] for k in arms}
    names = list(arms)
    for r in range(rounds):
        for j in range(len(names)):
            k = names[(r + j) % len(names)]
            ms[k].append(timed(arms[k], flush, r * 3 + j))
    per = T * n
    out = {"env_id": env_id, "log2_envs": log2n, "T": T, "action_dtype": dtype, "rounds": rounds}
    for k, v in ms.items():
        v = np.asarray(v) * 1e6 / per   # ns per env-step
        out[k + "_ns_per_env_step"] = {"median": float(np.median(v)), "min": float(v.min()), "max": float(v.max())}
    b = rollout_bytes(rolled, T, acts.element_size() * (1 if rolled.discrete else rolled.act_dim))
    med = out["rollout_ns_per_env_step"]["median"]
    out["rollout_bytes_per_env_step_from_shapes"] = round(b, 2)
    out["rollout_implied_TBps"] = round(b / med / 1e3, 3)
    out["rollout_implied_share_of_datasheet_3.35TBps"] = round(b / med / 1e3 / DATASHEET_TBPS, 3)
    out["rollout_speedup_vs_graph"] = round(out["graph_replay_ns_per_env_step"]["median"] / med, 3)
    for e in (eager, graphed, rolled):
        e.close()
    del g
    torch.cuda.empty_cache()
    return out


def main():
    p = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    p.add_argument("--rounds", type=int, default=5)
    p.add_argument("--out", default=None, help="also write the lines to this JSON-lines file")
    args = p.parse_args()
    assert torch.cuda.is_available(), "rollout_bench.py measures on the GPU"
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
