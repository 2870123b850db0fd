"""Time per batch step of closed-loop evaluation of a linear policy, four ways (DESIGN §4.12): T eager steps (the torch
restatement of the policy, then ``step()``), one replay of a graph of those T steps, ``rollout_linear(summary=False)``
and ``rollout_linear(summary=True)``.  All four compute the same actions bit for bit.

Timing follows rollout_bench.py's rules: every shape is warmed up, L2 is flushed before each timed call (bench.py's
L2Flush), each timed call gets one CUDA-event pair, and the arms alternate, round by round, in a rotating order.  Each
line gives the median over the rounds and the spread (min, max) per arm, in µs per batch step (one step of all N envs),
plus the bytes per env-step both rollout_linear arms must move (computed from shapes, not measured).  Prints the card
(name, power limit, max SM clock) before and after.
Usage: python scripts/rollout_linear_bench.py [--rounds R] [--out FILE]
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

# (env_id, log2 envs, T, per-env parameters, arms); LunarLander is not captured (its rollout_linear refuses capture,
# and the graph arm would time the same launches as the eager one)
ALL = ("eager", "graph_replay", "rollout_linear", "rollout_linear_summary")
WORKLOADS = [
    ("CartPole-v1", 20, 64, False, ALL), ("CartPole-v1", 20, 64, True, ALL),
    ("CartPole-v1", 20, 500, False, ALL), ("CartPole-v1", 20, 500, True, ALL),
    ("Pendulum-v1", 18, 64, True, ALL), ("MountainCar-v0", 18, 64, True, ALL), ("Acrobot-v1", 18, 64, True, ALL),
    ("LunarLander-v2", 16, 8, True, ("eager", "rollout_linear", "rollout_linear_summary")),
]


def policy(env, w, b, obs):
    """The documented arithmetic as torch elementwise ops (the tests' eager twin)."""
    z = b.expand(env.num_envs, b.shape[-1]).clone()
    for k in range(env.obs_dim):
        z = z + w[..., k] * obs[:, None, k]
    if not env.discrete:
        return z
    m, best = z[:, 0], torch.zeros(env.num_envs, dtype=torch.int64, device=z.device)
    for j in range(1, z.shape[1]):
        take = ~torch.isnan(m) & (torch.isnan(z[:, j]) | (z[:, j] > m))
        m = torch.where(take, z[:, j], m)
        best = torch.where(take, torch.full_like(best, j), best)
    return best


def linear_bytes(env, T, per_env, summary):
    """HBM bytes per env-step of one rollout_linear call, from shapes.  Per step (summary=False only): the action
    (int64, or float32 per element), the observation, the reward and both flags.  Per call: the float64 state and the
    TimeLimit counter loaded and stored, the per-env parameters loaded, the last observation stored, and (summary) the
    float64 return, int32 length and flag.  Not counted: final observations and PCG64 records of the envs that
    finish."""
    S = env._lib.b200gym_state_dim(env.kind) if env.kind < 5 else 0
    K = env.single_action_space.n if env.discrete else env.act_dim
    act = 8 if env.discrete else 4 * env.act_dim
    per_call = 2 * (8 * S + 4) + (4 * K * (env.obs_dim + 1) if per_env else 0) + 4 * env.obs_dim
    if summary:
        return (per_call + 8 + 4 + 1) / T
    return act + 4 * env.obs_dim + 8 + 2 + per_call / T


def run(env_id, log2n, T, per_env, arms_wanted, rounds, flush):
    n = 1 << log2n
    envs = {k: gym_b200.vector.make(env_id, n, device=0) for k in arms_wanted}
    obs = {}
    for i, (k, e) in enumerate(envs.items()):
        obs[k] = e.reset(seed=i)[0]
    e0 = next(iter(envs.values()))
    K = e0.single_action_space.n if e0.discrete else e0.act_dim
    g = torch.Generator(device="cpu").manual_seed(0)
    lead = (n,) if per_env else ()
    w = (0.5 * torch.randn(lead + (K, e0.obs_dim), generator=g)).to("cuda:0")
    b = (0.5 * torch.randn(lead + (K,), generator=g)).to("cuda:0")

    def loop(k):
        e = envs[k]
        o = obs[k]
        for _ in range(T):
            o = e.step(policy(e, w, b, o))[0]
        obs[k] = o

    arms = {}
    if "eager" in envs:
        arms["eager"] = lambda: loop("eager")
    if "graph_replay" in envs:
        loop("graph_replay")   # warm the step path before the capture
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            loop("graph_replay")
        arms["graph_replay"] = graph.replay
    if "rollout_linear" in envs:
        arms["rollout_linear"] = lambda: envs["rollout_linear"].rollout_linear(w, b, T)
    if "rollout_linear_summary" in envs:
        arms["rollout_linear_summary"] = lambda: envs["rollout_linear_summary"].rollout_linear(w, b, T, summary=True)
    for fn in arms.values():   # warm-up
        fn()
    torch.cuda.synchronize()
    ms = {k: [] for k in arms}
    names = list(arms)
    for r in range(rounds):
        for j in range(len(names)):
            k = names[(r + j) % len(names)]
            ms[k].append(timed(arms[k], flush, r * len(names) + j))
    out = {"env_id": env_id, "log2_envs": log2n, "T": T, "params": "per_env" if per_env else "shared",
           "rounds": rounds}
    for k, v in ms.items():
        v = np.asarray(v) * 1e3 / T   # µs per batch step
        out[k + "_us_per_batch_step"] = {"median": round(float(np.median(v)), 2), "min": round(float(v.min()), 2),
                                         "max": round(float(v.max()), 2)}
    ro = envs.get("rollout_linear") or e0
    out["rollout_linear_bytes_per_env_step_from_shapes"] = round(linear_bytes(ro, T, per_env, False), 2)
    out["rollout_linear_summary_bytes_per_env_step_from_shapes"] = round(linear_bytes(ro, T, per_env, True), 3)
    for k in ("eager", "graph_replay"):
        if k in ms:
            for a in ("rollout_linear", "rollout_linear_summary"):
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
    assert torch.cuda.is_available(), "rollout_linear_bench.py measures on the GPU"
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
