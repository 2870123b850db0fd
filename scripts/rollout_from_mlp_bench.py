"""Time of one closed-loop MLP-policy planning call from snapshot rows, three ways (DESIGN §4.20): the composed path
a caller writes without ``rollout_from_mlp`` (gather the branches' rows into a snapshot, ``restore`` it into a
planning batch of B envs, then ``rollout_mlp(summary=True)``, or ``rollout_mlp_noisy`` and a torch fold of its
rewards and flags over the first episode end), ``rollout_from_mlp``, and ``rollout_from_mlp(states=True)``.

The workloads are the issue's: Gumbel-sampled CartPole branches from MCTS-style leaves, MPPI on Pendulum with a
Gaussian-noised policy prior, deterministic per-branch Pendulum policies from common start rows (ES), and
LunarLander, whose ``rollout_from_mlp`` is itself composed launch by launch.  Every policy is a (64, 64) tanh MLP.
The composed noisy arm's torch fold sums in torch's order, so its returns are not bit for bit ``rollout_from_mlp``'s;
the script checks lengths, end flags and the step-0 actions for equality and reports the largest difference of the
returns.  The deterministic arms are compared bit for bit.

Timing follows rollout_bench.py's rules: every shape is warmed up, L2 is flushed before each timed call (bench.py's
L2Flush), each timed call gets one CUDA-event pair, and the arms alternate, round by round, in a rotating order.  Each
line gives the median and spread (min, max) per arm in µs per call.  Prints the card (name, power limit, max SM clock)
before and after.
Usage: python scripts/rollout_from_mlp_bench.py [--rounds R] [--out FILE]
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
from gym_b200.snapshot import EnvSnapshot  # noqa: E402
from rollout_bench import timed  # noqa: E402
from rollout_from_bench import fold  # noqa: E402
from sample_bench import card  # noqa: E402

HIDDEN = (64, 64)
# (name, env_id, log2 start rows, log2 branches per row, T, noise ("gumbel", "gauss" or None), per-branch policies)
WORKLOADS = [
    ("cartpole_gumbel", "CartPole-v1", 10, 10, 32, "gumbel", False),
    ("pendulum_gauss", "Pendulum-v1", 8, 10, 32, "gauss", False),
    ("pendulum_es_per_branch", "Pendulum-v1", 6, 10, 200, None, True),
    ("lunarlander", "LunarLander-v2", 4, 10, 8, None, False),
]


def run(name, env_id, log2r, log2k, T, noise_kind, per_branch, rounds, flush):
    R, K = 1 << log2r, 1 << log2k
    B = R * K
    src = gym_b200.vector.make(env_id, R, device=0)
    src.reset(seed=1)
    g = torch.Generator(device="cuda:0").manual_seed(0)
    for _ in range(5):   # start states a few steps into their episodes
        src.step(src.action_space.sample() if src.discrete else
                 torch.rand((R, src.act_dim), generator=g, device="cuda:0") * 2 - 1)
    snap = src.snapshot()
    Kout = int(src.single_action_space.n) if src.discrete else src.act_dim
    sizes = [src.obs_dim, *HIDDEN, Kout]
    P = sum(o * i + o for i, o in zip(sizes[:-1], sizes[1:]))
    if per_branch:   # policy j runs from every start row: branch b = j * R + r
        params = 0.3 * torch.randn((K, P), generator=g, device="cuda:0")
        params = params.repeat_interleave(R, 0).contiguous()
        rows = torch.arange(R, device="cuda:0").repeat(K)
    else:            # K branches of each start row
        params = 0.3 * torch.randn(P, generator=g, device="cuda:0")
        rows = torch.arange(R, device="cuda:0").repeat_interleave(K)
    noise = None
    if noise_kind == "gumbel":
        u = torch.rand((T, B, Kout), generator=g, device="cuda:0").clamp_(min=torch.finfo(torch.float32).tiny)
        noise = -torch.log(-torch.log(u))
    elif noise_kind == "gauss":
        noise = 0.3 * torch.randn((T, B, Kout), generator=g, device="cuda:0")
    plan = gym_b200.vector.make(env_id, B, device=0)
    runner = gym_b200.vector.make(env_id, 1, device=0)   # rollout_from_mlp touches none of its envs
    res = {}

    def composed():
        plan.restore(EnvSnapshot(snap.header, snap.rows[rows], snap.obs[rows]))
        if noise is None:
            res["composed"] = plan.rollout_mlp(params, HIDDEN, T, summary=True, activation="tanh") + (None,)
        else:
            a, _, _, rew, te, tr, _ = plan.rollout_mlp_noisy(params, HIDDEN, noise, activation="tanh")
            res["composed"] = fold(rew, te, tr) + (a[0],)

    def fused():
        res["fused"] = runner.rollout_from_mlp(snap, params, HIDDEN, T, noise=noise, rows=rows, activation="tanh")

    def fused_states():
        res["fused_states"] = runner.rollout_from_mlp(snap, params, HIDDEN, T, noise=noise, rows=rows, states=True,
                                                      activation="tanh")

    arms = {"composed": composed, "rollout_from_mlp": fused, "rollout_from_mlp_states": fused_states}
    for fn in arms.values():   # warm-up
        fn()
    torch.cuda.synchronize()
    ms = {k: [] for k in arms}
    names = list(arms)
    for r in range(rounds):
        for j in range(len(names)):
            k = names[(r + j) % len(names)]
            ms[k].append(timed(arms[k], flush, r * len(names) + j))
    out = {"workload": name, "env_id": env_id, "start_rows": R, "branches_per_row": K, "B": B, "T": T,
           "noise": noise_kind, "per_branch": per_branch, "hidden": list(HIDDEN), "rounds": rounds}
    for k, v in ms.items():
        v = np.asarray(v) * 1e3   # µs per call
        out[k + "_us_per_call"] = {"median": round(float(np.median(v)), 1), "min": round(float(v.min()), 1),
                                   "max": round(float(v.max()), 1)}
    for k in ("rollout_from_mlp", "rollout_from_mlp_states"):
        out[k + "_speedup_vs_composed"] = round(out["composed_us_per_call"]["median"] /
                                                out[k + "_us_per_call"]["median"], 3)
    c, f = res["composed"], res["fused"]
    out["lengths_and_ended_equal"] = bool(torch.equal(c[1], f[1]) and torch.equal(c[2], f[2]))
    if noise is None:
        out["returns_bitwise_equal"] = bool(torch.equal(c[0].view(torch.int64), f[0].view(torch.int64)))
    else:
        out["returns_max_abs_diff"] = float((c[0] - f[0]).abs().max())
        out["first_actions_equal"] = bool(torch.equal(c[3], f[3]))
    for e in (src, plan, runner):
        e.close()
    res.clear()
    torch.cuda.empty_cache()
    return out


def main():
    p = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    p.add_argument("--rounds", type=int, default=5)
    p.add_argument("--out", default=None, help="also write the lines to this JSON-lines file")
    args = p.parse_args()
    assert torch.cuda.is_available(), "rollout_from_mlp_bench.py measures on the GPU"
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
