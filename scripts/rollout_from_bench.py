"""Time of one planning call from snapshot rows, three ways (DESIGN §4.16): the composed path a planner writes without
``rollout_from`` (gather the branches' rows into a snapshot, ``restore`` it into a planning batch of B envs,
``rollout(actions)``, then fold the rewards and flags over the first episode end in torch), ``rollout_from``, and
``rollout_from(states=True)``.

The classic-control workloads are MPPI-shaped: R roots, each branched K times through ``rows``, with one sequence of
random actions per branch.  LunarLander's ``rollout_from`` is itself the composed path (its Box2D steps take
milliseconds), so its line records what the two cost side by side.  The composed arm's torch fold sums in torch's
order, so its returns are not bit for bit ``rollout_from``'s; the script checks lengths and end flags for equality and
reports the largest difference of the returns.

Timing follows rollout_bench.py's rules: every shape is warmed up, L2 is flushed before each timed call (bench.py's
L2Flush), each timed call gets one CUDA-event pair, and the arms alternate, round by round, in a rotating order.  Each
line gives the median and spread (min, max) per arm in µs per call and, from shapes (``bytes_per_branch``, not
measured), the HBM bytes/s ``rollout_from`` achieves against the H100 SXM's 3.35 TB/s.  Prints the card (name, power
limit, max SM clock) before and after.
Usage: python scripts/rollout_from_bench.py [--rounds R] [--out FILE]
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
from sample_bench import card  # noqa: E402

HBM_PEAK = 3.35e12
# (env_id, log2 roots, log2 branches per root, T, arms)
WORKLOADS = [
    ("CartPole-v1", 10, 10, 32, ("composed", "rollout_from", "rollout_from_states")),
    ("Pendulum-v1", 8, 10, 32, ("composed", "rollout_from", "rollout_from_states")),
    ("Acrobot-v1", 8, 10, 32, ("composed", "rollout_from", "rollout_from_states")),
    ("LunarLander-v2", 4, 10, 8, ("composed", "rollout_from")),
]


def bytes_per_branch(env, T, states):
    """HBM bytes one branch of rollout_from moves, from shapes: its root row, its T actions, the 13 bytes of summary
    (float64 return, int32 length, bool ended) and, with states, the end row and the float32 end observation."""
    R = env.snapshot_row_bytes
    act = 8 if env.discrete else 4 * env.act_dim
    return R + T * act + 13 + ((R + 4 * env.obs_dim) if states else 0)


def fold(rew, te, tr):
    """The planner's torch fold: each branch's return, length and end flag up to its first episode end."""
    done = te | tr
    upto = (done.to(torch.int32).cumsum(0) - done.to(torch.int32)) == 0   # steps up to and including the first end
    return torch.where(upto, rew, 0.0).sum(0), upto.sum(0, dtype=torch.int32), done.any(0)


def run(env_id, log2r, log2k, T, arms_wanted, rounds, flush):
    R, K = 1 << log2r, 1 << log2k
    B = R * K
    src = gym_b200.vector.make(env_id, R, device=0)
    src.reset(seed=1)
    g = torch.Generator(device="cuda:0").manual_seed(0)
    for _ in range(5):   # roots a few steps into their episodes
        src.step(src.action_space.sample() if src.discrete else
                 torch.rand((R, src.act_dim), generator=g, device="cuda:0") * 2 - 1)
    snap = src.snapshot()
    rows = torch.arange(R, device="cuda:0").repeat_interleave(K)
    if src.discrete:
        acts = torch.randint(0, int(src.single_action_space.n), (T, B), generator=g, device="cuda:0")
    else:
        lo, hi = float(src.single_action_space.low[0]), float(src.single_action_space.high[0])
        acts = lo + (hi - lo) * torch.rand((T, B, src.act_dim), generator=g, device="cuda:0")
    plan = gym_b200.vector.make(env_id, B, device=0)
    runner = gym_b200.vector.make(env_id, 1, device=0)   # rollout_from touches none of its envs
    res = {}

    def composed():
        plan.restore(EnvSnapshot(snap.header, snap.rows[rows], snap.obs[rows]))
        _, rew, te, tr, _ = plan.rollout(acts)
        res["composed"] = fold(rew, te, tr)

    def fused():
        res["rollout_from"] = runner.rollout_from(snap, acts, rows=rows)

    def fused_states():
        res["rollout_from_states"] = runner.rollout_from(snap, acts, rows=rows, states=True)

    arms = {k: v for k, v in (("composed", composed), ("rollout_from", fused), ("rollout_from_states", fused_states))
            if k in arms_wanted}
    for fn in arms.values():   # warm-up
        fn()
    torch.cuda.synchronize()
    ms = {k: [] for k in arms}
    names = list(arms)
    for r in range(rounds):
        for j in range(len(names)):
            k = names[(r + j) % len(names)]
            ms[k].append(timed(arms[k], flush, r * len(names) + j))
    out = {"env_id": env_id, "roots": R, "branches_per_root": K, "B": B, "T": T, "rounds": rounds}
    for k, v in ms.items():
        v = np.asarray(v) * 1e3   # µs per call
        out[k + "_us_per_call"] = {"median": round(float(np.median(v)), 1), "min": round(float(v.min()), 1),
                                   "max": round(float(v.max()), 1)}
    for k in ("rollout_from", "rollout_from_states"):
        if k not in ms:
            continue
        nbytes = bytes_per_branch(src, T, k.endswith("states"))
        sec = out[k + "_us_per_call"]["median"] * 1e-6
        out[k + "_bytes_per_branch_from_shapes"] = nbytes
        out[k + "_tb_per_s"] = round(B * nbytes / sec / 1e12, 3)
        out[k + "_share_of_hbm_peak"] = round(B * nbytes / sec / HBM_PEAK, 4)
        out[k + "_speedup_vs_composed"] = round(out["composed_us_per_call"]["median"] /
                                                out[k + "_us_per_call"]["median"], 3)
    # the arms compute the same thing: lengths and end flags equal, returns up to the fold's summation order
    c, f = res["composed"], res["rollout_from"]
    out["lengths_and_ended_equal"] = bool(torch.equal(c[1], f[1]) and torch.equal(c[2], f[2]))
    out["returns_max_abs_diff"] = float((c[0] - f[0]).abs().max())
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
    assert torch.cuda.is_available(), "rollout_from_bench.py measures on the GPU"
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
