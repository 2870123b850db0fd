"""Times `NormalizeReward(NormalizeObservation(gym_b200.vector.make(id, n))).step(a)` and the bare `step(a)` with
bench.py's timing rules: L2 flushed before every call, one CUDA-event pair per call on the launch stream, median /
p10 / p90.  The actions are drawn once per config, before timing.

Only the public API is used, so the same file times any version of the package: each `--tree DIR` is a source tree
with its library built (default: this one), and the trees are timed in alternation, one fresh process per tree and
round, so that the machine's drift falls on every tree alike.  Usage:
python scripts/normalize_bench.py [ENV_ID:LOG2N[:STACK] ...] [--tree DIR ...] [--rounds R] [--calls C].
Prints the card (name, power limit, max SM clock), one JSON line per tree, round and config, a summary line per
config (median over the rounds of each tree's median, with the min-max of the round medians) and the card again.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CONFIGS = ["CartPole-v1:20", "MountainCar-v0:18", "MountainCarContinuous-v0:18", "Pendulum-v1:18", "Acrobot-v1:18",
           "LunarLander-v2:16", "BipedalWalker-v3:16", "CartPole-v1:18:6"]


def worker(tree, configs, calls):
    sys.path.insert(0, tree)
    sys.path.insert(1, ROOT)
    sys.path.insert(2, os.path.join(ROOT, "scripts"))
    import torch

    import bench
    import gym_b200
    from gym_b200 import subenv
    from gym_b200.wrappers import NormalizeObservation, NormalizeReward
    from sample_bench import stats, time_flushed
    assert os.path.dirname(os.path.dirname(os.path.abspath(gym_b200.__file__))) == os.path.abspath(tree)
    torch.cuda.set_device(0)
    flush = bench.L2Flush(torch, torch.device("cuda:0"))
    for cfg in configs:
        env_id, log2n, *stack = cfg.split(":")
        n = 1 << int(log2n)
        kw = dict(wrappers=[subenv.FrameStack(int(stack[0]))]) if stack else {}
        line = {"workload": f"{env_id} num_envs=2^{log2n}" + (f" FrameStack({stack[0]})" if stack else ""), "calls": calls}
        for arm in ("bare", "normalized"):
            env = gym_b200.vector.make(env_id, n, **kw)
            if arm == "normalized":
                env = NormalizeReward(NormalizeObservation(env))
            env.reset(seed=0)
            env.action_space.seed(0)
            acts = [env.unwrapped.sample_actions().clone() for _ in range(8)]
            line[arm] = stats(time_flushed(lambda k: env.step(acts[k % len(acts)]), calls, flush))
            env.close()
        print(json.dumps(line), flush=True)


def main():
    p = argparse.ArgumentParser()
    p.add_argument("configs", nargs="*", default=CONFIGS)
    p.add_argument("--tree", action="append", default=None)
    p.add_argument("--rounds", type=int, default=3)
    p.add_argument("--calls", type=int, default=200)
    p.add_argument("--worker", default=None)
    args = p.parse_args()
    if args.worker:
        return worker(args.worker, args.configs, args.calls)
    sys.path.insert(0, os.path.join(ROOT, "scripts"))
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("normalize_bench.py needs a CUDA device")
    from sample_bench import card
    trees = [os.path.abspath(t) for t in (args.tree or [ROOT])]
    print(json.dumps(card()), flush=True)
    got = {}
    for r in range(args.rounds):
        for tree in trees:
            out = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", tree, "--calls", str(args.calls)]
                                 + args.configs, capture_output=True, text=True, check=True).stdout
            for ln in out.splitlines():
                line = json.loads(ln)
                print(json.dumps(dict(line, tree=tree, round=r)), flush=True)
                for arm in ("bare", "normalized"):
                    got.setdefault((line["workload"], arm, tree), []).append(line[arm]["median_us"])
    for cfg in dict.fromkeys(k[0] for k in got):
        summary = {"workload": cfg}
        for tree in trees:
            summary[tree] = {arm: {"median_us": float(np.median(got[(cfg, arm, tree)])),
                                   "min_us": float(min(got[(cfg, arm, tree)])),
                                   "max_us": float(max(got[(cfg, arm, tree)]))} for arm in ("bare", "normalized")}
        print(json.dumps(summary), flush=True)
    print(json.dumps(card()), flush=True)


if __name__ == "__main__":
    main()
