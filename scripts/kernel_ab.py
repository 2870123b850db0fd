"""Step kernels side by side on the classic-control kinds, with bench.py's timing rules (L2 flushed before every step,
one CUDA-event pair per step, median).  Usage: python scripts/kernel_ab.py ENV_ID:LOG2N ... [--kernels l,b]
[--rounds R].  The kernels are the B200GYM_KERNEL letters; they alternate within each round.  Prints one JSON line
per (env, kernel, round)."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
import gym_b200  # noqa: E402


def main():
    p = argparse.ArgumentParser()
    p.add_argument("configs", nargs="+")
    p.add_argument("--kernels", default="l,b")
    p.add_argument("--rounds", type=int, default=2)
    p.add_argument("--steps", type=int, default=300)
    args = p.parse_args()
    dev = torch.device("cuda:0")
    flush = bench.L2Flush(torch, dev)
    for cfg in args.configs:
        env_id, log2n = cfg.split(":")
        n = 1 << int(log2n)
        for r in range(args.rounds):
            for k in args.kernels.split(","):
                os.environ["B200GYM_KERNEL"] = k
                env = gym_b200.vector.make(env_id, n)
                env.reset(seed=0)
                gen = torch.Generator(device=dev).manual_seed(99)
                pool = bench.device_actions(torch, env, n, dev, gen, count=8)
                for w in range(20):
                    env.step(pool[w % 8])
                ms = bench.time_steps_flushed(torch, env, pool, args.steps, flush)
                env.close()
                print(json.dumps({"env": env_id, "log2n": int(log2n), "kernel": k, "round": r,
                                  "us_median": 1e3 * float(np.median(ms)), "us_p10": 1e3 * float(np.percentile(ms, 10)),
                                  "us_p90": 1e3 * float(np.percentile(ms, 90))}), flush=True)


if __name__ == "__main__":
    main()
