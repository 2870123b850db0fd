"""Times `gym_b200.wrappers.RecordEpisodeStatistics(gym_b200.vector.make(id, n)).step(a)` with bench.py's timing rules:
L2 flushed before every call, one CUDA-event pair per call on the launch stream, median / p10 / p90 (the numbers in
DESIGN.md §4.1).  The pair encloses the whole call, host bookkeeping included; the flush keeps the GPU busy while the
host prepares, so it measures device time.  The actions are drawn once per config, before timing.

Also one captured replay of `step(sample_actions())` behind the wrapper, per step: a warm-up, then windows of at least
1 s of back-to-back replays ending in a synchronise, wall clock / replays (as scripts/graph_bench.py).

Only the public API is used, so the same file times any version of the package.  Usage:
python scripts/episode_stats_bench.py [ENV_ID:LOG2N ...] [--calls C] [--graph ENV_ID:LOG2N] [--windows W].  Prints the
card (name, power limit, max SM clock), one JSON line per config, and the card again.
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

import bench  # noqa: E402
import gym_b200  # noqa: E402
from gym_b200.wrappers import RecordEpisodeStatistics  # noqa: E402
from graph_bench import calls_for, capture, window_ms  # noqa: E402
from sample_bench import card, stats, time_flushed  # noqa: E402

CONFIGS = ["CartPole-v1:20", "CartPole-v1:12", "Pendulum-v1:18", "Acrobot-v1:18", "LunarLander-v2:16"]


def eager_line(env_id, log2n, calls, flush):
    n = 1 << log2n
    env = RecordEpisodeStatistics(gym_b200.vector.make(env_id, n))
    env.reset(seed=0)
    env.action_space.seed(0)
    acts = [env.sample_actions().clone() for _ in range(8)]   # draws that the timed calls do not include
    ms = time_flushed(lambda k: env.step(acts[k % len(acts)]), calls, flush)
    count = env.episode_count
    env.close()
    return {"workload": f"{env_id} num_envs=2^{log2n}: RecordEpisodeStatistics(env).step(a), L2 flushed",
            "calls": calls, "step": stats(ms), "episodes_finished": count}


def graph_line(env_id, log2n, windows):
    env = RecordEpisodeStatistics(gym_b200.vector.make(env_id, 1 << log2n))
    env.reset(seed=0)
    env.action_space.seed(0)

    def step():
        env.step(env.sample_actions())
    step()   # puts the action stream on the device, as a captured sample_actions() requires
    graph = capture(step)
    calls = calls_for(graph.replay)
    ms = [window_ms(graph.replay, calls) for _ in range(windows)]
    env.close()
    return {"workload": f"{env_id} num_envs=2^{log2n}: one replay of a captured "
                        "RecordEpisodeStatistics(env).step(sample_actions())",
            "ms_per_step": float(np.median(ms)), "min": float(min(ms)), "max": float(max(ms)), "steps": calls}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("configs", nargs="*", default=CONFIGS)
    p.add_argument("--calls", type=int, default=300)
    p.add_argument("--graph", default="CartPole-v1:14")
    p.add_argument("--windows", type=int, default=3)
    args = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("episode_stats_bench.py needs a CUDA device")
    torch.cuda.set_device(0)
    print(json.dumps(card()), flush=True)
    flush = bench.L2Flush(torch, torch.device("cuda:0"))
    for cfg in args.configs:
        env_id, log2n = cfg.split(":")
        print(json.dumps(eager_line(env_id, int(log2n), args.calls, flush)), flush=True)
    if args.graph:
        env_id, log2n = args.graph.split(":")
        print(json.dumps(graph_line(env_id, int(log2n), args.windows)), flush=True)
    print(json.dumps(card()), flush=True)


if __name__ == "__main__":
    main()
