"""Per-step wall time of eager stepping against one CUDA graph replay of the same work (DESIGN §4.8).

For each config: eager `env.step(env.sample_actions())` against a graph that captured that pair, and, for the policy
config, `env.step(policy(obs))` with a small torch.nn MLP, eager against captured.  Timing follows bench.py's rules:
a warm-up, then windows of at least 1 s of back-to-back calls ending in a synchronise, wall clock / steps.  The two arms
alternate, window by window, so that other work on the host lands on both; the line gives the median window and the
spread (min, max) of each arm.  Usage: python scripts/graph_bench.py [ENV_ID:LOG2N ...] [--windows W]
[--policy ENV_ID:LOG2N].  Prints the card (name, power limit, max SM clock), one JSON line per config, and the card
again.
"""
import argparse
import json
import math
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import gym_b200  # noqa: E402
from sample_bench import card  # noqa: E402

MIN_WINDOW_S = 1.0
CONFIGS = ["CartPole-v1:10", "CartPole-v1:14", "CartPole-v1:17", "CartPole-v1:20", "LunarLander-v2:12",
           "LunarLander-v2:16"]


def window_ms(fn, calls):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(calls):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / calls * 1e3


def calls_for(fn):
    """Calls that fill a window of at least MIN_WINDOW_S, from a short timed run after the warm-up."""
    for _ in range(50):
        fn()
    ms = window_ms(fn, 50)
    return max(50, math.ceil(MIN_WINDOW_S * 1.1 * 1e3 / ms))


def compare(arms, windows):
    calls = {k: calls_for(fn) for k, fn in arms.items()}
    times = {k: [] for k in arms}
    for _ in range(windows):
        for k, fn in arms.items():
            times[k].append(window_ms(fn, calls[k]))
    out = {}
    for k, t in times.items():
        out[k] = {"ms_per_step": float(np.median(t)), "min": float(min(t)), "max": float(max(t)), "steps": calls[k]}
    eager, graph = (out[k]["ms_per_step"] for k in arms)
    out["eager_over_graph"] = eager / graph
    return out


def capture(fn):
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    return g


def sample_step_line(env_id, log2n, windows):
    env = gym_b200.vector.make(env_id, 1 << log2n)
    env.reset(seed=0)
    env.action_space.seed(0)

    def eager():
        env.step(env.sample_actions())
    eager()   # puts the action stream on the device, as a captured sample_actions() requires
    graph = capture(eager)
    res = compare({"eager": eager, "graph": graph.replay}, windows)
    env.close()
    return {"workload": f"{env_id} num_envs=2^{log2n}: step(sample_actions())", **res}


def policy_line(env_id, log2n, windows):
    n = 1 << log2n
    env = gym_b200.vector.make(env_id, n)
    obs, _ = env.reset(seed=0)
    torch.manual_seed(0)
    d = int(np.prod(env.single_observation_space.shape))
    net = torch.nn.Sequential(torch.nn.Linear(d, 64), torch.nn.Tanh(), torch.nn.Linear(64, 64), torch.nn.Tanh(),
                              torch.nn.Linear(64, int(env.single_action_space.n))).to(env.device)
    state = obs.clone()

    @torch.no_grad()
    def eager():
        o = env.step(net(state).argmax(-1))[0]
        state.copy_(o)
    # warm the policy's kernels on a side stream before the capture, as torch.cuda.graph's documentation asks
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            eager()
    torch.cuda.current_stream().wait_stream(side)
    graph = capture(eager)
    res = compare({"eager": eager, "graph": graph.replay}, windows)
    env.close()
    return {"workload": f"{env_id} num_envs=2^{log2n}: step(argmax(MLP {d}-64-64-{env.single_action_space.n}(obs)))",
            **res}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("configs", nargs="*", default=CONFIGS)
    p.add_argument("--policy", default="CartPole-v1:14")
    p.add_argument("--windows", type=int, default=3)
    args = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("graph_bench.py needs a CUDA device")
    torch.cuda.set_device(0)
    print(json.dumps(card()), flush=True)
    for cfg in args.configs:
        env_id, log2n = cfg.split(":")
        print(json.dumps(sample_step_line(env_id, int(log2n), args.windows)), flush=True)
    if args.policy:
        env_id, log2n = args.policy.split(":")
        print(json.dumps(policy_line(env_id, int(log2n), args.windows)), flush=True)
    print(json.dumps(card()), flush=True)


if __name__ == "__main__":
    main()
