"""Times `B200VectorEnv.sample_actions()` (space_sample_kernel) with bench.py's timing rules -- L2 flushed before every
call, one CUDA-event pair per call on the launch stream, median / p10 / p90 -- and the per-step wall time of three
random-action loops.  Usage: python scripts/sample_bench.py [ENV_ID:LOG2N ...] [--calls C] [--steps K].  Prints one
JSON line for the card, then one per config (the numbers in DESIGN.md §4.6).

Kernel time: events around the C entry point alone (b200gym_sample_space with the generator words prepared), and
around the whole `sample_actions()` call (host bookkeeping included; the flush keeps the GPU busy while the host
prepares, so the pair measures device time).  The floor is the output written once (the kernel reads nothing):
rows x cols x sizeof(element) at the data sheet's 3.35 TB/s -- a computed bound, not a measurement.

Loops (K steps after a warm-up, ending in a synchronise, wall clock / K): step(sample_actions()),
step(action_space.sample()) (host numpy draw + pageable host-to-device copy) and step(torch.randint / torch.rand).
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
import gym_b200  # noqa: E402
from gym_b200 import _lib  # noqa: E402

DATASHEET_BPS = 3.35e12


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
    except Exception as exc:   # the measurement still stands; the card line says why it is missing
        out = [f"nvidia-smi failed: {exc}"]
    return {"nvidia_smi": q, "gpus": out, "torch_device": torch.cuda.get_device_name(0)}


def stats(ms):
    ms = np.asarray(ms, dtype=np.float64)
    return {"median_us": float(np.median(ms)) * 1e3, "p10_us": float(np.percentile(ms, 10)) * 1e3,
            "p90_us": float(np.percentile(ms, 90)) * 1e3}


def time_flushed(fn, calls, flush):
    for k in range(5):
        fn(k)
    starts = [torch.cuda.Event(enable_timing=True) for _ in range(calls)]
    ends = [torch.cuda.Event(enable_timing=True) for _ in range(calls)]
    torch.cuda.synchronize()
    for k in range(calls):
        flush(k)
        starts[k].record()
        fn(k)
        ends[k].record()
    torch.cuda.synchronize()
    return [s.elapsed_time(e) for s, e in zip(starts, ends)]


def kernel_line(env_id, log2n, calls, flush):
    n = 1 << log2n
    env = gym_b200.vector.make(env_id, n)
    env.action_space.seed(0)
    n_choices, cols, low, high = env._sample_plan()
    out = env.sample_actions()
    lib, st = env._lib, env._stream()
    words = (ctypes.c_uint64 * 4)(0x12345, 0x6789, 0, 0x2b)
    lo = None if low is None else low.ctypes.data
    hi = None if high is None else high.ctypes.data

    def raw(k):
        _lib.check(lib.b200gym_sample_space(words, n, cols, n_choices, lo, hi, ctypes.c_void_p(out.data_ptr()), st))

    keep = []

    def api(k):
        keep.append(env.sample_actions())
        if len(keep) > 4:
            keep.pop(0)

    raw_ms = time_flushed(raw, calls, flush)
    api_ms = time_flushed(api, calls, flush)
    # the same launches back to back with L2 warm (code, table and output lines resident): one event pair around all
    s0, e0 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s0.record()
    for k in range(calls):
        raw(k)
    e0.record()
    torch.cuda.synchronize()
    warm_us = s0.elapsed_time(e0) / calls * 1e3
    nbytes = out.numel() * out.element_size()
    med = float(np.median(raw_ms)) * 1e-3
    env.close()
    return {"workload": f"{env_id} num_envs=2^{log2n}: sample_actions()", "calls": calls,
            "kernel": stats(raw_ms), "sample_actions_call": stats(api_ms), "kernel_warm_back_to_back_us": warm_us,
            "bytes_written": nbytes,
            "achieved_gbs": nbytes / med / 1e9, "of_datasheet_hbm": nbytes / med / DATASHEET_BPS,
            "floor_us_at_3.35TBps": nbytes / DATASHEET_BPS * 1e6}


def loop_line(env_id, log2n, steps):
    n = 1 << log2n
    env = gym_b200.vector.make(env_id, n)
    dev = env.device
    gen = torch.Generator(device=dev).manual_seed(0)

    def randint():
        if env.discrete:
            return torch.randint(0, env.single_action_space.n, (n,), device=dev, dtype=torch.int64, generator=gen)
        lo = float(env.single_action_space.low[0])
        hi = float(env.single_action_space.high[0])
        return torch.rand((n, env.act_dim), device=dev, generator=gen) * (hi - lo) + lo

    loops = {"step(sample_actions())": env.sample_actions, "step(action_space.sample())": env.action_space.sample,
             "step(torch.randint / torch.rand)": randint}
    res = {"workload": f"{env_id} num_envs=2^{log2n}: per-step wall time, {steps} steps ending in a synchronise"}
    for name, draw in loops.items():
        env.reset(seed=0)
        env.action_space.seed(0)
        for _ in range(10):
            env.step(draw())
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(steps):
            env.step(draw())
        torch.cuda.synchronize()
        res[name + " ms"] = (time.perf_counter() - t0) / steps * 1e3
    env.close()
    return res


def main():
    p = argparse.ArgumentParser()
    p.add_argument("configs", nargs="*", default=["CartPole-v1:20", "BipedalWalker-v3:16", "LunarLanderContinuous-v2:16"])
    p.add_argument("--calls", type=int, default=300)
    p.add_argument("--steps", type=int, default=1000)
    args = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sample_bench.py needs a CUDA device")
    torch.cuda.set_device(0)
    print(json.dumps(card()), flush=True)
    flush = bench.L2Flush(torch, torch.device("cuda:0"))
    for cfg in args.configs:
        env_id, log2n = cfg.split(":")
        print(json.dumps(kernel_line(env_id, int(log2n), args.calls, flush)), flush=True)
    for cfg in args.configs:
        env_id, log2n = cfg.split(":")
        print(json.dumps(loop_line(env_id, int(log2n), args.steps)), flush=True)
    print(json.dumps(card()), flush=True)


if __name__ == "__main__":
    main()
