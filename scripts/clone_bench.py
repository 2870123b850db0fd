"""Times b200gym_clone (env i <- env src[i], uniformly random sources) with bench.py's timing rules: L2 flushed before
every call, one CUDA-event pair per call, median / p10 / p90.  Usage: python scripts/clone_bench.py
[ENV_ID:LOG2N ...] [--calls C].  Prints one JSON line per config (the numbers in DESIGN.md §4.5).

Algorithmic bytes are one read of each source's state and one write of each destination's (2 x n x the unpadded row
bytes); the two-pass scheme (save every env into the scratch snapshot, load the gathered rows) moves more, reported as
moved_bytes."""
import argparse
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
import gym_b200  # noqa: E402
from gym_b200 import _lib  # noqa: E402

# unpadded per-env bytes of a snapshot row (include/b200gym.h): PCG64 record 32 + float64 state + 4 x Box2D record
# words + elapsed 4 + flags 1
STATE_BYTES = {"CartPole-v1": 32 + 4 * 8 + 5, "LunarLander-v2": 32 + 103 * 4 + 5,
               "BipedalWalkerHardcore-v3": 32 + 491 * 4 + 5}


def clone_line(env_id, log2n, calls, dev, flush, peak):
    n = 1 << log2n
    env = gym_b200.vector.make(env_id, n)
    env.reset(seed=0)
    gen = torch.Generator(device=dev).manual_seed(5)
    pool = [torch.randint(0, n, (n,), device=dev, dtype=torch.int64, generator=gen) for _ in range(4)]
    lib, h, st = env._lib, env._handle, env._stream()

    def clone(k):
        _lib.check(lib.b200gym_clone(h, ctypes.c_void_p(pool[k % 4].data_ptr()), st), h)

    for k in range(5):
        clone(k)
    starts = [torch.cuda.Event(enable_timing=True) for _ in range(calls)]
    ends = [torch.cuda.Event(enable_timing=True) for _ in range(calls)]
    torch.cuda.synchronize()
    for k in range(calls):
        flush(k)
        starts[k].record()
        clone(k)
        ends[k].record()
    torch.cuda.synchronize()
    if lib.b200gym_snapshot_index_error(h) != 0:
        raise RuntimeError("clone met an out-of-range source")
    row = env.snapshot_row_bytes
    env.close()
    ms = np.array([s.elapsed_time(e) for s, e in zip(starts, ends)], dtype=np.float64)
    med = float(np.median(ms))
    state = STATE_BYTES[env_id]
    alg, moved = 2 * n * state, 2 * n * (state + row)
    return {"workload": f"{env_id} num_envs=2^{log2n}, clone from uniformly random sources", "gpu": torch.cuda.get_device_name(dev),
            "ms_per_call": med, "ms_per_call_p10": float(np.percentile(ms, 10)),
            "ms_per_call_p90": float(np.percentile(ms, 90)), "calls": calls, "row_bytes": row,
            "state_bytes_per_env": state, "algorithmic_bytes": alg, "hbm_gbs": alg / (med * 1e-3) / 1e9,
            "hbm_frac": alg / (med * 1e-3) / 1e9 / peak, "moved_bytes": moved, "moved_gbs": moved / (med * 1e-3) / 1e9}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("configs", nargs="*", default=["CartPole-v1:20", "LunarLander-v2:16", "BipedalWalkerHardcore-v3:16"])
    p.add_argument("--calls", type=int, default=50)
    args = p.parse_args()
    dev = torch.device("cuda:0")
    flush = bench.L2Flush(torch, dev)
    peak, _ = bench.measured_hbm_peak()
    for cfg in args.configs:
        env_id, log2n = cfg.split(":")
        print(json.dumps(clone_line(env_id, int(log2n), args.calls, dev, flush, peak)), flush=True)


if __name__ == "__main__":
    main()
