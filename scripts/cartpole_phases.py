"""Where kernel B's time per tile goes: the CartPole step kernel (step_kernel_persistent_bulk) built with
-DB200_PHASE_CLOCKS, which adds up clock() cycles per phase.

Compute warps (lane 0 of each): waiting on the stage's `full` barrier, advance_env (inputs from the stage, the
lookahead's record prefetch, dynamics, TimeLimit, results into the stage), waiting for the PCG64 records of the
finishing envs (`record_wait`), the resets through the stage (`reset`), and the proxy fence + `done` arrive with the
final-observation and record stores after it.  The copy thread: waiting on `done`,
issuing the tile's bulk stores, waiting until they have read the stage, issuing the refill's bulk loads, and the final
wait until the last stores have read their stage.  Every CTA also stamps %globaltimer when its last compute warp
leaves the loop and when the CTA exits, relative to the CTA's start.  The instrumented build spills 8 to 16 bytes;
the default build spills none.

Builds the variant into a temporary directory (or takes --lib) and loads it through B200GYM_LIB.  Prints one JSON
line per shape: bench.py's (2^20 envs, L2 flushed before every step, median over steps) and 2^23 envs stepped back to
back (mean over steps).  Each bucket is given as a share of the loop time of its side and in cycles per tile."""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

COMPUTE = ["full_wait", "advance_env", "record_wait", "reset", "fence_arrive"]
COPY = ["done_wait", "store_issue", "wait_read", "load_issue", "final_wait_read"]
N_BUCKETS = 13   # enum PhaseBucket in csrc/b200gym.cu
N_STAMPS = 3     # g_phase_ns: CTA start, loop end, exit
MAX_CTAS = 4096


def build_variant(out_dir):
    from gym_b200 import build
    lib = os.path.join(out_dir, "libb200gym_phases.so")
    cmd = ([build._nvcc()] + build.NVCC_FLAGS + ["-DB200_PHASE_CLOCKS", "-o", lib] +
           [f for f in build.sources() if f.endswith(".cu")])
    subprocess.run(cmd, check=True)
    return lib


def read_clocks(lib, clear):
    cyc = (ctypes.c_ulonglong * N_BUCKETS)()
    ns = (ctypes.c_ulonglong * (MAX_CTAS * N_STAMPS))()
    if lib.b200gym_phase_clocks(cyc, ns, int(clear)) != 0:
        raise RuntimeError("b200gym_phase_clocks failed")
    c = np.array(cyc[:], dtype=np.float64)
    t = np.array(ns[:], dtype=np.float64).reshape(MAX_CTAS, N_STAMPS)
    return c, t[t[:, 0] > 0]


def summarise(c, t):
    """one launch's (or a sum of launches') counters -> shares, cycles per tile and CTA time stamps"""
    tiles = max(c[6], 1.0)
    comp = {k: c[b] for b, k in enumerate(COMPUTE)}
    copy = {k: c[7 + b] for b, k in enumerate(COPY)}
    comp_loop, copy_loop = max(c[5], 1.0), max(c[12], 1.0)
    out = {
        "compute_share": {k: v / comp_loop for k, v in comp.items()},
        "compute_cycles_per_warp_tile": {k: v / tiles for k, v in comp.items()},
        "compute_loop_cycles_per_warp_tile": comp_loop / tiles,
        # the copy thread handles one tile per 8 compute warp-tiles
        "copy_share": {k: v / copy_loop for k, v in copy.items() if k != "final_wait_read"},
        "copy_cycles_per_tile": {k: v / (tiles / 8) for k, v in copy.items()},
    }
    if len(t):
        rel = t[:, 1:] - t[:, :1]
        start_spread = t[:, 0] - t[:, 0].min()
        out["cta_us"] = {
            "start_spread_max": float(start_spread.max()) / 1e3,
            "loop_end_mean": float(rel[:, 0].mean()) / 1e3, "loop_end_max": float(rel[:, 0].max()) / 1e3,
            "exit_mean": float(rel[:, 1].mean()) / 1e3, "exit_max": float(rel[:, 1].max()) / 1e3,
        }
    return out


def median_of(dicts):
    """element-wise median of a list of nested dicts of floats"""
    first = dicts[0]
    if isinstance(first, dict):
        return {k: median_of([d[k] for d in dicts]) for k in first}
    return float(np.median(dicts))


def run(lib, torch, gym_b200, log2n, steps, warmup, flushed):
    n = 1 << log2n
    dev = torch.device("cuda")
    env = gym_b200.vector.make("CartPole-v1", n)
    env.reset(seed=0)
    gen = torch.Generator(device=dev).manual_seed(1)
    pool = torch.randint(0, 2, (16, n), device=dev, dtype=torch.int64, generator=gen)
    for k in range(warmup):
        env.step(pool[k % 16])
    torch.cuda.synchronize()
    read_clocks(lib, True)
    if flushed:
        buf = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
        rd = torch.zeros(32 << 20, dtype=torch.int64, device=dev)
        sink = torch.zeros(1, dtype=torch.int64, device=dev)
        per_step = []
        for k in range(steps):
            buf.fill_(k & 0xFF)   # as bench.py: 256 MiB written, then 256 MiB read so that L2 holds clean lines
            torch.sum(rd, dim=0, keepdim=True, out=sink)
            env.step(pool[k % 16])
            torch.cuda.synchronize()
            per_step.append(summarise(*read_clocks(lib, True)))
        res = median_of(per_step)
    else:
        for k in range(steps):
            env.step(pool[k % 16])
        torch.cuda.synchronize()
        c, _ = read_clocks(lib, True)
        res = summarise(c / steps, np.zeros((0, N_STAMPS)))
    env.close()
    res.update({"log2_envs": log2n, "steps": steps, "l2_flushed": flushed})
    return res


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--lib", help="an already built -DB200_PHASE_CLOCKS library (default: build one from the tree)")
    p.add_argument("--label", default="")
    p.add_argument("--steps", type=int, default=200)
    args = p.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        lib_path = args.lib or build_variant(tmp)
        os.environ["B200GYM_LIB"] = lib_path
        import torch
        import gym_b200
        from gym_b200 import _lib
        _lib.LIB_PATH = lib_path   # the package may have been imported (by the build) before B200GYM_LIB was set
        lib = _lib.load()
        lib.b200gym_phase_clocks.restype = ctypes.c_int
        lib.b200gym_phase_clocks.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
        for log2n, flushed, warmup in ((20, True, 100), (23, False, 10)):
            line = run(lib, torch, gym_b200, log2n, args.steps if flushed else max(args.steps // 5, 10), warmup, flushed)
            line["label"] = args.label
            print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
