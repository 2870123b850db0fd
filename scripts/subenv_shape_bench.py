"""Times the reshaping per-env wrapper chains and the action-stage kernel with bench.py's timing rules -- L2 flushed
before every call, one CUDA-event pair per call on the launch stream, median / p10 / p90.  Usage:
python scripts/subenv_shape_bench.py [--calls C] [--out FILE].  Prints one JSON line for the card (name, power
limit), one per workload (the numbers in DESIGN.md §4.7), then the card again.

Workloads:
  CartPole-v1 at 2^20 envs with FrameStack(4), and with FrameStack(4) + TimeAwareObservation: the chain kernel alone
      (b200gym_subenv_step_io over the last step's outputs), and `step()` with and without the chain;
  Pendulum-v1 at 2^18 envs with RescaleAction(-1, 1) + ClipAction: the action-stage kernel alone
      (b200gym_subenv_actions), and `step()` with and without the stages.
The floor is the kernel's HBM traffic counted from shapes (`chain_bytes`, `action_bytes`) at the data sheet's
3.35 TB/s -- a computed bound, not a measurement.  Terminal rows are written for finishing envs only and are left
out.
"""
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
from gym_b200 import _lib, subenv  # noqa: E402
from scripts.sample_bench import DATASHEET_BPS, card, stats, time_flushed  # noqa: E402


def chain_bytes(d, k, time_aware):
    """Per env-step of FrameStack(k) [+ TimeAwareObservation] over D float32 values: the flags (2), the reward read
    and written (16), the step's row read (4 D), the new frame written (4 D) and the k - 1 older ones read
    (4 D (k - 1)), the head read and written (8), the output row written (4 W), and t read and written (16)."""
    w = k * d + (1 if time_aware else 0)
    return 2 + 16 + 4 * d + 4 * d + 4 * d * (k - 1) + 8 + 4 * w + (16 if time_aware else 0)


def action_bytes(a):
    return 8 * a   # float32 actions read and written


def _line(workload, kernel_ms, nbytes_per_env, n, extra):
    med = float(np.median(kernel_ms)) * 1e-3
    nbytes = nbytes_per_env * n
    return dict({"workload": workload, "kernel": stats(kernel_ms), "bytes_per_env_step": nbytes_per_env,
                 "bytes": nbytes, "achieved_gbs": nbytes / med / 1e9, "of_datasheet_hbm": nbytes / med / DATASHEET_BPS,
                 "floor_us_at_3.35TBps": nbytes / DATASHEET_BPS * 1e6}, **extra)


def frame_stack_line(log2n, stages, calls, flush):
    n = 1 << log2n
    plain = gym_b200.vector.make("CartPole-v1", n, max_episode_steps=200)
    env = gym_b200.vector.make("CartPole-v1", n, max_episode_steps=200, wrappers=stages)
    gen = torch.Generator(device=env.device).manual_seed(0)
    acts = [torch.randint(0, 2, (n,), device=env.device, generator=gen) for _ in range(8)]
    plain.reset(seed=0)
    env.reset(seed=0)
    step_ms = time_flushed(lambda k: plain.step(acts[k % 8]), calls, flush)
    both_ms = time_flushed(lambda k: env.step(acts[k % 8]), calls, flush)
    out = env._out[env._flip]
    lib, h, st = env._lib, env._handle, env._stream()

    def ptr(k):
        return ctypes.c_void_p(out[k].data_ptr()) if k in out else None

    def chain(k):
        _lib.check(lib.b200gym_subenv_step_io(h, ptr("raw_obs"), ptr("obs"), ptr("reward"), ptr("terminated"),
                                              ptr("truncated"), ptr("raw_final_obs"), ptr("final_obs"),
                                              ptr("final_obs64"), ptr("ep_r"), ptr("ep_l"), st), h)

    chain_ms = time_flushed(chain, calls, flush)
    c = env._chain
    k = c.stack[0]
    res = _line(f"CartPole-v1 num_envs=2^{log2n}, chain {[repr(s) for s in stages]}, output {c.obs_shape}", chain_ms,
                chain_bytes(plain.obs_dim, k, c.time_aware), n,
                {"calls": calls, "step": stats(step_ms), "step+chain": stats(both_ms)})
    plain.close()
    env.close()
    return res


def action_line(log2n, stages, calls, flush):
    n = 1 << log2n
    plain = gym_b200.vector.make("Pendulum-v1", n, max_episode_steps=200)
    env = gym_b200.vector.make("Pendulum-v1", n, max_episode_steps=200, wrappers=stages)
    gen = torch.Generator(device=env.device).manual_seed(0)
    acts = [torch.rand((n, 1), device=env.device, generator=gen) * 3 - 1.5 for _ in range(8)]
    plain.reset(seed=0)
    env.reset(seed=0)
    step_ms = time_flushed(lambda k: plain.step(acts[k % 8]), calls, flush)
    both_ms = time_flushed(lambda k: env.step(acts[k % 8]), calls, flush)
    lib, h, st = env._lib, env._handle, env._stream()
    dst = torch.empty_like(acts[0])

    def kernel(k):
        _lib.check(lib.b200gym_subenv_actions(h, ctypes.c_void_p(acts[k % 8].data_ptr()),
                                              ctypes.c_void_p(dst.data_ptr()), st), h)

    kernel_ms = time_flushed(kernel, calls, flush)
    res = _line(f"Pendulum-v1 num_envs=2^{log2n}, action stages {[repr(s) for s in stages]}", kernel_ms,
                action_bytes(env.act_dim), n, {"calls": calls, "step": stats(step_ms), "step+stages": stats(both_ms)})
    plain.close()
    env.close()
    return res


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--calls", type=int, default=200)
    p.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("subenv_shape_bench.py needs a CUDA device")
    torch.cuda.set_device(0)
    lines = [card()]
    print(json.dumps(lines[-1]), flush=True)
    flush = bench.L2Flush(torch, torch.device("cuda:0"))
    for stages in ([subenv.FrameStack(4)], [subenv.FrameStack(4), subenv.TimeAwareObservation()]):
        lines.append(frame_stack_line(20, stages, args.calls, flush))
        print(json.dumps(lines[-1]), flush=True)
    lines.append(action_line(18, [subenv.RescaleAction(-1, 1), subenv.ClipAction()], args.calls, flush))
    print(json.dumps(lines[-1]), flush=True)
    lines.append(card())
    print(json.dumps(lines[-1]), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(json.dumps(x) for x in lines) + "\n")


if __name__ == "__main__":
    main()
