"""Compute floor of the CartPole step: 2^19 envs (about 35 MB of state, outputs and actions, under H100's 50 MB L2)
stepped with one action tensor and no L2 flush, so after the first steps every access hits L2 and what is left is the
kernel's arithmetic and issue.  One CUDA-event pair per step behind a short device sleep (the Python step call takes
about as long as the kernel at this size, so a back-to-back loop, or an event pair on an idle device, would time the
host).  Also times 2^23 envs back to back (there the GPU is the
bottleneck and every write-back falls inside the timed region).
Prints one JSON line; B200GYM_KERNEL / B200GYM_LIB select the kernel and the build as for bench.py."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import gym_b200  # noqa: E402


def per_step_median_us(log2n, steps, warmup):
    n = 1 << log2n
    env = gym_b200.vector.make("CartPole-v1", n)
    env.reset(seed=0)
    act = torch.randint(0, 2, (n,), device="cuda", dtype=torch.int64,
                        generator=torch.Generator(device="cuda").manual_seed(1))
    for _ in range(warmup):
        env.step(act)
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
    torch.cuda.synchronize()
    for s, e in ev:
        torch.cuda._sleep(200000)   # ~0.1 ms of device time: the launch is queued before the start event fires
        s.record()
        env.step(act)
        e.record()
    torch.cuda.synchronize()
    env.close()
    return float(np.median([s.elapsed_time(e) * 1e3 for s, e in ev]))


def back_to_back_us(log2n, steps, warmup):
    n = 1 << log2n
    env = gym_b200.vector.make("CartPole-v1", n)
    env.reset(seed=0)
    act = torch.randint(0, 2, (n,), device="cuda", dtype=torch.int64,
                        generator=torch.Generator(device="cuda").manual_seed(1))
    for _ in range(warmup):
        env.step(act)
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    best = float("inf")
    for _ in range(5):
        torch.cuda.synchronize()
        t0.record()
        for _ in range(steps):
            env.step(act)
        t1.record()
        torch.cuda.synchronize()
        best = min(best, t0.elapsed_time(t1) * 1e3 / steps)
    env.close()
    return best


if __name__ == "__main__":
    l2 = per_step_median_us(19, 400, 50)
    b2b = back_to_back_us(23, 40, 5)
    print(json.dumps({"kernel": os.environ.get("B200GYM_KERNEL", "default"),
                      "l2_resident_2p19_us": l2, "l2_resident_us_per_2p20": 2 * l2,
                      "back_to_back_2p23_us": b2b, "back_to_back_us_per_2p20": b2b / 8}))
