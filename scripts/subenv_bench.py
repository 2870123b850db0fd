"""Times the per-env wrapper chain (subenv_step_kernel) against the step it follows, with bench.py's timing rules -- L2
flushed before every call, one CUDA-event pair per call on the launch stream, median / p10 / p90.  Usage:
python scripts/subenv_bench.py [ENV_ID:LOG2N ...] [--calls C].  Prints one JSON line for the card, then one per config
(the numbers in DESIGN.md §4.7), then the card again.

Then, per --host config, the numpy backend end to end (host actions in, results in page-locked host memory), with
and without the chain.

Per config, with the PPO chain (RecordEpisodeStatistics, ClipAction on Box kinds, NormalizeObservation,
ClipObservation(-10, 10), NormalizeReward(0.99), ClipReward(-10, 10)):
  step        `step()` of the chain-less env
  step+chain  `step()` of the wrapped env (ClipAction launch, step, chain launch)
  chain       the chain kernel alone (b200gym_subenv_step over the last outputs)
The floor is the chain's HBM traffic counted from shapes at the data sheet's 3.35 TB/s -- a computed bound, not a
measurement: per env-step it reads and writes obs (4 D), reward (8), the observation statistics ((2 D + 1) x 8), the
reward statistics (4 x 8) and the episode accumulators (4 + 4), and reads the two flags (2).  Terminal rows and
episode fields are written for finishing envs only and are left out.
"""
import argparse
import ctypes
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
import gym_b200  # noqa: E402
from gym_b200 import _lib  # noqa: E402
from oracle.gen_subenv_fixtures import chains  # noqa: E402
from scripts.sample_bench import DATASHEET_BPS, card, stats, time_flushed  # noqa: E402


def chain_bytes(d):
    return 2 * (4 * d + 8 + (2 * d + 1) * 8 + 4 * 8 + 4 + 4) + 2


def config_line(env_id, log2n, calls, flush):
    n = 1 << log2n
    plain = gym_b200.vector.make(env_id, n, max_episode_steps=200)
    stages = chains(not plain.discrete)["ppo"]
    env = gym_b200.vector.make(env_id, n, max_episode_steps=200, wrappers=stages)
    gen = torch.Generator(device=env.device).manual_seed(0)
    if plain.discrete:
        acts = [torch.randint(0, plain.single_action_space.n, (n,), device=env.device, generator=gen) for _ in range(8)]
    else:
        hi = float(plain.single_action_space.high[0])
        acts = [(torch.rand((n, plain.act_dim), device=env.device, generator=gen) * 3 - 1.5) * hi for _ in range(8)]
    plain.reset(seed=0)
    env.reset(seed=0)
    step_ms = time_flushed(lambda k: plain.step(acts[k % 8]), calls, flush)
    both_ms = time_flushed(lambda k: env.step(acts[k % 8]), calls, flush)
    out = env._out[env._flip]
    lib, h, st = env._lib, env._handle, env._stream()

    def ptr(k):
        return ctypes.c_void_p(out[k].data_ptr()) if k in out else None

    def chain(k):
        _lib.check(lib.b200gym_subenv_step(h, ptr("obs"), ptr("reward"), ptr("terminated"), ptr("truncated"),
                                           ptr("final_obs"), ptr("final_obs64"), ptr("ep_r"), ptr("ep_l"), st), h)

    chain_ms = time_flushed(chain, calls, flush)
    nbytes = chain_bytes(plain.obs_dim) * n
    med = float(np.median(chain_ms)) * 1e-3
    plain.close()
    env.close()
    return {"workload": f"{env_id} num_envs=2^{log2n}, PPO chain {[repr(s) for s in stages]}", "calls": calls,
            "step": stats(step_ms), "step+chain": stats(both_ms), "chain_kernel": stats(chain_ms),
            "chain_bytes_per_env_step": chain_bytes(plain.obs_dim), "chain_bytes": nbytes,
            "chain_achieved_gbs": nbytes / med / 1e9, "chain_of_datasheet_hbm": nbytes / med / DATASHEET_BPS,
            "chain_floor_us_at_3.35TBps": nbytes / DATASHEET_BPS * 1e6}


def host_line(env_id, log2n, steps):
    """The numpy backend end to end: host actions in, every result in page-locked host memory (b200gym_step_host
    synchronises), wall clock per step over `steps` steps, with and without the PPO chain.  The chain kernel reads
    and writes the mapped host buffers in place."""
    n = 1 << log2n
    probe = gym_b200.vector.make(env_id, 1)
    stages = chains(not probe.discrete)["ppo"]
    probe.close()
    res = {"workload": f"{env_id} num_envs=2^{log2n}, numpy backend, per-step wall time over {steps} steps"}
    for name, wrap in (("step", False), ("step+chain", True)):
        env = gym_b200.vector.make(env_id, n, max_episode_steps=200, backend="numpy", copy=False, dense_infos=True,
                                   wrappers=stages if wrap else None)
        rng = np.random.default_rng(0)
        if env.discrete:
            acts = [rng.integers(0, env.single_action_space.n, size=n) for _ in range(4)]
        else:
            acts = [rng.uniform(-3, 3, size=(n, env.act_dim)).astype(np.float32) for _ in range(4)]
        env.reset(seed=0)
        for k in range(10):
            env.step(acts[k % 4])
        t0 = time.perf_counter()
        for k in range(steps):
            env.step(acts[k % 4])
        res[name + " ms"] = (time.perf_counter() - t0) / steps * 1e3
        env.close()
    return res


def main():
    p = argparse.ArgumentParser()
    p.add_argument("configs", nargs="*", default=["CartPole-v1:20", "Pendulum-v1:18", "LunarLander-v2:16"])
    p.add_argument("--calls", type=int, default=200)
    p.add_argument("--host", nargs="*", default=["CartPole-v1:20", "Pendulum-v1:18"],
                   help="ENV_ID:LOG2N configs timed end to end on the numpy backend")
    p.add_argument("--host-steps", type=int, default=200)
    p.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("subenv_bench.py needs a CUDA device")
    torch.cuda.set_device(0)
    lines = [card()]
    print(json.dumps(lines[-1]), flush=True)
    flush = bench.L2Flush(torch, torch.device("cuda:0"))
    for cfg in args.configs:
        env_id, log2n = cfg.split(":")
        lines.append(config_line(env_id, int(log2n), args.calls, flush))
        print(json.dumps(lines[-1]), flush=True)
    for cfg in args.host:
        env_id, log2n = cfg.split(":")
        lines.append(host_line(env_id, int(log2n), args.host_steps))
        print(json.dumps(lines[-1]), flush=True)
    lines.append(card())
    print(json.dumps(lines[-1]), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(json.dumps(x) for x in lines) + "\n")


if __name__ == "__main__":
    main()
