"""Time per batch step of collecting on-policy experience with a stochastic tanh MLP policy, four ways (DESIGN §4.15):
one replay of a graph of T eager steps (``nn.Sequential`` with ``nn.Tanh``, or ``torch.baddbmm`` and ``torch.tanh`` per
layer for per-env parameters, then a Gumbel-max sample for Discrete kinds or a Gaussian sample for Box kinds, then
``step()``), ``rollout_mlp_noisy(activation="tanh")`` on noise drawn in advance, ``rollout_mlp_noisy`` with the same
parameters and noise under ReLU (the cost of tanh is the ratio of the two), and ``rollout_mlp(activation="tanh",
summary=True)``.  LunarLander cannot be captured, so its first arm runs the T eager steps instead.  The eager arms run
through cuBLAS, so their actions are not bit for bit those of the rollouts; they are what a user would otherwise write.

Timing follows rollout_bench.py's rules: every shape is warmed up, L2 is flushed before each timed call (bench.py's
L2Flush), each timed call gets one CUDA-event pair, and the arms alternate, round by round, in a rotating order.  Each
line gives the median over the rounds and the spread (min, max) per arm, in µs per batch step (one step of all N envs),
and, from shapes (``noisy_bytes``, not measured), the HBM bytes/s the tanh ``rollout_mlp_noisy`` achieves.  Prints the
card (name, power limit, max SM clock) before and after.
Usage: python scripts/rollout_mlp_tanh_bench.py [--rounds R] [--out FILE]
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

import gym_b200  # noqa: E402
from bench import L2Flush  # noqa: E402
from rollout_bench import timed  # noqa: E402
from rollout_mlp_bench import HBM_PEAK, flops, layers, param_count, unpack  # noqa: E402
from rollout_mlp_noisy_bench import STD, draw_noise, noisy_bytes  # noqa: E402
from sample_bench import card  # noqa: E402

ROLLOUTS = ("tanh_rollout_mlp_noisy", "relu_rollout_mlp_noisy", "tanh_rollout_mlp_summary")
# (env_id, log2 envs, T, hidden, per-env parameters, arms): §4.14's rows
WORKLOADS = [
    ("CartPole-v1", 20, 64, (64, 64), False, ("graph_replay",) + ROLLOUTS),
    ("Pendulum-v1", 18, 64, (64, 64), False, ("graph_replay",) + ROLLOUTS),
    ("CartPole-v1", 16, 64, (64, 64), True, ("graph_replay",) + ROLLOUTS),
    ("LunarLander-v2", 16, 8, (64, 64), False, ("eager",) + ROLLOUTS),
]


def run(env_id, log2n, T, hidden, per_env, arms_wanted, rounds, flush):
    n = 1 << log2n
    envs = {k: gym_b200.vector.make(env_id, n, device=0) for k in arms_wanted}
    obs = {}
    for i, (k, e) in enumerate(envs.items()):
        obs[k] = e.reset(seed=i)[0]
    e0 = next(iter(envs.values()))
    K = int(e0.single_action_space.n if e0.discrete else e0.act_dim)
    torch.manual_seed(0)
    mods = []
    for j, (i, o) in enumerate(layers(e0, hidden)):
        mods += [torch.nn.Linear(i, o)] + ([torch.nn.Tanh()] if j < len(hidden) else [])
    net = torch.nn.Sequential(*mods).to("cuda:0")
    vec = torch.nn.utils.parameters_to_vector(net.parameters()).detach()
    params = (vec + 0.05 * torch.randn(n, vec.numel(), device="cuda:0")).contiguous() if per_env else vec.contiguous()
    views = unpack(e0, params, hidden) if per_env else None
    noise = draw_noise((T, n, K), e0.discrete)

    def forward(x):
        if not per_env:
            return net(x)
        x = x.unsqueeze(2)
        for j, (w, b) in enumerate(views):
            x = torch.baddbmm(b, w, x)
            if j < len(hidden):
                x = torch.tanh(x)
        return x.squeeze(2)

    def loop(k):
        e = envs[k]
        o = obs[k]
        with torch.no_grad():
            for _ in range(T):
                z = forward(o)
                a = (z + draw_noise(z.shape, True)).argmax(dim=1) if e.discrete else z + STD * torch.randn_like(z)
                o = e.step(a)[0]
        obs[k] = o

    arms = {}
    if "eager" in envs:
        arms["eager"] = lambda: loop("eager")
    if "graph_replay" in envs:
        loop("graph_replay")   # warm the step path and cuBLAS before the capture
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            loop("graph_replay")
        arms["graph_replay"] = graph.replay
    arms["tanh_rollout_mlp_noisy"] = lambda: envs["tanh_rollout_mlp_noisy"].rollout_mlp_noisy(
        params, hidden, noise, activation="tanh")
    arms["relu_rollout_mlp_noisy"] = lambda: envs["relu_rollout_mlp_noisy"].rollout_mlp_noisy(params, hidden, noise)
    arms["tanh_rollout_mlp_summary"] = lambda: envs["tanh_rollout_mlp_summary"].rollout_mlp(
        params, hidden, T, summary=True, activation="tanh")
    for fn in arms.values():   # warm-up
        fn()
    torch.cuda.synchronize()
    ms = {k: [] for k in arms}
    names = list(arms)
    for r in range(rounds):
        for j in range(len(names)):
            k = names[(r + j) % len(names)]
            ms[k].append(timed(arms[k], flush, r * len(names) + j))
    out = {"env_id": env_id, "log2_envs": log2n, "T": T, "hidden": list(hidden),
           "params": "per_env" if per_env else "shared", "P": param_count(e0, hidden), "K": K, "rounds": rounds}
    for k, v in ms.items():
        v = np.asarray(v) * 1e3 / T   # µs per batch step
        out[k + "_us_per_batch_step"] = {"median": round(float(np.median(v)), 2), "min": round(float(v.min()), 2),
                                         "max": round(float(v.max()), 2)}
    out["flops_per_env_step_from_shapes"] = flops(e0, hidden)
    nbytes = noisy_bytes(e0, T, hidden, per_env)
    sec = out["tanh_rollout_mlp_noisy_us_per_batch_step"]["median"] * 1e-6
    out["rollout_mlp_noisy_bytes_per_env_step_from_shapes"] = round(nbytes, 2)
    out["tanh_rollout_mlp_noisy_tb_per_s"] = round(n * nbytes / sec / 1e12, 3)
    out["tanh_rollout_mlp_noisy_share_of_hbm_peak"] = round(n * nbytes / sec / HBM_PEAK, 4)
    base = "graph_replay" if "graph_replay" in ms else "eager"
    for a in ("tanh_rollout_mlp_noisy", "tanh_rollout_mlp_summary"):
        out[f"{a}_speedup_vs_{base}"] = round(out[base + "_us_per_batch_step"]["median"] /
                                              out[a + "_us_per_batch_step"]["median"], 3)
    out["tanh_over_relu_rollout_mlp_noisy"] = round(out["tanh_rollout_mlp_noisy_us_per_batch_step"]["median"] /
                                                    out["relu_rollout_mlp_noisy_us_per_batch_step"]["median"], 3)
    for e in envs.values():
        e.close()
    arms.clear()
    torch.cuda.empty_cache()
    return out


def main():
    p = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    p.add_argument("--rounds", type=int, default=5)
    p.add_argument("--out", default=None, help="also write the lines to this JSON-lines file")
    args = p.parse_args()
    assert torch.cuda.is_available(), "rollout_mlp_tanh_bench.py measures on the GPU"
    assert args.rounds >= 3
    flush = L2Flush(torch, torch.device("cuda:0"))
    lines = [{"card": card()}]
    print(json.dumps(lines[0]), flush=True)
    for w in WORKLOADS:
        lines.append(run(*w, args.rounds, flush))
        print(json.dumps(lines[-1]), flush=True)
    lines.append({"card": card()})
    print(json.dumps(lines[-1]), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            f.writelines(json.dumps(x) + "\n" for x in lines)


if __name__ == "__main__":
    main()
