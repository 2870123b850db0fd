"""Time per batch step of one PPO collection step with normalised observations and rewards, a (64, 64) tanh actor and
critic, obs_norm, reward_norm and both clips at 10 (DESIGN §4.18):

1. ``graph_replay``: one replay of a graph of T eager steps (the observation normalised in torch, actor and critic
   ``nn.Sequential`` on it, a Gumbel-max sample for Discrete kinds or a Gaussian sample for Box kinds, ``step()``, the
   critic on that step's normalised ``infos["final_observation"]``), then the GAE loop in torch on the scaled rewards:
   the only way to run this collection without the keywords;
2. ``ac_norm``: ``rollout_actor_critic`` with ``obs_norm``, ``reward_norm`` and the clips;
3. ``ac_raw``: ``rollout_actor_critic`` without them;
4. ``noisy_norm`` / ``noisy_raw``: ``rollout_mlp_noisy`` with and without ``obs_norm`` and ``clip_obs``.

The noise of arms 2-4 is drawn in advance.  LunarLanderContinuous cannot be captured, so its first arm runs the T eager
steps instead.  The torch arm runs through cuBLAS, so its values are not bit for bit those of the rollout; it is what a
user would otherwise write.

Timing follows rollout_actor_critic_bench.py's rules: every shape is warmed up, L2 is flushed before each timed call
(bench.py's L2Flush), each timed call gets one CUDA-event pair, and the arms alternate, round by round, in a rotating
order.  Each line gives the median over the rounds and the spread (min, max) per arm, in µs per batch step (one step of
all N envs).  Prints the card (name, power limit, max SM clock) before and after.
Usage: python scripts/rollout_norm_bench.py [--rounds R] [--out FILE]
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
from rollout_actor_critic_bench import GAE_LAMBDA, GAMMA, gae_torch, mlp  # noqa: E402
from rollout_bench import timed  # noqa: E402
from rollout_mlp_noisy_bench import STD, draw_noise  # noqa: E402
from sample_bench import card  # noqa: E402

EPS, CLIP = 1e-8, 10.0
NORMED = ("ac_norm", "ac_raw", "noisy_norm", "noisy_raw")
# (env_id, log2 envs, T, hidden, first arm)
WORKLOADS = [
    ("CartPole-v1", 20, 64, (64, 64), "graph_replay"),
    ("Pendulum-v1", 18, 64, (64, 64), "graph_replay"),
    ("MountainCarContinuous-v0", 18, 64, (64, 64), "graph_replay"),
    ("Acrobot-v1", 18, 64, (64, 64), "graph_replay"),
    ("LunarLanderContinuous-v2", 16, 8, (64, 64), "eager"),
]


def run(env_id, log2n, T, hidden, first_arm, rounds, flush):
    n = 1 << log2n
    names = (first_arm,) + NORMED
    envs = {k: gym_b200.vector.make(env_id, n, device=0) for k in names}
    obs = {k: e.reset(seed=i)[0] for i, (k, e) in enumerate(envs.items())}
    e0 = envs[first_arm]
    K, D = int(e0.single_action_space.n if e0.discrete else e0.act_dim), e0.obs_dim
    torch.manual_seed(0)
    actor, critic = mlp(D, hidden, K), mlp(D, hidden, 1)
    pa = torch.nn.utils.parameters_to_vector(actor.parameters()).detach().contiguous()
    pc = torch.nn.utils.parameters_to_vector(critic.parameters()).detach().contiguous()
    noise = draw_noise((T, n, K), e0.discrete)
    f64 = dict(dtype=torch.float64, device="cuda:0")
    mean, var = 0.1 * torch.randn(D, **f64), torch.rand(D, **f64) + 0.5
    rvar = torch.rand(1, **f64) + 0.5

    def norm(o):
        return ((o.double() - mean) / torch.sqrt(var + EPS)).float().clamp(-CLIP, CLIP)

    def eager(k):
        e, o = envs[k], obs[k]
        values, vf, rews, tes, trs = [], [], [], [], []
        with torch.no_grad():
            for _ in range(T):
                x = norm(o)
                z = actor(x)
                values.append(critic(x)[:, 0])
                a = (z + draw_noise(z.shape, True)).argmax(dim=1) if e.discrete else z + STD * torch.randn_like(z)
                o, r, te, tr, info = e.step(a)
                vf.append(critic(norm(info["final_observation"]))[:, 0])
                rews.append(r)
                tes.append(te)
                trs.append(tr)
            values.append(critic(norm(o))[:, 0])
            rew = (torch.stack(rews) / torch.sqrt(rvar + EPS)).float().clamp(-CLIP, CLIP)
            adv = gae_torch(rew, torch.stack(tes), torch.stack(trs), torch.stack(values), torch.stack(vf))
        obs[k] = o
        return adv

    arms = {}
    if first_arm == "eager":
        arms["eager"] = lambda: eager("eager")
    else:
        eager("graph_replay")   # warm the step path and cuBLAS before the capture
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            eager("graph_replay")
        arms["graph_replay"] = g.replay
    kw = dict(gamma=GAMMA, gae_lambda=GAE_LAMBDA, activation="tanh")
    obs_kw = dict(obs_norm=(mean, var), norm_epsilon=EPS, clip_obs=CLIP)
    arms["ac_norm"] = lambda: envs["ac_norm"].rollout_actor_critic(pa, pc, hidden, noise, **kw, **obs_kw,
                                                                   reward_norm=rvar, clip_reward=CLIP)
    arms["ac_raw"] = lambda: envs["ac_raw"].rollout_actor_critic(pa, pc, hidden, noise, **kw)
    arms["noisy_norm"] = lambda: envs["noisy_norm"].rollout_mlp_noisy(pa, hidden, noise, activation="tanh", **obs_kw)
    arms["noisy_raw"] = lambda: envs["noisy_raw"].rollout_mlp_noisy(pa, hidden, noise, activation="tanh")
    for fn in arms.values():   # warm-up
        fn()
    torch.cuda.synchronize()
    ms = {k: [] for k in arms}
    order = list(arms)
    for r in range(rounds):
        for j in range(len(order)):
            k = order[(r + j) % len(order)]
            ms[k].append(timed(arms[k], flush, r * len(order) + j))
    out = {"env_id": env_id, "log2_envs": log2n, "T": T, "hidden": list(hidden), "activation": "tanh",
           "clip_obs": CLIP, "clip_reward": CLIP, "rounds": rounds}
    for k, v in ms.items():
        v = np.asarray(v) * 1e3 / T   # µs per batch step
        out[k + "_us_per_batch_step"] = {"median": round(float(np.median(v)), 2), "min": round(float(v.min()), 2),
                                         "max": round(float(v.max()), 2)}
    med = {k: out[k + "_us_per_batch_step"]["median"] for k in ms}
    out["ac_norm_speedup_vs_" + first_arm] = round(med[first_arm] / med["ac_norm"], 3)
    out["ac_norm_over_ac_raw"] = round(med["ac_norm"] / med["ac_raw"], 3)
    out["noisy_norm_over_noisy_raw"] = round(med["noisy_norm"] / med["noisy_raw"], 3)
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
    assert torch.cuda.is_available(), "rollout_norm_bench.py measures on the GPU"
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
