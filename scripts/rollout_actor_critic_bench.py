"""Time per batch step of one on-policy collection step of PPO / A2C with a (64, 64) tanh actor and critic, four ways
(DESIGN §4.17):

1. ``graph_replay``: one replay of a graph of T eager steps (actor and critic ``nn.Sequential``, a Gumbel-max sample for
   Discrete kinds or a Gaussian sample for Box kinds, ``step()``, and the critic on that step's
   ``infos["final_observation"]``), then the GAE loop in torch;
2. ``noisy_then_torch``: one replay of a graph of ``rollout_mlp_noisy``, then the critic ``nn.Sequential`` over the
   T + 1 stacked input observations and the T steps of final observations (one slice at a time, as the activations of
   all T * N rows at once do not fit), then the GAE loop in torch;
3. ``rollout_actor_critic``;
4. ``rollout_mlp_noisy`` alone: what the critic and the advantages cost is arm 3 minus arm 4.

The noise of arms 2-4 is drawn in advance.  LunarLander cannot be captured, so its first arm runs the T eager steps
instead, and it has no second arm.  The torch arms run through cuBLAS, so their values are not bit for bit those of the
rollout; they are what a user would otherwise write.

Timing follows rollout_bench.py's rules: every shape is warmed up, L2 is flushed before each timed call (bench.py's
L2Flush), each timed call gets one CUDA-event pair, and the arms alternate, round by round, in a rotating order.  Each
line gives the median over the rounds and the spread (min, max) per arm, in µs per batch step (one step of all N envs),
and, from shapes (not measured), the HBM bytes per env-step of ``rollout_actor_critic``'s two launches.  Prints the card
(name, power limit, max SM clock) before and after.
Usage: python scripts/rollout_actor_critic_bench.py [--rounds R] [--out FILE]
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
from rollout_mlp_bench import HBM_PEAK  # noqa: E402
from rollout_mlp_noisy_bench import STD, draw_noise, noisy_bytes  # noqa: E402
from sample_bench import card  # noqa: E402

GAMMA, GAE_LAMBDA = 0.99, 0.95
ALL = ("graph_replay", "noisy_then_torch", "rollout_actor_critic", "rollout_mlp_noisy")
# (env_id, log2 envs, T, hidden, arms)
WORKLOADS = [
    ("CartPole-v1", 20, 64, (64, 64), ALL),
    ("Pendulum-v1", 18, 64, (64, 64), ALL),
    ("Acrobot-v1", 18, 64, (64, 64), ALL),
    ("LunarLander-v2", 16, 8, (64, 64), ("eager", "rollout_actor_critic", "rollout_mlp_noisy")),
]


def ac_bytes(env, T, hidden):
    """HBM bytes per env-step of rollout_actor_critic, from shapes: rollout_mlp_noisy's (shared policy), plus the value
    and the advantage slot (8 B; the final-observation value is stored only where a step truncated) in the rollout
    kernel, plus gae_kernel's reward, two flags, value and advantage (18 B)."""
    return noisy_bytes(env, T, hidden, False) + 8 + 18


def mlp(D, hidden, K):
    sizes = [D] + list(hidden) + [K]
    mods = []
    for j, (i, o) in enumerate(zip(sizes[:-1], sizes[1:])):
        mods += [torch.nn.Linear(i, o)] + ([torch.nn.Tanh()] if j < len(sizes) - 2 else [])
    return torch.nn.Sequential(*mods).to("cuda:0")


def gae_torch(rew, te, tr, values, vf):
    """The GAE loop a user writes: CleanRL's, with the final-observation bootstrap of a time-limit end."""
    T = rew.shape[0]
    adv = torch.empty_like(values[:-1])
    last = torch.zeros_like(values[0])
    for t in reversed(range(T)):
        nextv = torch.where(te[t], 0.0, torch.where(tr[t], vf[t], values[t + 1]))
        delta = rew[t].float() + GAMMA * nextv - values[t]
        last = delta + (GAMMA * GAE_LAMBDA) * (~(te[t] | tr[t])) * last
        adv[t] = last
    return adv


def run(env_id, log2n, T, hidden, arms_wanted, rounds, flush):
    n = 1 << log2n
    envs = {k: gym_b200.vector.make(env_id, n, device=0) for k in arms_wanted}
    obs = {}
    for i, (k, e) in enumerate(envs.items()):
        obs[k] = e.reset(seed=i)[0]
    e0 = next(iter(envs.values()))
    K = int(e0.single_action_space.n if e0.discrete else e0.act_dim)
    torch.manual_seed(0)
    actor, critic = mlp(e0.obs_dim, hidden, K), mlp(e0.obs_dim, hidden, 1)
    pa = torch.nn.utils.parameters_to_vector(actor.parameters()).detach().contiguous()
    pc = torch.nn.utils.parameters_to_vector(critic.parameters()).detach().contiguous()
    noise = draw_noise((T, n, K), e0.discrete)

    def eager(k):
        e = envs[k]
        o = obs[k]
        values, vf, rews, tes, trs = [], [], [], [], []
        with torch.no_grad():
            for _ in range(T):
                z = actor(o)
                values.append(critic(o)[:, 0])
                a = (z + draw_noise(z.shape, True)).argmax(dim=1) if e.discrete else z + STD * torch.randn_like(z)
                o, r, te, tr, info = e.step(a)
                vf.append(critic(info["final_observation"])[:, 0])
                rews.append(r)
                tes.append(te)
                trs.append(tr)
            values.append(critic(o)[:, 0])
            adv = gae_torch(torch.stack(rews), torch.stack(tes), torch.stack(trs), torch.stack(values),
                            torch.stack(vf))
        obs[k] = o
        return adv

    first = obs.get("noisy_then_torch", obs[next(iter(obs))]).clone()

    def composed():
        e = envs["noisy_then_torch"]
        _, _, o, r, te, tr, info = e.rollout_mlp_noisy(pa, hidden, noise, activation="tanh")
        fin = info["final_observation"]
        with torch.no_grad():
            inp = torch.cat([first[None], o])
            values = torch.stack([critic(inp[t])[:, 0] for t in range(T + 1)])
            vf = torch.stack([critic(fin[t])[:, 0] for t in range(T)])
            adv = gae_torch(r, te, tr, values, vf)
        first.copy_(o[-1])
        return adv

    arms = {}
    if "eager" in envs:
        arms["eager"] = lambda: eager("eager")
    if "graph_replay" in envs:
        eager("graph_replay")   # warm the step path and cuBLAS before the capture
        torch.cuda.synchronize()
        g1 = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g1):
            eager("graph_replay")
        arms["graph_replay"] = g1.replay
    if "noisy_then_torch" in envs:
        composed()
        torch.cuda.synchronize()
        g2 = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g2):
            composed()
        arms["noisy_then_torch"] = g2.replay
    arms["rollout_actor_critic"] = lambda: envs["rollout_actor_critic"].rollout_actor_critic(
        pa, pc, hidden, noise, gamma=GAMMA, gae_lambda=GAE_LAMBDA, activation="tanh")
    arms["rollout_mlp_noisy"] = lambda: envs["rollout_mlp_noisy"].rollout_mlp_noisy(pa, hidden, noise,
                                                                                    activation="tanh")
    for fn in arms.values():   # warm-up
        fn()
    torch.cuda.synchronize()
    ms = {k: [] for k in arms}
    names = list(arms)
    for r in range(rounds):
        for j in range(len(names)):
            k = names[(r + j) % len(names)]
            ms[k].append(timed(arms[k], flush, r * len(names) + j))
    out = {"env_id": env_id, "log2_envs": log2n, "T": T, "hidden": list(hidden), "activation": "tanh",
           "P_actor": pa.numel(), "P_critic": pc.numel(), "K": K, "rounds": rounds}
    for k, v in ms.items():
        v = np.asarray(v) * 1e3 / T   # µs per batch step
        out[k + "_us_per_batch_step"] = {"median": round(float(np.median(v)), 2), "min": round(float(v.min()), 2),
                                         "max": round(float(v.max()), 2)}
    nbytes = ac_bytes(e0, T, hidden)
    sec = out["rollout_actor_critic_us_per_batch_step"]["median"] * 1e-6
    out["rollout_actor_critic_bytes_per_env_step_from_shapes"] = round(nbytes, 2)
    out["rollout_actor_critic_share_of_hbm_peak"] = round(n * nbytes / sec / HBM_PEAK, 4)
    ac = out["rollout_actor_critic_us_per_batch_step"]["median"]
    for base in ("graph_replay", "eager", "noisy_then_torch"):
        if base in ms:
            out[f"rollout_actor_critic_speedup_vs_{base}"] = round(out[base + "_us_per_batch_step"]["median"] / ac, 3)
    out["critic_and_gae_us_per_batch_step"] = round(ac - out["rollout_mlp_noisy_us_per_batch_step"]["median"], 2)
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
    assert torch.cuda.is_available(), "rollout_actor_critic_bench.py measures on the GPU"
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
