"""Freeze per-env wrapper chains of the real reference as tests/golden/reference/subenv_wrappers.npz.

Needs the unmodified reference installed as ``oracle/_ref`` (``oracle/make_ref.py``):

    python oracle/gen_subenv_fixtures.py

For the five classic-control ids x three chains it runs ``gym.vector.SyncVectorEnv`` over envs wrapped as
``gym.vector.make(id, n, wrappers=[...])`` wraps them, with a short TimeLimit so envs finish many times and a
``reset(seed=)`` in the middle, and stores what it returns.  It also stores the RAW outputs of the same run (the
same SyncVectorEnv over unwrapped envs, fed the clipped actions where the chain clips them), which the numpy
restatement of the chain (oracle/subenv_chain.py) and the chain-less engine are fed.  Test infrastructure.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from gym_b200 import subenv  # noqa: E402

CLASSIC = ["CartPole-v1", "MountainCar-v0", "MountainCarContinuous-v0", "Pendulum-v1", "Acrobot-v1"]
N, T, MID, MAX_STEPS = 8, 100, 50, 25
SEED, SEED_MID, ACTION_SEED = 3, 1000, 11


def chains(continuous):
    """name -> stage list (innermost first)."""
    ppo = [subenv.RecordEpisodeStatistics()] + ([subenv.ClipAction()] if continuous else []) + [
        subenv.NormalizeObservation(), subenv.ClipObservation(-10, 10), subenv.NormalizeReward(gamma=0.99),
        subenv.ClipReward(-10, 10)]
    reordered = [subenv.ClipObservation(-0.3, 0.3), subenv.NormalizeObservation(epsilon=1e-6),
                 subenv.ClipReward(-0.7, 0.7), subenv.NormalizeReward(gamma=0.9, epsilon=1e-7),
                 subenv.RecordEpisodeStatistics(deque_size=7)]
    return {"ppo": ppo, "stats": [subenv.RecordEpisodeStatistics()], "reordered": reordered}


def actions(env_id, rng):
    if env_id.startswith("CartPole"):
        return rng.integers(0, 2, size=(T, N))
    if env_id.startswith(("MountainCar-", "Acrobot")):
        return rng.integers(0, 3, size=(T, N))
    lim = 3.0 if env_id.startswith("Pendulum") else 1.5   # beyond the Box bounds, so that ClipAction bites
    return rng.uniform(-lim, lim, size=(T, N, 1)).astype(np.float32)


def reference_wrapper(gym, stage):
    """The reference wrapper a stage stands for, as a callable env -> env."""
    name, kw = stage.describe()
    if name == "RecordEpisodeStatistics":
        return lambda e: gym.wrappers.RecordEpisodeStatistics(e, deque_size=int(kw["deque_size"]))
    if name == "ClipAction":
        return gym.wrappers.ClipAction
    if name == "NormalizeObservation":
        return lambda e: gym.wrappers.NormalizeObservation(e, epsilon=kw["epsilon"])
    if name == "NormalizeReward":
        return lambda e: gym.wrappers.NormalizeReward(e, gamma=kw["gamma"], epsilon=kw["epsilon"])
    lo, hi = kw["low"], kw["high"]
    if name == "ClipObservation":
        return lambda e: gym.wrappers.TransformObservation(e, lambda o: np.clip(o, lo, hi))
    return lambda e: gym.wrappers.TransformReward(e, lambda r: np.clip(r, lo, hi))


def rollout(gym, env_id, stages, acts):
    """One SyncVectorEnv run -> dict of arrays.  stages None: unwrapped envs."""
    wrappers = [reference_wrapper(gym, s) for s in stages or []]

    def make():
        e = gym.make(env_id, max_episode_steps=MAX_STEPS, disable_env_checker=True)
        for w in wrappers:
            e = w(e)
        return e

    envs = gym.vector.SyncVectorEnv([make for _ in range(N)])
    D = envs.single_observation_space.shape[0]
    out = {"obs": np.zeros((T, N, D), np.float32), "reward": np.zeros((T, N)), "terminated": np.zeros((T, N), bool),
           "truncated": np.zeros((T, N), bool), "final_obs": np.zeros((T, N, D)), "final_f64": np.zeros((T, N), bool),
           "episode_r": np.full((T, N), np.nan, np.float32), "episode_l": np.full((T, N), -1, np.int32)}
    out["obs0"], _ = envs.reset(seed=SEED)
    for t in range(T):
        if t == MID:
            out["obs_mid"], _ = envs.reset(seed=SEED_MID)
        o, r, te, tr, info = envs.step(acts[t])
        out["obs"][t], out["reward"][t], out["terminated"][t], out["truncated"][t] = o, r, te, tr
        if "final_observation" in info:
            for i in np.flatnonzero(info["_final_observation"]):
                fo = info["final_observation"][i]
                out["final_obs"][t, i] = fo
                out["final_f64"][t, i] = fo.dtype == np.float64
                ep = info["final_info"][i].get("episode")
                if ep is not None:
                    assert type(ep["r"]) is np.float32 and type(ep["l"]) is np.int32
                    out["episode_r"][t, i], out["episode_l"][t, i] = ep["r"], ep["l"]
    envs.close()
    return out


def run_case(gym, env_id, stages):
    """-> (wrapped run, raw run, actions) of one id and chain."""
    acts = actions(env_id, np.random.default_rng(ACTION_SEED))
    raw_acts = acts
    if any(isinstance(s, subenv.ClipAction) for s in stages):
        space = gym.make(env_id, disable_env_checker=True).action_space
        raw_acts = np.clip(acts, space.low, space.high)
    return rollout(gym, env_id, stages, acts), rollout(gym, env_id, None, raw_acts), acts


def main():
    from oracle.ref_gym import import_reference
    gym = import_reference()
    z = {}
    for env_id in CLASSIC:
        for name, stages in chains(env_id in ("MountainCarContinuous-v0", "Pendulum-v1")).items():
            wrapped, raw, acts = run_case(gym, env_id, stages)
            key = f"{env_id}/{name}"
            z[f"{key}/actions"] = acts
            for k, v in wrapped.items():
                z[f"{key}/{k}"] = v
            for k, v in raw.items():
                if not k.startswith("episode") and k != "final_f64":
                    z[f"{key}/raw_{k}"] = v
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "reference", "subenv_wrappers.npz"), **z)


if __name__ == "__main__":
    main()
