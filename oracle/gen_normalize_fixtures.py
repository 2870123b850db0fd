"""Freeze the reference's vector normalisers as tests/golden/reference/normalize_wrappers.npz.

Needs the unmodified reference installed as ``oracle/_ref`` (``oracle/make_ref.py``):

    python oracle/gen_normalize_fixtures.py

For each classic-control id: ``NormalizeReward(NormalizeObservation(SyncVectorEnv(...)), gamma)`` over N envs with
a TimeLimit short enough to reset, T events (a reset at event 0, a ``reset(seed=)`` at event RESET, steps
otherwise), next to an unwrapped twin fed the same seeds and actions.  Per event: the twin's raw rows (what the
wrappers saw), the wrappers' float64 outputs, ``obs_rms`` and ``return_rms`` (mean, var, count) and ``returns``.
Test infrastructure, not product code.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle.gen_reference_fixtures import CLASSIC, actions  # noqa: E402
from oracle.ref_gym import import_reference  # noqa: E402

N, T, RESET, LIMIT, GAMMA = 16, 100, 50, 23, 0.9
SEEDS, ACTION_SEED = (2024, 777), 11
OUT = os.path.join(ROOT, "tests", "golden", "reference", "normalize_wrappers.npz")


def rollout(gym, env_id):
    def make():
        return gym.vector.SyncVectorEnv([lambda: gym.make(env_id, max_episode_steps=LIMIT, disable_env_checker=True)
                                         for _ in range(N)])
    from gym.wrappers import NormalizeObservation, NormalizeReward
    env = NormalizeReward(NormalizeObservation(make()), gamma=GAMMA)
    twin = make()
    acts = actions(env_id, np.random.default_rng(ACTION_SEED), T, N)
    D = twin.single_observation_space.shape[0]
    out = {"actions": acts, "raw_obs": np.zeros((T, N, D), np.float32), "obs": np.zeros((T, N, D)),
           "raw_reward": np.zeros((T, N)), "reward": np.zeros((T, N)), "terminated": np.zeros((T, N), bool),
           "truncated": np.zeros((T, N), bool), "returns": np.zeros((T, N)), "obs_mean": np.zeros((T, D)),
           "obs_var": np.zeros((T, D)), "obs_count": np.zeros(T), "ret_mean": np.zeros(T), "ret_var": np.zeros(T),
           "ret_count": np.zeros(T)}
    for t in range(T):
        if t in (0, RESET):
            seed = SEEDS[t != 0]
            o, _ = env.reset(seed=seed)
            raw, _ = twin.reset(seed=seed)
        else:
            o, r, te, tr, _ = env.step(acts[t])
            raw, rr, rte, rtr, _ = twin.step(acts[t])
            assert np.array_equal(te, rte) and np.array_equal(tr, rtr)
            out["reward"][t], out["raw_reward"][t], out["terminated"][t], out["truncated"][t] = r, rr, te, tr
        out["raw_obs"][t], out["obs"][t], out["returns"][t] = raw, o, env.returns
        rms = env.env.obs_rms
        out["obs_mean"][t], out["obs_var"][t], out["obs_count"][t] = rms.mean, rms.var, rms.count
        rms = env.return_rms
        out["ret_mean"][t], out["ret_var"][t], out["ret_count"][t] = rms.mean, rms.var, rms.count
    env.close()
    twin.close()
    assert out["terminated"].any() or out["truncated"].any()
    return out


def main():
    gym = import_reference()
    z = {"events": np.array([N, T, RESET, LIMIT]), "gamma": np.array(GAMMA), "seeds": np.array(SEEDS)}
    for env_id in CLASSIC:
        for k, v in rollout(gym, env_id).items():
            z[f"{env_id}/{k}"] = v
    np.savez_compressed(OUT, **z)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
