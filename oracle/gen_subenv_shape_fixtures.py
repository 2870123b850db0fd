"""Freeze reshaping per-env wrapper chains and action chains of the real reference as
tests/golden/reference/subenv_shape_wrappers.npz.

Needs the unmodified reference installed as ``oracle/_ref`` (``oracle/make_ref.py``), and ``python -O``: some runs
feed RescaleAction actions outside ``[min_action, max_action]``, which its ``assert`` s refuse otherwise
(rescale_action.py:71-75; the engine computes what the reference computes under ``-O``):

    python -O oracle/gen_subenv_shape_fixtures.py

In the style of oracle/gen_subenv_fixtures.py: for the five classic-control ids it runs ``gym.vector.SyncVectorEnv``
over envs wrapped as ``gym.vector.make(id, n, wrappers=[...])`` wraps them, with a short TimeLimit and a
``reset(seed=)`` in the middle, and stores what it returns, the single spaces it reports and the RAW outputs of the
same run (unwrapped envs fed the actions the chain's action stages produce).  Terminal rows are stored as
``np.asarray`` of what ``infos["final_observation"][i]`` holds (a LazyFrames for FrameStack chains), with a flag for
float64 ones.  Test infrastructure.

To keep the file small, it holds 4 envs x 48 steps per run (TimeLimit 12) and stores what several runs share once:
the actions and the raw run of an id under ``{id}/``, except where a chain's action stages change the raw run (then
under ``{id}/{chain}/raw_*``), a chain's rewards only where they differ from the raw ones, its flags not at all
(they are the raw run's) and its episode statistics only where it records them.  ``load_case`` puts a run's arrays
back together.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from gym_b200 import subenv  # noqa: E402
from oracle import gen_subenv_fixtures as base  # noqa: E402

CLASSIC = base.CLASSIC
CONTINUOUS = ("MountainCarContinuous-v0", "Pendulum-v1")
N, T, MID, MAX_STEPS = 4, 48, 24, 12   # every env finishes at least three times: at 12, 24 + 12 and 24 + 24
SEED, SEED_MID, ACTION_SEED = base.SEED, base.SEED_MID, base.ACTION_SEED
RAW_KEYS = ("obs0", "obs_mid", "obs", "reward", "terminated", "truncated", "final_obs")


def chains(continuous):
    """name -> stage list (innermost first) of the observation chains."""
    ppo = base.chains(continuous)["ppo"]
    return {"fs3": [subenv.FrameStack(3)],
            "norm_fs3": [subenv.NormalizeObservation(), subenv.FrameStack(3)],
            "fs3_norm_clip": [subenv.FrameStack(3), subenv.NormalizeObservation(), subenv.ClipObservation(-1.5, 1.5)],
            "fs4_flat": [subenv.FrameStack(4), subenv.FlattenObservation()],
            "time": [subenv.TimeAwareObservation()],
            "norm_time_fs2": [subenv.NormalizeObservation(), subenv.TimeAwareObservation(), subenv.FrameStack(2)],
            "ppo_time": ppo + [subenv.TimeAwareObservation()]}


def action_chains():
    """name -> stage list of the action chains (the continuous ids only)."""
    return {"rescale": [subenv.RescaleAction(-1, 1)],
            "clip_rescale": [subenv.ClipAction(), subenv.RescaleAction(-1, 1)],
            "rescale_clip": [subenv.RescaleAction(-1, 1), subenv.ClipAction()],
            "rescale_f32": [subenv.RescaleAction(np.array([-0.5], np.float32), np.array([0.75], np.float32)),
                            subenv.RecordEpisodeStatistics()]}


def cases():
    """[(env_id, chain name, stages)]"""
    out = []
    for env_id in CLASSIC:
        for name, stages in chains(env_id in CONTINUOUS).items():
            out.append((env_id, name, stages))
        if env_id in CONTINUOUS:
            for name, stages in action_chains().items():
                out.append((env_id, name, stages))
    return out


def actions(env_id, rng):
    """As oracle/gen_subenv_fixtures.py, (T, N) here; the continuous ones reach past [-1, 1] and past the Box
    bounds."""
    if env_id.startswith("CartPole"):
        return rng.integers(0, 2, size=(T, N))
    if env_id.startswith(("MountainCar-", "Acrobot")):
        return rng.integers(0, 3, size=(T, N))
    lim = 3.0 if env_id.startswith("Pendulum") else 1.5
    return rng.uniform(-lim, lim, size=(T, N, 1)).astype(np.float32)


def has_action_stages(stages):
    return any(isinstance(s, (subenv.ClipAction, subenv.RescaleAction)) for s in stages)


def load_case(z, env_id, name):
    """The arrays of one run from the loaded fixture `z` (a dict): the wrapped run's keys, "actions", and the raw
    run's as "raw_*" ("raw_actions" where the chain has action stages)."""
    shared, own = f"{env_id}/", f"{env_id}/{name}/"
    c = {k[len(shared):]: v for k, v in z.items() if k.startswith(shared) and "/" not in k[len(shared):]}
    c.update({k[len(own):]: v for k, v in z.items() if k.startswith(own)})
    c.setdefault("raw_actions", c["actions"])
    c.setdefault("reward", c["raw_reward"])
    c.setdefault("terminated", c["raw_terminated"])
    c.setdefault("truncated", c["raw_truncated"])
    c.setdefault("episode_r", np.full(c["raw_reward"].shape, np.nan, np.float32))
    c.setdefault("episode_l", np.full(c["raw_reward"].shape, -1, np.int32))
    return c


def reference_wrapper(gym, stage):
    name, kw = stage.describe()
    if name == "FrameStack":
        return lambda e: gym.wrappers.FrameStack(e, num_stack=int(kw["num_stack"]))
    if name == "TimeAwareObservation":
        return gym.wrappers.TimeAwareObservation
    if name == "FlattenObservation":
        return gym.wrappers.FlattenObservation
    if name == "RescaleAction":
        lo, hi = stage.kwargs["min_action"], stage.kwargs["max_action"]
        return lambda e: gym.wrappers.RescaleAction(e, min_action=lo, max_action=hi)
    return base.reference_wrapper(gym, stage)


def make_fn(gym, env_id, stages):
    wrappers = [reference_wrapper(gym, s) for s in stages or []]

    def make():
        e = gym.make(env_id, max_episode_steps=MAX_STEPS, disable_env_checker=True)
        for w in wrappers:
            e = w(e)
        return e
    return make


def rollout(gym, env_id, stages, acts):
    """One SyncVectorEnv run -> dict of arrays.  stages None: unwrapped envs."""
    envs = gym.vector.SyncVectorEnv([make_fn(gym, env_id, stages) for _ in range(N)])
    shape = envs.single_observation_space.shape
    out = {"obs": np.zeros((T, N) + shape, np.float32), "reward": np.zeros((T, N)),
           "terminated": np.zeros((T, N), bool), "truncated": np.zeros((T, N), bool),
           "final_obs": np.zeros((T, N) + shape), "final_f64": np.zeros((T, N), bool),
           "episode_r": np.full((T, N), np.nan, np.float32), "episode_l": np.full((T, N), -1, np.int32)}
    sp = envs.single_observation_space
    out["obs_low"], out["obs_high"] = sp.low, sp.high
    assert sp.dtype == np.float32
    if hasattr(envs.single_action_space, "low"):
        out["act_low"], out["act_high"] = envs.single_action_space.low, envs.single_action_space.high
    out["obs0"], _ = envs.reset(seed=SEED)
    for t in range(T):
        if t == MID:
            out["obs_mid"], _ = envs.reset(seed=SEED_MID)
        o, r, te, tr, info = envs.step(acts[t])
        out["obs"][t], out["reward"][t], out["terminated"][t], out["truncated"][t] = o, r, te, tr
        if "final_observation" in info:
            for i in np.flatnonzero(info["_final_observation"]):
                fo = np.asarray(info["final_observation"][i])
                out["final_obs"][t, i] = fo
                out["final_f64"][t, i] = fo.dtype == np.float64
                ep = info["final_info"][i].get("episode")
                if ep is not None:
                    out["episode_r"][t, i], out["episode_l"][t, i] = ep["r"], ep["l"]
    envs.close()
    return out


def raw_actions(gym, env_id, stages, acts):
    """The actions the unwrapped env sees: each row through the reference's action wrappers, outermost first."""
    if not has_action_stages(stages):
        return acts
    e = make_fn(gym, env_id, stages)()
    out = np.empty_like(acts)
    for idx in np.ndindex(acts.shape[:2]):
        a, w = acts[idx], e
        while isinstance(w, gym.Wrapper):
            if isinstance(w, gym.ActionWrapper):
                a = w.action(a)
            w = w.env
        assert a.dtype == np.float32
        out[idx] = a
    return out


def run_case(gym, env_id, stages):
    """-> (wrapped run, raw run, actions) of one id and chain."""
    acts = actions(env_id, np.random.default_rng(ACTION_SEED))
    raw_acts = raw_actions(gym, env_id, stages, acts)
    raw = rollout(gym, env_id, None, raw_acts)
    raw["actions"] = raw_acts
    return rollout(gym, env_id, stages, acts), raw, acts


def main():
    from oracle.ref_gym import import_reference
    if __debug__:
        raise SystemExit("run with python -O (see the module docstring)")
    gym = import_reference()
    z = {}
    for env_id, name, stages in cases():
        wrapped, raw, acts = run_case(gym, env_id, stages)
        if f"{env_id}/actions" not in z:
            z[f"{env_id}/actions"] = acts
        assert np.array_equal(z[f"{env_id}/actions"], acts)
        raw_prefix = f"{env_id}/{name}/raw_" if has_action_stages(stages) else f"{env_id}/raw_"
        for k in RAW_KEYS:
            if f"{raw_prefix}{k}" in z:   # a raw run without action stages is the same for every chain of the id
                assert np.array_equal(z[f"{raw_prefix}{k}"], raw[k]), (env_id, name, k)
            z[f"{raw_prefix}{k}"] = raw[k]
        if has_action_stages(stages):
            z[f"{raw_prefix}actions"] = raw["actions"]
        for k, v in wrapped.items():
            if k in ("reward", "terminated", "truncated") and np.array_equal(v.view(np.uint8), raw[k].view(np.uint8)):
                continue
            if k in ("episode_r", "episode_l") and not any(isinstance(s, subenv.RecordEpisodeStatistics)
                                                           for s in stages):
                assert (wrapped["episode_l"] == -1).all()
                continue
            z[f"{env_id}/{name}/{k}"] = v
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "reference", "subenv_shape_wrappers.npz"), **z)


if __name__ == "__main__":
    main()
