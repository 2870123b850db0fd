"""Subclasses of the REAL ``gym.Env`` / ``gym.vector.VectorEnv`` over the engine.

``B200VectorEnv`` / ``B200Env`` are self-contained (the engine must import without gym).  Inside an
installation that has openai/gym 0.26 these classes are what makes the engine a drop-in *by type*:

    isinstance(GymVectorEnv("CartPole-v1", 1 << 20), gym.vector.VectorEnv)          -> True
    gym.utils.env_checker.check_env(GymEnv("CartPole-v1"))                           -> passes
    gym.make("B200/CartPole-v1")    # gym_b200.plugin.make_env                       -> a GymEnv

They derive from both worlds -- the engine class first, so every method on the step/reset path is the
engine's -- and present ``gym.spaces`` objects (the reference's own ``Box`` / ``Discrete`` /
``batch_space``; gym/vector/vector_env.py:38-49, gym/core.py:35-84).  ``env.np_random`` /
``env.unwrapped._np_random`` (gym/core.py:75-84; read by ``check_reset_seed``,
gym/utils/env_checker.py:60-118) is a ``numpy.random.Generator`` built from the env's PCG64 state ON THE
DEVICE, so it shows exactly where the env's own stream is.

The classes are created on first use (``import gym`` happens here, not at ``import gym_b200``).
"""
import sys

import numpy as np

_cache = {}


def _to_gym_space(space, gym):
    from gym_b200 import spaces as own
    if isinstance(space, own.Box):
        return gym.spaces.Box(low=space.low, high=space.high, shape=space.shape, dtype=space.dtype.type)
    if isinstance(space, own.Discrete):
        return gym.spaces.Discrete(int(space.n), start=int(getattr(space, "start", 0)))
    if isinstance(space, own.MultiDiscrete):
        return gym.spaces.MultiDiscrete(space.nvec, dtype=space.dtype.type)
    raise TypeError(f"no gym.spaces equivalent for {space!r}")


def _device_generator(vec, index=0):
    """numpy Generator positioned where env `index`'s device PCG64 stream is (state, inc as 128-bit ints)."""
    _, _, rng = vec.get_state()
    w = rng[index].cpu().numpy().view(np.uint64)
    bg = np.random.PCG64(0)
    st = bg.state
    st["state"] = {"state": (int(w[0]) << 64) | int(w[1]), "inc": (int(w[2]) << 64) | int(w[3])}
    st["has_uint32"], st["uinteger"] = 0, 0
    bg.state = st
    return np.random.Generator(bg)


def classes():
    """-> (GymEnv, GymVectorEnv); needs an importable openai/gym 0.26."""
    if "classes" in _cache:
        return _cache["classes"]
    import gym
    from gym.vector.utils import batch_space as gym_batch_space

    from gym_b200.env import B200Env
    from gym_b200.vector_env import B200VectorEnv

    class GymVectorEnv(B200VectorEnv, gym.vector.VectorEnv):
        """``gym.vector.VectorEnv`` subclass (vector_env.py:12-275) whose reset_async / reset_wait /
        step_async / step_wait / close_extras / call are the engine's."""

        def __init__(self, env_id, num_envs, **kwargs):
            B200VectorEnv.__init__(self, env_id, num_envs, **kwargs)
            self.viewer = None
            self.single_observation_space = _to_gym_space(self.single_observation_space, gym)
            self.single_action_space = _to_gym_space(self.single_action_space, gym)
            self.observation_space = gym_batch_space(self.single_observation_space, n=self.num_envs)
            self.action_space = gym_batch_space(self.single_action_space, n=self.num_envs)

    class GymEnv(B200Env, gym.Env):
        """``gym.Env`` subclass (core.py:35-210) over a one-env engine handle."""

        def __init__(self, env_id, **kwargs):
            B200Env.__init__(self, env_id, **kwargs)
            self.observation_space = _to_gym_space(self.observation_space, gym)
            self.action_space = _to_gym_space(self.action_space, gym)

        @property
        def _np_random(self):
            if not self._vec._seeded:
                self._vec.seed(None)      # lazily seeded from OS entropy, like core.py:78-80
            return _device_generator(self._vec)

        @_np_random.setter
        def _np_random(self, value):
            # gym.Env.reset(seed=...) / `env.np_random = g` assign here; the stream lives on the device and is
            # (re)seeded by reset(seed=...) itself
            pass

    # pickle finds the classes through these module-level constructors (the classes themselves are built here)
    module = sys.modules[__name__]
    GymEnv._pickle_factory = staticmethod(module.GymEnv)
    GymVectorEnv._pickle_factory = staticmethod(module.GymVectorEnv)
    _cache["classes"] = (GymEnv, GymVectorEnv)
    return _cache["classes"]


def GymEnv(env_id, **kwargs):
    return classes()[0](env_id, **kwargs)


def GymVectorEnv(env_id, num_envs, **kwargs):
    return classes()[1](env_id, num_envs, **kwargs)
