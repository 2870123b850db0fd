"""``gym_b200.vector`` -- the ``gym.vector`` namespace of the engine."""
from gym_b200.vector_env import B200VectorEnv

__all__ = ["make", "B200VectorEnv", "VectorEnv"]

VectorEnv = B200VectorEnv


def make(id, num_envs=1, asynchronous=True, wrappers=None, disable_env_checker=None, **kwargs):
    """``gym.vector.make`` (gym/vector/__init__.py:12-73).

    ``asynchronous`` is accepted for signature compatibility: the GPU is the
    (only) asynchronous worker.  ``wrappers`` are applied to every sub-env on the
    device (``gym_b200.subenv`` lists the supported ones; anything else raises
    ``ValueError``).
    """
    return B200VectorEnv(id, num_envs, wrappers=wrappers, **kwargs)
