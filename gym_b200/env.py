"""``B200Env`` -- the single-environment facade (``gym.make(id)`` shape).

What the reference returns from ``gym.make`` is ``TimeLimit(OrderEnforcing(
PassiveEnvChecker(Env)))`` (gym/envs/registration.py:659-683).  This class is the
same contract on top of a one-env engine handle: numpy in, numpy out, no
autoreset (unless ``autoreset=True``, i.e. ``AutoResetWrapper``,
gym/wrappers/autoreset.py:35-61), ``ResetNeeded`` before the first reset
(gym/wrappers/order_enforcing.py:33-37), and ``truncated`` from the fused
TimeLimit counter.  It exists so that ``check_env``-style acceptance tests and
single-env agents run unchanged; the throughput path is ``B200VectorEnv``.
"""
import numpy as np

from gym_b200 import _lib, error
from gym_b200.vector_env import B200VectorEnv, _unpickle, refuse_capture

_NO_CAPTURE = "B200Env steps through host buffers and synchronises; capture a B200VectorEnv with backend='torch'"


class B200Env:
    def __init__(self, env_id, max_episode_steps=None, autoreset=False, device=None, **kwargs):
        if kwargs.get("wrappers"):
            raise ValueError("B200Env does not take per-env wrappers (they belong to B200VectorEnv)")
        self._vec = B200VectorEnv(env_id, 1, device=device, max_episode_steps=max_episode_steps,
                                  backend="numpy", copy=True, autoreset=autoreset, **kwargs)
        self.spec = self._vec.spec
        self.metadata = self._vec.metadata
        self.render_mode = None
        self.reward_range = self._vec.reward_range
        self.observation_space = self._vec.single_observation_space
        self.action_space = self._vec.single_action_space
        self._autoreset = bool(autoreset)

    # gym/core.py:86-151
    def reset(self, *, seed=None, options=None):
        refuse_capture("B200Env.reset()", _NO_CAPTURE)
        obs, _ = self._vec.reset(seed=seed, options=options)
        return obs[0], {}

    def step(self, action):
        refuse_capture("B200Env.step()", _NO_CAPTURE)
        v = self._vec
        if v.discrete:
            if not self.action_space.contains(action if not isinstance(action, np.ndarray) or action.shape == ()
                                              else action.reshape(())[()]):
                raise error.InvalidAction(f"{action!r} ({type(action)}) invalid")
            a = np.array([int(action)], dtype=np.int64)
        else:
            a = np.asarray(action, dtype=np.float32).reshape(1, v.act_dim)
        obs, rew, term, trunc, infos = v.step(a)
        info = {}
        if self._autoreset and "final_observation" in infos:
            info = {"final_observation": infos["final_observation"][0], "final_info": infos["final_info"][0]}
        # Pendulum returns np.float64 (pendulum.py:139); `spec` may have been replaced by gym.make (registration.py:657)
        reward = rew[0] if v.kind == _lib.KIND_PENDULUM else float(rew[0])
        return obs[0], reward, bool(term[0]), bool(trunc[0]), info

    @property
    def state(self):
        """``env.unwrapped.state`` of the reference classes, as a float64 vector."""
        st, _, _ = self._vec.get_state()
        return st[0].cpu().numpy()

    @property
    def unwrapped(self):
        return self

    @property
    def device(self):
        return self._vec.device

    # pickle / deepcopy carry the whole env state (B200VectorEnv.snapshot): the copy continues bit-identically
    _pickle_factory = None

    def _rebuild_args(self):
        v = self._vec
        kw = v._rebuild_env_kwargs()
        kw.update(max_episode_steps=v.max_episode_steps or 0, autoreset=self._autoreset, device=v.device.index)
        return (v.spec,), kw   # self.spec may be gym's own EnvSpec (gym.make replaces it)

    def _load_snapshot_payload(self, snap, seeded, has_reset):
        self._vec._load_snapshot_payload(snap, seeded, has_reset)

    def __reduce__(self):
        v = self._vec
        v._assert_open("pickle")
        args, kwargs = self._rebuild_args()
        payload = (v.snapshot().state_dict(), v._seeded, v._has_reset)
        return _unpickle, (type(self)._pickle_factory or type(self), args, kwargs, payload)

    def __deepcopy__(self, memo):
        v = self._vec
        v._assert_open("deepcopy")
        args, kwargs = self._rebuild_args()
        new = (type(self)._pickle_factory or type(self))(*args, **kwargs)
        new._load_snapshot_payload(v.snapshot(), v._seeded, v._has_reset)
        return new

    @property
    def _max_episode_steps(self):
        return self._vec.max_episode_steps

    def render(self):
        return None

    def close(self):
        self._vec.close()

    def __enter__(self):
        return self

    def __exit__(self, *args):
        self.close()
        return False

    def __repr__(self):
        return f"<B200Env<{self.spec.id}>>"
