"""Per-env wrapper chains: ``B200VectorEnv(id, n, wrappers=[...])`` / ``vector.make(id, n, wrappers=[...])``.

In gym 0.26 ``gym.vector.make(id, n, wrappers=[...])`` (gym/vector/__init__.py:56-63) gives every sub-env of a
``SyncVectorEnv`` its own wrapper stack, applied in list order on top of ``TimeLimit``.  The engine runs such a stack
on the device, one thread per env, after the step (csrc/subenv.cuh), bit-identical to the reference.  This differs
from ``gym_b200.wrappers``, whose wrappers wrap the *vector* env and keep statistics over the whole batch:

* statistics are per env (one RunningMeanStd per env, updated with a batch of one);
* the autoreset goes through the outermost wrapper, so a finishing env updates its observation statistics with its
  terminal and then its reset observation in the same step;
* episode statistics arrive in ``infos["final_info"][i]["episode"]`` and the float64 terminal rows of a normalised
  chain in ``infos["final_observation"]``.

The stages below stand for the reference's wrappers; the reference's own ``RecordEpisodeStatistics``, ``ClipAction``,
``NormalizeObservation`` and ``NormalizeReward`` classes (bare, or ``functools.partial`` with keyword arguments) are
accepted too.  ``ClipObservation`` / ``ClipReward`` stand for ``TransformObservation(env, lambda o: np.clip(o, lo, hi))``
/ ``TransformReward(env, lambda r: np.clip(r, lo, hi))``.
"""
import functools
import sys

import numpy as np

from gym_b200 import _lib

SUPPORTED = ("RecordEpisodeStatistics, ClipAction, NormalizeObservation, NormalizeReward, ClipObservation and "
             "ClipReward (gym_b200.subenv), or the reference's RecordEpisodeStatistics, ClipAction, "
             "NormalizeObservation and NormalizeReward classes")

# the Python type of each kind's raw reward (SyncVectorEnv stores them all as float64, but the wrappers see the scalar):
# a Python number (CartPole, MountainCar*, Acrobot), np.float64 (Pendulum, LunarLander*; LunarLander's +-100 are Python
# ints, exact in float32, so they need no rule of their own) or np.float32 (BipedalWalker*, except the -100 of a fall,
# a Python int: bipedal_walker.py:598-600)
REWARD_PY, REWARD_F64, REWARD_F32 = 0, 1, 2
RAW_REWARD_TYPE = {_lib.KIND_CARTPOLE: REWARD_PY, _lib.KIND_MOUNTAINCAR: REWARD_PY, _lib.KIND_MOUNTAINCAR_CONT: REWARD_PY,
                   _lib.KIND_PENDULUM: REWARD_F64, _lib.KIND_ACROBOT: REWARD_PY, _lib.KIND_LUNARLANDER: REWARD_F64,
                   _lib.KIND_BIPEDALWALKER: REWARD_F32, _lib.KIND_LUNARLANDER_CONT: REWARD_F64,
                   _lib.KIND_BIPEDALWALKER_HARDCORE: REWARD_F32}
INT_REWARD_ON_FALL = (_lib.KIND_BIPEDALWALKER, _lib.KIND_BIPEDALWALKER_HARDCORE)


class _Stage:
    """One wrapper of a chain: its name and keyword arguments."""

    def __init__(self, **kwargs):
        self.kwargs = kwargs

    def describe(self):
        return [type(self).__name__, {k: float(v) for k, v in sorted(self.kwargs.items())}]

    def __eq__(self, other):
        return type(self) is type(other) and self.describe() == other.describe()

    def __hash__(self):
        return hash(repr(self.describe()))

    def __repr__(self):
        return f"{type(self).__name__}({', '.join(f'{k}={v!r}' for k, v in sorted(self.kwargs.items()))})"


class RecordEpisodeStatistics(_Stage):
    """record_episode_statistics.py:79-151; ``deque_size`` is kept for the description only (the per-env queues are
    not exposed)."""

    def __init__(self, deque_size=100):
        super().__init__(deque_size=int(deque_size))


class ClipAction(_Stage):
    """clip_action.py:31-40 (Box action spaces only)."""

    def __init__(self):
        super().__init__()


class NormalizeObservation(_Stage):
    """normalize.py:49-94, one RunningMeanStd per env."""

    def __init__(self, epsilon=1e-8):
        super().__init__(epsilon=float(epsilon))


class NormalizeReward(_Stage):
    """normalize.py:97-144, one RunningMeanStd and discounted return per env."""

    def __init__(self, gamma=0.99, epsilon=1e-8):
        super().__init__(gamma=float(gamma), epsilon=float(epsilon))


class _Clip(_Stage):
    def __init__(self, low, high):
        low, high = float(low), float(high)
        if not (low <= high):
            raise ValueError(f"{type(self).__name__} needs low <= high, got {low} and {high}")
        super().__init__(low=low, high=high)


class ClipObservation(_Clip):
    """``TransformObservation(env, lambda o: np.clip(o, low, high))``."""


class ClipReward(_Clip):
    """``TransformReward(env, lambda r: np.clip(r, low, high))``."""


_OWN = (RecordEpisodeStatistics, ClipAction, NormalizeObservation, NormalizeReward, ClipObservation, ClipReward)
_REFERENCE = {"RecordEpisodeStatistics": RecordEpisodeStatistics, "ClipAction": ClipAction,
              "NormalizeObservation": NormalizeObservation, "NormalizeReward": NormalizeReward}


def _reference_stage(cls, kwargs):
    """The stage a class of the reference's gym.wrappers stands for, or None."""
    gym = sys.modules.get("gym")
    wrappers = getattr(gym, "wrappers", None) if gym is not None else None
    name = getattr(cls, "__name__", None)
    if wrappers is None or name not in _REFERENCE or getattr(wrappers, name, None) is not cls:
        return None
    try:
        return _REFERENCE[name](**kwargs)
    except TypeError as exc:
        raise ValueError(f"wrappers: {name} does not take {sorted(kwargs)}: {exc}") from None


def _stage(w):
    if isinstance(w, _OWN):
        return w
    if isinstance(w, type) and issubclass(w, _OWN):
        if issubclass(w, _Clip):
            raise ValueError(f"wrappers: {w.__name__} needs its bounds, e.g. {w.__name__}(-10, 10)")
        return w()
    cls, kwargs = w, {}
    if isinstance(w, functools.partial) and not w.args:
        cls, kwargs = w.func, dict(w.keywords)
    stage = _reference_stage(cls, kwargs) if isinstance(cls, type) else None
    if stage is None:
        raise ValueError(f"wrappers: {w!r} is not supported on the device; the supported per-env wrappers are "
                         f"{SUPPORTED}")
    return stage


def parse(wrappers):
    """``wrappers=`` (None, one wrapper or a list, innermost first) -> a list of stages, or None for no chain."""
    if wrappers is None:
        return None
    items = [wrappers] if (callable(wrappers) or isinstance(wrappers, _OWN)) else list(wrappers)
    stages = [_stage(w) for w in items]
    seen = set()
    for s in stages:
        if type(s) in seen:
            raise ValueError(f"wrappers: {type(s).__name__} appears twice; each per-env wrapper may appear once")
        seen.add(type(s))
    return stages or None


class Chain:
    """A parsed chain resolved for one env kind: the launch arguments and the per-env state tensors.

    The host resolves the dtype of the observation a ClipObservation sees: float32 (bounds rounded to float32) before
    NormalizeObservation, float64 after it.  The Python type of the reward can change from one env-step to the next (a
    BipedalWalker fall), so the kernel tracks it per env from the raw type given here (csrc/subenv.cuh)."""

    def __init__(self, stages, kind, obs_dim, action_space):
        self.stages = list(stages)
        self.kind, self.obs_dim = kind, int(obs_dim)
        self.clip_action = any(isinstance(s, ClipAction) for s in self.stages)
        if self.clip_action and not hasattr(action_space, "low"):
            raise ValueError(f"wrappers: ClipAction needs a Box action space, not {action_space!r}")
        self.norm_obs = any(isinstance(s, NormalizeObservation) for s in self.stages)
        self.norm_reward = any(isinstance(s, NormalizeReward) for s in self.stages)
        self.changes_rewards = any(isinstance(s, (NormalizeReward, ClipReward)) for s in self.stages)
        self.episode = any(isinstance(s, RecordEpisodeStatistics) for s in self.stages)
        self.raw_reward_type = RAW_REWARD_TYPE[kind]
        self.int_reward_on_fall = kind in INT_REWARD_ON_FALL
        self.act_low = self.act_high = None
        if self.clip_action:
            self.act_low = np.ascontiguousarray(action_space.low, dtype=np.float32)
            self.act_high = np.ascontiguousarray(action_space.high, dtype=np.float32)
        self.ops = []          # (op, p0, p1) of the device stages, in order
        obs_f32 = True
        for s in self.stages:
            kw = s.kwargs
            if isinstance(s, RecordEpisodeStatistics):
                self.ops.append((_lib.SUB_EPISODE, 0.0, 0.0))
            elif isinstance(s, NormalizeObservation):
                self.ops.append((_lib.SUB_NORM_OBS, kw["epsilon"], 0.0))
                obs_f32 = False
            elif isinstance(s, NormalizeReward):
                self.ops.append((_lib.SUB_NORM_REWARD, kw["gamma"], kw["epsilon"]))
            elif isinstance(s, ClipObservation):
                lo, hi = kw["low"], kw["high"]
                if obs_f32:
                    with np.errstate(over="ignore"):
                        lo, hi = float(np.float32(lo)), float(np.float32(hi))
                self.ops.append((_lib.SUB_CLIP_OBS, lo, hi))
            elif isinstance(s, ClipReward):
                self.ops.append((_lib.SUB_CLIP_REWARD, kw["low"], kw["high"]))
        self.state = None

    def describe(self):
        """What snapshots are tied to: the stages and their arguments, in order."""
        return [s.describe() for s in self.stages]

    def allocate(self, torch, n, device):
        """The per-env state at its initial values (RunningMeanStd: mean 0, var 1, count 1e-4; returns 0)."""
        d = self.obs_dim
        obs = torch.zeros((2 * d + 1, n), dtype=torch.float64, device=device)
        obs[d:2 * d] = 1.0
        obs[2 * d] = 1e-4
        rew = torch.zeros((4, n), dtype=torch.float64, device=device)
        rew[1] = 1.0
        rew[2] = 1e-4
        self.state = {"obs_stats": obs, "rew_stats": rew,
                      "ep_return": torch.zeros(n, dtype=torch.float32, device=device),
                      "ep_length": torch.zeros(n, dtype=torch.int32, device=device)}

    def struct(self):
        c = _lib.Subenv()
        c.num_stages = len(self.ops)
        for k, (op, p0, p1) in enumerate(self.ops):
            c.op[k], c.p0[k], c.p1[k] = op, p0, p1
        c.raw_reward_type = self.raw_reward_type
        c.int_reward_on_fall = 1 if self.int_reward_on_fall else 0
        st = self.state
        c.obs_stats = st["obs_stats"].data_ptr()
        c.rew_stats = st["rew_stats"].data_ptr()
        c.ep_return = st["ep_return"].data_ptr()
        c.ep_length = st["ep_length"].data_ptr()
        c.clip_action = 1 if self.clip_action else 0
        if self.clip_action:
            for k in range(len(self.act_low)):
                c.act_low[k], c.act_high[k] = float(self.act_low[k]), float(self.act_high[k])
        return c

    # snapshots: every per-env row follows its env; extras hold them env-major ((m, rows) and (m,))
    def snapshot_extra(self, pick):
        return {k: pick(v.t() if v.dim() == 2 else v) for k, v in self.state.items()}

    def restore_extra(self, extra, scatter):
        for k, v in self.state.items():
            if v.dim() == 2:
                t = v.t().contiguous()
                scatter(t, extra[k])
                v.copy_(t.t())
            else:
                scatter(v, extra[k])

    def clone_extra(self, src):
        for k, v in self.state.items():
            v.copy_(v.index_select(v.dim() - 1, src))
