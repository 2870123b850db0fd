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
``NormalizeObservation``, ``NormalizeReward``, ``FrameStack``, ``TimeAwareObservation``, ``FlattenObservation`` and
``RescaleAction`` classes (bare where they take no argument, or ``functools.partial`` with keyword arguments) are
accepted too.  ``ClipObservation`` / ``ClipReward`` stand for ``TransformObservation(env, lambda o: np.clip(o, lo, hi))``
/ ``TransformReward(env, lambda r: np.clip(r, lo, hi))``.

``FrameStack``, ``TimeAwareObservation`` and ``FlattenObservation`` change the observation's shape and dtype; the
chain resolves both at every position, and the env's observation spaces and output shapes follow.  Two deliberate
departures: a terminal row of a FrameStack chain arrives as an ndarray equal to ``np.asarray`` of the reference's
``LazyFrames``, and ``RescaleAction`` does not assert that actions lie in ``[min_action, max_action]`` (the engine
computes what the reference computes under ``python -O``).
"""
import functools
import sys

import numpy as np

from gym_b200 import _lib

SUPPORTED = ("RecordEpisodeStatistics, ClipAction, NormalizeObservation, NormalizeReward, ClipObservation, "
             "ClipReward, FrameStack, TimeAwareObservation, FlattenObservation and RescaleAction (gym_b200.subenv), or "
             "the reference's classes of the same names")
MAX_STACK = _lib.SUBENV_MAX_STACK   # FrameStack's num_stack

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


class FrameStack(_Stage):
    """frame_stack.py:125-190: the last ``num_stack`` observations, in the dtype they have at this position (a reset
    fills all of them with the reset observation).  ``lz4_compress=True`` is not supported."""

    def __init__(self, num_stack, lz4_compress=False):
        if lz4_compress:
            raise ValueError("wrappers: FrameStack(lz4_compress=True) is not supported on the device")
        if isinstance(num_stack, bool) or not isinstance(num_stack, (int, np.integer)) or not 1 <= num_stack <= MAX_STACK:
            raise ValueError(f"wrappers: FrameStack needs an int 1 <= num_stack <= {MAX_STACK}, got {num_stack!r}")
        super().__init__(num_stack=int(num_stack))


class TimeAwareObservation(_Stage):
    """time_aware_observation.py:24-71: appends the steps since the reset (a float64 observation, flattened)."""

    def __init__(self):
        super().__init__()


class FlattenObservation(_Stage):
    """flatten_observation.py / spaces/utils.py:138-141: flattens, rounding to the space's float32."""

    def __init__(self):
        super().__init__()


def _action_bound(v, what):
    """A RescaleAction bound that keeps the arithmetic in float32 -> float or float32 array."""
    if type(v) in (float, int):   # not np.float64, a subclass of float
        with np.errstate(over="ignore"):
            return float(np.float32(v))    # np.zeros(A, float32) + v: a Python number is weak (NEP 50)
    if isinstance(v, np.float32):
        return float(v)
    if isinstance(v, np.ndarray) and v.dtype == np.float32 and v.ndim <= 1:
        return v.copy()
    raise ValueError(f"wrappers: RescaleAction's {what} must be a Python number, an np.float32 or a float32 array of "
                     f"at most one dimension (anything else makes the actions float64), got {v!r}")


class RescaleAction(_Stage):
    """rescale_action.py:30-82: maps [min_action, max_action] affinely onto the action space below it, in float32.
    The range asserts of ``action()`` are not reproduced."""

    def __init__(self, min_action, max_action):
        lo, hi = _action_bound(min_action, "min_action"), _action_bound(max_action, "max_action")
        try:
            ok = bool(np.all(np.less_equal(lo, hi)))
        except ValueError:
            ok = False
        if not ok:
            raise ValueError(f"wrappers: RescaleAction needs min_action <= max_action, got {min_action!r} and "
                             f"{max_action!r}")
        super().__init__(min_action=lo, max_action=hi)

    def describe(self):
        def d(v):
            return [float(x) for x in v] if isinstance(v, np.ndarray) else float(v)
        return ["RescaleAction", {k: d(v) for k, v in sorted(self.kwargs.items())}]

    def __repr__(self):
        return "RescaleAction(" + ", ".join(f"{k}={v!r}" for k, v in sorted(self.describe()[1].items())) + ")"


_OWN = (RecordEpisodeStatistics, ClipAction, NormalizeObservation, NormalizeReward, ClipObservation, ClipReward,
        FrameStack, TimeAwareObservation, FlattenObservation, RescaleAction)
_REFERENCE = {"RecordEpisodeStatistics": RecordEpisodeStatistics, "ClipAction": ClipAction,
              "NormalizeObservation": NormalizeObservation, "NormalizeReward": NormalizeReward,
              "FrameStack": FrameStack, "TimeAwareObservation": TimeAwareObservation,
              "FlattenObservation": FlattenObservation, "RescaleAction": RescaleAction}


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
        if w in (FrameStack, RescaleAction):
            raise ValueError(f"wrappers: {w.__name__} needs its arguments")
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
    BipedalWalker fall), so the kernel tracks it per env from the raw type given here (csrc/subenv.cuh).

    It also resolves the spaces the wrapped env reports (``observation_space``, ``action_space``), the observation's
    shape and dtype at every position (``obs_shape``, ``final_f64``: the terminal rows are float64), and the action
    stages in the order they apply (``act_stages``: the outermost wrapper first, each with the bounds of the space
    below it)."""

    def __init__(self, stages, kind, obs_dim, action_space, observation_space=None):
        from gym_b200.spaces import Box
        self.stages = list(stages)
        self.kind, self.obs_dim = kind, int(obs_dim)
        self.clip_action = any(isinstance(s, ClipAction) for s in self.stages)
        acts = [s for s in self.stages if isinstance(s, (ClipAction, RescaleAction))]
        if acts and not hasattr(action_space, "low"):
            raise ValueError(f"wrappers: {type(acts[0]).__name__} needs a Box action space, not {action_space!r}")
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
        # action stages, innermost first: each sees the space below it; the outermost one applies first
        self.action_space = action_space
        self.act_stages = []   # (op, low, high, min, max) float32 (A,) in the order they apply
        for s in acts:
            low = np.asarray(self.action_space.low, np.float32)
            high = np.asarray(self.action_space.high, np.float32)
            if isinstance(s, ClipAction):
                self.act_stages.insert(0, (_lib.ACT_CLIP, low, high, low, high))
                continue
            shape = self.action_space.shape
            try:
                amin = np.zeros(shape, np.float32) + s.kwargs["min_action"]
                amax = np.zeros(shape, np.float32) + s.kwargs["max_action"]
            except ValueError:
                raise ValueError(f"wrappers: {s!r} does not fit the action shape {shape}") from None
            if amin.shape != shape or amax.shape != shape:
                raise ValueError(f"wrappers: {s!r} does not fit the action shape {shape}")
            assert amin.dtype == np.float32 and amax.dtype == np.float32
            self.act_stages.insert(0, (_lib.ACT_RESCALE, low, high, amin, amax))
            self.action_space = Box(low=amin, high=amax, shape=shape, dtype=np.float32)
        # observation stages: the shape, dtype and space at every position
        space = observation_space if observation_space is not None else Box(-np.inf, np.inf, (self.obs_dim,), np.float32)
        shape, obs_f32 = (self.obs_dim,), True
        self.norm_width = self.obs_dim      # width NormalizeObservation sees
        self.stack = None                   # (num_stack, frame width, frame float64) of FrameStack
        self.time_aware = False
        self.reshape = False
        self.ops = []          # (op, p0, p1) of the device stages, in order
        for s in self.stages:
            kw = s.kwargs
            width = int(np.prod(shape))
            if isinstance(s, RecordEpisodeStatistics):
                self.ops.append((_lib.SUB_EPISODE, 0.0, 0.0))
            elif isinstance(s, NormalizeObservation):
                self.ops.append((_lib.SUB_NORM_OBS, kw["epsilon"], 0.0))
                self.norm_width = width
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
            elif isinstance(s, FrameStack):
                k = kw["num_stack"]
                self.ops.append((_lib.SUB_FRAME_STACK, float(k), 0.0))
                self.stack = (k, width, not obs_f32)
                space = Box(low=np.repeat(space.low[np.newaxis, ...], k, axis=0),
                            high=np.repeat(space.high[np.newaxis, ...], k, axis=0), dtype=space.dtype)
                shape = (k,) + shape
            elif isinstance(s, TimeAwareObservation):
                self.ops.append((_lib.SUB_TIME_AWARE, 0.0, 0.0))
                self.time_aware = True
                space = Box(np.append(space.low, 0.0), np.append(space.high, np.inf), dtype=np.float32)
                shape, obs_f32 = (width + 1,), False
            elif isinstance(s, FlattenObservation):
                self.ops.append((_lib.SUB_FLATTEN, 0.0, 0.0))
                space = Box(space.low.flatten(), space.high.flatten(), dtype=space.dtype)
                assert space.dtype == np.float32
                shape, obs_f32 = (width,), True
            if isinstance(s, (FrameStack, TimeAwareObservation, FlattenObservation)):
                self.reshape = True
        self.observation_space = space
        self.obs_shape = tuple(shape)
        self.out_width = int(np.prod(shape))
        self.final_f64 = not obs_f32
        self.state = None

    def describe(self):
        """What snapshots are tied to: the stages and their arguments, in order."""
        return [s.describe() for s in self.stages]

    def allocate(self, torch, n, device):
        """The per-env state at its initial values (RunningMeanStd: mean 0, var 1, count 1e-4; returns 0; FrameStack's
        frames, head and TimeAwareObservation's t 0)."""
        d = self.norm_width
        obs = torch.zeros((2 * d + 1, n), dtype=torch.float64, device=device)
        obs[d:2 * d] = 1.0
        obs[2 * d] = 1e-4
        rew = torch.zeros((4, n), dtype=torch.float64, device=device)
        rew[1] = 1.0
        rew[2] = 1e-4
        self.state = {"obs_stats": obs, "rew_stats": rew,
                      "ep_return": torch.zeros(n, dtype=torch.float32, device=device),
                      "ep_length": torch.zeros(n, dtype=torch.int32, device=device)}
        if self.stack is not None:
            k, wf, f64 = self.stack
            self.state["history"] = torch.zeros((k * wf, n), dtype=torch.float64 if f64 else torch.float32,
                                                device=device)
            self.state["head"] = torch.zeros(n, dtype=torch.int32, device=device)
        if self.time_aware:
            self.state["t"] = torch.zeros(n, dtype=torch.int64, device=device)

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
        if "history" in st:
            c.history, c.head = st["history"].data_ptr(), st["head"].data_ptr()
        if "t" in st:
            c.t = st["t"].data_ptr()
        c.num_action_stages = len(self.act_stages)
        for s, (op, low, high, amin, amax) in enumerate(self.act_stages):
            c.action_op[s] = op
            for k in range(len(low)):
                c.action_low[s][k], c.action_high[s][k] = float(low[k]), float(high[k])
                c.action_min[s][k], c.action_max[s][k] = float(amin[k]), float(amax[k])
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
