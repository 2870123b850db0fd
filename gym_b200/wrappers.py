"""Vector-aware wrappers of the reference, re-built for device-resident batches (SURVEY.md 8f).

* ``RecordEpisodeStatistics``  gym/wrappers/record_episode_statistics.py:79-151
* ``NormalizeObservation`` / ``NormalizeReward``  gym/wrappers/normalize.py:50-144
* ``VectorListInfo``  gym/wrappers/vector_list_info.py:56-111
* ``step_api_compatibility``  gym/utils/step_api_compatibility.py:24-161

CUDA graphs: ``RecordEpisodeStatistics`` may be captured with the env it wraps (its ``"t"`` keeps the capture-time
value on replays); the normalisers and ``VectorListInfo`` refuse to be captured -- the normalisers pick their
statistics set by a host-side parity that a replay cannot flip, ``VectorListInfo`` synchronises.

The first three run on the device through the C ABI -- ``RecordEpisodeStatistics`` as one launch per
step over the rewards and flags the wrapped env returned, the normalisers as two launches per step with one pass
over the batch for the moments and, for sharded envs, an all-reduce of the 2 x dim batch sums in between -- with no
Python loop over the batch and no host synchronisation; the last two are host-side adapters.  They wrap
a ``B200VectorEnv`` with ``backend="torch"`` (or a ``ShardedVectorEnv``).
"""
import ctypes
import time
from collections import deque

import numpy as np

from gym_b200 import _lib
from gym_b200.vector_env import refuse_capture

_NORM_NO_CAPTURE = ("the running statistics are double-buffered by a host-side parity that replays would not flip, so "
                    "they would stop updating; step the normaliser eagerly")


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


class VectorWrapper:
    """Minimal ``gym.vector.VectorEnvWrapper`` (gym/vector/vector_env.py:277-332): forwards everything."""

    def __init__(self, env):
        self.env = env

    def __getattr__(self, name):
        if name.startswith("_"):
            raise AttributeError(name)
        return getattr(self.env, name)

    def reset(self, **kwargs):
        return self.env.reset(**kwargs)

    def step(self, actions):
        return self.env.step(actions)

    def rollout(self, actions):
        """Refused: a wrapper acts after every step, which a fused rollout of the env it wraps would skip (the
        statistics would not be recorded, the observations not normalised).  Step the wrapper instead."""
        from gym_b200 import error
        raise error.Error(f"{type(self).__name__} does not support rollout(): it acts after every step, and a fused "
                          "rollout of the wrapped env would skip it; call step() T times instead")

    def rollout_sampled(self, T):
        """Refused, as rollout(): step the wrapper with ``sample_actions()`` instead."""
        from gym_b200 import error
        raise error.Error(f"{type(self).__name__} does not support rollout_sampled(): it acts after every step, and a "
                          "fused rollout of the wrapped env would skip it; call step(sample_actions()) T times instead")

    def rollout_linear(self, weight, bias, T, *, summary=False):
        """Refused, as rollout(): step the wrapper with the policy's actions instead."""
        from gym_b200 import error
        raise error.Error(f"{type(self).__name__} does not support rollout_linear(): it acts after every step, and a "
                          "fused rollout of the wrapped env would skip it; call step() with the policy's actions T "
                          "times instead")

    def rollout_mlp(self, params, hidden, T, *, summary=False, activation="relu", head=None):
        """Refused, as rollout(): step the wrapper with the policy's actions instead."""
        from gym_b200 import error
        raise error.Error(f"{type(self).__name__} does not support rollout_mlp(): it acts after every step, and a "
                          "fused rollout of the wrapped env would skip it; call step() with the policy's actions T "
                          "times instead")

    def rollout_mlp_noisy(self, params, hidden, noise, *, activation="relu", head=None):
        """Refused, as rollout(): step the wrapper with the policy's actions instead."""
        from gym_b200 import error
        raise error.Error(f"{type(self).__name__} does not support rollout_mlp_noisy(): it acts after every step, and "
                          "a fused rollout of the wrapped env would skip it; call step() with the policy's actions T "
                          "times instead")

    def rollout_actor_critic(self, actor, critic, hidden, noise, *, gamma, gae_lambda, activation="relu"):
        """Refused, as rollout(): step the wrapper with the policy's actions instead."""
        from gym_b200 import error
        raise error.Error(f"{type(self).__name__} does not support rollout_actor_critic(): it acts after every step, "
                          "and a fused rollout of the wrapped env would skip it; call step() with the policy's actions "
                          "T times instead")

    def rollout_from(self, snap, actions, *, rows=None, states=False):
        """Refused, as rollout(): restore the snapshot into the wrapper's env and step the wrapper instead."""
        from gym_b200 import error
        raise error.Error(f"{type(self).__name__} does not support rollout_from(): it acts after every step, and a "
                          "fused rollout of the wrapped env would skip it; restore() the snapshot and call step() T "
                          "times instead")

    def rollout_from_mlp(self, snap, params, hidden, T, **kwargs):
        """Refused, as rollout_from()."""
        from gym_b200 import error
        raise error.Error(f"{type(self).__name__} does not support rollout_from_mlp(): it acts after every step, and a "
                          "fused rollout of the wrapped env would skip it; restore() the snapshot and call step() T "
                          "times instead")

    def close(self, **kwargs):
        return self.env.close(**kwargs)

    # B200VectorEnv.snapshot / restore / clone; a wrapper with per-env or running state extends them through the
    # hooks below, keeping its part of a snapshot in snap.extras under its own layer key
    def snapshot(self, indices=None):
        snap = self.env.snapshot(indices)
        extra = self._snapshot_extra(self.unwrapped._index_tensor(indices, "snapshot indices"))
        if extra is not None:
            snap.extras[self._layer_key()] = extra
        return snap

    def restore(self, snap, indices=None):
        obs, info = self.env.restore(snap, indices)
        key = self._layer_key()
        if self._has_snapshot_state():
            if key not in snap.extras:
                from gym_b200 import error
                raise error.Error(f"the snapshot carries no state for wrapper layer {key}")
            self._restore_extra(snap.extras[key], self.unwrapped._index_tensor(indices, "restore indices"))
        return self._restored_obs(obs), info

    def clone(self, src):
        import torch
        obs = self.env.clone(src)
        u = self.unwrapped
        src = u._index_tensor(src, "clone sources")
        self._clone_extra(u._in_range(src, torch.arange(u.num_envs, device=u.device)))
        return self._restored_obs(obs)

    def _layer_key(self):
        depth, e = 0, self.env
        while isinstance(e, VectorWrapper):
            depth, e = depth + 1, e.env
        return f"{depth}:{type(self).__name__}"

    def _has_snapshot_state(self):
        return False

    def _snapshot_extra(self, idx):
        return None

    def _restore_extra(self, extra, idx):
        pass

    def _clone_extra(self, src):
        pass

    def _restored_obs(self, obs):
        return obs

    @property
    def unwrapped(self):
        return self.env.unwrapped


def _pick(u, t, idx):
    """Rows `idx` of a per-env tensor (all rows: idx None); out-of-range entries read row 0."""
    return t.clone() if idx is None else t.index_select(0, u._in_range(idx, 0))


def _scatter(u, t, idx, values):
    """t[idx] = values for a per-env tensor (all rows: idx None); out-of-range entries land in a scratch row."""
    import torch
    if idx is None:
        t.copy_(values)
        return
    tmp = torch.cat([t, t[:1]])
    tmp.index_copy_(0, u._in_range(idx, u.num_envs), values.to(t.device))
    t.copy_(tmp[:u.num_envs])


def _rms_state(r):
    return {"stats": r.stats.clone(), "scratch": r.scratch.clone(), "cur": int(r.cur)}


def _set_rms_state(r, e):
    r.stats.copy_(e["stats"])
    r.scratch.copy_(e["scratch"])
    r.cur = int(e["cur"])


class RecordEpisodeStatistics(VectorWrapper):
    """Cumulative reward and length of every episode, kept on the device.

    ``infos["episode"] = {"r": float32 (N,), "l": int32 (N,), "t": float}`` with the ``_episode`` mask
    (rows valid where the mask is set), every step and without a host sync.  ``return_queue`` /
    ``length_queue`` (the last ``deque_size`` finished episodes) and ``episode_count`` synchronise on access.
    """

    def __init__(self, env, deque_size=100):
        super().__init__(env)
        import torch
        self._torch = torch
        n, dev = env.num_envs, env.device
        self.num_envs = n
        self.is_vector_env = True
        self.t0 = time.perf_counter()
        self.deque_size = int(deque_size)
        self.episode_returns = torch.zeros(n, dtype=torch.float32, device=dev)
        self.episode_lengths = torch.zeros(n, dtype=torch.int32, device=dev)
        self._ep_r = [torch.zeros(n, dtype=torch.float32, device=dev) for _ in range(2)]
        self._ep_l = [torch.zeros(n, dtype=torch.int32, device=dev) for _ in range(2)]
        self._ep_m = [torch.zeros(n, dtype=torch.bool, device=dev) for _ in range(2)]
        # one int64 word per slot: length << 32 | float32 bits of the return (written with a single store)
        self._ring = torch.zeros(max(self.deque_size, 1), dtype=torch.int64, device=dev)
        self._counter = torch.zeros(1, dtype=torch.int64, device=dev)
        self._flip = 0

    def reset(self, **kwargs):
        out = self.env.reset(**kwargs)
        self.episode_returns.zero_()
        self.episode_lengths.zero_()
        return out

    def step(self, actions):
        self._flip ^= 1
        k = self._flip
        obs, rew, term, trunc, infos = self.env.step(actions)
        # one launch over the rewards and flags step() returned: what a per-env wrapper chain or another wrapper made
        # of them is what gets summed
        env = self.env.unwrapped
        _lib.check(env._lib.b200gym_episode_stats(
            _p(rew), _p(term), _p(trunc), _p(self.episode_returns), _p(self.episode_lengths), _p(self._ep_r[k]),
            _p(self._ep_l[k]), _p(self._ep_m[k]), _p(self._ring), _p(self._counter),
            self.deque_size, self.num_envs, env._stream()))
        infos["episode"] = {"r": self._ep_r[k], "l": self._ep_l[k], "t": round(time.perf_counter() - self.t0, 6)}
        infos["_episode"] = self._ep_m[k]
        return obs, rew, term, trunc, infos

    # snapshots: the per-env accumulators follow the envs, the ring and the counter are saved and restored whole
    def _has_snapshot_state(self):
        return True

    def _snapshot_extra(self, idx):
        u = self.unwrapped
        return {"episode_returns": _pick(u, self.episode_returns, idx), "episode_lengths": _pick(u, self.episode_lengths, idx),
                "ring": self._ring.clone(), "counter": self._counter.clone()}

    def _restore_extra(self, e, idx):
        u = self.unwrapped
        _scatter(u, self.episode_returns, idx, e["episode_returns"])
        _scatter(u, self.episode_lengths, idx, e["episode_lengths"])
        self._ring.copy_(e["ring"])
        self._counter.copy_(e["counter"])

    def _clone_extra(self, src):
        self.episode_returns.copy_(self.episode_returns.index_select(0, src))
        self.episode_lengths.copy_(self.episode_lengths.index_select(0, src))

    @property
    def episode_count(self):
        return int(self._counter.item())

    def _queue(self, returns):
        return unpack_episode_ring(self._ring.cpu().numpy(), self.episode_count, self.deque_size, returns)

    @property
    def return_queue(self):
        return self._queue(True)

    @property
    def length_queue(self):
        return self._queue(False)


def unpack_episode_ring(words, count, deque_size, returns):
    """The ring written by b200gym_episode_stats -> the reference's deque (record_episode_statistics.py:90-91):
    slot (episode number mod size) holds length << 32 | float32 bits of the return; oldest kept episode first."""
    k = min(int(count), int(deque_size))
    words = np.ascontiguousarray(words).view(np.uint64)
    vals = (words & np.uint64(0xFFFFFFFF)).astype(np.uint32).view(np.float32) if returns else \
        (words >> np.uint64(32)).astype(np.int32)
    order = [(count - k + j) % max(int(deque_size), 1) for j in range(k)]
    return deque((vals[i].item() for i in order), maxlen=int(deque_size))


class _RunningMeanStd:
    """Device copy of RunningMeanStd's state (normalize.py:8-29): mean 0, var 1, count epsilon.

    ``stats[2][2*d + 1]`` = {mean, var, count} and ``scratch[2][2*d]`` = this step's batch sums, both
    double-buffered by step parity (include/b200gym.h); ``cur`` is the set holding the current statistics.
    ``work`` holds the moments launch's per-CTA partial sums (zero between launches, not part of the state)."""

    def __init__(self, torch, d, device, epsilon=1e-4):
        self.d = int(d)
        self.stats = torch.zeros((2, 2 * self.d + 1), dtype=torch.float64, device=device)
        self.stats[:, self.d:2 * self.d] = 1.0
        self.stats[:, 2 * self.d] = epsilon
        self.scratch = torch.zeros((2, 2 * self.d), dtype=torch.float64, device=device)
        self.work = torch.zeros(_lib.rms_work_size(self.d), dtype=torch.float64, device=device)
        self.cur = 0

    @property
    def mean(self):
        return self.stats[self.cur, :self.d]

    @property
    def var(self):
        return self.stats[self.cur, self.d:2 * self.d]

    @property
    def count(self):
        return self.stats[self.cur, 2 * self.d:]


def _shard_group(env, group):
    """The process group when the batch statistics must be combined across GPUs (None otherwise): the wrapped env is
    this rank's shard of a global batch (``first_index``/``ShardedVectorEnv(gather=None)``) and torch.distributed is
    up."""
    if group is False:
        return None
    try:
        import torch.distributed as dist
    except Exception:
        return None
    if not (dist.is_available() and dist.is_initialized()):
        return None
    if group is None and not getattr(env, "shards_global_batch", False):
        return None
    return dist.group.WORLD if group in (None, True) else group


def _batch_count(torch, env, group):
    """Rows of the global batch: this shard's rows summed over the group (shards may differ in size)."""
    n = env.num_envs
    if group is None:
        return float(n)
    import torch.distributed as dist
    t = torch.tensor([n], dtype=torch.float64, device=env.unwrapped.device)
    dist.all_reduce(t, group=group)
    return float(t.item())


class NormalizeObservation(VectorWrapper):
    """obs -> (obs - running_mean) / sqrt(running_var + epsilon), statistics over the whole batch.

    ``group``: a torch.distributed process group (or True for the default one) when ``env`` is ONE RANK'S SHARD of
    a global batch: the per-column batch sums are all-reduced over the group before the running statistics are
    updated (normalize.py:32-46 applied to the global batch), so every rank normalises with the same numbers; the
    batch count is the shards' env counts summed over the group, so the shards may differ in size.

    Rows must have 1, 2, 3, 4, 6, 8 or 24 elements (``ValueError`` otherwise).  The batch moments are float64 sums
    in a fixed order (the same batch gives the same statistics bit for bit); the reference's are float32 ``np.mean``
    / ``np.var`` of float32 observations, and its outputs float64 where these are float32 (DESIGN.md §4.9)."""

    def __init__(self, env, epsilon=1e-8, group=None):
        super().__init__(env)
        import torch
        self._torch = torch
        self.num_envs, self.is_vector_env = env.num_envs, True
        self.epsilon = float(epsilon)
        d = int(np.prod(env.single_observation_space.shape))   # statistics per element of the flattened row
        if d not in _lib.NORM_WIDTHS:
            raise ValueError(f"NormalizeObservation: observation rows of {d} elements; the device kernels take "
                             f"{', '.join(map(str, _lib.NORM_WIDTHS))}")
        self.obs_rms = _RunningMeanStd(torch, d, env.unwrapped.device)
        self._out = [None, None]
        self._flip = 0
        self._group = _shard_group(env, group)
        self._count = _batch_count(torch, env, self._group)

    def _normalize(self, obs, update=True):
        torch = self._torch
        self._flip ^= 1
        if self._out[self._flip] is None or self._out[self._flip].shape != obs.shape:
            self._out[self._flip] = torch.empty_like(obs)
        out = self._out[self._flip]
        env = self.env.unwrapped
        r, lib = self.obs_rms, env._lib
        n = obs.shape[0]
        d = obs.numel() // n
        st, sc = r.stats[r.cur], r.scratch[r.cur]
        with torch.cuda.device(obs.device):
            if update:
                _lib.check(lib.b200gym_rms_moments(_p(obs), 0, n, d, _p(st), _p(sc), _p(r.work), env._stream()))
                if self._group is not None:
                    import torch.distributed as dist
                    dist.all_reduce(sc, group=self._group)
            _lib.check(lib.b200gym_rms_apply_obs(_p(obs), _p(out), n, d, _p(st), _p(r.stats[r.cur ^ 1]), _p(sc),
                                                 _p(r.scratch[r.cur ^ 1]), self._count, self.epsilon,
                                                 1 if update else 0, env._stream()))
        if update:
            r.cur ^= 1
        return out

    # snapshots: the statistics are saved and restored whole and left alone by clone; restored / cloned
    # observations are normalised without updating them
    def _has_snapshot_state(self):
        return True

    def _snapshot_extra(self, idx):
        return _rms_state(self.obs_rms)

    def _restore_extra(self, e, idx):
        _set_rms_state(self.obs_rms, e)

    def _restored_obs(self, obs):
        return self._normalize(obs, update=False)

    def reset(self, **kwargs):
        refuse_capture("NormalizeObservation.reset()", _NORM_NO_CAPTURE)
        obs, info = self.env.reset(**kwargs)
        return self._normalize(obs), info

    def step(self, actions):
        refuse_capture("NormalizeObservation.step()", _NORM_NO_CAPTURE)
        obs, rew, term, trunc, infos = self.env.step(actions)
        return self._normalize(obs), rew, term, trunc, infos


class NormalizeReward(VectorWrapper):
    """Scale rewards so that the discounted return has unit running variance (normalize.py:98-144)."""

    def __init__(self, env, gamma=0.99, epsilon=1e-8, group=None):
        super().__init__(env)
        import torch
        self._torch = torch
        self.num_envs, self.is_vector_env = env.num_envs, True
        self.gamma, self.epsilon = float(gamma), float(epsilon)
        dev = env.unwrapped.device
        self.return_rms = _RunningMeanStd(torch, 1, dev)
        self.returns = None
        self._out = [None, None]
        self._flip = 0
        self._group = _shard_group(env, group)
        self._count = _batch_count(torch, env, self._group)

    def reset(self, **kwargs):
        refuse_capture("NormalizeReward.reset()", _NORM_NO_CAPTURE)
        return self.env.reset(**kwargs)

    def step(self, actions):
        torch = self._torch
        refuse_capture("NormalizeReward.step()", _NORM_NO_CAPTURE)
        obs, rew, term, trunc, infos = self.env.step(actions)
        if self.returns is None or self.returns.shape != rew.shape:
            self.returns = torch.zeros_like(rew)
        self._flip ^= 1
        if self._out[self._flip] is None or self._out[self._flip].shape != rew.shape:
            self._out[self._flip] = torch.empty_like(rew)
        out = self._out[self._flip]
        env = self.env.unwrapped
        r, lib = self.return_rms, env._lib
        n = rew.shape[0]
        st, sc = r.stats[r.cur], r.scratch[r.cur]
        with torch.cuda.device(rew.device):
            _lib.check(lib.b200gym_return_moments(_p(self.returns), _p(rew), self.gamma, n, _p(st), _p(sc), _p(r.work),
                                                  env._stream()))
            if self._group is not None:
                import torch.distributed as dist
                dist.all_reduce(sc, group=self._group)
            _lib.check(lib.b200gym_rms_apply_reward(_p(rew), _p(out), _p(self.returns), _p(term), _p(trunc), n, _p(st),
                                                    _p(r.stats[r.cur ^ 1]), _p(sc), _p(r.scratch[r.cur ^ 1]),
                                                    self._count, self.epsilon, env._stream()))
        r.cur ^= 1
        return obs, out, term, trunc, infos

    # snapshots: the per-env discounted returns follow the envs; the statistics are saved and restored whole and
    # left alone by clone
    def _has_snapshot_state(self):
        return True

    def _returns(self):
        u = self.unwrapped
        if self.returns is None:
            self.returns = self._torch.zeros(u.num_envs, dtype=self._torch.float64, device=u.device)
        return self.returns

    def _snapshot_extra(self, idx):
        return dict(_rms_state(self.return_rms), returns=_pick(self.unwrapped, self._returns(), idx))

    def _restore_extra(self, e, idx):
        _set_rms_state(self.return_rms, e)
        _scatter(self.unwrapped, self._returns(), idx, e["returns"])

    def _clone_extra(self, src):
        self.returns = self._returns().index_select(0, src)


class VectorListInfo(VectorWrapper):
    """Dict-of-arrays ``infos`` -> list of per-env dicts (vector_list_info.py:56-111).

    Host-side adapter for agents that expect the pre-0.25 info format; it synchronises and walks the
    batch in Python, so it is meant for small batches."""

    def _to_host(self, v):
        return v.detach().cpu().numpy() if hasattr(v, "detach") else v

    def _convert(self, infos):
        n = self.env.num_envs
        out = [{} for _ in range(n)]
        for k in list(infos.keys()):
            if k.startswith("_"):
                continue
            mask = np.asarray(self._to_host(infos[f"_{k}"])).astype(bool)
            if k == "episode":  # vector_list_info.py:86-111
                ep = {kk: self._to_host(vv) for kk, vv in infos[k].items()}
                for i in np.flatnonzero(mask):
                    out[i]["episode"] = {kk: (vv[i] if np.ndim(vv) else vv) for kk, vv in ep.items()}
                continue
            vals = self._to_host(infos[k])
            for i in np.flatnonzero(mask):
                out[i][k] = vals[i]
        return out

    def reset(self, **kwargs):
        refuse_capture("VectorListInfo.reset()", "it copies infos to the host")
        obs, infos = self.env.reset(**kwargs)
        return obs, self._convert(infos)

    def step(self, actions):
        refuse_capture("VectorListInfo.step()", "it copies infos to the host")
        obs, rew, term, trunc, infos = self.env.step(actions)
        return obs, rew, term, trunc, self._convert(infos)


def step_api_compatibility(step_returns, output_truncation_bool=True, is_vector_env=True):
    """5-tuple <-> 4-tuple step API for vector envs (gym/utils/step_api_compatibility.py:24-161).

    Works on numpy arrays and torch tensors alike (``|``, ``&``, ``~`` only)."""
    if output_truncation_bool:
        if len(step_returns) == 5:
            return step_returns
        obs, rew, dones, infos = step_returns
        trunc_key = infos.get("TimeLimit.truncated") if isinstance(infos, dict) else None
        truncated = trunc_key if trunc_key is not None else dones & ~dones
        return obs, rew, dones & ~truncated, truncated, infos
    if len(step_returns) == 4:
        return step_returns
    obs, rew, terminated, truncated, infos = step_returns
    done = terminated | truncated
    # like the reference (:114-118) the key only appears in steps where some env finished (for device tensors this
    # `any` is the one host synchronisation of the adapter)
    if isinstance(infos, dict) and bool(done.any()):
        infos["TimeLimit.truncated"] = truncated & ~terminated
    return obs, rew, done, infos
