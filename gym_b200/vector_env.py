"""``B200VectorEnv`` -- gym's ``VectorEnv`` API over the CUDA engine.

Presents the contract of ``gym.vector.VectorEnv`` (reference
gym/vector/vector_env.py:12-275) with the semantics of ``SyncVectorEnv``
(gym/vector/sync_vector_env.py:90-169): ``seed + i`` fan-out, per-env TimeLimit,
same-step autoreset with ``final_observation``.  One ``step()`` is one kernel
launch through the C ABI (``include/b200gym.h``); PyTorch is used only to own
device memory and streams.

Two output backends:

``backend="torch"`` (default, the fast path)
    ``step`` returns ``torch.cuda`` tensors: obs float32 (N, D), rewards float64
    (N,), terminated/truncated bool (N,).  No host synchronisation happens in
    ``step``.  ``infos`` always carries ``final_observation`` (dense (N, D)
    tensor, rows valid where the mask is set) and the ``_final_observation`` mask
    -- a dense, sync-free form of the reference's object arrays
    (vector_env.py:235-258).  Output tensors are double-buffered: the tensors
    returned by step t stay valid until step t+2 (``copy=True`` clones instead).

``backend="numpy"`` (drop-in for CPU agents and for the parity tests)
    host buffers in, host buffers out, through ``b200gym_step_host``; returns
    exactly what ``SyncVectorEnv.step`` returns, including the object-array
    ``infos`` that only appear when some env finished.
"""
import ctypes
import os

import numpy as np

from gym_b200 import _lib, envs as _envs, error
from gym_b200.registration import spec as _spec
from gym_b200.snapshot import FORMAT_VERSION, EnvSnapshot, check_compatible, env_config, host_indices
from gym_b200.spaces import batch_space, pcg64_skip, pcg64_state

_STATE_DEFAULT, _STATE_WAITING_RESET, _STATE_WAITING_STEP = "default", "reset", "step"


def _torch():
    import torch
    return torch


def seed_words(seed):
    """Non-negative int < 2**128 -> (c_uint32 * 4) little-endian entropy words."""
    seed = int(seed)
    if seed < 0:
        raise error.Error(f"Seed must be a non-negative integer or omitted, not {seed}")
    if seed >= 1 << 128:
        raise error.Error("gym_b200 supports seeds below 2**128")
    return (ctypes.c_uint32 * 4)(*[(seed >> (32 * k)) & 0xFFFFFFFF for k in range(4)])


def _unpickle(factory, args, kwargs, payload):
    """Rebuild an env pickled by ``B200VectorEnv.__reduce__`` / ``B200Env.__reduce__`` and load its snapshot."""
    env = factory(*args, **kwargs)
    state, seeded, has_reset = payload
    env._load_snapshot_payload(EnvSnapshot.from_state_dict(state, env.device), seeded, has_reset)
    return env


class FinalInfos(dict):
    """``infos`` of the torch backend: the done mask is materialised on first access."""

    def __init__(self, final_obs, terminated, truncated):
        super().__init__(final_observation=final_obs)
        self._t, self._u = terminated, truncated

    def _mask(self):
        if not dict.__contains__(self, "_final_observation"):
            dict.__setitem__(self, "_final_observation", self._t | self._u)
        return dict.__getitem__(self, "_final_observation")

    def __getitem__(self, k):
        if k == "_final_observation":
            return self._mask()
        return dict.__getitem__(self, k)

    def __contains__(self, k):
        return k == "_final_observation" or dict.__contains__(self, k)

    def get(self, k, default=None):
        return self[k] if k in self else default

    def keys(self):
        self._mask()
        return dict.keys(self)

    def items(self):
        self._mask()
        return dict.items(self)


class B200VectorEnv:
    """``num_envs`` copies of one registered env advanced by one CUDA kernel per step.

    Args mirror ``gym.vector.make(id, num_envs, **kwargs)`` (gym/vector/__init__.py:12-73)
    plus engine knobs:
        env_id: registered id ("CartPole-v1", ...) or an ``EnvSpec``.
        num_envs: environments owned by THIS handle (one GPU).
        device: CUDA device index / torch.device (default: current device).
        max_episode_steps: overrides the registry's TimeLimit cap (``make`` kwarg).
        backend: "torch" | "numpy" (see module docstring).
        copy: clone outputs every step (reference ``copy=True``); default False for torch.
        dense_infos: numpy backend only -- return ``final_observation`` as a dense (N, D) array
            plus mask every step instead of the reference's object arrays (use for large N).
        first_index: global index of env 0 when a batch is sharded across GPUs; the
            int-seed fan-out becomes ``seed + first_index + i``.
        **kwargs: env constructor kwargs (``g`` for Pendulum, ``goal_velocity`` for MountainCar*).
    """

    is_vector_env = True

    def __init__(self, env_id, num_envs, device=None, max_episode_steps=None, backend="torch",
                 copy=None, first_index=0, autoreset=True, dense_infos=False, **kwargs):
        self.spec = _spec(env_id)
        if backend not in ("torch", "numpy"):
            raise ValueError("backend must be 'torch' or 'numpy'")
        self.backend = backend
        self.copy = (backend == "numpy") if copy is None else bool(copy)
        self.num_envs = int(num_envs)
        if self.num_envs <= 0:
            raise ValueError("num_envs must be positive")
        self.first_index = int(first_index)
        self.dense_infos = bool(dense_infos)
        self.closed = True  # until construction succeeds
        self._handle = None
        ctor_kwargs = dict(self.spec.kwargs)
        ctor_kwargs.update(kwargs)
        self.kind, cfg_flags = _envs.resolve_variant(self.spec.kind, ctor_kwargs)
        self._info = _envs.KINDS[self.kind]
        self.metadata = dict(self._info.metadata)
        self.render_mode = None
        self.reward_range = (-float("inf"), float("inf"))

        params = _envs.resolve_params(self.kind, ctor_kwargs)
        self.env_kwargs = {k: v for k, v in ctor_kwargs.items() if k not in ("render_mode", "wind_idx", "torque_idx")}
        mes = self.spec.max_episode_steps if max_episode_steps is None else max_episode_steps
        self.max_episode_steps = None if (mes is None or int(mes) <= 0) else int(mes)

        self.single_observation_space, self.single_action_space = self._info.spaces(params)
        self.observation_space = batch_space(self.single_observation_space, n=self.num_envs)
        self.action_space = batch_space(self.single_action_space, n=self.num_envs)
        self.obs_dim = self.single_observation_space.shape[0]
        self.discrete = hasattr(self.single_action_space, "n")
        self.act_dim = 0 if self.discrete else self.single_action_space.shape[0]
        self._sample_cache = None   # (single action space, its sample_actions plan)

        lib = _lib.load()
        torch = _torch()
        if not torch.cuda.is_available():
            raise error.DependencyNotInstalled(
                "gym_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback")
        if device is None:
            index = torch.cuda.current_device()
        elif isinstance(device, int):
            index = device
        else:
            dev = torch.device(device)
            index = torch.cuda.current_device() if dev.index is None else dev.index
        self.device = torch.device("cuda", index)
        torch.cuda.init()
        with torch.cuda.device(self.device):
            torch.empty(1, device=self.device)  # make sure the primary context exists
            cfg = _lib.Config(kind=self.kind, max_episode_steps=self.max_episode_steps or 0,
                              autoreset=1 if autoreset else 0, flags=cfg_flags)
            for k in range(4):
                cfg.param[k] = params[k]
            handle = ctypes.c_void_p()
            _lib.check(lib.b200gym_create(ctypes.byref(cfg), self.num_envs, index, ctypes.byref(handle)))
        self._lib = lib
        self._handle = handle
        self.autoreset = bool(autoreset)
        self._params, self._cfg_flags = list(params), cfg_flags
        self._obs_dev = None
        if cfg_flags & _lib.LUNAR_ENABLE_WIND:
            # LunarLander.__init__ draws wind_idx, then torque_idx, from numpy's GLOBAL generator, once per env
            # object (lunar_lander.py:234-235); SyncVectorEnv builds the objects in index order.  `wind_idx=` /
            # `torque_idx=` (ints or arrays) pin them instead -- an engine extension for reproducible runs.
            draws = np.random.randint(-9999, 9999, size=2 * self.num_envs).reshape(self.num_envs, 2)
            wind = np.ascontiguousarray(np.broadcast_to(ctor_kwargs.get("wind_idx", draws[:, 0]), (self.num_envs,)),
                                        dtype=np.int32)
            torque = np.ascontiguousarray(np.broadcast_to(ctor_kwargs.get("torque_idx", draws[:, 1]), (self.num_envs,)),
                                          dtype=np.int32)
            _lib.check(lib.b200gym_lunar_wind_idx(handle, wind.ctypes.data, torque.ctypes.data, 1), handle)
        self.closed = False
        self._seeded = False
        self._has_reset = False
        self._state = _STATE_DEFAULT
        self._pending = None
        self._flip = 0
        self._out = None
        self._hio = None
        if backend == "torch":
            self._out = [self._alloc_outputs(), self._alloc_outputs()]
        else:
            self._map_host_buffers()

    # ------------------------------------------------------------------ buffers
    def _alloc_outputs(self):
        """One set of caller-owned output tensors (obs, reward, terminated, truncated, final_obs)."""
        torch = _torch()
        n, d, dev = self.num_envs, self.obs_dim, self.device
        return dict(
            obs=torch.zeros((n, d), dtype=torch.float32, device=dev),
            reward=torch.zeros((n,), dtype=torch.float64, device=dev),
            terminated=torch.zeros((n,), dtype=torch.bool, device=dev),
            truncated=torch.zeros((n,), dtype=torch.bool, device=dev),
            final_obs=torch.zeros((n, d), dtype=torch.float32, device=dev),
        )

    def _map_host_buffers(self):
        """numpy views of the library's page-locked staging buffers (b200gym_host_buffers)."""
        hio = _lib.HostIO()
        _lib.check(self._lib.b200gym_host_buffers(self._handle, ctypes.byref(hio)), self._handle)
        n, d = self.num_envs, self.obs_dim

        def view(ptr, ctype, shape, dtype):
            count = int(np.prod(shape))
            buf = (ctype * count).from_address(ptr)
            return np.frombuffer(buf, dtype=dtype).reshape(shape)

        if self.discrete:
            actions = view(hio.actions, ctypes.c_int64, (n,), np.int64)
        else:
            actions = view(hio.actions, ctypes.c_float, (n, self.act_dim), np.float32)
        self._hio = dict(
            actions=actions,
            obs=view(hio.obs, ctypes.c_float, (n, d), np.float32),
            reward=view(hio.reward, ctypes.c_double, (n,), np.float64),
            terminated=view(hio.terminated, ctypes.c_uint8, (n,), np.uint8),
            truncated=view(hio.truncated, ctypes.c_uint8, (n,), np.uint8),
            final_obs=view(hio.final_obs, ctypes.c_float, (n, d), np.float32),
        )

    def _stream(self):
        return ctypes.c_void_p(_torch().cuda.current_stream(self.device).cuda_stream)

    # ------------------------------------------------------------------ guards
    def _assert_open(self, what):
        if self.closed:
            raise error.ClosedEnvironmentError(f"Trying to operate on `{type(self).__name__}`, after a call to `close()`."
                                               if what is None else
                                               f"Trying to call `{what}` on `{type(self).__name__}` after `close()`.")

    # ------------------------------------------------------------------ seeding
    def seed(self, seed=None):
        """int -> env i gets ``seed + first_index + i``; list -> per-env seeds (None keeps a stream)."""
        self._assert_open("seed")
        if seed is None:
            if not self._seeded:
                # unseeded envs draw OS entropy (gym/utils/seeding.py:24 with seed=None)
                base = int.from_bytes(os.urandom(15), "little")
                _lib.check(self._lib.b200gym_seed_range(self._handle, seed_words(base), self.first_index,
                                                        self._stream()), self._handle)
                self._seeded = True
            return
        if isinstance(seed, (int, np.integer)):
            if seed < 0:
                raise error.Error(f"Seed must be a non-negative integer or omitted, not {seed}")
            _lib.check(self._lib.b200gym_seed_range(self._handle, seed_words(seed), self.first_index,
                                                    self._stream()), self._handle)
            self._seeded = True
            return
        seeds = list(seed)
        assert len(seeds) == self.num_envs, "one seed per environment is required"
        ent = np.zeros((self.num_envs, 4), dtype=np.uint32)
        mask = np.ones(self.num_envs, dtype=np.uint8)
        for i, s in enumerate(seeds):
            if s is None:
                mask[i] = 0
                continue
            if not (isinstance(s, (int, np.integer)) and s >= 0):
                raise error.Error(f"Seed must be a non-negative integer or omitted, not {s}")
            ent[i] = list(seed_words(s))
        if not self._seeded and not mask.all():
            self.seed(None)
        _lib.check(self._lib.b200gym_seed_each(self._handle, ent.ctypes.data, mask.ctypes.data, self._stream()),
                   self._handle)
        self._seeded = True

    # ------------------------------------------------------------------ reset
    def reset_async(self, seed=None, options=None):
        """Launch the reset kernel (the GPU is the asynchronous worker)."""
        self._assert_open("reset_async")
        if self._state != _STATE_DEFAULT:
            raise error.AlreadyPendingCallError(
                f"Calling `reset_async` while waiting for a pending call to `{self._state}` to complete",
                self._state)
        bounds = _envs.parse_reset_bounds(self.kind, options)
        self.seed(seed)
        bptr = None
        if bounds is not None:
            barr = (ctypes.c_double * 2)(*bounds)
            bptr = ctypes.cast(barr, ctypes.c_void_p)
        if self.backend == "torch":
            out = self._out[self._flip]
            _lib.check(self._lib.b200gym_reset(self._handle, None, bptr, ctypes.c_void_p(out["obs"].data_ptr()),
                                               self._stream()), self._handle)
            self._pending = out
        else:
            _torch().cuda.current_stream(self.device).synchronize()  # seeding ran on torch's stream
            _lib.check(self._lib.b200gym_reset_host(self._handle, None, bptr, None), self._handle)
        self._has_reset = True
        self._state = _STATE_WAITING_RESET

    def reset_wait(self, seed=None, options=None):
        self._assert_open("reset_wait")
        if self._state != _STATE_WAITING_RESET:
            raise error.NoAsyncCallError("Calling `reset_wait` without any prior call to `reset_async`.",
                                         _STATE_WAITING_RESET)
        self._state = _STATE_DEFAULT
        if self.backend == "torch":
            obs = self._pending["obs"]
            return (obs.clone() if self.copy else obs), {}
        obs = self._hio["obs"]
        return (obs.copy() if self.copy else obs), {}

    def reset(self, *, seed=None, options=None):
        """Reset every env; ``seed`` int fans out as seed+i (sync_vector_env.py:106-107)."""
        self.reset_async(seed=seed, options=options)
        return self.reset_wait(seed=seed, options=options)

    # ------------------------------------------------------------------ step
    def _device_actions(self, actions):
        """Bring `actions` to a contiguous device tensor of a dtype the kernel reads directly."""
        torch = _torch()
        if not isinstance(actions, torch.Tensor):
            actions = torch.as_tensor(np.asarray(actions))
        if self.discrete:
            if actions.dtype == torch.int64:
                code = _lib.ACT_I64
            elif actions.dtype == torch.int32:
                code = _lib.ACT_I32
            elif actions.dtype == torch.uint8:
                code = _lib.ACT_U8
            elif actions.dtype in (torch.int16, torch.int8, torch.bool):
                actions, code = actions.to(torch.int32), _lib.ACT_I32
            else:
                raise error.InvalidAction(f"Discrete actions must be integers, got {actions.dtype}")
            shape = (self.num_envs,)
        else:
            if actions.dtype != torch.float32:
                actions = actions.to(torch.float32)  # the Box dtype (e.g. pendulum.py:113-115)
            code = _lib.ACT_F32
            shape = (self.num_envs, self.act_dim)
        if actions.numel() != int(np.prod(shape)):
            raise error.InvalidAction(f"expected actions of shape {shape}, got {tuple(actions.shape)}")
        if actions.device != self.device:
            actions = actions.to(self.device, non_blocking=True)
        return actions.reshape(shape).contiguous(), code

    def step_async(self, actions):
        """Launch the fused step kernel on the current stream (no host sync)."""
        self._assert_open("step_async")
        if self._state != _STATE_DEFAULT:
            raise error.AlreadyPendingCallError(
                f"Calling `step_async` while waiting for a pending call to `{self._state}` to complete.",
                self._state)
        if not self._has_reset:
            raise error.ResetNeeded("Cannot call env.step() before calling env.reset()")
        if self.backend == "torch":
            # the reference asserts on an out-of-range Discrete action (cartpole.py:132); the device cannot raise and
            # this backend never waits for it, so the kernels flag it in host-visible memory and the error surfaces
            # at the next call (no synchronisation unless the flag is up)
            if self.discrete and self._lib.b200gym_invalid_seen(self._handle) == 1:
                self.check_actions()
            self._raise_snapshot_index_error()
            act, code = self._device_actions(actions)
            self._flip ^= 1
            out = self._out[self._flip]
            _lib.check(self._lib.b200gym_step(
                self._handle, ctypes.c_void_p(act.data_ptr()), code,
                ctypes.c_void_p(out["obs"].data_ptr()), ctypes.c_void_p(out["reward"].data_ptr()),
                ctypes.c_void_p(out["terminated"].data_ptr()), ctypes.c_void_p(out["truncated"].data_ptr()),
                ctypes.c_void_p(out["final_obs"].data_ptr()), self._stream()), self._handle)
            self._pending = out
            self._last_actions = act  # keep alive until the kernel has consumed it
        else:
            a = np.asarray(actions.cpu() if hasattr(actions, "cpu") else actions)
            if self.discrete:
                if not np.issubdtype(a.dtype, np.integer):
                    raise error.InvalidAction(f"Discrete actions must be integers, got {a.dtype}")
                a = np.ascontiguousarray(a.reshape(self.num_envs))
                # small batches are validated before anything is stepped, like the reference's assert
                # (cartpole.py:131-132); large ones rely on the kernel's own check (two passes over 2^20
                # actions on the host would cost more than the whole step) and raise right after the call
                if a.size <= 4096 and a.size and (a.min() < 0 or a.max() >= self.single_action_space.n):
                    bad = a[(a < 0) | (a >= self.single_action_space.n)][0]
                    raise error.InvalidAction(f"{bad!r} ({type(bad)}) invalid")
                code = {np.dtype(np.int64): _lib.ACT_I64, np.dtype(np.int32): _lib.ACT_I32,
                        np.dtype(np.uint8): _lib.ACT_U8}.get(a.dtype)
                if code is None:
                    a, code = a.astype(np.int64), _lib.ACT_I64
            else:
                a = np.ascontiguousarray(a, dtype=np.float32).reshape(self.num_envs, self.act_dim)
                code = _lib.ACT_F32
            h = self._hio
            # actions are read straight from the caller's array; the kernel writes the results into the
            # page-locked, device-mapped staging buffers; the invalid-action count comes back with the call
            count = ctypes.c_int64(0)
            _lib.check(self._lib.b200gym_step_host(
                self._handle, a.ctypes.data, code, None, None, None, None,
                h["final_obs"].ctypes.data if self.autoreset else None, ctypes.byref(count)), self._handle)
            if count.value:
                raise error.InvalidAction(f"{count.value} out-of-range Discrete action(s) were passed to step(); "
                                          "those environments were left untouched (NaN reward), the others have "
                                          "been stepped")
        self._state = _STATE_WAITING_STEP

    def step_wait(self, timeout=None):
        self._assert_open("step_wait")
        if self._state != _STATE_WAITING_STEP:
            raise error.NoAsyncCallError("Calling `step_wait` without any prior call to `step_async`.",
                                         _STATE_WAITING_STEP)
        self._state = _STATE_DEFAULT
        if self.backend == "torch":
            o = self._pending
            if self.copy:
                o = {k: v.clone() for k, v in o.items()}
            infos = FinalInfos(o["final_obs"], o["terminated"], o["truncated"])
            return o["obs"], o["reward"], o["terminated"], o["truncated"], infos
        h = self._hio
        term = h["terminated"].view(np.bool_)   # the kernel writes 0/1 bytes
        trunc = h["truncated"].view(np.bool_)
        obs, reward = h["obs"], h["reward"]
        if self.copy:
            obs, reward, term, trunc = obs.copy(), reward.copy(), term.copy(), trunc.copy()
        infos = {}
        if self.autoreset and self.dense_infos:
            # dense form for large batches: (N, D) array + mask (materialised on first access), no Python loop
            fo = h["final_obs"].copy() if self.copy else h["final_obs"]
            infos = FinalInfos(fo, term, trunc)
        elif self.autoreset:
            done = term | trunc
            if done.any():
                # vector_env.py:208-258: object arrays + `_key` masks, only when some env finished
                fo = np.full(self.num_envs, None, dtype=object)
                fi = np.full(self.num_envs, None, dtype=object)
                for i in np.flatnonzero(done):
                    fo[i] = h["final_obs"][i].copy()
                    fi[i] = {}
                infos = {"final_observation": fo, "_final_observation": done.copy(),
                         "final_info": fi, "_final_info": done.copy()}
        return obs, reward, term, trunc, infos

    def step(self, actions):
        """One SyncVectorEnv.step: (obs, rewards, terminateds, truncateds, infos)."""
        self.step_async(actions)
        return self.step_wait()

    def check_actions(self):
        """Number of out-of-range Discrete actions the device saw since the last check (syncs)."""
        count = ctypes.c_int64(0)
        _lib.check(self._lib.b200gym_invalid_actions(self._handle, self._stream(), ctypes.byref(count)),
                   self._handle)
        if count.value:
            raise error.InvalidAction(f"{count.value} out-of-range Discrete action(s) were passed to step()")
        return 0

    # ------------------------------------------------------------------ action sampling
    def _sample_plan(self):
        """(n_choices, cols, low, high) of the single action space, checked once per space object: Discrete(n) from 0
        batches to MultiDiscrete (n_choices = n), a bounded float32 Box of shape (A,) to a Box of shape (N, A)."""
        single = self.single_action_space
        if self._sample_cache is not None and self._sample_cache[0] is single:
            return self._sample_cache[1]
        if hasattr(single, "n") and int(getattr(single, "start", 0)) == 0:
            plan = (int(single.n), 1, None, None)
        elif (hasattr(single, "low") and np.dtype(single.dtype) == np.float32 and len(single.shape) == 1
              and 1 <= single.shape[0] <= 32 and np.all(np.isfinite(single.low)) and np.all(np.isfinite(single.high))):
            plan = (0, int(single.shape[0]), np.ascontiguousarray(single.low, dtype=np.float64),
                    np.ascontiguousarray(single.high, dtype=np.float64))
        else:
            raise error.Error(f"sample_actions supports Discrete(n) and bounded float32 Box action spaces, not {single!r}")
        self._sample_cache = (single, plan)
        return plan

    def sample_actions(self):
        """``self.action_space.sample()``, drawn on the device: the same values bit for bit (int64 (N,) for Discrete
        kinds, float32 (N, A) for continuous ones) as a tensor on ``self.device``, enqueued on torch's current stream
        with no synchronisation, ready for ``step()``.  The space's generator ends where ``sample()`` would leave it,
        so host and device sampling interleave freely.  ``backend="numpy"`` returns ``self.action_space.sample()``."""
        self._assert_open("sample_actions")
        space = self.action_space
        if self.backend == "numpy":
            return space.sample()
        n_choices, cols, low, high = self._sample_plan()
        shape = (self.num_envs,) if n_choices else (self.num_envs, cols)
        if (type(space).__name__ != ("MultiDiscrete" if n_choices else "Box") or tuple(space.shape) != shape
                or np.dtype(space.dtype) != (np.int64 if n_choices else np.float32)):
            raise error.Error(f"action_space {space!r} is no longer the batched space of {self.single_action_space!r}")
        bit_generator = space.np_random.bit_generator
        state = pcg64_state(bit_generator)
        s, inc = state["state"]["state"], state["state"]["inc"]
        mask = (1 << 64) - 1
        words = (ctypes.c_uint64 * 4)(s >> 64, s & mask, inc >> 64, inc & mask)
        torch = _torch()
        out = torch.empty(shape, dtype=torch.int64 if n_choices else torch.float32, device=self.device)
        _lib.check(self._lib.b200gym_sample_space(words, self.num_envs, cols, n_choices,
                                                  None if low is None else low.ctypes.data,
                                                  None if high is None else high.ctypes.data,
                                                  ctypes.c_void_p(out.data_ptr()), self._stream()))
        pcg64_skip(bit_generator, state, out.numel())
        return out

    # ------------------------------------------------------------------ state access
    def get_state(self):
        """(state float64 (N, S), elapsed int32 (N,), rng uint64 (N, 4)) as device tensors."""
        self._assert_open("get_state")
        torch = _torch()
        S = self._lib.b200gym_state_dim(self.kind)
        st = torch.empty((self.num_envs, S), dtype=torch.float64, device=self.device)
        el = torch.empty((self.num_envs,), dtype=torch.int32, device=self.device)
        rng = torch.empty((self.num_envs, 4), dtype=torch.int64, device=self.device)
        _lib.check(self._lib.b200gym_get_state(self._handle, ctypes.c_void_p(st.data_ptr()),
                                               ctypes.c_void_p(el.data_ptr()), ctypes.c_void_p(rng.data_ptr()),
                                               self._stream()), self._handle)
        return st, el, rng

    def lunar_bodies(self):
        """LunarLander only: (bodies float32 (N, 3, 6) = {c.x, c.y, angle, v.x, v.y, omega} of lander, leg(-1),
        leg(+1); flags int32 (N, 6) = {game_over, leg0, leg1, awake, elapsed, #touching contacts})."""
        self._assert_open("lunar_bodies")
        torch = _torch()
        bodies = torch.empty((self.num_envs, 18), dtype=torch.float32, device=self.device)
        flags = torch.empty((self.num_envs, 6), dtype=torch.int32, device=self.device)
        _lib.check(self._lib.b200gym_lunar_get_bodies(self._handle, ctypes.c_void_p(bodies.data_ptr()),
                                                      ctypes.c_void_p(flags.data_ptr()), self._stream()), self._handle)
        return bodies.view(self.num_envs, 3, 6), flags

    def box2d_overflows(self):
        """Box2D tasks: number of envs in which a touching pair was ever dropped because the scene's manifold table
        (8 pairs for LunarLander*, 10 for BipedalWalker*) was full -- i.e. where the physics knowingly departs from
        Box2D (include/b200gym.h: b200gym_box2d_overflows).  Synchronises."""
        self._assert_open("box2d_overflows")
        count = ctypes.c_int64(0)
        _lib.check(self._lib.b200gym_box2d_overflows(self._handle, self._stream(), ctypes.byref(count)), self._handle)
        return int(count.value)

    def box2d_list_counts(self, slots=1):
        """Box2D tasks, a diagnostic: (parked, resets) int32 arrays of `slots` entries -- how many envs the last step
        parked for the TOI kernel and queued for the compacted reset kernel, per launch range (the torch backend
        runs one range, counted in slot 0; the numpy backend counts chunk c in slot c).  A pass that runs inline
        leaves its counter at 0 (include/b200gym.h: b200gym_box2d_list_counts).  Synchronises."""
        self._assert_open("box2d_list_counts")
        parked = np.zeros(slots, dtype=np.int32)
        resets = np.zeros(slots, dtype=np.int32)
        _lib.check(self._lib.b200gym_box2d_list_counts(self._handle, self._stream(), int(slots), parked.ctypes.data,
                                                       resets.ctypes.data), self._handle)
        return parked, resets

    def lunar_wind_idx(self):
        """LunarLander(enable_wind=True) only: the per-env (wind_idx, torque_idx) int32 arrays
        (lunar_lander.py:234-235,461,472), read back from the device."""
        self._assert_open("lunar_wind_idx")
        wind = np.zeros(self.num_envs, dtype=np.int32)
        torque = np.zeros(self.num_envs, dtype=np.int32)
        _lib.check(self._lib.b200gym_lunar_wind_idx(self._handle, wind.ctypes.data, torque.ctypes.data, 0), self._handle)
        return wind, torque

    def walker_bodies(self):
        """BipedalWalker only: (bodies float32 (N, 5, 6) of hull, leg(-1), lower(-1), leg(+1), lower(+1);
        flags int32 (N, 4) = {game_over, legs[1] contact, legs[3] contact, #touching contacts})."""
        self._assert_open("walker_bodies")
        torch = _torch()
        bodies = torch.empty((self.num_envs, 30), dtype=torch.float32, device=self.device)
        flags = torch.empty((self.num_envs, 4), dtype=torch.int32, device=self.device)
        _lib.check(self._lib.b200gym_walker_get_bodies(self._handle, ctypes.c_void_p(bodies.data_ptr()),
                                                       ctypes.c_void_p(flags.data_ptr()), self._stream()), self._handle)
        return bodies.view(self.num_envs, 5, 6), flags

    def set_state(self, state=None, elapsed=None, rng=None):
        self._assert_open("set_state")
        torch = _torch()

        def prep(x, dtype):
            if x is None:
                return None, None
            t = torch.as_tensor(x).to(device=self.device, dtype=dtype).contiguous()
            return t, ctypes.c_void_p(t.data_ptr())

        st, pst = prep(state, torch.float64)
        el, pel = prep(elapsed, torch.int32)
        if rng is not None and not isinstance(rng, torch.Tensor):
            rng = torch.as_tensor(np.ascontiguousarray(rng).view(np.int64))
        rg, prg = prep(rng, torch.int64)
        _lib.check(self._lib.b200gym_set_state(self._handle, pst, pel, prg, self._stream()), self._handle)
        torch.cuda.current_stream(self.device).synchronize()
        if rng is not None:
            self._seeded = True
        if state is not None:
            self._has_reset = True

    # ------------------------------------------------------------------ snapshots
    # What pickle / deepcopy carry for a reference env (env.state, np_random, TimeLimit._elapsed_steps), taken for
    # any subset of the batch, on the device (include/b200gym.h: b200gym_snapshot_*, b200gym_clone).
    @property
    def snapshot_row_bytes(self):
        return int(self._lib.b200gym_snapshot_row_bytes(self.kind))

    def _snapshot_header(self):
        return {"version": FORMAT_VERSION, "kind": self.kind, "row_bytes": self.snapshot_row_bytes,
                "config": env_config(self.max_episode_steps, self.autoreset, self._params, self._cfg_flags)}

    def _raise_snapshot_index_error(self):
        if self._lib.b200gym_snapshot_index_error(self._handle) == 1:
            raise error.Error("an earlier snapshot(), restore() or clone() was given an out-of-range index; "
                              "those entries were skipped")

    def _index_tensor(self, indices, what):
        """None -> None; a CUDA tensor -> int64 on this device (range-checked by the kernels, reported by the next
        call); anything else -> checked on the host, then copied to the device."""
        if indices is None:
            return None
        torch = _torch()
        if isinstance(indices, torch.Tensor) and indices.is_cuda:
            if indices.dim() != 1 or indices.dtype.is_floating_point or indices.dtype == torch.bool:
                raise error.Error(f"{what} must be a 1-D integer tensor, got {indices.dtype} of shape "
                                  f"{tuple(indices.shape)}")
            return indices.to(device=self.device, dtype=torch.int64).contiguous()
        if isinstance(indices, torch.Tensor):
            indices = indices.numpy()
        return torch.from_numpy(host_indices(indices, self.num_envs, what)).to(self.device)

    def _in_range(self, idx, fallback):
        """idx with every out-of-range entry replaced by `fallback`'s: torch indexing must never see one."""
        torch = _torch()
        return torch.where((idx >= 0) & (idx < self.num_envs), idx, fallback)

    def _last_obs(self):
        """Device tensor (N, D) of the observations last returned (numpy backend: a view of the mapped staging
        buffer, written by the device without a host copy)."""
        if self.backend == "torch":
            return self._out[self._flip]["obs"]
        if self._obs_dev is None:
            from gym_b200.distributed import _DeviceMemory
            h = self._hio["obs"]   # page-locked and mapped: under unified addressing its host address is its device one
            self._obs_dev = _torch().as_tensor(_DeviceMemory(h.ctypes.data, h.shape, "<f4"), device=self.device)
        return self._obs_dev

    def _next_obs(self):
        """Where restored / cloned observations go: the next set of the double buffer (the step-(t+2) rule holds),
        or the staging buffer on the numpy backend."""
        if self.backend == "torch":
            self._flip ^= 1
            return self._out[self._flip]["obs"]
        return self._last_obs()

    def _obs_result(self, obs):
        if self.backend == "torch":
            return obs.clone() if self.copy else obs
        _torch().cuda.current_stream(self.device).synchronize()
        self._raise_snapshot_index_error()
        obs = self._hio["obs"]
        return obs.copy() if self.copy else obs

    def _check_idle(self, what):
        self._assert_open(what)
        if self._state != _STATE_DEFAULT:
            raise error.AlreadyPendingCallError(f"Calling `{what}` while waiting for a pending call to `{self._state}` "
                                                "to complete", self._state)
        self._raise_snapshot_index_error()

    def snapshot(self, indices=None):
        """-> ``EnvSnapshot`` of envs ``indices`` (default: all, in order): their engine state as device rows, the
        observations last returned for them and a header (format version, kind, row bytes, construction config)."""
        self._check_idle("snapshot")
        torch = _torch()
        idx = self._index_tensor(indices, "snapshot indices")
        m = self.num_envs if idx is None else int(idx.shape[0])
        rows = torch.empty((m, self.snapshot_row_bytes), dtype=torch.uint8, device=self.device)
        with torch.cuda.device(self.device):
            if m:
                _lib.check(self._lib.b200gym_snapshot_save(
                    self._handle, None if idx is None else ctypes.c_void_p(idx.data_ptr()), m,
                    ctypes.c_void_p(rows.data_ptr()), self._stream()), self._handle)
            obs = self._last_obs()
            obs = obs.clone() if idx is None else obs.index_select(0, self._in_range(idx, 0))
        if self.backend == "numpy":
            torch.cuda.current_stream(self.device).synchronize()
            self._raise_snapshot_index_error()
        return EnvSnapshot(self._snapshot_header(), rows, obs)

    def restore(self, snap, indices=None):
        """Load ``snap`` (row k into env ``indices[k]``; default: all envs, in order) -> ``(obs, {})`` like ``reset``,
        with the observations the snapshot was taken with.  The other envs are left as they are.  A snapshot of
        another kind or construction config raises ``error.Error``."""
        self._check_idle("restore")
        check_compatible(snap.header, self.kind, self.snapshot_row_bytes,
                         env_config(self.max_episode_steps, self.autoreset, self._params, self._cfg_flags))
        torch = _torch()
        m, n = len(snap), self.num_envs
        idx = self._index_tensor(indices, "restore indices")
        if idx is None and m != n:
            raise error.Error(f"a snapshot of {m} envs restores into {n} envs only with indices=")
        if idx is not None and int(idx.shape[0]) != m:
            raise error.Error(f"{int(idx.shape[0])} indices given for a snapshot of {m} envs")
        rows, sobs = snap.rows.to(self.device), snap.obs.to(self.device)
        with torch.cuda.device(self.device):
            if m:
                _lib.check(self._lib.b200gym_snapshot_load(
                    self._handle, ctypes.c_void_p(rows.data_ptr()), None,
                    None if idx is None else ctypes.c_void_p(idx.data_ptr()), m, self._stream()), self._handle)
            prev = self._last_obs()
            target = self._next_obs()
            if idx is None:
                target.copy_(sobs)
            else:   # row n of the scratch takes the observations of skipped (out-of-range) entries
                tmp = torch.empty((n + 1, self.obs_dim), dtype=torch.float32, device=self.device)
                tmp[:n].copy_(prev)
                tmp.index_copy_(0, self._in_range(idx, n), sobs)
                target.copy_(tmp[:n])
        if idx is None:
            self._has_reset = self._seeded = True
        return self._obs_result(target), {}

    def clone(self, src):
        """Env i becomes a copy of env ``src[i]`` for every i (duplicates allowed), on the device -> the new
        observations, gathered from the last ones."""
        self._check_idle("clone")
        torch = _torch()
        src = self._index_tensor(src, "clone sources")
        if src is None or int(src.shape[0]) != self.num_envs:
            raise error.Error(f"clone needs one source per env ({self.num_envs})")
        with torch.cuda.device(self.device):
            _lib.check(self._lib.b200gym_clone(self._handle, ctypes.c_void_p(src.data_ptr()), self._stream()),
                       self._handle)
            g = self._in_range(src, torch.arange(self.num_envs, device=self.device))   # a skipped env keeps its obs
            prev = self._last_obs()
            target = self._next_obs()
            if target is prev:
                target.copy_(prev.index_select(0, g))
            else:
                torch.index_select(prev, 0, g, out=target)
        return self._obs_result(target)

    # ------------------------------------------------------------------ pickle / deepcopy
    _pickle_factory = None   # module-level callable that rebuilds this class (gym_compat's classes are built at run time)

    def _rebuild_env_kwargs(self):
        kw = dict(self.env_kwargs)
        if self._cfg_flags & _lib.LUNAR_ENABLE_WIND:
            kw.update(wind_idx=0, torque_idx=0)   # the counters come back with the rows: no draw from numpy's generator
        return kw

    def _rebuild_args(self):
        kw = self._rebuild_env_kwargs()
        kw.update(device=self.device.index, max_episode_steps=self.max_episode_steps or 0, backend=self.backend,
                  copy=self.copy, first_index=self.first_index, autoreset=self.autoreset, dense_infos=self.dense_infos)
        return (self.spec, self.num_envs), kw

    def _load_snapshot_payload(self, snap, seeded, has_reset):
        self.restore(snap)
        self._seeded, self._has_reset = seeded, has_reset

    def __reduce__(self):
        """pickle: the constructor arguments + a host copy of the whole snapshot; unpickling rebuilds the handle on
        the same device index and loads the rows, so the copy continues bit-identically."""
        self._assert_open("pickle")
        args, kwargs = self._rebuild_args()
        payload = (self.snapshot().state_dict(), self._seeded, self._has_reset)
        return _unpickle, (type(self)._pickle_factory or type(self), args, kwargs, payload)

    def __deepcopy__(self, memo):
        """A new handle on the same device loaded from a snapshot, device to device."""
        self._assert_open("deepcopy")
        args, kwargs = self._rebuild_args()
        new = (type(self)._pickle_factory or type(self))(*args, **kwargs)
        new._load_snapshot_payload(self.snapshot(), self._seeded, self._has_reset)
        return new

    # ------------------------------------------------------------------ call / attrs
    def call_async(self, name, *args, **kwargs):
        self._assert_open("call_async")
        self._call = (name, args, kwargs)

    def call_wait(self, timeout=None):
        name, args, kwargs = self._call
        if name in ("wind_idx", "torque_idx") and self.env_kwargs.get("enable_wind", False):
            return tuple(int(v) for v in self.lunar_wind_idx()[name == "torque_idx"])
        value = self._attr(name)
        return tuple([value] * self.num_envs)

    def call(self, name, *args, **kwargs):
        """vector_env.py:146-159.  Serves the read-only attributes of the reference env class."""
        self.call_async(name, *args, **kwargs)
        return self.call_wait()

    def _attr(self, name):
        if name in self.env_kwargs:
            return self.env_kwargs[name]
        if name in self._info.attrs:
            return self._info.attrs[name]
        if name in self._info.kwargs:
            return self._info.kwargs[name][1]
        if name in ("spec", "metadata", "render_mode", "reward_range"):
            return getattr(self, name)
        if name in ("observation_space", "action_space"):
            return getattr(self, "single_" + name)
        if name == "_max_episode_steps":
            return self.max_episode_steps
        raise AttributeError(f"'{self._info.name}' env has no attribute '{name}' in gym_b200")

    def walker_terrain(self):
        """BipedalWalker* only: (terrain_y float32 (N, 200); obstacle boxes float32 (N, 40, 4) = {x0, y_low, x1,
        y_high} in creation order; number of boxes int32 (N,)) -- `env.terrain_y` and the hardcore `fd_polygon`
        bodies of the reference (bipedal_walker.py:309-316,336,365,377)."""
        self._assert_open("walker_terrain")
        torch = _torch()
        terrain = torch.empty((self.num_envs, 200), dtype=torch.float32, device=self.device)
        polys = torch.empty((self.num_envs, 40, 4), dtype=torch.float32, device=self.device)
        npoly = torch.empty((self.num_envs,), dtype=torch.int32, device=self.device)
        _lib.check(self._lib.b200gym_walker_get_terrain(self._handle, ctypes.c_void_p(terrain.data_ptr()),
                                                        ctypes.c_void_p(polys.data_ptr()), ctypes.c_void_p(npoly.data_ptr()),
                                                        self._stream()), self._handle)
        return terrain, polys, npoly

    def get_attr(self, name):
        return self.call(name)

    def set_attr(self, name, values):
        """vector_env.py:171-180: sub-env attributes are fixed at construction in the engine."""
        raise AttributeError(
            f"gym_b200 fixes env attributes at construction; pass `{name}` as a constructor kwarg instead")

    # ------------------------------------------------------------------ lifecycle
    def close_extras(self, **kwargs):
        if self._handle is not None:
            try:
                _torch().cuda.synchronize(self.device)
            except Exception:
                pass
            self._hio = None
            self._lib.b200gym_destroy(self._handle)
            self._handle = None

    def close(self, **kwargs):
        """vector_env.py:182-206: idempotent."""
        if self.closed:
            return
        self.close_extras(**kwargs)
        self.closed = True

    def __del__(self):
        if not getattr(self, "closed", True):
            self.close()

    @property
    def unwrapped(self):
        return self

    def __repr__(self):
        return f"{type(self).__name__}({self.spec.id}, {self.num_envs})"
