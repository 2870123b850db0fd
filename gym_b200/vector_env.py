"""``B200VectorEnv`` -- gym's ``VectorEnv`` API over the CUDA engine.

Presents the contract of ``gym.vector.VectorEnv`` (reference
gym/vector/vector_env.py:12-275) with the semantics of ``SyncVectorEnv``
(gym/vector/sync_vector_env.py:90-169): ``seed + i`` fan-out, per-env TimeLimit,
same-step autoreset with ``final_observation``.  One ``step()`` is one kernel
launch through the C ABI (``include/b200gym.h``); PyTorch is used only to own
device memory and streams.

Two output backends:

``backend="torch"`` (default, the fast path)
    ``step`` returns ``torch.cuda`` tensors: obs float32 (N, D) (with per-env wrappers: (N,) +
    ``single_observation_space.shape``), rewards float64
    (N,), terminated/truncated bool (N,).  No host synchronisation happens in
    ``step``.  ``infos`` always carries ``final_observation`` (dense (N, D)
    tensor, rows valid where the mask is set) and the ``_final_observation`` mask
    -- a dense, sync-free form of the reference's object arrays
    (vector_env.py:235-258).  Output tensors are double-buffered: the tensors
    returned by step t stay valid until step t+2 (``copy=True`` clones instead).
    ``step``, ``reset`` and ``sample_actions`` may be captured in a CUDA graph
    (``torch.cuda.graph``): replays are bit-identical to eager calls, and what
    cannot be captured raises ``error.Error`` (DESIGN.md §4.8).

``backend="numpy"`` (drop-in for CPU agents and for the parity tests)
    host buffers in, host buffers out, through ``b200gym_step_host``; returns
    exactly what ``SyncVectorEnv.step`` returns, including the object-array
    ``infos`` that only appear when some env finished.
"""
import ctypes
import math
import os
import time

import numpy as np

from gym_b200 import _lib, envs as _envs, error, subenv as _subenv
from gym_b200.registration import spec as _spec
from gym_b200.snapshot import FORMAT_VERSION, EnvSnapshot, check_compatible, env_config, host_indices
from gym_b200.spaces import batch_space, pcg64_skip, pcg64_state

_STATE_DEFAULT, _STATE_WAITING_RESET, _STATE_WAITING_STEP = "default", "reset", "step"


def _torch():
    import torch
    return torch


def capturing():
    """True while torch's current CUDA stream is being captured into a graph (no CUDA call if CUDA is not up)."""
    torch = _torch()
    return torch.cuda.is_initialized() and torch.cuda.is_current_stream_capturing()


def refuse_capture(what, why):
    """Raise ``error.Error`` for an operation that cannot be captured in a CUDA graph (before it makes any CUDA call,
    so the env stays usable and the capture can be abandoned cleanly)."""
    if capturing():
        raise error.Error(f"{what} cannot be captured in a CUDA graph: {why}")


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
    """``infos`` of the torch backend: the done masks (``_final_observation`` and, with per-env episode statistics,
    ``_final_info``) are materialised on first access -- or at once while a CUDA graph is being captured, so that they
    are outputs of the graph that every replay rewrites."""

    def __init__(self, final_obs, terminated, truncated, final_info=None, captured=None):
        super().__init__(final_observation=final_obs)
        self._t, self._u = terminated, truncated
        self._masks = ("_final_observation",)
        if final_info is not None:
            dict.__setitem__(self, "final_info", final_info)
            self._masks = ("_final_observation", "_final_info")
        if capturing() if captured is None else captured:
            for m in self._masks:
                self._mask(m)

    def _mask(self, k):
        if not dict.__contains__(self, k):
            other = [m for m in self._masks if dict.__contains__(self, m)]
            dict.__setitem__(self, k, dict.__getitem__(self, other[0]) if other else self._t | self._u)
        return dict.__getitem__(self, k)

    def __getitem__(self, k):
        if k in self._masks:
            return self._mask(k)
        return dict.__getitem__(self, k)

    def __contains__(self, k):
        return k in self._masks or dict.__contains__(self, k)

    def get(self, k, default=None):
        return self[k] if k in self else default

    def keys(self):
        for m in self._masks:
            self._mask(m)
        return dict.keys(self)

    def items(self):
        for m in self._masks:
            self._mask(m)
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
        wrappers: per-env wrappers, innermost first, as ``gym.vector.make(..., wrappers=[...])`` applies them to
            every sub-env (``gym_b200.subenv``); they run on the device after each step.
        **kwargs: env constructor kwargs (``g`` for Pendulum, ``goal_velocity`` for MountainCar*).
    """

    is_vector_env = True

    def __init__(self, env_id, num_envs, device=None, max_episode_steps=None, backend="torch",
                 copy=None, first_index=0, autoreset=True, dense_infos=False, wrappers=None, **kwargs):
        self.spec = _spec(env_id)
        stages = _subenv.parse(wrappers)
        if stages and not autoreset:
            raise ValueError("per-env wrappers need autoreset=True (SyncVectorEnv resets through them)")
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
        self._sample_record = None  # the action-space stream on the device (sample_actions)
        self._sample_mirror = None  # the host generator state the record holds, as far as the host knows
        self._chain = None
        if stages:
            # the chain's spaces are the wrapped env's (FrameStack / TimeAwareObservation / FlattenObservation reshape
            # the observation, RescaleAction rescales the action space)
            self._chain = _subenv.Chain(stages, self.kind, self.obs_dim, self.single_action_space,
                                        self.single_observation_space)
            self.single_observation_space = self._chain.observation_space
            self.single_action_space = self._chain.action_space
            self.observation_space = batch_space(self.single_observation_space, n=self.num_envs)
            self.action_space = batch_space(self.single_action_space, n=self.num_envs)
        self._obs_shape = tuple(self.single_observation_space.shape)   # of one env's output row

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
        self._captured = False   # whether the pending torch-backend step is being captured in a CUDA graph
        self._flip = 0
        self._out = None
        self._hio = None
        if self._chain is not None:
            self._chain.allocate(torch, self.num_envs, self.device)
            _lib.check(lib.b200gym_subenv_set(handle, ctypes.byref(self._chain.struct())), handle)
            self._t0 = time.perf_counter()
        if backend == "torch":
            self._out = [self._alloc_outputs(), self._alloc_outputs()]
            # {state_hi, state_lo, inc_hi, inc_lo, ticket} of b200gym_sample_space_stream
            self._sample_record = torch.zeros(8, dtype=torch.int64, device=self.device)
        else:
            self._map_host_buffers()

    # ------------------------------------------------------------------ buffers
    def _alloc_outputs(self):
        """One set of caller-owned output tensors (obs, reward, terminated, truncated, final_obs)."""
        torch = _torch()
        n, d, dev = self.num_envs, self.obs_dim, self.device
        shape = (n,) + self._obs_shape
        out = dict(
            obs=torch.zeros(shape, dtype=torch.float32, device=dev),
            reward=torch.zeros((n,), dtype=torch.float64, device=dev),
            terminated=torch.zeros((n,), dtype=torch.bool, device=dev),
            truncated=torch.zeros((n,), dtype=torch.bool, device=dev),
            final_obs=torch.zeros(shape, dtype=torch.float32, device=dev),
            **self._chain_outputs(torch, lambda shape, dtype: torch.zeros(shape, dtype=dtype, device=dev)),
        )
        if self._chain is not None and self._chain.reshape:
            # a reshaping chain reads the step's own (n, D) rows and writes the outputs above
            out["raw_obs"] = torch.zeros((n, d), dtype=torch.float32, device=dev)
            out["raw_final_obs"] = torch.zeros((n, d), dtype=torch.float32, device=dev)
        return out

    def _chain_outputs(self, torch, alloc):
        """The outputs a wrapper chain adds: float64 final observations where the chain's terminal rows are float64,
        the episode fields when it records episode statistics."""
        c, n, out = self._chain, self.num_envs, {}
        if c is not None and c.final_f64:
            out["final_obs64"] = alloc((n,) + self._obs_shape, torch.float64)
        if c is not None and c.episode:
            out["ep_r"] = alloc((n,), torch.float32)
            out["ep_l"] = alloc((n,), torch.int32)
        return out

    def _map_host_buffers(self):
        """numpy views of the library's page-locked staging buffers (b200gym_host_buffers)."""
        hio = _lib.HostIO()
        _lib.check(self._lib.b200gym_host_buffers(self._handle, ctypes.byref(hio)), self._handle)
        n, shape = self.num_envs, (self.num_envs,) + self._obs_shape

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
            obs=view(hio.obs, ctypes.c_float, shape, np.float32),
            reward=view(hio.reward, ctypes.c_double, (n,), np.float64),
            terminated=view(hio.terminated, ctypes.c_uint8, (n,), np.uint8),
            truncated=view(hio.truncated, ctypes.c_uint8, (n,), np.uint8),
            final_obs=view(hio.final_obs, ctypes.c_float, shape, np.float32),
        )
        if self._chain is not None:
            f64, ep_r, ep_l = ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_void_p()
            _lib.check(self._lib.b200gym_subenv_host_buffers(self._handle, ctypes.byref(f64), ctypes.byref(ep_r),
                                                             ctypes.byref(ep_l)), self._handle)
            if self._chain.final_f64:
                self._hio["final_obs64"] = view(f64.value, ctypes.c_double, shape, np.float64)
            if self._chain.episode:
                self._hio.update(ep_r=view(ep_r.value, ctypes.c_float, (n,), np.float32),
                                 ep_l=view(ep_l.value, ctypes.c_int32, (n,), np.int32))

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
        refuse_capture("seed(<list>)", "per-env seeds are staged through host memory and synchronise; seed with an int "
                       "or seed outside the capture")
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
        self._refuse_numpy_capture("reset")
        if seed is not None and not isinstance(seed, (int, np.integer)):
            refuse_capture("reset(seed=<list>)", "per-env seeds are staged through host memory and synchronise; "
                           "seed with an int or reset outside the capture")
        bounds = _envs.parse_reset_bounds(self.kind, options)
        self.seed(seed)
        bptr = None
        if bounds is not None:
            barr = (ctypes.c_double * 2)(*bounds)
            bptr = ctypes.cast(barr, ctypes.c_void_p)
        if self.backend == "torch":
            out = self._out[self._flip]
            raw = out.get("raw_obs", out["obs"])
            _lib.check(self._lib.b200gym_reset(self._handle, None, bptr, ctypes.c_void_p(raw.data_ptr()),
                                               self._stream()), self._handle)
            if self._chain is not None:
                _lib.check(self._lib.b200gym_subenv_reset_io(self._handle, None, ctypes.c_void_p(raw.data_ptr()),
                                                             ctypes.c_void_p(out["obs"].data_ptr()), self._stream()),
                           self._handle)
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

    def _refuse_numpy_capture(self, what):
        if self.backend == "numpy":
            refuse_capture(what, "backend='numpy' steps through page-locked host buffers and synchronises; capture "
                           "an env with backend='torch'")

    # ------------------------------------------------------------------ step
    def _device_actions(self, actions, captured=False, steps=False, n=None, what=None):
        """Bring `actions` to a contiguous device tensor of a dtype the kernel reads directly.  steps=True: a leading
        time axis of length >= 1, with the shape checked exactly (rollout).  n: the batch size (default num_envs)."""
        torch = _torch()
        n = self.num_envs if n is None else n
        what = what or ("rollout()" if steps else "step()")
        if captured and not (isinstance(actions, torch.Tensor) and actions.device == self.device):
            raise error.Error(f"{what} cannot be captured in a CUDA graph with actions that are not a CUDA tensor on "
                              f"{self.device}: the host-to-device copy cannot be replayed (got "
                              f"{type(actions).__name__}{' on ' + str(actions.device) if hasattr(actions, 'device') else ''})")
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
            shape = (n,)
        else:
            if actions.dtype != torch.float32:
                actions = actions.to(torch.float32)  # the Box dtype (e.g. pendulum.py:113-115)
            code = _lib.ACT_F32
            shape = (n, self.act_dim)
        if steps:
            if actions.dim() != len(shape) + 1 or tuple(actions.shape[1:]) != shape or actions.shape[0] < 1:
                raise error.InvalidAction(f"expected actions of shape (T, {', '.join(map(str, shape))}) with T >= 1, "
                                          f"got {tuple(actions.shape)}")
            shape = (actions.shape[0],) + shape
        elif actions.numel() != int(np.prod(shape)):
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
        self._refuse_numpy_capture("step")
        if self.backend == "torch":
            self._captured = captured = capturing()
            # the reference asserts on an out-of-range Discrete action (cartpole.py:132); the device cannot raise and
            # this backend never waits for it, so the kernels flag it in host-visible memory and the error surfaces
            # at the next call (no synchronisation unless the flag is up; none at all while a graph is captured: an
            # invalid action in a replay is reported by the next eager call)
            if self.discrete and not captured and self._lib.b200gym_invalid_seen(self._handle) == 1:
                self.check_actions()
            self._raise_snapshot_index_error()
            act, code = self._device_actions(actions, captured)
            c = self._chain
            if c is not None and c.act_stages:   # ClipAction / RescaleAction, outermost first
                staged = _torch().empty_like(act)
                _lib.check(self._lib.b200gym_subenv_actions(self._handle, ctypes.c_void_p(act.data_ptr()),
                                                            ctypes.c_void_p(staged.data_ptr()), self._stream()),
                           self._handle)
                act = staged
            self._flip ^= 1
            out = self._out[self._flip]

            def ptr(k):
                return ctypes.c_void_p(out[k].data_ptr()) if k in out else None
            raw_obs = ptr("raw_obs") or ptr("obs")
            raw_fin = ptr("raw_final_obs") or ptr("final_obs")
            _lib.check(self._lib.b200gym_step(
                self._handle, ctypes.c_void_p(act.data_ptr()), code, raw_obs, ptr("reward"), ptr("terminated"),
                ptr("truncated"), raw_fin, self._stream()), self._handle)
            if c is not None:
                _lib.check(self._lib.b200gym_subenv_step_io(
                    self._handle, raw_obs, ptr("obs"), ptr("reward"), ptr("terminated"), ptr("truncated"), raw_fin,
                    ptr("final_obs"), ptr("final_obs64"), ptr("ep_r"), ptr("ep_l"), self._stream()), self._handle)
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
                o = {k: v.clone() for k, v in o.items() if not k.startswith("raw_")}
            episode = {"episode": {"r": o["ep_r"], "l": o["ep_l"], "t": self._episode_time()}} if "ep_r" in o else None
            infos = FinalInfos(o.get("final_obs64", o["final_obs"]), o["terminated"], o["truncated"], episode,
                               self._captured)
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
            fo = h.get("final_obs64", h["final_obs"])
            episode = None
            if "ep_r" in h:
                ep_r, ep_l = (h["ep_r"].copy(), h["ep_l"].copy()) if self.copy else (h["ep_r"], h["ep_l"])
                episode = {"episode": {"r": ep_r, "l": ep_l, "t": self._episode_time()}}
            infos = FinalInfos(fo.copy() if self.copy else fo, term, trunc, episode, False)
        elif self.autoreset:
            done = term | trunc
            if done.any():
                # vector_env.py:208-258: object arrays + `_key` masks, only when some env finished
                fo = np.full(self.num_envs, None, dtype=object)
                fi = np.full(self.num_envs, None, dtype=object)
                final = h.get("final_obs64", h["final_obs"])
                t = self._episode_time() if "ep_r" in h else None
                for i in np.flatnonzero(done):
                    fo[i] = final[i].copy()
                    # a per-env RecordEpisodeStatistics puts its episode into the step info, which SyncVectorEnv
                    # moves to final_info[i] (record_episode_statistics.py:127-139, sync_vector_env.py:152-156)
                    fi[i] = {} if t is None else {"episode": {"r": h["ep_r"][i].copy(), "l": h["ep_l"][i].copy(),
                                                              "t": t}}
                infos = {"final_observation": fo, "_final_observation": done.copy(),
                         "final_info": fi, "_final_info": done.copy()}
        return obs, reward, term, trunc, infos

    def _episode_time(self):
        """RecordEpisodeStatistics' "t": wall seconds since the wrappers were built."""
        return round(time.perf_counter() - self._t0, 6)

    def step(self, actions):
        """One SyncVectorEnv.step: (obs, rewards, terminateds, truncateds, infos)."""
        self.step_async(actions)
        return self.step_wait()

    def rollout(self, actions):
        """T steps with actions known in advance -> ``(obs, rewards, terminateds, truncateds, infos)``, each with a
        leading T axis: what ``[self.step(a) for a in actions]`` returns, stacked, bit for bit, and the env left as those
        calls leave it.  ``actions``: (T, N) integers (Discrete) or (T, N, A) float32 (Box).  The outputs are new
        tensors that belong to the caller; ``infos["final_observation"]`` is (T, N, D), valid where
        ``infos["_final_observation"]`` (T, N) is set.  The classic-control kinds run the T steps in one launch with
        each env's state in registers (DESIGN.md §4.10).  May be captured in a CUDA graph."""
        captured = self._rollout_guards("rollout")
        act, code = self._device_actions(actions, captured, steps=True)
        T = int(act.shape[0])
        obs, reward, term, trunc, final_obs, last = self._rollout_outputs(T)
        _lib.check(self._lib.b200gym_rollout(
            self._handle, ctypes.c_void_p(act.data_ptr()), code, T, ctypes.c_void_p(obs.data_ptr()),
            ctypes.c_void_p(reward.data_ptr()), ctypes.c_void_p(term.data_ptr()), ctypes.c_void_p(trunc.data_ptr()),
            ctypes.c_void_p(final_obs.data_ptr()) if self.autoreset else None, ctypes.c_void_p(last.data_ptr()),
            self._stream()), self._handle)
        self._last_actions = act  # keep alive until the kernel has consumed it
        return obs, reward, term, trunc, FinalInfos(final_obs, term, trunc, None, captured)

    def rollout_sampled(self, T):
        """T steps of random actions -> ``(actions, obs, rewards, terminateds, truncateds, infos)``, each with a leading
        T axis: bit for bit what ``a = self.sample_actions(); self.step(a)`` repeated T times returns, stacked, with
        the env and the action space's generator left where that loop leaves them.  ``actions`` is int64 (T, N) for
        Discrete kinds and float32 (T, N, A) for Box kinds; the other five are as ``rollout()`` returns them.  The
        outputs are new tensors that belong to the caller.  The classic-control kinds draw the actions inside the
        rollout kernel, next to each env's state, so they are written once and never read back (DESIGN.md §4.11).

        May be captured in a CUDA graph once the device holds the generator, as ``sample_actions()``: each replay
        continues the stream on the device, and ``sync_action_space()`` brings the host generator there."""
        captured = self._rollout_guards("rollout_sampled")
        n_choices, cols, low, high, bit_generator, state, words = self._sample_begin("rollout_sampled()", captured)
        if isinstance(T, (bool, np.bool_)) or not isinstance(T, (int, np.integer)) or not 1 <= int(T) <= 2 ** 31 - 1:
            raise ValueError(f"rollout_sampled(T) needs an integer 1 <= T < 2**31, got {T!r}")
        T = int(T)
        torch = _torch()
        n = self.num_envs
        actions = torch.empty((T, n) if n_choices else (T, n, cols), dtype=torch.int64 if n_choices else torch.float32,
                              device=self.device)
        obs, reward, term, trunc, final_obs, last = self._rollout_outputs(T)
        _lib.check(self._lib.b200gym_rollout_sampled(
            self._handle, ctypes.c_void_p(self._sample_record.data_ptr()), words, n_choices,
            None if low is None else low.ctypes.data, None if high is None else high.ctypes.data, T,
            ctypes.c_void_p(actions.data_ptr()), ctypes.c_void_p(obs.data_ptr()), ctypes.c_void_p(reward.data_ptr()),
            ctypes.c_void_p(term.data_ptr()), ctypes.c_void_p(trunc.data_ptr()),
            ctypes.c_void_p(final_obs.data_ptr()) if self.autoreset else None, ctypes.c_void_p(last.data_ptr()),
            self._stream()), self._handle)
        self._sample_end(bit_generator, state, actions.numel(), captured)
        return actions, obs, reward, term, trunc, FinalInfos(final_obs, term, trunc, None, captured)

    def rollout_linear(self, weight, bias, T, *, summary=False, obs_norm=None, norm_epsilon=1e-8, clip_obs=None,
                       obs_moments=False):
        """T steps of a linear policy in closed loop: bit for bit what
        ``for t in range(T): a = policy(obs); obs, r, te, tr, info = self.step(a)`` returns, stacked, with ``obs``
        starting at the observation the env last returned, and the env left where that loop leaves it.

        With K = ``single_action_space.n`` (Discrete) or ``act_dim`` (Box) and D = ``obs_dim``, ``weight`` (K, D) and
        ``bias`` (K,) are one policy for every env, or ``weight`` (N, K, D) and ``bias`` (N, K) one per env: float32,
        contiguous, on the env's device.  The logits are ``z[j] = bias[j]``, then ``z[j] = z[j] + weight[j, k] * o[k]``
        for k = 0 .. D-1, every float32 product and sum rounded (no fused multiply-add).  The action is ``np.argmax(z)``
        (the first NaN, else the first maximum) for Discrete kinds and ``z`` itself, unclipped, for Box kinds.

        ``summary=False`` -> ``(actions, obs, rewards, terminateds, truncateds, infos)`` as ``rollout_sampled()``
        returns them.  ``summary=True`` -> ``(returns, lengths, ended)``, each (N,), over env i's first episode end
        within the call (t_end; T - 1 if none): float64 ``0.0 + rewards[0] + ... + rewards[t_end]`` in step order,
        int32 ``t_end + 1``, and bool; the env still takes all T steps, and no per-step tensor is allocated.

        The classic-control kinds run the T steps in one launch, the policy next to each env's state, and start from
        the observation of the current state (after ``set_state()``, that is the first input).  They may be captured in
        a CUDA graph: replays read the current contents of ``weight`` and ``bias``.  The Box2D kinds launch the policy
        and the step once per step and cannot be captured (DESIGN.md §4.12).

        ``obs_norm=(mean, var)``, ``norm_epsilon`` and ``clip_obs`` (keyword only) are ``rollout_mlp_noisy()``'s: the
        policy reads ``((o.double() - mean) / torch.sqrt(var + eps)).float().clamp(-c, c)`` in place of ``o``, while
        the returned ``obs`` and ``infos["final_observation"]`` stay raw.  The statistics are one shared (D,) pair,
        fixed for the call, and per-env ``weight`` / ``bias`` rows are allowed with them: ES and ARS perturb the policy
        and share the statistics.  ``obs_moments=True`` needs ``summary=True`` (full mode returns the observations
        themselves; there it raises ``ValueError``) and returns ``(returns, lengths, ended, obs_sum, obs_sumsq)``, the
        last two float64 (N, D): with ``o_t`` the raw float32 observation the policy read at step t (step 0's is the
        one the env last returned), over env i's first-episode inputs t = 0 .. ``lengths[i] - 1`` in step order,
        every operation rounded, no fused multiply-add::

            s = +0.0;  s = s + float64(o_t[k])
            q = +0.0;  q = q + float64(o_t[k]) * float64(o_t[k])

        so the count is ``lengths``.  It works with or without ``obs_norm``.  An ARS-V2 loop (Mania et al. 2018) with
        float64 running statistics, starting from the identity (V2-t keeps the b best directions' updates)::

            f64 = dict(dtype=torch.float64, device=dev)
            mean, var, count = torch.zeros(D, **f64), torch.ones(D, **f64), 0
            M = torch.zeros(K, D, device=dev)                                  # the policy, zero bias
            for it in range(iters):
                delta = torch.randn(N // 2, K, D, device=dev)
                W = torch.cat([M + nu * delta, M - nu * delta])                   # (N, K, D): +-directions
                ret, length, ended, s, q = envs.rollout_linear(
                    W, torch.zeros(N, K, device=dev), 1000, summary=True,
                    obs_norm=(mean, var), obs_moments=True)
                r = ret.float().reshape(2, -1)
                M += alpha / (N // 2 * r.std()) * ((r[0] - r[1])[:, None, None] * delta).sum(0)
                c = length.sum().item()                                           # Chan's merge of (c, S, Q)
                if c:
                    bm = s.sum(0) / c
                    bv = q.sum(0) / c - bm * bm
                    d, tot = bm - mean, count + c
                    var.copy_((var * count + bv * c + d * d * count * c / tot) / tot)
                    mean.add_(d * c / tot)
                    count = tot

        Replays of a captured graph read the current ``mean`` and ``var``; ``norm_epsilon`` and ``clip_obs`` are fixed
        at capture.  With the four keywords at their defaults the call is the one above, unchanged (DESIGN.md
        §4.19)."""
        what = "rollout_linear"
        captured = self._rollout_guards(what)
        per_env = self._linear_params(weight, bias)
        norm, moments = self._policy_norm_args(what, summary, obs_norm, norm_epsilon, clip_obs, obs_moments)
        vp = ctypes.c_void_p
        if norm is None:
            return self._policy_rollout(what, T, summary, captured, lambda T, outs, last, first: (
                self._lib.b200gym_rollout_linear(self._handle, vp(weight.data_ptr()), vp(bias.data_ptr()), int(per_env),
                                                 T, *outs, vp(last.data_ptr()), vp(first.data_ptr()), self._stream())))
        return self._policy_rollout(what, T, summary, captured, lambda T, outs, last, first, s=None, q=None: (
            self._lib.b200gym_rollout_linear_norm(self._handle, vp(weight.data_ptr()), vp(bias.data_ptr()),
                                                  int(per_env), T, *outs, vp(last.data_ptr()), vp(first.data_ptr()),
                                                  self._stream(), *norm, s, q)), moments)

    def rollout_mlp(self, params, hidden, T, *, summary=False, activation="relu", head=None, obs_norm=None,
                    norm_epsilon=1e-8, clip_obs=None, obs_moments=False):
        """T steps of an MLP policy in closed loop: ``rollout_linear()`` with the policy
        D -> hidden[0] (-> hidden[1]) -> K, the activation after every hidden layer and nothing after the last.

        ``hidden`` is a tuple of one or two widths, each 1 .. 64.  ``params`` packs one policy as P float32 values,
        layer by layer the weight (out, in) row-major and then the bias (out,): exactly
        ``torch.nn.utils.parameters_to_vector(nn.Sequential(nn.Linear(D, H1), nn.ReLU(), ..., nn.Linear(H_last, K)))``.
        Shape (P,) is one policy for every env, (N, P) one per env: float32, contiguous, on the env's device.

        Every unit is ``z[j] = bias[j]``, then ``z[j] = z[j] + W[j, k] * x[k]`` for k = 0 .. in-1, every float32
        product and sum rounded (no fused multiply-add).  ``activation`` (keyword only) is ``"relu"`` or ``"tanh"``:

        * ``"relu"``: a hidden unit's activation is ``z`` if ``z > 0`` or ``z`` is NaN, else +0.0 (NaN propagates,
          -0.0 becomes +0.0), so ``nn.ReLU`` gives the same bits;
        * ``"tanh"``: it is ``tanhf(z)`` of CUDA's math library, for the policies of CleanRL's PPO and
          Stable-Baselines3's ``MlpPolicy`` (``nn.Tanh``).  ``torch.tanh`` / ``nn.Tanh`` on the device gives the same
          bits: the two compile to the same instructions, and the tests check every float32 input against the torch
          build they run with.  Another torch or CUDA build is not covered by that check (DESIGN.md §4.15).

        The action is taken from the K outputs as ``rollout_linear()`` takes it from its logits.  Returns, guards,
        capture and the start from the current state are ``rollout_linear()``'s (DESIGN.md §4.13).

        ``obs_norm``, ``norm_epsilon``, ``clip_obs`` and ``obs_moments`` are ``rollout_linear()``'s, per-env ``params``
        rows included.  The deterministic evaluation of a CleanRL-style tanh actor trained on normalised observations
        (``rollout_actor_critic(..., obs_norm=(om, ov), clip_obs=10.0)``) reads the inputs it was trained on::

            ret, length, ended = envs.rollout_mlp(pa, (64, 64), 1000, summary=True, activation="tanh",
                                                  obs_norm=(om, ov), clip_obs=10.0)
            score = ret[ended].mean()                  # the mean first-episode return of the episodes that ended

        For Box kinds the action is the actor's mean output, unclipped, as ``rollout_linear()`` takes it (DESIGN.md
        §4.19).

        ``head`` (keyword only, Box kinds) is ``None`` (the default: the outputs are the action, as above),
        ``"tanh"`` or ``"tanh_normal"``: the tanh-squashed actors of TD3 / DDPG and SAC.  With A = ``act_dim`` and the
        action space's bounds, ``scale = float32(float32(high - low) / 2)`` and
        ``bias = float32(float32(high + low) / 2)`` (2 and 0 for Pendulum, 1 and 0 for the other Box kinds), every
        product and sum one rounded float32 operation, ``tanh`` as ``activation="tanh"`` and ``exp`` CUDA's ``expf``
        (on the device the bits of ``torch.exp``, checked for every float32 input against the torch build of the
        tests, DESIGN.md §4.21):

        * ``"tanh"``: K = A outputs z and ``a = tanh(z) * scale + bias``, the action of CleanRL's TD3 / DDPG ``Actor``;
        * ``"tanh_normal"``: K = 2A outputs, the mean ``m = z[:A]`` and the raw log-std ``z[A:]``, and
          ``a = tanh(m) * scale + bias``, the deterministic action (``mean``) of CleanRL's SAC ``Actor.get_action``.

        P counts K outputs; ``rollout_mlp_noisy()`` shows the packing of both actors.  The hidden widths stay 1 .. 64:
        CleanRL's defaults are 256 wide, so those actors must be trained at widths <= 64 to run here.  ``head`` is
        refused with ``obs_norm``, ``clip_obs`` or ``obs_moments`` and on Discrete kinds, before any CUDA call."""
        what = "rollout_mlp"
        captured = self._rollout_guards(what)
        code = self._mlp_head(what, head, obs_norm, clip_obs, obs_moments)
        h1, h2, per_env, act = self._mlp_params(params, hidden, activation, head=head)
        norm, moments = self._policy_norm_args(what, summary, obs_norm, norm_epsilon, clip_obs, obs_moments)
        vp = ctypes.c_void_p
        if code is not None:
            return self._policy_rollout(what, T, summary, captured, lambda T, outs, last, first: (
                self._lib.b200gym_rollout_mlp_head(self._handle, vp(params.data_ptr()), int(per_env), len(hidden), h1,
                                                   h2, T, *outs, vp(last.data_ptr()), vp(first.data_ptr()),
                                                   self._stream(), act, code)))
        if norm is None:
            return self._policy_rollout(what, T, summary, captured, lambda T, outs, last, first: (
                self._lib.b200gym_rollout_mlp_act(self._handle, vp(params.data_ptr()), int(per_env), len(hidden), h1,
                                                  h2, T, *outs, vp(last.data_ptr()), vp(first.data_ptr()),
                                                  self._stream(), act)))
        return self._policy_rollout(what, T, summary, captured, lambda T, outs, last, first, s=None, q=None: (
            self._lib.b200gym_rollout_mlp_norm(self._handle, vp(params.data_ptr()), int(per_env), len(hidden), h1, h2,
                                               T, *outs, vp(last.data_ptr()), vp(first.data_ptr()), self._stream(), act,
                                               *norm, s, q)), moments)

    def rollout_mlp_noisy(self, params, hidden, noise, *, activation="relu", head=None, obs_norm=None,
                          norm_epsilon=1e-8, clip_obs=None):
        """T steps of a stochastic MLP policy in closed loop, T = ``noise.shape[0]`` -> ``(actions, outputs, obs,
        rewards, terminateds, truncateds, infos)``: bit for bit what
        ``for t in range(T): z = mlp(obs); a = rule(z + noise[t]); obs, r, te, tr, info = self.step(a)`` returns,
        stacked, with ``obs`` starting at the observation the env last returned, and the env left where that loop
        leaves it.

        ``params``, ``hidden`` and ``activation`` are ``rollout_mlp()``'s, and z is its K outputs.  ``noise`` is
        float32 (T, N, K), contiguous, on the env's device, 1 <= T < 2**31, with K = ``single_action_space.n``
        (Discrete) or ``act_dim`` (Box).  Each ``z[k] + noise[t, i, k]`` is one rounded float32 add, IEEE NaN and infinity included; ``rule`` is
        ``np.argmax`` (the first NaN, else the first maximum) for Discrete kinds and the identity, unclipped, for Box
        kinds.  ``outputs`` is float32 (T, N, K), z before the noise; the other six are ``rollout_mlp()``'s.

        The sampling distribution is the noise's.  Gumbel noise makes the Discrete action an exact sample of
        ``softmax(outputs)``, so the log-probabilities of the actions come from ``outputs`` afterwards::

            u = torch.rand(T, N, K, device=dev).clamp_(min=torch.finfo(torch.float32).tiny)
            g = -torch.log(-torch.log(u))
            a, logits, obs, r, te, tr, info = envs.rollout_mlp_noisy(params, (64, 64), g)
            logp = torch.distributions.Categorical(logits=logits).log_prob(a)

        and scaled normal noise makes the Box action a sample of N(outputs, std**2)::

            std = log_std.exp()
            eps = torch.randn(T, N, K, device=dev)
            a, mean, obs, r, te, tr, info = envs.rollout_mlp_noisy(params, (64, 64), std * eps)
            logp = torch.distributions.Normal(mean, std).log_prob(a).sum(-1)

        A CleanRL-shaped tanh actor runs as it is, packed with ``parameters_to_vector``::

            actor = nn.Sequential(nn.Linear(D, 64), nn.Tanh(), nn.Linear(64, 64), nn.Tanh(), nn.Linear(64, K)).cuda()
            params = torch.nn.utils.parameters_to_vector(actor.parameters()).detach()
            a, logits, obs, r, te, tr, info = envs.rollout_mlp_noisy(params, (64, 64), g, activation="tanh")

        with ``g`` the Gumbel noise above (Discrete kinds), or ``std * eps`` in its place (Box kinds).

        Noise of -0.0 everywhere gives ``rollout_mlp()``'s actions (+0.0 would turn a -0.0 Box output into +0.0).
        Guards and the start from the current state are ``rollout_linear()``'s.  The classic-control kinds may be
        captured in a CUDA graph, and replays read the current contents of ``params`` and ``noise``, so filling the
        noise and rolling out can be one graph; the Box2D kinds cannot (DESIGN.md §4.14).

        ``obs_norm=(mean, var)`` (keyword only; two float64 (D,) tensors, contiguous, on the env's device, such as
        ``w.obs_rms.mean`` and ``w.obs_rms.var`` of a ``gym_b200.wrappers.NormalizeObservation`` ``w``) makes the policy
        read normalised observations, per element, in float64 with ``eps = norm_epsilon`` (real, finite, >= 0)::

            x = float32((float64(o) - mean) / sqrt(var + eps))
            x = clamp(x, -c, c)        # only with clip_obs = c, a real number > 0 taken as float32; NaN stays NaN

        which is ``((o.double() - mean) / torch.sqrt(var + eps)).float().clamp(-c, c)``: what NormalizeObservation
        returns for these statistics without an update.  The returned ``obs`` and ``infos["final_observation"]`` stay
        raw, so the caller can update its statistics from them.  The statistics are fixed for the call (the engine
        never updates them) and need one shared policy: per-env ``params`` rows with ``obs_norm`` raise ``ValueError``,
        as does ``clip_obs`` without ``obs_norm``.  A captured graph reads the current contents of ``mean`` and
        ``var``; ``norm_epsilon`` and ``clip_obs`` are fixed at capture.  With the three keywords at their defaults the
        call is the one above, unchanged (DESIGN.md §4.18).

        ``head`` (keyword only, Box kinds) is ``rollout_mlp()``'s, with the noise going into the head: ``noise`` is
        float32 (T, N, A) and ``outputs`` float32 (T, N, K), z before the head.  In the arithmetic of ``rollout_mlp()``:

        * ``"tanh"``: ``a = clamp((tanh(z) * scale + bias) + noise[t], low, high)``, where a NaN stays NaN as in
          ``torch.clamp``: CleanRL's TD3 / DDPG ``actor(obs) + noise`` and ``.clip(low, high)``;
        * ``"tanh_normal"``: with ``m = z[..., :A]``, ``s = z[..., A:]`` and ``eps = noise[t]``,
          ``ls = -5 + 3.5 * (tanh(s) + 1)``, ``x = m + eps * exp(ls)`` and ``a = tanh(x) * scale + bias``, unclipped:
          CleanRL's SAC ``Actor.get_action`` (``LOG_STD_MIN = -5``, ``LOG_STD_MAX = 2``;
          ``Normal(m, exp(ls)).rsample()`` is ``m + eps * exp(ls)``).  Its log-probabilities are recomputed from the
          observations at update time.

        A TD3 collection step of CleanRL's ``Actor`` (``fc1``, ``fc2``, ``fc_mu`` with ReLU; ``action_scale`` and
        ``action_bias`` are buffers, so ``parameters()`` is the packing), trained at (64, 64), filling a replay buffer
        with CleanRL's ``real_next_obs`` (the final observation where an episode ended)::

            params = torch.nn.utils.parameters_to_vector(actor.parameters()).detach()
            noise = torch.randn(T, N, A, device=dev) * (actor.action_scale * 0.1)        # exploration_noise = 0.1
            a, z, obs, r, te, tr, info = envs.rollout_mlp_noisy(params, (64, 64), noise, head="tanh")
            prev = torch.cat([obs0[None], obs[:-1]])       # obs0: what the env returned before the call
            done = info["_final_observation"]
            real_next = torch.where(done[..., None], info["final_observation"], obs)
            rb.add(prev.flatten(0, 1), real_next.flatten(0, 1), a.flatten(0, 1), r.flatten(), te.flatten())
            obs0 = obs[-1]

        and a SAC collection step of CleanRL's two-head ``Actor``, packed as one (2A, 64) output layer::

            params = torch.cat([p.reshape(-1) for p in (actor.fc1.weight, actor.fc1.bias, actor.fc2.weight,
                                actor.fc2.bias, actor.fc_mean.weight, actor.fc_logstd.weight, actor.fc_mean.bias,
                                actor.fc_logstd.bias)]).detach()
            a, z, obs, r, te, tr, info = envs.rollout_mlp_noisy(params, (64, 64), torch.randn(T, N, A, device=dev),
                                                                head="tanh_normal")

        with the same replay-buffer tuples.  The hidden widths stay 1 .. 64, so CleanRL's 256-wide defaults must be
        trained at <= 64.  Capture and the refusals are as without a head; ``head`` is also refused with ``obs_norm``
        or ``clip_obs`` and on Discrete kinds, before any CUDA call (DESIGN.md §4.21)."""
        what = "rollout_mlp_noisy"
        captured = self._rollout_guards(what)
        code = self._mlp_head(what, head, obs_norm, clip_obs)
        h1, h2, per_env, act = self._mlp_params(params, hidden, activation, what, head=head)
        T = self._noise_steps(noise)
        norm = self._norm_args(what, obs_norm, norm_epsilon, clip_obs, per_env=per_env)
        self._refuse_box2d_capture(what)
        vp = ctypes.c_void_p
        if code is not None:
            outputs = _torch().empty((T, self.num_envs, self._head_outputs(head)), dtype=noise.dtype,
                                     device=self.device)
            actions, obs, reward, term, trunc, infos = self._policy_rollout(
                what, T, False, captured, lambda T, outs, last, first: self._lib.b200gym_rollout_mlp_noisy_head(
                    self._handle, vp(params.data_ptr()), int(per_env), len(hidden), h1, h2, T, vp(noise.data_ptr()),
                    vp(outputs.data_ptr()), *outs[:6], vp(last.data_ptr()), vp(first.data_ptr()), self._stream(), act,
                    code))
            return actions, outputs, obs, reward, term, trunc, infos
        outputs = _torch().empty_like(noise)
        if norm is None:
            launch = lambda T, outs, last, first: self._lib.b200gym_rollout_mlp_noisy_act(  # noqa: E731
                self._handle, vp(params.data_ptr()), int(per_env), len(hidden), h1, h2, T, vp(noise.data_ptr()),
                vp(outputs.data_ptr()), *outs[:6], vp(last.data_ptr()), vp(first.data_ptr()), self._stream(), act)
        else:
            launch = lambda T, outs, last, first: self._lib.b200gym_rollout_mlp_noisy_norm(  # noqa: E731
                self._handle, vp(params.data_ptr()), 0, len(hidden), h1, h2, T, vp(noise.data_ptr()),
                vp(outputs.data_ptr()), *outs[:6], vp(last.data_ptr()), vp(first.data_ptr()), self._stream(), act,
                *norm[:4])
        actions, obs, reward, term, trunc, infos = self._policy_rollout(what, T, False, captured, launch)
        return actions, outputs, obs, reward, term, trunc, infos

    def rollout_actor_critic(self, actor, critic, hidden, noise, *, gamma, gae_lambda, activation="relu", obs_norm=None,
                             norm_epsilon=1e-8, clip_obs=None, reward_norm=None, clip_reward=None):
        """One on-policy collection step of PPO / A2C: ``rollout_mlp_noisy()`` with a critic evaluated next to each env's
        state, and the GAE advantages -> ``(actions, outputs, values, advantages, obs, rewards, terminateds,
        truncateds, infos)``.

        ``actions``, ``outputs``, ``obs``, ``rewards``, ``terminateds``, ``truncateds`` and ``infos`` are bit for bit
        what ``rollout_mlp_noisy(actor, hidden, noise, activation=activation)`` returns, and the env is left where that
        call leaves it.  ``actor`` is one packed actor, shape (P_actor,): per-env rows (N, P) raise ``ValueError``,
        because PPO and A2C train one network and per-env rows would double the kernels for no caller.  ``critic`` is
        one packed critic of shape (P_critic,), ``parameters_to_vector(nn.Sequential(nn.Linear(D, h1), act,
        [nn.Linear(h1, h2), act,] nn.Linear(h_last, 1)))``: the actor's ``hidden`` and ``activation`` (the defaults of
        CleanRL and Stable-Baselines3), ``rollout_mlp()``'s arithmetic with one output.  Both float32, contiguous, on
        the env's device.

        ``values`` is float32 (T + 1, N): ``values[t]`` is V(the observation step t acts on), starting at the one the
        env last returned, and ``values[T]`` is V(the observation the call leaves the env at), CleanRL's
        ``next_value``, bit-equal to the next call's ``values[0]``.  ``advantages`` is float32 (T, N), every float32
        operation rounded, no fused multiply-add, with ``g = float32(gamma)``, ``gl = float32(gamma * gae_lambda)``
        (the product in float64), ``r[t] = float32(rewards[t])`` and ``Vf[t]`` = V(``infos["final_observation"][t]``)::

            adv[T] = +0.0
            for t = T-1 .. 0:
                if terminated[t]:   delta = r[t] - values[t]
                elif truncated[t]:  delta = (r[t] + g * Vf[t]) - values[t]
                else:               delta = (r[t] + g * values[t+1]) - values[t]
                adv[t] = delta if (terminated[t] or truncated[t]) else delta + gl * adv[t+1]

        That is CleanRL's recursion with Stable-Baselines3's bootstrap of a time-limit end from the final observation.
        ``gamma`` and ``gae_lambda`` are required keywords, real and finite in [0, 1].  The env must autoreset (the
        bootstrap reads the final observations); ``autoreset=False`` raises ``error.Error``.

        A CleanRL-shaped PPO collection, Discrete actions::

            actor = nn.Sequential(nn.Linear(D, 64), nn.Tanh(), nn.Linear(64, 64), nn.Tanh(), nn.Linear(64, K)).cuda()
            critic = nn.Sequential(nn.Linear(D, 64), nn.Tanh(), nn.Linear(64, 64), nn.Tanh(), nn.Linear(64, 1)).cuda()
            pa = torch.nn.utils.parameters_to_vector(actor.parameters()).detach()
            pc = torch.nn.utils.parameters_to_vector(critic.parameters()).detach()
            first_obs = obs_now                                            # what the env last returned
            u = torch.rand(T, N, K, device=dev).clamp_(min=torch.finfo(torch.float32).tiny)
            g = -torch.log(-torch.log(u))                                 # Gumbel: samples softmax(logits)
            a, logits, values, adv, obs, r, te, tr, info = envs.rollout_actor_critic(
                pa, pc, (64, 64), g, gamma=0.99, gae_lambda=0.95, activation="tanh")
            obs_in = torch.cat([first_obs[None], obs[:-1]])               # the inputs the actions were taken at
            logp = torch.distributions.Categorical(logits=logits).log_prob(a)
            returns = adv + values[:-1]
            obs_now = obs[-1]

        For Box actions draw ``std * torch.randn(T, N, K)`` instead of ``g``; then ``outputs`` is the mean and
        ``logp = torch.distributions.Normal(mean, std).log_prob(a).sum(-1)``.

        Guards and the start from the current state are ``rollout_mlp_noisy()``'s.  The classic-control kinds run the
        rollout in one launch, both nets staged in shared memory, then one launch for the advantages; they may be
        captured in a CUDA graph, and replays read the current contents of ``actor``, ``critic`` and ``noise``, while
        ``gamma`` and ``gae_lambda`` are fixed at capture.  The Box2D kinds compose the same results launch by launch
        and cannot be captured (DESIGN.md §4.17).

        ``obs_norm``, ``norm_epsilon`` and ``clip_obs`` are ``rollout_mlp_noisy()``'s: with ``obs_norm``, the actor, the
        critic at every step, ``values[T]`` and the bootstrap ``Vf[t]`` all read the normalised observation.
        ``reward_norm=var`` (a float64 (1,) tensor on the env's device, such as ``w.return_rms.var`` of a
        ``gym_b200.wrappers.NormalizeReward``) scales the rewards the advantages read, NormalizeReward's division
        without a mean::

            r[t] = float32(rewards[t] / sqrt(var + eps))
            r[t] = clamp(r[t], -c_r, c_r)      # only with clip_reward = c_r, as clip_obs

        The returned ``rewards`` stay raw float64; ``values`` and ``advantages`` are in the scaled units.
        ``clip_reward`` without ``reward_norm`` raises ``ValueError``.  Replays of a captured graph read the current
        ``mean``, ``var`` and reward ``var``.  The engine never updates the statistics: a CleanRL-shaped continuous PPO
        holds them fixed for one collection and updates them from it, in float64 (Chan's merge for the observations,
        the discounted-return recurrence for the rewards)::

            f64 = dict(dtype=torch.float64, device=dev)                          # RunningMeanStd's start
            om, ov, oc = torch.zeros(D, **f64), torch.ones(D, **f64), 1e-4
            rm, rv, rc = torch.zeros(1, **f64), torch.ones(1, **f64), 1e-4
            ret = torch.zeros(N, **f64)
            for update in range(num_updates):
                eps_n = std * torch.randn(T, N, K, device=dev)
                a, mean, values, adv, obs, r, te, tr, info = envs.rollout_actor_critic(
                    pa, pc, (64, 64), eps_n, gamma=0.99, gae_lambda=0.95, activation="tanh",
                    obs_norm=(om, ov), clip_obs=10.0, reward_norm=rv, clip_reward=10.0)
                x = obs.double().reshape(-1, D)                                   # Chan et al. from T * N rows
                bm, bv, bc = x.mean(0), x.var(0, unbiased=False), x.shape[0]
                d, tot = bm - om, oc + bc
                ov.copy_((ov * oc + bv * bc + d * d * oc * bc / tot) / tot); om.add_(d * bc / tot); oc = tot
                rets = []
                for t in range(T):                                                # NormalizeReward's recurrence
                    ret = ret * 0.99 + r[t]
                    rets.append(ret)
                    ret = torch.where(te[t] | tr[t], torch.zeros_like(ret), ret)
                y = torch.stack(rets).reshape(-1)
                bm, bv, bc = y.mean(), y.var(unbiased=False), y.numel()
                d, tot = bm - rm, rc + bc
                rv.copy_((rv * rc + bv * bc + d * d * rc * bc / tot) / tot); rm.add_(d * bc / tot); rc = tot
                # the PPO update reads obs normalised with the statistics of this collection: normalise before
                # updating them, or keep a copy

        With every new keyword at its default the call is the one above, unchanged (DESIGN.md §4.18)."""
        what = "rollout_actor_critic"
        captured = self._rollout_guards(what)
        if not self.autoreset:
            raise error.Error(f"{what}() needs autoreset=True: the bootstrap of a truncated episode reads its final "
                              "observation, which only an autoresetting env reports")
        h1, h2, per_env, act = self._mlp_params(actor, hidden, activation, what)
        if per_env:
            raise ValueError(f"{what}() takes one actor shared by every env, shape ({actor.shape[1]},); got per-env rows "
                             f"{tuple(actor.shape)}")
        self._critic_params(critic, hidden, what)
        g, gl = self._gae_coefficients(gamma, gae_lambda, what)
        T = self._noise_steps(noise, what)
        norm = self._norm_args(what, obs_norm, norm_epsilon, clip_obs, reward_norm, clip_reward)
        self._refuse_box2d_capture(what)
        torch = _torch()
        outputs = torch.empty_like(noise)
        values = torch.empty((T + 1, self.num_envs), dtype=torch.float32, device=self.device)
        advantages = torch.empty((T, self.num_envs), dtype=torch.float32, device=self.device)
        vp = ctypes.c_void_p
        entry = self._lib.b200gym_rollout_actor_critic if norm is None else self._lib.b200gym_rollout_actor_critic_norm
        actions, obs, reward, term, trunc, infos = self._policy_rollout(
            what, T, False, captured, lambda T, outs, last, first: entry(
                self._handle, vp(actor.data_ptr()), vp(critic.data_ptr()), len(hidden), h1, h2, T,
                vp(noise.data_ptr()), vp(outputs.data_ptr()), *outs[:6], vp(values.data_ptr()),
                vp(advantages.data_ptr()), g, gl, vp(last.data_ptr()), vp(first.data_ptr()), self._stream(), act,
                *(() if norm is None else norm)))
        return actions, outputs, values, advantages, obs, reward, term, trunc, infos

    def _norm_args(self, what, obs_norm, eps, clip_obs, reward_norm=None, clip_reward=None, per_env=False):
        """Check the normalisation keywords of rollout_mlp_noisy() / rollout_actor_critic() without a CUDA call ->
        None when the observations and rewards are both left as they are, else the trailing arguments of the
        ``_norm`` entry points: (mean, var, eps, clip_obs, reward var, clip_reward), pointers or None, clips as
        float32 values with +inf for none."""
        torch = _torch()
        if isinstance(eps, (bool, np.bool_)) or not isinstance(eps, (int, float, np.integer, np.floating)) or not (
                math.isfinite(float(eps)) and float(eps) >= 0.0):
            raise ValueError(f"{what}() needs norm_epsilon a finite real number >= 0, got {eps!r}")

        def clip(c, name, given):
            if c is None:
                return math.inf
            if isinstance(c, (bool, np.bool_)) or not isinstance(c, (int, float, np.integer, np.floating)):
                raise ValueError(f"{what}() needs {name} a finite real number > 0, got {c!r}")
            with np.errstate(over="ignore"):
                f = np.float32(float(c)) if math.isfinite(float(c)) else np.float32(np.nan)
            if not (np.isfinite(f) and f > 0):
                raise ValueError(f"{what}() needs {name} a finite real number > 0 (as float32), got {c!r}")
            if not given:
                raise ValueError(f"{what}() got {name} without the statistics it clips")
            return float(f)

        def stats(x, name, shape):
            if not isinstance(x, torch.Tensor):
                raise ValueError(f"{what}() needs {name} as a torch tensor, got {type(x).__name__}")
            if x.dtype != torch.float64:
                raise ValueError(f"{what}() needs float64 {name}, got {x.dtype}")
            if x.device != self.device:
                raise ValueError(f"{what}() needs {name} on {self.device}, got {x.device}")
            if tuple(x.shape) != shape:
                raise ValueError(f"{what}() needs {name} of shape {shape}, got {tuple(x.shape)}")
            if not x.is_contiguous():
                raise ValueError(f"{what}() needs a contiguous {name}")
            return ctypes.c_void_p(x.data_ptr())

        mean = var = rvar = None
        if obs_norm is not None:
            if not isinstance(obs_norm, (tuple, list)) or len(obs_norm) != 2:
                raise ValueError(f"{what}() needs obs_norm as a (mean, var) pair, got {type(obs_norm).__name__}")
            if per_env:
                raise ValueError(f"{what}() with obs_norm needs one policy shared by every env, not per-env rows")
            mean = stats(obs_norm[0], "obs_norm mean", (self.obs_dim,))
            var = stats(obs_norm[1], "obs_norm var", (self.obs_dim,))
        c_obs = clip(clip_obs, "clip_obs", obs_norm is not None)
        if reward_norm is not None:
            rvar = stats(reward_norm, "reward_norm", (1,))
        c_rew = clip(clip_reward, "clip_reward", reward_norm is not None)
        if obs_norm is None and reward_norm is None:
            return None
        return mean, var, float(eps), c_obs, rvar, c_rew

    def _policy_norm_args(self, what, summary, obs_norm, eps, clip_obs, obs_moments):
        """Check rollout_linear()'s / rollout_mlp()'s normalisation and moment keywords without a CUDA call ->
        (None, False) when all four are at their defaults; else the statistics' arguments of the ``_norm`` entry points
        (mean, var, eps, clip_obs) and whether the moments are asked for."""
        if not isinstance(obs_moments, (bool, np.bool_)):
            raise ValueError(f"{what}() needs obs_moments True or False, got {obs_moments!r}")
        if obs_moments and not summary:
            raise ValueError(f"{what}() takes obs_moments=True only with summary=True: the full mode returns the "
                             "observations themselves")
        norm = self._norm_args(what, obs_norm, eps, clip_obs)
        if norm is None and not obs_moments:
            return None, False
        return (norm[:4] if norm is not None else (None, None, float(eps), math.inf)), bool(obs_moments)

    def _critic_params(self, critic, hidden, what):
        """Check rollout_actor_critic()'s critic, D -> hidden -> 1, without a CUDA call."""
        torch = _torch()
        sizes = [self.obs_dim] + [int(h) for h in hidden] + [1]
        P = sum(o * i + o for i, o in zip(sizes[:-1], sizes[1:]))
        if not isinstance(critic, torch.Tensor):
            raise ValueError(f"{what}() needs critic as a torch tensor, got {type(critic).__name__}")
        if critic.dtype != torch.float32:
            raise ValueError(f"{what}() needs a float32 critic, got {critic.dtype}")
        if critic.device != self.device:
            raise ValueError(f"{what}() needs the critic on {self.device}, got {critic.device}")
        if not critic.is_contiguous():
            raise ValueError(f"{what}() needs a contiguous critic")
        if tuple(critic.shape) != (P,):
            raise ValueError(f"{what}() with hidden {tuple(sizes[1:-1])} needs one critic of shape ({P},), shared by "
                             f"every env; got {tuple(critic.shape)}")

    @staticmethod
    def _gae_coefficients(gamma, gae_lambda, what):
        """Check gamma and gae_lambda (real, finite, in [0, 1]) -> (float32(gamma), float32(gamma * gae_lambda)),
        the product taken in float64, as Python floats that hold float32 values."""
        for name, x in (("gamma", gamma), ("gae_lambda", gae_lambda)):
            if isinstance(x, (bool, np.bool_)) or not isinstance(x, (int, float, np.integer, np.floating)) or not (
                    math.isfinite(float(x)) and 0.0 <= float(x) <= 1.0):
                raise ValueError(f"{what}() needs {name} a real number in [0, 1], got {x!r}")
        return float(np.float32(float(gamma))), float(np.float32(float(gamma) * float(gae_lambda)))

    def rollout_from(self, snap, actions, *, rows=None, states=False):
        """T steps of B branches, each from a snapshot row, without touching this env -> ``(returns, lengths, ended)``,
        and with ``states=True`` also an ``EnvSnapshot`` of the B end states.

        ``snap`` is an ``EnvSnapshot`` of this env or of any env of the same kind and construction config (anything
        else raises ``error.Error``).  ``rows`` is None (branch b starts from row b, B = ``len(snap)``) or B row indices,
        duplicates allowed: a CUDA tensor, whose out-of-range entries skip their branch (zero outputs, zero end row and
        observation) and make the next call raise, as ``snapshot()`` / ``restore()`` do; or a host sequence, checked
        here.  ``actions`` is (T, B) integers (Discrete) or (T, B, A) float32 (Box), as ``rollout()`` takes them.

        Bit for bit, with ``twin`` a fresh env of the same id and config with B envs::

            twin.restore(EnvSnapshot(snap.header, snap.rows[rows], snap.obs[rows]))
            obs, r, te, tr, info = twin.rollout(actions)

        the results are ``rollout_linear(summary=True)``'s fold of ``r``, ``te`` and ``tr`` over each branch's first
        episode end t_end (T - 1 if none): float64 ``0.0 + r[0] + ... + r[t_end]`` in step order, int32 ``t_end + 1``
        and bool; every branch takes all T steps.  The end states are ``twin.snapshot()``, with ``snap``'s header, and
        go straight back into ``rollout_from``.  So the autoresets of K branches from one root draw the same reset
        states, as K deep copies would; CartPole's ``autoreset=False`` flag comes from the row; an invalid Discrete
        action gives a NaN reward and counts in this env's invalid-action counter.  This env's state, RNG records,
        TimeLimit counters, observation buffers and action-space generator do not move, and it needs no ``reset()``.

        MPPI, R roots of ``real`` with K sampled action sequences each (here CartPole, with a placeholder cost)::

            snap = real.snapshot(roots)                                  # R rows
            rows = torch.arange(R, device=dev).repeat_interleave(K)      # R * K branches
            acts = torch.randint(0, 2, (T, R * K), device=dev)
            returns, lengths, ended = real.rollout_from(snap, acts, rows=rows)   # real does not move
            w = torch.softmax(returns.view(R, K) / temperature, dim=1)   # weights of the K sequences of each root

        Tree expansion, the end states fed back in::

            ret, _, _, leaves = real.rollout_from(snap, acts, rows=rows, states=True)
            best = ret.topk(16).indices.repeat_interleave(K)              # K children of each of the 16 best leaves
            ret2, _, _, deeper = real.rollout_from(leaves, acts2, rows=best, states=True)

        Refused where ``rollout()`` is (``backend="numpy"``, ``wrappers=``, a pending async call), before any CUDA call.
        The classic-control kinds run in one launch, one thread per branch, and may be captured in a CUDA graph: replays
        read the current contents of ``snap.rows``, ``rows`` and ``actions`` (the first call with CUDA-tensor ``rows``
        allocates the env's index-error flag, so make one outside the capture).  The Box2D kinds load the rows into a
        scratch batch the env keeps and step it launch by launch; they cannot be captured (DESIGN.md §4.16)."""
        captured, r, idx, B = self._from_rows("rollout_from", snap, rows)
        torch = _torch()
        m = int(r.shape[0])
        act, code = self._device_actions(actions, captured, steps=True, n=B, what="rollout_from()")
        T = int(act.shape[0])
        if T > 2 ** 31 - 1:
            raise error.Error(f"rollout_from() needs T < 2**31, got {T}")
        if self.discrete and code != _lib.ACT_I64:
            act, code = act.to(torch.int64), _lib.ACT_I64
        idx = self._device_rows(idx)
        vp = ctypes.c_void_p
        returns, lengths, ended, end_rows, end_obs = self._from_outputs(B, states)
        _lib.check(self._lib.b200gym_rollout_from(
            self._handle, vp(r.data_ptr()), m, None if idx is None else vp(idx.data_ptr()), B, vp(act.data_ptr()), code,
            T, vp(returns.data_ptr()), vp(lengths.data_ptr()), vp(ended.data_ptr()),
            vp(end_rows.data_ptr()) if states else None, vp(end_obs.data_ptr()) if states else None, self._stream()),
            self._handle)
        if states:
            return returns, lengths, ended, EnvSnapshot(snap.header, end_rows, end_obs)
        return returns, lengths, ended

    def rollout_from_mlp(self, snap, params, hidden, T, *, noise=None, rows=None, states=False, activation="relu",
                         obs_norm=None, norm_epsilon=1e-8, clip_obs=None):
        """T steps of an MLP policy in closed loop on B branches, each from a snapshot row, without touching this env
        -> ``(returns, lengths, ended, first_actions)``, and with ``states=True`` also an ``EnvSnapshot`` of the B end
        states.

        ``snap``, ``rows`` and ``states`` are ``rollout_from()``'s: B = ``len(rows)``, or ``len(snap)`` without rows;
        rows may repeat; an out-of-range CUDA-tensor row skips its branch and makes the next call raise.  ``params``,
        ``hidden`` and ``activation`` are ``rollout_mlp()``'s, with per-policy rows indexed by branch: shape (P,) is
        one policy for every branch, (B, P) one per branch (branch b's row b, not row ``rows[b]``).  ``T`` is an
        integer, 1 <= T < 2**31.  ``noise`` is None (the deterministic policy) or float32 (T, B, K), contiguous, on the
        env's device, with ``rollout_mlp_noisy()``'s rule ``rule(z + noise[t])``; a shape that disagrees with T or B
        raises ``ValueError``.  ``obs_norm``, ``norm_epsilon`` and ``clip_obs`` are ``rollout_mlp()``'s; ``noise``
        together with per-branch rows and ``obs_norm`` is refused, as ``rollout_mlp_noisy()`` refuses per-env rows
        with ``obs_norm``.

        ``returns`` (float64), ``lengths`` (int32) and ``ended`` (bool), each (B,), are ``rollout_from()``'s fold over
        each branch's first episode.  ``first_actions`` is the action each branch took at step 0, int64 (B,) for
        Discrete kinds and float32 (B, A) for Box kinds: the action a planner executes.  A skipped branch gets 0.

        Bit for bit, with ``twin`` a fresh env of the same id and config with B envs::

            twin.restore(EnvSnapshot(snap.header, snap.rows[rows], snap.obs[rows]))
            a, obs, r, te, tr, info = twin.rollout_mlp(params, hidden, T, activation=..., obs_norm=..., ...)  # no noise
            a, z, obs, r, te, tr, info = twin.rollout_mlp_noisy(params, hidden, noise, activation=..., ...)  # noise

        the results are ``rollout_from()``'s fold of ``r``, ``te`` and ``tr``, ``first_actions == a[0]``, and the end
        states are ``twin.snapshot()``.  The classic kinds' step 0 reads ``observe()`` of the row's state, the Box2D
        kinds' ``snap.obs[rows]``, which is what the restored twin reads.  This env's state, RNG records, TimeLimit
        counters, flags, observation buffers and action-space generator do not move, and it needs no ``reset()``.

        MCTS leaf evaluation with a Gumbel-sampled tanh actor, K samples from each of R leaves (CartPole)::

            rows = torch.arange(R, device=dev).repeat_interleave(K)            # R * K branches
            u = torch.rand(T, R * K, 2, device=dev).clamp_(min=torch.finfo(torch.float32).tiny)
            g = -torch.log(-torch.log(u))                                       # samples softmax(actor(o))
            ret, length, ended, a0 = real.rollout_from_mlp(leaves, pa, (64, 64), T, noise=g, rows=rows,
                                                           activation="tanh")
            value = ret.view(R, K).mean(1)                                      # each leaf's Monte-Carlo value

        MPPI on Pendulum with a policy prior, R roots of ``real`` and K samples of ``policy(o) + noise[t]`` each::

            snap = real.snapshot(roots)
            rows = torch.arange(R, device=dev).repeat_interleave(K)
            eps = sigma * torch.randn(T, R * K, 1, device=dev)
            ret, _, _, a0 = real.rollout_from_mlp(snap, prior, (64, 64), T, noise=eps, rows=rows, activation="tanh")
            w = torch.softmax(ret.view(R, K) / temperature, dim=1)              # weights of the K samples of each root
            u = (w[..., None] * a0.view(R, K, 1)).sum(1)                        # the action each root executes

        ES with antithetic per-branch policies on common start states, P pairs from S rows::

            delta = torch.randn(P, theta.numel(), device=dev)
            pop = torch.cat([theta + sigma * delta, theta - sigma * delta]).repeat_interleave(S, 0)   # (2 * P * S, n)
            rows = torch.arange(S, device=dev).repeat(2 * P)                    # every policy from the same S rows
            ret, _, _, _ = real.rollout_from_mlp(starts, pop, (64, 64), T, rows=rows, activation="tanh")
            f = ret.view(2, P, S).mean(2)
            theta += alpha / (2 * P * sigma) * ((f[0] - f[1])[:, None] * delta).sum(0)

        Refused where ``rollout_from()`` is (``backend="numpy"``, ``wrappers=``, a pending async call), and for bad
        parameters, noise or statistics, before any CUDA call and with the messages of ``rollout_from()``,
        ``rollout_mlp()`` and ``rollout_mlp_noisy()``.  The classic-control kinds run in one launch, one thread per
        branch, and may be captured in a CUDA graph: replays read the current ``snap.rows``, ``rows``, ``params``,
        ``noise`` and statistics.  The Box2D kinds compose the twin launch by launch in ``rollout_from()``'s scratch
        batch and cannot be captured (DESIGN.md §4.20)."""
        what = "rollout_from_mlp"
        captured, r, idx, B = self._from_rows(what, snap, rows)
        if isinstance(T, (bool, np.bool_)) or not isinstance(T, (int, np.integer)) or not 1 <= int(T) <= 2 ** 31 - 1:
            raise ValueError(f"{what}(T) needs an integer 1 <= T < 2**31, got {T!r}")
        T = int(T)
        h1, h2, per_branch, act = self._mlp_params(params, hidden, activation, what, n=B)
        if noise is not None and self._noise_steps(noise, what, n=B) != T:
            raise ValueError(f"{what}() needs noise of T = {T} steps, got {tuple(noise.shape)}")
        norm = self._norm_args(what, obs_norm, norm_epsilon, clip_obs, per_env=per_branch and noise is not None)
        mean, var, eps, c_obs = norm[:4] if norm is not None else (None, None, float(norm_epsilon), math.inf)
        torch = _torch()
        m = int(r.shape[0])
        box2d = self.kind in (_lib.KIND_LUNARLANDER, _lib.KIND_LUNARLANDER_CONT, _lib.KIND_BIPEDALWALKER,
                              _lib.KIND_BIPEDALWALKER_HARDCORE)
        o = snap.obs
        if box2d and not (isinstance(o, torch.Tensor) and o.dtype == torch.float32 and o.device == self.device
                          and tuple(o.shape) == (m, self.obs_dim) and o.is_contiguous()):
            raise error.Error(f"{what}() of a Box2D env needs the snapshot's observations as a contiguous float32 "
                              f"({m}, {self.obs_dim}) tensor on {self.device}")
        idx = self._device_rows(idx)
        vp = ctypes.c_void_p
        returns, lengths, ended, end_rows, end_obs = self._from_outputs(B, states)
        first = torch.empty(B, dtype=torch.int64, device=self.device) if self.discrete else torch.empty(
            (B, self.act_dim), dtype=torch.float32, device=self.device)
        _lib.check(self._lib.b200gym_rollout_from_mlp(
            self._handle, vp(r.data_ptr()), vp(o.data_ptr()) if box2d else None, m,
            None if idx is None else vp(idx.data_ptr()), B, vp(params.data_ptr()), int(per_branch), len(hidden), h1,
            h2, T, None if noise is None else vp(noise.data_ptr()), act, mean, var, eps, c_obs,
            vp(returns.data_ptr()), vp(lengths.data_ptr()), vp(ended.data_ptr()), vp(first.data_ptr()),
            vp(end_rows.data_ptr()) if states else None, vp(end_obs.data_ptr()) if states else None, self._stream()),
            self._handle)
        if states:
            return returns, lengths, ended, first, EnvSnapshot(snap.header, end_rows, end_obs)
        return returns, lengths, ended, first

    def _from_rows(self, what, snap, rows):
        """The guards of rollout_from() / rollout_from_mlp() and their snapshot and rows checks, all before any CUDA
        call -> (whether a CUDA graph is being captured, the snapshot's rows, the row indices (None, a CUDA tensor or
        a checked host int64 array), B)."""
        captured = self._rollout_guards(what, reset_needed=False)
        if self.kind in (_lib.KIND_LUNARLANDER, _lib.KIND_LUNARLANDER_CONT, _lib.KIND_BIPEDALWALKER,
                         _lib.KIND_BIPEDALWALKER_HARDCORE):
            refuse_capture(f"{what}() of a Box2D env", "it steps a scratch batch that is created on first use, "
                           "through a scratch allocation per call")
        if not isinstance(snap, EnvSnapshot):
            raise error.Error(f"{what}() needs an EnvSnapshot, got {type(snap).__name__}")
        R = self.snapshot_row_bytes
        check_compatible(snap.header, self.kind, R, self._snapshot_config())
        torch = _torch()
        r = snap.rows
        if not (isinstance(r, torch.Tensor) and r.dtype == torch.uint8 and r.device == self.device and r.dim() == 2
                and r.shape[1] == R and r.is_contiguous()):
            raise error.Error(f"{what}() needs the snapshot's rows as a contiguous uint8 (m, {R}) tensor on "
                              f"{self.device}")
        m = int(r.shape[0])
        if rows is None:
            idx, B = None, m
        elif isinstance(rows, torch.Tensor) and rows.is_cuda:
            if rows.dim() != 1 or rows.dtype.is_floating_point or rows.dtype == torch.bool or rows.device != self.device:
                raise error.Error(f"{what}() rows must be a 1-D integer tensor on {self.device}, got {rows.dtype} "
                                  f"of shape {tuple(rows.shape)} on {rows.device}")
            idx, B = rows, int(rows.shape[0])
        else:
            if captured:
                raise error.Error(f"{what}() cannot be captured in a CUDA graph with host rows: the host-to-device "
                                  "copy cannot be replayed; pass a CUDA tensor")
            idx = host_indices(rows.numpy() if isinstance(rows, torch.Tensor) else rows, m, f"{what} rows")
            B = int(idx.shape[0])
        if B < 1:
            raise error.Error(f"{what}() needs at least one branch, got B = 0")
        return captured, r, idx, B

    def _device_rows(self, idx):
        """_from_rows()'s row indices as the entry points take them: None, or int64 on the env's device."""
        if idx is None:
            return None
        torch = _torch()
        return (torch.from_numpy(idx) if isinstance(idx, np.ndarray) else idx).to(self.device, torch.int64).contiguous()

    def _from_outputs(self, B, states):
        """The outputs of rollout_from() / rollout_from_mlp(): returns, lengths, ended, and with states the end rows
        and observations (else None, None)."""
        torch = _torch()
        dev = self.device
        returns = torch.empty(B, dtype=torch.float64, device=dev)
        lengths = torch.empty(B, dtype=torch.int32, device=dev)
        ended = torch.empty(B, dtype=torch.bool, device=dev)
        end_rows = torch.empty((B, self.snapshot_row_bytes), dtype=torch.uint8, device=dev) if states else None
        end_obs = torch.empty((B, self.obs_dim), dtype=torch.float32, device=dev) if states else None
        return returns, lengths, ended, end_rows, end_obs

    def _noise_steps(self, noise, what="rollout_mlp_noisy", n=None):
        """Check rollout_mlp_noisy()'s or rollout_actor_critic()'s noise without a CUDA call -> T.  n: the batch it
        is drawn for (rollout_from_mlp()'s B), the env's num_envs when not given.  Its last axis is the action space's
        n or act_dim with or without a head= (a head's noise is A per env, whatever its K)."""
        n = self.num_envs if n is None else n
        torch = _torch()
        K = int(self.single_action_space.n if self.discrete else self.act_dim)
        if not isinstance(noise, torch.Tensor):
            raise ValueError(f"{what}() needs noise as a torch tensor, got {type(noise).__name__}")
        if noise.dtype != torch.float32:
            raise ValueError(f"{what}() needs float32 noise, got {noise.dtype}")
        if noise.device != self.device:
            raise ValueError(f"{what}() needs noise on {self.device}, got {noise.device}")
        if not noise.is_contiguous():
            raise ValueError(f"{what}() needs contiguous noise")
        if noise.dim() != 3 or tuple(noise.shape[1:]) != (n, K) or not 1 <= noise.shape[0] <= 2 ** 31 - 1:
            raise ValueError(f"{what}() needs noise (T, {n}, {K}) with 1 <= T < 2**31, got "
                             f"{tuple(noise.shape)}")
        return int(noise.shape[0])

    def _refuse_box2d_capture(self, what):
        """Raise if a Box2D env's policy rollout is being captured."""
        if self.kind in (_lib.KIND_LUNARLANDER, _lib.KIND_LUNARLANDER_CONT, _lib.KIND_BIPEDALWALKER,
                         _lib.KIND_BIPEDALWALKER_HARDCORE):
            refuse_capture(f"{what}() of a Box2D env", "its step 0 reads the observation rows the env last "
                           "returned, which alternate between two buffers from call to call, so a replay would read a "
                           "stale set")

    def _policy_rollout(self, what, T, summary, captured, launch, moments=False):
        """The checks after the parameters', the outputs, and the call of rollout_linear() / rollout_mlp() /
        rollout_mlp_noisy(), whose entry point ``launch(T, outs, last, first)`` calls with the output pointers, the
        buffer that receives the last observations and the observations the env last returned.  ``moments`` (summary
        mode only): the launch is also given the pointers of two new float64 (N, D) tensors, obs_sum and obs_sumsq,
        and they are returned after the summary."""
        if isinstance(T, (bool, np.bool_)) or not isinstance(T, (int, np.integer)) or not 1 <= int(T) <= 2 ** 31 - 1:
            raise ValueError(f"{what}(T) needs an integer 1 <= T < 2**31, got {T!r}")
        T = int(T)
        self._refuse_box2d_capture(what)
        first = self._out[self._flip]["obs"]   # the observations the env last returned, before the flip below
        sums = ()
        torch = _torch()
        n, dev, vp = self.num_envs, self.device, ctypes.c_void_p
        if summary:
            returns = torch.empty(n, dtype=torch.float64, device=dev)
            lengths = torch.empty(n, dtype=torch.int32, device=dev)
            ended = torch.empty(n, dtype=torch.bool, device=dev)
            self._flip ^= 1
            last = self._out[self._flip]["obs"]
            outs = [None] * 6 + [vp(returns.data_ptr()), vp(lengths.data_ptr()), vp(ended.data_ptr())]
            if moments:
                sums = tuple(torch.empty((n, self.obs_dim), dtype=torch.float64, device=dev) for _ in range(2))
        else:
            actions = torch.empty((T, n) if self.discrete else (T, n, self.act_dim),
                                  dtype=torch.int64 if self.discrete else torch.float32, device=dev)
            obs, reward, term, trunc, final_obs, last = self._rollout_outputs(T)
            outs = [vp(actions.data_ptr()), vp(obs.data_ptr()), vp(reward.data_ptr()), vp(term.data_ptr()),
                    vp(trunc.data_ptr()), vp(final_obs.data_ptr()) if self.autoreset else None, None, None, None]
        _lib.check(launch(T, outs, last, first, *(vp(x.data_ptr()) for x in sums)), self._handle)
        if summary:
            return (returns, lengths, ended) + sums
        return actions, obs, reward, term, trunc, FinalInfos(final_obs, term, trunc, None, captured)

    def _linear_params(self, weight, bias):
        """Check rollout_linear()'s parameters without a CUDA call -> whether they are per env."""
        torch = _torch()
        K = self.single_action_space.n if self.discrete else self.act_dim
        K, D, n = int(K), self.obs_dim, self.num_envs
        for name, x in (("weight", weight), ("bias", bias)):
            if not isinstance(x, torch.Tensor):
                raise ValueError(f"rollout_linear() needs {name} as a torch tensor, got {type(x).__name__}")
            if x.dtype != torch.float32:
                raise ValueError(f"rollout_linear() needs float32 {name}, got {x.dtype}")
            if x.device != self.device:
                raise ValueError(f"rollout_linear() needs {name} on {self.device}, got {x.device}")
            if not x.is_contiguous():
                raise ValueError(f"rollout_linear() needs a contiguous {name}")
        shared = tuple(weight.shape) == (K, D) and tuple(bias.shape) == (K,)
        per_env = tuple(weight.shape) == (n, K, D) and tuple(bias.shape) == (n, K)
        if not (shared or per_env):
            raise ValueError(f"rollout_linear() needs weight ({K}, {D}) and bias ({K},) for one policy, or weight "
                             f"({n}, {K}, {D}) and bias ({n}, {K}) for one per env; got {tuple(weight.shape)} and "
                             f"{tuple(bias.shape)}")
        return per_env

    def _mlp_head(self, what, head, obs_norm=None, clip_obs=None, obs_moments=False):
        """Check rollout_mlp()'s or rollout_mlp_noisy()'s head= without a CUDA call -> None for no head, else the
        b200gym_mlp_head code."""
        if head is None:
            return None
        if not isinstance(head, str) or head not in _lib.MLP_HEADS:
            raise ValueError(f"{what}() needs head None, 'tanh' or 'tanh_normal', got {head!r}")
        if self.discrete:
            raise ValueError(f"{what}() takes head= only for a Box action space, not "
                             f"{self.single_action_space!r}")
        if obs_norm is not None or clip_obs is not None or obs_moments:
            raise ValueError(f"{what}() does not take head= together with obs_norm, clip_obs or obs_moments")
        return _lib.MLP_HEADS[head]

    def _head_outputs(self, head):
        """K, the network outputs of head= (None, 'tanh' or 'tanh_normal') for a Box kind: act_dim, or 2 * act_dim
        for the SAC head's mean and log-std."""
        return int(self.act_dim) * (2 if head == "tanh_normal" else 1)

    def _mlp_params(self, params, hidden, activation, what="rollout_mlp", n=None, head=None):
        """Check rollout_mlp()'s or rollout_mlp_noisy()'s parameters without a CUDA call -> (h1, h2 (0 for one hidden
        layer), per_env, the b200gym_mlp_activation code).  n: the number of per-env rows (rollout_from_mlp()'s B),
        the env's num_envs when not given.  head: a head= that _mlp_head() accepted; it sets K."""
        n = self.num_envs if n is None else n
        torch = _torch()
        if not isinstance(activation, str) or activation not in _lib.MLP_ACTIVATIONS:
            raise ValueError(f"{what}() needs activation 'relu' or 'tanh', got {activation!r}")
        if not isinstance(hidden, (tuple, list)) or not 1 <= len(hidden) <= 2 or any(
                isinstance(h, (bool, np.bool_)) or not isinstance(h, (int, np.integer)) or not 1 <= int(h) <= 64
                for h in hidden):
            raise ValueError(f"{what}() needs hidden as a tuple of one or two widths, each 1 .. 64, got {hidden!r}")
        widths = [int(h) for h in hidden]
        K = self.single_action_space.n if self.discrete else self._head_outputs(head)
        sizes = [self.obs_dim] + widths + [int(K)]
        P = sum(o * i + o for i, o in zip(sizes[:-1], sizes[1:]))
        if not isinstance(params, torch.Tensor):
            raise ValueError(f"{what}() needs params as a torch tensor, got {type(params).__name__}")
        if params.dtype != torch.float32:
            raise ValueError(f"{what}() needs float32 params, got {params.dtype}")
        if params.device != self.device:
            raise ValueError(f"{what}() needs params on {self.device}, got {params.device}")
        if not params.is_contiguous():
            raise ValueError(f"{what}() needs contiguous params")
        per_env = tuple(params.shape) == (n, P)
        if not (per_env or tuple(params.shape) == (P,)):
            raise ValueError(f"{what}() with hidden {tuple(widths)} needs params ({P},) for one policy or "
                             f"({n}, {P}) for one per env; got {tuple(params.shape)}")
        return widths[0], widths[1] if len(widths) == 2 else 0, per_env, _lib.MLP_ACTIVATIONS[activation]

    def _rollout_guards(self, what, reset_needed=True):
        """The refusals of rollout() / rollout_sampled() / rollout_linear() / rollout_mlp() / rollout_mlp_noisy() /
        rollout_from(), all raised before any CUDA call -> whether a CUDA graph is being captured.  rollout_from()
        reads none of the env's state, so it passes reset_needed=False."""
        self._assert_open(what)
        if self.backend == "numpy":
            raise error.Error(f"{what}() needs backend='torch': backend='numpy' steps through host buffers")
        if self._chain is not None:
            raise error.Error(f"{what}() cannot run per-env wrappers (wrappers=): the chain runs after every step, "
                              "and the fused rollout kernel has no step boundary to run it at")
        if self._state != _STATE_DEFAULT:
            raise error.AlreadyPendingCallError(
                f"Calling `{what}` while waiting for a pending call to `{self._state}` to complete.", self._state)
        if reset_needed and not self._has_reset:
            raise error.ResetNeeded(f"Cannot call env.{what}() before calling env.reset()")
        captured = capturing()
        # the same poll as step_async: an invalid action of an earlier call raises here (not while capturing)
        if self.discrete and not captured and self._lib.b200gym_invalid_seen(self._handle) == 1:
            self.check_actions()
        self._raise_snapshot_index_error()
        return captured

    def _rollout_outputs(self, T):
        """(obs, reward, terminated, truncated, final_obs) with a leading T axis, new tensors, and the handle's buffer
        that receives the last observations."""
        torch = _torch()
        n, dev = self.num_envs, self.device
        shape = (T, n) + self._obs_shape
        obs = torch.empty(shape, dtype=torch.float32, device=dev)
        reward = torch.empty((T, n), dtype=torch.float64, device=dev)
        term = torch.empty((T, n), dtype=torch.bool, device=dev)
        trunc = torch.empty((T, n), dtype=torch.bool, device=dev)
        # without autoreset step() hands out a final_observation buffer that nothing writes
        final_obs = (torch.empty if self.autoreset else torch.zeros)(shape, dtype=torch.float32, device=dev)
        # the last observations also go to the next set of the double buffer, where snapshot() / clone() read them
        self._flip ^= 1
        return obs, reward, term, trunc, final_obs, self._out[self._flip]["obs"]

    def check_actions(self):
        """Number of out-of-range Discrete actions the device saw since the last check (syncs)."""
        refuse_capture("check_actions()", "it synchronises")
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
        so host and device sampling interleave freely.  ``backend="numpy"`` returns ``self.action_space.sample()``.

        May be captured in a CUDA graph once an eager call has put the generator on the device: each replay draws the
        next batch of the stream, which only the device follows until ``sync_action_space()`` (DESIGN §4.8)."""
        self._assert_open("sample_actions")
        space = self.action_space
        self._refuse_numpy_capture("sample_actions")
        if self.backend == "numpy":
            return space.sample()
        captured = capturing()
        n_choices, cols, low, high, bit_generator, state, words = self._sample_begin("sample_actions()", captured)
        shape = (self.num_envs,) if n_choices else (self.num_envs, cols)
        torch = _torch()
        out = torch.empty(shape, dtype=torch.int64 if n_choices else torch.float32, device=self.device)
        _lib.check(self._lib.b200gym_sample_space_stream(ctypes.c_void_p(self._sample_record.data_ptr()), words,
                                                         self.num_envs, cols, n_choices,
                                                         None if low is None else low.ctypes.data,
                                                         None if high is None else high.ctypes.data,
                                                         ctypes.c_void_p(out.data_ptr()), self._stream()))
        self._sample_end(bit_generator, state, out.numel(), captured)
        return out

    def _sample_begin(self, what, captured):
        """The launch arguments of a draw from the device record of the action space's stream (sample_actions(),
        rollout_sampled()) -> (n_choices, cols, low, high, bit generator, its state, override words or None)."""
        space = self.action_space
        n_choices, cols, low, high = self._sample_plan()
        shape = (self.num_envs,) if n_choices else (self.num_envs, cols)
        if (type(space).__name__ != ("MultiDiscrete" if n_choices else "Box") or tuple(space.shape) != shape
                or np.dtype(space.dtype) != (np.int64 if n_choices else np.float32)):
            raise error.Error(f"action_space {space!r} is no longer the batched space of {self.single_action_space!r}")
        bit_generator = space.np_random.bit_generator
        state = pcg64_state(bit_generator)
        s, inc = state["state"]["state"], state["state"]["inc"]
        # The draws come from the device record, which the launch also advances, so a captured call continues the
        # stream at every replay.  The mirror is what the host last left in the record: a host generator that differs
        # from it (drawn from or reseeded on the host) is passed as the override.
        in_sync = self._sample_mirror == (s, inc)
        if captured:
            if not in_sync:
                raise error.Error(f"{what} cannot be captured in a CUDA graph before the device holds the "
                                  f"action space's generator: call {what} once outside the capture (after "
                                  "any action_space.seed() or host draw)")
        mask = (1 << 64) - 1
        words = None if in_sync else (ctypes.c_uint64 * 4)(s >> 64, s & mask, inc >> 64, inc & mask)
        return n_choices, cols, low, high, bit_generator, state, words

    def _sample_end(self, bit_generator, state, count, captured):
        """After an eager launch that drew `count` elements: the host generator skips them and the mirror follows."""
        if not captured:   # a capture leaves the host where it is: replays advance the record alone
            pcg64_skip(bit_generator, state, count)
            st = pcg64_state(bit_generator)["state"]
            self._sample_mirror = (st["state"], st["inc"])

    def sync_action_space(self):
        """Move ``self.action_space``'s generator to where the device stream of ``sample_actions()`` is (synchronises).

        Replays of a CUDA graph that captured ``sample_actions()`` advance that stream on the device only; until this
        is called the host generator stays where the capture left it, and eager ``sample_actions()`` calls continue
        the device stream, not the host one.  torch backend only."""
        self._assert_open("sync_action_space")
        refuse_capture("sync_action_space()", "it synchronises")
        if self.backend == "numpy" or self._sample_mirror is None:
            return   # the host generator is the stream
        w = self._sample_record[:4].cpu().numpy().view(np.uint64)
        s, inc = (int(w[0]) << 64) | int(w[1]), (int(w[2]) << 64) | int(w[3])
        bit_generator = self.action_space.np_random.bit_generator
        st = bit_generator.state   # the buffered 32-bit draw stays, as sample_actions() leaves it
        st["state"] = {"state": s, "inc": inc}
        bit_generator.state = st
        self._sample_mirror = (s, inc)

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
        refuse_capture("set_state()", "it synchronises")
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

    def _snapshot_config(self):
        config = env_config(self.max_episode_steps, self.autoreset, self._params, self._cfg_flags)
        if self._chain is not None:
            config["wrappers"] = self._chain.describe()
        return config

    def _snapshot_header(self):
        return {"version": FORMAT_VERSION, "kind": self.kind, "row_bytes": self.snapshot_row_bytes,
                "config": self._snapshot_config()}

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
        refuse_capture(f"{what}()", "snapshots, restores and clones take host indices and synchronise")
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
            extras = {}
            if self._chain is not None:
                extras["subenv"] = self._chain.snapshot_extra(
                    lambda t: t.clone() if idx is None else t.index_select(0, self._in_range(idx, 0)))
        if self.backend == "numpy":
            torch.cuda.current_stream(self.device).synchronize()
            self._raise_snapshot_index_error()
        return EnvSnapshot(self._snapshot_header(), rows, obs, extras)

    def restore(self, snap, indices=None):
        """Load ``snap`` (row k into env ``indices[k]``; default: all envs, in order) -> ``(obs, {})`` like ``reset``,
        with the observations the snapshot was taken with.  The other envs are left as they are.  A snapshot of
        another kind or construction config raises ``error.Error``."""
        self._check_idle("restore")
        check_compatible(snap.header, self.kind, self.snapshot_row_bytes, self._snapshot_config())
        torch = _torch()
        m, n = len(snap), self.num_envs
        idx = self._index_tensor(indices, "restore indices")
        if idx is None and m != n:
            raise error.Error(f"a snapshot of {m} envs restores into {n} envs only with indices=")
        if idx is not None and int(idx.shape[0]) != m:
            raise error.Error(f"{int(idx.shape[0])} indices given for a snapshot of {m} envs")
        if self._chain is not None and "subenv" not in snap.extras:
            raise error.Error("the snapshot carries no state for this env's per-env wrappers")
        rows, sobs = snap.rows.to(self.device), snap.obs.to(self.device)
        with torch.cuda.device(self.device):
            if m:
                _lib.check(self._lib.b200gym_snapshot_load(
                    self._handle, ctypes.c_void_p(rows.data_ptr()), None,
                    None if idx is None else ctypes.c_void_p(idx.data_ptr()), m, self._stream()), self._handle)
            if self._chain is not None:
                self._chain.restore_extra(snap.extras["subenv"], lambda t, v: self._scatter_rows(t, idx, v))
            prev = self._last_obs()
            target = self._next_obs()
            if idx is None:
                target.copy_(sobs)
            else:   # row n of the scratch takes the observations of skipped (out-of-range) entries
                tmp = torch.empty((n + 1,) + self._obs_shape, dtype=torch.float32, device=self.device)
                tmp[:n].copy_(prev)
                tmp.index_copy_(0, self._in_range(idx, n), sobs)
                target.copy_(tmp[:n])
        if idx is None:
            self._has_reset = self._seeded = True
        return self._obs_result(target), {}

    def _scatter_rows(self, t, idx, values):
        """t[idx] = values along dim 0 (all rows: idx None); out-of-range entries land in a scratch row."""
        torch = _torch()
        values = values.to(self.device)
        if idx is None:
            t.copy_(values)
            return
        tmp = torch.cat([t, t[:1]])
        tmp.index_copy_(0, self._in_range(idx, self.num_envs), values)
        t.copy_(tmp[:self.num_envs])

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
            if self._chain is not None:
                self._chain.clone_extra(g)   # as deepcopy of the source sub-env would: its statistics come along
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
        if self._chain is not None:
            kw["wrappers"] = list(self._chain.stages)
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
