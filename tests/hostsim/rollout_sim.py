"""ctypes wrapper of tests/hostsim/rollout.cpp: the device source of rollout_kernel and kernel A on the CPU.

Built on demand with g++ into tests/hostsim/_build/ (git-ignored), with the flags of sim.py.
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_BUILD = os.path.join(_HERE, "_build")
_LIB = os.path.join(_BUILD, "librollout.so")
_SRCS = [os.path.join(_HERE, "rollout.cpp"), os.path.join(_HERE, "cuda_shim.h"),
         os.path.join(_ROOT, "include", "b200gym.h")] + [
    os.path.join(_ROOT, "gym_b200", "csrc", f) for f in ("rng.cuh", "envs.cuh", "glibc_trig.cuh", "b2lite.cuh",
                                                         "b2lite_toi.cuh", "lunar.cuh", "walker.cuh", "per_env.cuh",
                                                         "box2d_consts.h")]
_lib = None

# enum b200gym_action_dtype
ACT_I64, ACT_I32, ACT_U8, ACT_F32 = 0, 1, 2, 3
DTYPE_CODE = {np.dtype(np.int64): ACT_I64, np.dtype(np.int32): ACT_I32, np.dtype(np.uint8): ACT_U8,
              np.dtype(np.float32): ACT_F32}
# kind -> (obs_dim, act_dim, state_dim); enum b200gym_kind
DIMS = {0: (4, 0, 4), 1: (2, 0, 2), 2: (2, 1, 2), 3: (3, 1, 2), 4: (6, 0, 4)}


class _Batch(ctypes.Structure):
    """struct Batch of rollout.cpp"""
    _fields_ = [("kind", ctypes.c_int32), ("max_steps", ctypes.c_int32), ("autoreset", ctypes.c_int32),
                ("pad", ctypes.c_int32), ("n", ctypes.c_int64), ("param0", ctypes.c_double),
                ("state", ctypes.c_void_p), ("elapsed", ctypes.c_void_p), ("flags", ctypes.c_void_p),
                ("rng", ctypes.c_void_p)]


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB) or os.path.getmtime(_LIB) < max(os.path.getmtime(s) for s in _SRCS):
            os.makedirs(_BUILD, exist_ok=True)
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared",
                                   "-Wno-unknown-pragmas", "-o", _LIB, os.path.join(_HERE, "rollout.cpp")])
        L = ctypes.CDLL(_LIB)
        vp, i64, i32, bp = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.POINTER(_Batch)
        L.hs_ro_seed_range.argtypes = [bp, vp, i64]
        L.hs_ro_reset.restype = i64
        L.hs_ro_reset.argtypes = [bp, vp, vp]
        L.hs_ro_step.restype = i64
        L.hs_ro_step.argtypes = [bp, i32, vp, vp, vp, vp, vp, vp]
        L.hs_ro_rollout.restype = i64
        L.hs_ro_rollout.argtypes = [bp, i32, ctypes.c_int32, vp, vp, vp, vp, vp, vp, vp]
        _lib = L
    return _lib


class RolloutSim:
    """A batch of classic-control envs in the handle's layout, stepped on the CPU by the kernels' per-env drivers.
    ``step`` is one kernel-A launch, ``rollout`` one rollout_kernel launch; both return the outputs the torch backend
    returns (final observations zero where nothing was written) plus the number of invalid actions met."""

    def __init__(self, kind, num_envs, max_episode_steps=None, autoreset=True, param0=0.0):
        self.kind, self.n = int(kind), int(num_envs)
        self.obs_dim, self.act_dim, self.state_dim = DIMS[self.kind]
        self.state = np.zeros((self.state_dim, self.n), dtype=np.float64)   # SoA, as on the device
        self.elapsed = np.zeros(self.n, dtype=np.int32)
        self.flags = np.zeros(self.n, dtype=np.uint8)
        self.rng = np.zeros((self.n, 4), dtype=np.uint64)
        self._b = _Batch(kind=self.kind, max_steps=int(max_episode_steps or 0), autoreset=int(bool(autoreset)), pad=0,
                         n=self.n, param0=float(param0), state=self.state.ctypes.data,
                         elapsed=self.elapsed.ctypes.data, flags=self.flags.ctypes.data, rng=self.rng.ctypes.data)

    def reset(self, seed, bounds=None):
        words = np.array([(int(seed) >> (32 * k)) & 0xFFFFFFFF for k in range(4)], dtype=np.uint32)
        lib().hs_ro_seed_range(ctypes.byref(self._b), words.ctypes.data, 0)
        obs = np.zeros((self.n, self.obs_dim), dtype=np.float32)
        b = None if bounds is None else np.ascontiguousarray(bounds, dtype=np.float64)
        assert lib().hs_ro_reset(ctypes.byref(self._b), None if b is None else b.ctypes.data, obs.ctypes.data) == 0
        return obs

    def _outputs(self, lead):
        return (np.zeros(lead + (self.obs_dim,), dtype=np.float32), np.zeros(lead, dtype=np.float64),
                np.zeros(lead, dtype=np.uint8), np.zeros(lead, dtype=np.uint8),
                np.zeros(lead + (self.obs_dim,), dtype=np.float32))

    def step(self, actions):
        a = np.ascontiguousarray(actions)
        obs, rew, te, tr, fo = self._outputs((self.n,))
        bad = lib().hs_ro_step(ctypes.byref(self._b), DTYPE_CODE[a.dtype], a.ctypes.data, obs.ctypes.data,
                               rew.ctypes.data, te.ctypes.data, tr.ctypes.data, fo.ctypes.data)
        assert bad >= 0
        return obs, rew, te.astype(bool), tr.astype(bool), fo, int(bad)

    def rollout(self, actions, last_obs=None):
        """actions (T, n[, 1]) -> (obs, rew, term, trunc, final_obs) with a leading T axis, the invalid-action count;
        `last_obs` (n, obs_dim) float32, if given, receives obs[T-1] as the handle's own buffer does."""
        a = np.ascontiguousarray(actions)
        T = a.shape[0]
        obs, rew, te, tr, fo = self._outputs((T, self.n))
        last = np.zeros((self.n, self.obs_dim), dtype=np.float32) if last_obs is None else last_obs
        bad = lib().hs_ro_rollout(ctypes.byref(self._b), DTYPE_CODE[a.dtype], T, a.ctypes.data, obs.ctypes.data,
                                  rew.ctypes.data, te.ctypes.data, tr.ctypes.data, fo.ctypes.data, last.ctypes.data)
        assert bad >= 0
        return obs, rew, te.astype(bool), tr.astype(bool), fo, int(bad)

    def get_state(self):
        return self.state.T.copy(), self.elapsed.copy(), self.flags.copy(), self.rng.copy()
