"""ctypes wrapper of tests/hostsim/subenv.cpp: the device source of the per-env wrapper chains running on the CPU.

Built on demand with g++ into tests/hostsim/_build/ (git-ignored) with `-ffp-contract=off`, matching nvcc's
`-fmad=false`.
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_BUILD = os.path.join(_HERE, "_build")
_LIB = os.path.join(_BUILD, "libsubenv.so")
_SRCS = [os.path.join(_HERE, "subenv.cpp"), os.path.join(_HERE, "cuda_shim.h"),
         os.path.join(_ROOT, "gym_b200", "csrc", "subenv.cuh")]
_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB) or os.path.getmtime(_LIB) < max(os.path.getmtime(s) for s in _SRCS):
            os.makedirs(_BUILD, exist_ok=True)
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared",
                                   "-Wno-unknown-pragmas", "-o", _LIB, os.path.join(_HERE, "subenv.cpp")])
        L = ctypes.CDLL(_LIB)
        vp, i64, i32 = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int
        L.hs_subenv_step.argtypes = [vp, i32, i32, vp, vp, i32, i32, i64] + [vp] * 12
        L.hs_subenv_reset.argtypes = [vp, i32, i32, vp, vp, i32, i32, i64] + [vp] * 5
        L.hs_clip.argtypes = [vp, vp, i64, ctypes.c_float, ctypes.c_float]
        _lib = L
    return _lib


class HostChain:
    """The chain of a ``gym_b200.subenv.Chain`` (its resolved ``ops``) over n envs, state in numpy arrays laid out as
    on the device."""

    def __init__(self, chain, n):
        self.n, self.d = int(n), chain.obs_dim
        ops = chain.ops
        self.op = np.array([o[0] for o in ops] or [0], np.int32)
        self.p0 = np.array([o[1] for o in ops] or [0], np.float64)
        self.p1 = np.array([o[2] for o in ops] or [0], np.float64)
        self.raw_reward_type, self.int_reward_on_fall = chain.raw_reward_type, int(chain.int_reward_on_fall)
        self.k = len(ops)
        d = self.d
        self.obs_stats = np.zeros((2 * d + 1, n))
        self.obs_stats[d:2 * d] = 1.0
        self.obs_stats[2 * d] = 1e-4
        self.rew_stats = np.zeros((4, n))
        self.rew_stats[1] = 1.0
        self.rew_stats[2] = 1e-4
        self.ep_return = np.zeros(n, np.float32)
        self.ep_length = np.zeros(n, np.int32)

    def _head(self):
        return (self.op.ctypes.data, self.raw_reward_type, self.int_reward_on_fall, self.p0.ctypes.data,
                self.p1.ctypes.data, self.k, self.d, self.n, self.obs_stats.ctypes.data, self.rew_stats.ctypes.data, self.ep_return.ctypes.data,
                self.ep_length.ctypes.data)

    def reset(self, obs):
        obs = np.array(obs, np.float32, order="C")
        lib().hs_subenv_reset(*self._head(), obs.ctypes.data)
        return obs

    def step(self, obs, reward, terminated, truncated, final_obs):
        """-> obs, reward, final rows (float32 in place / float64), episode r / l (written for finishing envs only,
        NaN / -1 elsewhere)."""
        obs = np.array(obs, np.float32, order="C")
        reward = np.array(reward, np.float64, order="C")
        term = np.ascontiguousarray(terminated, np.uint8)
        trunc = np.ascontiguousarray(truncated, np.uint8)
        fin = np.array(final_obs, np.float32, order="C")
        fin64 = np.zeros((self.n, self.d))
        ep_r = np.full(self.n, np.nan, np.float32)
        ep_l = np.full(self.n, -1, np.int32)
        lib().hs_subenv_step(*self._head(), obs.ctypes.data, reward.ctypes.data, term.ctypes.data, trunc.ctypes.data,
                             fin.ctypes.data, fin64.ctypes.data, ep_r.ctypes.data, ep_l.ctypes.data)
        return obs, reward, fin, fin64, ep_r, ep_l


def clip(x, lo, hi):
    x = np.ascontiguousarray(x, np.float32)
    out = np.empty_like(x)
    lib().hs_clip(x.ctypes.data, out.ctypes.data, x.size, lo, hi)
    return out
