"""ctypes wrapper of tests/hostsim/rollout_policy_norm.cpp: the device source of rollout_linear_norm_kernel and
rollout_mlp_norm_kernel on the CPU.

Built on demand with g++ into tests/hostsim/_build/ (git-ignored), with the flags of rollout_sim.py.
"""
import ctypes
import math
import os
import subprocess

import numpy as np

from hostsim import rollout_sim
from hostsim.rollout_mlp_sim import MlpRolloutSim

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = os.path.join(rollout_sim._BUILD, "librollout_policy_norm.so")
_SRCS = rollout_sim._SRCS + [os.path.join(_HERE, "rollout_policy_norm.cpp")]
_lib = None

RELU, TANH = 0, 1


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB) or os.path.getmtime(_LIB) < max(os.path.getmtime(s) for s in _SRCS):
            os.makedirs(rollout_sim._BUILD, exist_ok=True)
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared",
                                   "-Wno-unknown-pragmas", "-o", _LIB, os.path.join(_HERE, "rollout_policy_norm.cpp")])
        L = ctypes.CDLL(_LIB)
        vp, i64, i32, f32, f64 = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_float, ctypes.c_double
        L.hs_linear_norm_rollout.restype = i64
        L.hs_linear_norm_rollout.argtypes = [ctypes.POINTER(rollout_sim._Batch), vp, vp, i32, ctypes.c_int32] + \
            [vp] * 10 + [vp, vp, f64, f32, vp, vp]
        L.hs_mlp_norm_rollout.restype = i64
        L.hs_mlp_norm_rollout.argtypes = [ctypes.POINTER(rollout_sim._Batch), vp, i32, i32, i32, i32,
                                          ctypes.c_int32] + [vp] * 10 + [vp, vp, f64, f32, vp, vp]
        _lib = L
    return _lib


def _ptr(x):
    return None if x is None else x.ctypes.data


class PolicyNormRolloutSim(MlpRolloutSim):
    """MlpRolloutSim plus the normalised closed-loop launches.  mean / var None: raw inputs."""

    def _policy_norm(self, call, T, summary, mean, var, eps, clip, moments, last_obs):
        m = None if mean is None else np.ascontiguousarray(mean, dtype=np.float64)
        v = None if var is None else np.ascontiguousarray(var, dtype=np.float64)
        c = math.inf if clip is None else float(np.float32(clip))
        last = np.zeros((self.n, self.obs_dim), dtype=np.float32) if last_obs is None else last_obs
        stats = [_ptr(m), _ptr(v), float(eps), c]
        if summary:
            ret = np.full(self.n, np.nan)
            length = np.full(self.n, -1, dtype=np.int32)
            ended = np.full(self.n, 7, dtype=np.uint8)
            s = q = None
            if moments:
                s = np.full((self.n, self.obs_dim), np.nan)
                q = np.full((self.n, self.obs_dim), np.nan)
            rc = call(*([None] * 6), ret.ctypes.data, length.ctypes.data, ended.ctypes.data, last.ctypes.data,
                      *stats, _ptr(s), _ptr(q))
            assert rc == 0
            return (ret, length, ended.astype(bool)) + ((s, q) if moments else ())
        if self.act_dim == 0:
            acts = np.full((T, self.n), -1, dtype=np.int64)
        else:
            acts = np.full((T, self.n, self.act_dim), np.nan, dtype=np.float32)
        obs, rew, te, tr, fo = self._outputs((T, self.n))
        rc = call(acts.ctypes.data, obs.ctypes.data, rew.ctypes.data, te.ctypes.data, tr.ctypes.data, fo.ctypes.data,
                  None, None, None, last.ctypes.data, *stats, None, None)
        assert rc == 0
        return acts, obs, rew, te.astype(bool), tr.astype(bool), fo

    def rollout_linear_norm(self, weight, bias, T, mean, var, eps, clip, summary=False, moments=False, last_obs=None):
        """-> rollout_linear's outputs; summary with moments: (returns, lengths, ended, obs_sum, obs_sumsq)."""
        w = np.ascontiguousarray(weight, dtype=np.float32)
        b = np.ascontiguousarray(bias, dtype=np.float32)
        per_env = w.ndim == 3
        call = lambda *a: lib().hs_linear_norm_rollout(  # noqa: E731
            ctypes.byref(self._b), w.ctypes.data, b.ctypes.data, int(per_env), int(T), *a)
        return self._policy_norm(call, T, summary, mean, var, eps, clip, moments, last_obs)

    def rollout_mlp_norm(self, params, hidden, T, mean, var, eps, clip, act=RELU, summary=False, moments=False,
                         last_obs=None):
        """-> rollout_mlp's outputs; summary with moments as rollout_linear_norm."""
        w = np.ascontiguousarray(params, dtype=np.float32)
        per_env = w.ndim == 2
        h1, h2 = (hidden[0], 0) if len(hidden) == 1 else hidden
        call = lambda *a: lib().hs_mlp_norm_rollout(  # noqa: E731
            ctypes.byref(self._b), w.ctypes.data, int(per_env), h1, h2, act, int(T), *a)
        return self._policy_norm(call, T, summary, mean, var, eps, clip, moments, last_obs)
