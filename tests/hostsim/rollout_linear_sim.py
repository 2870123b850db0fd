"""ctypes wrapper of tests/hostsim/rollout_linear.cpp: the device source of rollout_linear_kernel on the CPU.

Built on demand with g++ into tests/hostsim/_build/ (git-ignored), with the flags of rollout_sim.py.
"""
import ctypes
import os
import subprocess

import numpy as np

from hostsim import rollout_sim
from hostsim.rollout_sim import RolloutSim

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = os.path.join(rollout_sim._BUILD, "librollout_linear.so")
_SRCS = rollout_sim._SRCS + [os.path.join(_HERE, "rollout_linear.cpp")]
_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB) or os.path.getmtime(_LIB) < max(os.path.getmtime(s) for s in _SRCS):
            os.makedirs(rollout_sim._BUILD, exist_ok=True)
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared",
                                   "-Wno-unknown-pragmas", "-o", _LIB, os.path.join(_HERE, "rollout_linear.cpp")])
        L = ctypes.CDLL(_LIB)
        vp, i64, i32 = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int
        bp = ctypes.POINTER(rollout_sim._Batch)
        L.hs_rol_rollout.restype = i64
        L.hs_rol_rollout.argtypes = [bp, vp, vp, i32, ctypes.c_int32] + [vp] * 10
        L.hs_rol_observe.restype = i64
        L.hs_rol_observe.argtypes = [bp, vp]
        _lib = L
    return _lib


class LinearRolloutSim(RolloutSim):
    """RolloutSim plus ``rollout_linear``, one rollout_linear_kernel launch, and ``observe``."""

    def rollout_linear(self, weight, bias, T, summary=False, last_obs=None):
        """T steps of the linear policy (weight (K, D) / bias (K,), or (n, K, D) / (n, K)) -> summary=False:
        (actions, obs, rew, term, trunc, final_obs) with a leading T axis; summary=True: (returns, lengths, ended)."""
        w = np.ascontiguousarray(weight, dtype=np.float32)
        b = np.ascontiguousarray(bias, dtype=np.float32)
        per_env = w.ndim == 3
        last = np.zeros((self.n, self.obs_dim), dtype=np.float32) if last_obs is None else last_obs
        if summary:
            ret = np.full(self.n, np.nan)
            length = np.full(self.n, -1, dtype=np.int32)
            ended = np.full(self.n, 7, dtype=np.uint8)
            rc = lib().hs_rol_rollout(ctypes.byref(self._b), w.ctypes.data, b.ctypes.data, int(per_env), int(T),
                                      *([None] * 6), ret.ctypes.data, length.ctypes.data, ended.ctypes.data,
                                      last.ctypes.data)
            assert rc == 0
            return ret, length, ended.astype(bool)
        if self.act_dim == 0:
            acts = np.full((T, self.n), -1, dtype=np.int64)
        else:
            acts = np.full((T, self.n, self.act_dim), np.nan, dtype=np.float32)
        obs, rew, te, tr, fo = self._outputs((T, self.n))
        rc = lib().hs_rol_rollout(ctypes.byref(self._b), w.ctypes.data, b.ctypes.data, int(per_env), int(T),
                                  acts.ctypes.data, obs.ctypes.data, rew.ctypes.data, te.ctypes.data, tr.ctypes.data,
                                  fo.ctypes.data, None, None, None, last.ctypes.data)
        assert rc == 0
        return acts, obs, rew, te.astype(bool), tr.astype(bool), fo

    def observe(self):
        """Env<KIND>::observe of every env's state -> (n, obs_dim) float32."""
        obs = np.zeros((self.n, self.obs_dim), dtype=np.float32)
        assert lib().hs_rol_observe(ctypes.byref(self._b), obs.ctypes.data) == 0
        return obs
