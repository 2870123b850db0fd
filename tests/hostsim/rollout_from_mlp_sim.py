"""ctypes wrapper of tests/hostsim/rollout_from_mlp.cpp: the device source of rollout_from_mlp_kernel on the CPU.

Built on demand with g++ into tests/hostsim/_build/ (git-ignored), with the flags of rollout_sim.py.
"""
import ctypes
import math
import os
import subprocess

import numpy as np

from hostsim import rollout_sim
from hostsim.rollout_from_sim import RolloutFromSim

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = os.path.join(rollout_sim._BUILD, "librollout_from_mlp.so")
_SRCS = rollout_sim._SRCS + [os.path.join(_HERE, "rollout_from_mlp.cpp")]
_lib = None

RELU, TANH = 0, 1


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB) or os.path.getmtime(_LIB) < max(os.path.getmtime(s) for s in _SRCS):
            os.makedirs(rollout_sim._BUILD, exist_ok=True)
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared",
                                   "-Wno-unknown-pragmas", "-o", _LIB, os.path.join(_HERE, "rollout_from_mlp.cpp")])
        L = ctypes.CDLL(_LIB)
        vp, i64, i32 = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int
        L.hs_rfm_rollout_from_mlp.restype = i64
        L.hs_rfm_rollout_from_mlp.argtypes = [ctypes.POINTER(rollout_sim._Batch), vp, i64, vp, i64, vp, i32, i32, i32,
                                              i32, ctypes.c_int32, vp, vp, vp, ctypes.c_double, ctypes.c_float] + \
            [vp] * 7
        _lib = L
    return _lib


def _ptr(x):
    return None if x is None else x.ctypes.data


class RolloutFromMlpSim(RolloutFromSim):
    """RolloutFromSim plus ``rollout_from_mlp``, one rollout_from_mlp_kernel launch over snapshot rows (the batch's own
    arrays are neither read nor written by it: only its configuration is used)."""

    def rollout_from_mlp(self, rows, params, hidden, T, row_idx=None, noise=None, act=RELU, mean=None, var=None,
                         eps=1e-8, clip=None, states=False):
        """rows (m, row_bytes) uint8, params (P,) or (B, P), noise None or (T, B, K), row_idx (B,) int64 or None ->
        (returns, lengths, ended, first_actions, end_rows, end_obs, invalid, bad); end_rows / end_obs None unless
        states."""
        rows = np.ascontiguousarray(rows, dtype=np.uint8)
        idx = None if row_idx is None else np.ascontiguousarray(row_idx, dtype=np.int64)
        B = rows.shape[0] if idx is None else idx.shape[0]
        w = np.ascontiguousarray(params, dtype=np.float32)
        per_branch = w.ndim == 2
        h1, h2 = (hidden[0], 0) if len(hidden) == 1 else hidden
        e = None if noise is None else np.ascontiguousarray(noise, dtype=np.float32)
        m = None if mean is None else np.ascontiguousarray(mean, dtype=np.float64)
        v = None if var is None else np.ascontiguousarray(var, dtype=np.float64)
        c = math.inf if clip is None else float(np.float32(clip))
        # poisoned outputs: every byte must be written
        ret = np.full(B, np.nan)
        length = np.full(B, -1, dtype=np.int32)
        ended = np.full(B, 7, dtype=np.uint8)
        first = np.full(B, -1, dtype=np.int64) if self.act_dim == 0 else np.full((B, self.act_dim), np.nan,
                                                                                   dtype=np.float32)
        end_rows = np.full((B, rows.shape[1]), 0xAB, dtype=np.uint8) if states else None
        end_obs = np.full((B, self.obs_dim), np.nan, dtype=np.float32) if states else None
        bad = ctypes.c_ulonglong(0)
        invalid = lib().hs_rfm_rollout_from_mlp(
            ctypes.byref(self._b), rows.ctypes.data, rows.shape[0], _ptr(idx), B, w.ctypes.data, int(per_branch), h1,
            h2, act, int(T), _ptr(e), _ptr(m), _ptr(v), float(eps), c, ret.ctypes.data, length.ctypes.data,
            ended.ctypes.data, first.ctypes.data, _ptr(end_rows), _ptr(end_obs), ctypes.byref(bad))
        assert invalid >= 0
        return ret, length, ended.astype(bool), first, end_rows, end_obs, int(invalid), int(bad.value)
