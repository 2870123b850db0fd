"""ctypes wrapper of tests/hostsim/rollout_from.cpp: the device source of rollout_from_kernel on the CPU.

Built on demand with g++ into tests/hostsim/_build/ (git-ignored), with the flags of rollout_sim.py.
"""
import ctypes
import os
import subprocess

import numpy as np

from hostsim import rollout_sim
from hostsim.rollout_sim import RolloutSim

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = os.path.join(rollout_sim._BUILD, "librollout_from.so")
_SRCS = rollout_sim._SRCS + [os.path.join(_HERE, "rollout_from.cpp")]
_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB) or os.path.getmtime(_LIB) < max(os.path.getmtime(s) for s in _SRCS):
            os.makedirs(rollout_sim._BUILD, exist_ok=True)
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared",
                                   "-Wno-unknown-pragmas", "-o", _LIB, os.path.join(_HERE, "rollout_from.cpp")])
        L = ctypes.CDLL(_LIB)
        vp, i64 = ctypes.c_void_p, ctypes.c_int64
        bp = ctypes.POINTER(rollout_sim._Batch)
        L.hs_rf_rollout_from.restype = i64
        L.hs_rf_rollout_from.argtypes = [bp, vp, i64, vp, i64, vp, ctypes.c_int32, vp, vp, vp, vp, vp, vp]
        L.hs_rf_row_bytes.restype = i64
        L.hs_rf_row_bytes.argtypes = [bp]
        _lib = L
    return _lib


class RolloutFromSim(RolloutSim):
    """RolloutSim plus ``rollout_from``, one rollout_from_kernel launch over snapshot rows (the batch's own arrays are
    neither read nor written by it: only its configuration is used)."""

    @property
    def row_bytes(self):
        return int(lib().hs_rf_row_bytes(ctypes.byref(self._b)))

    def rollout_from(self, rows, actions, row_idx=None, states=False):
        """rows (m, row_bytes) uint8, actions (T, B[, 1]), row_idx (B,) int64 or None -> (returns, lengths, ended,
        end_rows, end_obs, invalid, bad); end_rows / end_obs None unless states."""
        rows = np.ascontiguousarray(rows, dtype=np.uint8)
        a = np.ascontiguousarray(actions, dtype=np.int64 if self.act_dim == 0 else np.float32)
        T, B = a.shape[0], a.shape[1]
        idx = None if row_idx is None else np.ascontiguousarray(row_idx, dtype=np.int64)
        # poisoned outputs: every byte must be written
        ret = np.full(B, np.nan)
        length = np.full(B, -1, dtype=np.int32)
        ended = np.full(B, 7, dtype=np.uint8)
        end_rows = np.full((B, rows.shape[1]), 0xAB, dtype=np.uint8) if states else None
        end_obs = np.full((B, self.obs_dim), np.nan, dtype=np.float32) if states else None
        bad = ctypes.c_ulonglong(0)
        invalid = lib().hs_rf_rollout_from(
            ctypes.byref(self._b), rows.ctypes.data, rows.shape[0], None if idx is None else idx.ctypes.data, B,
            a.ctypes.data, T, ret.ctypes.data, length.ctypes.data, ended.ctypes.data,
            None if end_rows is None else end_rows.ctypes.data, None if end_obs is None else end_obs.ctypes.data,
            ctypes.byref(bad))
        assert invalid >= 0
        return ret, length, ended.astype(bool), end_rows, end_obs, int(invalid), int(bad.value)
