"""ctypes wrapper of tests/hostsim/rollout_sampled.cpp: the device source of rollout_sampled_kernel on the CPU.

Built on demand with g++ into tests/hostsim/_build/ (git-ignored), with the flags of rollout_sim.py.
"""
import ctypes
import os
import subprocess

import numpy as np

from hostsim import rollout_sim
from hostsim.rollout_sim import RolloutSim

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = os.path.join(rollout_sim._BUILD, "librollout_sampled.so")
_SRCS = rollout_sim._SRCS + [os.path.join(_HERE, "rollout_sampled.cpp"),
                             os.path.join(rollout_sim._ROOT, "gym_b200", "csrc", "space_sample.cuh")]
_lib = None

RECORD_WORDS = 5


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB) or os.path.getmtime(_LIB) < max(os.path.getmtime(s) for s in _SRCS):
            os.makedirs(rollout_sim._BUILD, exist_ok=True)
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared",
                                   "-Wno-unknown-pragmas", "-o", _LIB, os.path.join(_HERE, "rollout_sampled.cpp")])
        L = ctypes.CDLL(_LIB)
        vp, i64, dbl = ctypes.c_void_p, ctypes.c_int64, ctypes.c_double
        L.hs_ros_rollout.restype = i64
        L.hs_ros_rollout.argtypes = [ctypes.POINTER(rollout_sim._Batch), vp, vp, i64, dbl, dbl, ctypes.c_int32,
                                     vp, vp, vp, vp, vp, vp, vp]
        _lib = L
    return _lib


def words(state, inc):
    m = (1 << 64) - 1
    return np.array([state >> 64, state & m, inc >> 64, inc & m], dtype=np.uint64)


def new_record():
    return np.zeros(RECORD_WORDS, dtype=np.uint64)


def record_state(record):
    w = [int(x) for x in record[:4]]
    return (w[0] << 64) | w[1], (w[2] << 64) | w[3]


class SampledRolloutSim(RolloutSim):
    """RolloutSim plus ``rollout_sampled``, one rollout_sampled_kernel launch."""

    def rollout_sampled(self, record, T, n_choices=0, low=0.0, high=0.0, override=None, last_obs=None):
        """T steps of actions drawn from `record` (uint64 [RECORD_WORDS], updated in place) or from `override`
        ((state, inc) or None) -> (actions, obs, rew, term, trunc, final_obs) with a leading T axis, the invalid-action
        count.  actions is int64 (T, n) when n_choices > 0, float32 (T, n, 1) otherwise."""
        if n_choices:
            acts = np.full((T, self.n), -1, dtype=np.int64)
        else:
            acts = np.full((T, self.n, 1), np.nan, dtype=np.float32)
        obs, rew, te, tr, fo = self._outputs((T, self.n))
        last = np.zeros((self.n, self.obs_dim), dtype=np.float32) if last_obs is None else last_obs
        ov = None if override is None else words(*override)
        bad = lib().hs_ros_rollout(ctypes.byref(self._b), record.ctypes.data, None if ov is None else ov.ctypes.data,
                                   int(n_choices), float(low), float(high), int(T), acts.ctypes.data, obs.ctypes.data,
                                   rew.ctypes.data, te.ctypes.data, tr.ctypes.data, fo.ctypes.data, last.ctypes.data)
        assert bad >= 0
        return acts, obs, rew, te.astype(bool), tr.astype(bool), fo, int(bad)
