"""ctypes wrapper of tests/hostsim/rollout_mlp_tanh.cpp: the tanh instantiations of rollout_mlp_kernel's and
rollout_mlp_noisy_kernel's device source on the CPU.

Built on demand with g++ into tests/hostsim/_build/ (git-ignored), with the flags of rollout_sim.py.
"""
import ctypes
import os
import subprocess

import numpy as np

from hostsim import rollout_sim
from hostsim.rollout_mlp_noisy_sim import MlpNoisyRolloutSim

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = os.path.join(rollout_sim._BUILD, "librollout_mlp_tanh.so")
_SRCS = rollout_sim._SRCS + [os.path.join(_HERE, "rollout_mlp_tanh.cpp")]
_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB) or os.path.getmtime(_LIB) < max(os.path.getmtime(s) for s in _SRCS):
            os.makedirs(rollout_sim._BUILD, exist_ok=True)
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared",
                                   "-Wno-unknown-pragmas", "-o", _LIB, os.path.join(_HERE, "rollout_mlp_tanh.cpp")])
        L = ctypes.CDLL(_LIB)
        vp, i64, i32 = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int
        L.hs_mlp_tanh_rollout.restype = i64
        L.hs_mlp_tanh_rollout.argtypes = [ctypes.POINTER(rollout_sim._Batch), vp, i32, i32, i32, ctypes.c_int32] + \
            [vp] * 10
        L.hs_mlp_noisy_tanh_rollout.restype = i64
        L.hs_mlp_noisy_tanh_rollout.argtypes = [ctypes.POINTER(rollout_sim._Batch), vp, i32, i32, i32,
                                                ctypes.c_int32] + [vp] * 9
        _lib = L
    return _lib


class MlpTanhRolloutSim(MlpNoisyRolloutSim):
    """MlpNoisyRolloutSim whose ``rollout_mlp`` and ``rollout_mlp_noisy`` run the tanh launches: the same arguments and
    returns, with tanh after every hidden layer."""

    def rollout_mlp(self, params, hidden, T, summary=False, last_obs=None):
        w = np.ascontiguousarray(params, dtype=np.float32)
        per_env = w.ndim == 2
        h1, h2 = (hidden[0], 0) if len(hidden) == 1 else hidden
        last = np.zeros((self.n, self.obs_dim), dtype=np.float32) if last_obs is None else last_obs
        if summary:
            ret = np.full(self.n, np.nan)
            length = np.full(self.n, -1, dtype=np.int32)
            ended = np.full(self.n, 7, dtype=np.uint8)
            rc = lib().hs_mlp_tanh_rollout(ctypes.byref(self._b), w.ctypes.data, int(per_env), h1, h2, int(T),
                                           *([None] * 6), ret.ctypes.data, length.ctypes.data, ended.ctypes.data,
                                           last.ctypes.data)
            assert rc == 0
            return ret, length, ended.astype(bool)
        if self.act_dim == 0:
            acts = np.full((T, self.n), -1, dtype=np.int64)
        else:
            acts = np.full((T, self.n, self.act_dim), np.nan, dtype=np.float32)
        obs, rew, te, tr, fo = self._outputs((T, self.n))
        rc = lib().hs_mlp_tanh_rollout(ctypes.byref(self._b), w.ctypes.data, int(per_env), h1, h2, int(T),
                                       acts.ctypes.data, obs.ctypes.data, rew.ctypes.data, te.ctypes.data,
                                       tr.ctypes.data, fo.ctypes.data, None, None, None, last.ctypes.data)
        assert rc == 0
        return acts, obs, rew, te.astype(bool), tr.astype(bool), fo

    def rollout_mlp_noisy(self, params, hidden, noise, last_obs=None):
        w = np.ascontiguousarray(params, dtype=np.float32)
        e = np.ascontiguousarray(noise, dtype=np.float32)
        T = e.shape[0]
        per_env = w.ndim == 2
        h1, h2 = (hidden[0], 0) if len(hidden) == 1 else hidden
        last = np.zeros((self.n, self.obs_dim), dtype=np.float32) if last_obs is None else last_obs
        outputs = np.full(e.shape, np.nan, dtype=np.float32)
        if self.act_dim == 0:
            acts = np.full((T, self.n), -1, dtype=np.int64)
        else:
            acts = np.full((T, self.n, self.act_dim), np.nan, dtype=np.float32)
        obs, rew, te, tr, fo = self._outputs((T, self.n))
        rc = lib().hs_mlp_noisy_tanh_rollout(ctypes.byref(self._b), w.ctypes.data, int(per_env), h1, h2, int(T),
                                             e.ctypes.data, outputs.ctypes.data, acts.ctypes.data, obs.ctypes.data,
                                             rew.ctypes.data, te.ctypes.data, tr.ctypes.data, fo.ctypes.data,
                                             last.ctypes.data)
        assert rc == 0
        return acts, outputs, obs, rew, te.astype(bool), tr.astype(bool), fo
