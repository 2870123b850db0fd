"""ctypes wrapper of tests/hostsim/rollout_mlp_head.cpp: the device source of rollout_mlp_head_kernel and
rollout_mlp_noisy_head_kernel on the CPU.

Built on demand with g++ into tests/hostsim/_build/ (git-ignored), with the flags of rollout_sim.py.
"""
import ctypes
import os
import subprocess

import numpy as np

from hostsim import rollout_sim
from hostsim.rollout_mlp_noisy_sim import MlpNoisyRolloutSim

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = os.path.join(rollout_sim._BUILD, "librollout_mlp_head.so")
_SRCS = rollout_sim._SRCS + [os.path.join(_HERE, "rollout_mlp_head.cpp")]
_lib = None

# enum b200gym_mlp_activation, enum b200gym_mlp_head
ACTIVATIONS = {"relu": 0, "tanh": 1}
HEADS = {"tanh": 1, "tanh_normal": 2}


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB) or os.path.getmtime(_LIB) < max(os.path.getmtime(s) for s in _SRCS):
            os.makedirs(rollout_sim._BUILD, exist_ok=True)
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared",
                                   "-Wno-unknown-pragmas", "-o", _LIB, os.path.join(_HERE, "rollout_mlp_head.cpp")])
        L = ctypes.CDLL(_LIB)
        vp, i64, i32 = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int
        L.hs_mlp_head_rollout.restype = i64
        L.hs_mlp_head_rollout.argtypes = [ctypes.POINTER(rollout_sim._Batch), vp, i32, i32, i32, ctypes.c_int32, i32,
                                          i32] + [vp] * 11
        L.hs_mlp_noisy_head_rollout.restype = i64
        L.hs_mlp_noisy_head_rollout.argtypes = [ctypes.POINTER(rollout_sim._Batch), vp, i32, i32, i32, ctypes.c_int32,
                                                i32, i32] + [vp] * 10
        _lib = L
    return _lib


class MlpHeadRolloutSim(MlpNoisyRolloutSim):
    """MlpNoisyRolloutSim plus ``rollout_mlp_head`` and ``rollout_mlp_noisy_head``, one launch each of the head kernels.
    ``bounds`` is float32 (low, high, scale, bias), the HeadBounds the launch is given."""

    def rollout_mlp_head(self, params, hidden, T, activation, head, bounds, summary=False, last_obs=None):
        w = np.ascontiguousarray(params, dtype=np.float32)
        b = np.ascontiguousarray(bounds, dtype=np.float32)
        per_env = w.ndim == 2
        h1, h2 = (hidden[0], 0) if len(hidden) == 1 else hidden
        last = np.zeros((self.n, self.obs_dim), dtype=np.float32) if last_obs is None else last_obs
        args = (ctypes.byref(self._b), w.ctypes.data, int(per_env), h1, h2, int(T), ACTIVATIONS[activation],
                HEADS[head], b.ctypes.data)
        if summary:
            ret = np.full(self.n, np.nan)
            length = np.full(self.n, -1, dtype=np.int32)
            ended = np.full(self.n, 7, dtype=np.uint8)
            rc = lib().hs_mlp_head_rollout(*args, *([None] * 6), ret.ctypes.data, length.ctypes.data,
                                           ended.ctypes.data, last.ctypes.data)
            assert rc == 0
            return ret, length, ended.astype(bool)
        acts = np.full((T, self.n, self.act_dim), np.nan, dtype=np.float32)
        obs, rew, te, tr, fo = self._outputs((T, self.n))
        rc = lib().hs_mlp_head_rollout(*args, acts.ctypes.data, obs.ctypes.data, rew.ctypes.data, te.ctypes.data,
                                       tr.ctypes.data, fo.ctypes.data, None, None, None, last.ctypes.data)
        assert rc == 0
        return acts, obs, rew, te.astype(bool), tr.astype(bool), fo

    def rollout_mlp_noisy_head(self, params, hidden, noise, activation, head, bounds, last_obs=None):
        w = np.ascontiguousarray(params, dtype=np.float32)
        e = np.ascontiguousarray(noise, dtype=np.float32)
        b = np.ascontiguousarray(bounds, dtype=np.float32)
        T = e.shape[0]
        K = self.act_dim * (2 if head == "tanh_normal" else 1)
        per_env = w.ndim == 2
        h1, h2 = (hidden[0], 0) if len(hidden) == 1 else hidden
        last = np.zeros((self.n, self.obs_dim), dtype=np.float32) if last_obs is None else last_obs
        outputs = np.full((T, self.n, K), np.nan, dtype=np.float32)
        acts = np.full((T, self.n, self.act_dim), np.nan, dtype=np.float32)
        obs, rew, te, tr, fo = self._outputs((T, self.n))
        rc = lib().hs_mlp_noisy_head_rollout(ctypes.byref(self._b), w.ctypes.data, int(per_env), h1, h2, int(T),
                                             ACTIVATIONS[activation], HEADS[head], b.ctypes.data, e.ctypes.data,
                                             outputs.ctypes.data, acts.ctypes.data, obs.ctypes.data, rew.ctypes.data,
                                             te.ctypes.data, tr.ctypes.data, fo.ctypes.data, last.ctypes.data)
        assert rc == 0
        return acts, outputs, obs, rew, te.astype(bool), tr.astype(bool), fo
