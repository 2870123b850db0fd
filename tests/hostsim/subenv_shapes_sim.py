"""ctypes wrapper of tests/hostsim/subenv_shapes.cpp: the reshaping wrapper chains and the action stages of
gym_b200/csrc/subenv.cuh running on the CPU.

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
_LIB = os.path.join(_BUILD, "libsubenv_shapes.so")
_SRCS = [os.path.join(_HERE, "subenv_shapes.cpp"), os.path.join(_HERE, "cuda_shim.h"),
         os.path.join(_ROOT, "gym_b200", "csrc", "subenv.cuh")]
_lib = None


class _State(ctypes.Structure):
    _fields_ = [(k, ctypes.c_void_p) for k in ("obs_stats", "rew_stats", "ep_return", "ep_length", "history", "head",
                                                 "t")]


class _Actions(ctypes.Structure):
    _fields_ = [("num", ctypes.c_int32), ("op", ctypes.c_int32 * 2)] + [
        (k, (ctypes.c_float * 4) * 2) for k in ("lo", "hi", "amin", "amax")]


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB) or os.path.getmtime(_LIB) < max(os.path.getmtime(s) for s in _SRCS):
            os.makedirs(_BUILD, exist_ok=True)
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared",
                                   "-Wno-unknown-pragmas", "-o", _LIB, os.path.join(_HERE, "subenv_shapes.cpp")])
        L = ctypes.CDLL(_LIB)
        vp, i64, i32 = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int
        head = [vp, vp, vp, i32, i32, i32, i32, i64, ctypes.POINTER(_State)]
        L.hs_shape_width.argtypes = [vp, vp, i32, i32, vp]
        L.hs_shape_step.argtypes = head + [vp] * 10
        L.hs_shape_reset.argtypes = head + [vp] * 2
        L.hs_actions.argtypes = [ctypes.POINTER(_Actions), vp, vp, i64, i32]
        _lib = L
    return _lib


class HostShapeChain:
    """A reshaping ``gym_b200.subenv.Chain`` (its resolved ``ops``) over n envs, state in numpy arrays laid out as on
    the device (``Chain.allocate``)."""

    def __init__(self, chain, n):
        assert chain.reshape, "the host build runs the reshaping path only"
        self.chain, self.n, self.d = chain, int(n), chain.obs_dim
        ops = chain.ops
        self.op = np.array([o[0] for o in ops], np.int32)
        self.p0 = np.array([o[1] for o in ops], np.float64)
        self.p1 = np.array([o[2] for o in ops], np.float64)
        f64 = ctypes.c_int32(0)
        self.W = lib().hs_shape_width(self.op.ctypes.data, self.p0.ctypes.data, len(ops), self.d, ctypes.byref(f64))
        self.out_f64 = bool(f64.value)
        assert self.W == chain.out_width and self.out_f64 == chain.final_f64
        w = chain.norm_width
        self.obs_stats = np.zeros((2 * w + 1, n))
        self.obs_stats[w:2 * w] = 1.0
        self.obs_stats[2 * w] = 1e-4
        self.rew_stats = np.zeros((4, n))
        self.rew_stats[1] = 1.0
        self.rew_stats[2] = 1e-4
        self.ep_return = np.zeros(n, np.float32)
        self.ep_length = np.zeros(n, np.int32)
        k, wf, hf64 = chain.stack if chain.stack is not None else (1, 1, False)
        self.history = np.zeros((k * wf, n), np.float64 if hf64 else np.float32)
        self.head = np.zeros(n, np.int32)
        self.t = np.zeros(n, np.int64)
        self._st = _State(*[a.ctypes.data for a in (self.obs_stats, self.rew_stats, self.ep_return, self.ep_length,
                                                    self.history, self.head, self.t)])

    def _head(self):
        c = self.chain
        return (self.op.ctypes.data, self.p0.ctypes.data, self.p1.ctypes.data, len(self.op), c.raw_reward_type,
                int(c.int_reward_on_fall), self.d, self.n, ctypes.byref(self._st))

    def _shape(self):
        return (self.n,) + self.chain.obs_shape

    def reset(self, obs):
        obs = np.array(obs, np.float32, order="C")
        out = np.zeros(self._shape(), np.float32)
        lib().hs_shape_reset(*self._head(), obs.ctypes.data, out.ctypes.data)
        return out

    def step(self, obs, reward, terminated, truncated, final_obs):
        """-> obs, reward, terminal rows (float64 or float32 as the chain's; written for finishing envs only, zero
        elsewhere), episode r / l (NaN / -1 where no episode ended)."""
        obs = np.array(obs, np.float32, order="C")
        reward = np.array(reward, np.float64, order="C")
        term = np.ascontiguousarray(terminated, np.uint8)
        trunc = np.ascontiguousarray(truncated, np.uint8)
        fin = np.array(final_obs, np.float32, order="C")
        out = np.zeros(self._shape(), np.float32)
        fin32 = np.zeros(self._shape(), np.float32)
        fin64 = np.zeros(self._shape(), np.float64)
        ep_r = np.full(self.n, np.nan, np.float32)
        ep_l = np.full(self.n, -1, np.int32)
        lib().hs_shape_step(*self._head(), obs.ctypes.data, out.ctypes.data, reward.ctypes.data, term.ctypes.data,
                            trunc.ctypes.data, fin.ctypes.data, fin32.ctypes.data, fin64.ctypes.data,
                            ep_r.ctypes.data, ep_l.ctypes.data)
        return out, reward, (fin64 if self.out_f64 else fin32), ep_r, ep_l


def actions(chain, x):
    """The chain's action stages (``Chain.act_stages``) over float32 actions x (N, A)."""
    x = np.ascontiguousarray(x, np.float32)
    b = _Actions()
    b.num = len(chain.act_stages)
    for s, (op, lo, hi, amin, amax) in enumerate(chain.act_stages):
        b.op[s] = op
        for k in range(len(lo)):
            b.lo[s][k], b.hi[s][k], b.amin[s][k], b.amax[s][k] = lo[k], hi[k], amin[k], amax[k]
    out = np.empty_like(x)
    lib().hs_actions(ctypes.byref(b), x.ctypes.data, out.ctypes.data, x.size, x.shape[-1])
    return out
