"""ctypes wrapper of tests/hostsim/sample_space.cpp: the device source of space_sample_kernel running on the CPU.

Built on demand with g++ into tests/hostsim/_build/ (git-ignored), with the flags sim.py uses for the step kernels'
host build (`-ffp-contract=off`, matching nvcc's `-fmad=false`: uniform()'s multiply and add round separately).
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_BUILD = os.path.join(_HERE, "_build")
_LIB = os.path.join(_BUILD, "libsample_space.so")
_SRCS = [os.path.join(_HERE, "sample_space.cpp"), os.path.join(_HERE, "cuda_shim.h")] + [
    os.path.join(_ROOT, "gym_b200", "csrc", f) for f in ("rng.cuh", "space_sample.cuh")]
_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB) or os.path.getmtime(_LIB) < max(os.path.getmtime(s) for s in _SRCS):
            os.makedirs(_BUILD, exist_ok=True)
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared",
                                   "-Wno-unknown-pragmas", "-o", _LIB, os.path.join(_HERE, "sample_space.cpp")])
        L = ctypes.CDLL(_LIB)
        vp, i64, i32 = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int
        L.hs_sample_space.argtypes = [vp, i64, i32, i64, vp, vp, vp, i64]
        L.hs_pcg64_jump.argtypes = [vp, ctypes.c_uint64, ctypes.c_uint64, i32]
        _lib = L
    return _lib


def _pcg64_words(state, inc):
    m = (1 << 64) - 1
    return np.array([state >> 64, state & m, inc >> 64, inc & m], dtype=np.uint64)


def pcg64_jump(state, inc, delta, table=False):
    """csrc/rng.cuh: the PCG64 state `delta` draws after `state`, by pcg64_jump (square-and-multiply, delta < 2**128)
    or by pcg64_jump_table (the sampling kernel's table walk, delta < 2**64)."""
    w = _pcg64_words(state, inc)
    lib().hs_pcg64_jump(w.ctypes.data, int(delta) >> 64, int(delta) & ((1 << 64) - 1), int(bool(table)))
    return (int(w[0]) << 64) | int(w[1])


def sample_space(state, inc, rows, cols=1, n_choices=0, low=None, high=None, blocks=0):
    """csrc/space_sample.cuh: what space_sample_kernel writes for a batched MultiDiscrete (n_choices = n, int64 (rows,))
    or bounded float32 Box (float32 (rows, cols), per-column float64 bounds), over the grid b200gym_sample_space
    launches (blocks = 0) or over `blocks` CTAs."""
    w = _pcg64_words(state, inc)
    if n_choices:
        out = np.full(rows, -1, dtype=np.int64)
        lo = hi = None
    else:
        out = np.full((rows, cols), np.nan, dtype=np.float32)
        lo = np.ascontiguousarray(low, dtype=np.float64)
        hi = np.ascontiguousarray(high, dtype=np.float64)
    lib().hs_sample_space(w.ctypes.data, int(rows), int(cols), int(n_choices), None if lo is None else lo.ctypes.data,
                          None if hi is None else hi.ctypes.data, out.ctypes.data, int(blocks))
    return out
