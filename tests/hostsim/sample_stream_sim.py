"""ctypes wrapper of tests/hostsim/sample_stream.cpp: the device source of space_sample_stream_kernel on the CPU.

Built on demand with g++ into tests/hostsim/_build/ (git-ignored), with the flags of sample_sim.py.
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_BUILD = os.path.join(_HERE, "_build")
_LIB = os.path.join(_BUILD, "libsample_stream.so")
_SRCS = [os.path.join(_HERE, "sample_stream.cpp"), os.path.join(_HERE, "cuda_shim.h")] + [
    os.path.join(_ROOT, "gym_b200", "csrc", f) for f in ("rng.cuh", "space_sample.cuh")]
_lib = None

RECORD_WORDS = 5


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB) or os.path.getmtime(_LIB) < max(os.path.getmtime(s) for s in _SRCS):
            os.makedirs(_BUILD, exist_ok=True)
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared",
                                   "-Wno-unknown-pragmas", "-o", _LIB, os.path.join(_HERE, "sample_stream.cpp")])
        L = ctypes.CDLL(_LIB)
        vp, i64, i32 = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int
        L.hs_sample_space_stream.argtypes = [vp, vp, i64, i32, i64, vp, vp, vp]
        _lib = L
    return _lib


def words(state, inc):
    m = (1 << 64) - 1
    return np.array([state >> 64, state & m, inc >> 64, inc & m], dtype=np.uint64)


def new_record():
    return np.zeros(RECORD_WORDS, dtype=np.uint64)


def sample_space_stream(record, rows, cols=1, n_choices=0, low=None, high=None, override=None):
    """One b200gym_sample_space_stream call on `record` (uint64 [RECORD_WORDS], updated in place); `override` is
    (state, inc) or None."""
    if n_choices:
        out = np.full(rows, -1, dtype=np.int64)
        lo = hi = None
    else:
        out = np.full((rows, cols), np.nan, dtype=np.float32)
        lo = np.ascontiguousarray(low, dtype=np.float64)
        hi = np.ascontiguousarray(high, dtype=np.float64)
    ov = None if override is None else words(*override)
    lib().hs_sample_space_stream(record.ctypes.data, None if ov is None else ov.ctypes.data, int(rows), int(cols),
                                 int(n_choices), None if lo is None else lo.ctypes.data,
                                 None if hi is None else hi.ctypes.data, out.ctypes.data)
    return out
