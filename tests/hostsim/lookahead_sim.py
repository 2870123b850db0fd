"""ctypes wrapper of tests/hostsim/lookahead.cpp: kernel B's CartPole lookahead and the step it predicts, on the CPU.

Built on demand with g++ into tests/hostsim/_build/ (git-ignored), with the flags of sim.py.
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_BUILD = os.path.join(_HERE, "_build")
_LIB = os.path.join(_BUILD, "liblookahead.so")
_SRCS = [os.path.join(_HERE, "lookahead.cpp"), os.path.join(_HERE, "cuda_shim.h"),
         os.path.join(_ROOT, "include", "b200gym.h")] + [
    os.path.join(_ROOT, "gym_b200", "csrc", f) for f in ("rng.cuh", "envs.cuh", "glibc_trig.cuh", "b2lite.cuh",
                                                         "b2lite_toi.cuh", "lunar.cuh", "walker.cuh", "per_env.cuh",
                                                         "box2d_consts.h")]
_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB) or os.path.getmtime(_LIB) < max(os.path.getmtime(s) for s in _SRCS):
            os.makedirs(_BUILD, exist_ok=True)
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared",
                                   "-Wno-unknown-pragmas", "-o", _LIB, os.path.join(_HERE, "lookahead.cpp")])
        L = ctypes.CDLL(_LIB)
        vp, i64, i32 = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int
        L.hs_cartpole_lookahead.argtypes = [vp, vp, vp, i64, i32, i32, vp, vp, vp, vp]
        _lib = L
    return _lib


def cartpole_lookahead(state, elapsed, actions, max_steps, autoreset=True):
    """Kernel B's lookahead for CartPole states [n][4] and the step it predicts.  Returns (will_terminate, step's
    terminated, will_reset, advance_env's return) as bool arrays."""
    state = np.ascontiguousarray(state, dtype=np.float64)
    n = state.shape[0]
    elapsed = np.ascontiguousarray(np.broadcast_to(elapsed, (n,)), dtype=np.int32)
    actions = np.ascontiguousarray(np.broadcast_to(actions, (n,)), dtype=np.int64)
    out = [np.zeros(n, dtype=np.uint8) for _ in range(4)]
    lib().hs_cartpole_lookahead(state.ctypes.data, elapsed.ctypes.data, actions.ctypes.data, n, int(max_steps),
                                int(bool(autoreset)), *(o.ctypes.data for o in out))
    return tuple(o.astype(bool) for o in out)
