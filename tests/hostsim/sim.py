"""ctypes wrapper of tests/hostsim/hostsim.cpp: the device source of the step and reset kernels running on the CPU.

Built on demand with g++ into tests/hostsim/_build/ (git-ignored), with the flags that make float32 arithmetic
round like the device build does (`-ffp-contract=off`, matching nvcc's `-fmad=false`).
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_BUILD = os.path.join(_HERE, "_build")
_LIB = os.path.join(_BUILD, "libhostsim.so")
# a second build of the same sources with tiny manifold tables (LunarLander 1 pair, BipedalWalker 2): forces the
# "table full" path that never triggers in normal play, so that its equivalence with the oracle can be tested
_LIB_SMALLCAP = os.path.join(_BUILD, "libhostsim_smallcap.so")
SMALLCAP = {"lunar": 1, "walker": 2}
_SRCS = [os.path.join(_HERE, "hostsim.cpp"), os.path.join(_HERE, "cuda_shim.h")] + [
    os.path.join(_ROOT, "gym_b200", "csrc", f) for f in ("rng.cuh", "envs.cuh", "glibc_trig.cuh", "b2lite.cuh", "b2lite_toi.cuh", "lunar.cuh",
                                                         "walker.cuh", "per_env.cuh", "box2d_consts.h",
                                                         "b2probe.cuh")]

KIND = {"LunarLander": 5, "BipedalWalker": 6, "LunarLanderContinuous": 7, "BipedalWalkerHardcore": 8}
_lib = None
_libs = {}


def lib(smallcap=False):
    global _lib
    if smallcap or _lib is None:
        if smallcap and "small" in _libs:
            return _libs["small"]
        path = _LIB_SMALLCAP if smallcap else _LIB
        extra = [f"-DB2L_LUNAR_MAX_VC={SMALLCAP['lunar']}", f"-DB2L_WALKER_MAX_VC={SMALLCAP['walker']}"] if smallcap else []
        if not os.path.exists(path) or os.path.getmtime(path) < max(os.path.getmtime(s) for s in _SRCS):
            os.makedirs(_BUILD, exist_ok=True)
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared",
                                   "-Wno-unknown-pragmas"] + extra + ["-o", path, os.path.join(_HERE, "hostsim.cpp")])
        L = ctypes.CDLL(path)
        vp, i64, i32, dbl = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_double
        L.hs_create.restype = vp
        L.hs_create.argtypes = [i32, i64, i32, i32, dbl, dbl, dbl, i32, i32]
        L.hs_destroy.argtypes = [vp]
        L.hs_seed_range.argtypes = [vp, vp, i64]
        L.hs_set_wind_idx.argtypes = [vp, vp, vp]
        L.hs_get_wind_idx.argtypes = [vp, vp, vp]
        L.hs_reset.argtypes = [vp, vp]
        L.hs_step.restype = i64
        L.hs_step.argtypes = [vp, vp, vp, vp, vp, vp, vp]
        L.hs_list_totals.argtypes = [vp, vp, vp]
        L.hs_walker_terrain.restype = i32
        L.hs_walker_terrain.argtypes = [vp, i64, vp, vp]
        L.hs_classic_create.restype = vp
        L.hs_classic_create.argtypes = [i32, i64, i32, dbl]
        L.hs_classic_destroy.argtypes = [vp]
        L.hs_classic_seed_range.argtypes = [vp, vp, i64]
        L.hs_classic_reset.argtypes = [vp, vp, vp]
        L.hs_classic_step.restype = i64
        L.hs_classic_step.argtypes = [vp, vp, vp, vp, vp, vp, vp]
        L.hs_classic_get_state.argtypes = [vp, vp, i32]
        L.hs_sincos_small.argtypes = [vp, i64, vp, vp]
        L.hs_overflows.restype = i64
        L.hs_overflows.argtypes = [vp]
        L.hs_glibc_trig.argtypes = [vp, i64, vp, vp]
        L.hs_glibc_sq_mismatches.restype = i64
        L.hs_glibc_sq_mismatches.argtypes = [ctypes.c_uint64, i64, dbl, dbl, ctypes.POINTER(i64)]
        L.hs_glibc_trig_mismatches.restype = i64
        L.hs_glibc_trig_mismatches.argtypes = [ctypes.c_uint64, i64, dbl, dbl]
        fp, f32 = ctypes.POINTER(ctypes.c_float), ctypes.c_float
        L.hs_toi_probe.restype = i32
        L.hs_toi_probe.argtypes = [i32, fp, f32, fp, f32, fp, fp, fp, fp, ctypes.POINTER(i32)]
        L.hs_box2d_probe.argtypes = [i32, vp, i64, vp]
        if smallcap:
            _libs["small"] = L
            return L
        _lib = L
    return _lib


def _seed_words(seed):
    s = int(seed)
    return np.array([(s >> (32 * k)) & 0xFFFFFFFF for k in range(4)], dtype=np.uint32)


class HostSim:
    """One batch of envs stepped by the device source on the CPU; same call shape as oracle.OracleLunar/OracleWalker.

    defer=True runs a step as the device does by default: a step pass, a TOI pass over the envs the step pass parked
    and a reset pass over the envs whose episode ended; defer=False solves both inline in the step pass
    (B200GYM_BOX2D_TOI_DEFER=0 / B200GYM_BOX2D_DEFER=0).  ranges > 1 splits every step into that many launch ranges,
    the last one ragged, as the host path splits a batch into chunks."""

    def __init__(self, name, num_envs, max_episode_steps, gravity=-10.0, enable_wind=False, wind_power=15.0,
                 turbulence_power=1.5, wind_idx=None, torque_idx=None, smallcap=False, defer=True, ranges=1):
        self._L = lib(smallcap)
        self.kind = KIND[name]
        self.n = int(num_envs)
        self.lunar = self.kind in (5, 7)
        self.obs_dim = 8 if self.lunar else 24
        self._h = self._L.hs_create(self.kind, self.n, int(max_episode_steps or 0), int(bool(enable_wind)), float(gravity),
                                  float(wind_power), float(turbulence_power), int(bool(defer)), int(ranges))
        assert self._h
        if wind_idx is not None:
            wi = np.ascontiguousarray(np.broadcast_to(wind_idx, (self.n,)), dtype=np.int32)
            ti = np.ascontiguousarray(np.broadcast_to(torque_idx, (self.n,)), dtype=np.int32)
            self._L.hs_set_wind_idx(self._h, wi.ctypes.data, ti.ctypes.data)

    def list_totals(self):
        """(envs taken by the TOI pass, envs taken by the reset pass) since construction."""
        t = np.zeros(2, dtype=np.int64)
        self._L.hs_list_totals(self._h, t[0:].ctypes.data, t[1:].ctypes.data)
        return int(t[0]), int(t[1])

    def overflows(self):
        """Number of envs whose manifold table ever overflowed."""
        return int(self._L.hs_overflows(self._h))

    def close(self):
        if getattr(self, "_h", None):
            self._L.hs_destroy(self._h)
            self._h = None

    __del__ = close

    def reset(self, seed=None):
        if seed is not None:
            self._L.hs_seed_range(self._h, _seed_words(seed).ctypes.data, 0)
        obs = np.zeros((self.n, self.obs_dim), dtype=np.float32)
        self._L.hs_reset(self._h, obs.ctypes.data)
        return obs

    def step(self, actions):
        if self.kind == 5:
            a = np.ascontiguousarray(actions, dtype=np.int64).reshape(self.n)
        else:
            a = np.ascontiguousarray(actions, dtype=np.float32).reshape(self.n, 2 if self.kind == 7 else 4)
        obs = np.zeros((self.n, self.obs_dim), dtype=np.float32)
        fo = np.zeros((self.n, self.obs_dim), dtype=np.float32)
        rew = np.zeros(self.n, dtype=np.float64)
        te = np.zeros(self.n, dtype=np.uint8)
        tr = np.zeros(self.n, dtype=np.uint8)
        bad = self._L.hs_step(self._h, a.ctypes.data, obs.ctypes.data, rew.ctypes.data, te.ctypes.data, tr.ctypes.data,
                            fo.ctypes.data)
        assert bad == 0
        return obs, rew, te.astype(bool), tr.astype(bool), fo

    def wind_idx(self):
        wi = np.zeros(self.n, dtype=np.int32)
        ti = np.zeros(self.n, dtype=np.int32)
        self._L.hs_get_wind_idx(self._h, wi.ctypes.data, ti.ctypes.data)
        return wi, ti

    def terrain(self, i=0):
        t = np.zeros(200, dtype=np.float32)
        boxes = np.zeros((40, 4), dtype=np.float32)
        k = self._L.hs_walker_terrain(self._h, int(i), t.ctypes.data, boxes.ctypes.data)
        return t, boxes[:k].copy()


class HostSimClassic:
    """The per-env drivers of reset_kernel and kernel A over Env<KIND> of gym_b200/csrc/envs.cuh on the CPU (autoreset
    mode); call shape of oracle.OracleVec."""

    # kind -> (obs_dim, act_dim, state_dim); enum b200gym_kind
    DIMS = {0: (4, 0, 4), 1: (2, 0, 2), 2: (2, 1, 2), 3: (3, 1, 2), 4: (6, 0, 4)}

    def __init__(self, kind, num_envs, max_episode_steps, param0=0.0):
        self.kind, self.n = int(kind), int(num_envs)
        self.obs_dim, self.act_dim, self.state_dim = self.DIMS[self.kind]
        self._h = lib().hs_classic_create(self.kind, self.n, int(max_episode_steps or 0), float(param0))
        assert self._h

    def close(self):
        if getattr(self, "_h", None):
            lib().hs_classic_destroy(self._h)
            self._h = None

    __del__ = close

    def reset(self, seed=None, bounds=None):
        if seed is not None:
            lib().hs_classic_seed_range(self._h, _seed_words(seed).ctypes.data, 0)
        obs = np.zeros((self.n, self.obs_dim), dtype=np.float32)
        b = None if bounds is None else np.asarray(bounds, dtype=np.float64)
        lib().hs_classic_reset(self._h, None if b is None else b.ctypes.data, obs.ctypes.data)
        return obs

    def step(self, actions):
        if self.act_dim == 0:
            a = np.ascontiguousarray(actions, dtype=np.int64).reshape(self.n)
        else:
            a = np.ascontiguousarray(actions, dtype=np.float32).reshape(self.n)
        obs = np.zeros((self.n, self.obs_dim), dtype=np.float32)
        fo = np.zeros((self.n, self.obs_dim), dtype=np.float32)
        rew = np.zeros(self.n, dtype=np.float64)
        te = np.zeros(self.n, dtype=np.uint8)
        tr = np.zeros(self.n, dtype=np.uint8)
        bad = lib().hs_classic_step(self._h, a.ctypes.data, obs.ctypes.data, rew.ctypes.data, te.ctypes.data,
                                    tr.ctypes.data, fo.ctypes.data)
        assert bad == 0
        return obs, rew, te.astype(bool), tr.astype(bool), fo

    def state(self):
        s = np.zeros((self.n, self.state_dim), dtype=np.float64)
        lib().hs_classic_get_state(self._h, s.ctypes.data, self.state_dim)
        return s


def glibc_trig(x):
    """csrc/glibc_trig.cuh: gt::sin / gt::cos on an array of float64 arguments."""
    x = np.ascontiguousarray(x, dtype=np.float64)
    sn, cs = np.empty_like(x), np.empty_like(x)
    lib().hs_glibc_trig(x.ctypes.data, x.size, sn.ctypes.data, cs.ctypes.data)
    return sn, cs


def glibc_trig_mismatches(seed, n, lo, hi):
    """How many of n pseudo-random arguments in [lo, hi) give a sin or cos that differs bitwise from libm's."""
    return int(lib().hs_glibc_trig_mismatches(int(seed), int(n), float(lo), float(hi)))


def glibc_sq_mismatches(seed, n, lo, hi):
    """(#arguments where gt::sq(x) != libm pow(x, 2.0), #arguments where pow(x, 2.0) != x * x) of n in [lo, hi)."""
    neq = ctypes.c_int64(0)
    bad = lib().hs_glibc_sq_mismatches(int(seed), int(n), float(lo), float(hi), ctypes.byref(neq))
    return int(bad), int(neq.value)


def sincos_small(x):
    """csrc/envs.cuh: sincos_small on an array of float64 angles."""
    x = np.ascontiguousarray(x, dtype=np.float64)
    sn, cs = np.zeros_like(x), np.zeros_like(x)
    lib().hs_sincos_small(x.ctypes.data, x.size, sn.ctypes.data, cs.ctypes.data)
    return sn, cs


def shape_verts(shape):
    """Vertices (n, 2) float32 and local centre (2,) of task polygon `shape` as the device constants hold them."""
    fp = ctypes.POINTER(ctypes.c_float)
    out = np.zeros(16, dtype=np.float32)
    lc = np.zeros(2, dtype=np.float32)
    f = lib().hs_shape_verts
    f.restype = ctypes.c_int
    f.argtypes = [ctypes.c_int, fp, fp]
    n = f(int(shape), out.ctypes.data_as(fp), lc.ctypes.data_as(fp))
    return out[:2 * n].reshape(n, 2).copy(), lc


def toi_probe(shape, c0, a0, c1, a1, edge=None, box=None):
    """The device source's b2TimeOfImpact + its conservative shortcut for one sweep of a task polygon (0 lander, 1 its
    leg, 2 walker hull, 3 / 4 walker upper / lower leg) against a static edge ((x1, y1), (x2, y2)) or an axis-aligned
    box (x0, ylo, x1, yhi) -> (state, t, cannot_touch); state 3 = touching."""
    fp = ctypes.POINTER(ctypes.c_float)
    arr = lambda x: np.ascontiguousarray(x, dtype=np.float32).ravel()
    C0, C1 = arr(c0), arr(c1)
    V1, V2 = (arr(edge[0]), arr(edge[1])) if edge is not None else (arr([0, 0]), arr([0, 0]))
    B = arr(box) if box is not None else None
    t = ctypes.c_float(0.0)
    ct = ctypes.c_int(0)
    p = lambda a: a.ctypes.data_as(fp)
    st = lib().hs_toi_probe(int(shape), p(C0), float(a0), p(C1), float(a1), p(V1), p(V2), p(B) if B is not None else None,
                            ctypes.byref(t), ctypes.byref(ct))
    return int(st), float(t.value), bool(ct.value)



def box2d_probe(op, records):
    """csrc/b2probe.cuh on the CPU: op on float32 records (n, 16) -> (n, 16), what b200gym_selftest_box2d computes."""
    rec = np.ascontiguousarray(records, dtype=np.float32).reshape(-1, 16)
    out = np.zeros_like(rec)
    lib().hs_box2d_probe(int(op), rec.ctypes.data, rec.shape[0], out.ctypes.data)
    return out
