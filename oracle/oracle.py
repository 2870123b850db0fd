"""ctypes front-end of the CPU ORACLE (test infrastructure, NOT product code).

Wraps ``oracle/libgymoracle.so`` (built from ``oracle/gym_oracle.c``), the plain-C
restatement of gym 0.26.2's classic-control ``step()/reset()`` path.  Only
``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` /
``--impl reference`` legs may import this module; nothing under ``gym_b200/``
does.  Parity status: pinned (see ``oracle/gen_golden.py`` and ``tests/golden``).
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libgymoracle.so")

KINDS = {
    "CartPole": 0,
    "MountainCar": 1,
    "MountainCarContinuous": 2,
    "Pendulum": 3,
    "Acrobot": 4,
}

# gym/envs/__init__.py:11-60 registry constants restated: id -> (kind, max_episode_steps)
ENV_IDS = {
    "CartPole-v0": ("CartPole", 200),
    "CartPole-v1": ("CartPole", 500),
    "MountainCar-v0": ("MountainCar", 200),
    "MountainCarContinuous-v0": ("MountainCarContinuous", 999),
    "Pendulum-v1": ("Pendulum", 200),
    "Acrobot-v1": ("Acrobot", 500),
}


def build(force=False):
    """Compile the oracle with the recipe in oracle/Makefile (gcc, no FMA contraction)."""
    srcs = [os.path.join(_HERE, f) for f in ("gym_oracle.c", "lunar_oracle.c", "walker_oracle.c", "gym_oracle.h", "lunar_oracle.h",
                                           "walker_oracle.h", "b2lite.h", "np_rng.h")]
    if (force or not os.path.exists(_LIB_PATH)
            or os.path.getmtime(_LIB_PATH) < max(os.path.getmtime(s) for s in srcs)):
        subprocess.check_call(["make", "-s", "-C", _HERE, "libgymoracle.so"])
    return _LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = ctypes.CDLL(_LIB_PATH)
        vp, i64, i32, dbl = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_double
        L.orc_vec_create.restype = vp
        L.orc_vec_create.argtypes = [i32, i64, i32, dbl]
        L.orc_vec_destroy.argtypes = [vp]
        L.orc_seed_sequence.argtypes = [vp, vp]
        L.orc_vec_seed_env.argtypes = [vp, i64, vp]
        L.orc_vec_seed_range.argtypes = [vp, vp, i64]
        L.orc_vec_get_rng.argtypes = [vp, vp]
        L.orc_vec_set_rng.argtypes = [vp, vp]
        L.orc_vec_next_double.restype = dbl
        L.orc_vec_next_double.argtypes = [vp, i64]
        L.orc_vec_reset.argtypes = [vp, vp, vp, vp]
        L.orc_vec_step.restype = i64
        L.orc_vec_step.argtypes = [vp, vp, vp, vp, vp, vp, vp, i32]
        L.orc_vec_get_state.argtypes = [vp, vp, vp]
        L.orc_vec_set_state.argtypes = [vp, vp, vp]
        L.orc_lunar_create.restype = vp
        L.orc_lunar_create.argtypes = [i64, i32]
        L.orc_lunar_create_ex.restype = vp
        L.orc_lunar_create_ex.argtypes = [i64, i32, i32, i32, dbl, dbl, dbl]
        L.orc_lunar_set_wind_idx.argtypes = [vp, vp, vp]
        L.orc_lunar_get_wind_idx.argtypes = [vp, vp, vp]
        L.orc_lunar_step_cont.argtypes = [vp, vp, vp, vp, vp, vp, vp]
        L.orc_lunar_step_mt.restype = i64
        L.orc_lunar_step_mt.argtypes = [vp, vp, vp, vp, vp, vp, vp, i32]
        L.orc_lunar_step_cont_mt.argtypes = [vp, vp, vp, vp, vp, vp, vp, i32]
        L.orc_walker_step_mt.argtypes = [vp, vp, vp, vp, vp, vp, vp, i32]
        L.orc_lunar_engines.argtypes = [i32, i32, vp, dbl, dbl, dbl, dbl, dbl, vp, vp, vp]
        L.orc_lunar_destroy.argtypes = [vp]
        L.orc_lunar_seed_range.argtypes = [vp, vp, i64]
        L.orc_lunar_reset.argtypes = [vp, vp]
        L.orc_lunar_step.restype = i64
        L.orc_lunar_step.argtypes = [vp, vp, vp, vp, vp, vp, vp]
        L.orc_lunar_get_bodies.argtypes = [vp, i64, vp, vp]
        L.orc_lunar_get_terrain.argtypes = [vp, i64, vp]
        L.orc_walker_create.restype = vp
        L.orc_walker_create.argtypes = [i64, i32]
        L.orc_walker_create_ex.restype = vp
        L.orc_walker_create_ex.argtypes = [i64, i32, i32]
        L.orc_walker_action_flow.argtypes = [dbl, vp, vp, vp, vp]
        L.orc_walker_get_polys.restype = i32
        L.orc_walker_get_polys.argtypes = [vp, i64, vp]
        L.orc_walker_destroy.argtypes = [vp]
        L.orc_walker_seed_range.argtypes = [vp, vp, i64]
        L.orc_walker_reset.argtypes = [vp, vp]
        L.orc_walker_step.restype = None
        L.orc_walker_step.argtypes = [vp, vp, vp, vp, vp, vp, vp]
        L.orc_walker_get_terrain.argtypes = [vp, i64, vp]
        L.orc_walker_get_bodies.argtypes = [vp, i64, vp, vp]
        L.orc_rng_sequence.argtypes = [vp, vp, i64, vp]
        for f in ("orc_obs_dim", "orc_act_dim", "orc_state_dim", "orc_num_actions"):
            getattr(L, f).argtypes = [i32]
        _lib = L
    return _lib


def seed_words(seed):
    """Non-negative int (< 2**128) -> four little-endian uint32 entropy words."""
    seed = int(seed)
    if seed < 0 or seed >= 1 << 128:
        raise ValueError("oracle supports 0 <= seed < 2**128")
    return np.array([(seed >> (32 * k)) & 0xFFFFFFFF for k in range(4)], dtype=np.uint32)


def seed_sequence(seed):
    """SeedSequence(seed).generate_state(4, np.uint64) through the C restatement."""
    out = np.zeros(4, dtype=np.uint64)
    ent = seed_words(seed)
    lib().orc_seed_sequence(ent.ctypes.data, out.ctypes.data)
    return out


def _ptr(a):
    return None if a is None else a.ctypes.data


class OracleVec:
    """SyncVectorEnv([make(id)] * n) restated in C: TimeLimit + same-step autoreset fused."""

    def __init__(self, env_id, num_envs, max_episode_steps=None, param0=None):
        if env_id in ENV_IDS:
            kind_name, default_max = ENV_IDS[env_id]
        else:
            kind_name, default_max = env_id, 0
        self.kind = KINDS[kind_name]
        self.kind_name = kind_name
        self.n = int(num_envs)
        self.max_episode_steps = default_max if max_episode_steps is None else int(max_episode_steps)
        if param0 is None:
            param0 = 10.0 if kind_name == "Pendulum" else 0.0
        L = lib()
        self.obs_dim = L.orc_obs_dim(self.kind)
        self.act_dim = L.orc_act_dim(self.kind)
        self.state_dim = L.orc_state_dim(self.kind)
        self.num_actions = L.orc_num_actions(self.kind)
        self._h = L.orc_vec_create(self.kind, self.n, self.max_episode_steps, float(param0))
        if not self._h:
            raise ValueError("orc_vec_create failed")

    def close(self):
        if getattr(self, "_h", None):
            lib().orc_vec_destroy(self._h)
            self._h = None

    __del__ = close

    # -- RNG ------------------------------------------------------------
    def seed(self, seed, first=0):
        """int -> env i gets seed+first+i; sequence -> per-env seeds (None keeps the stream)."""
        L = lib()
        if isinstance(seed, (int, np.integer)):
            L.orc_vec_seed_range(self._h, seed_words(seed).ctypes.data, int(first))
        else:
            assert len(seed) == self.n
            for i, s in enumerate(seed):
                if s is not None:
                    L.orc_vec_seed_env(self._h, i, seed_words(s).ctypes.data)

    def get_rng(self):
        out = np.zeros((self.n, 4), dtype=np.uint64)
        lib().orc_vec_get_rng(self._h, out.ctypes.data)
        return out

    def set_rng(self, rng):
        rng = np.ascontiguousarray(rng, dtype=np.uint64).reshape(self.n, 4)
        lib().orc_vec_set_rng(self._h, rng.ctypes.data)

    def next_double(self, i=0):
        return lib().orc_vec_next_double(self._h, int(i))

    # -- env API ----------------------------------------------------------
    def reset(self, seed=None, bounds=None, mask=None):
        if seed is not None:
            self.seed(seed)
        obs = np.zeros((self.n, self.obs_dim), dtype=np.float32)
        b = None if bounds is None else np.asarray(bounds, dtype=np.float64)
        m = None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8)
        lib().orc_vec_reset(self._h, _ptr(m), _ptr(b), obs.ctypes.data)
        return obs

    def step(self, actions, nthreads=1):
        if self.act_dim == 0:
            a = np.ascontiguousarray(actions, dtype=np.int64).reshape(self.n)
        else:
            a = np.ascontiguousarray(actions, dtype=np.float32).reshape(self.n, self.act_dim)
        obs = np.zeros((self.n, self.obs_dim), dtype=np.float32)
        final_obs = np.zeros((self.n, self.obs_dim), dtype=np.float32)
        reward = np.zeros(self.n, dtype=np.float64)
        term = np.zeros(self.n, dtype=np.uint8)
        trunc = np.zeros(self.n, dtype=np.uint8)
        bad = lib().orc_vec_step(self._h, a.ctypes.data, obs.ctypes.data, reward.ctypes.data,
                                 term.ctypes.data, trunc.ctypes.data, final_obs.ctypes.data,
                                 int(nthreads))
        if bad:
            raise AssertionError(f"{bad} invalid discrete action(s)")
        return obs, reward, term.astype(bool), trunc.astype(bool), final_obs

    def get_state(self):
        s = np.zeros((self.n, self.state_dim), dtype=np.float64)
        e = np.zeros(self.n, dtype=np.int32)
        lib().orc_vec_get_state(self._h, s.ctypes.data, e.ctypes.data)
        return s, e

    def set_state(self, state=None, elapsed=None):
        s = None if state is None else np.ascontiguousarray(state, dtype=np.float64)
        e = None if elapsed is None else np.ascontiguousarray(elapsed, dtype=np.int32)
        lib().orc_vec_set_state(self._h, _ptr(s), _ptr(e))


def set_box2d_max_contacts(lunar=8, walker=10):
    """Manifold-table capacity of the two Box2D scenes (defaults = the CUDA scenes' kMaxVC); process-wide.
    Tests shrink it (together with a small-table build of the device source) to exercise the overflow rule."""
    L = lib()
    L.orc_lunar_set_max_contacts(int(lunar))
    L.orc_walker_set_max_contacts(int(walker))


def set_box2d_toi(on=True):
    """Continuous collision (b2World::SolveTOI, oracle/b2lite_toi.h) of the two Box2D scenes; process-wide, on by
    default like Box2D's m_continuousPhysics.  Tests switch it off to show what it prevents."""
    L = lib()
    L.orc_lunar_set_toi(int(bool(on)))
    L.orc_walker_set_toi(int(bool(on)))


def toi_probe(poly, c0, a0, c1, a1, v1, v2):
    """b2TimeOfImpact of a convex polygon (local vertices) sweeping from (c0, a0) to (c1, a1) against the static edge
    v1-v2 -> (state, t); state 3 = touching, 4 = separated, 2 = overlapped, 1 = failed."""
    f = lib().orc_b2l_toi_probe
    f.restype = ctypes.c_int
    fp = ctypes.POINTER(ctypes.c_float)
    f.argtypes = [fp, ctypes.c_int, fp, ctypes.c_float, fp, ctypes.c_float, fp, fp, fp]
    arr = lambda x: np.ascontiguousarray(x, dtype=np.float32).ravel()
    P, C0, C1, V1, V2 = arr(poly), arr(c0), arr(c1), arr(v1), arr(v2)
    t = ctypes.c_float(0.0)
    as_p = lambda a: a.ctypes.data_as(fp)
    st = f(as_p(P), len(P) // 2, as_p(C0), float(a0), as_p(C1), float(a1), as_p(V1), as_p(V2), ctypes.byref(t))
    return int(st), float(t.value)


def distance_probe(poly, c, a, v1, v2):
    """b2Distance (GJK) between a convex polygon (local vertices) placed at (c, a) and the static edge v1-v2, without
    radii -> (distance, number of simplex vertices at termination)."""
    f = lib().orc_b2l_distance_probe
    f.restype = ctypes.c_float
    fp = ctypes.POINTER(ctypes.c_float)
    f.argtypes = [fp, ctypes.c_int, fp, ctypes.c_float, fp, fp, ctypes.POINTER(ctypes.c_int)]
    arr = lambda x: np.ascontiguousarray(x, dtype=np.float32).ravel()
    P, C, V1, V2 = arr(poly), arr(c), arr(v1), arr(v2)
    cnt = ctypes.c_int(0)
    p_ = lambda z: z.ctypes.data_as(fp)
    d = f(p_(P), len(P) // 2, p_(C), float(a), p_(V1), p_(V2), ctypes.byref(cnt))
    return float(d), int(cnt.value)


class OracleLunar:
    """SyncVectorEnv([make("LunarLander-v2")] * n) restated in C (oracle/lunar_oracle.c).

    PARITY UNPINNED: the rigid-body arithmetic restates Box2D 2.3 from its published design;
    box2d-py is not installable here, so it cannot be checked against the real library."""

    obs_dim, act_dim, num_actions = 8, 0, 4

    def __init__(self, num_envs, max_episode_steps=1000, continuous=False, gravity=-10.0, enable_wind=False,
                 wind_power=15.0, turbulence_power=1.5, wind_idx=None, torque_idx=None):
        self.n = int(num_envs)
        self.continuous = bool(continuous)
        self._h = lib().orc_lunar_create_ex(self.n, int(max_episode_steps or 0), int(self.continuous), int(bool(enable_wind)),
                                            float(gravity), float(wind_power), float(turbulence_power))
        if wind_idx is not None:
            # the per-object np.random.randint(-9999, 9999) draws of LunarLander.__init__ (lunar_lander.py:234-235)
            wi = np.ascontiguousarray(np.broadcast_to(wind_idx, (self.n,)), dtype=np.int32)
            ti = np.ascontiguousarray(np.broadcast_to(torque_idx, (self.n,)), dtype=np.int32)
            lib().orc_lunar_set_wind_idx(self._h, wi.ctypes.data, ti.ctypes.data)

    def wind_idx(self):
        wi = np.zeros(self.n, dtype=np.int32)
        ti = np.zeros(self.n, dtype=np.int32)
        lib().orc_lunar_get_wind_idx(self._h, wi.ctypes.data, ti.ctypes.data)
        return wi, ti

    def overflows(self):
        """Number of envs in which a touching pair was ever dropped because the manifold table was full."""
        f = lib().orc_lunar_overflows
        f.restype, f.argtypes = ctypes.c_int64, [ctypes.c_void_p]
        return int(f(self._h))

    def toi_stats(self):
        """(b2TimeOfImpact evaluations, TOI sub-steps) summed over all envs since creation."""
        out = np.zeros(3, dtype=np.int64)
        lib().orc_lunar_toi_stats(ctypes.c_void_p(self._h), ctypes.c_void_p(out.ctypes.data))
        self.toi_events_max = int(out[2])     # most TOI sub-steps any env ran in one world step
        return int(out[0]), int(out[1])

    def set_body_velocity(self, i, body, vx, vy, w=0.0):
        """test hook: overwrite the velocity of one body (0 lander, 1 / 2 legs) of env i"""
        f = lib().orc_lunar_set_body_velocity
        f.restype, f.argtypes = None, [ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_float, ctypes.c_float, ctypes.c_float]
        f(self._h, int(i), int(body), float(vx), float(vy), float(w))

    def close(self):
        if getattr(self, "_h", None):
            lib().orc_lunar_destroy(self._h)
            self._h = None

    __del__ = close

    def reset(self, seed=None, first=0):
        """env k is seeded seed + first + k: the oracle stands in for envs [first, first + n) of a larger batch"""
        if seed is not None:
            lib().orc_lunar_seed_range(self._h, seed_words(seed).ctypes.data, int(first))
        obs = np.zeros((self.n, 8), dtype=np.float32)
        lib().orc_lunar_reset(self._h, obs.ctypes.data)
        return obs

    def step(self, actions, nthreads=1):
        obs = np.zeros((self.n, 8), dtype=np.float32)
        fo = np.zeros((self.n, 8), dtype=np.float32)
        rew = np.zeros(self.n, dtype=np.float64)
        te = np.zeros(self.n, dtype=np.uint8)
        tr = np.zeros(self.n, dtype=np.uint8)
        if self.continuous:
            a = np.ascontiguousarray(actions, dtype=np.float32).reshape(self.n, 2)
            lib().orc_lunar_step_cont_mt(self._h, a.ctypes.data, obs.ctypes.data, rew.ctypes.data, te.ctypes.data,
                                         tr.ctypes.data, fo.ctypes.data, int(nthreads))
            return obs, rew, te.astype(bool), tr.astype(bool), fo
        a = np.ascontiguousarray(actions, dtype=np.int64).reshape(self.n)
        bad = lib().orc_lunar_step_mt(self._h, a.ctypes.data, obs.ctypes.data, rew.ctypes.data, te.ctypes.data,
                                      tr.ctypes.data, fo.ctypes.data, int(nthreads))
        if bad:
            raise AssertionError(f"{bad} invalid discrete action(s)")
        return obs, rew, te.astype(bool), tr.astype(bool), fo

    def terrain(self, i=0):
        """the 11 terrain vertex heights (smooth_y) of env i"""
        y = np.zeros(11, dtype=np.float32)
        lib().orc_lunar_get_terrain(self._h, int(i), y.ctypes.data)
        return y

    def bodies(self, i=0):
        out = np.zeros(18, dtype=np.float32)
        flags = np.zeros(6, dtype=np.int32)
        lib().orc_lunar_get_bodies(self._h, int(i), out.ctypes.data, flags.ctypes.data)
        return out.reshape(3, 6), flags


class OracleWalker:
    """SyncVectorEnv([make("BipedalWalker-v3")] * n) restated in C (oracle/walker_oracle.c).
    PARITY UNPINNED for the Box2D arithmetic (see oracle/b2lite.h)."""

    obs_dim, act_dim, num_actions = 24, 4, 0

    def __init__(self, num_envs, max_episode_steps=1600, hardcore=False):
        self.n = int(num_envs)
        self._h = lib().orc_walker_create_ex(self.n, int(max_episode_steps or 0), int(bool(hardcore)))

    def overflows(self):
        """Number of envs in which a touching pair was ever dropped because the manifold table was full."""
        f = lib().orc_walker_overflows
        f.restype, f.argtypes = ctypes.c_int64, [ctypes.c_void_p]
        return int(f(self._h))

    def toi_stats(self):
        """(b2TimeOfImpact evaluations, TOI sub-steps) summed over all envs since creation."""
        out = np.zeros(3, dtype=np.int64)
        lib().orc_walker_toi_stats(ctypes.c_void_p(self._h), ctypes.c_void_p(out.ctypes.data))
        self.toi_events_max = int(out[2])     # most TOI sub-steps any env ran in one world step
        return int(out[0]), int(out[1])

    def close(self):
        if getattr(self, "_h", None):
            lib().orc_walker_destroy(self._h)
            self._h = None

    __del__ = close

    def reset(self, seed=None, first=0):
        """env k is seeded seed + first + k (see OracleLunar.reset)"""
        if seed is not None:
            lib().orc_walker_seed_range(self._h, seed_words(seed).ctypes.data, int(first))
        obs = np.zeros((self.n, 24), dtype=np.float32)
        lib().orc_walker_reset(self._h, obs.ctypes.data)
        return obs

    def step(self, actions, nthreads=1):
        a = np.ascontiguousarray(actions, dtype=np.float32).reshape(self.n, 4)
        obs = np.zeros((self.n, 24), dtype=np.float32)
        fo = np.zeros((self.n, 24), dtype=np.float32)
        rew = np.zeros(self.n, dtype=np.float64)
        te = np.zeros(self.n, dtype=np.uint8)
        tr = np.zeros(self.n, dtype=np.uint8)
        lib().orc_walker_step_mt(self._h, a.ctypes.data, obs.ctypes.data, rew.ctypes.data, te.ctypes.data,
                                 tr.ctypes.data, fo.ctypes.data, int(nthreads))
        return obs, rew, te.astype(bool), tr.astype(bool), fo

    def terrain(self, i=0):
        y = np.zeros(200, dtype=np.float32)
        lib().orc_walker_get_terrain(self._h, int(i), y.ctypes.data)
        return y

    def polys(self, i=0):
        """hardcore obstacles of env i as rows {x0, ylo, x1, yhi} (float32), in creation order"""
        out = np.zeros((40, 4), dtype=np.float32)
        k = lib().orc_walker_get_polys(self._h, int(i), out.ctypes.data)
        return out[:k].copy()

    def bodies(self, i=0):
        out = np.zeros(30, dtype=np.float32)
        flags = np.zeros(4, dtype=np.int32)
        lib().orc_walker_get_bodies(self._h, int(i), out.ctypes.data, flags.ctypes.data)
        return out.reshape(5, 6), flags


def walker_action_flow(shaping_delta, action):
    """The action-dependent arithmetic of BipedalWalker.step in walker_oracle.c (test hook)."""
    a = np.ascontiguousarray(action, dtype=np.float32)
    ms, mt = np.zeros(4, dtype=np.float32), np.zeros(4, dtype=np.float32)
    r = ctypes.c_double(0.0)
    lib().orc_walker_action_flow(float(shaping_delta), a.ctypes.data, ms.ctypes.data, mt.ctypes.data, ctypes.byref(r))
    return ms, mt, r.value


class WalkerHeuristic:
    """The demo gait controller of gym/envs/box2d/bipedal_walker.py:775-854 ("suboptimal, have no notion of
    balance"): a three-state machine (stay on one leg / put the other down / push off) with PD targets on the hip
    and knee angles.  One instance drives one env; call it with the observation, get the next action."""

    STAY_ON_ONE_LEG, PUT_OTHER_DOWN, PUSH_OFF = 1, 2, 3
    SPEED = 0.29
    SUPPORT_KNEE_ANGLE = +0.1

    def __init__(self):
        self.state = self.STAY_ON_ONE_LEG
        self.moving_leg = 0
        self.supporting_knee_angle = self.SUPPORT_KNEE_ANGLE
        self.a = np.array([0.0, 0.0, 0.0, 0.0])

    def __call__(self, s):
        moving, supporting = self.moving_leg, 1 - self.moving_leg
        mb, sb = 4 + 5 * moving, 4 + 5 * supporting
        hip_targ, knee_targ = [None, None], [None, None]
        hip_todo, knee_todo = [0.0, 0.0], [0.0, 0.0]
        if self.state == self.STAY_ON_ONE_LEG:
            hip_targ[moving] = 1.1
            knee_targ[moving] = -0.6
            self.supporting_knee_angle += 0.03
            if s[2] > self.SPEED:
                self.supporting_knee_angle += 0.03
            self.supporting_knee_angle = min(self.supporting_knee_angle, self.SUPPORT_KNEE_ANGLE)
            knee_targ[supporting] = self.supporting_knee_angle
            if s[sb + 0] < 0.10:
                self.state = self.PUT_OTHER_DOWN
        if self.state == self.PUT_OTHER_DOWN:
            hip_targ[moving] = +0.1
            knee_targ[moving] = self.SUPPORT_KNEE_ANGLE
            knee_targ[supporting] = self.supporting_knee_angle
            if s[mb + 4]:
                self.state = self.PUSH_OFF
                self.supporting_knee_angle = min(s[mb + 2], self.SUPPORT_KNEE_ANGLE)
        if self.state == self.PUSH_OFF:
            knee_targ[moving] = self.supporting_knee_angle
            knee_targ[supporting] = +1.0
            if s[sb + 2] > 0.88 or s[2] > 1.2 * self.SPEED:
                self.state = self.STAY_ON_ONE_LEG
                self.moving_leg = 1 - moving
        for leg in (0, 1):
            if hip_targ[leg]:
                hip_todo[leg] = 0.9 * (hip_targ[leg] - s[4 + 5 * leg]) - 0.25 * s[5 + 5 * leg]
            if knee_targ[leg]:
                knee_todo[leg] = 4.0 * (knee_targ[leg] - s[6 + 5 * leg]) - 0.25 * s[7 + 5 * leg]
            hip_todo[leg] -= 0.9 * (0 - s[0]) - 1.5 * s[1]
            knee_todo[leg] -= 15.0 * s[3]
        a = np.array([hip_todo[0], knee_todo[0], hip_todo[1], knee_todo[1]])
        return np.clip(0.5 * a, -1.0, 1.0)


def rng_sequence(seed, ops):
    """Draws of Generator(PCG64(SeedSequence(seed))): op 0 uniform(-1,1), 1 integers(5,10), 2 random(),
    3 integers(1,5) -- through the C restatement (oracle/np_rng.h)."""
    ops = np.ascontiguousarray(ops, dtype=np.int32)
    out = np.zeros(len(ops), dtype=np.float64)
    lib().orc_rng_sequence(seed_words(seed).ctypes.data, ops.ctypes.data, len(ops), out.ctypes.data)
    return out


def lunar_engines(continuous, action, ang, posx, posy, disp0, disp1):
    """The engine arithmetic of lunar_oracle.c alone (test hook): impulses / points as Box2D receives them."""
    ca = np.zeros(2, dtype=np.float32)
    act = 0
    if continuous:
        ca[:] = action
    else:
        act = int(action)
    out = np.zeros(8, dtype=np.float32)
    cost = np.zeros(2, dtype=np.float64)
    on = np.zeros(2, dtype=np.int32)
    lib().orc_lunar_engines(int(continuous), act, ca.ctypes.data, float(ang), float(posx), float(posy), float(disp0),
                            float(disp1), out.ctypes.data, cost.ctypes.data, on.ctypes.data)
    return out, cost, on


def lunar_heuristic(s, continuous=False):
    """gym/envs/box2d/lunar_lander.py:726-777, used by the behavioural test."""
    angle_targ = s[0] * 0.5 + s[2] * 1.0
    angle_targ = min(max(angle_targ, -0.4), 0.4)
    hover_targ = 0.55 * np.abs(s[0])
    angle_todo = (angle_targ - s[4]) * 0.5 - (s[5]) * 1.0
    hover_todo = (hover_targ - s[1]) * 0.5 - (s[3]) * 0.5
    if s[6] or s[7]:
        angle_todo = 0
        hover_todo = -(s[3]) * 0.5
    if continuous:
        return np.clip(np.array([hover_todo * 20 - 1, -angle_todo * 20]), -1, +1)
    a = 0
    if hover_todo > np.abs(angle_todo) and hover_todo > 0.05:
        a = 2
    elif angle_todo < -0.05:
        a = 3
    elif angle_todo > +0.05:
        a = 1
    return a
