"""ctypes wrapper of tests/hostsim/rollout_norm.cpp: the device source of rollout_mlp_noisy_norm_kernel,
rollout_actor_critic_norm_kernel and gae_scaled_kernel on the CPU.

Built on demand with g++ into tests/hostsim/_build/ (git-ignored), with the flags of rollout_sim.py.
"""
import ctypes
import math
import os
import subprocess

import numpy as np

from hostsim import rollout_sim
from hostsim.rollout_actor_critic_sim import ActorCriticRolloutSim

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = os.path.join(rollout_sim._BUILD, "librollout_norm.so")
_SRCS = rollout_sim._SRCS + [os.path.join(_HERE, "rollout_norm.cpp")]
_lib = None

RELU, TANH = 0, 1


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB) or os.path.getmtime(_LIB) < max(os.path.getmtime(s) for s in _SRCS):
            os.makedirs(rollout_sim._BUILD, exist_ok=True)
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared",
                                   "-Wno-unknown-pragmas", "-o", _LIB, os.path.join(_HERE, "rollout_norm.cpp")])
        L = ctypes.CDLL(_LIB)
        vp, i64, i32, f32, f64 = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_float, ctypes.c_double
        L.hs_mlp_noisy_norm_rollout.restype = i64
        L.hs_mlp_noisy_norm_rollout.argtypes = [ctypes.POINTER(rollout_sim._Batch), vp, i32, i32, i32,
                                                ctypes.c_int32] + [vp] * 11 + [f64, f32]
        L.hs_actor_critic_norm_rollout.restype = i64
        L.hs_actor_critic_norm_rollout.argtypes = [ctypes.POINTER(rollout_sim._Batch), vp, vp, i32, i32, i32,
                                                   ctypes.c_int32] + [vp] * 10 + [f32, f32, vp, vp, vp, f64, f32, vp,
                                                                                   f32]
        L.hs_gae_scaled.restype = None
        L.hs_gae_scaled.argtypes = [i64, ctypes.c_int32, f32, f32, f64, f64, f32, vp, vp, vp, vp, vp]
        L.hs_norm_elems.restype = None
        L.hs_norm_elems.argtypes = [i64, vp, f64, f64, f64, f32, vp]
        _lib = L
    return _lib


def _clip(c):
    return math.inf if c is None else float(np.float32(c))


def gae_scaled(g, gl, ret_var, eps, clip_r, reward, term, trunc, values, held):
    """gae_scaled_env over (T, n) rows (gae() of rollout_actor_critic_sim with the rewards scaled)."""
    reward = np.ascontiguousarray(reward, dtype=np.float64)
    T, n = reward.shape
    te = np.ascontiguousarray(term, dtype=np.uint8)
    tr = np.ascontiguousarray(trunc, dtype=np.uint8)
    v = np.ascontiguousarray(values, dtype=np.float32)
    adv = np.array(held, dtype=np.float32, order="C")
    lib().hs_gae_scaled(n, T, g, gl, float(ret_var), float(eps), _clip(clip_r), reward.ctypes.data, te.ctypes.data,
                        tr.ctypes.data, v.ctypes.data, adv.ctypes.data)
    return adv


def norm_elems(o, mean, var, eps, clip):
    """norm_obs_elem over the float32 array o with one column's statistics."""
    o = np.ascontiguousarray(o, dtype=np.float32)
    x = np.empty_like(o)
    lib().hs_norm_elems(o.size, o.ctypes.data, float(mean), float(var), float(eps), _clip(clip), x.ctypes.data)
    return x


class NormRolloutSim(ActorCriticRolloutSim):
    """ActorCriticRolloutSim plus the normalised launches."""

    def _acts(self, T):
        if self.act_dim == 0:
            return np.full((T, self.n), -1, dtype=np.int64)
        return np.full((T, self.n, self.act_dim), np.nan, dtype=np.float32)

    def rollout_mlp_noisy_norm(self, params, hidden, noise, mean, var, eps, clip, act=RELU, last_obs=None):
        """-> (actions, outputs, obs, rew, term, trunc, final_obs), as rollout_mlp_noisy."""
        w = np.ascontiguousarray(params, dtype=np.float32)
        e = np.ascontiguousarray(noise, dtype=np.float32)
        m = np.ascontiguousarray(mean, dtype=np.float64)
        v = np.ascontiguousarray(var, dtype=np.float64)
        T = e.shape[0]
        h1, h2 = (hidden[0], 0) if len(hidden) == 1 else hidden
        last = np.zeros((self.n, self.obs_dim), dtype=np.float32) if last_obs is None else last_obs
        outputs = np.full(e.shape, np.nan, dtype=np.float32)
        acts = self._acts(T)
        obs, rew, te, tr, fo = self._outputs((T, self.n))
        rc = lib().hs_mlp_noisy_norm_rollout(ctypes.byref(self._b), w.ctypes.data, h1, h2, act, int(T), e.ctypes.data,
                                             outputs.ctypes.data, acts.ctypes.data, obs.ctypes.data, rew.ctypes.data,
                                             te.ctypes.data, tr.ctypes.data, fo.ctypes.data, last.ctypes.data,
                                             m.ctypes.data, v.ctypes.data, float(eps), _clip(clip))
        assert rc == 0
        return acts, outputs, obs, rew, te.astype(bool), tr.astype(bool), fo

    def rollout_actor_critic_norm(self, actor, critic, hidden, noise, g, gl, mean, var, eps, clip, ret_var=None,
                                  clip_r=None, act=RELU, last_obs=None):
        """-> (actions, outputs, values, advantages, obs, rew, term, trunc, final_obs), as rollout_actor_critic."""
        wa = np.ascontiguousarray(actor, dtype=np.float32)
        wc = np.ascontiguousarray(critic, dtype=np.float32)
        e = np.ascontiguousarray(noise, dtype=np.float32)
        m = np.ascontiguousarray(mean, dtype=np.float64)
        v = np.ascontiguousarray(var, dtype=np.float64)
        rv = None if ret_var is None else np.array([ret_var], dtype=np.float64)
        T = e.shape[0]
        h1, h2 = (hidden[0], 0) if len(hidden) == 1 else hidden
        last = np.zeros((self.n, self.obs_dim), dtype=np.float32) if last_obs is None else last_obs
        outputs = np.full(e.shape, np.nan, dtype=np.float32)
        values = np.full((T + 1, self.n), np.nan, dtype=np.float32)
        adv = np.full((T, self.n), np.nan, dtype=np.float32)
        acts = self._acts(T)
        obs, rew, te, tr, fo = self._outputs((T, self.n))
        rc = lib().hs_actor_critic_norm_rollout(
            ctypes.byref(self._b), wa.ctypes.data, wc.ctypes.data, h1, h2, act, int(T), e.ctypes.data,
            outputs.ctypes.data, acts.ctypes.data, obs.ctypes.data, rew.ctypes.data, te.ctypes.data, tr.ctypes.data,
            fo.ctypes.data, values.ctypes.data, adv.ctypes.data, g, gl, last.ctypes.data, m.ctypes.data, v.ctypes.data,
            float(eps), _clip(clip), None if rv is None else rv.ctypes.data, _clip(clip_r))
        assert rc == 0
        return acts, outputs, values, adv, obs, rew, te.astype(bool), tr.astype(bool), fo
