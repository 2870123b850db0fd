"""ctypes wrapper of tests/hostsim/rollout_actor_critic.cpp: the device source of rollout_actor_critic_kernel and
gae_kernel on the CPU.

Built on demand with g++ into tests/hostsim/_build/ (git-ignored), with the flags of rollout_sim.py.
"""
import ctypes
import os
import subprocess

import numpy as np

from hostsim import rollout_sim
from hostsim.rollout_mlp_noisy_sim import MlpNoisyRolloutSim

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = os.path.join(rollout_sim._BUILD, "librollout_actor_critic.so")
_SRCS = rollout_sim._SRCS + [os.path.join(_HERE, "rollout_actor_critic.cpp")]
_lib = None

RELU, TANH = 0, 1


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB) or os.path.getmtime(_LIB) < max(os.path.getmtime(s) for s in _SRCS):
            os.makedirs(rollout_sim._BUILD, exist_ok=True)
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared",
                                   "-Wno-unknown-pragmas", "-o", _LIB, os.path.join(_HERE, "rollout_actor_critic.cpp")])
        L = ctypes.CDLL(_LIB)
        vp, i64, i32, f32 = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_float
        L.hs_actor_critic_rollout.restype = i64
        L.hs_actor_critic_rollout.argtypes = [ctypes.POINTER(rollout_sim._Batch), vp, vp, i32, i32, i32,
                                              ctypes.c_int32] + [vp] * 10 + [f32, f32, vp]
        L.hs_gae.restype = None
        L.hs_gae.argtypes = [i64, ctypes.c_int32, f32, f32, vp, vp, vp, vp, vp]
        _lib = L
    return _lib


def gae(g, gl, reward, term, trunc, values, held):
    """gae_env over (T, n) rows: reward float64, term / trunc bool, values (T + 1, n) float32, held (T, n) float32
    with V(final obs) where a step truncated without terminating -> advantages (T, n)."""
    reward = np.ascontiguousarray(reward, dtype=np.float64)
    T, n = reward.shape
    te = np.ascontiguousarray(term, dtype=np.uint8)
    tr = np.ascontiguousarray(trunc, dtype=np.uint8)
    v = np.ascontiguousarray(values, dtype=np.float32)
    adv = np.array(held, dtype=np.float32, order="C")
    assert v.shape == (T + 1, n) and adv.shape == (T, n) and te.shape == tr.shape == (T, n)
    lib().hs_gae(n, T, g, gl, reward.ctypes.data, te.ctypes.data, tr.ctypes.data, v.ctypes.data, adv.ctypes.data)
    return adv


class ActorCriticRolloutSim(MlpNoisyRolloutSim):
    """MlpNoisyRolloutSim plus ``rollout_actor_critic``, the rollout and GAE launches of one call."""

    def rollout_actor_critic(self, actor, critic, hidden, noise, g, gl, act=RELU, last_obs=None):
        """T = len(noise) steps of the noisy actor with the critic; g, gl the float32 GAE coefficients ->
        (actions, outputs, values, advantages, obs, rew, term, trunc, final_obs) with a leading T (T + 1) axis."""
        wa = np.ascontiguousarray(actor, dtype=np.float32)
        wc = np.ascontiguousarray(critic, dtype=np.float32)
        e = np.ascontiguousarray(noise, dtype=np.float32)
        T = e.shape[0]
        h1, h2 = (hidden[0], 0) if len(hidden) == 1 else hidden
        last = np.zeros((self.n, self.obs_dim), dtype=np.float32) if last_obs is None else last_obs
        outputs = np.full(e.shape, np.nan, dtype=np.float32)
        values = np.full((T + 1, self.n), np.nan, dtype=np.float32)
        adv = np.full((T, self.n), np.nan, dtype=np.float32)
        if self.act_dim == 0:
            acts = np.full((T, self.n), -1, dtype=np.int64)
        else:
            acts = np.full((T, self.n, self.act_dim), np.nan, dtype=np.float32)
        obs, rew, te, tr, fo = self._outputs((T, self.n))
        rc = lib().hs_actor_critic_rollout(ctypes.byref(self._b), wa.ctypes.data, wc.ctypes.data, h1, h2, act, int(T),
                                           e.ctypes.data, outputs.ctypes.data, acts.ctypes.data, obs.ctypes.data,
                                           rew.ctypes.data, te.ctypes.data, tr.ctypes.data, fo.ctypes.data,
                                           values.ctypes.data, adv.ctypes.data, g, gl, last.ctypes.data)
        assert rc == 0
        return acts, outputs, values, adv, obs, rew, te.astype(bool), tr.astype(bool), fo
