"""ctypes binding of ``libb200gym.so`` -- the reference-side stub of INTEGRATION.md.

The shared library is built in-tree by ``gym_b200.build.build()`` (nvcc,
``-gencode arch=compute_90a,code=sm_90a``).  There is no CPU fallback: if the
library is missing, ``load()`` raises ``DependencyNotInstalled`` and every env
constructor fails loudly.
"""
import ctypes
import os

from gym_b200 import error

_HERE = os.path.dirname(os.path.abspath(__file__))
# B200GYM_LIB points at an alternative build of the same library (A/B tuning runs only)
LIB_PATH = os.environ.get("B200GYM_LIB") or os.path.join(_HERE, "libb200gym.so")

# enum b200gym_kind (include/b200gym.h)
KIND_CARTPOLE = 0
KIND_MOUNTAINCAR = 1
KIND_MOUNTAINCAR_CONT = 2
KIND_PENDULUM = 3
KIND_ACROBOT = 4
KIND_LUNARLANDER = 5
KIND_BIPEDALWALKER = 6
KIND_LUNARLANDER_CONT = 7
KIND_BIPEDALWALKER_HARDCORE = 8

# b200gym_config.flags
LUNAR_ENABLE_WIND = 1

# enum b200gym_action_dtype
ACT_I64, ACT_I32, ACT_U8, ACT_F32 = 0, 1, 2, 3

# enum b200gym_mlp_activation, by the name rollout_mlp(activation=) takes
MLP_ACTIVATIONS = {"relu": 0, "tanh": 1}

# enum b200gym_mlp_head, by the name rollout_mlp(head=) takes
MLP_HEADS = {"tanh": 1, "tanh_normal": 2}


class Config(ctypes.Structure):
    """struct b200gym_config"""
    _fields_ = [
        ("kind", ctypes.c_int32),
        ("max_episode_steps", ctypes.c_int32),
        ("autoreset", ctypes.c_int32),
        ("flags", ctypes.c_int32),
        ("param", ctypes.c_double * 4),
    ]


class HostIO(ctypes.Structure):
    """struct b200gym_host_io"""
    _fields_ = [
        ("actions", ctypes.c_void_p),
        ("obs", ctypes.c_void_p),
        ("reward", ctypes.c_void_p),
        ("terminated", ctypes.c_void_p),
        ("truncated", ctypes.c_void_p),
        ("final_obs", ctypes.c_void_p),
    ]


# B200GYM_RMS_WORK_SIZE(dim): float64 words of the normalisers' moments work buffer
RMS_MAX_CTAS = 1056
NORM_WIDTHS = (1, 2, 3, 4, 6, 8, 24)


def rms_work_size(dim):
    return 1 + 2 * int(dim) * RMS_MAX_CTAS


SUBENV_MAX_STAGES = 8
SUBENV_MAX_STACK = 64
SUBENV_MAX_ACTION_STAGES = 2
# enum b200gym_subenv_op
SUB_EPISODE, SUB_NORM_OBS, SUB_NORM_REWARD, SUB_CLIP_OBS, SUB_CLIP_REWARD = 0, 1, 2, 3, 4
SUB_FRAME_STACK, SUB_TIME_AWARE, SUB_FLATTEN = 5, 6, 7
# enum b200gym_subenv_action_op
ACT_CLIP, ACT_RESCALE = 0, 1


class Subenv(ctypes.Structure):
    """struct b200gym_subenv"""
    _fields_ = [
        ("num_stages", ctypes.c_int32),
        ("op", ctypes.c_int32 * SUBENV_MAX_STAGES),
        ("raw_reward_type", ctypes.c_int32),
        ("int_reward_on_fall", ctypes.c_int32),
        ("p0", ctypes.c_double * SUBENV_MAX_STAGES),
        ("p1", ctypes.c_double * SUBENV_MAX_STAGES),
        ("obs_stats", ctypes.c_void_p),
        ("rew_stats", ctypes.c_void_p),
        ("ep_return", ctypes.c_void_p),
        ("ep_length", ctypes.c_void_p),
        ("clip_action", ctypes.c_int32),
        ("act_low", ctypes.c_float * 4),
        ("act_high", ctypes.c_float * 4),
        ("history", ctypes.c_void_p),
        ("head", ctypes.c_void_p),
        ("t", ctypes.c_void_p),
        ("num_action_stages", ctypes.c_int32),
        ("action_op", ctypes.c_int32 * SUBENV_MAX_ACTION_STAGES),
        ("action_low", (ctypes.c_float * 4) * SUBENV_MAX_ACTION_STAGES),
        ("action_high", (ctypes.c_float * 4) * SUBENV_MAX_ACTION_STAGES),
        ("action_min", (ctypes.c_float * 4) * SUBENV_MAX_ACTION_STAGES),
        ("action_max", (ctypes.c_float * 4) * SUBENV_MAX_ACTION_STAGES),
    ]


class P2PLayout(ctypes.Structure):
    """struct b200gym_p2p_layout"""
    _fields_ = [
        ("base", ctypes.c_void_p),
        ("set_bytes", ctypes.c_uint64),
        ("off_obs", ctypes.c_uint64),
        ("off_reward", ctypes.c_uint64),
        ("off_terminated", ctypes.c_uint64),
        ("off_truncated", ctypes.c_uint64),
        ("rows", ctypes.c_int64),
    ]


# every symbol include/b200gym.h declares: name -> (restype, argtypes)
_vp, _i64, _i32 = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int
SIGNATURES = {
    "b200gym_obs_dim": (_i32, [_i32]),
    "b200gym_act_dim": (_i32, [_i32]),
    "b200gym_num_actions": (_i32, [_i32]),
    "b200gym_state_dim": (_i32, [_i32]),
    "b200gym_version": (_i32, []),
    "b200gym_last_error": (ctypes.c_char_p, [_vp]),
    "b200gym_create": (_i32, [ctypes.POINTER(Config), _i64, _i32, ctypes.POINTER(_vp)]),
    "b200gym_destroy": (None, [_vp]),
    "b200gym_num_envs": (_i64, [_vp]),
    "b200gym_device": (_i32, [_vp]),
    "b200gym_seed_range": (_i32, [_vp, _vp, _i64, _vp]),
    "b200gym_seed_each": (_i32, [_vp, _vp, _vp, _vp]),
    "b200gym_reset": (_i32, [_vp, _vp, _vp, _vp, _vp]),
    "b200gym_step": (_i32, [_vp, _vp, _i32, _vp, _vp, _vp, _vp, _vp, _vp]),
    "b200gym_rollout": (_i32, [_vp, _vp, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "b200gym_rollout_sampled": (_i32, [_vp, _vp, _vp, _i64, _vp, _vp, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "b200gym_rollout_linear": (_i32, [_vp, _vp, _vp, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                      _vp]),
    "b200gym_rollout_mlp": (_i32, [_vp, _vp, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                   _vp, _vp, _vp, _vp]),
    "b200gym_rollout_mlp_noisy": (_i32, [_vp, _vp, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                         _vp, _vp, _vp, _vp]),
    "b200gym_rollout_mlp_act": (_i32, [_vp, _vp, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                       _vp, _vp, _vp, _vp, _vp, _i32]),
    "b200gym_rollout_mlp_noisy_act": (_i32, [_vp, _vp, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp,
                                             _vp, _vp, _vp, _vp, _vp, _i32]),
    "b200gym_rollout_mlp_head": (_i32, [_vp, _vp, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                        _vp, _vp, _vp, _vp, _vp, _i32, _i32]),
    "b200gym_rollout_mlp_noisy_head": (_i32, [_vp, _vp, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp,
                                              _vp, _vp, _vp, _vp, _vp, _i32, _i32]),
    "b200gym_rollout_actor_critic": (_i32, [_vp, _vp, _vp, _i32, _i32, _i32, _i32] + [_vp] * 10 +
                                     [ctypes.c_float, ctypes.c_float, _vp, _vp, _vp, _i32]),
    "b200gym_rollout_mlp_noisy_norm": (_i32, [_vp, _vp, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp,
                                               _vp, _vp, _vp, _vp, _vp, _i32, _vp, _vp, ctypes.c_double,
                                               ctypes.c_float]),
    "b200gym_rollout_actor_critic_norm": (_i32, [_vp, _vp, _vp, _i32, _i32, _i32, _i32] + [_vp] * 10 +
                                          [ctypes.c_float, ctypes.c_float, _vp, _vp, _vp, _i32, _vp, _vp,
                                           ctypes.c_double, ctypes.c_float, _vp, ctypes.c_float]),
    "b200gym_rollout_linear_norm": (_i32, [_vp, _vp, _vp, _i32, _i32] + [_vp] * 12 +
                                    [_vp, _vp, ctypes.c_double, ctypes.c_float, _vp, _vp]),
    "b200gym_rollout_mlp_norm": (_i32, [_vp, _vp, _i32, _i32, _i32, _i32, _i32] + [_vp] * 12 +
                                 [_i32, _vp, _vp, ctypes.c_double, ctypes.c_float, _vp, _vp]),
    "b200gym_invalid_actions": (_i32, [_vp, _vp, ctypes.POINTER(_i64)]),
    "b200gym_invalid_seen": (_i32, [_vp]),
    "b200gym_host_buffers": (_i32, [_vp, ctypes.POINTER(HostIO)]),
    "b200gym_step_host": (_i32, [_vp, _vp, _i32, _vp, _vp, _vp, _vp, _vp, ctypes.POINTER(_i64)]),
    "b200gym_reset_host": (_i32, [_vp, _vp, _vp, _vp]),
    "b200gym_get_state": (_i32, [_vp, _vp, _vp, _vp, _vp]),
    "b200gym_set_state": (_i32, [_vp, _vp, _vp, _vp, _vp]),
    "b200gym_snapshot_row_bytes": (_i64, [_i32]),
    "b200gym_snapshot_save": (_i32, [_vp, _vp, _i64, _vp, _vp]),
    "b200gym_snapshot_load": (_i32, [_vp, _vp, _vp, _vp, _i64, _vp]),
    "b200gym_clone": (_i32, [_vp, _vp, _vp]),
    "b200gym_snapshot_index_error": (_i32, [_vp]),
    "b200gym_rollout_from": (_i32, [_vp, _vp, _i64, _vp, _i64, _vp, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp]),
    "b200gym_rollout_from_mlp": (_i32, [_vp, _vp, _vp, _i64, _vp, _i64, _vp, _i32, _i32, _i32, _i32, _i32, _vp, _i32,
                                        _vp, _vp, ctypes.c_double, ctypes.c_float, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "b200gym_lunar_get_bodies": (_i32, [_vp, _vp, _vp, _vp]),
    "b200gym_lunar_wind_idx": (_i32, [_vp, _vp, _vp, _i32]),
    "b200gym_walker_get_bodies": (_i32, [_vp, _vp, _vp, _vp]),
    "b200gym_walker_get_terrain": (_i32, [_vp, _vp, _vp, _vp, _vp]),
    "b200gym_p2p_create": (_i32, [_vp, _i32, _i32, _vp, _vp]),
    "b200gym_p2p_connect": (_i32, [_vp, _vp]),
    "b200gym_step_p2p": (_i32, [_vp, _vp, _i32, _vp, _vp, ctypes.POINTER(_i32)]),
    "b200gym_p2p_status": (_i32, [_vp, _vp, ctypes.POINTER(_i32)]),
    "b200gym_episode_stats": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32, _i64, _vp]),
    "b200gym_rms_moments": (_i32, [_vp, _i32, _i64, _i32, _vp, _vp, _vp, _vp]),
    "b200gym_return_moments": (_i32, [_vp, _vp, ctypes.c_double, _i64, _vp, _vp, _vp, _vp]),
    "b200gym_rms_apply_obs": (_i32, [_vp, _vp, _i64, _i32, _vp, _vp, _vp, _vp, ctypes.c_double, ctypes.c_double, _i32, _vp]),
    "b200gym_rms_apply_reward": (_i32, [_vp, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _vp, ctypes.c_double, ctypes.c_double,
                                        _vp]),
    "b200gym_sample_space": (_i32, [_vp, _i64, _i32, _i64, _vp, _vp, _vp, _vp]),
    "b200gym_sample_space_stream": (_i32, [_vp, _vp, _i64, _i32, _i64, _vp, _vp, _vp, _vp]),
    "b200gym_subenv_set": (_i32, [_vp, ctypes.POINTER(Subenv)]),
    "b200gym_subenv_step": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "b200gym_subenv_reset": (_i32, [_vp, _vp, _vp, _vp]),
    "b200gym_subenv_width": (_i32, [_vp]),
    "b200gym_subenv_step_io": (_i32, [_vp] * 12),
    "b200gym_subenv_reset_io": (_i32, [_vp] * 5),
    "b200gym_subenv_actions": (_i32, [_vp] * 4),
    "b200gym_clip_actions": (_i32, [_vp, _vp, _i64, _i32, _vp, _vp, _vp]),
    "b200gym_subenv_host_buffers": (_i32, [_vp, ctypes.POINTER(_vp), ctypes.POINTER(_vp), ctypes.POINTER(_vp)]),
    "b200gym_box2d_overflows": (_i32, [_vp, _vp, ctypes.POINTER(_i64)]),
    "b200gym_box2d_list_counts": (_i32, [_vp, _vp, _i32, _vp, _vp]),
    "b200gym_selftest_trig": (_i32, [_vp, _i64, _vp, _vp, _vp, _vp]),
    "b200gym_selftest_tanh": (_i32, [_vp, _i64, _vp, _vp]),
    "b200gym_selftest_exp": (_i32, [_vp, _i64, _vp, _vp]),
    "b200gym_selftest_box2d": (_i32, [_i32, _vp, _i64, _vp, _vp]),
    "b200gym_selftest": (_i32, [_i32, _i64, ctypes.c_uint64, ctypes.POINTER(_i64)]),
}

_lib = None


def load():
    """dlopen the in-tree library and type every entry point; raises if it is not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise error.DependencyNotInstalled(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(gym_b200 has no CPU fallback)")
    lib = ctypes.CDLL(LIB_PATH)
    for name, (restype, argtypes) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError here = header and library disagree
        fn.restype = restype
        fn.argtypes = argtypes
    _lib = lib
    return lib


def last_error(handle=None):
    msg = load().b200gym_last_error(handle)
    return msg.decode() if msg else ""


def check(rc, handle=None):
    if rc != 0:
        raise RuntimeError("b200gym: " + last_error(handle))
