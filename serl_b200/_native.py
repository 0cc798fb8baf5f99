"""ctypes binding of the C-ABI library (include/serl_b200.h): the only module that binds it.  The product path has no CPU
fallback: importing succeeds without a GPU (so host logic is testable), but the library must exist and every compute call
fails loudly when CUDA is unavailable.  tests/test_capi.py holds the signatures and constants below to the header,
tests/test_td3_oracle.py those of include/serl_td3.h (TD3_SIGNATURES, TD3Desc, TD3_*), tests/test_td3_wide.py its wide
bounds, tests/test_td3_per.py those of include/serl_td3_per.h (PER_SIGNATURES, TD3PerDesc, PER_MAX_CAPACITY),
tests/test_deep_actor.py those of include/serl_route.h (ROUTE_SIGNATURES)."""
import ctypes
import os

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get('SERL_B200_LIB') or os.path.join(HERE, 'libserl_b200.so')   # SERL_B200_LIB: e.g. the --exact validation build

ACTIVATIONS = {'tanh': 0, 'elu': 1, 'relu': 2}        # SERL_ACT_* ('relu' is the reference's LeakyReLU(0.01))
PLANT_VARIANTS = ['h2000_v90', 'ice', 'cg', 'cg_for', 'h2000_v150', 'h10000_v90', 'cg_timed', 'cg_timed_post']   # SERL_PLANT_*
FAULTS = ['none', 'be', 'jr', 'sa', 'se']             # SERL_FAULT_*
TRACE_COLS = 22
TRACK_COLS = 4
REPLAY_COLS = 20
MODE_GUST = 1 << 24
MODE_GUST_UP = 1 << 25
ROLLOUT_GUST = 1
ROLLOUT_STAGGER = 2
ROLLOUT_PER_ACTOR_REFS = 4
ROLLOUT_INCREMENTAL = 8
ROLLOUT_SYMMETRIC = 16
ROLLOUT_SUITE = 32
STATUS_NONFINITE = 1
STATUS_GUST_FLAG = 2
# include/serl_td3.h (K7, the fused TD3 learner)
TD3_CRITIC_HIDDEN = 64
TD3_MAX_BATCH = 128
TD3_MAX_HIDDEN = 320
TD3_MAX_WIDE_LAYERS = 8
TD3_CHAMPION_TARGET = 1
TD3_STATUS_INDEX = 4
TD3_MAX_GROUP = 64
# include/serl_td3_per.h (prioritized replay's priority tree)
PER_MAX_CAPACITY = 1 << 30


class ActorShape(ctypes.Structure):
    _fields_ = [('state_dim', ctypes.c_int32), ('action_dim', ctypes.c_int32), ('hidden', ctypes.c_int32),
                ('num_layers', ctypes.c_int32), ('activation', ctypes.c_int32)]


class RolloutDesc(ctypes.Structure):
    """serl_rollout_desc (include/serl_b200.h)"""
    _fields_ = [('d_weights', ctypes.c_void_p), ('pop', ctypes.c_int32), ('shape', ActorShape),
                ('d_ref_levels', ctypes.c_void_p), ('d_ref_starts', ctypes.c_void_p), ('d_env_mode', ctypes.c_void_p),
                ('n_envs', ctypes.c_int32), ('horizon', ctypes.c_int32), ('d_action_noise', ctypes.c_void_p),
                ('d_returns', ctypes.c_void_p), ('d_steps', ctypes.c_void_p), ('d_fitness', ctypes.c_void_p),
                ('d_trace', ctypes.c_void_p), ('d_actions', ctypes.c_void_p),
                ('t_max', ctypes.c_double), ('smooth_width', ctypes.c_double),
                ('d_env_order', ctypes.c_void_p), ('d_replay', ctypes.c_void_p), ('replay_env', ctypes.c_int32),
                ('d_status', ctypes.c_void_p), ('sm_limit', ctypes.c_int32),
                ('widths', ctypes.c_void_p), ('n_widths', ctypes.c_int32), ('d_sensor_noise', ctypes.c_void_p),
                ('flags', ctypes.c_int32), ('d_track', ctypes.c_void_p), ('d_cost', ctypes.c_void_p)]


class TD3Desc(ctypes.Structure):
    """serl_td3_desc (include/serl_td3.h)"""
    _fields_ = [('shape', ActorShape), ('d_state', ctypes.c_void_p),
                ('d_replay', ctypes.c_void_p), ('replay_cols', ctypes.c_int32), ('n_valid', ctypes.c_int32),
                ('batch', ctypes.c_int32), ('n_steps', ctypes.c_int32),
                ('first_iteration', ctypes.c_int64), ('critic_adam_steps', ctypes.c_int64), ('actor_adam_steps', ctypes.c_int64),
                ('gamma', ctypes.c_double), ('tau', ctypes.c_double), ('lr', ctypes.c_double), ('noise_sd', ctypes.c_double),
                ('noise_clip', ctypes.c_double), ('policy_update_freq', ctypes.c_int32),
                ('caps_lambda_t', ctypes.c_double), ('caps_lambda_s', ctypes.c_double), ('caps_eps_sd', ctypes.c_double),
                ('max_grad_norm', ctypes.c_double), ('flags', ctypes.c_int32), ('seed', ctypes.c_uint64),
                ('cluster_size', ctypes.c_int32), ('d_indices', ctypes.c_void_p), ('d_losses', ctypes.c_void_p),
                ('d_rec_indices', ctypes.c_void_p), ('d_rec_noise', ctypes.c_void_p), ('d_rec_caps', ctypes.c_void_p),
                ('d_status', ctypes.c_void_p)]


class TD3PerDesc(ctypes.Structure):
    """serl_td3_per_desc (include/serl_td3.h)"""
    _fields_ = [('d_tree', ctypes.c_void_p), ('capacity', ctypes.c_int32), ('n_valid', ctypes.c_int32),
                ('alpha', ctypes.c_double), ('beta0', ctypes.c_double), ('beta_frames', ctypes.c_double),
                ('d_rec_weights', ctypes.c_void_p), ('d_rec_td', ctypes.c_void_p)]


_vp, _i32, _i64, _f64, _int, _shape = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64, ctypes.c_double, ctypes.c_int, ctypes.POINTER(ActorShape)
# entry point -> (restype, argtypes), in the header's order; every entry point returning a serl_status takes the stream last
SIGNATURES = {
    'serl_actor_num_params': (_i64, [_shape]),
    'serl_rollout_run': (_int, [ctypes.POINTER(RolloutDesc), _vp]),
    'serl_actor_forward': (_int, [_vp, _shape, _vp, _i32, _vp, _vp]),
    'serl_actor_num_params_wide': (_i64, [_vp, _i32]),
    'serl_actor_forward_wide': (_int, [_vp, _vp, _i32, _i32, _vp, _i32, _vp, _vp]),
    'serl_smoothness': (_int, [_vp, _vp, _i32, _i32, _f64, _vp, _vp]),
    'serl_plant_init': (_int, [_vp, _vp, _i32, _vp]),
    'serl_plant_step': (_int, [_vp, _vp, _vp, _i32, _vp]),
    'serl_plant_step_timed': (_int, [_vp, _vp, _vp, _vp, _i32, _vp]),
    'serl_ssne_select': (_int, [_vp, _i32, _vp, _i32, _vp, _vp, _vp]),
    'serl_ssne_clone': (_int, [_vp, _i32, _i32, _vp, _i32, _vp]),
    'serl_ssne_crossover': (_int, [_vp, _i32, _i32, _vp, _i32, _vp, _vp]),
    'serl_ssne_mutate': (_int, [_vp, _i32, _i32, _vp, _i32, _vp, _vp, _vp, ctypes.c_float, ctypes.c_float, _vp]),
    'serl_plan_create': (_vp, [_vp, _vp, _vp, _vp, _i32, _vp, _i32, _vp, _i32, _vp, _i32, _vp, _i32, _f64]),
    'serl_plan_sizes': (None, [_vp, _vp]),
    'serl_plan_copy': (None, [_vp] * 7),
    'serl_plan_destroy': (None, [_vp]),
    'serl_launch_count': (_i64, []),
    'serl_last_error': (ctypes.c_char_p, []),
}
# the entry points of include/serl_td3.h (included by serl_b200.h), bound the same way
TD3_SIGNATURES = {
    'serl_td3_state_floats': (_i64, [_shape]),
    'serl_td3_learn': (_int, [ctypes.POINTER(TD3Desc), ctypes.POINTER(TD3PerDesc), _i32, _vp]),
}
# include/serl_td3_per.h: the priority tree's entry points
PER_SIGNATURES = {
    'serl_per_tree_doubles': (_i64, [_i32]),
    'serl_per_rebuild': (_int, [_vp, _i32, _vp]),
    'serl_per_insert': (_int, [_vp, _i32, _i32, _i32, _i32, _vp]),
    'serl_per_update': (_int, [_vp, _i32, _vp, _vp, _i32, _f64, _vp]),
    'serl_per_sample': (_int, [_vp, _i32, _i32, _i32, ctypes.c_uint64, _i64, _f64, _vp, _vp, _vp]),
}
# include/serl_route.h: the kernel of a uniform actor (host only, no stream)
ROUTE_SIGNATURES = {
    'serl_actor_tc_widths': (_i32, [_shape, _vp, _i32]),
}
_lib = None


class NativeError(RuntimeError):
    pass


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise NativeError('serl_b200: %s is missing — build it with `python -m serl_b200.build` '
                              '(there is no CPU fallback)' % LIB_PATH)
        L = ctypes.CDLL(LIB_PATH)
        for name, (restype, argtypes) in {**SIGNATURES, **TD3_SIGNATURES, **PER_SIGNATURES, **ROUTE_SIGNATURES}.items():
            f = getattr(L, name)
            f.restype, f.argtypes = restype, argtypes
        _lib = L
    return _lib


def check(rc, what):
    if rc != 0:
        raise NativeError('%s failed (%d): %s' % (what, rc, lib().serl_last_error().decode()))


def call(name, *args, device=None):
    """lib().<name>(*args, stream) for a serl_status entry point: tensors and arrays go as pointers (`args` keeps them alive through
    the call), the stream is the current one of `device` (default: the first tensor's device); a failure raises NativeError."""
    device = device or next((a.device for a in args if isinstance(a, torch.Tensor)), None)
    ptrs = [a.data_ptr() if isinstance(a, torch.Tensor) else a.ctypes if isinstance(a, np.ndarray) else a for a in args]
    check(getattr(lib(), name)(*ptrs, torch.cuda.current_stream(device).cuda_stream), name)
