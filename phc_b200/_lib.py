"""ctypes binding of libphc_b200.so -- the ONLY compute path of phc_b200 (there is no CPU / eager fallback).

Mirrors include/phc_b200.h one to one.  Loading fails loudly (ImportError naming the build command) when the
shared object is absent; every wrapper raises PhcError on a non-zero return code.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# PHC_LIB_PATH: experiment builds of the SAME sources (phc_b200.build.build_variant); default = the in-tree library
LIB_PATH = os.environ.get("PHC_LIB_PATH") or os.path.join(_HERE, "lib", "libphc_b200.so")

PHC_FLAG_UPRIGHT = 1 << 0
PHC_FLAG_LOCAL_ROOT_OBS = 1 << 1
PHC_FLAG_ROOT_HEIGHT_OBS = 1 << 2
PHC_FLAG_POWER_REWARD = 1 << 3
PHC_FLAG_EARLY_TERM = 1 << 4
PHC_FLAG_NO_COLLISION = 1 << 5
PHC_FLAG_TERM_USE_MEAN = 1 << 6
PHC_FLAG_OBS_ONLY = 1 << 7
PHC_FLAG_REWARD_FROM_CACHE = 1 << 8
PHC_FLAG_ZERO_OUT_FAR = 1 << 9
PHC_FLAG_CYCLE_MOTION = 1 << 10
PHC_FLAG_NO_SPECIALISE = 1 << 11
PHC_FLAG_SUBSET_REWARD = 1 << 12
PHC_FLAG_TASK_OBS_KP = 1 << 13
PHC_FLAG_RECOVERY = 1 << 14
PHC_FLAG_AMP_CURRENT = 1 << 15
PHC_ACT_NONE, PHC_ACT_RELU, PHC_ACT_SILU, PHC_ACT_SILU_BWD, PHC_ACT_RELU_BITS, PHC_ACT_MASK_BITS = 0, 1, 2, 3, 4, 5
PHC_MAX_KEY_BODIES = 8
PHC_MAX_BODIES = 64
PHC_LANE_BODIES = 32
PHC_MAX_AMP_JOINTS = 64
PHC_MAX_EXT_BODIES = 8
PHC_EVAL_ACC_FIELDS = 8

_p = C.c_void_p


class PhcError(RuntimeError):
    pass


class PhcMotionLib(C.Structure):
    _fields_ = [("frames_body", _p), ("frames_joint", _p), ("motion_len", _p), ("motion_dt", _p),
                ("motion_num_frames", _p), ("length_starts", _p), ("num_frames_total", C.c_int64),
                ("num_motions", C.c_int32), ("num_bodies", C.c_int32), ("body_stride", C.c_int32),
                ("joint_stride", C.c_int32), ("num_ext_bodies", C.c_int32), ("num_dofs", C.c_int32)]


class PhcMotionStateOut(C.Structure):
    _fields_ = [(n, _p) for n in ("rg_pos", "rb_rot", "body_vel", "body_ang_vel", "dof_pos", "dof_vel", "root_pos",
                                  "root_rot", "root_vel", "root_ang_vel", "rg_pos_t", "rg_rot_t", "body_vel_t", "body_ang_vel_t")]


class PhcStepArgs(C.Structure):
    _fields_ = [
        ("body_state", _p), ("dof_state", _p), ("dof_force", _p), ("bodies_per_env", C.c_int32),
        ("progress", _p), ("motion_ids", _p), ("env_motion", _p), ("start_times", _p), ("start_offsets", _p), ("global_offset", _p),
        ("cycle_counter", _p), ("only_where", _p), ("lib", PhcMotionLib),
        ("num_envs", C.c_int32), ("time_steps", C.c_int32), ("dt", C.c_float), ("traj_dt", C.c_float),
        ("flags", C.c_uint32),
        ("k_pos", C.c_float), ("k_rot", C.c_float), ("k_vel", C.c_float), ("k_ang_vel", C.c_float),
        ("w_pos", C.c_float), ("w_rot", C.c_float), ("w_vel", C.c_float), ("w_ang_vel", C.c_float),
        ("power_coef", C.c_float), ("term_thresh", C.c_float * PHC_MAX_BODIES), ("term_dist_mean", C.c_float),
        ("ext_parent", C.c_int32 * PHC_MAX_EXT_BODIES), ("ext_pos", (C.c_float * 3) * PHC_MAX_EXT_BODIES),
        ("num_key_bodies", C.c_int32), ("key_bodies", C.c_int32 * PHC_MAX_KEY_BODIES),
        ("amp_joints", C.c_int32 * PHC_MAX_AMP_JOINTS), ("num_amp_joints", C.c_int32),
        ("obs", _p), ("obs_stride", C.c_int64), ("rew", _p), ("reward_raw", _p), ("reset", _p), ("terminate", _p),
        ("amp_out", _p), ("amp_hist_in", _p), ("amp_out_stride", C.c_int64), ("amp_steps", C.c_int32),
        ("ref_body_pos", _p), ("ref_body_rot", _p), ("ref_body_vel", _p), ("ref_body_ang_vel", _p),
        ("ref_cache", _p),
        ("close_distance", C.c_float), ("far_distance", C.c_float), ("max_episode_length", C.c_int32), ("point_goal", _p),
        ("cycle_phase", _p), ("mpjpe", _p), ("body_pos_gt", _p), ("ring_head", _p),
        ("num_track", C.c_int32), ("track_slot", C.c_int8 * PHC_MAX_BODIES), ("occlusion", _p), ("shape_params", _p), ("num_shape", C.c_int32),
        ("limb_weights", _p), ("num_limb", C.c_int32), ("recovery_counter", _p),
    ]


class PhcGemmDesc(C.Structure):
    _fields_ = [("A", _p), ("lda", C.c_int64), ("a_kmajor", C.c_int32), ("B", _p), ("ldb", C.c_int64), ("b_kmajor", C.c_int32),
                ("C", _p), ("ldc", C.c_int64), ("M", C.c_int32), ("N", C.c_int32), ("K", C.c_int32), ("alpha", C.c_float),
                ("bias", _p), ("act", C.c_int32), ("aux", _p), ("ldaux", C.c_int64), ("accumulate", C.c_int32), ("k_splits", C.c_int32),
                ("B_lo", _p), ("B_img", _p), ("A_img", _p)]


class PhcGemmImageDesc(C.Structure):
    _fields_ = [("B", _p), ("ldb", C.c_int64), ("b_kmajor", C.c_int32), ("N", C.c_int32), ("K", C.c_int32), ("img", _p)]


class PhcColsumDesc(C.Structure):
    _fields_ = [("X", _p), ("ld", C.c_int64), ("M", C.c_int32), ("N", C.c_int32), ("alpha", C.c_float), ("out", _p)]


PHC_GEMM_GROUP_MAX = 8
PHC_GEMM_FP32_3XTF32, PHC_GEMM_TF32_SINGLE_PASS = 0, 1

# name -> (restype, argtypes); must list every symbol include/phc_b200.h declares (tests check this)
SIGNATURES = {
    "phc_version": (C.c_int, []),
    "phc_last_error": (C.c_char_p, []),
    "phc_compiled_sm": (C.c_int, []),
    "phc_launch_count": (C.c_int64, []),
    "phc_env_motion_gather": (C.c_int, [C.POINTER(PhcMotionLib), _p, C.c_int64, _p, _p]),
    "phc_motion_body_stride": (C.c_int, [C.c_int32]),
    "phc_reset_bookkeeping": (C.c_int, [_p, _p, _p, C.c_int64, _p, _p, _p, _p, _p, _p, _p, _p]),
    "phc_motion_dof_stride": (C.c_int, [C.c_int32]),
    "phc_motion_pack_dofs": (C.c_int, [_p, _p, C.c_int64, C.c_int32, _p, _p]),
    "phc_amp_obs_dim_robot": (C.c_int, [C.c_int32, C.c_int32, C.c_uint32]),
    "phc_motion_joint_stride": (C.c_int, [C.c_int32]),
    "phc_motion_pack": (C.c_int, [_p, _p, _p, _p, _p, _p, C.c_int64, C.c_int32, _p, _p, _p]),
    "phc_motion_load_workspace_bytes": (C.c_int64, [C.c_int64, C.c_int32]),
    "phc_motion_load": (C.c_int, [_p, _p, _p, _p, _p, _p, _p, _p, C.c_int64, C.c_int32, C.c_int32, _p, _p, _p, _p, _p, _p, _p, _p]),
    "phc_motion_state": (C.c_int, [C.POINTER(PhcMotionLib), _p, _p, _p, C.c_int64, C.POINTER(PhcMotionStateOut), _p]),
    "phc_self_obs_dim": (C.c_int, [C.c_int32, C.c_uint32]),
    "phc_task_obs_dim": (C.c_int, [C.c_int32, C.c_int32]),
    "phc_task_obs_dim_flags": (C.c_int, [C.c_int32, C.c_int32, C.c_uint32]),
    "phc_amp_obs_dim": (C.c_int, [C.c_int32, C.c_int32, C.c_uint32]),
    "phc_env_step": (C.c_int, [C.POINTER(PhcStepArgs), _p]),
    "phc_env_step_fast_launches": (C.c_int64, []),
    "phc_amp_obs_demo": (C.c_int, [C.POINTER(PhcMotionLib), _p, _p, C.c_int64, C.c_int32, C.c_int32, C.c_float,
                                   C.c_uint32, _p, C.c_int32, _p, C.c_int32, _p, C.c_int64, _p, C.c_int32, _p]),
    "phc_amp_obs_demo_ring": (C.c_int, [C.POINTER(PhcMotionLib), _p, _p, C.c_int64, C.c_int32, C.c_int32, C.c_float,
                                        C.c_uint32, _p, C.c_int32, _p, C.c_int32, _p, C.c_int64, _p, C.c_int32, _p, _p]),
    "phc_amp_window_export_ring": (C.c_int, [_p, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_int32, _p, _p, C.c_int64, _p]),
    "phc_ring_advance": (C.c_int, [_p, C.c_int32, _p]),
    "phc_launch_count_add": (None, [C.c_int64]),
    "phc_amp_window_export": (C.c_int, [_p, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_int32, _p, C.c_int64, _p]),
    "phc_set_env_state": (C.c_int, [C.POINTER(PhcMotionLib), _p, _p, _p, _p, C.c_int64, _p, C.c_int32, _p, _p]),
    "phc_getup_reset": (C.c_int, [_p, _p, _p, _p, _p, _p, _p, C.c_int32, _p, _p, C.c_int64, _p, _p, _p, C.c_int64, _p, C.c_int32, _p,
                                  C.c_int32, _p, _p, _p, _p, _p, _p]),
    "phc_amp_ring_fill": (C.c_int, [_p, C.c_int64, C.c_int64, C.c_int32, C.c_int32, _p, _p, _p]),
    "phc_eval_metrics_step": (C.c_int, [_p, C.c_int64, C.c_int64, C.c_int64, _p, _p, C.c_int32, C.c_int64, C.c_int32, _p, _p, _p]),
    "phc_episode_stats": (C.c_int, [_p, _p, C.c_int64, _p, _p, _p, _p, C.c_int32, _p]),
    "phc_gae": (C.c_int, [_p, _p, _p, _p, C.c_int32, C.c_int64, C.c_float, C.c_float, _p, _p, _p]),
    "phc_adv_norm_workspace_bytes": (C.c_int64, [C.c_int64]),
    "phc_adv_norm": (C.c_int, [_p, _p, C.c_int64, C.c_int32, _p, _p, _p]),
    "phc_gemm": (C.c_int, [_p, C.c_int64, C.c_int32, _p, C.c_int64, C.c_int32, _p, C.c_int64, C.c_int32, C.c_int32,
                           C.c_int32, C.c_float, _p, C.c_int32, _p, C.c_int64, C.c_int32, C.c_int32, _p]),
    "phc_split_tf32": (C.c_int, [_p, C.c_int64, C.c_int64, C.c_int32, _p, _p, C.c_int64, _p]),
    "phc_gemm_tc5": (C.c_int, [_p, _p, C.c_int64, C.c_int32, _p, _p, C.c_int64, C.c_int32, _p, _p, _p, C.c_int64, C.c_int32, C.c_int32,
                               C.c_int32, C.c_float, _p, C.c_int32, _p, C.c_int64, C.c_int32, C.c_int32, _p]),
    "phc_gemm_group": (C.c_int, [C.POINTER(PhcGemmDesc), C.c_int32, _p]),
    "phc_split_lo": (C.c_int, [_p, _p, C.c_int64, _p]),
    "phc_gemm_image_floats": (C.c_int64, [C.c_int32, C.c_int32]),
    "phc_gemm_make_images": (C.c_int, [C.POINTER(PhcGemmImageDesc), C.c_int32, _p]),
    "phc_gemm_tc5s": (C.c_int, [_p, C.c_int64, C.c_int32, _p, C.c_int64, C.c_int32, _p, C.c_int64, C.c_int32, C.c_int32,
                                C.c_int32, C.c_float, _p, C.c_int32, _p, C.c_int64, C.c_int32, C.c_int32, _p]),
    "phc_gemm_tc5s_set_ctas": (C.c_int, [C.c_int32]),
    "phc_gemm_tc5s_set_sched": (C.c_int, [C.c_int32]),
    "phc_gemm_tc5s_set_tile": (C.c_int, [C.c_int32]),
    "phc_gemm_set_precision": (C.c_int, [C.c_int32]),
    "phc_colsum_group": (C.c_int, [C.POINTER(PhcColsumDesc), C.c_int32, _p]),
    "phc_colsum": (C.c_int, [_p, C.c_int64, C.c_int32, C.c_int32, C.c_float, _p, C.c_int32, _p]),
    "phc_rms_apply": (C.c_int, [_p, C.c_int64, C.c_int64, C.c_int32, _p, _p, C.c_float, C.c_int32, _p, C.c_int64, _p, _p]),
    "phc_rms_apply_update": (C.c_int, [_p, C.c_int64, C.c_int64, C.c_int32, _p, _p, C.c_float, _p, C.c_int64, _p, _p, _p, _p, _p, _p]),
    "phc_rms_workspace_bytes": (C.c_int64, [C.c_int32]),
    "phc_rms_update": (C.c_int, [_p, C.c_int64, C.c_int64, C.c_int32, _p, _p, _p, _p, _p, _p]),
    "phc_gaussian_sample": (C.c_int, [_p, C.c_int64, _p, _p, C.c_int64, C.c_int32, _p, _p, _p, _p, _p]),
    "phc_ppo_actor_grad": (C.c_int, [_p, C.c_int64, _p, _p, _p, _p, _p, _p, C.c_int64, C.c_int32, C.c_float, C.c_float,
                                     C.c_float, _p, C.c_int64, _p, _p]),
    "phc_ppo_grads_gather": (C.c_int, [_p, C.c_int64, _p, _p, _p, _p, _p, _p, _p, C.c_int64, _p, _p, C.c_int64, C.c_int32, C.c_float, C.c_float,
                                       C.c_float, C.c_float, _p, C.c_int64, _p, C.c_int64, _p, _p]),
    "phc_ppo_critic_grad": (C.c_int, [_p, C.c_int64, _p, C.c_int64, C.c_float, C.c_float, _p, C.c_int64, _p, _p]),
    "phc_disc_logit_grad": (C.c_int, [_p, C.c_int64, C.c_int64, C.c_int64, C.c_float, _p, C.c_int64, _p, _p]),
    "phc_disc_reward": (C.c_int, [_p, C.c_int64, _p, C.c_int64, C.c_float, C.c_float, C.c_float, _p, _p, _p]),
    "phc_relu_mask_row": (C.c_int, [_p, C.c_int64, _p, C.c_int64, C.c_int32, _p, C.c_int64, _p]),
    "phc_scale_sumsq": (C.c_int, [_p, C.c_int64, C.c_int64, C.c_int32, C.c_float, _p, _p]),
    "phc_axpy2d": (C.c_int, [_p, C.c_int64, _p, C.c_int64, C.c_int64, C.c_int32, C.c_float, _p, _p]),
    "phc_mcp_combine": (C.c_int, [_p, C.c_int64, _p, C.c_int64, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_int32, _p, C.c_int64, _p]),
    "phc_pd_targets": (C.c_int, [_p, C.c_int64, C.c_int64, C.c_int32, C.c_int32, _p, _p, _p, _p, _p, C.c_int64, _p]),
    "phc_act_backward": (C.c_int, [_p, C.c_int64, _p, C.c_int64, C.c_int64, C.c_int32, C.c_int32, _p]),
    "phc_grad_sumsq": (C.c_int, [_p, C.c_int64, _p, _p]),
    "phc_adam_step": (C.c_int, [_p, _p, _p, _p, C.c_int64, _p, C.c_float, C.c_float, C.c_float, C.c_float, C.c_float,
                                C.c_float, C.c_int64, _p]),
}

_lib = None


def load() -> C.CDLL:
    """Load (once) and type the shared library.  No fallback: a missing library is an error."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(f"{LIB_PATH} is missing -- build it with `python -m phc_b200.build` "
                          f"(or __graft_entry__.build()); phc_b200 has no CPU / PyTorch fallback path")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)      # AttributeError here = header and library out of sync
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = load().phc_last_error().decode(errors="replace")
        raise PhcError(f"{what or 'phc call'} failed with code {rc}: {msg}")
