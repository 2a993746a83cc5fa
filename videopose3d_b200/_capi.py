"""ctypes binding of the C-ABI library ``libvp3d_b200.so`` (see ``include/vp3d_b200.h``).

The shared library is the product; this module only mirrors its structs and turns negative status
codes into Python exceptions.  There is deliberately no fallback: if the library is missing the
import of the model classes still works (so ``state_dict`` handling can be unit-tested on CPU) but
every compute call raises ``RuntimeError``.
"""
import ctypes
import os

VP3D_MAX_WIDTHS = 8
VP3D_MAX_LAYERS = 2 * (VP3D_MAX_WIDTHS - 1)

VP3D_VARIANT_DILATED = 0
VP3D_VARIANT_STRIDED = 1
VP3D_PRECISION_BF16 = 0
VP3D_PRECISION_BF16X3 = 1
VP3D_PRECISION_MIXED = 2
VP3D_PRECISION_FP16 = 3
VP3D_PRECISION_INT8 = 4
VP3D_PACK_CONV = 1
VP3D_PACK_BN_EVAL = 2
VP3D_PACK_CONV_T = 4
VP3D_PACK_EXPAND_T = 8
VP3D_TRAIN_FROZEN_BN = 1
VP3D_BN_SYNC_FORWARD, VP3D_BN_SYNC_BACKWARD = 0, 1
VP3D_SEMI_POS, VP3D_SEMI_TRAJ, VP3D_SEMI_PROJ, VP3D_SEMI_BONE = 1, 2, 4, 8
VP3D_EVAL_MPJPE, VP3D_EVAL_P_MPJPE, VP3D_EVAL_N_MPJPE, VP3D_EVAL_VELOCITY = 1, 2, 4, 8
VP3D_POSE_LOSS_MPJPE, VP3D_POSE_LOSS_N_MPJPE, VP3D_POSE_LOSS_P_MPJPE, VP3D_POSE_LOSS_VELOCITY = 1, 2, 4, 8
VP3D_STREAM_AUGMENT = 1
VP3D_STREAM_PROVISIONAL = 4
VP3D_STREAM_INT8 = 16
VP3D_STREAM_HELD = 64
VP3D_CLIPS_AUGMENT = 1
VP3D_INT8_CALIB_AMAX, VP3D_INT8_CALIB_PERCENTILE, VP3D_INT8_CALIB_MSE = 0, 1, 2

_LIB_NAME = "libvp3d_b200.so"
_LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_lib", _LIB_NAME)
# development hook: another build of the same library (the time-stamping `make dbg` build that
# tools/timeline.py drives); never a different implementation
_LIB_PATH = os.environ.get("VP3D_LIB_PATH", _LIB_PATH)

c_float_p = ctypes.POINTER(ctypes.c_float)
STAGE_FN = ctypes.CFUNCTYPE(None, ctypes.c_int, ctypes.c_void_p)
# vp3d_bn_exchange_fn(layer, phase, slots, floats_per_rank, user)
BN_EXCHANGE_FN = ctypes.CFUNCTYPE(None, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int,
                                  ctypes.c_void_p)


class Config(ctypes.Structure):
    _fields_ = [
        ("num_joints_in", ctypes.c_int),
        ("in_features", ctypes.c_int),
        ("num_joints_out", ctypes.c_int),
        ("num_widths", ctypes.c_int),
        ("filter_widths", ctypes.c_int * VP3D_MAX_WIDTHS),
        ("causal", ctypes.c_int),
        ("channels", ctypes.c_int),
        ("dense", ctypes.c_int),
        ("variant", ctypes.c_int),
        ("precision", ctypes.c_int),
    ]


class Weights(ctypes.Structure):
    _fields_ = [
        ("expand_conv_weight", ctypes.c_void_p),
        ("expand_bn", ctypes.c_void_p * 4),
        ("layers_conv_weight", ctypes.c_void_p * VP3D_MAX_LAYERS),
        ("layers_bn", (ctypes.c_void_p * 4) * VP3D_MAX_LAYERS),
        ("shrink_weight", ctypes.c_void_p),
        ("shrink_bias", ctypes.c_void_p),
    ]


class Grads(ctypes.Structure):
    _fields_ = [
        ("expand_conv_weight", ctypes.c_void_p),
        ("expand_bn", ctypes.c_void_p * 2),
        ("layers_conv_weight", ctypes.c_void_p * VP3D_MAX_LAYERS),
        ("layers_bn", (ctypes.c_void_p * 2) * VP3D_MAX_LAYERS),
        ("shrink_weight", ctypes.c_void_p),
        ("shrink_bias", ctypes.c_void_p),
    ]


class AdamTensor(ctypes.Structure):
    """vp3d_adam_tensor (include/vp3d_b200.h)."""
    _fields_ = [
        ("param", ctypes.c_void_p),
        ("grad", ctypes.c_void_p),
        ("exp_avg", ctypes.c_void_p),
        ("exp_avg_sq", ctypes.c_void_p),
        ("max_exp_avg_sq", ctypes.c_void_p),
        ("numel", ctypes.c_int64),
    ]


class GatherDesc(ctypes.Structure):
    """vp3d_gather_desc (include/vp3d_b200.h)."""
    _fields_ = [
        ("src", ctypes.c_void_p),
        ("seq_first", ctypes.c_void_p),
        ("seq_len", ctypes.c_void_p),
        ("rows", ctypes.c_void_p),
        ("src_joint", ctypes.c_void_p),
        ("out", ctypes.c_void_p),
        ("n_windows", ctypes.c_int32),
        ("frames", ctypes.c_int32),
        ("joints", ctypes.c_int32),
        ("features", ctypes.c_int32),
        ("first_offset", ctypes.c_int32),
    ]


class ConvDesc(ctypes.Structure):
    _fields_ = [
        ("a", ctypes.c_void_p),
        ("a_planes", ctypes.c_int),
        ("samples", ctypes.c_int),
        ("a_rows", ctypes.c_int),
        ("a_ld", ctypes.c_int),
        ("w", ctypes.c_void_p),
        ("taps", ctypes.c_int),
        ("k_per_tap", ctypes.c_int),
        ("n_pad", ctypes.c_int),
        ("per_sample_tiles", ctypes.c_int),
        ("tap_row_step", ctypes.c_int),
        ("tap_col_step", ctypes.c_int),
        ("out_rows", ctypes.c_int),
        ("precision", ctypes.c_int),
        ("scale", ctypes.c_void_p),
        ("shift", ctypes.c_void_p),
        ("relu", ctypes.c_int),
        ("res", ctypes.c_void_p),
        ("res_planes", ctypes.c_int),
        ("res_plane_stride", ctypes.c_longlong),
        ("res_ld", ctypes.c_int),
        ("res_rows_per_sample", ctypes.c_int),
        ("res_row_step", ctypes.c_int),
        ("res_row_off", ctypes.c_int),
        ("res_sample_div", ctypes.c_int),
        ("res_col_begin", ctypes.c_int),
        ("res_cols", ctypes.c_int),
        ("res_check_rows", ctypes.c_int),
        ("out", ctypes.c_void_p),
        ("out_planes", ctypes.c_int),
        ("out_plane_stride", ctypes.c_longlong),
        ("out_ld", ctypes.c_int),
        ("out_f32", ctypes.c_void_p),
        ("out_f32_ld", ctypes.c_int),
        ("n_valid", ctypes.c_int),
        ("stats", ctypes.c_void_p),
        ("bnb_z", ctypes.c_void_p),
        ("bnb_scale", ctypes.c_void_p),
        ("bnb_shift", ctypes.c_void_p),
        ("bnb_mean", ctypes.c_void_p),
        ("bnb_invstd", ctypes.c_void_p),
        ("bnb_sums", ctypes.c_void_p),
        ("bnb_c", ctypes.c_int),
        ("bnb_p", ctypes.c_float),
        ("bnb_seed", ctypes.c_ulonglong),
        ("bnb_layer", ctypes.c_int),
        ("lo_row_begin", ctypes.c_int),
        ("lo_row_end", ctypes.c_int),
        ("a_plane_stride", ctypes.c_longlong),
        ("out_u8", ctypes.c_void_p),
        ("out_u8_ld", ctypes.c_int),
        ("out_u8_inv_scale", ctypes.c_float),
    ]


class WgradDesc(ctypes.Structure):
    """vp3d_wgrad_desc (include/vp3d_b200.h)."""
    _fields_ = [
        ("dz", ctypes.c_void_p),
        ("dz_ld", ctypes.c_int),
        ("x", ctypes.c_void_p),
        ("x_ld", ctypes.c_int),
        ("planes", ctypes.c_int),
        ("rows", ctypes.c_longlong),
        ("per_sample", ctypes.c_int),
        ("samples", ctypes.c_int),
        ("x_rows", ctypes.c_longlong),
        ("taps", ctypes.c_int),
        ("tap_row_step", ctypes.c_int),
        ("tap_col_step", ctypes.c_int),
        ("c_out", ctypes.c_int),
        ("c_in_cols", ctypes.c_int),
        ("c_in", ctypes.c_int),
        ("taps_out", ctypes.c_int),
        ("merged", ctypes.c_int),
        ("grad", ctypes.c_void_p),
        ("partial", ctypes.c_void_p),
        ("partial_bytes", ctypes.c_size_t),
    ]


class StreamSlotsHeader(ctypes.Structure):
    """vp3d_stream_slots_header: what vp3d_stream_import checks of a slot blob on the host."""
    _fields_ = [
        ("version", ctypes.c_int32),
        ("n", ctypes.c_int32),
        ("cfg", Config),
        ("flags", ctypes.c_int32),
        ("rings", ctypes.c_int32),
        ("planes", ctypes.c_int32),
        ("f16", ctypes.c_int32),
        ("lookahead", ctypes.c_int32),
        ("H", ctypes.c_int32 * VP3D_MAX_WIDTHS),
        ("ld", ctypes.c_int32 * VP3D_MAX_WIDTHS),
        ("int8_snap", ctypes.c_int32),
        ("int8_mask", ctypes.c_uint32),
        ("act_scale", ctypes.c_float * VP3D_MAX_LAYERS),
        ("slot_bytes", ctypes.c_int64),
    ]


_P, _I, _LL, _F, _SZ = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong, ctypes.c_float, ctypes.c_size_t

# name -> (restype, argtypes); also the list the CPU test checks against include/vp3d_b200.h
SIGNATURES = {
    "vp3d_version": (ctypes.c_int, []),
    "vp3d_last_error": (ctypes.c_char_p, []),
    "vp3d_set_sm_limit": (ctypes.c_int, [ctypes.c_int]),
    "vp3d_set_pdl": (ctypes.c_int, [ctypes.c_int]),
    "vp3d_plan_create": (ctypes.c_int, [ctypes.POINTER(Config), ctypes.POINTER(ctypes.c_void_p)]),
    "vp3d_plan_destroy": (None, [ctypes.c_void_p]),
    "vp3d_receptive_field": (ctypes.c_int, [ctypes.c_void_p]),
    "vp3d_total_causal_shift": (ctypes.c_int, [ctypes.c_void_p]),
    "vp3d_set_weights": (ctypes.c_int, [ctypes.c_void_p, ctypes.POINTER(Weights), ctypes.c_int,
                                        ctypes.c_void_p]),
    "vp3d_output_frames": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int]),
    "vp3d_workspace_bytes": (ctypes.c_size_t, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int]),
    "vp3d_forward_eval": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                         ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                         ctypes.c_size_t, ctypes.c_void_p]),
    "vp3d_calibrate_int8": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int,
                                           ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t,
                                           ctypes.c_void_p, ctypes.c_void_p]),
    "vp3d_int8_hist_bytes": (ctypes.c_size_t, [ctypes.c_void_p]),
    "vp3d_calibrate_int8_hist": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int,
                                                ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t,
                                                ctypes.c_void_p, ctypes.c_void_p]),
    "vp3d_int8_thresholds_scratch_bytes": (ctypes.c_size_t, [ctypes.c_int]),
    "vp3d_int8_thresholds": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                                            ctypes.c_double, ctypes.c_void_p, ctypes.c_void_p,
                                            ctypes.c_size_t, ctypes.c_void_p]),
    "vp3d_set_int8_scales": (ctypes.c_int, [ctypes.c_void_p, ctypes.POINTER(ctypes.c_float),
                                            ctypes.c_int]),
    "vp3d_set_int8_blocks": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_uint32]),
    "vp3d_int8_packs": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p,
                                       ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "vp3d_forward_eval_host": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                              ctypes.c_int, ctypes.c_int]),
    "vp3d_forward_eval_host_submit": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p,
                                                     ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                                                     ctypes.c_int]),
    "vp3d_forward_eval_host_wait": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int]),
    "vp3d_train_workspace_bytes": (ctypes.c_size_t, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int]),
    "vp3d_forward_train": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                          ctypes.c_int, ctypes.c_int, ctypes.POINTER(Weights),
                                          ctypes.POINTER(ctypes.c_float), ctypes.c_float,
                                          ctypes.c_ulonglong, ctypes.c_void_p, ctypes.c_size_t,
                                          ctypes.c_void_p]),
    "vp3d_backward": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.POINTER(Grads),
                                     ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
    "vp3d_backward_staged": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.POINTER(Grads),
                                            ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p,
                                            ctypes.c_void_p, ctypes.c_void_p]),
    "vp3d_forward_train_ex": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                             ctypes.c_int, ctypes.c_int, ctypes.POINTER(Weights),
                                             ctypes.POINTER(ctypes.c_float), ctypes.c_float,
                                             ctypes.c_ulonglong, ctypes.c_int, ctypes.c_void_p,
                                             ctypes.c_size_t, ctypes.c_void_p]),
    "vp3d_backward_ex": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.POINTER(Grads),
                                        ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t,
                                        ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "vp3d_set_bn_sync": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                        ctypes.c_void_p]),
    "vp3d_last_launch_count": (ctypes.c_int, [ctypes.c_void_p]),
    "vp3d_profile_launch": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int]),
    "vp3d_profile_read": (ctypes.c_int, [ctypes.c_void_p, ctypes.POINTER(ctypes.c_float),
                                         ctypes.POINTER(ctypes.c_int)]),
    "vp3d_conv_gemm": (ctypes.c_int, [ctypes.POINTER(ConvDesc), ctypes.c_void_p]),
    "vp3d_conv_gemm_instance": (ctypes.c_int, [ctypes.POINTER(ConvDesc),
                                               ctypes.POINTER(ctypes.c_int)]),
    "vp3d_conv_gemm_instances": (ctypes.c_int, [ctypes.POINTER(ctypes.c_int), ctypes.c_int]),
    "vp3d_wgrad_gemm": (ctypes.c_int, [ctypes.POINTER(WgradDesc), ctypes.c_void_p]),
    "vp3d_bn_stats_finalize": (_I, [_P, _I, _I, _I, _I, _P, _P, _P, _P, _F, _F, _P, _P, _P, _P, _I,
                                    _I, _P, _SZ, _P, _I, _P]),
    "vp3d_ordered_col_sums": (_I, [_P, _I, _I, _I, _I, _I, _P, _P, _P, _P, _P, _SZ, _P, _I, _P]),
    "vp3d_bn_apply": (_I, [_P, _LL, _P, _LL, _I, _LL, _I, _P, _P, _F, ctypes.c_ulonglong, _I, _P,
                           _LL, _I, _I, _I, _I, _P]),
    "vp3d_bn_bwd_reduce": (_I, [_P, _LL, _P, _LL, _I, _LL, _I, _P, _P, _P, _P, _F,
                                ctypes.c_ulonglong, _I, _P, _SZ, _P, _P, _SZ, _P, _I, _P]),
    "vp3d_bn_bwd_apply": (_I, [_P, _LL, _P, _LL, _P, _LL, _I, _LL, _I, _P, _P, _P, _P, _F,
                               ctypes.c_ulonglong, _I, _P, _P, _P, _I, _I, _P]),
    "vp3d_gather_windows": (ctypes.c_int, [ctypes.POINTER(GatherDesc), ctypes.c_void_p]),
    "vp3d_gather_cameras": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int32, ctypes.c_void_p,
                                           ctypes.c_int32, ctypes.c_void_p, ctypes.c_void_p]),
    "vp3d_adam_step": (ctypes.c_int, [ctypes.POINTER(AdamTensor), ctypes.c_int32, ctypes.c_int64,
                                      ctypes.c_double, ctypes.c_double, ctypes.c_double,
                                      ctypes.c_double, ctypes.c_double, ctypes.c_void_p]),
    "vp3d_adam_step_packed": (ctypes.c_int, [ctypes.c_void_p, ctypes.POINTER(Weights),
                                             ctypes.POINTER(AdamTensor), ctypes.c_int32, ctypes.c_int64,
                                             ctypes.c_double, ctypes.c_double, ctypes.c_double,
                                             ctypes.c_double, ctypes.c_double, ctypes.c_void_p]),
    "vp3d_projected_mpjpe_fwd_bwd": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                                    ctypes.c_void_p, ctypes.c_int64, ctypes.c_int32,
                                                    ctypes.c_int32, ctypes.c_int32, ctypes.c_void_p,
                                                    ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "vp3d_semi_loss_scratch_bytes": (ctypes.c_size_t, []),
    "vp3d_semi_loss_fwd_bwd": (ctypes.c_int, [ctypes.c_void_p] * 6 + [ctypes.c_int64, ctypes.c_int64]
                               + [ctypes.c_int32] * 4 + [ctypes.c_void_p] * 4
                               + [ctypes.c_size_t, ctypes.c_void_p]),
    "vp3d_mpjpe_fwd_bwd": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                          ctypes.c_int64, ctypes.c_int32, ctypes.c_void_p,
                                          ctypes.c_void_p, ctypes.c_void_p]),
    "vp3d_mpjpe_scratch_bytes": (ctypes.c_size_t, [ctypes.c_int64]),
    "vp3d_mpjpe_fwd_bwd_ex": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                             ctypes.c_int64, ctypes.c_int32, ctypes.c_void_p,
                                             ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t,
                                             ctypes.c_void_p]),
    "vp3d_projected_mpjpe_scratch_bytes": (ctypes.c_size_t, [ctypes.c_int64, ctypes.c_int32]),
    "vp3d_projected_mpjpe_fwd_bwd_ex": (ctypes.c_int, [ctypes.c_void_p] * 4
                                        + [ctypes.c_int64, ctypes.c_int32, ctypes.c_int32,
                                           ctypes.c_int32] + [ctypes.c_void_p] * 4
                                        + [ctypes.c_size_t, ctypes.c_void_p]),
    "vp3d_pose_errors_scratch_bytes": (ctypes.c_size_t, [ctypes.c_int64]),
    "vp3d_pose_errors": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int32, ctypes.c_void_p,
                                        ctypes.c_void_p, ctypes.c_int64, ctypes.c_int32,
                                        ctypes.c_int32, ctypes.c_void_p, ctypes.c_void_p,
                                        ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
    "vp3d_pose_loss_scratch_bytes": (ctypes.c_size_t, [ctypes.c_int32, ctypes.c_int64]),
    "vp3d_pose_loss_fwd_bwd": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int32,
                                              ctypes.c_int64, ctypes.c_int32,
                                              ctypes.POINTER(ctypes.c_double)] + [ctypes.c_void_p] * 5
                               + [ctypes.c_size_t, ctypes.c_void_p]),
    "vp3d_stream_lookahead": (ctypes.c_int, [ctypes.c_void_p]),
    "vp3d_stream_state_bytes": (ctypes.c_size_t, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int]),
    "vp3d_stream_init": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t,
                                        ctypes.c_int, ctypes.c_int, ctypes.c_void_p]),
    "vp3d_stream_state_bytes_ex": (ctypes.c_size_t, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                                                     ctypes.c_int]),
    "vp3d_stream_init_ex": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t,
                                           ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                           ctypes.c_void_p, ctypes.c_void_p]),
    "vp3d_stream_push": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                        ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p,
                                        ctypes.c_void_p, ctypes.c_void_p]),
    "vp3d_stream_push_ex": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                           ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p,
                                           ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                           ctypes.c_void_p, ctypes.c_void_p]),
    "vp3d_stream_push_counts": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                               ctypes.c_int] + [ctypes.c_void_p] * 8),
    "vp3d_stream_push_provisional": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p,
                                                    ctypes.c_void_p, ctypes.c_int]
                                     + [ctypes.c_void_p] * 8),
    "vp3d_stream_push_held": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                             ctypes.c_int] + [ctypes.c_void_p] * 4
                              + [ctypes.c_int, ctypes.c_int] + [ctypes.c_void_p] * 5),
    "vp3d_stream_finish": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                          ctypes.c_void_p, ctypes.c_void_p]),
    "vp3d_stream_release": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p]),
    "vp3d_stream_slot_bytes": (ctypes.c_size_t, [ctypes.c_void_p, ctypes.c_int]),
    "vp3d_stream_export": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                          ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t,
                                          ctypes.POINTER(StreamSlotsHeader), ctypes.c_void_p]),
    "vp3d_stream_import": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                          ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t,
                                          ctypes.POINTER(StreamSlotsHeader), ctypes.c_void_p]),
    "vp3d_stream_pack_detections": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int,
                                                   ctypes.c_int, ctypes.c_void_p, ctypes.c_int64,
                                                   ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p,
                                                   ctypes.c_void_p]),
    "vp3d_clips_workspace_bytes": (ctypes.c_size_t, [ctypes.c_void_p, ctypes.c_int64, ctypes.c_int]),
    "vp3d_forward_clips": (ctypes.c_int, [ctypes.c_void_p] * 4 + [ctypes.c_int, ctypes.c_int64,
                                                                  ctypes.c_int]
                           + [ctypes.c_void_p] * 5 + [ctypes.c_size_t, ctypes.c_void_p]),
}

_lib = None
_load_error = None


def lib_path():
    return _LIB_PATH


def load():
    """Load the shared library once; raise RuntimeError (never fall back) if it is unavailable."""
    global _lib, _load_error
    if _lib is not None:
        return _lib
    if _load_error is not None:
        raise RuntimeError(_load_error)
    if not os.path.exists(_LIB_PATH):
        _load_error = (f"{_LIB_PATH} not found: build it with `make` (or "
                       f"`python -c 'import __graft_entry__ as g; g.build()'`); "
                       "videopose3d_b200 has no CPU / PyTorch fallback")
        raise RuntimeError(_load_error)
    try:
        lib = ctypes.CDLL(_LIB_PATH)
    except OSError as e:  # pragma: no cover - depends on the machine
        _load_error = f"failed to load {_LIB_PATH}: {e}"
        raise RuntimeError(_load_error)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(status, what):
    if status == 0:
        return
    msg = load().vp3d_last_error().decode("utf-8", "replace")
    if status == -1:
        raise ValueError(f"{what}: {msg}")
    if status == -2:
        raise NotImplementedError(f"{what}: {msg}")
    raise RuntimeError(f"{what}: {msg} (status {status})")
