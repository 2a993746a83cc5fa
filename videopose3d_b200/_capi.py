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
VP3D_PACK_CONV = 1
VP3D_PACK_BN_EVAL = 2
VP3D_PACK_CONV_T = 4
VP3D_SEMI_POS, VP3D_SEMI_TRAJ, VP3D_SEMI_PROJ, VP3D_SEMI_BONE = 1, 2, 4, 8
VP3D_EVAL_MPJPE, VP3D_EVAL_P_MPJPE, VP3D_EVAL_N_MPJPE, VP3D_EVAL_VELOCITY = 1, 2, 4, 8

_LIB_NAME = "libvp3d_b200.so"
_LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_lib", _LIB_NAME)
# development hook: another build of the same library (the time-stamping `make dbg` build that
# tools/timeline.py drives); never a different implementation
_LIB_PATH = os.environ.get("VP3D_LIB_PATH", _LIB_PATH)

c_float_p = ctypes.POINTER(ctypes.c_float)
STAGE_FN = ctypes.CFUNCTYPE(None, ctypes.c_int, ctypes.c_void_p)


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
    ]


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
    "vp3d_last_launch_count": (ctypes.c_int, [ctypes.c_void_p]),
    "vp3d_profile_launch": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int]),
    "vp3d_profile_read": (ctypes.c_int, [ctypes.c_void_p, ctypes.POINTER(ctypes.c_float),
                                         ctypes.POINTER(ctypes.c_int)]),
    "vp3d_conv_gemm": (ctypes.c_int, [ctypes.POINTER(ConvDesc), ctypes.c_void_p]),
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
    "vp3d_pose_errors_scratch_bytes": (ctypes.c_size_t, [ctypes.c_int64]),
    "vp3d_pose_errors": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int32, ctypes.c_void_p,
                                        ctypes.c_void_p, ctypes.c_int64, ctypes.c_int32,
                                        ctypes.c_int32, ctypes.c_void_p, ctypes.c_void_p,
                                        ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
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
