"""ctypes binding of libsegtran_b200.so (the C ABI declared in include/segtran_b200.h).

The library is built in-tree by ``__graft_entry__.build()`` / ``make``.  There is no fallback:
if the shared object is missing or a call fails, an exception is raised.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libsegtran_b200.so")

SX_F32, SX_BF16 = 0, 1
SX_OP_TF32, SX_OP_BF16 = 0, 1
SX_MAJOR_K, SX_MAJOR_MN = 0, 1
SX_BIAS_NONE, SX_BIAS_N, SX_BIAS_M = 0, 1, 2
SX_ACT_NONE, SX_ACT_GELU, SX_ACT_GELU_BWD = 0, 1, 2
SX_SCHED_WARMUP_LINEAR, SX_SCHED_WARMUP_CONSTANT = 0, 1
SX_CONSIST_BCE, SX_CONSIST_MARGIN = 0, 1
SX_HEAD_DMAP_NONE, SX_HEAD_DMAP_INTERP, SX_HEAD_DMAP_UNFOLD, SX_HEAD_DMAP_UNFOLD_INTERLEAVED = 0, 1, 2, 3
SX_HEAD_SRC_DEPTH_MAJOR, SX_HEAD_SRC_SLICE_MAJOR = 0, 1
SX_LABEL_U8, SX_LABEL_I16, SX_LABEL_I32, SX_LABEL_I64, SX_LABEL_F32 = 0, 1, 2, 3, 4


class SxError(RuntimeError):
    pass


class sx_operand(C.Structure):
    _fields_ = [("ptr", C.c_void_p), ("major", C.c_int32), ("_pad", C.c_int32), ("ld", C.c_int64),
                ("stride_z0", C.c_int64), ("stride_z1", C.c_int64)]


class sx_gemm_args(C.Structure):
    _fields_ = [("op_dtype", C.c_int32), ("M", C.c_int32), ("N", C.c_int32), ("K", C.c_int32), ("Z0", C.c_int32),
                ("Z1", C.c_int32), ("A", sx_operand), ("B", sx_operand), ("C", C.c_void_p), ("c_dtype", C.c_int32),
                ("round_tf32", C.c_int32), ("ldc", C.c_int64), ("c_stride_z0", C.c_int64), ("c_stride_z1", C.c_int64),
                ("alpha", C.c_float), ("bias_mode", C.c_int32), ("bias", C.c_void_p), ("bias_stride_z0", C.c_int64),
                ("bias_stride_z1", C.c_int64), ("act", C.c_int32), ("accumulate", C.c_int32), ("preact", C.c_void_p),
                ("split_k", C.c_int32), ("_pad2", C.c_int32), ("amax", C.c_void_p), ("drop_p", C.c_float),
                ("_pad3", C.c_uint32), ("drop_seed", C.c_uint64), ("drop_seed_dev", C.c_void_p), ("addend", C.c_void_p),
                ("part", C.c_void_p), ("part_floats", C.c_int64)]


class sx_gemm_tout(C.Structure):
    _fields_ = [("ct", C.c_void_p), ("ldct", C.c_int64), ("ct_stride_z0", C.c_int64), ("ct_stride_z1", C.c_int64)]


class sx_sw_weights(C.Structure):
    _fields_ = [("wx", C.c_void_p), ("wy", C.c_void_p), ("wz", C.c_void_p), ("nx", C.c_int32), ("ny", C.c_int32),
                ("nz", C.c_int32), ("_pad", C.c_int32)]


class sx_posbias(C.Structure):
    _fields_ = [("table", C.c_void_p), ("pd", C.c_int32), ("R", C.c_int32), ("grid", C.c_int32 * 3), ("w", C.c_float)]


class sx_attn_probs_args(C.Structure):
    _fields_ = [("B", C.c_int32), ("M", C.c_int32), ("U1", C.c_int32), ("U2", C.c_int32), ("d", C.c_int32),
                ("round_tf32", C.c_int32), ("Q", C.c_void_p), ("q_ld", C.c_int64), ("q_bstride", C.c_int64),
                ("K", C.c_void_p), ("k_ld", C.c_int64), ("k_bstride", C.c_int64), ("alpha", C.c_float),
                ("clip", C.c_float), ("P", C.c_void_p), ("S", C.c_void_p), ("ldp", C.c_int64), ("lse", C.c_void_p),
                ("rowmax", C.c_void_p), ("stat", C.c_void_p), ("diag", C.c_void_p), ("drop_p", C.c_float),
                ("_pad", C.c_uint32), ("drop_seed", C.c_uint64), ("drop_seed_dev", C.c_void_p), ("posbias", sx_posbias)]


class sx_attn_probs_tout(C.Structure):
    _fields_ = [("pt", C.c_void_p), ("ldpt", C.c_int64)]


class sx_consist_args(C.Structure):
    _fields_ = [("B", C.c_int32), ("N", C.c_int32), ("A", C.c_int32), ("K", C.c_int32), ("variant", C.c_int32),
                ("round_r", C.c_int32), ("Xo", C.c_void_p), ("xo_ld", C.c_int64), ("xo_bstride", C.c_int64),
                ("Xt", C.c_void_p), ("xt_ld", C.c_int64), ("xt_bstride", C.c_int64), ("X", C.c_void_p),
                ("x_ld", C.c_int64), ("x_bstride", C.c_int64), ("F", C.c_void_p), ("mu", C.c_void_p), ("R", C.c_void_p),
                ("ldr", C.c_int64), ("out", C.c_void_p), ("cap", C.c_void_p), ("cap_scale", C.c_float),
                ("_pad", C.c_int32), ("part", C.c_void_p), ("part_floats", C.c_int64)]


class sx_head_dropout_args(C.Structure):
    _fields_ = [("src", C.c_void_p), ("B", C.c_int32), ("Fs", C.c_int32), ("Ds", C.c_int32), ("Fo", C.c_int32),
                ("HW", C.c_int64), ("Dk", C.c_int32), ("dmap", C.c_int32), ("K", C.c_int32), ("src_layout", C.c_int32),
                ("Wc", C.c_void_p), ("bc", C.c_void_p), ("p", C.c_float), ("_pad2", C.c_uint32), ("seed", C.c_uint64),
                ("seed_dev", C.c_void_p), ("part", C.c_void_p), ("part_floats", C.c_int64)]


class sx_resample_grid(C.Structure):
    _fields_ = [("lin", C.c_int32 * 3), ("lout", C.c_int32 * 3), ("ratio", C.c_float * 3)]


class sx_crop_operand(C.Structure):
    _fields_ = [("x", C.c_void_p), ("stride", C.c_int64 * 5), ("y", C.c_void_p), ("C", C.c_int32), ("_pad", C.c_int32)]


_P, _I, _L, _F, _U64, _D = C.c_void_p, C.c_int32, C.c_int64, C.c_float, C.c_uint64, C.c_double

# name -> argtypes (every function returns int; 0 = success)
_PROTOS = {
    "sx_gemm": [C.POINTER(sx_gemm_args), C.POINTER(sx_gemm_tout), _P],
    "sx_gemm_debug_set": [C.c_char_p, _L],
    "sx_attn_probs_fwd": [C.POINTER(sx_attn_probs_args), C.POINTER(sx_attn_probs_tout), _P],
    "sx_attn_consist_fwd": [C.POINTER(sx_consist_args), _P],
    "sx_attn_consist_bwd": [C.POINTER(sx_consist_args), _P, _P, _I, _I, _L, _L, _P, _P, _P, _L, _L, _P],
    "sx_clamp_if": [_P, _L, _I, _L, _P, _F, _P, _L, _P, _L, _P],
    "sx_reduce_max": [_P, _L, _P, _P],
    "sx_pos_lsinu_fwd": [_P, _P, _L, _I, _P, _P, _I, _P, _P],
    "sx_pos_lsinu_bwd": [_P, _P, _L, _I, _P, _P, _I, _P, _P, _P, _P, _P, _L, _P],
    "sx_prologue_fwd": [_P, _L, _I, _I, _P, _P, _P, _I, _L, _F, _P, _F, _U64, _P, _P, _I, _P, _P],
    "sx_prologue_bwd": [_P, _P, _L, _I, _I, _P, _P, _P, _I, _L, _F, _P, _F, _U64, _P, _P, _P, _P, _P, _P, _P, _P, _L, _P],
    "sx_softmax_fwd": [_P, _L, _I, _L, _P, _F, _F, _U64, _P, _P, _L, _I, _P, _P, _P],
    "sx_softmax_bwd": [_P, _L, _P, _L, _P, _L, _I, _P, _F, _F, _U64, _P, _L, _P, _L, _I, _P],
    "sx_softmax_posbias_fwd": [_P, _L, _I, _L, _P, _F, _F, _U64, _P, _P, _L, _I, _P, _P, C.POINTER(sx_posbias), _P],
    "sx_softmax_posbias_bwd": [_P, _L, _P, _L, _P, _L, _I, _P, _F, _F, _U64, _P, _L, _P, _L, _I, C.POINTER(sx_posbias),
                               _P, _P, _L, _P],
    "sx_layernorm_fwd": [_P, _L, _I, _P, _P, _P, _I, _P, _P],
    "sx_layernorm_bwd": [_P, _P, _L, _I, _P, _P, _P, _I, _P, _P, _P, _L, _P],
    "sx_ln_softaggr_fwd": [_P, _I, _I, _I, _I, _P, _P, _P, _P, _F, _U64, _P, _P, _P, _P, _P],
    "sx_ln_softaggr_bwd": [_P, _P, _I, _I, _I, _I, _P, _P, _P, _F, _U64, _P, _P, _P, _P, _I, _P, _P, _P, _P, _P, _L, _P],
    "sx_softaggr_fwd": [_P, _I, _I, _I, _I, _P, _P, _P, _P, _P],
    "sx_softaggr_bwd": [_P, _P, _I, _I, _I, _I, _P, _P, _P, _P, _P],
    "sx_gelu_bwd": [_P, _P, _L, _F, _U64, _P, _P, _I, _P],
    "sx_seed_derive": [_P, _U64, _P, _P],
    "sx_seed_advance": [_P, _U64, _P],
    "sx_convert": [_P, _I, _L, _P, _I, _I, _P],
    "sx_sw_accumulate": [_P, _I, _I, _I, _I, _P, _P, _I, _I, _I, _I, _I, _I, _I, C.POINTER(sx_sw_weights), _P],
    "sx_sw_finalize": [_P, _P, _I, _L, _I, _P, _P],
    "sx_sw_gather": [_P, _I, _I, _I, _I, _I, _P, _I, _I, _I, _I, _I, _P, _P],
    "sx_sw2d_accumulate": [_P, _I, _I, _I, _I, _I, _I, _P, _P, _I, _I, _I, _I, _I, C.POINTER(sx_sw_weights), _P],
    "sx_sw2d_finalize": [_P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _P, _P, _P],
    "sx_eval2d_counts": [_P, _I, _I, _I, _I, _P, _I, _I, _P, _P],
    "sx_mask_counts": [_P, _P, _I, _L, _P, _L, _P],
    "sx_surface": [_P, _I, _I, _I, _I, _I, _P, _P],
    "sx_edt_sq": [_P, _I, _I, _I, _I, _P, _P],
    "sx_surface_hist": [_P, _P, _I, _L, _I, _P, _L, _P],
    "sx_surface_stats": [_P, _I, _I, _L, _P, _L, _P],
    "sx_brats_map_label": [_P, _I, _I, _L, _I, _P, _P],
    "sx_draw_resized_crop": [_P, _U64, _I, _I, _I, _I, _I, _I, _F, _F, _I, _P, _P],
    "sx_resized_crop": [C.POINTER(sx_crop_operand), C.POINTER(sx_crop_operand), _I, _I, _I, _I, _I, _I, _I, _P, _P],
    "sx_split_tf32": [_P, _L, _P, _P, _P],
    "sx_split_tf32_cat": [_P, _I, _I, _I, _I, _L, _L, _L, _L, _I, _I, _P, _P],
    "sx_transpose": [_P, _L, _I, _I, _I, _P, _P],
    "sx_colsum_batched": [_P, _I, _L, _I, _L, _L, _I, _L, _P, _P, _L, _P],
    "sx_dot": [_P, _P, _L, _P, _P, _L, _P],
    "sx_add": [_P, _P, _L, _P, _P],
    "sx_rowsum": [_P, _L, _L, _L, _I, _P, _P, _L, _P],
    "sx_scale": [_P, _L, _P, _F, _P, _P],
    "sx_head_contract_fwd": [_P, _P, _P, _I, _I, _L, _I, _P, _I, _P],
    "sx_head_contract_bwd_data": [_P, _P, _I, _I, _L, _I, _P, _P],
    "sx_head_contract_bwd_weight": [_P, _P, _I, _I, _L, _I, _P, _P, _L, _P],
    "sx_head_dropout_fwd": [C.POINTER(sx_head_dropout_args), _P, _P],
    "sx_head_dropout_bwd": [C.POINTER(sx_head_dropout_args), _P, _P, _I, _P, _P],
    "sx_token_scores": [_P, _P, _I, _I, _I, _I, _P, _P],
    "sx_token_scores_bwd": [_P, _P, _I, _I, _I, _I, _P, _P],
    "sx_subpixel_resize_fwd": [_P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _P, _P],
    "sx_subpixel_resize_bwd": [_P, _I, _I, _I, _I, _I, _I, _I, _I, _P, _P],
    "sx_resize_axis_fwd": [_P, _L, _I, _I, _L, _P, _I, _P],
    "sx_resize_axis_bwd": [_P, _L, _I, _I, _L, _P, _P],
    "sx_resize_tokens_fwd": [_P, _L, _L, _L, _P, _L, _L, _L, _I, _I, _I, _I, C.POINTER(sx_resample_grid), _I, _P],
    "sx_resize_tokens_bwd": [_P, _L, _L, _L, _P, _L, _L, _L, _I, _I, _I, _I, C.POINTER(sx_resample_grid), _I, _P],
    "sx_groupnorm_fwd": [_P, _I, _I, _L, _I, _P, _P, _F, _P, _P, _P, _I, _P],
    "sx_groupnorm_bwd": [_P, _P, _I, _I, _L, _I, _P, _P, _P, _P, _P, _P, _P, _P],
    "sx_groupnorm_slices_fwd": [_P, _I, _I, _I, _L, _I, _P, _P, _F, _P, _P, _P, _I, _P],
    "sx_groupnorm_slices_bwd": [_P, _P, _I, _I, _I, _L, _I, _P, _P, _P, _P, _P, _P, _P, _P],
    "sx_seg_loss_fwd": [_P, _P, _I, _I, _L, _P, _P, _F, _P, _P, _P, _P],
    "sx_seg_loss_bwd": [_P, _P, _I, _I, _L, _P, _P, _F, _P, _P, _P],
    "sx_adam_step": [_P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _P, _P, _D, _D, _D, _F, _F, _F, _L, _I, _P, _P, _P, _P, _P, _P],
    "sx_sgemm_small": [_P, _P, _P, _I, _I, _I, _L, _L, _L, _L, _L, _L, _I, _L, _L, _L, _F, _I, _P],
}
# every symbol include/segtran_b200.h declares (checked by tests/test_abi.py)
EXPORTS = sorted(list(_PROTOS) + ["sx_version", "sx_last_error", "sx_device_info"])

_lib = None


def lib():
    """The loaded CDLL; raises if the extension has not been built (no fallback path exists)."""
    global _lib
    if _lib is None:
        if not os.path.isfile(LIB_PATH):
            raise SxError("segtran_b200: %s is missing - run `python -c 'import __graft_entry__ as g; g.build()'` "
                          "or `make` at the repo root (there is no CPU / PyTorch fallback)" % LIB_PATH)
        l = C.CDLL(LIB_PATH)
        l.sx_version.restype = C.c_int
        l.sx_last_error.restype = C.c_char_p
        l.sx_device_info.argtypes = [C.POINTER(C.c_int)] * 3
        l.sx_device_info.restype = C.c_int
        for name, at in _PROTOS.items():
            f = getattr(l, name)
            f.argtypes = at
            f.restype = C.c_int
        _lib = l
    return _lib


def check(rc, what):
    if rc != 0:
        raise SxError("%s failed (rc=%d): %s" % (what, rc, lib().sx_last_error().decode("utf-8", "replace")))


# kernels launched per C-ABI call (for bench.py's gpu_launches claim); default 1
_LAUNCHES = {"sx_pos_lsinu_bwd": 3, "sx_ln_softaggr_bwd": 2, "sx_prologue_bwd": 3, "sx_layernorm_bwd": 3, "sx_gemm_debug_set": 0,
             "sx_attn_probs_fwd": 2, "sx_colsum_batched": 2, "sx_dot": 2, "sx_head_contract_bwd_weight": 2,
             "sx_softmax_posbias_bwd": 2, "sx_attn_consist_fwd": 2, "sx_head_dropout_bwd": 2, "sx_edt_sq": 3}
launch_count = 0
_hook = None          # optional callable(name, args) -> context manager, installed by bench.py for per-kernel timing


def set_hook(h):
    global _hook
    _hook = h


def call(name, *args):
    global launch_count
    launch_count += _LAUNCHES.get(name, 1)
    if _hook is None:
        check(getattr(lib(), name)(*args), name)
    else:
        with _hook(name, args):
            check(getattr(lib(), name)(*args), name)
