"""ctypes binding of the C-ABI library (include/lgb200.h).

The shared library is built in-tree by `__graft_entry__.build()` at
glue-factory_b200/csrc/liblgb200.so.  There is no fallback: if the library is
missing, or the device is not an H100 (sm_90), every entry point raises.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "liblgb200.so")

F32, BF16 = 0, 1

_lib = None
_device_checked = False

_vp, _i, _i64, _f, _sz = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_float, ctypes.c_size_t
_d = ctypes.c_double

# name -> (restype, argtypes); mirrors include/lgb200.h one to one
SIGNATURES = {
    "lgb200_abi_version": (_i, []),
    "lgb200_last_error": (ctypes.c_char_p, []),
    "lgb200_check_device": (_i, []),
    "lgb200_rope_split_fwd": (_i, [_vp, _vp, _vp, _vp, _vp, _i64, _i, _i, _vp]),
    "lgb200_rope_split_bwd": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i, _i, _vp]),
    "lgb200_rope_split_fwd_hd": (_i, [_vp, _vp, _vp, _vp, _vp, _i64, _i, _i, _i, _vp]),
    "lgb200_rope_split_bwd_hd": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i, _i, _i, _vp]),
    "lgb200_attn_fwd": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _f, _i, _vp]),
    "lgb200_attn_bwd_ws_floats": (_i64, [_i, _i, _i, _i]),
    "lgb200_attn_bwd": (_i, [_vp] * 10 + [_i, _i, _i, _i, _i, _f, _i, _vp]),
    "lgb200_attn_fwd_hd": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _f, _i, _i, _vp]),
    "lgb200_attn_bwd_hd": (_i, [_vp] * 10 + [_i, _i, _i, _i, _i, _f, _i, _i, _vp]),
    "lgb200_attn_fwd_varlen": (_i, [_vp] * 9 + [_i, _i, _i, _i, _i, _f, _i, _i, _vp]),
    "lgb200_adaptive_compact_ws_ints": (_i64, [_i, _i]),
    "lgb200_adaptive_compact": (_i, [_vp] * 18 + [_f, _f] + [_i] * 10 + [_vp]),
    "lgb200_adaptive_compact_varlen": (_i, [_vp] * 19 + [_f, _f] + [_i] * 10 + [_vp]),
    "lgb200_ln_gelu_fwd": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i64, _i, _f, _i, _vp]),
    "lgb200_ln_gelu_bwd_parts": (_i, [_i64]),
    "lgb200_ln_gelu_bwd": (_i, [_vp] * 10 + [_i64, _i, _i, _vp]),
    "lgb200_gemm_bf16": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i64, _i64, _i64, _i64, _i64, _i64, _i, _f, _vp]),
    "lgb200_gemm_splitk_ws_floats": (_i64, [_i, _i, _i]),
    "lgb200_gemm_bf16_splitk": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _i, _i64, _i64, _i64, _vp, _vp]),
    "lgb200_linear": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i64, _i64, _i64, _i, _f, _i, _vp]),
    "lgb200_assign_ws_bytes": (_sz, [_i, _i, _i]),
    "lgb200_assign_lse": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "lgb200_assign_scores": (_i, [_vp] * 16 + [_i, _i, _i, _vp]),
    "lgb200_assign_bwd": (_i, [_vp] * 8 + [_i, _i, _i, _i, _vp]),
    "lgb200_assign_fused_lse": (_i, [_vp, _vp, _f, _vp, _vp, _i, _i, _i, _i, _vp]),
    "lgb200_assign_fused_stats": (_i, [_vp, _vp, _f] + [_vp] * 10 + [_i, _i, _i, _i, _vp]),
    "lgb200_assign_fused_bwd": (_i, [_vp, _vp, _f] + [_vp] * 9 + [_i, _i, _i, _i, _vp]),
    "lgb200_assign_pos_fwd": (_i, [_vp, _vp, _vp, _f] + [_vp] * 5 + [_i] * 4 + [_vp]),
    "lgb200_assign_pos_bwd": (_i, [_vp] * 7 + [_i] * 4 + [_vp]),
    "lgb200_assign_bwd_sparse": (_i, [_vp] * 8 + [_i, _i, _i, _i, _vp]),
    "lgb200_filter_matches": (_i, [_vp, _vp, _vp, _f, _vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "lgb200_assign_lse_varlen": (_i, [_vp] * 5 + [_i, _i, _i, _vp]),
    "lgb200_assign_scores_varlen": (_i, [_vp] * 17 + [_i] * 5 + [_vp]),
    "lgb200_filter_matches_varlen": (_i, [_vp, _vp, _vp, _f] + [_vp] * 7 + [_i] * 5 + [_vp]),
    "lgb200_head_logsig": (_i, [_vp, _vp, _vp, _i64, _vp]),
    "lgb200_head_token_bwd_ws_floats": (_i, [_i]),
    "lgb200_head_token_fwd": (_i, [_vp] * 9 + [_i64, _i, _i, _vp]),
    "lgb200_head_token_bwd": (_i, [_vp] * 9 + [_i64, _i, _i, _vp]),
    "lgb200_head_terms_fwd": (_i, [_vp] * 14 + [_f] + [_vp] * 6 + [_i, _i, _i, _vp]),
    "lgb200_head_terms_bwd": (_i, [_vp] * 13 + [_f] + [_vp] * 3 + [_i, _i, _i, _vp]),
    "lgb200_heads_ws_bytes": (_sz, [_i, _i, _i]),
    "lgb200_log_double_softmax": (_i, [_vp, _f, _vp, _vp, _i, _i, _i, _vp]),
    "lgb200_log_double_softmax_dev": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "lgb200_log_double_softmax_varlen": (_i, [_vp] * 8 + [_i] * 5 + [_vp]),
    "lgb200_line_scores_varlen": (_i, [_vp] * 5 + [_i] * 5 + [_vp]),
    "lgb200_junction_mean_varlen": (_i, [_vp] * 4 + [_i, _i, _vp]),
    "lgb200_line_scores_train": (_i, [_vp] * 5 + [_i] * 5 + [_vp]),
    "lgb200_line_scores_bwd": (_i, [_vp] * 10 + [_i] * 5 + [_vp]),
    "lgb200_junction_sum": (_i, [_vp] * 4 + [_i, _i, _i, _vp]),
    "lgb200_sinkhorn": (_i, [_vp, _f, _i, _vp, _vp, _i, _i, _i, _vp]),
    "lgb200_sinkhorn_fwd": (_i, [_vp, _f, _i, _vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "lgb200_sinkhorn_bwd": (_i, [_vp, _f, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "lgb200_sinkhorn_fwd_dev": (_i, [_vp, _vp, _i, _vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "lgb200_sinkhorn_bwd_dev": (_i, [_vp, _vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "lgb200_sinkhorn_varlen_ws_bytes": (_sz, [_i, _i, _i]),
    "lgb200_sinkhorn_varlen": (_i, [_vp, _vp, _i, _vp, _vp, _vp] + [_i] * 5 + [_vp]),
    "lgb200_ot_nll_fwd": (_i, [_vp] * 7 + [_i, _i, _i, _vp]),
    "lgb200_ot_nll_bwd": (_i, [_vp] * 8 + [_i, _i, _i, _vp]),
    "lgb200_ot_nll_fwd_sparse": (_i, [_vp] * 8 + [_i, _i, _i, _vp]),
    "lgb200_ot_nll_bwd_sparse": (_i, [_vp] * 8 + [_i, _i, _i, _vp]),
    "lgb200_ot_filter_stats": (_i, [_vp] * 4 + [_i, _i, _i, _vp]),
    "lgb200_gt_homography_ws_bytes": (_sz, [_i, _i, _i]),
    "lgb200_gt_from_homography": (_i, [_vp, _vp, _vp, _vp, _f, _f, _vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "lgb200_gt_from_reprojection": (_i, [_vp] * 8 + [_f, _f, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "lgb200_gt_epipolar_unmatched": (_i, [_vp] * 5 + [_f, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "lgb200_gt_line_sample": (_i, [_vp, _vp, _i, _i, _i, _vp]),
    "lgb200_lsap": (_i, [_vp, _vp, _vp, _i, _i, _i, _vp]),
    "lgb200_gt_lines_ws_bytes": (_sz, [_i, _i, _i]),
    "lgb200_gt_line_matches": (_i, [_vp] * 10 + [_i] * 5 + [_d] * 3 + [_vp] * 4 + [_i, _i, _i, _vp]),
    "lgb200_adam_flat": (_i, [_vp, _vp, _vp, _vp, _i64, _vp, _f, _f, _f, _f, _f, _i, _vp, _f, _vp, _vp, _vp, _vp]),
    "lgb200_adamw_flat": (_i, [_vp, _vp, _vp, _vp, _i64, _vp, _f, _f, _f, _f, _f, _i, _vp, _f, _vp, _vp, _vp, _vp]),
    "lgb200_sgd_flat": (_i, [_vp, _vp, _vp, _i64, _vp, _f, _f, _f, _i, _f, _i, _vp, _f, _vp, _vp, _vp, _vp]),
    "lgb200_rmsprop_flat": (_i, [_vp, _vp, _vp, _vp, _vp, _i64, _vp, _f, _f, _f, _f, _f, _f, _vp, _vp, _vp, _vp]),
    "lgb200_flat_grad_check": (_i, [_vp, _i64, _vp, _vp]),
    "lgb200_flat_grad_norm_ws_bytes": (_sz, [_i64]),
    "lgb200_flat_grad_norm": (_i, [_vp, _i64, _i64, _f, _vp, _f, _vp, _vp, _vp, _vp, _vp]),
    "lgb200_amp_update": (_i, [_vp, _vp, _vp, _vp, _f, _f, _i, _vp]),
    "lgb200_cast_bf16": (_i, [_vp, _vp, _i64, _vp]),
    "lgb200_colsum_slabs": (_i, [_i64, _i]),
    "lgb200_colsum": (_i, [_vp, _vp, _vp, _vp, _i64, _i, _i, _vp]),
    "lgb200_bn_stats": (_i, [_vp, _vp, _vp, _vp, _i64, _i, _i, _vp]),
    "lgb200_bn_relu_fwd": (_i, [_vp] * 6 + [_f, _f] + [_vp] * 3 + [_i64, _i, _i, _vp]),
    "lgb200_bn_running_update": (_i, [_vp, _vp, _vp, _f, _i, _vp]),
    "lgb200_bn_relu_bwd_reduce": (_i, [_vp] * 9 + [_i64, _i, _i, _vp]),
    "lgb200_bn_relu_bwd": (_i, [_vp] * 9 + [_i64, _i, _i, _vp]),
    "lgb200_posenc_wgrad_blocks": (_i, []),
    "lgb200_posenc_wgrad": (_i, [_vp, _vp, _vp, _i64, _i, _i, _vp]),
    "lgb200_mask_counts": (_i, [_vp, _vp, _vp, _i, _i, _i, _vp]),
    "lgb200_residual_add_cast": (_i, [_vp, _vp, _vp, _vp, _i64, _i, _vp]),
    "lgb200_add_f32_cast": (_i, [_vp, _vp, _vp, _vp, _i64, _i, _vp]),
    "lgb200_residual_add_cast_pitched": (_i, [_vp, _vp, _vp, _vp, _i64, _i64, _i64, _i, _vp]),
    "lgb200_sp_conv1a": (_i, [_vp, _i, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "lgb200_sp_conv": (_i, [_vp, _i, _vp, _vp, _vp] + [_i] * 7 + [_vp]),
    "lgb200_sp_nms": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _i, _vp]),
    "lgb200_sp_count": (_i, [_vp, _f, _vp, _i, _i, _i, _vp]),
    "lgb200_sp_select": (_i, [_vp, _f, _i, _i, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "lgb200_sp_sample": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp]),
    "lgb200_spo_conv1a": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "lgb200_spo_conv": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _vp] + [_i] * 7 + [_vp]),
    "lgb200_spo_bn_apply": (_i, [_vp, _vp, _vp, _vp, _f, _vp, _i, _i, _i, _i, _i, _vp]),
}


class Lgb200Error(RuntimeError):
    pass


def load(check_device=True):
    """dlopen the library and bind every symbol declared in include/lgb200.h."""
    global _lib, _device_checked
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise Lgb200Error(
                f"{LIB_PATH} not found: the CUDA extension has not been built "
                "(run `python __graft_entry__.py`). There is no CPU fallback.")
        lib = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)  # AttributeError if the symbol is missing
            fn.restype = res
            fn.argtypes = args
        if lib.lgb200_abi_version() != 2:
            raise Lgb200Error("liblgb200.so ABI version mismatch")
        _lib = lib
    if check_device and not _device_checked:
        import torch

        if not torch.cuda.is_available():
            raise Lgb200Error("no CUDA device: the lgb200 matcher runs on H100 (sm_90a) only, there is no CPU fallback")
        rc = _lib.lgb200_check_device()
        if rc != 0:
            raise Lgb200Error(_lib.lgb200_last_error().decode())
        _device_checked = True
    return _lib


# kernels launched per entry point (for bench.py's gpu_launches accounting)
KERNELS_PER_CALL = {
    "lgb200_rope_split_fwd": 1, "lgb200_rope_split_bwd": 1, "lgb200_attn_fwd": 1, "lgb200_attn_bwd": 3,  # prep + fused + dQ convert (or prep + dQ + dKV; shared-qk cross: 2, passed by the caller)
    "lgb200_ln_gelu_fwd": 1, "lgb200_ln_gelu_bwd": 1, "lgb200_gemm_bf16": 1, "lgb200_assign_lse": 2,
    "lgb200_assign_scores": 2, "lgb200_assign_bwd": 1, "lgb200_filter_matches": 1, "lgb200_log_double_softmax": 3,
    "lgb200_adam_flat": 1, "lgb200_cast_bf16": 1, "lgb200_colsum": 1, "lgb200_residual_add_cast": 1,
    "lgb200_gemm_bf16_splitk": 2, "lgb200_gt_from_homography": 3, "lgb200_gt_from_reprojection": 3, "lgb200_gt_epipolar_unmatched": 2, "lgb200_gt_line_matches": 5, "lgb200_flat_grad_check": 1, "lgb200_flat_grad_norm": 2, "lgb200_amp_update": 1,
    "lgb200_ot_nll_fwd": 2, "lgb200_ot_nll_bwd": 1, "lgb200_ot_filter_stats": 2, "lgb200_bn_running_update": 1,
    "lgb200_attn_fwd_hd": 1, "lgb200_attn_bwd_hd": 3,  # prep + dQ + dKV (fp32: delta + dQ + dKV)
    "lgb200_rope_split_fwd_hd": 1, "lgb200_rope_split_bwd_hd": 1,
    "lgb200_adamw_flat": 1, "lgb200_sgd_flat": 1, "lgb200_rmsprop_flat": 1,
    "lgb200_attn_fwd_varlen": 1, "lgb200_adaptive_compact": 2, "lgb200_adaptive_compact_varlen": 2,  # decide + gather
    "lgb200_assign_lse_varlen": 2, "lgb200_assign_scores_varlen": 2, "lgb200_filter_matches_varlen": 1,
    "lgb200_log_double_softmax_varlen": 4, "lgb200_line_scores_varlen": 1, "lgb200_junction_mean_varlen": 1,
    "lgb200_line_scores_train": 1, "lgb200_line_scores_bwd": 1, "lgb200_junction_sum": 1,
    "lgb200_sinkhorn_varlen": 2,  # item table + persistent iterations
    "lgb200_ot_nll_fwd_sparse": 2, "lgb200_assign_pos_fwd": 1, "lgb200_assign_pos_bwd": 1,
    "lgb200_assign_bwd_sparse": 1, "lgb200_ot_nll_bwd_sparse": 1,
}
launch_count = 0          # running total of kernels launched through `call`
timed_entry = None        # entry-point name or a set of names: every call of them is bracketed by CUDA events
timed_events = []         # [(start_event, end_event, tag)]; tag = (name, timed_tagger(name, args)) when a tagger is set
timed_tag = None
timed_tagger = None       # optional callable (name, args) -> hashable, e.g. to tell self- from cross-attention launches


def call(name, *args, launches=None):
    """Invoke an entry point; a negative return code becomes a Python exception carrying the
    library's message (reference convention: Python exceptions / asserts, lightglue.py:413-414).
    launches: kernels this call launches, when it differs from KERNELS_PER_CALL[name]."""
    global launch_count
    lib = load()
    if timed_entry is not None and (timed_entry == name or (isinstance(timed_entry, (set, frozenset)) and name in timed_entry)):
        import torch

        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        rc = getattr(lib, name)(*args)
        e.record()
        timed_events.append((s, e, (name, timed_tagger(name, args)) if timed_tagger is not None else timed_tag))
    else:
        rc = getattr(lib, name)(*args)
    if rc != 0:
        raise Lgb200Error(f"{name} failed ({rc}): {lib.lgb200_last_error().decode()}")
    launch_count += launches if launches is not None else KERNELS_PER_CALL.get(name, 1)


def stream_ptr():
    import torch

    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def ptr(t):
    """Device pointer of a tensor (None -> NULL)."""
    if t is None:
        return None
    return ctypes.c_void_p(t.data_ptr())
