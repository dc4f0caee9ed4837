"""ctypes binding of libesr_b200.so (the C ABI declared in include/esr_b200.h).

There is no CPU or PyTorch fallback: if the shared library is missing or a call fails, an exception is raised.
"""
import ctypes
import os

_PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_PKG, "libesr_b200.so")

_lib = None

c_void_p = ctypes.c_void_p
c_int = ctypes.c_int
c_i64 = ctypes.c_int64
c_size_t = ctypes.c_size_t
c_float = ctypes.c_float

# name -> (restype, argtypes); must list every symbol of include/esr_b200.h (tests/test_capi_symbols.py checks)
SIGNATURES = {
    "esr_version": (c_int, []),
    "esr_last_error": (ctypes.c_char_p, []),
    "esr_launch_count": (c_i64, []),
    "esr_scatter_cnt": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_i64, c_int, c_int,
                                c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "esr_scatter_image": (c_int, [c_void_p, c_void_p, c_void_p, c_i64, c_int, c_int, c_int, c_void_p, c_void_p]),
    "esr_scatter_mask": (c_int, [c_void_p, c_void_p, c_void_p, c_i64, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "esr_time_bin_bounds": (c_int, [c_void_p, c_i64, c_int, c_void_p, c_void_p]),
    "esr_scatter_voxel": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_i64, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "esr_expand_count": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "esr_expand_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int, c_int, c_i64]),
    "esr_expand_emit": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p,
                                c_void_p, c_int, c_int,
                                c_void_p, c_void_p, c_i64, c_i64, c_void_p, c_void_p, c_size_t, c_void_p]),
    "esr_cnt2event_fused_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "esr_cnt2event_fused": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_i64, c_void_p,
                                    c_size_t, c_void_p]),
}


class ConvDesc(ctypes.Structure):
    """struct esr_conv_desc of include/esr_b200.h"""
    _fields_ = [
        ("src", c_void_p * 3), ("src_C", c_int * 3), ("src_n_img", c_int * 3), ("src_img", c_void_p * 3),
        ("n_src", c_int), ("H", c_int), ("W", c_int), ("n_img", c_int), ("ntaps", c_int), ("cout", c_int),
        ("wpacked", c_void_p), ("bias", c_void_p), ("act", c_int), ("act_from", c_int), ("res_mode", c_int),
        ("epi_mode", c_int), ("res", c_void_p), ("res_C", c_int), ("res_n_img", c_int), ("res_img", c_void_p),
        ("out", c_void_p), ("out_C", c_int), ("out_n_img", c_int), ("out_coff", c_int),
        ("out_f32", c_void_p), ("out_f32_C", c_int), ("h_prev", c_void_p), ("h_n_img", c_int), ("z_buf", c_void_p),
    ]


SIGNATURES.update({
    "esr_conv_tc": (c_int, [ctypes.POINTER(ConvDesc), c_void_p]),
    "esr_conv_tc_chunked": (c_int, [ctypes.POINTER(ConvDesc), ctypes.POINTER(c_int), ctypes.POINTER(c_int), c_void_p]),
    "esr_conv_weight_bytes": (c_size_t, [c_int, c_int, c_int]),
    "esr_pack_conv_weight": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "esr_split_from_nchw": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "esr_split_to_nchw": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
})


class ConvSmallDesc(ctypes.Structure):
    """struct esr_conv_small_desc of include/esr_b200.h"""
    _fields_ = [
        ("kind", c_int), ("path", c_int), ("in_f32", c_void_p), ("in_", c_void_p), ("in_n_img", c_int), ("in_img", c_void_p),
        ("H_in", c_int), ("W_in", c_int), ("pad_top", c_int), ("pad_bottom", c_int), ("pad_left", c_int), ("pad_right", c_int),
        ("w", c_void_p), ("bias", c_void_p), ("w_head", c_void_p), ("b_head", c_void_p), ("n_img", c_int),
        ("out", c_void_p), ("out_n_img", c_int), ("out_f32", c_void_p),
        ("crop_top", c_int), ("crop_left", c_int), ("out_H", c_int), ("out_W", c_int),
        ("agg_feats", c_void_p), ("agg_n_img", c_int), ("agg_att", c_void_p), ("agg_idx", c_void_p), ("agg_N", c_int),
        ("workspace", c_void_p), ("workspace_bytes", c_size_t),
    ]


SIGNATURES.update({
    "esr_conv_small_workspace_bytes": (c_size_t, [c_int, c_int]),
    "esr_conv_small": (c_int, [ctypes.POINTER(ConvSmallDesc), c_void_p]),
})


class GlueDesc(ctypes.Structure):
    """struct esr_glue_desc of include/esr_b200.h"""
    _fields_ = [
        ("op", c_int), ("n_img", c_int), ("N", c_int), ("H", c_int), ("W", c_int), ("C", c_int),
        ("in_", c_void_p), ("in_n_img", c_int), ("in2", c_void_p), ("in2_n_img", c_int), ("idx", c_void_p),
        ("maps", c_void_p), ("sk", c_void_p), ("ck_in", c_void_p), ("att", c_void_p),
        ("w0", c_void_p), ("b0", c_void_p), ("w1", c_void_p), ("b1", c_void_p),
        ("mx", c_void_p), ("ck", c_void_p), ("out", c_void_p), ("out_n_img", c_int),
    ]


SIGNATURES["esr_glue"] = (c_int, [ctypes.POINTER(GlueDesc), c_void_p])


SIGNATURES.update({
    "esr_net_param_bytes": (c_size_t, []),
    "esr_net_pack_params": (c_int, [c_void_p, c_void_p, c_void_p]),
    "esr_net_param_bytes_n": (c_size_t, [c_int]),
    "esr_net_pack_params_n": (c_int, [c_int, c_void_p, c_void_p, c_void_p]),
    "esr_net_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int, c_int]),
    "esr_net_create": (c_int, [ctypes.POINTER(c_void_p), c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_size_t, c_void_p]),
    "esr_net_destroy": (c_int, [c_void_p]),
    "esr_net_reset_states": (c_int, [c_void_p, c_void_p]),
    "esr_net_reset_sample_states": (c_int, [c_void_p, c_int, c_void_p]),
    "esr_net_forward": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "esr_net_forward_profiled": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p,
                                         c_void_p, c_void_p, c_void_p, c_void_p]),
    "esr_net_get_states": (c_int, [c_void_p, c_void_p, c_void_p]),
    "esr_net_set_states": (c_int, [c_void_p, c_void_p, c_void_p]),
})


SIGNATURES.update({
    "esr_ts_search": (c_int, [c_void_p, c_i64, c_void_p, c_i64, c_void_p, c_void_p]),
    "esr_gather_events": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_i64, c_void_p, c_void_p,
                                  c_void_p, c_void_p, c_void_p]),
    "esr_gather_events_aug": (c_int, [c_void_p] * 7 + [c_int, c_int, c_int, c_i64] + [c_void_p] * 5),
    "esr_encode_frames_multi": (c_int, [c_void_p, c_void_p, c_int, c_i64] + [c_int] * 4 + [c_void_p] * 3),
    "esr_metrics_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int]),
    "esr_metrics_planes": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, ctypes.c_double, c_void_p, c_void_p, c_size_t, c_void_p]),
    "esr_lpips_param_bytes": (c_size_t, []),
    "esr_lpips_pack_params": (c_int, [c_void_p, c_void_p, c_void_p]),
    "esr_lpips_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "esr_lpips_create": (c_int, [ctypes.POINTER(c_void_p), c_int, c_int, c_int, c_void_p, c_void_p, c_size_t]),
    "esr_lpips_destroy": (c_int, [c_void_p]),
    "esr_lpips_forward": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "esr_render_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "esr_render_event_cnt": (c_int, [c_void_p] + [c_int] * 7 + [c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "esr_events_to_columns": (c_int, [c_void_p, c_int, c_i64, c_void_p, c_i64] + [c_void_p] * 5),
})

SIGNATURES.update({
    "esr_dcn_v2_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "esr_dcn_v2_workspace_bytes_ex": (c_size_t, [c_int] * 11),
    "esr_dcn_v2_backward_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "esr_dcn_v2_backward": (c_int, [c_void_p] * 6 + [c_int] * 10 + [c_void_p] * 6 + [c_size_t, c_void_p]),
    "esr_dcn_v2_forward": (c_int, [c_void_p] * 5 + [c_int] * 10 + [c_void_p, c_void_p, c_size_t, c_void_p]),
    "esr_conv2d_workspace_bytes": (c_size_t, [c_int] * 7),
    "esr_conv2d_split_bytes": (c_size_t, [c_int] * 7),
    "esr_conv2d_forward": (c_int, [c_void_p] * 3 + [c_int] * 8 + [c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "esr_conv2d_backward": (c_int, [c_void_p] * 5 + [c_int] * 8 + [c_void_p] * 4 + [c_size_t, c_void_p]),
    "esr_upsample2x_forward": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "esr_upsample2x_backward": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "esr_resize_planes": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "esr_gru_hr": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "esr_gru_hr_backward": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "esr_gru_blend": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "esr_gru_blend_backward": (c_int, [c_void_p] * 4 + [c_int, c_int] + [c_void_p] * 4),
    "esr_mse_loss": (c_int, [c_void_p, c_void_p, c_size_t, c_void_p, c_void_p, c_float, c_void_p]),
    "esr_adam_step": (c_int, [c_void_p] * 5 + [c_size_t, c_void_p] + [c_float] * 5 + [c_void_p]),
    "esr_adam_step_dev": (c_int, [c_void_p] * 5 + [c_size_t, c_void_p, c_void_p, c_void_p]),
})

# the *_ex training entry points: a `flags` word before the workspace (DETERMINISTIC = ESR_DETERMINISTIC of the header)
DETERMINISTIC = 1
SIGNATURES.update({
    "esr_conv2d_workspace_bytes_ex": (c_size_t, [c_int] * 8),
    "esr_conv2d_backward_ex": (c_int, [c_void_p] * 5 + [c_int] * 8 + [c_void_p] * 3 + [c_int, c_void_p, c_size_t, c_void_p]),
    "esr_dcn_v2_backward_workspace_bytes_ex": (c_size_t, [c_int] * 11),
    "esr_dcn_v2_backward_ex": (c_int, [c_void_p] * 6 + [c_int] * 10 + [c_void_p] * 5 + [c_int, c_void_p, c_size_t, c_void_p]),
    "esr_mse_loss_workspace_bytes_ex": (c_size_t, [c_size_t, c_int]),
    "esr_mse_loss_ex": (c_int, [c_void_p, c_void_p, c_size_t, c_void_p, c_void_p, c_float, c_int, c_void_p, c_size_t, c_void_p]),
})


SIGNATURES["esr_resize_frames_cubic"] = (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p])
SIGNATURES["esr_resize_frames_cubic_u8"] = (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p])


class ESRError(RuntimeError):
    pass


def lib():
    """The loaded library.  Raises if it has not been built (python -m esr_b200.build)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ESRError(f"{LIB_PATH} not found: build it with `python -m esr_b200.build` "
                           "(there is no CPU fallback)")
        l = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(l, name)
            fn.restype = res
            fn.argtypes = args
        _lib = l
    return _lib


def check(rc, what):
    if rc != 0:
        msg = lib().esr_last_error().decode("utf-8", "replace")
        if rc == -2:
            raise ValueError(f"{what}: negative dimensions are not allowed ({msg})")
        raise ESRError(f"{what} failed (code {rc}): {msg}")


def stream_ptr():
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def ptr(t):
    """Device (or host) address of a torch tensor / None."""
    if t is None:
        return None
    return ctypes.c_void_p(t.data_ptr())
