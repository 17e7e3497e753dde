"""ctypes binding of libpropainter_b200.so (C ABI in include/propainter_b200.h).

There is no fallback: if the library is missing or a call fails, we raise.  Raw device pointers
(``tensor.data_ptr()``) and the current CUDA stream are passed; the library never allocates or syncs.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# PROPAINTER_B200_LIB selects another build of the same ABI (e.g. an experiment compiled with different -D flags)
LIB_PATH = os.environ.get("PROPAINTER_B200_LIB") or os.path.join(_HERE, "libpropainter_b200.so")

c_void_p, c_int, c_long, c_float, c_size_t = ctypes.c_void_p, ctypes.c_int, ctypes.c_long, ctypes.c_float, ctypes.c_size_t

PP_MAX_WINDOW = 32


class PPAttnParams(ctypes.Structure):
    _fields_ = [("qkv", c_void_p), ("pool", c_void_p), ("key_tok", c_void_p), ("flags", c_void_p), ("out", c_void_p),
                ("ld_qkv", c_int), ("ld_pool", c_int), ("ld_out", c_int),
                ("t", c_int), ("NT", c_int), ("WN", c_int), ("NKO", c_int), ("NP", c_int), ("C", c_int),
                ("kf_start", c_int), ("kf_step", c_int), ("nkf", c_int), ("scale_log2", c_float)]


PP_CONV_MAX_SEG = 4


class PPConvSeg(ctypes.Structure):
    _fields_ = [("x", c_void_p), ("ld", c_int), ("C", c_int)]


class PPConvParams(ctypes.Structure):
    _fields_ = [("seg", PPConvSeg * PP_CONV_MAX_SEG), ("nseg", c_int),
                ("n", c_int), ("H", c_int), ("W", c_int), ("KH", c_int), ("KW", c_int),
                ("w_packed", c_void_p), ("Cout", c_int), ("bias", c_void_p),
                ("pre", c_void_p), ("ld_pre", c_int), ("res", c_void_p), ("ld_res", c_int),
                ("out", c_void_p), ("ld_out", c_int),
                ("act", c_int), ("slope", c_float), ("post_relu", c_int), ("round_tf32", c_int),
                ("bn", c_int), ("tile_w", c_int), ("tile_m", c_int)]


class PPWindowIds(ctypes.Structure):
    _fields_ = [("n", c_int), ("frame", c_int * PP_MAX_WINDOW), ("first", c_int * PP_MAX_WINDOW)]


# symbol -> (restype, argtypes); the CPU test-suite checks every symbol of the header is exported
SIGNATURES = {
    "pp_abi_version": (c_int, []),
    "pp_error_string": (ctypes.c_char_p, [c_int]),
    "pp_corr_build": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_void_p]),
    "pp_corr_pool_pyramid": (c_int, [c_void_p, c_long, c_int, c_int, c_void_p]),
    "pp_corr_lookup": (c_int, [c_void_p, c_void_p, c_void_p, c_long, c_int, c_int, c_void_p]),
    "pp_corr_lookup_ldg": (c_int, [c_void_p, c_void_p, c_void_p, c_long, c_int, c_int, c_void_p]),
    "pp_corr_lookup_f16": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_long, c_int, c_int, c_void_p]),
    "pp_corr_lookup_ldg_f16": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_long, c_int, c_int, c_void_p]),
    "pp_corr_fmap_pyramid": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "pp_corr_lookup_otf": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "pp_corr_lookup_r": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_long, c_int, c_int, c_void_p]),
    "pp_corr_lookup_ldg_r": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_long, c_int, c_int, c_void_p]),
    "pp_corr_lookup_otf_r": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_int,
                                     c_void_p]),
    "pp_upflow8": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "pp_convex_upsample": (c_int, [c_void_p, c_int, c_float, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "pp_img_prop_scan_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "pp_img_prop_scan": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_int,
                                 c_int, c_int, c_int, c_void_p]),
    "pp_img_prop_scan_u8h_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "pp_img_prop_scan_u8h": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_int, c_int,
                                     c_int, c_int, c_int, c_int, c_void_p]),
    "pp_prop_cond": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p,
                             c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "pp_deform_align_workspace_bytes": (c_size_t, [c_int, c_int]),
    "pp_deform_align": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_float, c_void_p, c_void_p, c_void_p,
                                c_int, c_int, c_int, c_int, c_int, c_void_p, c_size_t, c_void_p]),
    "pp_conv2d_umma": (c_int, [ctypes.POINTER(PPConvParams), c_void_p]),
    "pp_conv2d_umma_plan": (c_int, [ctypes.POINTER(PPConvParams)] + [c_void_p] * 5),
    "pp_conv2d_umma_f16": (c_int, [ctypes.POINTER(PPConvParams), c_void_p, c_int, c_void_p]),
    "pp_conv2d_umma_plan_f16": (c_int, [ctypes.POINTER(PPConvParams)] + [c_void_p] * 5),
    "pp_deform_gather": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_float, c_void_p, c_int, c_int,
                                 c_int, c_int, c_void_p]),
    "pp_flow_warp_fbcheck": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_int,
                                     c_int, c_void_p]),
    "pp_deform_gather_f16": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_float, c_void_p, c_int,
                                     c_int, c_int, c_int, c_void_p]),
    "pp_flow_warp_fbcheck_f16": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int,
                                         c_int, c_void_p]),
    "pp_gen_prep": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                            c_void_p]),
    "pp_gen_prep_f16": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                                c_void_p]),
    "pp_window_mask": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "pp_sparse_window_attn": (c_int, [ctypes.POINTER(PPAttnParams), c_int, c_void_p]),
    "pp_sparse_window_attn_mma": (c_int, [ctypes.POINTER(PPAttnParams), c_int, c_void_p]),
    "pp_sparse_window_attn_f16": (c_int, [ctypes.POINTER(PPAttnParams), c_int, c_void_p]),
    "pp_ffn_overlap_add_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int]),
    "pp_ffn_overlap_add": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_size_t,
                                   c_void_p]),
    "pp_ffn_overlap_add_f16": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_size_t,
                                       c_void_p]),
    "pp_gru_gate": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_long, c_int, c_void_p]),
    "pp_gru_update": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_long, c_int, c_void_p]),
    "pp_raft_pack_motion": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_long, c_void_p]),
    "pp_gru_gate_f16": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_long, c_int, c_void_p]),
    "pp_gru_update_f16": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p, c_long, c_int,
                                  c_void_p]),
    "pp_raft_pack_motion_f16": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_long, c_void_p]),
    "pp_raft_pack_motion_n": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_long, c_int, c_void_p]),
    "pp_bias_act": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p, c_int, c_long, c_int, c_int, c_float, c_int,
                            c_void_p]),
    "pp_bias_act_pre": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_long, c_int, c_int, c_float,
                                c_int, c_void_p]),
    "pp_bias_act_f16": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_int, c_long, c_int,
                                c_int, c_float, c_int, c_void_p]),
    "pp_bias_act_f16_res": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p, c_int, c_long, c_int, c_int, c_float, c_int,
                                    c_void_p]),
    "pp_pool_depthwise": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "pp_add_layernorm": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_long, c_int, c_float, c_void_p]),
    "pp_pool_depthwise_f16": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int,
                                      c_void_p]),
    "pp_add_layernorm_f16": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_long, c_int,
                                     c_float, c_void_p]),
    "pp_instance_norm_workspace_bytes": (c_size_t, [c_int, c_long, c_int]),
    "pp_instance_norm": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_long, c_int, c_float, c_int, c_int, c_void_p, c_size_t,
                                 c_void_p]),
    "pp_upsample2x_bilinear": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "pp_upsample2x_bilinear_f16": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "pp_sc_fold_f16": (c_int, [c_void_p, c_long, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "pp_mask_dilate": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "pp_u8_to_frames": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "pp_u8_to_frames_resized": (c_int, [c_void_p, c_void_p] + [c_int] * 5 + [c_void_p]),
    "pp_resample_coeffs_bicubic": (c_int, [c_int, c_int, c_void_p, c_void_p, c_long]),
    "pp_resample_index_nearest": (c_int, [c_int, c_int, c_void_p]),
    "pp_resample_coeffs_linear_cv": (c_int, [c_int, c_int, c_int, c_void_p, c_void_p]),
    "pp_resize_u8_bicubic_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "pp_resize_u8_bicubic": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p,
                                     c_int, c_void_p, c_size_t, c_void_p]),
    "pp_resize_u8_nearest": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "pp_resize_u8_bilinear_cv": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                         c_void_p]),
    "pp_composite_blend_u8": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, ctypes.POINTER(PPWindowIds), c_int, c_int,
                                      c_void_p]),
    "pp_composite_blend_f32": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, ctypes.POINTER(PPWindowIds), c_int, c_int,
                                       c_void_p]),
    "pp_resample_coeffs_linear_f32": (c_int, [c_int, c_int, c_int, c_void_p, c_void_p]),
    "pp_resize_flow_linear_cv": (c_int, [c_void_p, c_void_p] + [c_int] * 5 + [c_void_p] * 5),
    "pp_extrapolate_u8": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p] + [c_int] * 9 + [c_void_p]),
    "pp_mask_overlay_u8": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "pp_flow_maxrad": (c_int, [c_void_p, c_void_p] + [c_int] * 5 + [ctypes.c_float, c_void_p]),
    "pp_flow_to_image_u8": (c_int, [c_void_p, c_void_p, c_void_p] + [c_int] * 5 + [ctypes.c_float, c_int, c_void_p]),
    "pp_flow_occlusion": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "pp_warp_error_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "pp_warp_error": (c_int, [c_void_p] * 5 + [c_int] * 3 + [c_void_p, c_size_t, c_void_p]),
    "pp_i3d_input": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "pp_maxpool3d_same": (c_int, [c_void_p, c_int, c_void_p, c_int] + [c_int] * 11 + [c_void_p]),
    "pp_mean_thw": (c_int, [c_void_p, c_int, c_void_p, c_int, c_long, c_int, c_void_p]),
    "pp_cutie_topk_readout": (c_int, [c_void_p, c_void_p, c_void_p, c_long] + [c_int] * 3 + [c_void_p, c_void_p] + [c_int] * 3 +
                              [c_void_p] * 4),
    "pp_cutie_frame_in": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "pp_cutie_labels": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_void_p]),
}

_lib = None


def lib():
    """Load (once) and return the shared library; raises if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} not found: build the CUDA extension first (python -c 'import __graft_entry__ as g; "
                "g.build()').  propainter_b200 has no CPU or PyTorch fallback.")
        handle = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(handle, name)          # AttributeError if a symbol is missing
            fn.restype, fn.argtypes = res, args
        if handle.pp_abi_version() != 2:
            raise RuntimeError("libpropainter_b200.so ABI version mismatch")
        _lib = handle
    return _lib


def check(code, what):
    if code != 0:
        raise RuntimeError(f"{what} failed: {lib().pp_error_string(code).decode()} ({code})")
