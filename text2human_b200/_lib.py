"""ctypes binding of libt2h.so (the C ABI declared in include/t2h.h).

The library is built in-tree by ``__graft_entry__.build()`` /
``text2human_b200/csrc/Makefile``.  There is no CPU or PyTorch fallback: if the
shared object is missing, loading fails loudly.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libt2h.so")

ABI_VERSION = 202  # T2H_VERSION of include/t2h.h that the structs below mirror
MAX_TAPS = 16
OUT_F32, OUT_PLANES = 0, 1
BIAS_NONE, BIAS_COL, BIAS_ROW = 0, 1, 2
ACT_NONE, ACT_GELU, ACT_RELU, ACT_LRELU = 0, 1, 2, 3
CVT_PLAIN, CVT_UP2X, CVT_S2D, CVT_MAXPOOL2, CVT_BILINEAR2X = 0, 1, 2, 3, 4
NGP_MAX_BLOCKS = 1024  # T2H_NGP_MAX_BLOCKS: t2h_nchw_grad_to_planes' scratch is this many rows of c_pad doubles


class TapGemmParams(C.Structure):
    """Mirror of ``t2h_tapgemm_params`` (include/t2h.h) — field order matters."""
    _fields_ = [
        ("a", C.c_void_p), ("a_terms", C.c_int32), ("a_term_imgs", C.c_int32),
        ("a_imgs", C.c_int32), ("a_bcast", C.c_int32),
        ("n_img", C.c_int32), ("H", C.c_int32), ("W", C.c_int32), ("tile_rows", C.c_int32),
        ("a_H", C.c_int32), ("a_W", C.c_int32), ("C", C.c_int32),
        ("a_sw", C.c_int64), ("a_sh", C.c_int64), ("a_sn", C.c_int64),
        ("b", C.c_void_p), ("b_terms", C.c_int32), ("b_term_g", C.c_int32),
        ("b_groups", C.c_int32), ("b_groups2", C.c_int32), ("b_batched", C.c_int32),
        ("b_batched_h", C.c_int32), ("n_out", C.c_int32),
        ("b_sn", C.c_int64), ("b_sg", C.c_int64), ("b_sg2", C.c_int64),
        ("ntaps", C.c_int32),
        ("tap_dy", C.c_int32 * MAX_TAPS), ("tap_dx", C.c_int32 * MAX_TAPS),
        ("tap_img_off", C.c_int32 * MAX_TAPS),
        ("nterms", C.c_int32),
        ("d", C.c_void_p), ("d_mode", C.c_int32), ("d_terms", C.c_int32),
        ("d_plane", C.c_int64),
        ("d_sn", C.c_int64), ("d_sh", C.c_int64), ("d_sw", C.c_int64), ("d_sc", C.c_int64),
        ("bias", C.c_void_p), ("bias_mode", C.c_int32), ("act", C.c_int32),
        ("alpha", C.c_float),
        ("residual", C.c_void_p),
        ("gn_stats", C.c_void_p), ("gn_cpg", C.c_int32), ("a_mn", C.c_int32), ("b_mn", C.c_int32), ("bias_sn", C.c_int64), ("k_split", C.c_int32),
        ("use_tap_w", C.c_int32), ("tap_w", C.c_int32 * MAX_TAPS), ("accumulate", C.c_int32),
        ("k_partials", C.c_int32), ("d_slab", C.c_int64),
        ("nb_sums", C.c_void_p), ("nb_stats", C.c_void_p), ("nb_gamma", C.c_void_p), ("nb_beta", C.c_void_p),
        ("nb_eps", C.c_float), ("nb_act", C.c_int32), ("nb_groups", C.c_int32),
    ]


class ConvWgradParams(C.Structure):
    """Mirror of ``t2h_conv_wgrad_params`` (include/t2h.h) — field order matters."""
    _fields_ = [
        ("dy", C.c_void_p), ("dy_terms", C.c_int32), ("dy_term_imgs", C.c_int32), ("dy_imgs", C.c_int32),
        ("n_img", C.c_int32), ("H", C.c_int32), ("W", C.c_int32), ("cout", C.c_int32),
        ("dy_sw", C.c_int64), ("dy_sh", C.c_int64), ("dy_sn", C.c_int64),
        ("x", C.c_void_p), ("x_terms", C.c_int32), ("x_term_imgs", C.c_int32), ("x_imgs", C.c_int32),
        ("x_H", C.c_int32), ("x_W", C.c_int32), ("cin", C.c_int32),
        ("x_sw", C.c_int64), ("x_sh", C.c_int64), ("x_sn", C.c_int64),
        ("ntaps", C.c_int32),
        ("tap_dy", C.c_int32 * MAX_TAPS), ("tap_dx", C.c_int32 * MAX_TAPS), ("tap_img_off", C.c_int32 * MAX_TAPS),
        ("dw", C.c_void_p), ("dw_tap_stride", C.c_int64), ("dw_ld", C.c_int64),
        ("alpha", C.c_float), ("nterms", C.c_int32), ("k_split", C.c_int32),
    ]


# name -> (restype, argtypes); every symbol include/t2h.h declares
_I, _L, _P, _F = C.c_int, C.c_int64, C.c_void_p, C.c_float
SIGNATURES = {
    "t2h_version": (_I, []),
    "t2h_last_error": (C.c_char_p, []),
    "t2h_device_info": (_I, [C.POINTER(_I)] * 3),
    "t2h_tapgemm": (_I, [C.POINTER(TapGemmParams), _P]),
    "t2h_debug_read": (_I, [C.POINTER(C.c_longlong), _I]),
    "t2h_nchw_to_planes": (_I, [_P, _P, _I, _I, _I, _I, _I, _I, _P]),
    "t2h_nchw_grad_to_planes": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _F, _P]),
    "t2h_nhwc_to_nchw": (_I, [_P, _P, _I, _I, _I, _I, _P]),
    "t2h_nchw_to_nhwc": (_I, [_P, _P, _I, _I, _I, _I, _P]),
    "t2h_f32_to_planes": (_I, [_P, _P, _I, _I, _I, _I, _I, _I, _P]),
    "t2h_f32_to_planes_bcast": (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _P]),
    "t2h_gn_stats": (_I, [_P, _P, _I, _I, _I, _I, _P]),
    "t2h_gn_apply": (_I, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _F, _I, _I, _P]),
    "t2h_add_inplace": (_I, [_P, _P, _L, _P]),
    "t2h_softmax_rows": (_I, [_P, _P, _L, _I, _F, _I, _P]),
    "t2h_attn_fwd": (_I, [_P, _I, _L, _L, _L, _I, _I, _I, _I, _I, _I, _I, _F, _P, _L, _L, _P]),
    "t2h_vq_search": (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _L, _P, _P, _P, _P, _P, _P,
                           _P, _L, _P]),
    "t2h_vq_workspace_bytes": (_L, [_L, _I, _I]),
    "t2h_vq_gather": (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _P, _P, _P]),
    "t2h_vq_bwd_patch": (_I, [_P] * 9 + [_I] * 7 + [_F, _F, _P]),
    "t2h_texture_mask": (_I, [_P, _P, _P, _I, _P, _I, _L, _P]),
    "t2h_u8_to_planes": (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _F, _F, _I, _P]),
    "t2h_mask_to_ids": (_I, [_P, _P, _I, _I, _I, _I, _I, _P]),
    "t2h_onehot_to_planes": (_I, [_P, _P, _I, _I, _I, _I, _I, _I, _P]),
    "t2h_embed_sum": (_I, [_P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _P]),
    "t2h_layernorm": (_I, [_P, _P, _P, _P, _L, _I, _F, _I, _P]),
    "t2h_layernorm_scatter": (_I, [_P, _P, _P, _P, _L, _I, _F, _I, _P, _L, _P]),
    "t2h_splitk_reduce_ln": (_I, [_P, _I, _L, _P, _P, _P, _P, _P, _F, _P, _I, _P, _L, _L, _I, _P]),
    "t2h_pack_u8": (_I, [_P, _P, _I, _I, _I, _I, _F, _F, _P]),
    "t2h_argmax_heads": (_I, [_P, _P, _P, _L, _I, _I, _P]),
    "t2h_shape_attr_embed": (_I, [_P] * 11 + [_I, _I, _I, _I, _P]),
    "t2h_f32_to_planes_t": (_I, [_P, _P, _P, _I, _I, _I, _I, _F, _P]),
    "t2h_planes_transpose": (_I, [_P, _P, _I, _I, _I, _L, _L, _L, _L, _L, _L, _I, _P]),
    "t2h_colsum": (_I, [_P, _P, _L, _I, _P]),
    "t2h_gelu_fwd": (_I, [_P, _P, _L, _I, _P]),
    "t2h_gelu_bwd": (_I, [_P, _P, _P, _P, _L, _I, _P]),
    "t2h_layernorm_bwd_fused": (_I, [_P, _P, _P, _P, _P, _P, _L, _I, _F, _I, _P, _I, _P, _P]),
    "t2h_softmax_bwd_planes": (_I, [_P, _P, _P, _L, _I, _F, _I, _F, _P]),
    "t2h_layernorm_bwd": (_I, [_P, _P, _P, _P, _P, _P, _L, _I, _F, _I, _P]),
    "t2h_softmax_bwd": (_I, [_P, _P, _P, _L, _I, _F, _I, _P]),
    "t2h_ce_heads": (_I, [_P, _P, _P, _P, _P, _P, _L, _I, _I, _P]),
    "t2h_head_grads_absmax": (_I, [_P, _I, _I, _I, _I, _P, _P]),
    "t2h_head_grads_to_planes": (_I, [_P, _I, _I, _I, _I, _F, _I, _P, _P]),
    "t2h_head_grads_to_planes_sums": (_I, [_P, _I, _I, _I, _I, _F, _I, _P, _P, _P, _P]),
    "t2h_embed_bwd": (_I, [_P, _P, _P, _L, _I, _I, _P]),
    "t2h_adam": (_I, [_P, _P, _P, _P, _L, _F, _F, _F, _F, _I, _F, _P]),
    "t2h_conv_wgrad": (_I, [C.POINTER(ConvWgradParams), _P]),
    "t2h_norm_bwd": (_I, [_P, _P, _P, _P, _P, _P, _P, _P, _I, _P, _P, _P, _I, _I, _I, _I, _F, _I, _P, _I, _P]),
    "t2h_bn_update_running": (_I, [_P, _P, _P, _L, _F, _I, _P]),
    "t2h_lrelu_bwd": (_I, [_P, _P, _P, _P, _I, _L, _P]),
    "t2h_sumpool2": (_I, [_P, _P, _I, _I, _I, _I, _P]),
    "t2h_planes_s2d": (_I, [_P, _P, _I, _I, _I, _I, _I, _P]),
    "t2h_vq_bwd": (_I, [_P, _P, _P, _P, _P, _P, _P, _L, _I, _I, _I, _F, _F, _P]),
    "t2h_l1_loss": (_I, [_P, _P, _P, _P, _L, _F, _P]),
    "t2h_bce_logits": (_I, [_P, _P, _I, _I, _I, _I, _I, _F, _P, _P, _I, _P, _P]),
    "t2h_hinge_loss": (_I, [_P, _P, _P, _L, _F, _F, _P]),
    "t2h_diffaug_fwd": (_I, [_P, _P, _P, _P, _P, _I, _I, _I, _P]),
    "t2h_diffaug_bwd": (_I, [_P, _P, _P, _P, _P, _I, _I, _I, _P]),
    "t2h_adaptive_weight": (_I, [_P, _P, _L, _F, _F, _F, _P, _P]),
    "t2h_axpy_dev": (_I, [_P, _P, _P, _P, _L, _P]),
    "t2h_norm_bwd_drop": (_I, [_P, _P, _P, _P, _P, _P, _I, _P, _P, _I, _P, _P, _P, _I, _I, _I, _I, _F, _I, _P]),
    "t2h_norm_apply_ex": (_I, [_P, _P, _P, _P, _P, _I, _P, _P, _I, _I, _I, _I, _F, _I, _I, _P]),
    "t2h_maxpool2_bcast_bwd": (_I, [_P, _I, _P, _P, _I, _P, _P, _I, _I, _I, _I, _I, _I, _P]),
    "t2h_bilinear2x_bwd": (_I, [_P, _P, _I, _I, _I, _I, _P]),
    "t2h_ce_logits": (_I, [_P, _P, _I, _I, _I, _I, _I, _F, _P, _P, _I, _P, _P]),
    "t2h_shape_attr_embed_bwd": (_I, [_P] * 13 + [_I, _I, _I, _I, _P]),
    "t2h_routed_head_ce": (_I, [_P, _P, _P, _P, _P, _L, _I, _I, _I, _F, _P, _P, _P, _P, _P, _P, _P, _P]),
    "t2h_lpips_scale_fwd": (_I, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _P]),
    "t2h_lpips_scale_bwd": (_I, [_P, _I, _P, _F, _P, _I, _I, _I, _P]),
    "t2h_lpips_head": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _F, _F, _P, _P, _P, _I, _P]),
    "t2h_lpips_head_chunks": (_I, [_I, _I]),
    "t2h_relu_bwd": (_I, [_P, _P, _P, _I, _L, _P]),
    "t2h_sample_step": (_I, [_P, _P, _P, _P, _P, _L, _I, _I, _F, _F, C.c_uint64, C.c_uint32, _L, _P]),
}

_lib = None


class T2HError(RuntimeError):
    pass


def load():
    """Load libt2h.so (once).  Raises if the extension has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise T2HError(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(or `make -C text2human_b200/csrc`). There is no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if a declared symbol is missing
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc):
    if rc != 0:
        raise T2HError(f"libt2h error {rc}: {load().t2h_last_error().decode()}")
