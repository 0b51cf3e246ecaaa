"""ctypes binding of libmarconet_b200.so (the C ABI declared in include/marconet_b200.h).

The product path has NO fallback: if the shared library is missing or a symbol cannot be
resolved this module raises at import of the first operator, loudly.
"""
import ctypes
import os
from ctypes import c_longlong, POINTER, Structure, c_char_p, c_double, c_float, c_int, c_int32, c_int64, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libmarconet_b200.so")

# enums (mirror include/marconet_b200.h)
ACT_NONE, ACT_RELU, ACT_LRELU02, ACT_TANH, ACT_GELU, ACT_SIGMOID, ACT_RSQRT_EPS = range(7)
PREC_FP32_SIMT, PREC_F16X3_TC, PREC_BF16X3_TC, PREC_F16X1_TC = range(4)


class ConvParams(Structure):
    _fields_ = [
        ("x", c_void_p), ("N", c_int), ("H", c_int), ("W", c_int), ("Cin", c_int), ("x_cs", c_int),
        ("w", c_void_p), ("KH", c_int), ("KW", c_int), ("stride_h", c_int), ("stride_w", c_int),
        ("pad_h", c_int), ("pad_w", c_int), ("Cout", c_int),
        ("y", c_void_p), ("y_cs", c_int),
        ("bias", c_void_p),
        ("out_scale", c_void_p), ("out_scale_stride", c_int),
        ("residual", c_void_p), ("res_cs", c_int),
        ("res_broadcast_n", c_int),
        ("act", c_int), ("act_gain", c_float),
        ("y2", c_void_p), ("y2_cs", c_int), ("y2_scale", c_void_p), ("y2_scale_stride", c_int),
        ("valid_w", c_void_p),
        ("workspace", c_void_p), ("workspace_bytes", c_int64),
        ("split_k", c_int),
        ("precision", c_int),
        ("w_tc_hi", c_void_p), ("w_tc_lo", c_void_p), ("w_tc_scale", c_void_p),
        ("gn_mean_rstd", c_void_p), ("gn_gamma", c_void_p), ("gn_beta", c_void_p), ("gn_swish", c_int),
        ("x_scale", c_float), ("x_absmax", c_void_p), ("range_flag", c_void_p), ("range_tag", c_int32),
        ("y2_ptrs", c_void_p), ("gn_stats_out", c_void_p),
    ]


CONV_KERNELS = ("small", "simt", "tc1", "tc2")     # mn_conv_kernel


class ConvPlan(Structure):
    _fields_ = [("kernel", c_int), ("precision", c_int), ("nt", c_int), ("TN", c_int), ("TH", c_int), ("TW", c_int), ("splits", c_int),
                ("gn_fused", c_int), ("gn_stats_out", c_int), ("cs", c_int), ("m_tiles", c_int), ("work_items", c_int),
                ("hstages", c_int), ("bstages", c_int), ("ctas", c_int)]


class DemodDesc(Structure):
    _fields_ = [("wsq", c_void_p), ("s_off", c_int32), ("cin", c_int32), ("cout", c_int32), ("out_off", c_int32)]


class Window(Structure):
    _fields_ = [("line", c_int32), ("x1", c_int32), ("x2", c_int32), ("y1", c_int32)]


class LqCrop(Structure):
    _fields_ = [("img", c_void_p), ("row_pitch", c_int64), ("h", c_int), ("w", c_int), ("cn", c_int), ("fx", c_double), ("fy", c_double),
                ("dh", c_int), ("dw", c_int)]


class SrPiece(Structure):
    _fields_ = [("line", c_int32), ("src_x0", c_int32), ("width", c_int32), ("dst", c_void_p), ("dst_pitch", c_int64)]


class FigurePrior(Structure):
    _fields_ = [("img", c_void_p), ("stride_c", c_int64), ("stride_h", c_int64), ("stride_w", c_int64)]


class FigureImage(Structure):
    _fields_ = [("img", c_void_p), ("row_pitch", c_int64), ("fig", c_void_p), ("fig_pitch", c_int64), ("marks", c_void_p), ("priors", c_void_p),
                ("h", c_int32), ("w", c_int32), ("S", c_int32), ("W", c_int32), ("n_top", c_int32), ("n_bot", c_int32), ("n_chars", c_int32)]


PRED_SLOTS = 16     # MN_PRED_SLOTS


class CharPred(Structure):
    _fields_ = [("x1", c_double * PRED_SLOTS), ("x2", c_double * PRED_SLOTS), ("label", c_int32 * PRED_SLOTS), ("n_kept", c_int32),
                ("n_decoded", c_int32)]


class PredRow(Structure):
    _fields_ = [("a", c_double), ("scale", c_double), ("lo", c_double), ("hi", c_double), ("out", c_void_p)]


LABEL_SLOTS = 64    # MN_LABEL_SLOTS


class LabelRow(Structure):
    _fields_ = [("n", c_int32), ("label", c_int32 * LABEL_SLOTS)]


class LerpRow(Structure):
    _fields_ = [("w1", c_int32), ("w2", c_int32), ("s", c_float), ("t", c_float)]


class PriorTile(Structure):
    _fields_ = [("dst", c_void_p), ("dst_pitch", c_int64)]


class ResizeImage(Structure):
    _fields_ = [("src", c_void_p), ("src_pitch", c_int64), ("h", c_int32), ("w", c_int32), ("dst", c_void_p), ("dst_pitch", c_int64),
                ("dh", c_int32), ("dw", c_int32), ("scale_x", c_double), ("scale_y", c_double)]


class Region(Structure):
    _fields_ = [("page", c_void_p), ("page_pitch", c_int64), ("sr", c_void_p), ("sr_pitch", c_int64), ("chain", c_void_p),
                ("page_h", c_int32), ("page_w", c_int32), ("sr_h", c_int32), ("sr_w", c_int32),
                ("x0", c_int32), ("y0", c_int32), ("x1", c_int32), ("y1", c_int32), ("feather", c_int32), ("n_chain", c_int32)]


class WarpImage(Structure):
    _fields_ = [("src", c_void_p), ("src_pitch", c_int64), ("h", c_int32), ("w", c_int32), ("dst", c_void_p), ("dst_pitch", c_int64),
                ("dh", c_int32), ("dw", c_int32), ("m", c_double * 6)]


REGION_RECT, REGION_AFFINE = 0, 1


class RegionAffine(Structure):
    _fields_ = [("r", Region), ("kind", c_int32), ("kx", c_float), ("ky", c_float), ("pad", c_int32), ("n", c_double * 6)]


class WarpPerspectiveImage(Structure):
    _fields_ = [("src", c_void_p), ("src_pitch", c_int64), ("h", c_int32), ("w", c_int32), ("dst", c_void_p), ("dst_pitch", c_int64),
                ("dh", c_int32), ("dw", c_int32), ("m", c_double * 9)]


REGION_PERSPECTIVE = 2


class RegionQuad(Structure):
    _fields_ = [("r", Region), ("kind", c_int32), ("kx", c_float), ("ky", c_float), ("pad", c_int32), ("n", c_double * 9)]


class VerticalColumn(Structure):
    _fields_ = [("src", c_void_p), ("src_pitch", c_int64), ("dst", c_void_p), ("dst_pitch", c_int64), ("cells", c_void_p),
                ("dh", c_int32), ("dw", c_int32), ("n_cells", c_int32), ("w", c_int32)]


class RemapCurvedImage(Structure):
    _fields_ = [("src", c_void_p), ("src_pitch", c_int64), ("h", c_int32), ("w", c_int32), ("dst", c_void_p), ("dst_pitch", c_int64),
                ("dh", c_int32), ("dw", c_int32), ("curve", c_void_p), ("n_seg", c_int32), ("pad", c_int32)]


REGION_CURVED = 3


class RegionCurved(Structure):
    _fields_ = [("q", RegionQuad), ("curve", c_void_p), ("n_seg", c_int32), ("pad", c_int32)]


BLOCK_MAX_LINES = 256   # MN_BLOCK_MAX_LINES
INK_AUTO, INK_DARK, INK_LIGHT = 0, 1, 2


class BlockLines(Structure):
    _fields_ = [("n_lines", c_int32), ("threshold", c_int32), ("ink", c_int32), ("pad", c_int32),
                ("rect", c_int32 * (4 * BLOCK_MAX_LINES))]


class TextBlock(Structure):
    _fields_ = [("img", c_void_p), ("pitch", c_int64), ("x0", c_int32), ("y0", c_int32), ("w", c_int32), ("h", c_int32),
                ("vertical", c_int32), ("polarity", c_int32), ("min_ink", c_int32), ("gap", c_int32), ("min_height", c_int32),
                ("pad", c_int32), ("hist", c_void_p), ("prof", c_void_p), ("scratch", c_void_p), ("out", c_void_p)]


class SkewBlock(Structure):
    _fields_ = [("b", TextBlock), ("table", c_void_p), ("scores", c_void_p), ("profiles", c_void_p), ("n_ang", c_int32),
                ("stride", c_int32), ("chosen", c_int32), ("L", c_int32), ("M", c_int32), ("pad", c_int32), ("u_min", c_double),
                ("v_min", c_double), ("c", c_double), ("s", c_double)]


# name -> (restype, argtypes); every symbol include/marconet_b200.h declares
SYMBOLS = {
    "mn_last_error": (c_char_p, []),
    "mn_version": (c_int, []),
    "mn_device_is_sm90": (c_int, []),
    "mn_set_max_ctas": (c_int, [c_int]),
    "mn_conv2d_nhwc": (c_int, [POINTER(ConvParams), c_void_p]),
    "mn_conv2d_plan": (c_int, [POINTER(ConvParams), POINTER(ConvPlan)]),
    "mn_groupnorm_stats": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p, c_void_p, c_void_p, c_void_p]),
    "mn_groupnorm_finalize": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p, c_void_p, c_void_p]),
    "mn_groupnorm_apply": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int,
                                   c_void_p, c_void_p]),
    "mn_conv_pack_weights_tc": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "mn_pixelnorm": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "mn_select_text": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_void_p]),
    "mn_set_pdl": (c_int, [c_int]),
    "mn_check_labels": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "mn_char_windows": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "mn_char_windows_ragged": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                       c_void_p]),
    "mn_demod": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "mn_demod_batched": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_void_p, c_int, c_int, c_void_p]),
    "mn_resample_modulate": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "mn_resample_modulate_ragged": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "mn_torgb": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "mn_groupnorm_swish": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int,
                                   c_float, c_int, c_void_p, c_void_p, c_void_p]),
    "mn_adain_concat": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "mn_window_scatter": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int,
                                  c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "mn_swish": (c_int, [c_void_p, c_void_p, c_longlong, c_void_p]),
    "mn_row_mean_std": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_float, c_void_p]),
    "mn_adain_rows": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "mn_layernorm": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_float, c_void_p]),
    "mn_linear_small_m": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_float, c_void_p]),
    "mn_linear_small_m_ex": (c_int, [c_void_p, c_longlong, c_longlong, c_int, c_longlong, c_void_p, c_void_p, c_void_p, c_longlong, c_void_p,
                                     c_int, c_int, c_int, c_int, c_int, c_float, c_void_p]),
    "mn_linear_small_m_ws": (c_int, [c_void_p, c_longlong, c_longlong, c_int, c_longlong, c_void_p, c_void_p, c_void_p, c_longlong, c_void_p,
                                     c_int, c_int, c_int, c_int, c_int, c_float, c_void_p, c_longlong, c_void_p]),
    "mn_preprocess_lq_u8": (c_int, [c_void_p, c_int, c_int, c_int, c_double, c_double, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "mn_postprocess_sr_u8": (c_int, [c_void_p, c_longlong, c_longlong, c_longlong, c_longlong, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "mn_preprocess_lq_u8_batched": (c_int, [c_void_p, c_int, c_int, c_void_p, c_int, c_int, c_void_p]),
    "mn_postprocess_sr_u8_pieces": (c_int, [c_void_p, c_longlong, c_longlong, c_longlong, c_longlong, c_int, c_int, c_int, c_void_p, c_int, c_int,
                                            c_void_p]),
    "mn_figure_u8": (c_int, [c_void_p, c_int, c_int, c_void_p]),
    "mn_decode_predictions": (c_int, [c_void_p, c_longlong, c_int, c_int, c_void_p, c_longlong, c_void_p, c_int, c_int, c_void_p]),
    "mn_decode_labels": (c_int, [c_void_p, c_longlong, c_int, c_int, c_void_p, c_int, c_int, c_void_p]),
    "mn_style_lerp": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_void_p, c_int, c_void_p]),
    "mn_prior_tiles_u8": (c_int, [c_void_p, c_longlong, c_longlong, c_longlong, c_longlong, c_void_p, c_int, c_void_p]),
    "mn_resize_cubic_u8_batched": (c_int, [c_void_p, c_int, c_int, c_longlong, c_void_p]),
    "mn_composite_regions_u8": (c_int, [c_void_p, c_int, c_longlong, c_void_p]),
    "mn_warp_affine_u8_batched": (c_int, [c_void_p, c_int, c_int, c_longlong, c_void_p]),
    "mn_composite_regions_affine_u8": (c_int, [c_void_p, c_int, c_longlong, c_void_p]),
    "mn_warp_perspective_u8_batched": (c_int, [c_void_p, c_int, c_int, c_longlong, c_void_p]),
    "mn_composite_regions_quad_u8": (c_int, [c_void_p, c_int, c_longlong, c_void_p]),
    "mn_vertical_layout_u8_batched": (c_int, [c_void_p, c_int, c_longlong, c_void_p]),
    "mn_vertical_unlayout_u8_batched": (c_int, [c_void_p, c_int, c_longlong, c_void_p]),
    "mn_remap_curved_u8_batched": (c_int, [c_void_p, c_int, c_int, c_longlong, c_void_p]),
    "mn_composite_regions_curved_u8": (c_int, [c_void_p, c_int, c_longlong, c_void_p]),
    "mn_find_lines_u8": (c_int, [c_void_p, c_int, c_longlong, c_void_p, c_longlong, c_void_p]),
    "mn_find_lines_skewed_u8": (c_int, [c_void_p, c_void_p, c_int, c_longlong, c_void_p, c_longlong, c_void_p]),
    "mn_token_mix": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_float, c_void_p]),
    "mn_attention": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_float, c_void_p]),
    "mn_nchw_to_nhwc": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "mn_nhwc_to_nchw": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
}

_lib = None


def load():
    """Load the shared library and bind every declared symbol. Raises RuntimeError when unavailable."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.isfile(LIB_PATH):
        raise RuntimeError(
            f"marconet_b200: CUDA library {LIB_PATH} is missing. Build it with "
            f"`python -m marconet_b200.build` (nvcc, sm_90a). There is no CPU/PyTorch fallback.")
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SYMBOLS.items():
        try:
            fn = getattr(lib, name)
        except AttributeError as e:
            raise RuntimeError(f"marconet_b200: symbol {name} missing from {LIB_PATH}") from e
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc, what):
    if rc != 0:
        msg = load().mn_last_error().decode(errors="replace")
        raise RuntimeError(f"{what} failed (status {rc}): {msg}")
