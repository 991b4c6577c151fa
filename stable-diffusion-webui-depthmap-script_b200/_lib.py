"""ctypes binding of include/depthmap_b200.h.  Fails loudly: no library -> ImportError-like RuntimeError, no GPU -> RuntimeError."""
from __future__ import annotations

import ctypes
import os
import sys
import threading

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("DEPTHMAP_B200_LIB", os.path.join(_HERE, "_native", "libdepthmap_b200.so"))

DM_OK, DM_E_INVALID, DM_E_CUDA, DM_E_OOM, DM_E_UNSUPPORTED, DM_E_WORKSPACE = 0, -1, -2, -3, -4, -5
DM_DEPTH_U16, DM_DEPTH_ND64 = 0, 1
DM_FILL = {"none": 0, "naive": 1, "naive_interpolating": 2, "polylines_soft": 3, "polylines_sharp": 4}
DM_EYE_WARP, DM_EYE_IDENTITY, DM_EYE_SKIP = 0, 1, 2
DM_PACK_STRIDED, DM_PACK_ANAGLYPH = 0, 1
DM_PNG_INVERT = 1


class StereoParams(ctypes.Structure):
    _fields_ = [
        ("div_px", ctypes.c_double * 2),
        ("sep_px", ctypes.c_double * 2),
        ("exponent", ctypes.c_double),
        ("eye_mode", ctypes.c_int32 * 2),
        ("fill", ctypes.c_int32),
        ("pack", ctypes.c_int32),
        ("anaglyph_red_eye", ctypes.c_int32),
        ("depth_kind", ctypes.c_int32),
        ("reserved", ctypes.c_int32),
        ("dst_row_stride", ctypes.c_int64 * 2),
        ("dst_img_stride", ctypes.c_int64 * 2),
    ]


class GemmDesc(ctypes.Structure):
    """mirror of dm_gemm_desc (include/depthmap_b200.h)"""
    _fields_ = [
        ("M", ctypes.c_int32), ("N", ctypes.c_int32), ("K", ctypes.c_int32),
        ("epi", ctypes.c_int32), ("act", ctypes.c_int32),
        ("bias", ctypes.c_void_p),
        ("C", ctypes.c_void_p), ("ldc", ctypes.c_int32),
        ("C2", ctypes.c_void_p),
        ("R", ctypes.c_void_p), ("ldr", ctypes.c_int32),
        ("R2", ctypes.c_void_p), ("ldr2", ctypes.c_int32),
        ("X", ctypes.c_void_p), ("ldx", ctypes.c_int32),
        ("gamma", ctypes.c_void_p),
        ("head_b2", ctypes.c_float),
        ("ps_s", ctypes.c_int32), ("ps_cout", ctypes.c_int32), ("ps_h", ctypes.c_int32), ("ps_w", ctypes.c_int32),
    ]


EPI_STORE_F16, EPI_RESID_F32, EPI_PIXSHUF, EPI_HEAD, EPI_STORE_F32 = 0, 1, 2, 3, 4
ACT_NONE, ACT_GELU, ACT_RELU = 0, 1, 2

_lock = threading.Lock()
_lib = None

# every symbol include/depthmap_b200.h declares; tests check the built library exports all of them
EXPORTS = [
    "dm_last_error", "dm_version", "dm_device_name",
    "dm_normalize_u16_workspace_bytes", "dm_normalize_u16", "dm_normalize_u16_outliers_workspace_bytes", "dm_normalize_u16_outliers",
    "dm_stereo_workspace_bytes", "dm_stereo", "dm_stereo_pack", "dm_depth_to_nd64", "dm_convert_to_i16_f64",
    "dm_normalmap_workspace_bytes", "dm_normalmap",
    "dm_gemm_ex", "dm_conv3x3_ex", "dm_gemm_f16", "dm_conv3x3_f16", "dm_attention_f16", "dm_attention_relpos_f16",
    "dm_preprocess_patchify", "dm_preprocess_patchify_f32_crops",
    "dm_assemble_tokens", "dm_layernorm_f16", "dm_resize_bilinear_nhwc_f16", "dm_resize_f32", "dm_im2col_s2_f16", "dm_concat_readout_f16",
    "dm_zoe_preprocess_patchify", "dm_layernorm_post_f16", "dm_attention_small_f16", "dm_cast_f32_f16", "dm_zoe_select_softplus",
    "dm_resize_add_nhwc_f16", "dm_zoe_attractor", "dm_zoe_clb_final", "dm_zoe_tta_combine",
    "dm_zoe_seed_bins", "dm_zoe_attractor_single", "dm_zoe_clb_single",
    "dm_video_workspace_bytes", "dm_video_blend", "dm_video_minmax", "dm_video_scale_f32", "dm_video_select_init", "dm_video_select_hist",
    "dm_video_select_pick", "dm_video_select_bounds", "dm_video_scale_f64",
    "dm_dinov2_pos_embed", "dm_beit_rel_table", "dm_vit_pos_embed",
    "dm_leres_stem_im2col", "dm_maxpool3x3s2_nhwc_f16", "dm_subsample2_nhwc_f16", "dm_add_f16", "dm_resize_f32_ld",
    "dm_boost_partials", "dm_unet_first_cols", "dm_unet_down_cols", "dm_unet_up_cols", "dm_unet_interleave", "dm_unet_final", "dm_unet_first", "dm_unet_last", "dm_sum_chunks_f32", "dm_boost_minmax",
    "dm_boost_merge_input", "dm_boost_post", "dm_boost_fit_sums", "dm_boost_blend", "dm_boost_resize_cubic", "dm_boost_u8_to_planar",
    "dm_leres_stem_im2col_f32", "dm_leres_stem_im2col_f32_batch", "dm_boost_minmax_normalise", "dm_boost_quantise_crops_u8",
    "dm_circular_halo_f16", "dm_conv3x3_circular_ex", "dm_im2col_s2_circular_f16", "dm_leres_stem_im2col_circular",
    "dm_leres_stem_im2col_f32_circular", "dm_leres_stem_im2col_f32_batch_circular",
    "dm_midas_stem_im2col", "dm_midas_stem_im2col_circular", "dm_midas_stem_im2col_f32_crops", "dm_midas_stem_im2col_f32_crops_circular",
    "dm_resize_bilinear_half_nhwc_f16",
    "dm_gemm_split_ex", "dm_conv3x3_split_ex", "dm_attention_split", "dm_preprocess_patchify_split", "dm_assemble_tokens_f32",
    "dm_layernorm_split", "dm_resize_bilinear_nhwc_split",
    "dm_preprocess_patchify_ragged", "dm_leres_stem_im2col_ragged", "dm_leres_stem_im2col_ragged_circular", "dm_midas_stem_im2col_ragged",
    "dm_midas_stem_im2col_ragged_circular", "dm_zoe_preprocess_patchify_ragged", "dm_resize_f32_ragged", "dm_zoe_tta_combine_ragged",
    "dm_png_encode_bound", "dm_png_encode_workspace_bytes", "dm_png_encode", "dm_depth_combine_rgb",
]


def load() -> ctypes.CDLL:
    global _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"depthmap_b200: native library missing ({LIB_PATH}). Build it with "
                f"`python {os.path.join(_HERE, 'csrc', 'build.py')}` — there is no CPU fallback.")
        L = ctypes.CDLL(LIB_PATH)
        c = ctypes
        vp, i32, i64, f32, sz = c.c_void_p, c.c_int, c.c_int64, c.c_float, c.c_size_t
        L.dm_last_error.restype = c.c_char_p
        L.dm_version.restype = i32
        L.dm_device_name.argtypes = [c.c_char_p, i32]
        L.dm_normalize_u16_workspace_bytes.argtypes = [i32]
        L.dm_normalize_u16_workspace_bytes.restype = sz
        L.dm_normalize_u16.argtypes = [vp, i32, i32, i32, i32, i32, f32, f32, vp, vp, vp, sz, vp]
        L.dm_normalize_u16_outliers_workspace_bytes.argtypes = [i32]
        L.dm_normalize_u16_outliers_workspace_bytes.restype = sz
        L.dm_normalize_u16_outliers.argtypes = [vp, i32, i32, i32, i32, ctypes.POINTER(ctypes.c_int64), ctypes.c_double, ctypes.c_double, vp, vp, vp, sz, vp]
        L.dm_stereo_workspace_bytes.argtypes = [i32, i32, i32]
        L.dm_stereo_workspace_bytes.restype = sz
        L.dm_stereo.argtypes = [vp, vp, i32, i32, i32, c.POINTER(StereoParams), vp, vp, vp, sz, vp]
        L.dm_stereo_pack.argtypes = [vp, i32, i32, i32, i32, vp, vp]
        L.dm_depth_to_nd64.argtypes = [vp, i32, i32, c.c_longlong, vp, vp, vp]
        L.dm_convert_to_i16_f64.argtypes = [vp, c.c_longlong, vp, vp]
        L.dm_normalmap_workspace_bytes.argtypes = [i32, i32, i32, i32, i32, i32]
        L.dm_normalmap_workspace_bytes.restype = sz
        L.dm_normalmap.argtypes = [vp, i32, i32, i32, i32, i32, i32, i32, vp, vp, sz, vp]
        if hasattr(L, "dm_video_blend"):
            ll, dbl = c.c_longlong, c.c_double
            L.dm_video_workspace_bytes.restype = sz
            L.dm_video_blend.argtypes = [vp, ll, i32, i32, i32, i32, i32, vp, vp]
            L.dm_video_minmax.argtypes = [vp, ll, vp, vp, sz, vp]
            L.dm_video_scale_f32.argtypes = [vp, ll, vp, vp, vp]
            L.dm_video_select_init.argtypes = [vp, c.POINTER(ll), vp]
            L.dm_video_select_hist.argtypes = [vp, ll, i32, vp, vp]
            L.dm_video_select_pick.argtypes = [vp, i32, vp]
            L.dm_video_select_bounds.argtypes = [vp, dbl, dbl, vp, vp]
            L.dm_video_scale_f64.argtypes = [vp, ll, vp, vp, vp]
        L.dm_dinov2_pos_embed.argtypes = [vp, i32, i32, i32, i32, vp]
        L.dm_beit_rel_table.argtypes = [vp, i32, i32, i32, i32, vp]
        L.dm_vit_pos_embed.argtypes = [vp, i32, i32, i32, i32, vp]
        _bind_optional(L)
        _lib = L
        return L


def _bind_optional(L):
    """Model entry points (present once the tensor-core units are linked in)."""
    c = ctypes
    vp, i32, i64, f32, sz = c.c_void_p, c.c_int, c.c_int64, c.c_float, c.c_size_t
    if hasattr(L, "dm_gemm_f16"):
        L.dm_gemm_f16.argtypes = [vp, i32, vp, i32, vp, vp, i32, i32, i32, i32, i32, i32, vp]
        L.dm_conv3x3_f16.argtypes = [vp, i32, i32, i32, i32, vp, vp, vp, i32, i32, vp]
        L.dm_gemm_ex.argtypes = [vp, i32, vp, i32, c.POINTER(GemmDesc), vp]
        L.dm_conv3x3_ex.argtypes = [vp, i32, i32, i32, i32, vp, c.POINTER(GemmDesc), vp]
        L.dm_circular_halo_f16.argtypes = [vp, i32, i32, i32, i32, vp, vp]
        L.dm_conv3x3_circular_ex.argtypes = [vp, vp, i32, i32, i32, i32, vp, c.POINTER(GemmDesc), vp]
        L.dm_gemm_split_ex.argtypes = [vp, i32, vp, i32, vp, c.POINTER(GemmDesc), vp]
        L.dm_conv3x3_split_ex.argtypes = [vp, vp, i32, i32, i32, i32, vp, vp, c.POINTER(GemmDesc), vp]
    if hasattr(L, "dm_attention_f16"):
        L.dm_attention_f16.argtypes = [vp, i32, i32, i32, f32, vp, i32, vp, vp]
        L.dm_attention_relpos_f16.argtypes = [vp, i32, i32, i32, i32, f32, vp, i32, vp, vp]
        L.dm_attention_split.argtypes = [vp, i32, i32, i32, f32, vp, vp]
    if hasattr(L, "dm_layernorm_f16"):
        L.dm_preprocess_patchify.argtypes = [vp, i32, i32, i32, i32, i32, i32, c.POINTER(c.c_float), c.POINTER(c.c_float),
                                             c.POINTER(c.c_int), vp, i32, vp]
        L.dm_preprocess_patchify_f32_crops.argtypes = [vp, i32, i32, vp, i32, i32, i32, i32, c.POINTER(c.c_float), c.POINTER(c.c_float),
                                                       c.POINTER(c.c_int), vp, i32, vp]
        L.dm_assemble_tokens.argtypes = [vp, vp, vp, vp, i32, i32, i32, vp]
        L.dm_layernorm_f16.argtypes = [vp, c.c_longlong, i32, vp, vp, f32, vp, i32, i32, vp]
        L.dm_resize_bilinear_nhwc_f16.argtypes = [vp, i32, i32, i32, i32, vp, i32, i32, vp]
        L.dm_preprocess_patchify_split.argtypes = L.dm_preprocess_patchify.argtypes
        L.dm_assemble_tokens_f32.argtypes = L.dm_assemble_tokens.argtypes
        L.dm_layernorm_split.argtypes = L.dm_layernorm_f16.argtypes
        L.dm_resize_bilinear_nhwc_split.argtypes = L.dm_resize_bilinear_nhwc_f16.argtypes
        L.dm_resize_f32.argtypes = [vp, i32, i32, i32, vp, i32, i32, i32, vp]
        L.dm_im2col_s2_f16.argtypes = [vp, i32, i32, i32, i32, vp, vp]
        L.dm_im2col_s2_circular_f16.argtypes = [vp, i32, i32, i32, i32, vp, vp]
        L.dm_concat_readout_f16.argtypes = [vp, i32, i32, i32, vp, vp]
    if hasattr(L, "dm_leres_stem_im2col"):
        L.dm_leres_stem_im2col.argtypes = [vp, i32, i32, i32, i32, i32, c.POINTER(c.c_float), c.POINTER(c.c_float), vp, vp]
        L.dm_leres_stem_im2col_circular.argtypes = L.dm_leres_stem_im2col.argtypes
        L.dm_maxpool3x3s2_nhwc_f16.argtypes = [vp, i32, i32, i32, i32, vp, vp]
        L.dm_subsample2_nhwc_f16.argtypes = [vp, i32, i32, i32, i32, vp, vp]
        L.dm_add_f16.argtypes = [vp, vp, vp, c.c_longlong, vp]
        L.dm_resize_f32_ld.argtypes = [vp, i32, i32, i32, i32, vp, i32, i32, i32, vp]
    if hasattr(L, "dm_midas_stem_im2col"):
        fp, ip = c.POINTER(c.c_float), c.POINTER(c.c_int)
        L.dm_midas_stem_im2col.argtypes = [vp, i32, i32, i32, i32, i32, fp, fp, ip, vp, vp]
        L.dm_midas_stem_im2col_circular.argtypes = L.dm_midas_stem_im2col.argtypes
        L.dm_midas_stem_im2col_f32_crops.argtypes = [vp, i32, i32, vp, i32, i32, i32, fp, fp, ip, vp, vp]
        L.dm_midas_stem_im2col_f32_crops_circular.argtypes = L.dm_midas_stem_im2col_f32_crops.argtypes
        L.dm_resize_bilinear_half_nhwc_f16.argtypes = [vp, i32, i32, i32, i32, vp, i32, i32, vp]
    if hasattr(L, "dm_unet_first_cols"):
        ll = c.c_longlong
        L.dm_unet_first_cols.argtypes = [vp, i32, i32, vp, i32, vp]
        L.dm_unet_down_cols.argtypes = [vp, i32, i32, i32, vp, i32, vp]
        L.dm_unet_up_cols.argtypes = [vp, i32, vp, i32, i32, i32, vp, i32, vp]
        L.dm_unet_interleave.argtypes = [vp, i32, i32, i32, i32, vp, vp]
        L.dm_unet_final.argtypes = [vp, i32, i32, i32, f32, vp, vp]
        L.dm_boost_minmax.argtypes = [vp, ll, vp, vp]
        L.dm_sum_chunks_f32.argtypes = [vp, i32, ll, i32, vp, vp, vp]
        L.dm_unet_first.argtypes = [vp, i32, i32, vp, vp, vp]
        L.dm_unet_last.argtypes = [vp, i32, vp, i32, i32, i32, vp, f32, vp, vp]
        L.dm_boost_merge_input.argtypes = [vp, vp, ll, vp, vp, vp, vp]
        L.dm_boost_post.argtypes = [vp, ll, vp, i32, vp, vp]
        L.dm_boost_fit_sums.argtypes = [vp, vp, ll, vp, vp]
        L.dm_boost_minmax_normalise.argtypes = [vp, ll, vp, vp, vp, vp]
        L.dm_boost_blend.argtypes = [vp, i32, vp, vp, i32, vp, i32, i32, i32, i32, i32, vp]
        L.dm_boost_resize_cubic.argtypes = [vp, i32, ll, i32, i32, vp, i32, ll, i32, i32, i32, vp]
        L.dm_boost_u8_to_planar.argtypes = [vp, i32, i32, vp, vp]
        L.dm_boost_quantise_crops_u8.argtypes = [vp, i32, i32, vp, i32, i32, i32, vp, vp]
        L.dm_leres_stem_im2col_f32.argtypes = [vp, i32, i32, i32, i32, i32, i32, i32, i32, c.POINTER(c.c_float), c.POINTER(c.c_float), vp, vp]
        L.dm_leres_stem_im2col_f32_batch.argtypes = [vp, i32, i32, vp, i32, i32, i32, c.POINTER(c.c_float), c.POINTER(c.c_float), vp, vp]
        L.dm_leres_stem_im2col_f32_circular.argtypes = L.dm_leres_stem_im2col_f32.argtypes
        L.dm_leres_stem_im2col_f32_batch_circular.argtypes = L.dm_leres_stem_im2col_f32_batch.argtypes
    if hasattr(L, "dm_zoe_clb_final"):
        L.dm_zoe_preprocess_patchify.argtypes = [vp, i32, i32, i32, i32, i32, i32, i32, i32, vp, i32, vp]
        L.dm_layernorm_post_f16.argtypes = [vp, c.c_longlong, i32, vp, vp, f32, vp, vp]
        L.dm_attention_small_f16.argtypes = [vp, i32, i32, i32, f32, vp, vp]
        L.dm_cast_f32_f16.argtypes = [vp, c.c_longlong, vp, vp]
        L.dm_zoe_select_softplus.argtypes = [vp, i32, vp, i32, i32, i32, vp, vp]
        L.dm_resize_add_nhwc_f16.argtypes = [vp, vp, i32, i32, i32, i32, vp, i32, i32, vp]
        L.dm_zoe_attractor.argtypes = [vp, i32, vp, i32, vp, i32, i32, i32, i32, i32, vp, vp]
        L.dm_zoe_clb_final.argtypes = [vp, i32, vp, i32, vp, vp, i32, vp, vp, vp, vp, i32, i32, i32, i32, i32, f32, f32, vp, vp]
        L.dm_zoe_tta_combine.argtypes = [vp, i32, i32, i32, i32, i32, i32, i32, vp, vp]
        L.dm_zoe_seed_bins.argtypes = [vp, i32, c.c_longlong, i32, f32, f32, vp, vp]
        L.dm_zoe_attractor_single.argtypes = [vp, i32, i32, i32, vp, i32, i32, i32, i32, i32, i32, f32, f32, vp, vp]
        L.dm_zoe_clb_single.argtypes = [vp, i32, vp, i32, vp, vp, vp, vp, vp, vp, f32, i32, i32, i32, i32, i32, f32, f32, vp, vp]
    if hasattr(L, "dm_resize_f32_ragged"):
        _bind_ragged(L)
    if hasattr(L, "dm_png_encode"):
        L.dm_png_encode_bound.argtypes = [i32, i32, i32, i32]
        L.dm_png_encode_bound.restype = sz
        L.dm_png_encode_workspace_bytes.argtypes = [i32, i32, i32, i32, i32]
        L.dm_png_encode_workspace_bytes.restype = sz
        L.dm_png_encode.argtypes = [vp, i32, i32, i32, i32, i32, i32, vp, sz, vp, vp, sz, vp]
        L.dm_depth_combine_rgb.argtypes = [vp, vp, i32, i32, i32, i32, i32, vp, vp]


def _bind_ragged(L):
    """the ragged-batch twins (include/depthmap_b200.h): packed buffer, its size, host and device descriptors, then the twin's own
    arguments"""
    c = ctypes
    vp, i32, ll, fp, ip = c.c_void_p, c.c_int, c.c_longlong, c.POINTER(c.c_float), c.POINTER(c.c_int)
    rag = [vp, ll, vp, vp, i32]
    L.dm_preprocess_patchify_ragged.argtypes = rag + [i32, i32, i32, fp, fp, ip, i32, vp, i32, vp]
    L.dm_leres_stem_im2col_ragged.argtypes = rag + [i32, i32, fp, fp, vp, vp]
    L.dm_leres_stem_im2col_ragged_circular.argtypes = L.dm_leres_stem_im2col_ragged.argtypes
    L.dm_midas_stem_im2col_ragged.argtypes = rag + [i32, i32, fp, fp, ip, vp, vp]
    L.dm_midas_stem_im2col_ragged_circular.argtypes = L.dm_midas_stem_im2col_ragged.argtypes
    L.dm_zoe_preprocess_patchify_ragged.argtypes = rag + [i32, i32, i32, vp, i32, vp]
    L.dm_resize_f32_ragged.argtypes = [vp, i32, i32, i32, vp, ll, vp, vp, i32, vp]
    L.dm_zoe_tta_combine_ragged.argtypes = [vp, i32, i32, i32, vp, ll, vp, vp, vp]


class Ragged:
    """A ragged image list for the *_ragged entry points: `sizes` [(h, w)] packed back to back from offset 0, `unit` elements per
    pixel (3 for uint8 RGB, 1 for an fp32 map).  `host` is the dm_ragged_image array (int64 offset, int32 h, int32 w per image),
    `dev` its copy on `device` (None without a device: a layout only); `size` the packed element count."""

    def __init__(self, sizes, unit, device):
        import torch
        self.sizes = [(int(h), int(w)) for h, w in sizes]
        self.B, self.unit = len(self.sizes), unit
        rec = np.zeros(self.B, dtype=[("offset", "<i8"), ("h", "<i4"), ("w", "<i4")])
        off = 0
        self.offsets = []
        for i, (h, w) in enumerate(self.sizes):
            rec[i] = (off, h, w)
            self.offsets.append(off)
            off += h * w * unit
        self.size = off
        self.host = rec
        self.dev = torch.from_numpy(rec.view(np.uint8).copy()).to(device) if device is not None else None

    def args(self, packed):
        """(packed buffer, size, host descriptors, device descriptors, B): the leading arguments of every ragged entry point"""
        return packed, self.size, self.host.ctypes.data, self.dev, self.B

    def split(self, packed):
        """views of the B images of a packed tensor of this layout: [h, w] (unit 1) or [h, w, 3] (unit 3)"""
        shape = () if self.unit == 1 else (self.unit,)
        return [packed[o:o + h * w * self.unit].view(h, w, *shape) for o, (h, w) in zip(self.offsets, self.sizes)]


def check(rc: int, what: str = ""):
    if rc == DM_OK:
        return
    msg = load().dm_last_error().decode("utf-8", "replace")
    if rc == DM_E_OOM:
        raise RuntimeError(f"CUDA out of memory. {msg}")  # src/core.py:310 matches 'out of memory'
    if rc == DM_E_INVALID:
        raise ValueError(msg or what)
    if rc == DM_E_UNSUPPORTED:
        raise NotImplementedError(msg or what)
    raise RuntimeError(f"depthmap_b200 {what} failed ({rc}): {msg}")


def require_cuda():
    import torch
    if not torch.cuda.is_available():
        raise RuntimeError("depthmap_b200: no CUDA device visible; the H100 kernels have no CPU fallback")
    return torch.device("cuda", torch.cuda.current_device())


def stream_ptr():
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return t.data_ptr() if t is not None else None


def _gemm_desc(M, N, K, epi, act, bias, C, ldc, C2, R, ldr, R2, ldr2, X, ldx, gamma, head_b2, ps=None):
    return GemmDesc(M, N, K, epi, act, _ptr(bias), _ptr(C), ldc, _ptr(C2), _ptr(R), ldr, _ptr(R2), ldr2, _ptr(X), ldx, _ptr(gamma), head_b2,
                    *(ps or (0, 0, 0, 0)))


class Ops:
    """Checked kernel calls on the current torch stream, with a running count of the kernels they issue (`launches`)."""

    def __init__(self):
        import torch
        self._tensor = torch.Tensor
        self.L = load()
        for name in ("dm_gemm_ex", "dm_conv3x3_ex", "dm_attention_f16", "dm_layernorm_f16"):
            if not hasattr(self.L, name):
                raise RuntimeError(f"depthmap_b200: native library lacks {name}; rebuild csrc (no fallback exists)")
        self.launches = 0

    def call(self, name, *args, launches=1):
        """L.name(*args, stream): a tensor goes in as its data pointer, None as NULL; a status other than DM_OK raises.
        `launches`: the kernels this call issues."""
        T = self._tensor
        check(getattr(self.L, name)(*[a.data_ptr() if isinstance(a, T) else a for a in args], stream_ptr()), name)
        self.launches += launches

    def gemm(self, A, lda, W, ldw, M, N, K, epi=EPI_STORE_F16, act=ACT_NONE, bias=None, C=None, ldc=0, C2=None,
             R=None, ldr=0, R2=None, ldr2=0, X=None, ldx=0, gamma=None, head_b2=0.0, ps=None):
        d = _gemm_desc(M, N, K, epi, act, bias, C, ldc, C2, R, ldr, R2, ldr2, X, ldx, gamma, head_b2, ps)
        self.call("dm_gemm_ex", A, lda, W, ldw, ctypes.byref(d))

    def conv3x3(self, act_t, B, H, W_, Cin, Wt, Cout, epi=EPI_STORE_F16, act=ACT_NONE, bias=None, C=None, C2=None,
                R=None, R2=None, X=None, gamma=None, head_b2=0.0, ldx=1, halo=None):
        """pad-1 3x3 convolution; with a `halo` scratch tensor (at least B*(H+2)*(W_+2)*Cin fp16) the padding is circular"""
        d = _gemm_desc(0, Cout, 0, epi, act, bias, C, Cout, C2, R, Cout, R2, Cout, X, ldx, gamma, head_b2)
        if halo is None:
            self.call("dm_conv3x3_ex", act_t, B, H, W_, Cin, Wt, ctypes.byref(d))
        else:
            if halo.numel() < B * (H + 2) * (W_ + 2) * Cin:
                raise ValueError(f"conv3x3: halo scratch of {halo.numel()} elements is too small for [{B}, {H + 2}, {W_ + 2}, {Cin}]")
            self.call("dm_conv3x3_circular_ex", act_t, halo, B, H, W_, Cin, Wt, ctypes.byref(d), launches=2)


    def gemm_split(self, A, lda, W, ldw, wscale, M, N, K, epi=EPI_STORE_F16, act=ACT_NONE, bias=None, C=None, ldc=0, C2=None,
                   R=None, ldr=0, R2=None, ldr2=0, X=None, ldx=0, gamma=None, head_b2=0.0, ps=None):
        """split-mode GEMM (dm_gemm_split_ex): A, W split operands of depth K (3x the logical one), wscale the weights' [N] factor;
        ldc / ldr / ldr2 are the split rows' pitches (>= 3N)"""
        d = _gemm_desc(M, N, K, epi, act, bias, C, ldc, C2, R, ldr, R2, ldr2, X, ldx, gamma, head_b2, ps)
        self.call("dm_gemm_split_ex", A, lda, W, ldw, wscale, ctypes.byref(d))

    def conv3x3_split(self, act_t, B, H, W_, Cin, Wt, wscale, Cout, epi=EPI_STORE_F16, act=ACT_NONE, bias=None, C=None, C2=None,
                      R=None, R2=None, X=None, gamma=None, head_b2=0.0, ldx=1, halo=None):
        """split-mode pad-1 3x3 convolution on split NHWC activations (Cin, Cout logical); circular padding with a `halo` scratch
        of at least B*(H+2)*(W_+2)*3*Cin fp16"""
        d = _gemm_desc(0, Cout, 0, epi, act, bias, C, 3 * Cout, C2, R, 3 * Cout, R2, 3 * Cout, X, ldx, gamma, head_b2)
        if halo is not None and halo.numel() < B * (H + 2) * (W_ + 2) * 3 * Cin:
            raise ValueError(f"conv3x3_split: halo scratch of {halo.numel()} elements is too small for [{B}, {H + 2}, {W_ + 2}, {3 * Cin}]")
        self.call("dm_conv3x3_split_ex", act_t, halo, B, H, W_, Cin, Wt, wscale, ctypes.byref(d), launches=1 if halo is None else 2)


class GraphCache:
    """CUDA-graph replay of a fixed launch sequence, keyed by shape.  At a key, the first call runs eagerly (it allocates), the
    second captures and later calls replay; inside a capture someone else started the kernels are plain launches.  A failed
    capture is reported once and leaves the caller eager: the graph is an optimisation over the same kernels.  A replay adds the
    captured kernels to ops.launches.  `env` = "0" keeps everything eager."""

    def __init__(self, ops, env, what):
        self.ops, self.what = ops, what
        self.enabled = os.environ.get(env, "1") != "0"
        self._graphs, self._calls = {}, {}

    def clear(self):
        self._graphs.clear()
        self._calls.clear()

    def run(self, key, fn, *inputs, copy_out=False):
        """fn(*inputs) -> output tensor.  A replay copies `inputs` into the captured ones and returns the captured output buffer,
        which the next replay at this key overwrites, or with copy_out a copy of it."""
        import torch
        capturing = torch.cuda.is_current_stream_capturing()
        g = self._graphs.get(key)
        if g is not None and not capturing:
            graph, static_in, out, n = g
            for s, x in zip(static_in, inputs):
                s.copy_(x)
            graph.replay()
            self.ops.launches += n
            return out.clone() if copy_out else out
        calls = self._calls[key] = self._calls.get(key, 0) + 1
        if self.enabled and calls >= 2 and not capturing:
            try:
                graph = torch.cuda.CUDAGraph()
                static_in = [x.clone() for x in inputs]
                n0 = self.ops.launches
                with torch.cuda.graph(graph):
                    out = fn(*static_in)
                self._graphs[key] = (graph, static_in, out, self.ops.launches - n0)
                graph.replay()
                return out.clone() if copy_out else out
            except Exception as e:  # noqa: BLE001 — an optimisation only: the same kernels run eagerly
                sys.stderr.write(f"[depthmap_b200] {self.what} graph capture failed ({e}); running eagerly\n")
                torch.cuda.synchronize()
                self.enabled = False
        return fn(*inputs)
