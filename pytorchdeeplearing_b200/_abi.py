"""ctypes binding of ``libb200seg.so`` (C ABI: ``include/b200seg.h``) -- the ONLY product backend.

``CudaBackend`` exposes one method per ``b200seg_*`` entry point with torch tensors as
arguments; it extracts raw device pointers / shapes / pitches and passes the current CUDA
stream.  PyTorch is plumbing here (allocator, streams); no torch operator computes anything.
"""
from __future__ import annotations

import ctypes as C
import os
import struct
import threading
from typing import Optional

import torch

K3, K1, DOWN, UP = 0, 1, 2, 3
F32, BF16, BF16_TC, BF16_HALO, BF16_HALO_WS = 0, 1, 2, 3, 4
I64 = 16
U8, I32 = 17, 18          # mask dtypes of the segmentation metrics
I16 = 19                  # volumes of the whole-volume resample
NORM_NONE, NORM_MEANSTD, NORM_PCTL = 0, 1, 2
# operations of b200seg_morphology (B200SEG_MORPH_*) and its largest radius
MORPH_OPS = {"dilate": 0, "erode": 1, "open": 2, "close": 3}
MORPH_MAX_RADIUS = 64
# kernel families of b200seg_conv / b200seg_wgrad (include/b200seg.h: B200SEG_CONV_*, B200SEG_WGRAD_*)
CONV_PATHS = ("PW_MMA", "TC", "HALO2D", "HALO3", "HALO_WS", "STEM_MMA", "STEM", "SMALLCIN", "GENERIC")
WGRAD_PATHS = ("HALO_MMA", "TC", "STEM_MMA", "STEM", "SMALLCIN", "GENERIC")
# output tile geometries of the HALO_WS family (B200SEG_WS_GEOM_*): 8 x 16 column tiles, flattened padded rows
HALO_WS_GEOMS = ("COLUMN", "FLAT")
# voxels per sample a 3x3x3 layer needs before its weights are packed for the halo-staged kernels (16/32 channels)
# and the weight-streaming halo kernel (64/128 channels); smaller layers take the TMA implicit-GEMM kernel
HALO_MIN_VOX = 128 * 128
HALO_WS_MIN_VOX = 1000

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libb200seg.so")


class TensorDesc(C.Structure):
    _fields_ = [("ptr", C.c_void_p), ("n", C.c_int32), ("d", C.c_int32), ("h", C.c_int32), ("w", C.c_int32),
                ("c", C.c_int32), ("ld", C.c_int64), ("dtype", C.c_int32)]


class PackDesc(C.Structure):   # include/b200seg.h: struct b200seg_pack_desc
    _fields_ = [("src", C.c_void_p), ("dst", C.c_void_p), ("st", C.c_int64), ("sk", C.c_int64), ("sn2", C.c_int64),
                ("sn1", C.c_int64), ("out_dtype", C.c_int32), ("T", C.c_int32), ("K", C.c_int32), ("N2", C.c_int32),
                ("N1", C.c_int32), ("flip", C.c_int32), ("block_start", C.c_int32), ("nblocks", C.c_int32)]


# activation after the norm (B200SEG_ACT_*): nn.ReLU, nn.LeakyReLU(0.01)
ACT_RELU, ACT_LEAKY = 0, 1


class GnDesc(C.Structure):     # include/b200seg.h: struct b200seg_gn
    _fields_ = [("stats", C.c_void_p), ("gamma", C.c_void_p), ("beta", C.c_void_p), ("scale", C.c_void_p),
                ("groups", C.c_int32), ("vox", C.c_int64), ("eps", C.c_float), ("act", C.c_int32)]


_PT = C.POINTER(TensorDesc)
_PG = C.POINTER(GnDesc)
_vp, _i, _i64, _f, _d = C.c_void_p, C.c_int, C.c_int64, C.c_float, C.c_double

_SIGNATURES = {
    "b200seg_version": ([], C.c_int),
    "b200seg_last_error": ([], C.c_char_p),
    "b200seg_init": ([_i], C.c_int),
    "b200seg_pack_weight": ([_vp, _vp, _i, _i, _i, _i, _i, _i64, _i64, _i64, _i64, _i, _i, _vp], C.c_int),
    "b200seg_unpack_wgrad": ([_vp, _vp, _i, _i, _i, _i64, _i64, _i64, _i, _vp], C.c_int),
    "b200seg_pack_weights_multi": ([_vp, _i, _i, _i, _vp], C.c_int),
    "b200seg_unpack_wgrads_multi": ([_vp, _i, _i, _i, _vp], C.c_int),
    "b200seg_upload_table": ([_vp, _i64, _vp, _i, _vp], C.c_int),
    "b200seg_conv": ([_i, _i, _PT, _vp, _i, _vp, _PT, _vp, _PT, _i, _vp], C.c_int),
    "b200seg_conv_path": ([_i, _i, _PT, _i, _PT, _PT], C.c_int),
    "b200seg_conv_halo_ws_geometry": ([_i, _i, _PT, _i, _PT, _PT], C.c_int),
    "b200seg_conv_bwdstats_supported": ([_i, _i, _PT, _i, _PT, _PT, _PT], C.c_int),
    "b200seg_conv_bwdstats": ([_i, _i, _PT, _vp, _i, _PT, _PT, _PT, _PG, _vp, _i, _vp], C.c_int),
    "b200seg_conv_tc_eligible": ([_i, _i, _i], C.c_int),
    "b200seg_conv_halo_eligible": ([_i, _i, _i], C.c_int),
    "b200seg_conv_halo_ws_ntile": ([_i, _i, _i], C.c_int),
    "b200seg_wgrad": ([_i, _i, _PT, _PT, _vp, _i, _vp], C.c_int),
    "b200seg_wgrad_path": ([_i, _i, _PT, _PT], C.c_int),
    "b200seg_gn_finalize": ([_vp, _vp, _vp, _vp, _i, _i, _i, _i64, _f, _vp, _vp, _i, _vp], C.c_int),
    "b200seg_apply": ([_PT, _vp, _PT, _vp, _PT, _PT, _i, _vp], C.c_int),
    "b200seg_apply_gn": ([_PT, _PG, _PT, _PG, _PT, _PT, _i, _vp], C.c_int),
    "b200seg_gn_bwd_reduce_gn": ([_PT, _PT, _PG, _vp, _i, _vp], C.c_int),
    "b200seg_gn_bwd_apply_gn": ([_PT, _PT, _PG, _vp, _PT, _vp, _vp, _vp, _i, _i, _vp], C.c_int),
    "b200seg_gn_bwd_fused_supported": ([_PT, _PT, _PT, _i], C.c_int),
    "b200seg_gn_bwd_fused_gn": ([_PT, _PT, _PG, _vp, _vp, _PT, _vp, _vp, _vp, _i, _vp], C.c_int),
    "b200seg_gn_bwd_reduce": ([_PT, _PT, _vp, _vp, _i, _vp], C.c_int),
    "b200seg_gn_bwd_finalize": ([_vp, _vp, _vp, _vp, _i, _i, _i, _i64, _vp, _vp, _vp, _vp, _i, _vp], C.c_int),
    "b200seg_gn_bwd_apply": ([_PT, _PT, _vp, _vp, _PT, _i, _vp], C.c_int),
    "b200seg_colsum": ([_PT, _vp, _i, _vp], C.c_int),
    "b200seg_pool_fwd": ([_PT, _PT, _i, _i, _vp], C.c_int),
    "b200seg_pool_bwd": ([_PT, _PT, _PT, _PT, _i, _i, _vp], C.c_int),
    "b200seg_upsample2_add": ([_PT, _PT, _PT, _i, _vp], C.c_int),
    "b200seg_upsample2_bwd": ([_PT, _PT, _i, _vp], C.c_int),
    "b200seg_head_probs": ([_vp, _vp, _i64, _i, _i, _vp], C.c_int),
    "b200seg_head_fwd": ([_PT, _vp, _vp, _vp, _vp, _i, _i, _vp], C.c_int),
    "b200seg_stem_gn_supported": ([_PT, _i, _i], C.c_int),
    "b200seg_stem_gn_stats": ([_PT, _vp, _vp, _vp, _vp, _vp, _vp, _i, _vp], C.c_int),
    "b200seg_stem_gn_apply": ([_PT, _vp, _vp, _vp, _vp, _PG, _PG, _PT, _i, _vp], C.c_int),
    "b200seg_stem_gn_bwd_sums": ([_PT, _vp, _vp, _vp, _vp, _PG, _PG, _PT, _vp, _vp, _i, _vp], C.c_int),
    "b200seg_stem_gn_bwd": ([_PT, _vp, _vp, _vp, _vp, _PG, _PG, _PT, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _vp],
                            C.c_int),
    "b200seg_up_gn_supported": ([_PT, _i, _i], C.c_int),
    "b200seg_up_gn_stats": ([_PT, _vp, _vp, _vp, _i, _vp], C.c_int),
    "b200seg_up_gn_apply": ([_PT, _vp, _vp, _PG, _PT, _i, _vp], C.c_int),
    "b200seg_up_gn_bwd_sums": ([_PT, _vp, _vp, _PG, _PT, _vp, _i, _vp], C.c_int),
    "b200seg_up_gn_bwd": ([_PT, _vp, _vp, _PG, _PT, _vp, _vp, _PT, _vp, _vp, _vp, _i, _vp], C.c_int),
    "b200seg_head_bwd_supported": ([_i, _i], C.c_int),
    "b200seg_head_bwd": ([_PT, _vp, _vp, _PT, _vp, _vp, _i, _i, _vp], C.c_int),
    "b200seg_loss_partials": ([_vp, _vp, _i, _i, _i64, _i, _f, _f, _vp, _vp, _i, _vp], C.c_int),
    "b200seg_loss_finalize": ([_vp, _i, _i, _vp, _f, _f, _vp, _vp, _i, _vp], C.c_int),
    "b200seg_loss_bwd": ([_vp, _vp, _i, _i64, _i, _vp, _vp, _vp, _i, _vp], C.c_int),
    "b200seg_loss_partials_ss": ([_vp, _vp, _i, _i, _i64, _vp, _vp, _i, _vp], C.c_int),
    "b200seg_loss_bwd_ss": ([_vp, _vp, _i, _i64, _vp, _vp, _vp, _i, _vp], C.c_int),
    "b200seg_radix_sort_workspace": ([_i, _i64], C.c_int64),
    "b200seg_radix_sort_pairs": ([_vp, _vp, _vp, _vp, _i, _i64, _vp, _i64, _i, _vp], C.c_int),
    "b200seg_lovasz_workspace": ([_i, _i64, _i, _i], C.c_int64),
    "b200seg_lovasz_fwd": ([_vp, _vp, _i, _i64, _i, _i, _i, _i64, _vp, _i64, _vp, _vp, _vp, _i, _vp], C.c_int),
    "b200seg_lovasz_bwd": ([_vp, _vp, _i, _i64, _i, _i, _vp, _vp, _vp, _vp, _i, _vp], C.c_int),
    "b200seg_lovasz_hinge_workspace": ([_i, _i64, _i], C.c_int64),
    "b200seg_lovasz_hinge_fwd": ([_vp, _vp, _i, _i64, _i, _i, _i64, _vp, _i64, _vp, _vp, _vp, _i, _vp], C.c_int),
    "b200seg_lovasz_hinge_bwd": ([_vp, _i64, _vp, _vp, _i, _vp], C.c_int),
    "b200seg_segmetric3d_workspace": ([_i, _i, _i, _i], C.c_int64),
    "b200seg_segmetric3d": ([_vp, _i, _vp, _i, _i, _i, _i, _i, _vp, _vp, _i64, _vp, _vp, _vp, _i, _vp], C.c_int),
    "b200seg_segmetric3d_points": ([_vp, _i, _vp, _i, _i, _i, _i, _i, _vp, _vp, _i64, _i64, _i64, _vp, _vp, _vp, _vp,
                                    _i, _vp], C.c_int),
    "b200seg_ssim_workspace": ([_i, _i, _i, _i, _i, _i, _i], C.c_int64),
    "b200seg_ssim_fwd": ([_i, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp, _vp, _vp, _i64, _i, _vp], C.c_int),
    "b200seg_ssim_finalize": ([_i, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _i64, _vp, _vp, _i, _vp], C.c_int),
    "b200seg_ssim_bwd": ([_i, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp, _vp, _i, _vp, _vp, _vp, _vp, _i, _vp],
                         C.c_int),
    "b200seg_cldice_workspace": ([_i, _i, _i, _i, _i], C.c_int64),
    "b200seg_cldice_skeleton": ([_vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp, _i, _vp, _vp, _vp, _i, _vp, _i64, _i, _vp],
                                C.c_int),
    "b200seg_cldice_finalize": ([_i, _i, _i, _i, _i, _i, _i, _vp, _d, _d, _i, _vp, _i64, _vp, _vp, _i, _vp], C.c_int),
    "b200seg_cldice_bwd": ([_vp, _vp, _i, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _vp],
                           C.c_int),
    "b200seg_cldice_norm": ([_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp, _vp, _i, _vp], C.c_int),
    "b200seg_cldice_norm_bwd": ([_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _i, _vp], C.c_int),
    "b200seg_metric_partials": ([_vp, _vp, _i, _i, _i64, _i, _f, _vp, _i, _vp], C.c_int),
    "b200seg_metric_finalize": ([_vp, _i, _i, _vp, _i, _vp], C.c_int),
    "b200seg_adam_step": ([_vp, _vp, _vp, _vp, _i64, _vp, _d, _d, _d, _f, _d, _i, _vp, _i, _i, _vp], C.c_int),
    "b200seg_dropout_masks": ([_vp, _vp, _i, _i, C.c_double, _vp, _i, _vp], C.c_int),
    "b200seg_head_mask": ([_PT, _vp, _vp, _vp, _i, _f, _i, _vp], C.c_int),
    "b200seg_mask_logits": ([_vp, _i64, _i, _f, _vp, _i, _vp], C.c_int),
    "b200seg_cls_head_fwd": ([_PT, _vp, _vp, _vp, _vp, _i, _i, _vp, _vp, _vp, _i, _vp], C.c_int),
    "b200seg_cls_head_bwd": ([_vp, _vp, _vp, _vp, _vp, _i, _i, _vp, _PT, _vp, _vp, _vp, _vp, _i, _vp], C.c_int),
    "b200seg_stage_u8_sums": ([_vp, _i, _i64, _vp, _i, _vp], C.c_int),
    "b200seg_stage_u8_normalize": ([_vp, _i, _i64, _vp, _vp, _i, _i, _vp], C.c_int),
    "b200seg_stage_labels_u8": ([_vp, _i64, _i, _vp, _i, _vp], C.c_int),
    "b200seg_resample_workspace": ([_i, _i, _i, _i], C.c_int64),
    "b200seg_resample_linear": ([_vp, _i, _i, _i, _i, _vp, _i, _i, _i, _i, _f, _f, _vp, _vp, _i64, _i, _vp], C.c_int),
    "b200seg_normalize": ([_i, _vp, _i, _i, _i, _vp, _i64, _vp, _i, _vp], C.c_int),
    "b200seg_resample_nearest_u8": ([_vp, _i, _i, _i, _vp, _i, _i, _i, _i, _i, _i, _vp, _i, _vp], C.c_int),
    "b200seg_resize_linear_u8": ([_vp, _vp, _i, _i, _i, _vp, _i, _i, _vp], C.c_int),
    "b200seg_augment2d_workspace": ([_i64], C.c_int64),
    "b200seg_augment2d": ([_vp, _vp, _vp, _i, _i64, _i, _vp, _i64, _vp, _vp, _i64, _i, _vp], C.c_int),
    "b200seg_augment3d_workspace": ([_i, _i, _i, _i], C.c_int64),
    "b200seg_augment3d": ([_vp, _vp, _i, _i, _i, _i, _i, _i, _vp, _i, C.c_double, _i, C.c_double, _i, _vp, _vp, _i, _i,
                           _vp, _i64, _i, _vp], C.c_int),
    "b200seg_components_workspace": ([_i, _i, _i], C.c_int64),
    "b200seg_largest_component": ([_vp, _i, _i, _i, _i, _vp, _i64, _vp, _vp, _i, _vp], C.c_int),
    "b200seg_morphology_workspace": ([_i, _i, _i, _i, _i, _i], C.c_int64),
    "b200seg_morphology": ([_vp, _i, _i, _i, _i, _i, _i, _i, _vp, _i64, _vp, _i, _vp], C.c_int),
    "b200seg_label_bbox_workspace": ([], C.c_int64),
    "b200seg_label_bbox": ([_vp, _i, _i, _i, _i, _i, _vp, _i64, _vp, _i, _vp], C.c_int),
    "b200seg_gradcam_workspace": ([_i, _i, _i, _i], C.c_int64),
    "b200seg_gradcam_layer": ([_PT, _PT, _i, _i, _i, _i, _vp, _i64, _vp, _i, _vp], C.c_int),
    "b200seg_gradcam_scale": ([_vp, _i, _i, _i, _vp, _i64, _i, _vp], C.c_int),
    "b200seg_gradcam_target": ([_vp, _i, _i, _i, _vp, _vp, _i, _vp], C.c_int),
    "b200seg_warp3d": ([_vp, _vp, _i, _vp, _i, _i, _i, _i, _i, _vp, _vp, _i, _vp], C.c_int),
    "b200seg_warp3d_bwd": ([_vp, _vp, _i, _vp, _vp, _i, _i, _i, _i, _vp, _i, _vp], C.c_int),
}

EXPORTED_SYMBOLS = tuple(_SIGNATURES.keys())

_lib = None
_lib_lock = threading.Lock()


def load_library(path: Optional[str] = None):
    """dlopen the in-tree library and declare every prototype.  Raises if it is missing:
    there is no fallback implementation."""
    global _lib
    with _lib_lock:
        if _lib is not None and path is None:
            return _lib
        p = path or os.environ.get("B200SEG_LIB") or LIB_PATH      # B200SEG_LIB: an alternative build (A/B timing)
        if not os.path.exists(p):
            raise RuntimeError(
                f"{p} not found: build it with `python -m pytorchdeeplearing_b200.build` "
                "(or __graft_entry__.build()). pytorchdeeplearing_b200 has no non-CUDA fallback.")
        lib = C.CDLL(p)
        for name, (argtypes, restype) in _SIGNATURES.items():
            fn = getattr(lib, name)          # AttributeError if the symbol is not exported
            fn.argtypes = argtypes
            fn.restype = restype
        if lib.b200seg_version() < 201:
            raise RuntimeError("libb200seg.so is older than the Python binding")
        if path is None:
            _lib = lib
        return lib


RESIZE_SRC_BYTES = 16      # sizeof(struct b200seg_resize_src)


def resize_src_table(entries) -> bytes:
    """[(byte offset, h, w)] of a ragged uint8 batch -> the host bytes of its ``b200seg_resize_src`` table"""
    return b"".join(struct.pack("<qii", int(o), int(h), int(w)) for o, h, w in entries)


# stage bits and blur kinds of b200seg_augment2d (B200SEG_AUG2D_*)
AUG2D_HFLIP, AUG2D_VFLIP, AUG2D_BLUR, AUG2D_WARP, AUG2D_LUT = 1, 2, 4, 8, 16
AUG2D_BLURS = {"motion": 1, "median": 2, "box": 3}
AUG2D_MAX_TAPS = 8
AUG2D_MAX_SIDE = 8192
AUG2D_PARAM_BYTES = 416    # sizeof(struct b200seg_aug2d_param)


def aug2d_param_entry(src, dst, mask_src, mask_dst, h, w, c, flags, blur=0, taps=(), minv=None, lut=None,
                      filter_cn=None) -> bytes:
    """one ``b200seg_aug2d_param``: byte offsets, size, stage bits, blur kind, motion taps [(dy, dx, weight)],
    inverse 2x3 matrix (fp64) and the 256-byte table"""
    taps = list(taps)
    if len(taps) > AUG2D_MAX_TAPS:
        raise ValueError(f"at most {AUG2D_MAX_TAPS} motion-kernel taps, got {len(taps)}")
    wt = [float(t[2]) for t in taps] + [0.0] * (AUG2D_MAX_TAPS - len(taps))
    dy = [int(t[0]) for t in taps] + [0] * (AUG2D_MAX_TAPS - len(taps))
    dx = [int(t[1]) for t in taps] + [0] * (AUG2D_MAX_TAPS - len(taps))
    m = [0.0] * 6 if minv is None else [float(v) for v in minv]
    table = bytes(256) if lut is None else bytes(lut)
    assert len(table) == 256
    return struct.pack("<4q6d8f8b8b8i", int(src), int(dst), int(mask_src), int(mask_dst), *m, *wt, *dy, *dx,
                       int(h), int(w), int(c), int(flags), int(blur), len(taps),
                       int(c if filter_cn is None else filter_cn), 0) + table


# fill modes and rescale forms of b200seg_augment3d (B200SEG_AUG_*, B200SEG_RESCALE_*)
AUG_MODES = {"nearest": 0, "constant": 1, "reflect": 2, "wrap": 3, "mirror": 4}
RESCALE_NONE, RESCALE_F32, RESCALE_F64 = 0, 1, 2
AUG3D_PARAM_BYTES = 120    # sizeof(struct b200seg_aug3d_param)


def aug3d_param_table(entries) -> bytes:
    """[(3x3 matrix, offset[3], channel shifts (<= 4 floats), flip bits)] -> the host bytes of a
    ``b200seg_aug3d_param`` table (fp64 matrix and offset, fp32 shifts, int32 flip bits)"""
    out = []
    for m, off, shifts, flip in entries:
        sh = [float(v) for v in shifts] + [0.0] * (4 - len(shifts))
        out.append(struct.pack("<9d3d4fii", *[float(v) for v in m], *[float(v) for v in off], *sh, int(flip), 0))
    return b"".join(out)


def _dt(t: torch.Tensor) -> int:
    if t.dtype == torch.float32:
        return F32
    if t.dtype == torch.bfloat16:
        return BF16
    raise TypeError(f"unsupported activation dtype {t.dtype}")


def _desc(t: Optional[torch.Tensor]):
    """(N,D,H,W,C) view with unit channel stride and pitch = stride of W -> TensorDesc."""
    if t is None:
        return None
    if t.dim() != 5:
        raise ValueError(f"expected (N,D,H,W,C), got {tuple(t.shape)}")
    n, d, h, w, c = t.shape
    sn, sd, sh, sw, sc = t.stride()
    ld = sw if w > 1 else (sh // w if h > 1 else (sd // (h * w) if d > 1 else max(sn // (d * h * w), c)))
    if c > 1 and sc != 1:
        raise ValueError("channel stride must be 1 (channels-last)")
    ok = (w == 1 or sw == ld) and (h == 1 or sh == ld * w) and (d == 1 or sd == ld * w * h) and \
         (n == 1 or sn == ld * w * h * d)
    if not ok or ld < c:
        raise ValueError(f"tensor is not an NDHWC view with a channel pitch: shape {tuple(t.shape)} strides {t.stride()}")
    return TensorDesc(t.data_ptr(), n, d, h, w, c, ld, _dt(t))


def _p(t: Optional[torch.Tensor]):
    return None if t is None else t.data_ptr()


def _ref(d):
    return None if d is None else C.byref(d)


class PackedWeight:
    """Packed conv operand + its layout code (B200SEG_F32 / BF16 = [tap][K][N]; BF16_TC = [tap][N][K] K-major
    for the wgmma path).  Keeps what is needed to re-pack for the CUDA-core path."""
    __slots__ = ("t", "code", "src", "kind", "which", "dims")

    def __init__(self, t, code, src, kind, which, dims):
        self.t, self.code, self.src, self.kind, self.which, self.dims = t, code, src, kind, which, dims


class _PackPlan:
    __slots__ = ("outs", "table", "ndesc", "blocks", "anchor")

    def __init__(self, outs, table, ndesc, blocks, anchor):
        self.outs, self.table, self.ndesc, self.blocks, self.anchor = outs, table, ndesc, blocks, anchor


class CudaBackend:
    name = "cuda-sm90a"
    use_tc = True      # bf16 convolutions of the shapes the library accepts always take its tensor-core kernels

    def __init__(self):
        if not torch.cuda.is_available():
            raise RuntimeError("pytorchdeeplearing_b200 needs a CUDA device (built for sm_90a); none is available "
                               "and there is no CPU fallback")
        self.lib = load_library()
        self._inited = set()
        self._keep_tables = []     # device descriptor tables stay referenced while launches that read them may be pending
        self.launch_count = 0      # kernels launched through the C ABI (one per successful entry-point call)

    # ------------------------------------------------------------------ plumbing
    def _ds(self, t: torch.Tensor):
        dev = t.device.index if t.device.index is not None else torch.cuda.current_device()
        if dev not in self._inited:
            self._check(self.lib.b200seg_init(dev))
            self._inited.add(dev)
        return dev, torch.cuda.current_stream(dev).cuda_stream

    def _check(self, rc: int):
        if rc != 0:
            msg = self.lib.b200seg_last_error()
            raise RuntimeError(f"libb200seg error {rc}: {msg.decode() if msg else ''}")
        self.launch_count += 1

    # ------------------------------------------------------------------ weights
    def _pack_plan(self, w, kind, which, dtype, dims, allow_tc=True, vox=None):
        """-> (out_shape, layout code, (T, K, N2, N1, st, sk, sn2, sn1, flip)) for one conv operand; for the
        grouped layout the last element is a LIST of (src element offset, dst element offset, args) parts."""
        a, b = w.shape[0], w.shape[1]
        t = w.numel() // (a * b)
        od = F32 if dtype == torch.float32 else BF16
        if (allow_tc and dtype == torch.bfloat16 and kind == K3 and dims == 3
                and vox is not None and vox >= HALO_WS_MIN_VOX):
            cin, cout = (b, a) if which == "fwd" else (a, b)
            nt = self.lib.b200seg_conv_halo_ws_ntile(kind, cin, cout)
            if nt > 0:
                g = cout // nt
                if which == "fwd":      # [co/NT][t][ci/8][co%NT][ci%8]
                    parts = [(i * nt * b * t, i * t * b * nt, (t, b // 8, nt, 8, 1, 8 * t, b * t, t, 0)) for i in range(g)]
                else:                   # [ci/NT][T-1-t][co/8][ci%NT][co%8]
                    parts = [(i * nt * t, i * t * a * nt, (t, a // 8, nt, 8, 1, 8 * b * t, t, b * t, 1)) for i in range(g)]
                return (g, t, cin // 8, nt, 8), BF16_HALO_WS, parts
        if (allow_tc and dtype == torch.bfloat16 and kind == K3
                and vox is not None and vox >= HALO_MIN_VOX):
            cin, cout = (b, a) if which == "fwd" else (a, b)
            if self.lib.b200seg_conv_halo_eligible(kind, cin, cout):
                if which == "fwd":      # [t][ci/8][co][ci%8]
                    return (t, b // 8, a, 8), BF16_HALO, (t, b // 8, a, 8, 1, 8 * t, b * t, t, 0)
                return (t, a // 8, b, 8), BF16_HALO, (t, a // 8, b, 8, 1, 8 * b * t, t, b * t, 1)   # [T-1-t][co/8][ci][co%8]
        tc = False
        if allow_tc and dtype == torch.bfloat16:
            # (kind, Cin, Cout) of the op that will consume the packed operand
            if which == "fwd":
                op = (kind, a, b) if kind == UP else (kind, b, a)
            else:
                op = {K3: (K3, a, b), K1: (K1, a, b), DOWN: (UP, a, b), UP: (DOWN, b, a)}[kind]
            tc = bool(self.lib.b200seg_conv_tc_eligible(*op))
        if tc:
            # K-major rows for the wgmma path: [tap][N][K]
            gather_like = (which == "fwd" and kind != UP) or (which == "dgrad" and kind == UP)
            if which == "dgrad" and kind in (K3, K1):      # [T-1-t][ci][co]
                return (t, b, a), BF16_TC, (t, b, 1, a, 1, t, 0, b * t, 1)
            if gather_like:                                 # W (A,B,t) -> [t][A][B]
                return (t, a, b), BF16_TC, (t, a, 1, b, 1, b * t, 0, t, 0)
            return (t, b, a), BF16_TC, (t, b, 1, a, 1, t, 0, b * t, 0)   # [t][B][A]  (UP fwd, DOWN dgrad)
        if which == "fwd":
            if kind == UP:      # W (Ci,Co,t) -> [ci][t*Co + co]
                return (a, t * b), od, (1, a, t, b, 0, b * t, 1, t, 0)
            return (t, b, a), od, (t, b, 1, a, 1, t, 0, b * t, 0)       # W (Co,Ci,t) -> [t][ci][co]
        if kind in (K3, K1):   # [T-1-t][co][ci]
            return (t, a, b), od, (t, a, 1, b, 1, b * t, 0, t, 1)
        if kind == DOWN:       # W (Co,Ci,t) -> [co][t*Ci + ci]
            return (a, t * b), od, (1, a, t, b, 0, b * t, 1, t, 0)
        return (t, b, a), od, (t, b, 1, a, 1, t, 0, b * t, 0)           # UP: W (Ci,Co,t) -> [t][co][ci]

    def pack_weight(self, w, kind, which, dtype, dims, allow_tc=True, vox=None):
        """``vox``: voxels per sample of the layer's output (lets the backend pick the halo-staged kernel for the
        full-resolution 16/32-channel layers)."""
        dev, st = self._ds(w)
        shape, code, args = self._pack_plan(w, kind, which, dtype, dims, allow_tc, vox)
        out = torch.empty(shape, dtype=dtype, device=w.device)
        od = F32 if dtype == torch.float32 else BF16
        parts = args if isinstance(args, list) else [(0, 0, args)]
        for so, do, (T, K, N2, N1, s_t, s_k, s_n2, s_n1, flip) in parts:
            self._check(self.lib.b200seg_pack_weight(w.data_ptr() + so * w.element_size(),
                                                     out.data_ptr() + do * out.element_size(), od, T, K, N2, N1,
                                                     s_t, s_k, s_n2, s_n1, flip, dev, st))
        return PackedWeight(out, code, w, kind, which, dims)

    def _table_alloc(self, descs, device):
        """ctypes descriptor array -> (device tensor allocated on the current stream, host bytes, size)"""
        arr = (PackDesc * len(descs))(*descs)
        nbytes = C.sizeof(arr)
        pad = (nbytes + 15) // 16 * 16
        buf = (C.c_char * pad)()
        C.memmove(buf, arr, nbytes)
        return torch.empty(pad, dtype=torch.uint8, device=device), buf, pad

    def _table_upload(self, tab, st):
        """the descriptor bytes reach the device as kernel ARGUMENTS (no host-to-device memcpy: b200seg_upload_table)"""
        devt, buf, pad = tab
        dev = devt.device.index if devt.device.index is not None else torch.cuda.current_device()
        self._check(self.lib.b200seg_upload_table(C.cast(buf, C.c_void_p), pad, devt.data_ptr(), dev, st))
        self._keep_tables.append(devt)
        if len(self._keep_tables) > 64 and not torch.cuda.is_current_stream_capturing():
            self._keep_tables.pop(0)
        return devt

    def _launch_stream(self, dev, stream, after):
        """raw handle of the stream a launch goes to: the current one, or ``stream`` once it has been made to wait for
        the event ``after`` (default: for everything the current stream has enqueued so far)"""
        if stream is None:
            return torch.cuda.current_stream(dev).cuda_stream
        if after is not None:
            stream.wait_event(after)
        else:
            stream.wait_stream(torch.cuda.current_stream(dev))
        return stream.cuda_stream

    def pack_plan(self, reqs):
        """reqs: [(w, kind, which, dtype, dims, vox)] -> plan: the outputs and the descriptor table are ALLOCATED (on the
        current stream), nothing is launched.  ``plan.outs`` is the [PackedWeight] list."""
        descs, outs, blocks = [], [], 0
        for (w, kind, which, dtype, dims, vox) in reqs:
            shape, code, args = self._pack_plan(w, kind, which, dtype, dims, True, vox)
            out = torch.empty(shape, dtype=dtype, device=w.device)
            parts = args if isinstance(args, list) else [(0, 0, args)]
            for so, do, (T, K, N2, N1, s_t, s_k, s_n2, s_n1, flip) in parts:
                nb = max(1, min(256, (T * K * N2 * N1 + 4095) // 4096))
                descs.append(PackDesc(w.data_ptr() + so * w.element_size(), out.data_ptr() + do * out.element_size(),
                                      s_t, s_k, s_n2, s_n1, F32 if dtype == torch.float32 else BF16, T, K, N2, N1,
                                      flip, blocks, nb))
                blocks += nb
            outs.append(PackedWeight(out, code, w, kind, which, dims))
        return _PackPlan(outs, self._table_alloc(descs, reqs[0][0].device), len(descs), blocks, reqs[0][0])

    def pack_launch(self, plan, stream=None, after=None):
        """the two launches of a plan (table upload + ONE pack kernel), on the current stream or on ``stream`` (which
        first waits for the event ``after``, or for the current stream); the CALLER makes consumers wait for ``stream``"""
        dev, _ = self._ds(plan.anchor)
        st = self._launch_stream(dev, stream, after)
        table = self._table_upload(plan.table, st)
        self._check(self.lib.b200seg_pack_weights_multi(table.data_ptr(), plan.ndesc, plan.blocks, dev, st))
        return plan.outs

    def pack_many(self, reqs, stream=None):
        """reqs: [(w, kind, which, dtype, dims, vox)] -> [PackedWeight]: ONE launch for all operands."""
        if not reqs:
            return []
        return self.pack_launch(self.pack_plan(reqs), stream)

    def unpack_many(self, items, stream=None):
        """items: [(dwp [t][k][n], grad view)] -> parameter-layout gradients, ONE launch (on ``stream`` if given, after
        it has waited for the current stream; see ``pack_many``)."""
        if not items:
            return
        dev, st = self._ds(items[0][0])
        descs, blocks = [], 0
        for dwp, grad in items:
            t, k, n = dwp.shape
            nb = max(1, min(256, (dwp.numel() + 4095) // 4096))
            descs.append(PackDesc(dwp.data_ptr(), grad.data_ptr(), 1, t, k * t, 0, F32, t, k, n, 1, 0, blocks, nb))
            blocks += nb
        tab = self._table_alloc(descs, items[0][0].device)
        st = self._launch_stream(dev, stream, None)
        table = self._table_upload(tab, st)
        self._check(self.lib.b200seg_unpack_wgrads_multi(table.data_ptr(), len(descs), blocks, dev, st))

    def unpack_wgrad(self, dwp, grad, kind, dims):
        t, k, n = dwp.shape
        dev, st = self._ds(dwp)
        # dwp[t][k][n] -> grad[n][k][t]  (gather kinds: (Co,Ci,t); UP: (Ci,Co,t))
        self._check(self.lib.b200seg_unpack_wgrad(dwp.data_ptr(), grad.data_ptr(), t, k, n, 1, t, k * t, dev, st))

    # ------------------------------------------------------------------ conv family
    @staticmethod
    def _needs_repack(wpk, x, y):
        # the wgmma paths need bf16 activations on both sides (e.g. a 16-channel fp32 network input)
        return wpk.code in (BF16_TC, BF16_HALO, BF16_HALO_WS) and not (x.dtype == torch.bfloat16 and
                                                                      y.dtype == torch.bfloat16)

    def conv(self, kind, dims, x, wpk, bias, y, stats, addend):
        dev, st = self._ds(x)
        if self._needs_repack(wpk, x, y):
            wpk = self.pack_weight(wpk.src, wpk.kind, wpk.which, torch.bfloat16, wpk.dims, allow_tc=False)
        dx, dy, da = _desc(x), _desc(y), _desc(addend)
        self._check(self.lib.b200seg_conv(kind, dims, C.byref(dx), wpk.t.data_ptr(), wpk.code, _p(bias), C.byref(dy),
                                          _p(stats), _ref(da), dev, st))

    def conv_path(self, kind, dims, x, wpk, y, addend=None):
        """name (CONV_PATHS) of the kernel family ``conv`` would launch for these arguments; launches nothing"""
        code = BF16 if self._needs_repack(wpk, x, y) else wpk.code
        dx, dy, da = _desc(x), _desc(y), _desc(addend)
        rc = self.lib.b200seg_conv_path(kind, dims, C.byref(dx), code, C.byref(dy), _ref(da))
        if rc < 0:
            raise RuntimeError(f"libb200seg error {rc}: {self.lib.b200seg_last_error().decode()}")
        return CONV_PATHS[rc]

    def conv_halo_ws_geometry(self, kind, dims, x, wpk, y, addend=None):
        """output tile geometry (HALO_WS_GEOMS) the HALO_WS kernel family would use for these arguments; raises where
        ``conv`` would take another family; launches nothing"""
        code = BF16 if self._needs_repack(wpk, x, y) else wpk.code
        dx, dy, da = _desc(x), _desc(y), _desc(addend)
        rc = self.lib.b200seg_conv_halo_ws_geometry(kind, dims, C.byref(dx), code, C.byref(dy), _ref(da))
        if rc < 0:
            raise RuntimeError(f"libb200seg error {rc}: {self.lib.b200seg_last_error().decode()}")
        return HALO_WS_GEOMS[rc]

    def wgrad_path(self, kind, dims, a, b):
        """name (WGRAD_PATHS) of the kernel family ``wgrad`` would launch for these arguments; launches nothing"""
        da, db = _desc(a), _desc(b)
        rc = self.lib.b200seg_wgrad_path(kind, dims, C.byref(da), C.byref(db))
        if rc < 0:
            raise RuntimeError(f"libb200seg error {rc}: {self.lib.b200seg_last_error().decode()}")
        return WGRAD_PATHS[rc]

    def conv_bwdstats_ok(self, kind, dims, x, wpk, y, addend, yfwd):
        """can ``conv_bwdstats`` take this data-gradient convolution (3-D halo-staged 16/32-channel 3x3x3 layers)?"""
        if wpk.code not in (BF16_HALO, BF16_HALO_WS) or x.dtype != torch.bfloat16 or y.dtype != torch.bfloat16:
            return False
        # with 16 output channels the layer is traffic bound once it also reads the producer's raw output, so the
        # fused form is used for 32 output channels only
        if y.shape[-1] == 16:
            return False
        dx, dy, da, df = _desc(x), _desc(y), _desc(addend), _desc(yfwd)
        return bool(self.lib.b200seg_conv_bwdstats_supported(kind, dims, C.byref(dx), wpk.code, C.byref(dy), _ref(da),
                                                             C.byref(df)))

    def conv_bwdstats(self, kind, dims, x, wpk, y, addend, yfwd, gn, sums):
        """y = conv(x, wpk) [+ addend] AND sums[n][c][0:2] += {g*m, g*m*yfwd} of the layer (yfwd, gn) whose activation
        gradient y is: the GroupNorm-backward reduce pass folded into the data-gradient epilogue"""
        dev, st = self._ds(x)
        dx, dy, da, df, gg = _desc(x), _desc(y), _desc(addend), _desc(yfwd), self._gn(gn)
        self._check(self.lib.b200seg_conv_bwdstats(kind, dims, C.byref(dx), wpk.t.data_ptr(), wpk.code, C.byref(dy),
                                                   _ref(da), C.byref(df), C.byref(gg), sums.data_ptr(), dev, st))

    def wgrad(self, kind, dims, a, b, dwp):
        dev, st = self._ds(a)
        da, db = _desc(a), _desc(b)
        self._check(self.lib.b200seg_wgrad(kind, dims, C.byref(da), C.byref(db), dwp.data_ptr(), dev, st))

    # ------------------------------------------------------------------ GroupNorm
    def gn_finalize(self, stats, gamma, beta, scale, vox, groups, eps, coef, mr):
        dev, st = self._ds(stats)
        n, c = stats.shape[0], stats.shape[1]
        self._check(self.lib.b200seg_gn_finalize(stats.data_ptr(), gamma.data_ptr(), beta.data_ptr(), _p(scale), n, c,
                                                 groups, vox, eps, coef.data_ptr(), mr.data_ptr(), dev, st))

    def apply(self, y1, c1, y2, c2, res, out):
        dev, st = self._ds(y1)
        d1, d2, dr, do = _desc(y1), _desc(y2), _desc(res), _desc(out)
        self._check(self.lib.b200seg_apply(C.byref(d1), c1.data_ptr(), _ref(d2), _p(c2), _ref(dr), C.byref(do), dev, st))

    # fused-coefficient forms: gn = (stats, gamma, beta, scale|None, vox, groups, eps[, act]); act defaults to ACT_RELU
    @staticmethod
    def _gn(gn):
        if gn is None:
            return None
        stats, gamma, beta, scale, vox, groups, eps = gn[:7]
        act = gn[7] if len(gn) > 7 else ACT_RELU
        return GnDesc(stats.data_ptr(), gamma.data_ptr(), beta.data_ptr(), _p(scale), groups, vox, eps, act)

    def apply_gn(self, y1, gn1, y2, gn2, res, out):
        dev, st = self._ds(y1)
        d1, d2, dr, do = _desc(y1), _desc(y2), _desc(res), _desc(out)
        g1, g2 = self._gn(gn1), self._gn(gn2)
        self._check(self.lib.b200seg_apply_gn(C.byref(d1), C.byref(g1), _ref(d2), _ref(g2), _ref(dr), C.byref(do),
                                              dev, st))

    def gn_bwd_reduce_gn(self, g, y, gn, sums):
        dev, st = self._ds(y)
        dg, dy, gg = _desc(g), _desc(y), self._gn(gn)
        self._check(self.lib.b200seg_gn_bwd_reduce_gn(C.byref(dg), C.byref(dy), C.byref(gg), sums.data_ptr(), dev, st))

    def gn_bwd_apply_gn(self, g, y, gn, sums, dy, dgamma, dbeta, dbias, sum_y_from_stats=False):
        dev, st = self._ds(y)
        dg, dyy, dd, gg = _desc(g), _desc(y), _desc(dy), self._gn(gn)
        self._check(self.lib.b200seg_gn_bwd_apply_gn(C.byref(dg), C.byref(dyy), C.byref(gg), sums.data_ptr(),
                                                     C.byref(dd), dgamma.data_ptr(), dbeta.data_ptr(), _p(dbias),
                                                     1 if sum_y_from_stats else 0, dev, st))

    def gn_bwd_fused_ok(self, g, y, dy):
        dev, _ = self._ds(y)
        dg, dyy, dd = _desc(g), _desc(y), _desc(dy)
        return bool(self.lib.b200seg_gn_bwd_fused_supported(C.byref(dg), C.byref(dyy), C.byref(dd), dev))

    def gn_bwd_fused_gn(self, g, y, gn, sums, counter, dy, dgamma, dbeta, dbias):
        """sums [N][C][3] fp64 and counter (>= 4 bytes) zero on entry; one launch instead of reduce + apply"""
        dev, st = self._ds(y)
        dg, dyy, dd, gg = _desc(g), _desc(y), _desc(dy), self._gn(gn)
        self._check(self.lib.b200seg_gn_bwd_fused_gn(C.byref(dg), C.byref(dyy), C.byref(gg), sums.data_ptr(),
                                                     counter.data_ptr(), C.byref(dd), dgamma.data_ptr(),
                                                     dbeta.data_ptr(), _p(dbias), dev, st))

    # ------------------------------------------------------------------ fused input block (csrc/stem_gn.cu)
    # w3 / w1: the packed forward operands of the two stems (pack_weight(..., "fwd", torch.bfloat16, ...)); the raw
    # stem outputs are never stored: every call recomputes them from the fp32 image x (N,D,H,W,1)
    def stem_gn_ok(self, x, cout, dims):
        """can the fused input-block kernels take this image (3-D, fp32, one channel, 16 output channels)?"""
        if x.dtype != torch.float32 or x.dim() != 5 or x.shape[-1] != 1:
            return False
        return bool(self.lib.b200seg_stem_gn_supported(C.byref(_desc(x)), cout, dims))

    def _stem_operand(self, wpk):
        if wpk.code != BF16:
            wpk = self.pack_weight(wpk.src, wpk.kind, wpk.which, torch.bfloat16, wpk.dims, allow_tc=False)
        return wpk.t.data_ptr()

    def stem_gn_stats(self, x, w3, b3, w1, b1, stats3, stats1):
        dev, st = self._ds(x)
        self._check(self.lib.b200seg_stem_gn_stats(C.byref(_desc(x)), self._stem_operand(w3), _p(b3),
                                                   self._stem_operand(w1), _p(b1), stats3.data_ptr(),
                                                   stats1.data_ptr(), dev, st))

    def stem_gn_apply(self, x, w3, b3, w1, b1, gn3, gn1, out):
        dev, st = self._ds(x)
        g3, g1, do = self._gn(gn3), self._gn(gn1), _desc(out)
        self._check(self.lib.b200seg_stem_gn_apply(C.byref(_desc(x)), self._stem_operand(w3), _p(b3),
                                                   self._stem_operand(w1), _p(b1), C.byref(g3), C.byref(g1),
                                                   C.byref(do), dev, st))

    def stem_gn_bwd_sums(self, x, w3, b3, w1, b1, gn3, gn1, g, sums3, sums1):
        dev, st = self._ds(x)
        g3, g1, dg = self._gn(gn3), self._gn(gn1), _desc(g)
        self._check(self.lib.b200seg_stem_gn_bwd_sums(C.byref(_desc(x)), self._stem_operand(w3), _p(b3),
                                                      self._stem_operand(w1), _p(b1), C.byref(g3), C.byref(g1),
                                                      C.byref(dg), sums3.data_ptr(), sums1.data_ptr(), dev, st))

    def stem_gn_bwd(self, x, w3, b3, w1, b1, gn3, gn1, g, sums3, sums1, dw3, dw1, dgamma, dbeta, db3, db1):
        dev, st = self._ds(x)
        g3, g1, dg = self._gn(gn3), self._gn(gn1), _desc(g)
        self._check(self.lib.b200seg_stem_gn_bwd(C.byref(_desc(x)), self._stem_operand(w3), _p(b3),
                                                 self._stem_operand(w1), _p(b1), C.byref(g3), C.byref(g1),
                                                 C.byref(dg), sums3.data_ptr(), sums1.data_ptr(), dw3.data_ptr(),
                                                 dw1.data_ptr(), dgamma.data_ptr(), dbeta.data_ptr(), _p(db3),
                                                 _p(db1), dev, st))

    # ------------------------------------------------------------------ fused first layer of up_tr32 (csrc/up_gn.cu)
    # w: the packed forward operand of the transposed convolution (pack_weight(..., "fwd", torch.bfloat16, ...) on the
    # pointwise mma.sync path); the raw output is never stored: every call recomputes it from x (N,D,H,W,32)
    def up_gn_ok(self, x, wpk, cout, dims):
        """can the fused up_tr32 kernels take this input (3-D, bf16, 32 -> 16 channels) and forward operand?"""
        if x.dtype != torch.bfloat16 or x.dim() != 5 or wpk is None or wpk.code != BF16_TC:
            return False
        return bool(self.lib.b200seg_up_gn_supported(C.byref(_desc(x)), cout, dims))

    def up_gn_stats(self, x, wpk, bias, stats):
        dev, st = self._ds(x)
        self._check(self.lib.b200seg_up_gn_stats(C.byref(_desc(x)), wpk.t.data_ptr(), _p(bias), stats.data_ptr(),
                                                 dev, st))

    def up_gn_apply(self, x, wpk, bias, gn, out):
        dev, st = self._ds(x)
        gg, do = self._gn(gn), _desc(out)
        self._check(self.lib.b200seg_up_gn_apply(C.byref(_desc(x)), wpk.t.data_ptr(), _p(bias), C.byref(gg),
                                                 C.byref(do), dev, st))

    def up_gn_bwd_sums(self, x, wpk, bias, gn, g, sums):
        dev, st = self._ds(x)
        gg, dg = self._gn(gn), _desc(g)
        self._check(self.lib.b200seg_up_gn_bwd_sums(C.byref(_desc(x)), wpk.t.data_ptr(), _p(bias), C.byref(gg),
                                                    C.byref(dg), sums.data_ptr(), dev, st))

    def up_gn_bwd(self, x, wpk, bias, gn, g, sums, dw, dx, dgamma, dbeta, dbias):
        dev, st = self._ds(x)
        gg, dg, dd = self._gn(gn), _desc(g), _desc(dx)
        self._check(self.lib.b200seg_up_gn_bwd(C.byref(_desc(x)), wpk.t.data_ptr(), _p(bias), C.byref(gg), C.byref(dg),
                                               sums.data_ptr(), dw.data_ptr(), C.byref(dd), dgamma.data_ptr(),
                                               dbeta.data_ptr(), _p(dbias), dev, st))

    def gn_bwd_reduce(self, g, y, coef, sums):
        dev, st = self._ds(y)
        dg, dy = _desc(g), _desc(y)
        self._check(self.lib.b200seg_gn_bwd_reduce(C.byref(dg), C.byref(dy), coef.data_ptr(), sums.data_ptr(), dev, st))

    def gn_bwd_finalize(self, sums, mr, gamma, scale, vox, groups, coef3, dgamma, dbeta, dbias):
        dev, st = self._ds(sums)
        n, c = sums.shape[0], sums.shape[1]
        self._check(self.lib.b200seg_gn_bwd_finalize(sums.data_ptr(), mr.data_ptr(), gamma.data_ptr(), _p(scale), n, c,
                                                     groups, vox, coef3.data_ptr(), dgamma.data_ptr(),
                                                     dbeta.data_ptr(), _p(dbias), dev, st))

    def gn_bwd_apply(self, g, y, coef, coef3, dy):
        dev, st = self._ds(y)
        dg, dyy, dd = _desc(g), _desc(y), _desc(dy)
        self._check(self.lib.b200seg_gn_bwd_apply(C.byref(dg), C.byref(dyy), coef.data_ptr(), coef3.data_ptr(),
                                                  C.byref(dd), dev, st))

    def colsum(self, dy, out):
        dev, st = self._ds(dy)
        d = _desc(dy)
        self._check(self.lib.b200seg_colsum(C.byref(d), out.data_ptr(), dev, st))

    # ------------------------------------------------------------------ pooling
    def pool_fwd(self, x, out, dims):
        dev, st = self._ds(x)
        dx, do = _desc(x), _desc(out)
        self._check(self.lib.b200seg_pool_fwd(C.byref(dx), C.byref(do), dims, dev, st))

    def pool_bwd(self, x, g_out, addend, g_x, dims):
        dev, st = self._ds(x)
        dx, dg, da, do = _desc(x), _desc(g_out), _desc(addend), _desc(g_x)
        self._check(self.lib.b200seg_pool_bwd(C.byref(dx), C.byref(dg), _ref(da), C.byref(do), dims, dev, st))

    # ------------------------------------------------------------------ trilinear 2x upsample + skip add (UNet3dthin)
    def upsample_add(self, a, e, s):
        """s (N,2D,2H,2W,C) = up2(a) + e for a (N,D,H,W,C); e has s's shape"""
        dev, st = self._ds(a)
        da, de, ds = _desc(a), _desc(e), _desc(s)
        self._check(self.lib.b200seg_upsample2_add(C.byref(da), C.byref(de), C.byref(ds), dev, st))

    def upsample_bwd(self, g_s, g_a):
        """g_a (N,D,H,W,C) = up2^T(g_s), written"""
        dev, st = self._ds(g_s)
        dg, da = _desc(g_s), _desc(g_a)
        self._check(self.lib.b200seg_upsample2_bwd(C.byref(dg), C.byref(da), dev, st))

    # ------------------------------------------------------------------ head + losses
    def head_probs(self, logits, probs):
        dev, st = self._ds(logits)
        c = logits.shape[-1]
        self._check(self.lib.b200seg_head_probs(logits.data_ptr(), probs.data_ptr(), logits.numel() // c, c, dev, st))

    def head_fwd(self, x, w, bias, logits, probs):
        """logits/probs (N,D,H,W,nc) fp32 contiguous; w the (nc,Cin,1..) conv parameter. False if unsupported."""
        nc = logits.shape[-1]
        if nc > 8 or x.shape[-1] % 4 != 0:
            return False
        dev, st = self._ds(x)
        dx = _desc(x)
        self._check(self.lib.b200seg_head_fwd(C.byref(dx), w.data_ptr(), _p(bias), logits.data_ptr(), _p(probs),
                                              nc, dev, st))
        return True

    def head_bwd(self, x, dlogits, w, dx, dw, db):
        nc = dlogits.shape[-1]
        if not self.lib.b200seg_head_bwd_supported(x.shape[-1], nc):
            return False
        dev, st = self._ds(x)
        d1, d2 = _desc(x), _desc(dx)
        self._check(self.lib.b200seg_head_bwd(C.byref(d1), dlogits.data_ptr(), w.data_ptr(), C.byref(d2),
                                              dw.data_ptr(), db.data_ptr(), nc, dev, st))
        return True

    def cls_head_fwd(self, x, w1, b1, w2, b2, pooled, hidden, logits):
        """classifier head (ResNet2d / ResNet3d): x (N,D,H,W,C) -> pooled [N][C], hidden [N][Hd], logits [N][K] fp32;
        w1/b1/w2/b2 the nn.Linear parameters"""
        dev, st = self._ds(x)
        dx = _desc(x)
        self._check(self.lib.b200seg_cls_head_fwd(C.byref(dx), w1.data_ptr(), b1.data_ptr(), w2.data_ptr(),
                                                  b2.data_ptr(), w1.shape[0], w2.shape[0], pooled.data_ptr(),
                                                  hidden.data_ptr(), logits.data_ptr(), dev, st))

    def cls_head_bwd(self, dlogits, pooled, hidden, w1, w2, work, dx, dw1, db1, dw2, db2):
        """d logits [N][K] -> dw1, db1, dw2, db2 (written) and dx (N,D,H,W,C) = the broadcast pooled gradient;
        work: fp32 scratch of N*(Hd + C) elements"""
        dev, st = self._ds(dlogits)
        d = _desc(dx)
        self._check(self.lib.b200seg_cls_head_bwd(dlogits.data_ptr(), pooled.data_ptr(), hidden.data_ptr(),
                                                  w1.data_ptr(), w2.data_ptr(), w1.shape[0], w2.shape[0],
                                                  work.data_ptr(), C.byref(d), dw1.data_ptr(), db1.data_ptr(),
                                                  dw2.data_ptr(), db2.data_ptr(), dev, st))

    @staticmethod
    def _label_dtype(labels):
        if labels.dtype == torch.int64:
            return I64
        if labels.dtype == torch.float32:
            return F32
        raise TypeError(f"labels must be int64 (or fp32 soft targets for the binary losses), got {labels.dtype}")

    @staticmethod
    def part_size(c):
        """doubles in the loss partial-sum buffer (include/b200seg.h: b200seg_loss_partials)"""
        return 3 * c + 4 if c > 1 else 7

    def loss_partials(self, logits, labels, gamma, alpha_f, part, metric=None):
        """logits (N, ..., C) fp32 channels-last contiguous; labels (N, ...) int64 / fp32; metric [N][C][3] fp64 or None"""
        dev, st = self._ds(logits)
        n, c = logits.shape[0], logits.shape[-1]
        self._check(self.lib.b200seg_loss_partials(logits.data_ptr(), labels.data_ptr(), self._label_dtype(labels), n,
                                                   logits.numel() // (n * c), c, gamma, alpha_f, part.data_ptr(),
                                                   _p(metric), dev, st))

    def loss_finalize(self, part, c, terms, alpha, gamma, alpha_f, loss, lcoef):
        dev, st = self._ds(part)
        self._check(self.lib.b200seg_loss_finalize(part.data_ptr(), c, terms, alpha.data_ptr(), gamma, alpha_f,
                                                   loss.data_ptr(), lcoef.data_ptr(), dev, st))

    def loss_bwd(self, logits, labels, lcoef, gscale, dlogits):
        dev, st = self._ds(logits)
        c = logits.shape[-1]
        self._check(self.lib.b200seg_loss_bwd(logits.data_ptr(), labels.data_ptr(), self._label_dtype(labels),
                                              logits.numel() // c, c, lcoef.data_ptr(), gscale.data_ptr(),
                                              dlogits.data_ptr(), dev, st))

    def loss_partials_ss(self, logits, labels, part, metric=None):
        """BinarySSLoss sums (include/b200seg.h: b200seg_loss_partials_ss), same part size as the binary losses"""
        dev, st = self._ds(logits)
        n = logits.shape[0]
        self._check(self.lib.b200seg_loss_partials_ss(logits.data_ptr(), labels.data_ptr(), self._label_dtype(labels),
                                                      n, logits.numel() // n, part.data_ptr(), _p(metric), dev, st))

    def loss_bwd_ss(self, logits, labels, lcoef, gscale, dlogits):
        dev, st = self._ds(logits)
        self._check(self.lib.b200seg_loss_bwd_ss(logits.data_ptr(), labels.data_ptr(), self._label_dtype(labels),
                                                 logits.numel(), lcoef.data_ptr(), gscale.data_ptr(),
                                                 dlogits.data_ptr(), dev, st))

    def radix_sort_pairs(self, keys, vals):
        """keys uint32 bit patterns in int32 [nseg, len], vals int32 [nseg, len] -> (keys, vals) sorted per row,
        ascending by unsigned key, ties in input order"""
        dev, st = self._ds(keys)
        assert keys.dtype == torch.int32 and vals.dtype == torch.int32 and keys.shape == vals.shape and keys.dim() == 2
        keys, vals = keys.contiguous(), vals.contiguous()
        nseg, ln = keys.shape
        ko, vo = torch.empty_like(keys), torch.empty_like(vals)
        nb = int(self.lib.b200seg_radix_sort_workspace(nseg, ln))
        ws = torch.empty(max(nb, 1), dtype=torch.uint8, device=keys.device)
        self._check(self.lib.b200seg_radix_sort_pairs(keys.data_ptr(), vals.data_ptr(), ko.data_ptr(), vo.data_ptr(),
                                                      nseg, ln, ws.data_ptr(), nb, dev, st))
        return ko, vo

    def lovasz_fwd(self, logits, labels, per_image, ignore, loss, coef, seg_scale):
        """logits (N, ..., C) fp32 channels-last contiguous, labels int64 (N, ...); coef like logits;
        seg_scale fp32 [N*C if per_image else C].  ignore: None or an int label value"""
        dev, st = self._ds(logits)
        n, c = logits.shape[0], logits.shape[-1]
        vox = logits.numel() // (n * c)
        nb = int(self.lib.b200seg_lovasz_workspace(n, vox, c, 1 if per_image else 0))
        ws = torch.empty(max(nb, 1), dtype=torch.uint8, device=logits.device)
        self._check(self.lib.b200seg_lovasz_fwd(logits.data_ptr(), labels.data_ptr(), n, vox, c,
                                                1 if per_image else 0, 0 if ignore is None else 1,
                                                0 if ignore is None else int(ignore), ws.data_ptr(), nb,
                                                loss.data_ptr(), coef.data_ptr(), seg_scale.data_ptr(), dev, st))

    def lovasz_bwd(self, logits, labels, per_image, coef, seg_scale, gscale, dlogits):
        dev, st = self._ds(logits)
        n, c = logits.shape[0], logits.shape[-1]
        self._check(self.lib.b200seg_lovasz_bwd(logits.data_ptr(), labels.data_ptr(), n, logits.numel() // (n * c), c,
                                                1 if per_image else 0, coef.data_ptr(), seg_scale.data_ptr(),
                                                gscale.data_ptr(), dlogits.data_ptr(), dev, st))

    def lovasz_hinge_fwd(self, logits, labels, per_image, ignore, loss, coef, bad=None):
        """logits (N, ..., 1) fp32 contiguous, labels int64 with N*vox elements; coef like logits (d loss / d logits);
        bad: None or int64 [1] (labels other than 0, 1 and ignore).  ignore: None or an int label value"""
        dev, st = self._ds(logits)
        n = logits.shape[0]
        vox = logits.numel() // n
        nb = int(self.lib.b200seg_lovasz_hinge_workspace(n, vox, 1 if per_image else 0))
        ws = torch.empty(max(nb, 1), dtype=torch.uint8, device=logits.device)
        self._check(self.lib.b200seg_lovasz_hinge_fwd(logits.data_ptr(), labels.data_ptr(), n, vox,
                                                      1 if per_image else 0, 0 if ignore is None else 1,
                                                      0 if ignore is None else int(ignore), ws.data_ptr(), nb,
                                                      loss.data_ptr(), coef.data_ptr(), _p(bad), dev, st))

    def lovasz_hinge_bwd(self, coef, gscale, dlogits):
        dev, st = self._ds(coef)
        self._check(self.lib.b200seg_lovasz_hinge_bwd(coef.data_ptr(), coef.numel(), gscale.data_ptr(),
                                                      dlogits.data_ptr(), dev, st))

    # ------------------------------------------------------------------ 3-D segmentation metrics (model/metric.py:11-142)
    _MASK_DTYPES = {torch.bool: U8, torch.uint8: U8, torch.int32: I32, torch.int64: I64}

    def _segmetric_args(self, real, pred, spacing_zyx):
        """real, pred (N, D, H, W) contiguous masks of one shape; spacing_zyx fp64 (N, 3) on the same device"""
        assert real.shape == pred.shape and real.dim() == 4 and real.is_contiguous() and pred.is_contiguous()
        assert spacing_zyx.dtype == torch.float64 and spacing_zyx.is_contiguous() and spacing_zyx.numel() >= 3 * real.shape[0]
        rdt, pdt = self._MASK_DTYPES.get(real.dtype), self._MASK_DTYPES.get(pred.dtype)
        if rdt is None or pdt is None:
            raise TypeError(f"masks must be bool, uint8, int32 or int64, got {real.dtype} / {pred.dtype}")
        n, d, h, w = real.shape
        nb = int(self.lib.b200seg_segmetric3d_workspace(n, d, h, w))
        ws = torch.empty(max(nb, 1), dtype=torch.uint8, device=real.device)
        return (real.data_ptr(), rdt, pred.data_ptr(), pdt, n, d, h, w, spacing_zyx.data_ptr(), ws.data_ptr(), nb), ws

    def segmetric3d(self, real, pred, spacing_zyx, counts, metrics, flags):
        """counts int64 [N][6] = {R, P, I, U, S_r, S_p}, metrics fp64 [N][9] (Seg_Metirc3d's order), flags int32 [N]"""
        dev, st = self._ds(real)
        args, ws = self._segmetric_args(real, pred, spacing_zyx)
        self._check(self.lib.b200seg_segmetric3d(*args, counts.data_ptr(), metrics.data_ptr(), flags.data_ptr(), dev, st))

    def segmetric3d_points(self, real, pred, spacing_zyx, real_idx, pred_idx, real2pred, pred2real):
        """C-order linear voxel indices of both surfaces (int64) and each point's distance to the other surface (fp64);
        the four outputs are sized from the surface counts of ``segmetric3d``"""
        dev, st = self._ds(real)
        args, ws = self._segmetric_args(real, pred, spacing_zyx)
        self._check(self.lib.b200seg_segmetric3d_points(*args, real_idx.numel(), pred_idx.numel(), real_idx.data_ptr(),
                                                        pred_idx.data_ptr(), real2pred.data_ptr(), pred2real.data_ptr(),
                                                        dev, st))

    # ------------------------------------------------------------------ SSIM / SSIM3D (model/lossesSSIM.py:49-93)
    @staticmethod
    def _ssim_geom(img):
        """(dims, N, C, D, H, W) and the host {n, c, d, h, w} element strides of an fp32 (N,C,H,W) / (N,C,D,H,W) image"""
        if img.dim() == 4:
            n, c, h, w = img.shape
            sn, sc, sh, sw = img.stride()
            return (2, n, c, 1, h, w), (C.c_int64 * 5)(sn, sc, 0, sh, sw)
        return (3,) + tuple(img.shape), (C.c_int64 * 5)(*img.stride())

    # ------------------------------------------------------------------ voxelmorph warp (csrc/warp3d.cu)
    def warp3d(self, ddf, image, label, moved_image, moved_label):
        """ddf fp32 contiguous (N, D, H, W, 3); image / label fp32 contiguous (N, C, D, H, W) or None; the moved
        tensors likewise"""
        dev, st = self._ds(ddf)
        n, d, h, w = ddf.shape[:4]
        ci = image.shape[1] if image is not None else 0
        cl = label.shape[1] if label is not None else 0
        self._check(self.lib.b200seg_warp3d(ddf.data_ptr(), _p(image), ci, _p(label), cl, n, d, h, w, _p(moved_image),
                                            _p(moved_label), dev, st))

    def warp3d_bwd(self, ddf, image, gmoved, addend, gddf):
        """gddf (N, D, H, W, 3) = d loss / d ddf from gmoved (N, C, D, H, W) [+ addend (N, D, H, W, 3)]"""
        dev, st = self._ds(ddf)
        n, d, h, w = ddf.shape[:4]
        self._check(self.lib.b200seg_warp3d_bwd(ddf.data_ptr(), image.data_ptr(), image.shape[1], gmoved.data_ptr(),
                                                _p(addend), n, d, h, w, gddf.data_ptr(), dev, st))

    def ssim_fwd(self, img1, img2, window_size, taps, coef):
        """img1, img2 fp32 of one shape, any strides; taps fp32 host [window_size]; coef fp64 [4][map voxels] or None.
        -> the workspace holding the partial sums of the map (input of ssim_finalize)"""
        dev, st = self._ds(img1)
        geom, s1 = self._ssim_geom(img1)
        _, s2 = self._ssim_geom(img2)
        nb = int(self.lib.b200seg_ssim_workspace(*geom, window_size))
        ws = torch.empty(max(nb, 8) // 8, dtype=torch.float64, device=img1.device)
        t = (C.c_float * window_size)(*[float(v) for v in taps])
        self._check(self.lib.b200seg_ssim_fwd(geom[0], img1.data_ptr(), C.cast(s1, _vp), img2.data_ptr(), C.cast(s2, _vp),
                                              *geom[1:], window_size, C.cast(t, _vp), _p(coef), ws.data_ptr(), nb,
                                              dev, st))
        return ws

    def ssim_finalize(self, img1, window_size, size_average, ws, acc, value, reduce=True):
        """acc fp64 / value fp32: {sum, count} / [1] (size_average), else [N] (2-D) or [N][W'] (3-D); reduce=False
        recomputes value from acc only"""
        dev, st = self._ds(acc)
        geom, _ = self._ssim_geom(img1)
        self._check(self.lib.b200seg_ssim_finalize(*geom, window_size, int(bool(size_average)), int(bool(reduce)),
                                                   ws.data_ptr(), ws.numel() * 8, acc.data_ptr(), value.data_ptr(),
                                                   dev, st))

    def ssim_bwd(self, img1, img2, window_size, taps, coef, size_average, gout, acc, grad1, grad2):
        """grad1 / grad2: fp32 contiguous in the images' shape, or None"""
        dev, st = self._ds(img1)
        geom, s1 = self._ssim_geom(img1)
        _, s2 = self._ssim_geom(img2)
        t = (C.c_float * window_size)(*[float(v) for v in taps])
        self._check(self.lib.b200seg_ssim_bwd(geom[0], img1.data_ptr(), C.cast(s1, _vp), img2.data_ptr(), C.cast(s2, _vp),
                                              *geom[1:], window_size, C.cast(t, _vp), coef.data_ptr(),
                                              int(bool(size_average)), gout.data_ptr(), acc.data_ptr(), _p(grad1),
                                              _p(grad2), dev, st))

    # ------------------------------------------------------------------ soft-clDice (model/lossescldice.py)
    @staticmethod
    def _cl_field(t):
        """(float pointer, host strides, labels pointer) of an fp32 (N, C, [D,] H, W) field, or of int64 labels
        (N, [D,] H, W) whose one-hot stands for the field"""
        if t is None:
            return None, None, None
        if t.dtype == torch.int64:
            return None, None, t.data_ptr()
        _, s = CudaBackend._ssim_geom(t)
        return t.data_ptr(), s, None

    @staticmethod
    def _cl_shape(x):
        return (x.shape[0], x.shape[1], 1) + tuple(x.shape[2:]) if x.dim() == 4 else tuple(x.shape)

    def cldice_workspace(self, x):
        nb = int(self.lib.b200seg_cldice_workspace(*self._cl_shape(x)))
        return torch.empty(max(nb, 8) // 8, dtype=torch.float64, device=x.device)

    def cldice_skeleton(self, x, rounds, fields, other=None, pass_=0, ws=None):
        """x fp32 (any strides) or int64 labels with ``fields``' (N, C) leading extents; fields fp32 [nfields][...];
        other (fp32 or int64 labels) adds the epilogue sums into half ``pass_`` of ``ws``"""
        dev, st = self._ds(fields)
        xp, xs, xl = self._cl_field(x)
        op, os_, ol = self._cl_field(other)
        shape = self._cl_shape(fields[0])
        self._check(self.lib.b200seg_cldice_skeleton(xp, None if xs is None else C.cast(xs, _vp), xl, *shape, rounds,
                                                     fields.data_ptr(), fields.shape[0], op,
                                                     None if os_ is None else C.cast(os_, _vp), ol, pass_, _p(ws),
                                                     0 if ws is None else ws.numel() * 8, dev, st))

    def cldice_finalize(self, shape, per_class, labels, alpha, smooth, eps, ws, stats, loss, reduce=True):
        dev, st = self._ds(stats)
        self._check(self.lib.b200seg_cldice_finalize(*shape, int(bool(per_class)), int(bool(labels)), _p(alpha),
                                                     float(smooth), float(eps), int(bool(reduce)), _p(ws),
                                                     0 if ws is None else ws.numel() * 8, stats.data_ptr(),
                                                     loss.data_ptr(), dev, st))

    def cldice_bwd(self, x, rounds, fields, grad, scratch, grad_skeleton=None, target=None, target_skeleton=None,
                   stats=None, gout=None):
        dev, st = self._ds(grad)
        _, xs = self._ssim_geom(x)
        tp, ts, tl = self._cl_field(target)
        self._check(self.lib.b200seg_cldice_bwd(x.data_ptr(), C.cast(xs, _vp), *self._cl_shape(x), rounds, _p(fields),
                                                _p(grad_skeleton), tp, None if ts is None else C.cast(ts, _vp), tl,
                                                _p(target_skeleton), _p(stats), _p(gout), grad.data_ptr(),
                                                _p(scratch), dev, st))

    def cldice_norm(self, cl, vessel, sums, out):
        dev, st = self._ds(cl)
        _, cs = self._ssim_geom(cl)
        _, vs = self._ssim_geom(vessel)
        self._check(self.lib.b200seg_cldice_norm(cl.data_ptr(), C.cast(cs, _vp), vessel.data_ptr(), C.cast(vs, _vp),
                                                 *self._cl_shape(cl), sums.data_ptr(), out.data_ptr(), dev, st))

    def cldice_norm_bwd(self, cl, vessel, sums, gout, grad_cl, grad_vessel):
        dev, st = self._ds(cl)
        _, cs = self._ssim_geom(cl)
        _, vs = self._ssim_geom(vessel)
        self._check(self.lib.b200seg_cldice_norm_bwd(cl.data_ptr(), C.cast(cs, _vp), vessel.data_ptr(),
                                                     C.cast(vs, _vp), *self._cl_shape(cl), sums.data_ptr(),
                                                     gout.data_ptr(), _p(grad_cl), _p(grad_vessel), dev, st))

    # ------------------------------------------------------------------ per-step accuracy (model/metric.py)
    def metric_partials(self, probs, labels, threshold, metric):
        """probs (N, ..., C) fp32 channels-last contiguous; metric [N][C][3] fp64 (+=)"""
        dev, st = self._ds(probs)
        n, c = probs.shape[0], probs.shape[-1]
        self._check(self.lib.b200seg_metric_partials(probs.data_ptr(), labels.data_ptr(), self._label_dtype(labels), n,
                                                     probs.numel() // (n * c), c, threshold, metric.data_ptr(), dev, st))

    def metric_finalize(self, metric, out):
        dev, st = self._ds(metric)
        n, c = metric.shape[0], metric.shape[1]
        self._check(self.lib.b200seg_metric_finalize(metric.data_ptr(), n, c, out.data_ptr(), dev, st))

    # ------------------------------------------------------------------ optimizer / dropout masks / inference head
    def adam_step(self, param, grad, exp_avg, exp_avg_sq, state, lr, beta1, beta2, eps, weight_decay, decoupled,
                  gscale=None, tick=True):
        dev, st = self._ds(param)
        self._check(self.lib.b200seg_adam_step(param.data_ptr(), grad.data_ptr(), exp_avg.data_ptr(),
                                               exp_avg_sq.data_ptr(), param.numel(), state.data_ptr(), lr, beta1,
                                               beta2, eps, weight_decay, 1 if decoupled else 0, _p(gscale),
                                               1 if tick else 0, dev, st))
        if tick:
            self.launch_count += 1

    def upload_bytes(self, raw: bytes, device):
        """host bytes -> new device uint8 tensor through kernel arguments (b200seg_upload_table; no memcpy node)"""
        pad = (len(raw) + 15) // 16 * 16
        buf = (C.c_char * pad)()
        C.memmove(buf, raw, len(raw))
        devt = torch.empty(pad, dtype=torch.uint8, device=device)
        dev = device.index if device.index is not None else torch.cuda.current_device()
        self._check(self.lib.b200seg_upload_table(C.cast(buf, C.c_void_p), pad, devt.data_ptr(), dev,
                                                  torch.cuda.current_stream(dev).cuda_stream))
        return devt

    def upload_into(self, raw: bytes, dst: torch.Tensor):
        """host bytes -> EXISTING device tensor (len(raw) <= dst bytes, multiple of 16)"""
        pad = (len(raw) + 15) // 16 * 16
        buf = (C.c_char * pad)()
        C.memmove(buf, raw, len(raw))
        dev, st = self._ds(dst)
        self._check(self.lib.b200seg_upload_table(C.cast(buf, C.c_void_p), pad, dst.data_ptr(), dev, st))

    def dropout_masks(self, rng, table, nmasks, total, p_drop, out):
        """rng: int64 [2] device {seed, offset}; table: int32 [nmasks][3] device {first, count, first element index
        within the (global-batch) draw}; out fp32 [total]"""
        dev, st = self._ds(out)
        self._check(self.lib.b200seg_dropout_masks(rng.data_ptr(), table.data_ptr(), nmasks, total, p_drop,
                                                   out.data_ptr(), dev, st))

    def head_mask(self, x, w, bias, mask, threshold):
        """x (N,D,H,W,Cin); mask uint8 (N,D,H,W). False if the fused path does not take the shape."""
        nc = w.shape[0]
        if nc > 8 or x.shape[-1] % 4 != 0:
            return False
        dev, st = self._ds(x)
        dx = _desc(x)
        self._check(self.lib.b200seg_head_mask(C.byref(dx), w.data_ptr(), _p(bias), mask.data_ptr(), nc, threshold,
                                               dev, st))
        return True

    # ------------------------------------------------------------------ input staging (SURVEY 8f-4)
    def stage_images_u8(self, img, out):
        """out[n] = (img[n] - mean_n) / std_n  (float64 arithmetic, population std; model/dataset.py:141-142) for a
        dense uint8 batch ``img`` [N, ...]; ``out`` fp32 or bf16 with the same number of elements."""
        dev, st = self._ds(img)
        assert img.dtype == torch.uint8 and img.is_contiguous() and out.is_contiguous() and out.numel() == img.numel()
        n = img.shape[0]
        per = img.numel() // n
        sums = torch.zeros((n, 2), dtype=torch.int64, device=img.device)      # uint64 bit patterns
        self._check(self.lib.b200seg_stage_u8_sums(img.data_ptr(), n, per, sums.data_ptr(), dev, st))
        self._check(self.lib.b200seg_stage_u8_normalize(img.data_ptr(), n, per, sums.data_ptr(), out.data_ptr(),
                                                        _dt(out), dev, st))
        return out

    def stage_labels_u8(self, lab, out, binarize=True):
        """out = lab.long(), with y[y != 0] = 1 (model/modelUnet.py:130) when ``binarize``"""
        dev, st = self._ds(lab)
        assert lab.dtype == torch.uint8 and out.dtype == torch.int64 and lab.is_contiguous() and out.is_contiguous()
        self._check(self.lib.b200seg_stage_labels_u8(lab.data_ptr(), lab.numel(), 1 if binarize else 0, out.data_ptr(),
                                                     dev, st))
        return out

    # ------------------------------------------------------------------ whole-volume 3-D inference (csrc/resample.cu)
    _VOL_DTYPES = {torch.uint8: U8, torch.int16: I16, torch.int32: I32, torch.float32: F32}

    def resample_workspace(self, mode, out_zyx, device):
        """uint8 workspace of b200seg_resample_workspace bytes; its first 8 fp64 are the stats of b200seg_normalize"""
        nb = int(self.lib.b200seg_resample_workspace(mode, *out_zyx))
        return torch.empty(max(nb, 256), dtype=torch.uint8, device=device)

    def resample_linear(self, src, ratio_zyx, out, mode=NORM_NONE, lower=0.0, upper=0.0, ws=None):
        """src dense (D, H, W) uint8 / int16 / int32 / fp32 -> out dense fp32 (oD, oH, oW); ratio_zyx host floats"""
        dev, st = self._ds(src)
        code = self._VOL_DTYPES.get(src.dtype)
        if code is None:
            raise TypeError(f"volumes must be uint8, int16, int32 or float32, got {src.dtype}")
        assert src.dim() == 3 and src.is_contiguous() and out.dim() == 3 and out.is_contiguous()
        assert out.dtype == torch.float32
        r = (C.c_double * 3)(*[float(v) for v in ratio_zyx])
        self._check(self.lib.b200seg_resample_linear(src.data_ptr(), code, *src.shape, C.cast(r, _vp), *out.shape, mode,
                                                     lower, upper, out.data_ptr(), _p(ws),
                                                     0 if ws is None else ws.numel(), dev, st))

    def normalize(self, mode, x, ws, out):
        """x: the fp32 output of resample_linear(..., mode, ws=ws) -> out (a separate fp32 buffer of x's size)"""
        dev, st = self._ds(x)
        assert x.dim() == 3 and x.is_contiguous() and out.is_contiguous() and out.numel() == x.numel()
        self._check(self.lib.b200seg_normalize(mode, x.data_ptr(), *x.shape, ws.data_ptr(), ws.numel(), out.data_ptr(),
                                               dev, st))

    def resample_nearest_u8(self, src, ratio_zyx, valid_zyx, out):
        """src dense uint8 (D, H, W) -> out dense uint8: the NN resample in the valid corner, 0 elsewhere"""
        dev, st = self._ds(src)
        assert src.dtype == torch.uint8 and out.dtype == torch.uint8 and src.dim() == 3 and out.dim() == 3
        assert src.is_contiguous() and out.is_contiguous()
        r = (C.c_double * 3)(*[float(v) for v in ratio_zyx])
        self._check(self.lib.b200seg_resample_nearest_u8(src.data_ptr(), *src.shape, C.cast(r, _vp), *valid_zyx,
                                                         *out.shape, out.data_ptr(), dev, st))

    # ------------------------------------------------------------------ 2-D image resize (csrc/resize2d.cu)
    def resize_linear(self, src, desc, out):
        """cv2.resize(INTER_LINEAR) of a ragged uint8 batch: src a uint8 device buffer holding every sample's rows,
        desc int64 [N, 2] device: the bytes of ``resize_src_table`` (struct b200seg_resize_src), out dense
        (N, oH, oW) uint8 (the cv2 bytes) or fp32 (v / 255)"""
        dev, st = self._ds(src)
        assert src.dtype == torch.uint8 and src.is_contiguous() and desc.dtype == torch.int64 and desc.is_contiguous()
        assert out.dim() == 3 and out.is_contiguous() and desc.shape == (out.shape[0], 2)
        mode = {torch.uint8: U8, torch.float32: F32}[out.dtype]
        n, oh, ow = out.shape
        self._check(self.lib.b200seg_resize_linear_u8(src.data_ptr(), desc.data_ptr(), n, oh, ow, out.data_ptr(), mode,
                                                      dev, st))

    # ------------------------------------------------------------------ 2-D augmentation (csrc/augment2d.cu)
    def augment2d_workspace(self, out_bytes, device):
        """uint8 workspace of b200seg_augment2d_workspace bytes (the blurred images)"""
        nb = int(self.lib.b200seg_augment2d_workspace(int(out_bytes)))
        return torch.empty(max(nb, 16), dtype=torch.uint8, device=device)

    def augment2d(self, src, params, n, max_hw, stages, out, msrc=None, mout=None, ws=None):
        """Segmenation_Aug's stages on a ragged uint8 batch: src / msrc flat uint8 device buffers holding every
        image / mask, params uint8 device bytes of n ``aug2d_param_entry`` entries, out / mout flat uint8 outputs,
        ws a workspace of ``augment2d_workspace(out.numel())`` when ``stages`` has AUG2D_BLUR"""
        dev, st = self._ds(src)
        for t in (src, out, msrc, mout, ws, params):
            assert t is None or (t.dtype == torch.uint8 and t.is_contiguous())
        assert params.numel() >= n * AUG2D_PARAM_BYTES
        self._check(self.lib.b200seg_augment2d(src.data_ptr(), _p(msrc), params.data_ptr(), int(n), int(max_hw),
                                               int(stages), out.data_ptr(), out.numel(), _p(mout), _p(ws),
                                               0 if ws is None else ws.numel(), dev, st))

    # ------------------------------------------------------------------ 3-D augmentation warp (csrc/augment3d.cu)
    def augment3d_workspace(self, n, dhw, device):
        """uint8 workspace of b200seg_augment3d_workspace bytes (the channel shift's min / max partials)"""
        nb = int(self.lib.b200seg_augment3d_workspace(n, *dhw))
        return torch.empty(max(nb, 16), dtype=torch.uint8, device=device)

    def augment3d(self, x, y, params, x_out, y_out, mode=0, cval=0.0, shift=False, rescale=0.0,
                  rescale_mode=RESCALE_NONE, binarize=False, ws=None):
        """ImageDataGenerator3D's order-0 warp of a batch: x dense fp32 (N, D, H, W, C), C in {1, 3, 4}; y dense
        uint8 / fp32 (N, D, H, W); params uint8 device bytes of ``aug3d_param_table`` (N entries); x_out like x;
        y_out like y, or int64 (with ``binarize``: y != 0)"""
        dev, st = self._ds(x)
        assert x.dtype == torch.float32 and x.dim() == 5 and x.is_contiguous() and x_out.is_contiguous()
        assert x_out.dtype == torch.float32 and x_out.shape == x.shape
        assert y.is_contiguous() and y_out.is_contiguous() and y.shape == x.shape[:4] and y_out.shape == y.shape
        assert params.dtype == torch.uint8 and params.numel() >= x.shape[0] * AUG3D_PARAM_BYTES
        codes = {torch.uint8: U8, torch.float32: F32, torch.int64: I64}
        n, d, h, w, c = x.shape
        self._check(self.lib.b200seg_augment3d(x.data_ptr(), y.data_ptr(), codes[y.dtype], n, d, h, w, c,
                                               params.data_ptr(), mode, float(cval), 1 if shift else 0, float(rescale),
                                               rescale_mode, x_out.data_ptr(), y_out.data_ptr(), codes[y_out.dtype],
                                               1 if binarize else 0, _p(ws), 0 if ws is None else ws.numel(), dev,
                                               st))

    # ------------------------------------------------------------------ mask post-processing (csrc/postprocess.cu)
    _PP_DTYPES = {torch.bool: U8, torch.uint8: U8, torch.int16: I16, torch.int32: I32, torch.int64: I64,
                  torch.float32: F32}

    def _pp_mask(self, mask, allow_f32=False):
        """dense (H, W) or (D, H, W) mask -> (dtype code, dims, D, H, W)"""
        code = self._PP_DTYPES.get(mask.dtype)
        if code is None or (code == F32 and not allow_f32):
            raise TypeError(f"unsupported mask dtype {mask.dtype}")
        assert mask.dim() in (2, 3) and mask.is_contiguous()
        dims = mask.dim()
        return (code, dims) + ((1,) + tuple(mask.shape) if dims == 2 else tuple(mask.shape))

    def largest_component(self, mask, out, stats):
        """out uint8 like mask: 1 on the face-connected component with the most voxels (ties: first in C order);
        stats int64 [2] = {components, voxels of the largest}"""
        dev, st = self._ds(mask)
        code, _, d, h, w = self._pp_mask(mask)
        assert out.dtype == torch.uint8 and out.is_contiguous() and out.numel() == mask.numel()
        assert stats.dtype == torch.int64 and stats.numel() >= 2
        nb = int(self.lib.b200seg_components_workspace(d, h, w))
        ws = torch.empty(max(nb, 1), dtype=torch.uint8, device=mask.device)
        self._check(self.lib.b200seg_largest_component(mask.data_ptr(), code, d, h, w, ws.data_ptr(), nb,
                                                       out.data_ptr(), stats.data_ptr(), dev, st))

    def morphology(self, mask, radius, op, out):
        """op: MORPH_* code; out uint8 like mask (0/1)"""
        dev, st = self._ds(mask)
        code, dims, d, h, w = self._pp_mask(mask, allow_f32=True)
        assert out.dtype == torch.uint8 and out.is_contiguous() and out.numel() == mask.numel()
        nb = int(self.lib.b200seg_morphology_workspace(dims, d, h, w, radius, op))
        ws = torch.empty(max(nb, 1), dtype=torch.uint8, device=mask.device)
        self._check(self.lib.b200seg_morphology(mask.data_ptr(), code, dims, d, h, w, radius, op, ws.data_ptr(), nb,
                                                out.data_ptr(), dev, st))

    def label_bbox(self, mask, box):
        """box int64 [2 dims + 1] = {x0, y0, [z0,] sx, sy, [sz,] voxels equal to 1}"""
        dev, st = self._ds(mask)
        code, dims, d, h, w = self._pp_mask(mask)
        assert box.dtype == torch.int64 and box.numel() >= 2 * dims + 1
        nb = int(self.lib.b200seg_label_bbox_workspace())
        ws = torch.empty(nb, dtype=torch.uint8, device=mask.device)
        self._check(self.lib.b200seg_label_bbox(mask.data_ptr(), code, dims, d, h, w, ws.data_ptr(), nb,
                                                box.data_ptr(), dev, st))

    # ------------------------------------------------------------------ Grad-CAM (csrc/gradcam.cu)
    def gradcam_target(self, logits, target, dlogits, category):
        """logits [N][K] fp32 -> dlogits [N][K] fp32 one-hot of each row's class and category [N] int64; target: a
        class for every row, or -1 for the arg-max of each row"""
        dev, st = self._ds(logits)
        n, k = logits.shape
        assert logits.is_contiguous() and dlogits.is_contiguous() and dlogits.shape == logits.shape
        assert category.dtype == torch.int64 and category.numel() == n
        self._check(self.lib.b200seg_gradcam_target(logits.data_ptr(), n, k, int(target), dlogits.data_ptr(),
                                                    category.data_ptr(), dev, st))

    def gradcam(self, stages, out):
        """stages: [(act, grad)] in forward order, each (N, 1, h, w, C) channels-last; out: fp32 (N, H, W) contiguous,
        the Grad-CAM map (per-stage scale and resize, mean over the stages, final scale)"""
        dev, st = self._ds(out)
        n, H, W = out.shape
        assert out.dtype == torch.float32 and out.is_contiguous()
        nb = max(int(self.lib.b200seg_gradcam_workspace(a.shape[0], a.shape[2], a.shape[3], a.shape[4]))
                 for a, _ in stages)
        ws = torch.empty(max(nb, 1), dtype=torch.uint8, device=out.device)
        for i, (a, g) in enumerate(stages):
            da, dg = _desc(a), _desc(g)
            self._check(self.lib.b200seg_gradcam_layer(C.byref(da), C.byref(dg), H, W, i, len(stages), ws.data_ptr(),
                                                       nb, out.data_ptr(), dev, st))
        self._check(self.lib.b200seg_gradcam_scale(out.data_ptr(), n, H, W, ws.data_ptr(), nb, dev, st))

    def mask_logits(self, logits, threshold, mask):
        dev, st = self._ds(logits)
        c = logits.shape[-1]
        self._check(self.lib.b200seg_mask_logits(logits.data_ptr(), logits.numel() // c, c, threshold,
                                                 mask.data_ptr(), dev, st))
