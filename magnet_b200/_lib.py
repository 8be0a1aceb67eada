"""ctypes binding of libmagnet_b200.so (the C ABI in include/magnet_b200.h).

There is NO fallback: if the shared library is missing or does not export the ABI, importing
the ops raises.  Device pointers are passed as integers (``tensor.data_ptr()``), the stream as
``torch.cuda.current_stream().cuda_stream``.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import os

PKG = Path(__file__).resolve().parent
# MAGNET_B200_LIB selects a tuning build (magnet_b200.build.build(defines=..., tag=...)); default = production
LIB_PATH = Path(os.environ["MAGNET_B200_LIB"]) if os.environ.get("MAGNET_B200_LIB") else PKG / "libmagnet_b200.so"

MAGNET_ABI_VERSION = 4
MAGNET_MAX_PLANES = 256

OK, ERR_NULL, ERR_SHAPE, ERR_UNSUPPORTED, ERR_CUDA, ERR_ALIGN = 0, -1, -2, -3, -4, -5
DEPTH_VOLUME, DEPTH_GAUSS, DEPTH_PLANES = 0, 1, 2
SRC_NCHW, SRC_TILED32, SRC_PIXC, SRC_SPLIT16, SRC_HALF16 = 0, 1, 2, 3, 4
DTYPE_F16, DTYPE_BF16 = 0, 1
INDEX_I32, INDEX_I64 = 0, 1
VARIANT_AUTO, VARIANT_DIRECT, VARIANT_CELLS, VARIANT_CELLS_NOREUSE, VARIANT_TMA, VARIANT_MMA = 0, 1, 2, 3, 4, 5
MAGNET_METRICS_MAX_PRED = 8
MAGNET_METRICS_COLS = 13

MAGNET_HIDDEN_CHANNELS = 128
MAGNET_GNET_SCRATCH_BYTES = 16
MAGNET_MASK_MAX_PRED = 8


class CostArgs(C.Structure):
    """Mirror of ``struct magnet_cost_args``."""
    _fields_ = [
        ("B", C.c_int32), ("V", C.c_int32), ("D", C.c_int32), ("C", C.c_int32), ("H", C.c_int32), ("W", C.c_int32),
        ("depth_mode", C.c_int32), ("src_layout", C.c_int32), ("consistency", C.c_int32), ("softmax", C.c_int32),
        ("variant", C.c_int32), ("kappa", C.c_float),
        ("ref_feat", C.c_void_p), ("src_feat", C.c_void_p), ("src_gmm", C.c_void_p), ("rays", C.c_void_p),
        ("cams", C.c_void_p), ("d_volume", C.c_void_p), ("ref_gmm", C.c_void_p), ("k_host", C.c_void_p),
        ("out", C.c_void_p),
    ]


class CostFBwdArgs(C.Structure):
    """Mirror of ``struct magnet_cost_f_bwd_args``."""
    _fields_ = [("fwd", C.POINTER(CostArgs)), ("prob", C.c_void_p), ("grad_out", C.c_void_p), ("workspace", C.c_void_p),
                ("grad_ref", C.c_void_p), ("grad_src", C.c_void_p)]


class CostBwdArgs(C.Structure):
    """Mirror of ``struct magnet_cost_bwd_args``."""
    _fields_ = [("fwd", C.POINTER(CostArgs)), ("ref_feat", C.c_void_p), ("src_feat", C.c_void_p), ("src_gmm", C.c_void_p),
                ("grad_out", C.c_void_p), ("workspace", C.c_void_p), ("grad_ref", C.c_void_p), ("grad_src", C.c_void_p),
                ("grad_depth", C.c_void_p)]


class CostGeomBwdArgs(C.Structure):
    """Mirror of ``struct magnet_cost_geom_bwd_args``."""
    _fields_ = [("fwd", C.POINTER(CostArgs))] + [
        (n, C.c_void_p) for n in ("ref_feat", "src_feat", "src_gmm", "grad_out", "prob", "score", "workspace",
                                  "grad_cams", "grad_rays", "grad_depth")]


class DepthMetricsArgs(C.Structure):
    """Mirror of ``struct magnet_depth_metrics_args``."""
    _fields_ = [("P", C.c_int32), ("B", C.c_int32), ("H", C.c_int32), ("W", C.c_int32), ("k", C.c_int32),
                ("row0", C.c_int32), ("row1", C.c_int32), ("col0", C.c_int32), ("col1", C.c_int32),
                ("min_depth", C.c_float), ("max_depth", C.c_float),
                ("pred", C.POINTER(C.c_void_p)), ("up_mask", C.c_void_p), ("gt", C.c_void_p), ("workspace", C.c_void_p),
                ("out", C.c_void_p)]


class DepthMetricsNearestArgs(C.Structure):
    """Mirror of ``struct magnet_depth_metrics_nearest_args``."""
    _fields_ = [("P", C.c_int32), ("B", C.c_int32), ("H", C.c_int32), ("W", C.c_int32), ("h", C.c_int32),
                ("w", C.c_int32), ("row0", C.c_int32), ("row1", C.c_int32), ("col0", C.c_int32), ("col1", C.c_int32),
                ("min_depth", C.c_float), ("max_depth", C.c_float),
                ("pred", C.POINTER(C.c_void_p)), ("gt", C.c_void_p), ("workspace", C.c_void_p), ("out", C.c_void_p)]


class GnetArgs(C.Structure):
    """Mirror of ``struct magnet_gnet_args``."""
    _fields_ = [("B", C.c_int32), ("D", C.c_int32), ("H", C.c_int32), ("W", C.c_int32),
                ("cost", C.c_void_p), ("invariant", C.c_void_p), ("packed_weights", C.c_void_p), ("prev_gmm", C.c_void_p),
                ("scratch", C.c_void_p), ("out", C.c_void_p)]


class GnetTrainArgs(C.Structure):
    """Mirror of ``struct magnet_gnet_train_args``."""
    _fields_ = [("B", C.c_int32), ("D", C.c_int32), ("H", C.c_int32), ("W", C.c_int32)] + [
        (n, C.c_void_p) for n in ("cost", "invariant", "packed_weights", "prev_gmm", "scratch", "out", "saved", "grad_out",
                                  "workspace", "grad_invariant", "grad_w0_cost", "grad_w1", "grad_b1", "grad_w2", "grad_b2",
                                  "grad_w3", "grad_b3", "grad_prev")]


class MaskUpsampleArgs(C.Structure):
    """Mirror of ``struct magnet_mask_upsample_args``."""
    _fields_ = [("P", C.c_int32), ("B", C.c_int32), ("H", C.c_int32), ("W", C.c_int32), ("k", C.c_int32),
                ("pre0", C.c_void_p), ("packed_weights", C.c_void_p), ("pred", C.POINTER(C.c_void_p)),
                ("out", C.POINTER(C.c_void_p))]


class MaskTrainArgs(C.Structure):
    """Mirror of ``struct magnet_mask_train_args``."""
    _fields_ = [("P", C.c_int32), ("B", C.c_int32), ("H", C.c_int32), ("W", C.c_int32), ("k", C.c_int32),
                ("pre0", C.c_void_p), ("packed_weights", C.c_void_p), ("pred", C.POINTER(C.c_void_p)),
                ("gt", C.c_void_p), ("gt_mask", C.c_void_p), ("pred_scale", C.POINTER(C.c_float)),
                ("save_maps", C.c_int32), ("pred_grad", C.c_int32), ("partial", C.c_void_p), ("saved", C.c_void_p),
                ("grad_scale", C.c_void_p), ("workspace", C.c_void_p)] + [
        (n, C.c_void_p) for n in ("grad_pre0", "grad_w1", "grad_b1", "grad_w2", "grad_b2", "grad_w3", "grad_b3")] + [
        ("grad_pred", C.POINTER(C.c_void_p))]


_P, _I32, _I64, _F32, _SZ, _ST = C.c_void_p, C.c_int32, C.c_int64, C.c_float, C.c_size_t, C.c_int
_OUT = C.POINTER(C.c_int)

# (restype, argtypes) of every symbol include/magnet_b200.h declares; `lib()` checks the library exports each one
SIGNATURES = {
    "magnet_abi_version": (C.c_int, []),
    "magnet_strerror": (C.c_char_p, [C.c_int]),
    "magnet_last_cuda_error": (C.c_char_p, []),
    "magnet_launch_count": (C.c_uint64, []),
    "magnet_cost_launch_info": (_ST, [C.POINTER(CostArgs), _OUT, _OUT, _OUT]),
    "magnet_cost_volume_f32": (_ST, [C.POINTER(CostArgs), _P]),
    "magnet_cost_volume_indexed_f32": (_ST, [C.POINTER(CostArgs), _P, _I32, _P]),
    "magnet_cost_indexed_launch_info": (_ST, [C.POINTER(CostArgs), _P, _I32, _OUT, _OUT, _OUT]),
    "magnet_check_src_index": (_ST, [_P] + [_I32] * 4 + [_P, _P, _P]),
    "magnet_cost_volume_f_bwd_f32": (_ST, [C.POINTER(CostFBwdArgs), _P]),
    "magnet_cost_volume_bwd_f32": (_ST, [C.POINTER(CostBwdArgs), _P]),
    "magnet_cost_geom_workspace_bytes": (_SZ, [_I32] * 4),
    "magnet_cost_volume_geom_bwd_f32": (_ST, [C.POINTER(CostGeomBwdArgs), _P]),
    "magnet_pack_cameras_f32": (_ST, [_P, _P, _I64, _I64, _I64, _I64, _P, _I64, _I64, _I64, _P, _I32, _I32, _P, _P]),
    "magnet_repack_tiled32_f32": (_ST, [_P, _P] + [_I32] * 4 + [_P]),
    "magnet_repack_pixc_f32": (_ST, [_P, _P, _P] + [_I32] * 4 + [_P]),
    "magnet_split16_bytes": (_SZ, [_I32] * 3),
    "magnet_repack_split16_f32": (_ST, [_P, _P, _P] + [_I32] * 4 + [_P]),
    "magnet_half16_bytes": (_SZ, [_I32] * 3),
    "magnet_repack_half16": (_ST, [_P, _I32, _P, _P] + [_I32] * 4 + [_P]),
    "magnet_sample_depths_f32": (_ST, [_P, _P] + [_I32] * 3 + [_P, _P]),
    "magnet_gaussian_update_fwd_f32": (_ST, [_P, _P, _I32, _I32, _P, _P]),
    "magnet_gaussian_update_bwd_f32": (_ST, [_P, _P, _P, _I32, _I32, _P, _P]),
    "magnet_convex_upsample_fwd_f32": (_ST, [_P, _P] + [_I32] * 5 + [_P, _P]),
    "magnet_convex_upsample_bwd_f32": (_ST, [_P, _P, _P] + [_I32] * 5 + [_P, _P, _P]),
    "magnet_convex_upsample_bwd_det_f32": (_ST, [_P, _P, _P] + [_I32] * 5 + [_P, _P, _P]),
    "magnet_relative_poses_f32": (_ST, [_P, _P, _I32, _I32, _P, _P, _P]),
    "magnet_camera_rays_f32": (_ST, [_P] + [_I32] * 3 + [_P, _P, _P]),
    "magnet_upsample_nll_partials": (_ST, [_I32] * 4),
    "magnet_upsample_nll_fwd_f32": (_ST, [_P] * 4 + [_I32] * 4 + [_P, _P]),
    "magnet_upsample_nll_bwd_f32": (_ST, [_P] * 4 + [_F32] + [_I32] * 4 + [_P, _P, _P]),
    "magnet_upsample_nll_bwd_dev_f32": (_ST, [_P] * 5 + [_I32] * 4 + [_P, _P, _P]),
    "magnet_upsample_nll_bwd_det_workspace_bytes": (_SZ, [_I32] * 4),
    "magnet_upsample_nll_bwd_det_f32": (_ST, [_P] * 4 + [_F32] + [_I32] * 4 + [_P, _P, _P, _P]),
    "magnet_upsample_nll_bwd_dev_det_f32": (_ST, [_P] * 5 + [_I32] * 4 + [_P, _P, _P, _P]),
    "magnet_dnet_nll_fwd_f32": (_ST, [_P] * 4 + [_I32] * 4 + [_P, _P]),
    "magnet_dnet_nll_bwd_f32": (_ST, [_P] * 4 + [_F32] + [_I32] * 4 + [_P, _P, _P]),
    "magnet_dnet_nll_bwd_dev_f32": (_ST, [_P] * 5 + [_I32] * 4 + [_P, _P, _P]),
    "magnet_dnet_nll_bwd_det_f32": (_ST, [_P] * 4 + [_F32] + [_I32] * 4 + [_P, _P, _P, _P]),
    "magnet_dnet_nll_bwd_dev_det_f32": (_ST, [_P] * 5 + [_I32] * 4 + [_P, _P, _P, _P]),
    "magnet_fnet_l1_partials": (_ST, [_I32] * 3),
    "magnet_fnet_l1_fwd_f32": (_ST, [_P] * 4 + [_I32] * 4 + [_P, _P]),
    "magnet_fnet_l1_bwd_f32": (_ST, [_P] * 4 + [_F32, _P] + [_I32] * 4 + [_P, _P]),
    "magnet_plane_depth_f32": (_ST, [_P, _P] + [_I32] * 5 + [_P, _P]),
    "magnet_depth_metrics_workspace": (C.c_int64, [C.POINTER(DepthMetricsArgs)]),
    "magnet_depth_metrics_f32": (_ST, [C.POINTER(DepthMetricsArgs), _P]),
    "magnet_depth_metrics_var_f32": (_ST, [C.POINTER(DepthMetricsArgs), _P]),
    "magnet_depth_metrics_nearest_workspace": (C.c_int64, [C.POINTER(DepthMetricsNearestArgs)]),
    "magnet_depth_metrics_nearest_f32": (_ST, [C.POINTER(DepthMetricsNearestArgs), _P]),
    "magnet_gnet_weights_bytes": (_SZ, [_I32]),
    "magnet_gnet_pack_weights_f32": (_ST, [_P] * 7 + [_I32, _P, _P]),
    "magnet_gnet_update_f32": (_ST, [C.POINTER(GnetArgs), _P]),
    "magnet_gnet_train_weights_bytes": (_SZ, [_I32]),
    "magnet_gnet_saved_bytes": (_SZ, [_I32] * 3),
    "magnet_gnet_bwd_workspace_bytes": (_SZ, [_I32] * 4),
    "magnet_gnet_pack_train_weights_f32": (_ST, [_P] * 7 + [_I32, _P, _P]),
    "magnet_gnet_train_fwd_f32": (_ST, [C.POINTER(GnetTrainArgs), _P]),
    "magnet_gnet_bwd_f32": (_ST, [C.POINTER(GnetTrainArgs), _P]),
    "magnet_mask_weights_bytes": (_SZ, [_I32]),
    "magnet_mask_pack_weights_f32": (_ST, [_P] * 8),
    "magnet_mask_upsample_f32": (_ST, [C.POINTER(MaskUpsampleArgs), _P]),
    "magnet_mask_train_weights_bytes": (_SZ, [_I32]),
    "magnet_mask_saved_bytes": (_SZ, [_I32] * 4),
    "magnet_mask_bwd_workspace_bytes": (_SZ, [_I32] * 3),
    "magnet_mask_train_det_workspace_bytes": (_SZ, [_I32] * 4),
    "magnet_mask_train_partials": (_ST, [_I32] * 3),
    "magnet_mask_pack_train_weights_f32": (_ST, [_P] * 8),
    "magnet_mask_train_fwd_f32": (_ST, [C.POINTER(MaskTrainArgs), _P]),
    "magnet_mask_train_fwd_dev_f32": (_ST, [C.POINTER(MaskTrainArgs), _P, _P]),
    "magnet_mask_train_fwd_det_f32": (_ST, [C.POINTER(MaskTrainArgs), _P]),
    "magnet_mask_train_fwd_dev_det_f32": (_ST, [C.POINTER(MaskTrainArgs), _P, _P]),
    "magnet_mask_bwd_f32": (_ST, [C.POINTER(MaskTrainArgs), _P]),
    "magnet_dnet_weights_bytes": (_SZ, [_I32]),
    "magnet_dnet_pack_weights_f32": (_ST, [_P] * 8 + [_I32, _P, _P]),
    "magnet_dnet_depth_f32": (_ST, [_P, _P] + [_I32] * 4 + [_P, _P]),
    "magnet_dnet_upsample_f32": (_ST, [_P] * 3 + [_I32] * 4 + [_P, _P]),
}
EXPORTS = tuple(SIGNATURES)


class MagnetError(RuntimeError):
    pass


_lib = None


def lib() -> C.CDLL:
    """Load (once) and type the shared library.  Raises if it is missing — never falls back."""
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        raise MagnetError(
            f"{LIB_PATH} not found: build it with `python -m magnet_b200.build` (or __graft_entry__.build()). "
            "magnet_b200 has no CPU / PyTorch fallback for the matching path.")
    L = C.CDLL(str(LIB_PATH))
    for name, (restype, argtypes) in SIGNATURES.items():
        if not hasattr(L, name):
            raise MagnetError(f"{LIB_PATH} does not export {name}")
        fn = getattr(L, name)
        fn.restype, fn.argtypes = restype, argtypes
    if L.magnet_abi_version() != MAGNET_ABI_VERSION:
        raise MagnetError(f"ABI version mismatch: library {L.magnet_abi_version()} != binding {MAGNET_ABI_VERSION}")
    _lib = L
    return L


def check(status: int, what: str) -> None:
    """Status -> RuntimeError (the reference's operators raise plain Python exceptions)."""
    if status == OK:
        return
    L = lib()
    msg = L.magnet_strerror(status).decode()
    if status == ERR_CUDA:
        msg += ": " + L.magnet_last_cuda_error().decode()
    raise MagnetError(f"{what} failed ({status}): {msg}")


def launch_count() -> int:
    return int(lib().magnet_launch_count())
