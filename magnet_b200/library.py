"""The inference entry points as ``torch.library`` custom ops (``torch.ops.magnet_b200.*``), so that torch.compile,
CUDA-graph trees and torch.export see each launch as one node instead of a graph break.

Each op's CUDA implementation is the eager ``ops`` function: the argument checks and the ctypes argument structs stay
in ``ops.py``, in one place.  The ``ops`` functions call the op only while torch.compile traces
(``torch.compiler.is_compiling()``); eager calls go to the C entry points directly (DESIGN §3.18).  Every op allocates
its outputs; the one that writes into an argument, ``depth_metrics_update``, declares it in ``mutates_args``.  Each
``register_fake`` states the output shapes and dtypes the eager function returns, from shapes and host arithmetic only.

Training entry points stay ``torch.autograd.Function``s and are not registered.
"""
from __future__ import annotations

from typing import List, Optional, Tuple

import torch
from torch import Tensor

from . import _lib, ops

_NS = "magnet_b200"


def _op(name: str, mutates_args=()):
    return torch.library.custom_op(f"{_NS}::{name}", mutates_args=mutates_args, device_types="cuda")


def _f32(x: Tensor, *shape) -> Tensor:
    return x.new_empty(shape, dtype=torch.float32)


def _bytes(x: Tensor, n: int) -> Tensor:
    return x.new_empty((n,), dtype=torch.uint8)


# --- cameras and sampling --------------------------------------------------------------------------------------------

@_op("pack_cameras")
def pack_cameras(intM: Tensor, R: Tensor, t: Tensor, is_valid: Tensor) -> Tensor:
    return ops.pack_cameras(intM, R, t, is_valid)


@pack_cameras.register_fake
def _(intM, R, t, is_valid):
    return _f32(intM, R.shape[0] * R.shape[1], 16)


@_op("relative_poses")
def relative_poses(ext_ref: Tensor, ext_nghbr: Tensor) -> Tuple[Tensor, Tensor]:
    return ops.relative_poses(ext_ref, ext_nghbr)


@relative_poses.register_fake
def _(ext_ref, ext_nghbr):
    V, B = ext_nghbr.shape[0], ext_nghbr.shape[1]
    return _f32(ext_ref, B, V, 4, 4), ext_ref.new_empty((B, V), dtype=torch.int32)


@_op("camera_rays")
def camera_rays(raw_intrinsics: Tensor, H: int, W: int) -> Tuple[Tensor, Tensor]:
    out = ops.camera_rays(raw_intrinsics, H, W)
    return out["intM"], out["unit_ray_array_2D"]


@camera_rays.register_fake
def _(raw_intrinsics, H, W):
    B = raw_intrinsics.shape[0]
    return _f32(raw_intrinsics, B, 3, 3), _f32(raw_intrinsics, B, 3, H * W)


@_op("sample_depths")
def sample_depths(gmm: Tensor, k: List[float]) -> Tensor:
    return ops.sample_depths(gmm, k)


@sample_depths.register_fake
def _(gmm, k):
    B, _, H, W = gmm.shape
    return _f32(gmm, B, len(k), H, W)


# --- source repacks --------------------------------------------------------------------------------------------------

@_op("repack_tiled32")
def repack_tiled32(x: Tensor) -> Tensor:
    return ops.repack_tiled32(x)


@repack_tiled32.register_fake
def _(x):
    N, C, H, W = x.shape
    return _f32(x, N, H, (W + 31) // 32, C // 4, 32, 4)


@_op("repack_pixc")
def repack_pixc(x: Tensor, gmm: Optional[Tensor]) -> Tensor:
    return ops.repack_pixc(x, gmm)


@repack_pixc.register_fake
def _(x, gmm):
    N, C, H, W = x.shape
    return _f32(x, N, H, W, C + 4)


@_op("repack_split16")
def repack_split16(x: Tensor, gmm: Optional[Tensor]) -> Tensor:
    return ops.repack_split16(x, gmm)


@repack_split16.register_fake
def _(x, gmm):
    N, _, H, W = x.shape
    return _bytes(x, ops.packed_bytes(_lib.SRC_SPLIT16, int(N), int(H), int(W)))


@_op("repack_half16")
def repack_half16(x: Tensor, gmm: Optional[Tensor]) -> Tensor:
    return ops.repack_half16(x, gmm)


@repack_half16.register_fake
def _(x, gmm):
    N, _, H, W = x.shape
    return _bytes(x, ops.packed_bytes(_lib.SRC_HALF16, int(N), int(H), int(W)))


# --- matching --------------------------------------------------------------------------------------------------------

@_op("cost_volume")
def cost_volume(ref_feat: Tensor, src_feat: Tensor, rays: Tensor, cams: Tensor, V: int, src_layout: int,
                consistency: bool, src_gmm: Optional[Tensor], kappa: float, d_volume: Optional[Tensor],
                ref_gmm: Optional[Tensor], k: Optional[List[float]], planes: bool, softmax: bool, variant: int,
                ref_split: Optional[Tensor]) -> Tensor:
    return ops.cost_volume(ref_feat, src_feat, rays, cams, V=V, src_layout=src_layout, consistency=consistency,
                           src_gmm=src_gmm, kappa=kappa, d_volume=d_volume, ref_gmm=ref_gmm, k=k, planes=planes,
                           softmax=softmax, variant=variant, ref_split=ref_split)


@cost_volume.register_fake
def _(ref_feat, src_feat, rays, cams, V, src_layout, consistency, src_gmm, kappa, d_volume, ref_gmm, k, planes,
      softmax, variant, ref_split):
    B, _, H, W = ref_feat.shape
    D = d_volume.shape[1] if d_volume is not None else len(k)
    return ref_feat.new_empty((B, D, H, W), dtype=torch.float32)


@_op("gaussian_update")
def gaussian_update(d_output: Tensor, ref_gmm: Tensor) -> Tensor:
    return ops.GaussianUpdate.apply(d_output, ref_gmm)


@gaussian_update.register_fake
def _(d_output, ref_gmm):
    return d_output.new_empty(d_output.shape, dtype=torch.float32)


@_op("pack_gnet_weights")
def pack_gnet_weights(weights: List[Tensor], D: int) -> Tensor:
    return ops._pack_gnet(weights, D)


@pack_gnet_weights.register_fake
def _(weights, D):
    return _bytes(weights[0], ops.gnet_weights_bytes(D))


@_op("gnet_update")
def gnet_update(cost: Tensor, invariant: Tensor, packed: Tensor, prev_gmm: Tensor) -> Tensor:
    return ops.gnet_update(cost, invariant, packed, prev_gmm)


@gnet_update.register_fake
def _(cost, invariant, packed, prev_gmm):
    B, _, H, W = cost.shape
    return _f32(cost, B, 2, H, W)


# --- upsampling ------------------------------------------------------------------------------------------------------

@_op("convex_upsample")
def convex_upsample(depth: Tensor, up_mask: Tensor, k: int) -> Tensor:
    return ops.ConvexUpsample.apply(depth, up_mask, k)


@convex_upsample.register_fake
def _(depth, up_mask, k):
    B, CH, H, W = depth.shape
    return _f32(depth, B, CH, k * H, k * W)


@_op("pack_mask_weights")
def pack_mask_weights(weights: List[Tensor]) -> Tensor:
    return ops._pack_mask(weights)


@pack_mask_weights.register_fake
def _(weights):
    return _bytes(weights[0], ops.mask_weights_bytes(4))


@_op("mask_upsample")
def mask_upsample(pre0: Tensor, packed: Tensor, preds: List[Tensor], k: int) -> List[Tensor]:
    return ops.mask_upsample(pre0, packed, preds, k)


@mask_upsample.register_fake
def _(pre0, packed, preds, k):
    B, _, H, W = pre0.shape
    return [_f32(pre0, B, 2, 4 * H, 4 * W) for _ in preds]


# --- D-Net heads -----------------------------------------------------------------------------------------------------

@_op("pack_dnet_weights")
def pack_dnet_weights(weights: List[Tensor], k: int) -> Tensor:
    return ops._pack_dnet(weights, k)


@pack_dnet_weights.register_fake
def _(weights, k):
    return _bytes(weights[0], ops.dnet_weights_bytes(k))


@_op("dnet_depth")
def dnet_depth(pre_d: Tensor, packed: Tensor, sigma: bool) -> Tensor:
    return ops.dnet_depth(pre_d, packed, sigma)


@dnet_depth.register_fake
def _(pre_d, packed, sigma):
    B, _, H, W = pre_d.shape
    return _f32(pre_d, B, 2, H, W)


@_op("dnet_upsample")
def dnet_upsample(pre_m: Tensor, packed: Tensor, raw: Tensor, k: int) -> Tensor:
    return ops.dnet_upsample(pre_m, packed, raw, k)


@dnet_upsample.register_fake
def _(pre_m, packed, raw, k):
    B, _, H, W = pre_m.shape
    return _f32(pre_m, B, 2, 4 * H, 4 * W)


# --- evaluation ------------------------------------------------------------------------------------------------------

@_op("plane_depth")
def plane_depth(volume: Tensor, planes: List[float], scores: bool) -> Tensor:
    return ops.plane_depth(volume, planes, scores=scores)


@plane_depth.register_fake
def _(volume, planes, scores):
    B, _, H, W = volume.shape
    return _f32(volume, B, 1, H, W)


@_op("depth_metrics")
def depth_metrics(preds: List[Tensor], gt: Tensor, min_depth: float, max_depth: float, crop: Optional[str],
                  up_mask: Optional[Tensor], k: Optional[int], nearest: bool, variance: bool) -> Tensor:
    return ops.depth_metrics(preds, gt, min_depth=min_depth, max_depth=max_depth, crop=crop, up_mask=up_mask, k=k,
                             nearest=nearest, variance=variance)


def _metric_rows(preds, gt):
    return gt.new_empty((len(preds), gt.shape[0], _lib.MAGNET_METRICS_COLS), dtype=torch.float64)


@depth_metrics.register_fake
def _(preds, gt, min_depth, max_depth, crop, up_mask, k, nearest, variance):
    return _metric_rows(preds, gt)


@_op("depth_metrics_update", mutates_args=("acc",))
def depth_metrics_update(acc: Tensor, preds: List[Tensor], gt: Tensor, min_depth: float, max_depth: float,
                         crop: Optional[str], up_mask: Optional[Tensor], k: Optional[int], nearest: bool,
                         variance: bool) -> Tensor:
    """``DepthMetrics.update``: the (P,B,13) rows of ``depth_metrics``, added into the (P,14) accumulator ``acc``."""
    from .metrics import accumulate
    rows = ops.depth_metrics(preds, gt, min_depth=min_depth, max_depth=max_depth, crop=crop, up_mask=up_mask, k=k,
                             nearest=nearest, variance=variance)
    accumulate(acc, rows)
    return rows


@depth_metrics_update.register_fake
def _(acc, preds, gt, min_depth, max_depth, crop, up_mask, k, nearest, variance):
    return _metric_rows(preds, gt)


OPS = ("pack_cameras", "relative_poses", "camera_rays", "sample_depths", "repack_tiled32", "repack_pixc",
       "repack_split16", "repack_half16", "cost_volume", "gaussian_update", "pack_gnet_weights", "gnet_update",
       "convex_upsample", "pack_mask_weights", "mask_upsample", "pack_dnet_weights", "dnet_depth", "dnet_upsample",
       "plane_depth", "depth_metrics", "depth_metrics_update")
