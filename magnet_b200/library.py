"""The inference entry points as ``torch.library`` custom ops (``torch.ops.magnet_b200.*``), so that torch.compile,
CUDA-graph trees and torch.export see each launch as one node instead of a graph break.

Each op's CUDA implementation is the eager ``ops`` function: the argument checks and the ctypes argument structs stay
in ``ops.py``, in one place.  The ``ops`` functions call the op only while torch.compile traces
(``torch.compiler.is_compiling()``); eager calls go to the C entry points directly (DESIGN §3.18).  Every op allocates
its outputs; the one that writes into an argument, ``depth_metrics_update``, declares it in ``mutates_args``.  Each
``register_fake`` states the output shapes and dtypes the eager function returns, from shapes and host arithmetic only.

The training launches are ops too (``TRAIN_OPS``), tied to their backward ops with ``register_autograd``: the G-Net
head, the fused mask loss, the upsample-NLL and F-Net losses, the F volume, and the backwards of ``gaussian_update`` and
``convex_upsample``; D-Net's loss is the pair in ``DNET_TRAIN_OPS``.  What an autograd Function keeps on ``ctx``
(packed weights, saved maps) is an op output here.
The loss ops take the number of supervised pixels as a device tensor and normalise on the device, with the eager
arithmetic inside the op (DESIGN §3.18), so a compiled step has no host read and can be captured in a CUDA graph.
"""
from __future__ import annotations

from typing import List, Optional, Tuple

import torch
from torch import Tensor

from . import _lib, ops

_NS = "magnet_b200"


def _op(name: str, mutates_args=()):
    return torch.library.custom_op(f"{_NS}::{name}", mutates_args=mutates_args, device_types="cuda")


def _grads(ctx, need_from: int, grads):
    """``grads`` with None where ``ctx.needs_input_grad[need_from + i]`` is False."""
    return [g if n else None for g, n in zip(grads, ctx.needs_input_grad[need_from:])]


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


@_op("check_src_index")
def check_src_index(src_index: Tensor, n_src: int) -> Tuple[Tensor, Tensor]:
    """``ops.check_src_index_device``: (int32 table with out-of-range entries replaced by 0, (B,) int32 flags)."""
    return ops.check_src_index_device(src_index, n_src)


@check_src_index.register_fake
def _(src_index, n_src):
    B, V = src_index.shape
    return src_index.new_empty((B, V), dtype=torch.int32), src_index.new_empty((B,), dtype=torch.int32)


@_op("cost_volume_indexed")
def cost_volume_indexed(ref_feat: Tensor, src_feat: Tensor, rays: Tensor, cams: Tensor, V: int, src_layout: int,
                        consistency: bool, src_gmm: Optional[Tensor], kappa: float, d_volume: Optional[Tensor],
                        ref_gmm: Optional[Tensor], k: Optional[List[float]], planes: bool, softmax: bool, variant: int,
                        ref_split: Optional[Tensor], src_index: Tensor, n_src: Optional[int]) -> Tensor:
    """``cost_volume`` with view (b, v) reading source image ``src_index[b, v]`` of the n_src images the source operand
    holds (None: as many as it holds, ``ops.source_images``).  The table is range-checked on the device, never read
    back: the forward reads the sanitised table, and the (D, H, W) block of every sample with an entry outside
    [0, n_src) is then set to NaN."""
    B, C, H, W = ref_feat.shape
    n_img = _source_images(src_layout, src_feat, C, H, W, n_src)
    if src_index.dim() != 2 or tuple(src_index.shape) != (B, V):
        raise _lib.MagnetError(f"src_index must have shape (B, V) = {(B, V)}, got {tuple(src_index.shape)}")
    table, bad = ops.check_src_index_device(src_index, n_img)
    vol = ops.cost_volume(ref_feat, src_feat, rays, cams, V=V, src_layout=src_layout, consistency=consistency,
                          src_gmm=src_gmm, kappa=kappa, d_volume=d_volume, ref_gmm=ref_gmm, k=k, planes=planes,
                          softmax=softmax, variant=variant, ref_split=ref_split, src_index=table, n_src=n_img,
                          check_index=False)
    return vol.masked_fill_((bad != 0).view(B, 1, 1, 1), float("nan"))


def _source_images(src_layout: int, src_feat: Tensor, C, H, W, n_src: Optional[int]) -> int:
    """The source images of an indexed volume: those the operand holds (a packed buffer's count from its size), which
    ``n_src`` must equal when given."""
    n_img = ops.source_images(src_layout, src_feat, int(C), int(H), int(W))
    if n_src is not None and n_src != n_img:
        raise _lib.MagnetError(f"n_src={n_src} does not match src_feat, which holds {n_img} source images")
    return n_img


@cost_volume_indexed.register_fake
def _(ref_feat, src_feat, rays, cams, V, src_layout, consistency, src_gmm, kappa, d_volume, ref_gmm, k, planes,
      softmax, variant, ref_split, src_index, n_src):
    B, C, H, W = ref_feat.shape
    _source_images(src_layout, src_feat, C, H, W, n_src)
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


# --- training: backwards of the update and the upsampling -------------------------------------------------------------

@_op("gaussian_update_bwd")
def gaussian_update_bwd(grad_out: Tensor, d_output: Tensor, ref_gmm: Tensor) -> Tensor:
    return ops.gaussian_update_bwd(grad_out, d_output, ref_gmm)


@gaussian_update_bwd.register_fake
def _(grad_out, d_output, ref_gmm):
    return d_output.new_empty(d_output.shape, dtype=torch.float32)


def _gaussian_update_setup(ctx, inputs, output):
    ctx.save_for_backward(*inputs)


def _gaussian_update_backward(ctx, grad):
    d_output, ref_gmm = ctx.saved_tensors
    return gaussian_update_bwd(grad, d_output, ref_gmm), None


gaussian_update.register_autograd(_gaussian_update_backward, setup_context=_gaussian_update_setup)


@_op("convex_upsample_bwd")
def convex_upsample_bwd(grad_out: Tensor, depth: Tensor, up_mask: Tensor, k: int) -> Tuple[Tensor, Tensor]:
    return ops.convex_upsample_bwd(grad_out, depth, up_mask, k)


@convex_upsample_bwd.register_fake
def _(grad_out, depth, up_mask, k):
    return _f32(depth, *depth.shape), _f32(up_mask, *up_mask.shape)


def _convex_upsample_setup(ctx, inputs, output):
    depth, up_mask, ctx.k = inputs
    ctx.save_for_backward(depth, up_mask)


def _convex_upsample_backward(ctx, grad):
    depth, up_mask = ctx.saved_tensors
    return (*convex_upsample_bwd(grad, depth, up_mask, ctx.k), None)


convex_upsample.register_autograd(_convex_upsample_backward, setup_context=_convex_upsample_setup)


# --- training: G-Net head --------------------------------------------------------------------------------------------

@_op("gnet_train_fwd")
def gnet_train_fwd(cost: Tensor, invariant: Tensor, w0: Tensor, w1: Tensor, b1: Tensor, w2: Tensor, b2: Tensor,
                   w3: Tensor, b3: Tensor, prev_gmm: Tensor) -> Tuple[Tensor, Tensor, Tensor]:
    """``GnetHeadTrain``'s forward: (updated Gaussian, packed training weights, saved hidden maps)."""
    out, packed, saved, _, _ = ops.gnet_train_fwd(cost, invariant, (w0, w1, b1, w2, b2, w3, b3), prev_gmm)
    return out, packed, saved


@gnet_train_fwd.register_fake
def _(cost, invariant, w0, w1, b1, w2, b2, w3, b3, prev_gmm):
    B, D, H, W = cost.shape
    L = _lib.lib()
    return (_f32(cost, B, 2, H, W), _bytes(cost, int(L.magnet_gnet_train_weights_bytes(D))),
            _f32(cost, int(L.magnet_gnet_saved_bytes(B, H, W)) // 4))


@_op("gnet_bwd")
def gnet_bwd(grad_out: Tensor, cost: Tensor, prev_gmm: Tensor, packed: Tensor, saved: Tensor,
             need: List[bool]) -> List[Tensor]:
    """[grad of the invariant, of W0[:, :D], W1, b1, W2, b2, W3, b3, of prev_gmm]; an empty tensor where ``need`` (8
    flags: the weights and prev_gmm) is False."""
    return [_empty_if_none(g, cost) for g in ops.gnet_bwd(grad_out, cost, prev_gmm, packed, saved, need)]


def _empty_if_none(g, like):
    return like.new_empty((0,), dtype=torch.float32) if g is None else g


@gnet_bwd.register_fake
def _(grad_out, cost, prev_gmm, packed, saved, need):
    B, D, H, W = cost.shape
    shapes = [s for _, s in ops.gnet_weight_shapes(D)] + [(B, 2, H, W)]
    return [_f32(cost, B, _lib.MAGNET_HIDDEN_CHANNELS, H, W)] + [_f32(cost, *(s if n else (0,))) for s, n in zip(shapes, need)]


def _gnet_train_setup(ctx, inputs, output):
    cost, prev_gmm = inputs[0], inputs[9]
    ctx.save_for_backward(cost, prev_gmm, output[1], output[2])


def _gnet_train_backward(ctx, grad, _packed, _saved):
    cost, prev_gmm, packed, saved = ctx.saved_tensors
    need = [bool(n) for n in ctx.needs_input_grad[2:10]]
    return (None, *_grads(ctx, 1, gnet_bwd(grad, cost, prev_gmm, packed, saved, need)))


gnet_train_fwd.register_autograd(_gnet_train_backward, setup_context=_gnet_train_setup)


# --- training: the fused mask head, upsampling and loss --------------------------------------------------------------

@_op("mask_train_fwd")
def mask_train_fwd(pre0: Tensor, w1: Tensor, b1: Tensor, w2: Tensor, b2: Tensor, w3: Tensor, b3: Tensor, gt: Tensor,
                   gt_mask: Tensor, count: Tensor, preds: List[Tensor], gamma: float, save_maps: bool,
                   pred_grad: bool) -> Tuple[Tensor, Tensor, Tensor]:
    """``MaskLossTrain``'s forward with the number of supervised pixels ``count`` on the device: (loss, packed training
    weights, saved).  The prediction scales gamma_p / count are formed on the device and read by the kernel when it
    runs; the loss is formed from the partials as the eager forward forms it (NaN for count 0)."""
    P = len(preds)
    gammas = ops.loss_weights(gamma, P)
    # the weights are filled on the device (a host-to-device copy could not be captured in a CUDA graph)
    num = torch.stack([torch.full((), g, dtype=torch.float64, device=pre0.device) for g in gammas])
    scales = ops.device_scales(num, count)
    partial, packed, saved = ops.mask_train_fwd(pre0, (w1, b1, w2, b2, w3, b3), preds, gt, gt_mask, save_maps,
                                                pred_grad, scales)
    terms = ops.loss_term(partial.view(-1, P).sum(0, dtype=torch.float64), count)
    loss = 0.0
    for i in range(P):
        loss = loss + gammas[i] * terms[i]
    return loss, packed, saved


@mask_train_fwd.register_fake
def _(pre0, w1, b1, w2, b2, w3, b3, gt, gt_mask, count, preds, gamma, save_maps, pred_grad):
    B, _, H, W = pre0.shape
    return (pre0.new_empty((), dtype=torch.float32), _bytes(pre0, int(_lib.lib().magnet_mask_train_weights_bytes(4))),
            _f32(pre0, ops.mask_saved_floats(len(preds), B, H, W, save_maps)))


@_op("mask_bwd")
def mask_bwd(grad_loss: Tensor, packed: Tensor, saved: Tensor, P: int, B: int, H: int, W: int,
             need_layers: List[bool], pred_grad: bool) -> List[Tensor]:
    """[grad of pre0, of W1, b1, W2, b2, W3, b3, then of each of the P predictions]; an empty tensor where
    ``need_layers`` (7 flags: pre0 and the six tensors) or ``pred_grad`` is False."""
    g = ops.mask_bwd(grad_loss, packed, saved, (P, B, H, W), need_layers, [pred_grad] * P)
    return [_empty_if_none(t, saved) for t in g]


@mask_bwd.register_fake
def _(grad_loss, packed, saved, P, B, H, W, need_layers, pred_grad):
    shapes = [(B, _lib.MAGNET_HIDDEN_CHANNELS, H, W)] + [s for _, s in ops.mask_weight_shapes()]
    return ([_f32(saved, *(s if n else (0,))) for s, n in zip(shapes, need_layers)]
            + [_f32(saved, *((B, 2, H, W) if pred_grad else (0,))) for _ in range(P)])


def _mask_train_setup(ctx, inputs, output):
    pre0, preds, pred_grad = inputs[0], inputs[10], inputs[13]
    B, _, H, W = pre0.shape
    ctx.shape, ctx.pred_grad = (len(preds), B, H, W), pred_grad
    ctx.save_for_backward(output[1], output[2])


def _mask_train_backward(ctx, grad, _packed, _saved):
    packed, saved = ctx.saved_tensors
    P = ctx.shape[0]
    need = [bool(n) for n in ctx.needs_input_grad[:7]]
    g = mask_bwd(grad, packed, saved, *ctx.shape, need, ctx.pred_grad)
    preds = list(g[7:]) if ctx.pred_grad else [None] * P
    return (*_grads(ctx, 0, g[:7]), None, None, None, preds, None, None, None)


mask_train_fwd.register_autograd(_mask_train_backward, setup_context=_mask_train_setup)


# --- training: the module path's upsample-NLL loss -------------------------------------------------------------------

@_op("upsample_nll_fwd")
def upsample_nll_fwd(depth: Tensor, up_mask: Tensor, gt: Tensor, gt_mask: Tensor, k: int, count: Tensor,
                     weight: float) -> Tensor:
    """``weight * UpsampleNLL(depth, up_mask, gt, gt_mask, k, count)`` with ``count`` on the device: one term of
    ``magnet_loss``, weighted as the eager sum weights it (NaN for count 0)."""
    partial, _ = ops.upsample_nll_fwd(depth, up_mask, gt, gt_mask, k)
    return ops.loss_term(partial.sum(dtype=torch.float64), count) * weight


@upsample_nll_fwd.register_fake
def _(depth, up_mask, gt, gt_mask, k, count, weight):
    return depth.new_empty((), dtype=torch.float32)


@_op("upsample_nll_bwd")
def upsample_nll_bwd(grad: Tensor, depth: Tensor, up_mask: Tensor, gt: Tensor, gt_mask: Tensor, k: int, count: Tensor,
                     weight: float) -> Tuple[Tensor, Tensor]:
    """The gradients of ``upsample_nll_fwd`` w.r.t. (depth, up_mask): the term's upstream gradient ``grad * weight``
    over ``count`` in float64, rounded once to fp32 (0 for count 0), read by the kernel from device memory."""
    scale = ops.device_scales(grad.to(torch.float32) * weight, count)
    return ops.upsample_nll_bwd(depth, up_mask, gt, gt_mask, k, scale)


@upsample_nll_bwd.register_fake
def _(grad, depth, up_mask, gt, gt_mask, k, count, weight):
    return _f32(depth, *depth.shape), _f32(up_mask, *up_mask.shape)


def _upsample_nll_setup(ctx, inputs, output):
    depth, up_mask, gt, gt_mask, ctx.k, count, ctx.weight = inputs
    ctx.save_for_backward(depth, up_mask, gt, gt_mask, count)


def _upsample_nll_backward(ctx, grad):
    depth, up_mask, gt, gt_mask, count = ctx.saved_tensors
    g_depth, g_mask = upsample_nll_bwd(grad, depth, up_mask, gt, gt_mask, ctx.k, count, ctx.weight)
    return g_depth, g_mask, None, None, None, None, None


upsample_nll_fwd.register_autograd(_upsample_nll_backward, setup_context=_upsample_nll_setup)


# --- training: D-Net's upsample-NLL loss (DnetLoss) ------------------------------------------------------------------

@_op("dnet_nll_fwd")
def dnet_nll_fwd(raw: Tensor, up_mask: Tensor, gt: Tensor, gt_mask: Tensor, k: int, count: Tensor) -> Tensor:
    """``UpsampleNLL(raw, up_mask, gt, gt_mask, k, count, dnet=True)`` with ``count`` on the device (NaN for count
    0)."""
    partial, _ = ops.upsample_nll_fwd(raw, up_mask, gt, gt_mask, k, dnet=True)
    return ops.loss_term(partial.sum(dtype=torch.float64), count)


@dnet_nll_fwd.register_fake
def _(raw, up_mask, gt, gt_mask, k, count):
    return raw.new_empty((), dtype=torch.float32)


@_op("dnet_nll_bwd")
def dnet_nll_bwd(grad: Tensor, raw: Tensor, up_mask: Tensor, gt: Tensor, gt_mask: Tensor, k: int,
                 count: Tensor) -> Tuple[Tensor, Tensor]:
    """The gradients of ``dnet_nll_fwd`` w.r.t. (raw, up_mask): the upstream gradient over ``count`` in float64, rounded
    once to fp32 (0 for count 0), read by the kernel from device memory."""
    scale = ops.device_scales(grad.to(torch.float32), count)
    return ops.upsample_nll_bwd(raw, up_mask, gt, gt_mask, k, scale, dnet=True)


@dnet_nll_bwd.register_fake
def _(grad, raw, up_mask, gt, gt_mask, k, count):
    return _f32(raw, *raw.shape), _f32(up_mask, *up_mask.shape)


def _dnet_nll_setup(ctx, inputs, output):
    raw, up_mask, gt, gt_mask, ctx.k, count = inputs
    ctx.save_for_backward(raw, up_mask, gt, gt_mask, count)


def _dnet_nll_backward(ctx, grad):
    raw, up_mask, gt, gt_mask, count = ctx.saved_tensors
    g_raw, g_mask = dnet_nll_bwd(grad, raw, up_mask, gt, gt_mask, ctx.k, count)
    return g_raw, g_mask, None, None, None, None


dnet_nll_fwd.register_autograd(_dnet_nll_backward, setup_context=_dnet_nll_setup)


# --- training: F-Net's L1 loss and the F volume ----------------------------------------------------------------------

@_op("fnet_l1_fwd")
def fnet_l1_fwd(scores: Tensor, planes: List[float], gt: Tensor, mask: Tensor, count: Tensor) -> Tensor:
    """``FnetL1Loss`` with ``count`` on the device (NaN for count 0)."""
    partial = ops.fnet_l1_fwd(scores, planes, gt, mask)[0]
    return ops.loss_term(partial.sum(dtype=torch.float64), count)


@fnet_l1_fwd.register_fake
def _(scores, planes, gt, mask, count):
    return scores.new_empty((), dtype=torch.float32)


@_op("fnet_l1_bwd")
def fnet_l1_bwd(grad: Tensor, scores: Tensor, planes: List[float], gt: Tensor, mask: Tensor, count: Tensor) -> Tensor:
    """The gradient of ``fnet_l1_fwd`` w.r.t. the scores: the eager kernel scale fp32(1 / count) (0 for count 0) times
    the upstream gradient, one fp32 product as the kernel forms it, read from device memory."""
    grad_scale = ops.device_scales(torch.ones_like(count, dtype=torch.float64), count) * grad.to(torch.float32)
    return ops.fnet_l1_bwd(scores, planes, gt, mask, 1.0, grad_scale)


@fnet_l1_bwd.register_fake
def _(grad, scores, planes, gt, mask, count):
    return _f32(scores, *scores.shape)


def _fnet_l1_setup(ctx, inputs, output):
    scores, ctx.planes, gt, mask, count = inputs
    ctx.save_for_backward(scores, gt, mask, count)


def _fnet_l1_backward(ctx, grad):
    scores, gt, mask, count = ctx.saved_tensors
    return fnet_l1_bwd(grad, scores, ctx.planes, gt, mask, count), None, None, None, None


fnet_l1_fwd.register_autograd(_fnet_l1_backward, setup_context=_fnet_l1_setup)


@_op("cost_volume_f")
def cost_volume_f(ref_feat: Tensor, nghbr_feat: Tensor, src: Tensor, ref_split: Optional[Tensor], rays: Tensor,
                  cams: Tensor, V: int, layout: int, variant: int, planes: List[float], softmax: bool,
                  tc_bwd: bool) -> Tensor:
    """The F volume of training (``_CostVolumeF``): ``src`` / ``ref_split`` are the source maps in ``layout`` and the
    reference split the forward reads (``homography.repack_source``); ``ref_feat`` / ``nghbr_feat`` the NCHW maps it is
    differentiable in.  With ``tc_bwd`` and a SPLIT16 / HALF16 layout the backward runs on the tensor cores on the same
    buffers, otherwise on the CUDA cores on the NCHW maps."""
    ref = ref_feat if layout == _lib.SRC_HALF16 else ref_feat.float()
    return ops.cost_volume(ref.detach(), src, rays, cams, V=V, src_layout=layout, consistency=False, k=planes,
                           planes=True, softmax=softmax, variant=variant, ref_split=ref_split)


@cost_volume_f.register_fake
def _(ref_feat, nghbr_feat, src, ref_split, rays, cams, V, layout, variant, planes, softmax, tc_bwd):
    B, _, H, W = ref_feat.shape
    return _f32(ref_feat, B, len(planes), H, W)


@_op("cost_volume_f_bwd")
def cost_volume_f_bwd(grad_out: Tensor, ref_feat: Tensor, nghbr_feat: Tensor, rays: Tensor, cams: Tensor, V: int,
                      planes: List[float], prob: Optional[Tensor], softmax: bool, ref_split: Optional[Tensor],
                      src_split: Optional[Tensor], layout: int) -> Tuple[Tensor, Tensor]:
    """The gradients of ``cost_volume_f`` w.r.t. (ref_feat, nghbr_feat), in their dtypes: the tensor-core kernel on the
    forward's buffers for a SPLIT16 / HALF16 ``layout``, else the CUDA-core kernel on the fp32 NCHW maps."""
    shape_only = layout == _lib.SRC_HALF16
    ref, src = (ref_feat, nghbr_feat) if shape_only else (ref_feat.float(), nghbr_feat.float())
    g_ref, g_src = ops.cost_volume_f_bwd(ref, src, rays, cams, planes, V, prob, grad_out.contiguous(), softmax=softmax,
                                         ref_split=ref_split, src_split=src_split,
                                         split_layout=layout if layout in ops.PACKED_LAYOUTS else _lib.SRC_SPLIT16)
    return g_ref.to(ref_feat.dtype), g_src.to(nghbr_feat.dtype)


@cost_volume_f_bwd.register_fake
def _(grad_out, ref_feat, nghbr_feat, rays, cams, V, planes, prob, softmax, ref_split, src_split, layout):
    return ref_feat.new_empty(ref_feat.shape), nghbr_feat.new_empty(nghbr_feat.shape)


def _cost_volume_f_setup(ctx, inputs, output):
    ref_feat, nghbr_feat, src, ref_split, rays, cams, V, layout, _, planes, softmax, tc_bwd = inputs
    ctx.layout = layout if tc_bwd and layout in ops.PACKED_LAYOUTS else _lib.SRC_NCHW
    packed = ctx.layout in ops.PACKED_LAYOUTS
    ctx.V, ctx.planes, ctx.softmax = V, planes, softmax
    ctx.save_for_backward(ref_feat, nghbr_feat, rays, cams, output if softmax else None, ref_split if packed else None,
                          src if packed else None)


def _cost_volume_f_backward(ctx, grad):
    ref_feat, nghbr_feat, rays, cams, prob, ref_split, src_split = ctx.saved_tensors
    g_ref, g_src = cost_volume_f_bwd(grad, ref_feat, nghbr_feat, rays, cams, ctx.V, ctx.planes, prob, ctx.softmax,
                                     ref_split, src_split, ctx.layout)
    return (g_ref, g_src) + (None,) * 10


cost_volume_f.register_autograd(_cost_volume_f_backward, setup_context=_cost_volume_f_setup)


OPS = ("pack_cameras", "relative_poses", "camera_rays", "sample_depths", "repack_tiled32", "repack_pixc",
       "repack_split16", "repack_half16", "cost_volume", "gaussian_update", "pack_gnet_weights", "gnet_update",
       "convex_upsample", "pack_mask_weights", "mask_upsample", "pack_dnet_weights", "dnet_depth", "dnet_upsample",
       "plane_depth", "depth_metrics", "depth_metrics_update")
# the frame-table path of sequence evaluation (DESIGN §3.17 / §3.18): the device-side range check and the indexed volume
SEQUENCE_OPS = ("check_src_index", "cost_volume_indexed")
TRAIN_OPS = ("gaussian_update_bwd", "convex_upsample_bwd", "gnet_train_fwd", "gnet_bwd", "mask_train_fwd", "mask_bwd",
             "upsample_nll_fwd", "upsample_nll_bwd", "fnet_l1_fwd", "fnet_l1_bwd", "cost_volume_f", "cost_volume_f_bwd")
# D-Net training (DESIGN §3.19): the fused DnetLoss and its backward.  Training ops like TRAIN_OPS, listed apart so
# that TRAIN_OPS stays the set of MaGNet and F-Net training launches its registration tests enumerate.
DNET_TRAIN_OPS = ("dnet_nll_fwd", "dnet_nll_bwd")
