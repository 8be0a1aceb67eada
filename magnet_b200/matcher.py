"""H100-native matching loop: the iteration of models/MAGNET.py:150-169 with the sampler fused into
the cost kernel and the Gaussian update as one kernel, prepared once per forward.

The reference inlines the sampler (MAGNET.py:154-156) and the update (inside GNET.forward, :60-69),
so they are only reachable through this alternative loop (or the ``GNET`` mirror below); the
cost-volume function itself is also available as a pure drop-in (``magnet_b200.homography``).  Both take the source
layout and kernel of each call from ``homography.route``; under the default variant the fused sampler keeps the
global-gather kernel where the drop-in takes the TMA-staged one.
In inference the per-iteration G-Net head and update run as one fused kernel (``fused_gnet_applies``); with
``fused_train=True`` so do training iterations of the head (``fused_gnet_trains``, with a fused backward).  With
``fused_upsample=True``, inference runs the mask head after its first convolution and the upsampling of every
prediction as one fused kernel too (``fused_mask_applies``), and ``MagnetHead.train_loss`` runs the same part of the
mask head, the upsampling and the training loss as one differentiable fused op (``fused_mask_trains``).  Autocast and
the hoisted x_d3 convolutions (G-Net's and the mask head's first layer) stay ordinary ``nn.Module``s (cuDNN).
"""
from __future__ import annotations

from typing import Callable, List, Optional, Sequence

import torch
import torch.nn as nn

from . import _lib, ops
from .homography import (_CostVolumeCW, camera_inputs, check_geometry_grad, geometry_grad_enabled, repack_source, route,
                         wants_cw_grad)
from .ops import PACKED_LAYOUTS
from .sampling import depth_sampling


class GNET(nn.Module):
    """Mirror of the reference's ``GNET`` (models/MAGNET.py:47-70): same sub-module names and shapes
    (``gnet.0 .. gnet.6``), hence state-dict compatible; the update equations run in the
    ``magnet_gaussian_update`` kernels (forward + backward) instead of six elementwise ATen ops."""

    def __init__(self, ch_in: int, ch_out: int = 2):
        super().__init__()
        h_dim = 128
        self.gnet = nn.Sequential(
            nn.Conv2d(ch_in, h_dim, 3, padding=1), nn.ReLU(inplace=True),
            nn.Conv2d(h_dim, h_dim, 1), nn.ReLU(inplace=True),
            nn.Conv2d(h_dim, h_dim, 1), nn.ReLU(inplace=True),
            nn.Conv2d(h_dim, ch_out, 1),
        )

    def forward(self, cost_volume: torch.Tensor, ref_gmm: torch.Tensor) -> torch.Tensor:
        # under torch.autocast the convolutions return half tensors: the update kernel reads fp32
        return ops.gaussian_update(self.gnet(cost_volume).float(), ref_gmm.float())

    # --- SURVEY §8 f-3: G-Net input assembly without the per-iteration cat ------------------------------------
    # The reference concatenates [cost_volume (D ch), x_d3 (256 ch)] every iteration (MAGNET.py:167, a 197 MB copy at
    # config 2) and runs the 3x3 conv over all D+256 channels.  x_d3 does not change across iterations, and a
    # convolution is linear in its input channels:  conv(cat[cv, x]) = conv(cv, W[:, :D]) + conv(x, W[:, D:]) + b.
    def invariant_part(self, x_d3: torch.Tensor, n_cost_channels: int) -> torch.Tensor:
        """conv(x_d3, W[:, D:]) + b of the first layer — computed once per forward."""
        c0 = self.gnet[0]
        return nn.functional.conv2d(x_d3, c0.weight[:, n_cost_channels:], c0.bias, padding=1)

    def raw_from_parts(self, cost_volume: torch.Tensor, invariant: torch.Tensor) -> torch.Tensor:
        """The raw (mu_1, sigma_1) output given the cost volume and the precomputed invariant part."""
        c0 = self.gnet[0]
        y = nn.functional.conv2d(cost_volume, c0.weight[:, :cost_volume.shape[1]], None, padding=1) + invariant
        for layer in list(self.gnet)[1:]:
            y = layer(y)
        return y


class MatchingPlan:
    """Everything about one batch that does not change across the N_iter iterations, prepared once:
    device intrinsics / rays, camera-constant table, source features in the layouts ``cost()`` reads.

    Each ``cost()`` call takes its source layout and kernel from ``homography.route`` (the drop-in's rule, except that
    AUTO keeps the global-gather kernel where the drop-in would take the TMA-staged one); a layout is packed on first
    use.  The feature maps may be fp16 / bf16 (torch.autocast): of one half dtype, they go to the single-plane HALF16
    layout wherever the fp32 maps would go to SPLIT16; every other layout reads their fp32 upcast (made once).  The
    Gaussians are upcast; volumes are fp32."""

    def __init__(self, ref_feat, nghbr_feat, nghbr_gmms, nghbr_poses, is_valid, cam_intrins, *, thres: int = 5):
        if torch.is_grad_enabled() and not geometry_grad_enabled():
            check_geometry_grad(nghbr_poses=nghbr_poses, intM=cam_intrins['intM'],
                                unit_ray_array_2D=cam_intrins['unit_ray_array_2D'])
        # the caller's camera tensors: a plan built under geometry_grad() is differentiable in them on every cost()
        # call, wherever that call runs (the switch is latched here); a plan built outside never is
        self._cam_in = camera_inputs(nghbr_poses[:, :, :3, :3], nghbr_poses[:, :, :3, 3], cam_intrins) \
            if geometry_grad_enabled() else (None,) * 4
        dev = ref_feat.device
        self.B, self.C, self.H, self.W = ref_feat.shape
        self.V = nghbr_feat.shape[0] // self.B
        self.kappa = float(thres)
        self.ref_feat = ref_feat.detach().contiguous()
        self.src_gmm = nghbr_gmms.detach().float().contiguous()
        self._f32 = {}
        self.rays = cam_intrins['unit_ray_array_2D'].detach().to(dev, torch.float32).contiguous()
        intM = cam_intrins['intM'].detach().to(dev, torch.float32).contiguous()
        R, t = nghbr_poses.detach()[:, :, :3, :3], nghbr_poses.detach()[:, :, :3, 3]
        self.cams = ops.pack_cameras(intM, R, t, is_valid.to(dev, torch.int32))
        self._nghbr_feat = nghbr_feat.detach()
        self._ref_in, self._src_in = ref_feat, nghbr_feat   # the caller's tensors: cost() is differentiable in them
        self._packed = {}
        self._ref_split = None

    def _fp32(self, which: str) -> torch.Tensor:
        """The reference ('ref') or source ('src') features in fp32: the plan's own when they are fp32, else their
        upcast, made on first use."""
        x = self.ref_feat if which == "ref" else self._nghbr_feat
        if x.dtype == torch.float32:
            return x
        if which not in self._f32:
            self._f32[which] = x.float()
        return self._f32[which]

    def _ref_operand(self, layout: int) -> torch.Tensor:
        return self.ref_feat if layout == _lib.SRC_HALF16 else self._fp32("ref")

    def _source(self, layout: int):
        """Source maps in ``layout`` (built on first use; the cross-check variants read other layouts than production)."""
        if layout not in self._packed:
            feat = self._nghbr_feat if layout == _lib.SRC_HALF16 else self._fp32("src")
            self._packed[layout], ref_split = repack_source(layout, feat, self.src_gmm, self._ref_operand(layout))
            if ref_split is not None:
                self._ref_split = ref_split
        return self._packed[layout]

    def cost(self, gmm: torch.Tensor, k, out: Optional[torch.Tensor] = None, variant=_lib.VARIANT_AUTO):
        """Fused sampler + CW cost volume for the current Gaussian (B,2,H,W).  Differentiable in the plan's feature maps
        and in ``gmm`` when grad mode is on and one of them requires grad (then ``out`` must be None); detached
        otherwise."""
        gmm = gmm.float()                                  # differentiable upcast (a no-op for fp32)
        grad = wants_cw_grad(gmm, self._ref_in, self._src_in, *self._cam_in)
        if grad:
            if out is not None:
                raise _lib.MagnetError("cost(out=...) writes into a caller buffer and cannot be differentiated")
            k = ops.k_array(k)
        layout, fv = route(self.C, self.V, len(k), variant, _lib.DEPTH_GAUSS, self.ref_feat.dtype,
                           self._nghbr_feat.dtype, differentiable=grad)

        def run():
            src = self._source(layout)
            packed = layout in PACKED_LAYOUTS
            vol = ops.cost_volume(self._ref_operand(layout), src, self.rays, self.cams, V=self.V, src_layout=layout,
                                  consistency=True, src_gmm=self.src_gmm, kappa=self.kappa, ref_gmm=gmm.detach(),
                                  k=k, out=out, variant=fv, ref_split=self._ref_split if packed else None)
            return vol, layout, fv, (self._ref_split, src) if packed else None

        if grad:
            return _CostVolumeCW.apply(gmm, self._ref_in, self._src_in, self.src_gmm, run,
                                       (self.rays, self.cams, self.V, self.kappa, k), *self._cam_in)
        return run()[0]


def matching_loop(plan: MatchingPlan, ref_gmms: torch.Tensor, x_d3: torch.Tensor,
                  g_net_convs, n_iter: int, k: Sequence[float],
                  variant=_lib.VARIANT_AUTO, detach_cost: bool = True, fused_train: bool = False) -> List[torch.Tensor]:
    """pred_list of MAGNET.py:150-169: [ref_gmms, pred_1, ..., pred_n_iter] at quarter resolution.

    ``g_net_convs`` is either a callable mapping the (B, D+256, H, W) concatenation [cost volume, x_d3] to the
    raw (B,2,H,W) G-Net output (``GNET.gnet``, the reference's data flow), or a ``GNET`` module — then the
    iteration-invariant x_d3 half of the first convolution is computed once and the per-iteration ``cat`` is
    skipped (f-3).  Gradients flow exactly where the reference lets them: through the update into the conv
    weights, never into the cost volume (MAGNET.py:167 detaches it).  With ``detach_cost=False`` the cost volume stays
    in the graph, so feature maps that require grad (a trainable F-Net upstream) receive gradients through it; the
    Gaussian that places the hypotheses stays detached, as in the reference (MAGNET.py:153).  When nothing needs a
    gradient (see ``fused_gnet_applies``), a ``GNET``'s head and the update of each iteration are one fused kernel, with
    the weights packed once per call.  With ``fused_train`` and a head to train (see ``fused_gnet_trains``), each
    iteration is one differentiable fused op (``ops.gnet_head_train``) instead of the module chain."""
    karr = ops.k_array(k)
    preds = [ref_gmms]
    split = isinstance(g_net_convs, GNET)
    inv = g_net_convs.invariant_part(x_d3, len(karr)) if split else None
    packed = None
    for _ in range(n_iter):
        cur = preds[-1].detach().float()                   # a half ref_gmms (autocast) enters the update as fp32
        if detach_cost:
            with torch.no_grad():
                cv = plan.cost(cur, karr, variant=variant)
        else:
            cv = plan.cost(cur, karr, variant=variant)
        if fused_gnet_applies(g_net_convs, cv, inv):
            if packed is None:                             # the weights are read once per call
                packed = ops.pack_gnet_weights(g_net_convs, cv.shape[1])
            preds.append(ops.gnet_update(cv, inv, packed, cur))
            continue
        if fused_train and fused_gnet_trains(g_net_convs, cv, inv):
            preds.append(ops.gnet_head_train(cv, inv, g_net_convs, cur))
            continue
        raw = g_net_convs.raw_from_parts(cv, inv) if split else g_net_convs(torch.cat([cv, x_d3], dim=1))
        preds.append(ops.gaussian_update(raw.float(), cur))   # raw is half under autocast
    return preds


def fused_gnet_applies(g_net_convs, cv: torch.Tensor, inv: Optional[torch.Tensor]) -> bool:
    """Whether an iteration of ``matching_loop`` runs the fused G-Net head (``ops.gnet_update``) instead of the module
    path (``raw_from_parts`` + ``gaussian_update``): the split data flow of a ``GNET``, nothing to differentiate (grad
    mode off, or no requires_grad among the head's parameters, the cost volume and the invariant), no CUDA autocast,
    fp32 weights and 1 <= D <= MAGNET_MAX_PLANES cost channels.  The fused head has no backward."""
    if not isinstance(g_net_convs, GNET) or inv is None:
        return False
    params = list(g_net_convs.parameters())
    if torch.is_grad_enabled() and (cv.requires_grad or inv.requires_grad or any(p.requires_grad for p in params)):
        return False
    if torch.is_autocast_enabled("cuda"):
        return False
    if any(p.dtype != torch.float32 for p in params) or cv.dtype != torch.float32 or inv.dtype != torch.float32:
        return False
    return 1 <= cv.shape[1] <= _lib.MAGNET_MAX_PLANES


def fused_gnet_trains(g_net_convs, cv: torch.Tensor, inv: Optional[torch.Tensor]) -> bool:
    """Whether a training iteration of ``matching_loop(..., fused_train=True)`` runs the differentiable fused head
    (``ops.gnet_head_train``): the split data flow of a ``GNET``, grad mode on and a head parameter or the invariant
    requiring grad, a cost volume that does not (the fused backward has no gradient into it), no CUDA autocast, fp32
    weights and volume and 1 <= D <= MAGNET_MAX_PLANES cost channels."""
    if not isinstance(g_net_convs, GNET) or inv is None:
        return False
    params = list(g_net_convs.parameters())
    if not torch.is_grad_enabled() or not (inv.requires_grad or any(p.requires_grad for p in params)):
        return False
    if cv.requires_grad or torch.is_autocast_enabled("cuda"):
        return False
    if any(p.dtype != torch.float32 for p in params) or cv.dtype != torch.float32 or inv.dtype != torch.float32:
        return False
    return 1 <= cv.shape[1] <= _lib.MAGNET_MAX_PLANES


def fused_mask_applies(mask_head, pre0: Optional[torch.Tensor], preds, k: int) -> bool:
    """Whether ``MagnetHead(fused_upsample=True).forward`` runs the fused mask head and upsampling
    (``ops.mask_upsample``) instead of ``mask_head(x_d3)`` + ``convex_upsample`` per prediction: a mask head with the
    reference's structure and k == 4, nothing to differentiate (grad mode off, or no requires_grad among the mask
    head's parameters, pre0 and the predictions), no CUDA autocast, fp32 weights, pre0 and predictions.  pre0 may be
    None when it is not computed yet.  The inference kernel has no backward; training takes the fused path of
    ``fused_mask_trains``."""
    if int(k) != 4 or ops.mask_head_layers(mask_head) is None:
        return False
    params = list(mask_head.parameters())
    preds = [preds] if isinstance(preds, torch.Tensor) else list(preds)
    tensors = preds + ([pre0] if pre0 is not None else [])
    if torch.is_grad_enabled() and (any(p.requires_grad for p in params) or any(t.requires_grad for t in tensors)):
        return False
    if torch.is_autocast_enabled("cuda"):
        return False
    return all(p.dtype == torch.float32 for p in params) and all(t.dtype == torch.float32 for t in tensors)


def fused_mask_trains(mask_head, pre0: Optional[torch.Tensor], preds, k: int, gt: Optional[torch.Tensor] = None) -> bool:
    """Whether ``MagnetHead(fused_upsample=True).train_loss`` runs the differentiable fused mask head, upsampling and
    loss (``ops.mask_head_loss``) instead of ``mask_head(x_d3)`` + ``magnet_loss``: a mask head with the reference's
    structure and k == 4, grad mode on with something to differentiate (a mask-head parameter, pre0 or a prediction
    requiring grad), 1 <= P <= MAGNET_MASK_MAX_PRED predictions, no CUDA autocast, fp32 weights, pre0, predictions and
    gt.  pre0 and gt may be None when they are not known yet."""
    if int(k) != 4 or ops.mask_head_layers(mask_head) is None:
        return False
    params = list(mask_head.parameters())
    preds = [preds] if isinstance(preds, torch.Tensor) else list(preds)
    if not 1 <= len(preds) <= _lib.MAGNET_MASK_MAX_PRED:
        return False
    tensors = preds + ([pre0] if pre0 is not None else [])
    if not torch.is_grad_enabled() or not (any(p.requires_grad for p in params) or any(t.requires_grad for t in tensors)):
        return False
    if torch.is_autocast_enabled("cuda"):
        return False
    tensors += [gt] if gt is not None else []
    return all(p.dtype == torch.float32 for p in params) and all(t.dtype == torch.float32 for t in tensors)


def fused_dnet_applies(depth_head, mask_head, x_feat: torch.Tensor, k: int) -> bool:
    """Whether ``DnetHead.forward`` runs the fused D-Net heads (``ops.dnet_depth`` / ``ops.dnet_upsample``) instead of
    the module chain: heads with the reference's structure (``mask_head`` None when it is not run) and k == 4 when the
    mask head is run, nothing to differentiate (grad mode off, or no requires_grad among the heads' parameters and
    x_feat), no CUDA autocast, fp32 weights and x_feat.  The fused kernels have no backward."""
    if ops.dnet_head_layers(depth_head, mask_head) is None:
        return False
    if mask_head is not None and int(k) != 4:
        return False
    params = list(depth_head.parameters()) + (list(mask_head.parameters()) if mask_head is not None else [])
    if torch.is_grad_enabled() and (x_feat.requires_grad or any(p.requires_grad for p in params)):
        return False
    if torch.is_autocast_enabled("cuda"):
        return False
    return all(p.dtype == torch.float32 for p in params) and x_feat.dtype == torch.float32


class DnetHead(nn.Module):
    """D-Net after its trunk: the depth head and the mask head of the reference's ``Decoder``
    (models/submodules/D_dense_depth.py:147-161,187-195) and DNET's activations (models/DNET.py:56-67), on the fused
    kernels where ``fused_dnet_applies`` holds (DESIGN §3.15).

    ``depth_head`` and ``mask_head`` have the reference's structure and names, so a reference checkpoint's
    ``d_net.decoder.depth_head.*`` / ``d_net.decoder.mask_head.*`` entries load with that prefix stripped.
    ``forward(x_feat)`` with x_feat (B, in_dim, h, w), the decoder's output:
      dnet=True:  (B,2,kh,kw) [mu, var], what ``DNET(args)(img)`` returns for that trunk output;
      dnet=False: ((B,2,h,w) [mu, sigma], x_feat), the ``DNET(args, dnet=False)`` contract, so
                  ``nn.Sequential(trunk, DnetHead(dnet=False))`` is a ``d_net`` for ``MAGNET``.  The mask head is built
                  (a checkpoint loads strictly) but not run.
    Where the rule does not hold (training, autocast, other dtypes, other structures or k) the module chain runs, with
    ``ops.convex_upsample`` and torch's elu / sqrt, and stays differentiable."""

    def __init__(self, in_dim: int = 256, downsample_ratio: int = 4, dnet: bool = True):
        super().__init__()
        h_dim = 128
        self.downsample_ratio, self.dnet = downsample_ratio, dnet
        self.depth_head = nn.Sequential(
            nn.Conv2d(in_dim, h_dim, 3, padding=1), nn.ReLU(inplace=True),
            nn.Conv2d(h_dim, h_dim, 1), nn.ReLU(inplace=True),
            nn.Conv2d(h_dim, 2, 1),
        )
        self.mask_head = nn.Sequential(
            nn.Conv2d(in_dim, h_dim, 3, padding=1), nn.ReLU(inplace=True),
            nn.Conv2d(h_dim, h_dim, 1), nn.ReLU(inplace=True),
            nn.Conv2d(h_dim, 9 * downsample_ratio * downsample_ratio, 1),
        )

    @staticmethod
    def _pre(head: nn.Sequential, x: torch.Tensor) -> torch.Tensor:
        """The head's 3x3 convolution before its ReLU (cuDNN), the part that stays outside the fused kernels."""
        c0 = head[0]
        return nn.functional.conv2d(x, c0.weight, c0.bias, c0.stride, c0.padding, c0.dilation, c0.groups)

    def forward(self, x_feat: torch.Tensor):
        k = self.downsample_ratio
        mask_head = self.mask_head if self.dnet else None
        if fused_dnet_applies(self.depth_head, mask_head, x_feat, k):
            packed = ops.pack_dnet_weights(self.depth_head, mask_head)
            raw = ops.dnet_depth(self._pre(self.depth_head, x_feat), packed, sigma=not self.dnet)
            if not self.dnet:
                return raw, x_feat
            return ops.dnet_upsample(self._pre(self.mask_head, x_feat), packed, raw, k)
        depth = self.depth_head(x_feat)
        if not self.dnet:                                   # activation_G_magnet (DNET.py:62-67)
            mu, v = torch.split(depth, 1, dim=1)
            return torch.cat([mu, torch.sqrt(nn.functional.elu(v) + 1.0 + 1e-10)], dim=1), x_feat
        up = ops.convex_upsample(depth.float(), self.mask_head(x_feat).float(), k)
        mu, v = torch.split(up, 1, dim=1)                   # activation_G (DNET.py:56-60)
        return torch.cat([mu, nn.functional.elu(v) + 1.0 + 1e-10], dim=1)


class MagnetHead(nn.Module):
    """G-Net + mask head + convex upsampling of the reference's ``MAGNET`` (models/MAGNET.py:100-118,
    150-175) operating on backbone outputs; D-Net / F-Net are supplied by the caller (they need
    checkpoints / torch.hub in the reference and are out of scope, SURVEY §2.1 #3-4)."""

    def __init__(self, n_samples: int = 5, sampling_range: float = 3, n_iter: int = 3, thres: int = 5,
                 downsample_ratio: int = 4, dnet_fdim: int = 256, detach_cost: bool = True, fused_train: bool = False,
                 fused_upsample: bool = False):
        super().__init__()
        self.n_iter, self.thres, self.downsample_ratio = n_iter, thres, downsample_ratio
        # True: forward runs the mask head after its first convolution and the upsampling of every prediction as one
        # fused kernel where fused_mask_applies holds (inference), and train_loss runs that part and the loss as one
        # differentiable fused op where fused_mask_trains holds; the full mask is then never computed
        self.fused_upsample = fused_upsample
        # True: training iterations of the G-Net head run the differentiable fused kernels where fused_gnet_trains holds
        self.fused_train = fused_train
        # True: G-Net reads a detached cost volume (MAGNET.py:167).  False: the volume stays in the graph, so a trainable
        # F-Net upstream receives gradients through the matching.
        self.detach_cost = detach_cost
        self.k_list = depth_sampling(sampling_range, n_samples)
        self.g_net = GNET(ch_in=dnet_fdim + n_samples, ch_out=2)
        h_dim = 128
        self.mask_head = nn.Sequential(
            nn.Conv2d(dnet_fdim, h_dim, 3, padding=1), nn.ReLU(inplace=True),
            nn.Conv2d(h_dim, h_dim, 1), nn.ReLU(inplace=True),
            nn.Conv2d(h_dim, h_dim, 1), nn.ReLU(inplace=True),
            nn.Conv2d(h_dim, 9 * downsample_ratio * downsample_ratio, 1),
        )

    @staticmethod
    def upsample(depth, up_mask, k):
        """upsample_depth_via_mask (MAGNET.py:15-27) — fused kernels, no (B,2,9,k,k,H,W) temporaries (f-2)."""
        return ops.convex_upsample(depth.float(), up_mask.float(), k)

    def mask_pre(self, x_d3: torch.Tensor) -> torch.Tensor:
        """The mask head's first layer before its ReLU, conv3x3(x_d3, W0) + b0: the part of the mask head that stays on
        cuDNN when the rest runs fused (``ops.mask_upsample``).  The same convolution ``mask_head[0]`` computes."""
        c0 = self.mask_head[0]
        return nn.functional.conv2d(x_d3, c0.weight, c0.bias, c0.stride, c0.padding, c0.dilation, c0.groups)

    def forward(self, ref_feat, nghbr_feat, ref_gmms, nghbr_gmms, x_d3, nghbr_poses, is_valid, cam_intrins):
        k = self.downsample_ratio
        if self.fused_upsample:
            preds = self._predictions(ref_feat, nghbr_feat, ref_gmms, nghbr_gmms, x_d3, nghbr_poses, is_valid,
                                      cam_intrins)
            if fused_mask_applies(self.mask_head, None, preds, k):
                pre0 = self.mask_pre(x_d3)
                if fused_mask_applies(self.mask_head, pre0, preds, k):
                    return ops.mask_upsample(pre0, ops.pack_mask_weights(self.mask_head), preds, k)
            mask = self.mask_head(x_d3).float()
        else:
            preds, mask = self.forward_quarter(ref_feat, nghbr_feat, ref_gmms, nghbr_gmms, x_d3, nghbr_poses, is_valid,
                                               cam_intrins)
        return [self.upsample(pr, mask, k) for pr in preds]

    def _predictions(self, ref_feat, nghbr_feat, ref_gmms, nghbr_gmms, x_d3, nghbr_poses, is_valid, cam_intrins):
        plan = MatchingPlan(ref_feat, nghbr_feat, nghbr_gmms, nghbr_poses, is_valid, cam_intrins, thres=self.thres)
        preds = matching_loop(plan, ref_gmms, x_d3, self.g_net, self.n_iter, self.k_list, detach_cost=self.detach_cost,
                              fused_train=self.fused_train)
        return preds[1:]

    def forward_quarter(self, ref_feat, nghbr_feat, ref_gmms, nghbr_gmms, x_d3, nghbr_poses, is_valid, cam_intrins):
        """The N_iter quarter-resolution predictions and the upsampling mask, NOT upsampled: what the fused
        upsample + NLL loss (``loss`` below) consumes during training.  Under torch.autocast every input may be half;
        the predictions and the mask are fp32."""
        preds = self._predictions(ref_feat, nghbr_feat, ref_gmms, nghbr_gmms, x_d3, nghbr_poses, is_valid, cam_intrins)
        return preds, self.mask_head(x_d3).float()

    def loss(self, preds_quarter, mask, gt_depth, gt_depth_mask, gamma: float = 0.8):
        """MagnetLoss 'gaussian' (utils/losses.py:34-50) of the upsampled predictions without materialising them."""
        return ops.magnet_loss([p.float() for p in preds_quarter], mask.float(), gt_depth.float(), gt_depth_mask,
                               self.downsample_ratio, gamma)

    def train_loss(self, ref_feat, nghbr_feat, ref_gmms, nghbr_gmms, x_d3, nghbr_poses, is_valid, cam_intrins, gt_depth,
                   gt_depth_mask, gamma: float = 0.8):
        """The scalar loss of one training step: ``loss(*forward_quarter(...), gt_depth, gt_depth_mask, gamma)``.  With
        ``fused_upsample`` and ``fused_mask_trains`` holding, the mask head after ``mask_pre`` runs with the upsampling
        and the loss as one differentiable fused op (``ops.mask_head_loss``): the 144-channel mask is never computed."""
        k = self.downsample_ratio
        if self.fused_upsample:
            preds = self._predictions(ref_feat, nghbr_feat, ref_gmms, nghbr_gmms, x_d3, nghbr_poses, is_valid,
                                      cam_intrins)
            if fused_mask_trains(self.mask_head, None, preds, k, gt_depth):
                pre0 = self.mask_pre(x_d3)
                if fused_mask_trains(self.mask_head, pre0, preds, k, gt_depth):
                    return ops.mask_head_loss(pre0, self.mask_head, preds, gt_depth, gt_depth_mask, k, gamma)
            mask = self.mask_head(x_d3).float()
        else:
            preds, mask = self.forward_quarter(ref_feat, nghbr_feat, ref_gmms, nghbr_gmms, x_d3, nghbr_poses, is_valid,
                                               cam_intrins)
        return self.loss(preds, mask, gt_depth, gt_depth_mask, gamma)


class MAGNET(nn.Module):
    """The reference's ``MAGNET`` (models/MAGNET.py:73-175) with the matching loop on the H100 kernels.

    Same forward signature and return value: ``forward(ref_img, nghbr_imgs, nghbr_poses, is_valid, cam_intrins,
    mode)`` -> list of N_iter upsampled (B,2,H,W) Gaussians.  The backbones are passed in (the reference builds
    them from checkpoints / torch.hub, out of scope here): ``d_net(imgs) -> ((N,2,h,w) [mu, sigma], (N,256,h,w))``
    and ``f_net(imgs) -> (N,C,h,w)`` as DNET.py:62-67 / F_psmnet.py:122-124; they are frozen and run under
    ``no_grad`` in ``eval()`` mode exactly like MAGNET.py:82-92,133-144.  ``g_net`` / ``mask_head`` have the
    reference's parameter names, so ``load_state_dict`` of a reference checkpoint's head works."""

    def __init__(self, d_net: nn.Module, f_net: nn.Module, n_samples: int = 5, sampling_range: float = 3,
                 weighting: str = "CW5", train_iter: int = 3, test_iter: int = 3, downsample_ratio: int = 4,
                 dnet_fdim: int = 256, fused_train: bool = False, fused_upsample: bool = False):
        super().__init__()
        self.d_net, self.f_net = d_net, f_net
        for net in (self.d_net, self.f_net):
            for prm in net.parameters():
                prm.requires_grad = False
            net.eval()
        self.train_iter, self.test_iter = train_iter, test_iter
        thres = int(weighting.split('CW')[1])                   # "CW5" -> kappa = 5 (MAGNET.py:159)
        self.head = MagnetHead(n_samples=n_samples, sampling_range=sampling_range, n_iter=train_iter, thres=thres,
                               downsample_ratio=downsample_ratio, dnet_fdim=dnet_fdim, fused_train=fused_train,
                               fused_upsample=fused_upsample)
        self.g_net, self.mask_head = self.head.g_net, self.head.mask_head   # reference attribute names

    def train(self, mode: bool = True):
        super().train(mode)
        self.d_net.eval()        # frozen backbones stay in eval (the reference's model.train() flips them — SURVEY §2.3 quirk)
        self.f_net.eval()
        return self

    def forward(self, ref_img, nghbr_imgs, nghbr_poses, is_valid, cam_intrins, mode='train'):
        B = ref_img.shape[0]
        with torch.no_grad():
            imgs = torch.cat((ref_img, nghbr_imgs), dim=0)
            mono_gmms, x_d3 = self.d_net(imgs)
            feat = self.f_net(imgs)
        self.head.n_iter = self.train_iter if mode == 'train' else self.test_iter
        return self.head(feat[:B], feat[B:], mono_gmms[:B].detach(), mono_gmms[B:].detach(), x_d3[:B], nghbr_poses,
                         is_valid, cam_intrins)


def sid_planes(min_depth: float, max_depth: float, n: int = 80, device=None) -> torch.Tensor:
    """The F-Net plane depths of train_FNet.py:56-66: centres of n spacing-increasing-discretisation (SID) bins on
    [min_depth, max_depth], evaluated in float64 and rounded to float32, shape (1, n, 1, 1)."""
    import numpy as np
    idx = np.arange(n + 1)
    gamma = 1 - min_depth
    bounds = np.exp(np.log(max_depth + gamma) * idx / n) - gamma
    centre = (bounds[:-1] + bounds[1:]) / 2
    return torch.from_numpy(centre.astype(np.float32)).view(1, n, 1, 1).to(device)


class MagnetF(nn.Module):
    """The reference's ``MAGNET_F`` (models/MAGNET.py:179-202) — F-Net + plane-sweep volume — with the volume, its
    backward and the training loss on the H100 kernels.  The attribute is ``f_net``, so a reference F-Net state dict
    loads; ``f_net(imgs) -> (N, C, h, w)`` as F_psmnet.py:122-124 (cuDNN, trained)."""

    def __init__(self, f_net: nn.Module):
        super().__init__()
        self.f_net = f_net

    def _features(self, ref_img, nghbr_imgs):
        B = ref_img.shape[0]
        feat = self.f_net(torch.cat((ref_img, nghbr_imgs), dim=0))
        return feat[:B], feat[B:]

    def forward(self, ref_img, nghbr_imgs, nghbr_poses, is_valid, cam_intrins, d_center):
        """(B, D, h, w) probability volume over the planes ``d_center`` (1, D, 1, 1), the reference's contract."""
        from .homography import plane_sweep_f
        ref_feat, nghbr_feat = self._features(ref_img, nghbr_imgs)
        return plane_sweep_f(d_center, ref_feat, nghbr_feat, nghbr_poses[:, :, :3, :3], nghbr_poses[:, :, :3, 3],
                             is_valid, cam_intrins, softmax=True)

    def loss(self, ref_img, nghbr_imgs, nghbr_poses, is_valid, cam_intrins, d_center, gt_dmap, min_depth: float,
             max_depth: float):
        """The L1 loss of train_FNet.py:87-108: gt above max_depth is zeroed, gt is nearest-resized to the volume's
        grid and supervises where it exceeds min_depth; the soft-argmin depth comes from the fused loss kernel on the
        plane-sweep scores (no probability volume, no prediction map), and both backwards run in CUDA kernels."""
        from .homography import _plane_list, plane_sweep_f
        ref_feat, nghbr_feat = self._features(ref_img, nghbr_imgs)
        scores = plane_sweep_f(d_center, ref_feat, nghbr_feat, nghbr_poses[:, :, :3, :3], nghbr_poses[:, :, :3, 3],
                               is_valid, cam_intrins, softmax=False)
        gt_dmap = gt_dmap.float()
        gt = torch.where(gt_dmap > max_depth, torch.zeros_like(gt_dmap), gt_dmap)
        gt = nn.functional.interpolate(gt, size=[scores.shape[2], scores.shape[3]], mode='nearest')
        return ops.fnet_l1_loss(scores, _plane_list(d_center), gt.contiguous(), gt > min_depth)

    def predict(self, ref_img, nghbr_imgs, nghbr_poses, is_valid, cam_intrins, d_center):
        """F-Net's soft-argmin depth map (train_FNet.py:96 / :180) on the volume's grid, (B, 1, h, w) float32: the
        plane-sweep scores followed by ``ops.plane_depth`` with the softmax fused in, so the probability volume is never
        written.  The prediction is bit for bit the one ``loss`` supervises.  Inference
        only: it runs under ``torch.no_grad()`` and the result carries no graph.  Score it against the full-resolution
        GT with ``DepthMetrics.update(pred, gt, nearest=True)``."""
        from .homography import _plane_list, plane_sweep_f
        with torch.no_grad():
            ref_feat, nghbr_feat = self._features(ref_img, nghbr_imgs)
            scores = plane_sweep_f(d_center, ref_feat, nghbr_feat, nghbr_poses[:, :, :3, :3], nghbr_poses[:, :, :3, 3],
                                   is_valid, cam_intrins, softmax=False)
            return ops.plane_depth(scores, _plane_list(d_center), scores=True)


def install(homography_module=None) -> None:
    """Rebind the reference's operators to the H100 kernels so that ``MAGNET.forward`` /
    ``MAGNET_F.forward`` / ``test_MaGNet.py`` run unchanged:

        import models.submodules.homography as homography   # the reference's module
        import magnet_b200; magnet_b200.install(homography)

    With no argument the module is looked up in ``sys.modules`` under its reference name."""
    import sys

    from . import homography as ours

    ours_lib = _lib.lib()   # fail now, loudly, if the CUDA library is missing
    del ours_lib
    mod = homography_module or sys.modules.get("models.submodules.homography")
    if mod is None:
        raise _lib.MagnetError("models.submodules.homography is not imported; pass the module to install()")
    mod.est_costvolume_CW = ours.est_costvolume_CW
    mod.est_costvolume_F = ours.est_costvolume_F
