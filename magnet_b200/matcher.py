"""H100-native matching loop: the iteration of models/MAGNET.py:150-169 with the sampler fused into
the cost kernel and the Gaussian update as one kernel, prepared once per forward.

The reference inlines the sampler (MAGNET.py:154-156) and the update (inside GNET.forward, :60-69),
so they are only reachable through this alternative loop (or the ``GNET`` mirror below); the
cost-volume function itself is also available as a pure drop-in (``magnet_b200.homography``).
The G-Net / mask-head convolutions stay ordinary ``nn.Module``s (cuDNN), as north_star states.
"""
from __future__ import annotations

from typing import Callable, List, Optional, Sequence

import torch
import torch.nn as nn

from . import _lib, ops
from .homography import (MMA_MIN_PLANES, _CostVolumeCW, check_geometry_grad, differentiable_layout,
                         wants_cw_grad)
from .ops import HALF_DTYPES, PACKED_LAYOUTS
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
    device intrinsics / rays, camera-constant table, source features in the gather layout.

    The feature maps may be fp16 / bf16 (torch.autocast).  Of one half dtype, they go to the single-plane HALF16
    layout wherever the fp32 maps would go to SPLIT16; every other layout reads their fp32 upcast (made once).  The
    Gaussians are upcast; volumes are fp32."""

    def __init__(self, ref_feat, nghbr_feat, nghbr_gmms, nghbr_poses, is_valid, cam_intrins, *,
                 thres: int = 5, src_layout: int = _lib.SRC_SPLIT16):
        if torch.is_grad_enabled():
            check_geometry_grad(nghbr_poses=nghbr_poses, intM=cam_intrins['intM'],
                                unit_ray_array_2D=cam_intrins['unit_ray_array_2D'])
        dev = ref_feat.device
        self.B, self.C, self.H, self.W = ref_feat.shape
        self.V = nghbr_feat.shape[0] // self.B
        self.kappa = float(thres)
        self.ref_feat = ref_feat.detach().contiguous()
        self.src_gmm = nghbr_gmms.detach().float().contiguous()
        # the half dtype of both feature maps (tensor-core kernels on HALF16 buffers), or None (fp32 maps, or upcast)
        self.half = ref_feat.dtype if ref_feat.dtype == nghbr_feat.dtype and ref_feat.dtype in HALF_DTYPES else None
        self._f32 = {}
        self.rays = cam_intrins['unit_ray_array_2D'].to(dev, torch.float32).contiguous()
        intM = cam_intrins['intM'].to(dev, torch.float32).contiguous()
        R, t = nghbr_poses[:, :, :3, :3], nghbr_poses[:, :, :3, 3]
        self.cams = ops.pack_cameras(intM, R, t, is_valid.to(dev, torch.int32))
        self._nghbr_feat = nghbr_feat.detach()
        self._ref_in, self._src_in = ref_feat, nghbr_feat   # the caller's tensors: cost() is differentiable in them
        self._packed = {}
        self._ref_split = None
        # Production: the tensor-core kernel on the fp16 hi/lo planes (C == 64 and at least half a chunk of hypotheses,
        # decided per cost() call); otherwise the global-gather kernel (TILED32), which needs no staging window and
        # no per-thread scratch.  Pass src_layout=SRC_PIXC / variant=VARIANT_TMA for the TMA-staged
        # CUDA-core kernel.  Layouts are packed on first use.
        if src_layout == _lib.SRC_SPLIT16 and not (self.C == 64 and self.V <= 16):
            src_layout = _lib.SRC_TILED32
        if src_layout == _lib.SRC_PIXC and not (self.C in (16, 32, 64) and self.V <= 16):
            src_layout = _lib.SRC_TILED32
        if src_layout == _lib.SRC_TILED32 and self.C % 4 != 0:
            src_layout = _lib.SRC_NCHW
        self.layout = src_layout

    def _fp32(self, which: str) -> torch.Tensor:
        """The reference ('ref') or source ('src') features in fp32: the plan's own when they are fp32, else their
        upcast, made on first use."""
        x = self.ref_feat if which == "ref" else self._nghbr_feat
        if x.dtype == torch.float32:
            return x
        if which not in self._f32:
            self._f32[which] = x.float()
        return self._f32[which]

    def _tc_layout(self, layout: int) -> int:
        """The tensor-core layout the plan's maps take: HALF16 for half maps of one dtype, else SPLIT16."""
        return _lib.SRC_HALF16 if layout == _lib.SRC_SPLIT16 and self.half is not None else layout

    def _ref_operand(self, layout: int) -> torch.Tensor:
        return self.ref_feat if layout == _lib.SRC_HALF16 else self._fp32("ref")

    def _source(self, layout: int):
        """Source maps in ``layout`` (built on first use; the cross-check variants read other layouts than production)."""
        if layout not in self._packed:
            if layout == _lib.SRC_PIXC:
                self._packed[layout] = ops.repack_pixc(self._fp32("src"), self.src_gmm)
            elif layout == _lib.SRC_SPLIT16:
                self._packed[layout] = ops.repack_split16(self._fp32("src"), self.src_gmm)
                self._ref_split = ops.repack_split16(self._fp32("ref"))
            elif layout == _lib.SRC_HALF16:
                self._packed[layout] = ops.repack_half16(self._nghbr_feat, self.src_gmm)
                self._ref_split = ops.repack_half16(self.ref_feat)
            elif layout == _lib.SRC_TILED32:
                self._packed[layout] = ops.repack_tiled32(self._fp32("src"))
            else:
                self._packed[layout] = self._fp32("src").contiguous()
        return self._packed[layout]

    def cost(self, gmm: torch.Tensor, k, out: Optional[torch.Tensor] = None, variant=_lib.VARIANT_AUTO):
        """Fused sampler + CW cost volume for the current Gaussian (B,2,H,W).  Differentiable in the plan's feature maps
        and in ``gmm`` when grad mode is on and one of them requires grad (then ``out`` must be None); detached
        otherwise."""
        gmm = gmm.float()                                  # differentiable upcast (a no-op for fp32)
        if wants_cw_grad(gmm, self._ref_in, self._src_in):
            return self._cost_differentiable(gmm, k, out, variant)
        layout = self.layout
        n_planes = len(k)
        if layout == _lib.SRC_SPLIT16 and variant == _lib.VARIANT_AUTO and n_planes < MMA_MIN_PLANES:
            layout = _lib.SRC_TILED32 if self.C % 4 == 0 else _lib.SRC_NCHW   # few hypotheses: the gather kernel is faster
        if variant == _lib.VARIANT_TMA:
            layout = _lib.SRC_PIXC                         # the TMA-staged kernel fetches its windows from PIXC
        elif variant == _lib.VARIANT_MMA:
            layout = _lib.SRC_SPLIT16                      # the tensor-core kernel reads the fp16 hi/lo planes
        elif layout in (_lib.SRC_PIXC, _lib.SRC_SPLIT16) and variant in (_lib.VARIANT_DIRECT, _lib.VARIANT_CELLS, _lib.VARIANT_CELLS_NOREUSE):
            layout = _lib.SRC_TILED32                      # the global-gather kernels read TILED32
        layout = self._tc_layout(layout)
        src = self._source(layout)
        return ops.cost_volume(self._ref_operand(layout), src, self.rays, self.cams, V=self.V, src_layout=layout,
                               consistency=True, src_gmm=self.src_gmm, kappa=self.kappa, ref_gmm=gmm.detach(),
                               k=k, out=out, variant=variant,
                               ref_split=self._ref_split if layout in PACKED_LAYOUTS else None)


    def _cost_differentiable(self, gmm, k, out, variant):
        if out is not None:
            raise _lib.MagnetError("cost(out=...) writes into a caller buffer and cannot be differentiated")
        karr = ops.k_array(k)
        layout = differentiable_layout(self.C, self.V, len(karr), variant, split16_ok=self.layout == _lib.SRC_SPLIT16,
                                       half=self.half is not None)

        def run():
            packed = layout in PACKED_LAYOUTS
            fv = variant if packed else _lib.VARIANT_DIRECT
            src = self._source(layout)
            vol = ops.cost_volume(self._ref_operand(layout), src, self.rays, self.cams, V=self.V, src_layout=layout,
                                  consistency=True, src_gmm=self.src_gmm, kappa=self.kappa, ref_gmm=gmm.detach(),
                                  k=karr, variant=fv, ref_split=self._ref_split if packed else None)
            return vol, layout, fv, (self._ref_split, src) if packed else None

        return _CostVolumeCW.apply(gmm, self._ref_in, self._src_in, self.src_gmm, run,
                                   (self.rays, self.cams, self.V, self.kappa, karr))


def matching_loop(plan: MatchingPlan, ref_gmms: torch.Tensor, x_d3: torch.Tensor,
                  g_net_convs, n_iter: int, k: Sequence[float],
                  variant=_lib.VARIANT_AUTO, detach_cost: bool = True) -> List[torch.Tensor]:
    """pred_list of MAGNET.py:150-169: [ref_gmms, pred_1, ..., pred_n_iter] at quarter resolution.

    ``g_net_convs`` is either a callable mapping the (B, D+256, H, W) concatenation [cost volume, x_d3] to the
    raw (B,2,H,W) G-Net output (``GNET.gnet``, the reference's data flow), or a ``GNET`` module — then the
    iteration-invariant x_d3 half of the first convolution is computed once and the per-iteration ``cat`` is
    skipped (f-3).  Gradients flow exactly where the reference lets them: through the update into the conv
    weights, never into the cost volume (MAGNET.py:167 detaches it).  With ``detach_cost=False`` the cost volume stays
    in the graph, so feature maps that require grad (a trainable F-Net upstream) receive gradients through it; the
    Gaussian that places the hypotheses stays detached, as in the reference (MAGNET.py:153)."""
    karr = ops.k_array(k)
    preds = [ref_gmms]
    split = isinstance(g_net_convs, GNET)
    inv = g_net_convs.invariant_part(x_d3, len(karr)) if split else None
    for _ in range(n_iter):
        cur = preds[-1].detach().float()                   # a half ref_gmms (autocast) enters the update as fp32
        if detach_cost:
            with torch.no_grad():
                cv = plan.cost(cur, karr, variant=variant)
        else:
            cv = plan.cost(cur, karr, variant=variant)
        raw = g_net_convs.raw_from_parts(cv, inv) if split else g_net_convs(torch.cat([cv, x_d3], dim=1))
        preds.append(ops.gaussian_update(raw.float(), cur))   # raw is half under autocast
    return preds


class MagnetHead(nn.Module):
    """G-Net + mask head + convex upsampling of the reference's ``MAGNET`` (models/MAGNET.py:100-118,
    150-175) operating on backbone outputs; D-Net / F-Net are supplied by the caller (they need
    checkpoints / torch.hub in the reference and are out of scope, SURVEY §2.1 #3-4)."""

    def __init__(self, n_samples: int = 5, sampling_range: float = 3, n_iter: int = 3, thres: int = 5,
                 downsample_ratio: int = 4, dnet_fdim: int = 256, detach_cost: bool = True):
        super().__init__()
        self.n_iter, self.thres, self.downsample_ratio = n_iter, thres, downsample_ratio
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

    def forward(self, ref_feat, nghbr_feat, ref_gmms, nghbr_gmms, x_d3, nghbr_poses, is_valid, cam_intrins):
        preds, mask = self.forward_quarter(ref_feat, nghbr_feat, ref_gmms, nghbr_gmms, x_d3, nghbr_poses, is_valid,
                                           cam_intrins)
        return [self.upsample(pr, mask, self.downsample_ratio) for pr in preds]

    def forward_quarter(self, ref_feat, nghbr_feat, ref_gmms, nghbr_gmms, x_d3, nghbr_poses, is_valid, cam_intrins):
        """The N_iter quarter-resolution predictions and the upsampling mask, NOT upsampled: what the fused
        upsample + NLL loss (``loss`` below) consumes during training.  Under torch.autocast every input may be half;
        the predictions and the mask are fp32."""
        plan = MatchingPlan(ref_feat, nghbr_feat, nghbr_gmms, nghbr_poses, is_valid, cam_intrins, thres=self.thres)
        preds = matching_loop(plan, ref_gmms, x_d3, self.g_net, self.n_iter, self.k_list, detach_cost=self.detach_cost)
        return preds[1:], self.mask_head(x_d3).float()

    def loss(self, preds_quarter, mask, gt_depth, gt_depth_mask, gamma: float = 0.8):
        """MagnetLoss 'gaussian' (utils/losses.py:34-50) of the upsampled predictions without materialising them."""
        return ops.magnet_loss([p.float() for p in preds_quarter], mask.float(), gt_depth.float(), gt_depth_mask,
                               self.downsample_ratio, gamma)


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
                 dnet_fdim: int = 256):
        super().__init__()
        self.d_net, self.f_net = d_net, f_net
        for net in (self.d_net, self.f_net):
            for prm in net.parameters():
                prm.requires_grad = False
            net.eval()
        self.train_iter, self.test_iter = train_iter, test_iter
        thres = int(weighting.split('CW')[1])                   # "CW5" -> kappa = 5 (MAGNET.py:159)
        self.head = MagnetHead(n_samples=n_samples, sampling_range=sampling_range, n_iter=train_iter, thres=thres,
                               downsample_ratio=downsample_ratio, dnet_fdim=dnet_fdim)
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
