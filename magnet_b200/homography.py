"""Drop-in replacements for ``models.submodules.homography`` of the reference.

Same function names, argument order, argument meaning and return contract as
``est_costvolume_CW`` (homography.py:79-121) and ``est_costvolume_F`` (homography.py:10-47), so
that ``MAGNET.forward`` (models/MAGNET.py:160-164) and ``MAGNET_F.forward`` (:197-200) run
unchanged after ``magnet_b200.install()``.

What the wrapper does around the single kernel launch (all of it hoisted out of the reference's
per-(batch, view) Python loop):
  * ``cam_intrins`` / ``is_valid`` arrive as CPU tensors (test_MaGNet.py:36-50): uploaded once and
    cached across the N_iter calls of one forward (keyed by object identity + version counter);
  * ``R`` / ``t`` arrive as non-contiguous views of ``nghbr_poses`` (MAGNET.py:147-148): passed to
    ``magnet_pack_cameras_f32`` with their strides, no copy;
  * ``nghbr_feat`` / ``nghbr_gmms`` / ``ref_feat`` arrive NCHW: split once per forward into the fp16 hi/lo planes the
    tensor-core kernel's TMA boxes fetch (C == 64; else the pixel-major PIXC layout of the TMA-staged CUDA-core kernel;
    cached the same way; bypassed under CUDA-graph capture).  fp16 / bf16 maps (torch.autocast) of one dtype go
    to the single-plane HALF16 layout where SPLIT16 would be used; in every other case they are upcast to fp32
    once (cached) and take the fp32 rules.  Volumes are fp32, gradients come back in each input's dtype.
Both volumes are differentiable as in the reference: the CW volume w.r.t. both feature maps and the depth volume
(magnet_cost_volume_bwd_f32; built only when grad mode is on and one of them requires grad, so that G-Net training,
where none does, runs exactly the no-grad path), the F volume w.r.t. both feature maps (magnet_cost_volume_f_bwd_f32)
for F-Net training.
"""
from __future__ import annotations

import weakref
from typing import Dict, Tuple

import torch

from . import _lib, ops


class _PrepCache:
    """Cache of per-forward preparations (uploads, repacks, camera tables), keyed on the CALLER's tensors.

    An entry is valid only while the same tensor objects are alive and unmodified: the key holds each source
    tensor's storage pointer, ``_version``, shape, strides and device, plus a weakref to the object the caller
    passed (never to a ``detach()`` temporary), so a freed-and-reallocated tensor at the same address cannot alias a
    stale entry.  Writers that do not bump ``_version`` (a CUDA-graph replay, NCCL, a non-torch kernel) are invisible
    to this key; therefore the cache is BYPASSED while the current stream is being captured (the preparation kernels
    then become part of the graph and replay with the data), and ``clear_cache()`` / ``prep_cache(False)`` exist for
    callers that refill buffers behind torch's back."""

    def __init__(self, capacity: int = 8):
        self.capacity = capacity
        self.enabled = True
        self._items: Dict[Tuple, Tuple[tuple, object]] = {}

    @staticmethod
    def _sig(tensors):
        return tuple((t.data_ptr(), t._version, tuple(t.shape), tuple(t.stride()), str(t.device)) for t in tensors)

    def _usable(self, tensors) -> bool:
        if not self.enabled:
            return False
        if any(t.is_cuda for t in tensors) and torch.cuda.is_current_stream_capturing():
            return False
        return True

    def get(self, kind: str, tensors, extra=()):
        if not self._usable(tensors):
            return None
        key = (kind,) + self._sig(tensors) + tuple(extra)
        hit = self._items.get(key)
        if hit is not None:
            refs, value = hit
            if all(r() is t for r, t in zip(refs, tensors)):
                return value
            del self._items[key]
        return None

    def put(self, kind: str, tensors, value, extra=()):
        if not self._usable(tensors):
            return value
        key = (kind,) + self._sig(tensors) + tuple(extra)
        for dead in [k for k, (refs, _) in self._items.items() if any(r() is None for r in refs)]:
            del self._items[dead]                      # drop preparations whose source tensor is gone
        if len(self._items) >= self.capacity:
            self._items.pop(next(iter(self._items)))
        self._items[key] = (tuple(weakref.ref(t) for t in tensors), value)
        return value

    def clear(self):
        self._items.clear()


_cache = _PrepCache()


def clear_cache() -> None:
    _cache.clear()


def prep_cache(enabled: bool) -> None:
    """Enable / disable the per-forward preparation cache (disabled: every call repacks and re-uploads)."""
    _cache.enabled = bool(enabled)
    if not enabled:
        _cache.clear()


def _device_intrinsics(cam_intrins, device):
    intM, rays = cam_intrins['intM'], cam_intrins['unit_ray_array_2D']
    hit = _cache.get("intr", (intM, rays), (str(device),))
    if hit is not None:
        return hit
    value = (intM.to(device=device, dtype=torch.float32).contiguous(),
             rays.to(device=device, dtype=torch.float32).contiguous())
    return _cache.put("intr", (intM, rays), value, (str(device),))


def _camera_table(cam_intrins, R, t, is_valid, device):
    """K*R, K*t per (b, v): 2 KB, one 3 us kernel.  Cached on the tensors R and t are views OF (MAGNET.py:147-148
    slices nghbr_poses once per forward) — both bases, with their version counters — plus the views' geometry."""
    intM_d, _ = _device_intrinsics(cam_intrins, device)
    rbase = R._base if R._base is not None else R
    tbase = t._base if t._base is not None else t
    src = (rbase, tbase, is_valid, cam_intrins['intM'])
    extra = (R.data_ptr(), tuple(R.shape), tuple(R.stride()), t.data_ptr(), tuple(t.shape), tuple(t.stride()))
    hit = _cache.get("cams", src, extra)
    if hit is not None:
        return hit
    valid_d = is_valid.to(device=device, dtype=torch.int32)
    return _cache.put("cams", src, ops.pack_cameras(intM_d, R, t, valid_d), extra)


MMA_MIN_PLANES = 32   # below half a 64-hypothesis chunk the all-pairs GEMM is wasted: the gather kernel does only the needed taps


def _wants_split16(C: int, V: int, variant: int, D: int) -> bool:
    if variant == _lib.VARIANT_MMA:
        return C == 64 and V <= 16
    return variant == _lib.VARIANT_AUTO and C == 64 and V <= 16 and D >= MMA_MIN_PLANES


def wants_half16(ref_dtype, src_dtype, C: int, V: int, variant: int, D: int) -> bool:
    """The dispatch rule of half-precision feature maps: the single-plane HALF16 layout when both maps have the same
    half dtype and the SPLIT16 conditions hold; otherwise (False) both maps are upcast and today's fp32 rules apply."""
    return ref_dtype == src_dtype and ref_dtype in ops.HALF_DTYPES and _wants_split16(C, V, variant, D)


def _f32(x):
    """x as an fp32 tensor: x itself when it is fp32 (the same object, so that caches keyed on it still hit), else a
    detached upcast cached on x (once per forward)."""
    if x.dtype == torch.float32:
        return x
    hit = _cache.get("f32", (x,))
    if hit is None:
        hit = _cache.put("f32", (x,), x.detach().float())
    return hit


def _wants_pixc(C: int, V: int, variant: int) -> bool:
    return variant in (_lib.VARIANT_AUTO, _lib.VARIANT_TMA) and C in (16, 32, 64) and V <= 16


def _packed_source(nghbr_feat, nghbr_gmms, V, variant, ref_feat=None, D=MMA_MIN_PLANES):
    """The source maps in the layout the selected kernel reads, repacked once per forward (cached on the caller's
    tensor objects): SPLIT16 (fp16 hi/lo planes + Gaussian table, also of the reference features) for the tensor-core
    production kernel (C == 64 and at least MMA_MIN_PLANES hypotheses), PIXC (features + Gaussians, pixel-major) for the TMA-staged CUDA-core kernel, TILED32 for the
    global-gather kernels, NCHW when the channel count fits none.  Half-precision maps: HALF16 by ``wants_half16``,
    else upcast.  Returns (source, layout, reference split or None)."""
    C = nghbr_feat.shape[1]
    if ref_feat is not None and wants_half16(ref_feat.dtype, nghbr_feat.dtype, C, V, variant, D):
        src = (nghbr_feat,) if nghbr_gmms is None else (nghbr_feat, nghbr_gmms)
        hit = _cache.get("half16", src)
        if hit is None:
            hit = _cache.put("half16", src, ops.repack_half16(nghbr_feat.detach(),
                                                              None if nghbr_gmms is None else _f32(nghbr_gmms)))
        ref = _cache.get("half16ref", (ref_feat,))
        if ref is None:
            ref = _cache.put("half16ref", (ref_feat,), ops.repack_half16(ref_feat.detach()))
        return hit, _lib.SRC_HALF16, ref
    nghbr_feat = _f32(nghbr_feat)
    nghbr_gmms = None if nghbr_gmms is None else _f32(nghbr_gmms)
    ref_feat = None if ref_feat is None else _f32(ref_feat)
    if _wants_split16(C, V, variant, D) and ref_feat is not None:
        src = (nghbr_feat,) if nghbr_gmms is None else (nghbr_feat, nghbr_gmms)
        hit = _cache.get("split16", src)
        if hit is None:
            hit = _cache.put("split16", src, ops.repack_split16(nghbr_feat.detach(),
                                                                None if nghbr_gmms is None else nghbr_gmms.detach()))
        ref = _cache.get("split16ref", (ref_feat,))
        if ref is None:
            ref = _cache.put("split16ref", (ref_feat,), ops.repack_split16(ref_feat.detach()))
        return hit, _lib.SRC_SPLIT16, ref
    if variant == _lib.VARIANT_MMA:
        raise _lib.MagnetError(f"MAGNET_VARIANT_MMA needs C == 64 and V <= 16, got C={C}, V={V}")
    if _wants_pixc(C, V, variant):
        src = (nghbr_feat,) if nghbr_gmms is None else (nghbr_feat, nghbr_gmms)
        hit = _cache.get("pixc", src)
        if hit is None:
            hit = _cache.put("pixc", src, ops.repack_pixc(nghbr_feat.detach(),
                                                          None if nghbr_gmms is None else nghbr_gmms.detach()))
        return hit, _lib.SRC_PIXC, None
    if variant == _lib.VARIANT_TMA:
        raise _lib.MagnetError(f"MAGNET_VARIANT_TMA needs C in (16, 32, 64) and V <= 16, got C={C}, V={V}")
    if C % 4 != 0:
        return nghbr_feat.detach().contiguous(), _lib.SRC_NCHW, None
    hit = _cache.get("tiled32", (nghbr_feat,))
    if hit is None:
        hit = _cache.put("tiled32", (nghbr_feat,), ops.repack_tiled32(nghbr_feat.detach()))
    return hit, _lib.SRC_TILED32, None


def check_geometry_grad(**named) -> None:
    """The cost volume is differentiable in the feature maps and the depths only: raise instead of silently dropping
    the gradient of a camera tensor."""
    for name, x in named.items():
        if isinstance(x, torch.Tensor) and x.requires_grad:
            raise _lib.MagnetError(f"{name} requires grad, but the cost volume is differentiable only in the feature "
                                   "maps and the depth hypotheses (detach the camera tensors)")


def wants_cw_grad(*tensors) -> bool:
    """The differentiable CW path is taken only when grad mode is on and one of the differentiable inputs requires
    grad; otherwise the no-grad path runs (same kernels, nothing saved, no autograd node)."""
    return torch.is_grad_enabled() and any(x is not None and x.requires_grad for x in tensors)


class _CostVolumeCW(torch.autograd.Function):
    """Cost volume with per-pixel depths (d_volume, or the Gaussian + k of the fused sampler), differentiable in the
    depth source and both feature maps.  ``run()`` launches the forward kernel and returns (volume, layout, variant,
    (ref split, source split) or None): the backward (magnet_cost_volume_bwd_f32) reproduces that kernel's consistency
    mask.  After a SPLIT16 forward the feature gradients run on the tensor cores on the same split buffers (the rule of
    _PlaneSweepF), otherwise on the CUDA cores; the depth gradient always on the CUDA cores.  The source Gaussians get
    no gradient (the mask is piecewise constant)."""

    @staticmethod
    def forward(ctx, depth, ref_feat, nghbr_feat, nghbr_gmms, run, spec):
        out, layout, variant, splits = run()
        ctx.save_for_backward(depth.detach(), ref_feat.detach(), nghbr_feat.detach(), nghbr_gmms.detach())
        ctx.spec, ctx.fwd, ctx.splits = spec, (layout, variant), splits or (None, None)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        depth, ref_in, src_in, gmm = ctx.saved_tensors
        rays, cams, V, kappa, karr = ctx.spec
        need_d, need_ref, need_src = ctx.needs_input_grad[:3]
        # the CUDA-core kernel reads fp32 NCHW maps: always after a non-HALF16 forward, for the depth gradient after one
        upcast = need_d or ctx.fwd[0] != _lib.SRC_HALF16
        ref, src = (ref_in.float(), src_in.float()) if upcast else (ref_in, src_in)
        g_ref, g_src, g_d = ops.cost_volume_bwd(
            ref, src, gmm.float(), rays, cams, grad_out.contiguous(), V=V, kappa=kappa,
            d_volume=depth if karr is None else None, ref_gmm=depth if karr is not None else None, k=karr,
            fwd_layout=ctx.fwd[0], fwd_variant=ctx.fwd[1], need_ref=need_ref, need_src=need_src, need_depth=need_d,
            ref_split=ctx.splits[0], src_split=ctx.splits[1])
        g_ref = None if g_ref is None else g_ref.to(ref_in.dtype)
        g_src = None if g_src is None else g_src.to(src_in.dtype)
        return g_d, g_ref, g_src, None, None, None


def differentiable_layout(C: int, V: int, D: int, variant: int, split16_ok: bool = True, half=False) -> int:
    """Source layout of a differentiable CW forward: SPLIT16 (tensor cores) where the no-grad path would use it, else
    NCHW with the DIRECT kernel — the two forward kernels whose consistency mask the backward reproduces.  ``half``:
    both feature maps have one half dtype, so HALF16 replaces SPLIT16 (wants_half16)."""
    if variant not in (_lib.VARIANT_AUTO, _lib.VARIANT_MMA, _lib.VARIANT_DIRECT):
        raise _lib.MagnetError("a differentiable CW volume runs on the tensor-core or the DIRECT kernel (variant AUTO, MMA "
                               f"or DIRECT), got variant {variant}")
    if C > 64:
        raise _lib.MagnetError(f"the CW backward supports C <= 64 channels, got C={C}")
    if split16_ok and _wants_split16(C, V, variant, D):
        return _lib.SRC_HALF16 if half else _lib.SRC_SPLIT16
    if variant == _lib.VARIANT_MMA:
        raise _lib.MagnetError(f"MAGNET_VARIANT_MMA needs C == 64 and V <= 16, got C={C}, V={V}")
    return _lib.SRC_NCHW


def est_costvolume_CW(d_volume, ref_feat, nghbr_feat, ref_gmms, nghbr_gmms,
                      R, t, is_valid, cam_intrins, thres, variant=_lib.VARIANT_AUTO):
    """Consistency-weighted multi-view cost volume — drop-in for homography.est_costvolume_CW.

    d_volume (B,D,H,W); ref_feat (B,C,H,W); nghbr_feat (V*B,C,H,W) view-major; ref_gmms unused (as in
    the reference, SURVEY A.5 #7); nghbr_gmms (V*B,2,H,W) [mu, sigma]; R (B,V,3,3), t (B,V,3) device
    views; is_valid (B,V) int CPU or device; cam_intrins dict of 'intM' (B,3,3) and
    'unit_ray_array_2D' (B,3,H*W), CPU or device; thres int.  Returns (B,D,H,W) float32 on
    ref_feat.device, freshly allocated.  Differentiable, as the reference, in d_volume, ref_feat and nghbr_feat when
    grad mode is on and one of them requires grad (the camera tensors must not require grad); detached otherwise.
    Any of the tensors may be fp16 / bf16 (torch.autocast): the volume is fp32, each gradient has its input's dtype."""
    device = ref_feat.device
    B = d_volume.shape[0]
    V = int(nghbr_feat.shape[0] / B)
    if torch.is_grad_enabled():
        check_geometry_grad(R=R, t=t, intM=cam_intrins['intM'], unit_ray_array_2D=cam_intrins['unit_ray_array_2D'])
    d_volume = d_volume.float()                            # differentiable upcast (a no-op for fp32)
    if wants_cw_grad(d_volume, ref_feat, nghbr_feat):
        D, C = int(d_volume.shape[1]), int(ref_feat.shape[1])
        half = wants_half16(ref_feat.dtype, nghbr_feat.dtype, C, V, variant, D)
        layout = differentiable_layout(C, V, D, variant, half=half)
        _, rays_d = _device_intrinsics(cam_intrins, device)
        cams = _camera_table(cam_intrins, R, t, is_valid, device)

        def run():
            if layout in ops.PACKED_LAYOUTS:
                src, _, ref_split = _packed_source(nghbr_feat, nghbr_gmms, V, variant, ref_feat, D)
                fv = variant
            else:
                src, ref_split, fv = _f32(nghbr_feat).detach().contiguous(), None, _lib.VARIANT_DIRECT
            ref = (ref_feat if layout == _lib.SRC_HALF16 else _f32(ref_feat)).detach()
            out = ops.cost_volume(ref, src, rays_d, cams, V=V, src_layout=layout, consistency=True,
                                  src_gmm=_f32(nghbr_gmms).detach(), kappa=float(thres), d_volume=d_volume.detach(),
                                  variant=fv, ref_split=ref_split)
            return out, layout, fv, (ref_split, src) if layout in ops.PACKED_LAYOUTS else None

        return _CostVolumeCW.apply(d_volume, ref_feat, nghbr_feat, nghbr_gmms, run,
                                   (rays_d, cams, V, float(thres), None))
    with torch.no_grad():
        _, rays_d = _device_intrinsics(cam_intrins, device)
        cams = _camera_table(cam_intrins, R, t, is_valid, device)
        src, layout, ref_split = _packed_source(nghbr_feat, nghbr_gmms, V, variant, ref_feat, int(d_volume.shape[1]))
        ref = (ref_feat if layout == _lib.SRC_HALF16 else _f32(ref_feat)).detach()
        return ops.cost_volume(ref, src, rays_d, cams, V=V, src_layout=layout, consistency=True,
                               src_gmm=_f32(nghbr_gmms).detach(), kappa=float(thres), d_volume=d_volume.detach(),
                               variant=variant, ref_split=ref_split)


def _plane_list(d_center):
    """The D plane depths as host floats.  ``d_center`` is a constant of the training run (train_FNet.py:56-66): the
    device -> host read happens once per tensor, not once per step."""
    hit = _cache.get("planes", (d_center,))
    if hit is None:
        hit = _cache.put("planes", (d_center,), d_center.detach().reshape(-1).cpu().tolist())
    return hit


class _CostVolumeF(torch.autograd.Function):
    """Plane-sweep probability volume for F-Net training (homography.py:10-75), forward + backward kernels."""

    @staticmethod
    def forward(ctx, ref_feat, nghbr_feat, planes, rays_d, cams, V, variant):
        src, layout, ref_split = _packed_source(nghbr_feat, None, V, variant, ref_feat, len(planes))
        ref = (ref_feat if layout == _lib.SRC_HALF16 else _f32(ref_feat)).detach()
        out = ops.cost_volume(ref, src, rays_d, cams, V=V, src_layout=layout, consistency=False,
                              k=planes, planes=True, softmax=True, variant=variant, ref_split=ref_split)
        ctx.save_for_backward(ref_feat.detach(), nghbr_feat.detach(), out, rays_d, cams)
        ctx.planes, ctx.V = planes, V
        return out

    @staticmethod
    def backward(ctx, grad_out):
        ref_feat, nghbr_feat, out, rays_d, cams = ctx.saved_tensors
        g_ref, g_src = ops.cost_volume_f_bwd(ref_feat.float(), nghbr_feat.float(), rays_d, cams, ctx.planes, ctx.V, out,
                                             grad_out.contiguous(), softmax=True)
        return g_ref.to(ref_feat.dtype), g_src.to(nghbr_feat.dtype), None, None, None, None, None


class _PlaneSweepF(torch.autograd.Function):
    """Plane-sweep volume of ``MagnetF`` — the 1/V-averaged scores (``softmax=False``, what the fused F-Net loss reads)
    or the probabilities — differentiable in both feature maps.  The backward runs on the tensor cores whenever the
    forward read SPLIT16 buffers (C == 64, V <= 16, at least MMA_MIN_PLANES planes), on the same buffers; otherwise
    the CUDA-core kernel reads the NCHW maps."""

    @staticmethod
    def forward(ctx, ref_feat, nghbr_feat, planes, rays_d, cams, V, softmax):
        src, layout, ref_split = _packed_source(nghbr_feat, None, V, _lib.VARIANT_AUTO, ref_feat, len(planes))
        ref = (ref_feat if layout == _lib.SRC_HALF16 else _f32(ref_feat)).detach()
        out = ops.cost_volume(ref, src, rays_d, cams, V=V, src_layout=layout, consistency=False,
                              k=planes, planes=True, softmax=softmax, ref_split=ref_split)
        ctx.save_for_backward(ref_feat.detach(), nghbr_feat.detach(), out if softmax else None, rays_d, cams)
        ctx.splits = (ref_split, src) if layout in ops.PACKED_LAYOUTS else (None, None)
        ctx.layout = layout
        ctx.planes, ctx.V, ctx.softmax = planes, V, softmax
        return out

    @staticmethod
    def backward(ctx, grad_out):
        ref_feat, nghbr_feat, out, rays_d, cams = ctx.saved_tensors
        ref_split, src_split = ctx.splits
        if ctx.layout == _lib.SRC_HALF16:                  # the NCHW maps only supply the shapes
            ref, src = ref_feat, nghbr_feat
        else:
            ref, src = ref_feat.float(), nghbr_feat.float()
        g_ref, g_src = ops.cost_volume_f_bwd(ref, src, rays_d, cams, ctx.planes, ctx.V, out,
                                             grad_out.contiguous(), softmax=ctx.softmax, ref_split=ref_split,
                                             src_split=src_split, split_layout=ctx.layout)
        return g_ref.to(ref_feat.dtype), g_src.to(nghbr_feat.dtype), None, None, None, None, None


def plane_sweep_f(d_center, ref_feat, nghbr_feat, R, t, is_valid, cam_intrins, softmax=True):
    """The F volume of est_costvolume_F (softmax=True) or its 1/V-averaged scores (softmax=False), with the
    tensor-core backward where the forward ran on the tensor cores (MagnetF's path; est_costvolume_F keeps the
    CUDA-core backward)."""
    device = ref_feat.device
    V = int(nghbr_feat.shape[0] / ref_feat.shape[0])
    planes = _plane_list(d_center)
    _, rays_d = _device_intrinsics(cam_intrins, device)
    cams = _camera_table(cam_intrins, R, t, is_valid, device)
    return _PlaneSweepF.apply(ref_feat, nghbr_feat, planes, rays_d, cams, V, softmax)


def est_costvolume_F(d_center, ref_feat, nghbr_feat, R, t, is_valid, cam_intrins, variant=_lib.VARIANT_AUTO):
    """Fronto-parallel plane-sweep volume with softmax over planes — drop-in (forward) for
    homography.est_costvolume_F.  d_center (1,D,1,1); the rest as in est_costvolume_CW."""
    device = ref_feat.device
    B = ref_feat.shape[0]
    V = int(nghbr_feat.shape[0] / B)
    planes = _plane_list(d_center)
    _, rays_d = _device_intrinsics(cam_intrins, device)
    cams = _camera_table(cam_intrins, R, t, is_valid, device)
    return _CostVolumeF.apply(ref_feat, nghbr_feat, planes, rays_d, cams, V, variant)
