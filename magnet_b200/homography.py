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
    cached the same way; bypassed under CUDA-graph capture).
The CW volume is not differentiable (its inputs never require grad in the reference, SURVEY §3.2);
the F volume is differentiable w.r.t. both feature maps (magnet_cost_volume_f_bwd_f32) for F-Net training.
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


def _wants_pixc(C: int, V: int, variant: int) -> bool:
    return variant in (_lib.VARIANT_AUTO, _lib.VARIANT_TMA) and C in (16, 32, 64) and V <= 16


def _packed_source(nghbr_feat, nghbr_gmms, V, variant, ref_feat=None, D=MMA_MIN_PLANES):
    """The source maps in the layout the selected kernel reads, repacked once per forward (cached on the caller's
    tensor objects): SPLIT16 (fp16 hi/lo planes + Gaussian table, also of the reference features) for the tensor-core
    production kernel (C == 64 and at least MMA_MIN_PLANES hypotheses), PIXC (features + Gaussians, pixel-major) for the TMA-staged CUDA-core kernel, TILED32 for the
    global-gather kernels, NCHW when the channel count fits none.  Returns (source, layout, reference split or None)."""
    C = nghbr_feat.shape[1]
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


def est_costvolume_CW(d_volume, ref_feat, nghbr_feat, ref_gmms, nghbr_gmms,
                      R, t, is_valid, cam_intrins, thres, variant=_lib.VARIANT_AUTO):
    """Consistency-weighted multi-view cost volume — drop-in for homography.est_costvolume_CW.

    d_volume (B,D,H,W); ref_feat (B,C,H,W); nghbr_feat (V*B,C,H,W) view-major; ref_gmms unused (as in
    the reference, SURVEY A.5 #7); nghbr_gmms (V*B,2,H,W) [mu, sigma]; R (B,V,3,3), t (B,V,3) device
    views; is_valid (B,V) int CPU or device; cam_intrins dict of 'intM' (B,3,3) and
    'unit_ray_array_2D' (B,3,H*W), CPU or device; thres int.  Returns (B,D,H,W) float32 on
    ref_feat.device, freshly allocated, detached."""
    device = ref_feat.device
    B = d_volume.shape[0]
    V = int(nghbr_feat.shape[0] / B)
    with torch.no_grad():
        _, rays_d = _device_intrinsics(cam_intrins, device)
        cams = _camera_table(cam_intrins, R, t, is_valid, device)
        src, layout, ref_split = _packed_source(nghbr_feat, nghbr_gmms, V, variant, ref_feat, int(d_volume.shape[1]))
        return ops.cost_volume(ref_feat.detach(), src, rays_d, cams, V=V, src_layout=layout, consistency=True,
                               src_gmm=nghbr_gmms.detach(), kappa=float(thres), d_volume=d_volume.detach(),
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
        out = ops.cost_volume(ref_feat.detach(), src, rays_d, cams, V=V, src_layout=layout, consistency=False,
                              k=planes, planes=True, softmax=True, variant=variant, ref_split=ref_split)
        ctx.save_for_backward(ref_feat.detach(), nghbr_feat.detach(), out, rays_d, cams)
        ctx.planes, ctx.V = planes, V
        return out

    @staticmethod
    def backward(ctx, grad_out):
        ref_feat, nghbr_feat, out, rays_d, cams = ctx.saved_tensors
        g_ref, g_src = ops.cost_volume_f_bwd(ref_feat, nghbr_feat, rays_d, cams, ctx.planes, ctx.V, out,
                                             grad_out.contiguous(), softmax=True)
        return g_ref, g_src, None, None, None, None, None


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
