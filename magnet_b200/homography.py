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
  * ``nghbr_feat`` / ``nghbr_gmms`` / ``ref_feat`` arrive NCHW: repacked once per forward (cached the same way;
    bypassed under CUDA-graph capture) into the source layout ``route()`` picks for the call — the one rule shared
    with ``MatchingPlan``: the fp16 hi/lo planes the tensor-core kernel's TMA boxes fetch (C == 64 and at least
    MMA_MIN_PLANES hypotheses), or for fp16 / bf16 maps of one dtype (torch.autocast) their single-plane HALF16
    form; else the pixel-major PIXC layout of the TMA-staged CUDA-core kernel, TILED32 or NCHW, read from fp32 maps
    (half maps upcast once, cached).  Volumes are fp32, gradients come back in each input's dtype.
Both volumes are differentiable as in the reference: the CW volume w.r.t. both feature maps and the depth volume
(magnet_cost_volume_bwd_f32; built only when grad mode is on and one of them requires grad, so that G-Net training,
where none does, runs exactly the no-grad path), the F volume w.r.t. both feature maps (magnet_cost_volume_f_bwd_f32)
for F-Net training.  Inside ``geometry_grad()`` both are differentiable in the cameras too (R, t, intM and the rays;
magnet_cost_volume_geom_bwd_f32).
"""
from __future__ import annotations

import contextlib
import threading
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
    then become part of the graph and replay with the data) and while torch.compile traces (the key reads data
    pointers, and a compiled graph replays its preparations with the data too), and ``clear_cache()`` /
    ``prep_cache(False)`` exist for callers that refill buffers behind torch's back.

    Entries are per stream: the key also holds the current stream of the device the preparation is made on (``device``,
    else the first CUDA source tensor's).  A preparation is enqueued and allocated on that stream, so only calls on the
    same stream may read it: they are ordered after its kernels, and once the entry is dropped the caching allocator
    hands its memory only to later work of that stream.  A call on another stream prepares again.  ``capacity`` counts
    per stream (one CW call holds four or five entries), so streams that alternate do not evict each other's entries.
    The dict is guarded by a lock, so host threads may share the cache; the preparations themselves run outside it."""

    def __init__(self, capacity: int = 8):
        self.capacity = capacity
        self.enabled = True
        self._items: Dict[Tuple, Tuple[tuple, object]] = {}
        self._lock = threading.Lock()

    @staticmethod
    def _key(kind, tensors, extra, device):
        if device is None:
            device = next((t.device for t in tensors if t.is_cuda), None)
        elif not isinstance(device, torch.device):
            device = torch.device(device)
        stream = None
        if device is not None and device.type == "cuda":
            # the raw handle: torch.cuda.current_stream builds a Stream object, several microseconds per lookup
            index = torch.cuda.current_device() if device.index is None else device.index
            stream = (index, torch._C._cuda_getCurrentRawStream(index))
        sig = tuple((t.data_ptr(), t._version, tuple(t.shape), tuple(t.stride()), str(t.device)) for t in tensors)
        return (kind, stream) + sig + tuple(extra)

    def _usable(self, tensors) -> bool:
        if not self.enabled or torch.compiler.is_compiling():
            return False
        if any(t.is_cuda for t in tensors) and torch.cuda.is_current_stream_capturing():
            return False
        return True

    def get(self, kind: str, tensors, extra=(), device=None):
        if not self._usable(tensors):
            return None
        key = self._key(kind, tensors, extra, device)
        with self._lock:
            hit = self._items.get(key)
            if hit is not None:
                refs, value = hit
                if all(r() is t for r, t in zip(refs, tensors)):
                    return value
                del self._items[key]
        return None

    def put(self, kind: str, tensors, value, extra=(), device=None):
        if not self._usable(tensors):
            return value
        key = self._key(kind, tensors, extra, device)
        refs = tuple(weakref.ref(t) for t in tensors)
        with self._lock:
            for dead in [k for k, (rs, _) in self._items.items() if any(r() is None for r in rs)]:
                del self._items[dead]                  # drop preparations whose source tensor is gone
            same = [k for k in self._items if k[1] == key[1]]
            if len(same) >= self.capacity:
                del self._items[same[0]]               # the stream's oldest entry (dicts keep insertion order)
            self._items[key] = (refs, value)
        return value

    def clear(self):
        with self._lock:
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
    hit = _cache.get("intr", (intM, rays), (str(device),), device)
    if hit is not None:
        return hit
    value = (intM.detach().to(device=device, dtype=torch.float32).contiguous(),
             rays.detach().to(device=device, dtype=torch.float32).contiguous())
    return _cache.put("intr", (intM, rays), value, (str(device),), device)


def _camera_table(cam_intrins, R, t, is_valid, device):
    """K*R, K*t per (b, v): 2 KB, one 3 us kernel.  Cached on the tensors R and t are views OF (MAGNET.py:147-148
    slices nghbr_poses once per forward) — both bases, with their version counters — plus the views' geometry."""
    intM_d, _ = _device_intrinsics(cam_intrins, device)
    if torch.compiler.is_compiling():                  # no cache while tracing, and its key reads data pointers
        return ops.pack_cameras(intM_d, R, t, is_valid.to(device=device, dtype=torch.int32))
    rbase = R._base if R._base is not None else R
    tbase = t._base if t._base is not None else t
    src = (rbase, tbase, is_valid, cam_intrins['intM'])
    extra = (R.data_ptr(), tuple(R.shape), tuple(R.stride()), t.data_ptr(), tuple(t.shape), tuple(t.stride()))
    hit = _cache.get("cams", src, extra, device)
    if hit is not None:
        return hit
    valid_d = is_valid.to(device=device, dtype=torch.int32)
    return _cache.put("cams", src, ops.pack_cameras(intM_d, R, t, valid_d), extra, device)


MMA_MIN_PLANES = 32   # below half a 64-hypothesis chunk the all-pairs GEMM is wasted: the gather kernel does only the needed taps


def _tensor_cores(C: int, V: int, variant: int, D: int) -> bool:
    return C == 64 and V <= 16 and (variant == _lib.VARIANT_MMA or (variant == _lib.VARIANT_AUTO and D >= MMA_MIN_PLANES))


def wants_half16(ref_dtype, src_dtype, C: int, V: int, variant: int, D: int) -> bool:
    """The half-precision part of ``route``: the single-plane HALF16 layout when the tensor-core kernel runs and both
    feature maps have the same half dtype; otherwise (False) both maps are upcast and the fp32 layouts apply."""
    return _tensor_cores(C, V, variant, D) and ref_dtype == src_dtype and ref_dtype in ops.HALF_DTYPES


def route(C: int, V: int, D: int, variant: int, depth_mode: int, ref_dtype, src_dtype,
          differentiable: bool = False) -> Tuple[int, int]:
    """(source layout, kernel variant) of one cost-volume forward of C channels, V views and D hypotheses: the one rule
    of ``est_costvolume_CW``, ``est_costvolume_F``, ``plane_sweep_f`` and ``MatchingPlan.cost``.

    The tensor-core kernel (C == 64, V <= 16, and variant MMA, or AUTO with at least MMA_MIN_PLANES hypotheses) reads
    HALF16 when both feature maps have the same half dtype, else SPLIT16; MMA is refused anywhere else.  Otherwise a
    differentiable CW forward takes NCHW with the DIRECT kernel (the backward reproduces the consistency masks of these
    two forwards only); a plain forward takes PIXC for the TMA-staged CUDA-core kernel (variant TMA, which is refused
    where PIXC does not fit, or AUTO outside the fused sampler), else TILED32 for the global-gather kernels, or NCHW
    when C is not a multiple of 4.  Every layout but HALF16 reads fp32 maps (half maps upcast once)."""
    if differentiable:
        if variant not in (_lib.VARIANT_AUTO, _lib.VARIANT_MMA, _lib.VARIANT_DIRECT):
            raise _lib.MagnetError("a differentiable CW volume runs on the tensor-core or the DIRECT kernel (variant AUTO, "
                                   f"MMA or DIRECT), got variant {variant}")
        if C > 64:
            raise _lib.MagnetError(f"the CW backward supports C <= 64 channels, got C={C}")
    if _tensor_cores(C, V, variant, D):
        return (_lib.SRC_HALF16 if wants_half16(ref_dtype, src_dtype, C, V, variant, D) else _lib.SRC_SPLIT16), variant
    if variant == _lib.VARIANT_MMA:
        raise _lib.MagnetError(f"MAGNET_VARIANT_MMA needs C == 64 and V <= 16, got C={C}, V={V}")
    if differentiable:
        return _lib.SRC_NCHW, _lib.VARIANT_DIRECT
    pixc = C in (16, 32, 64) and V <= 16
    if variant == _lib.VARIANT_TMA and not pixc:
        raise _lib.MagnetError(f"MAGNET_VARIANT_TMA needs C in (16, 32, 64) and V <= 16, got C={C}, V={V}")
    # AUTO: the fused sampler (DEPTH_GAUSS) stays on the global-gather kernel, which is faster than the TMA-staged one there
    if pixc and (variant == _lib.VARIANT_TMA or (variant == _lib.VARIANT_AUTO and depth_mode != _lib.DEPTH_GAUSS)):
        return _lib.SRC_PIXC, variant
    return (_lib.SRC_TILED32 if C % 4 == 0 else _lib.SRC_NCHW), variant


def differentiable_layout(C: int, V: int, D: int, variant: int, half: bool = False) -> int:
    """The source layout ``route`` gives a differentiable CW forward, for feature maps of one half dtype (``half``) or
    fp32: HALF16 / SPLIT16 on the tensor cores, else NCHW (read by the DIRECT kernel)."""
    dtype = torch.float16 if half else torch.float32
    return route(C, V, D, variant, _lib.DEPTH_VOLUME, dtype, dtype, differentiable=True)[0]


def repack_source(layout: int, nghbr_feat, nghbr_gmms=None, ref_feat=None):
    """(source maps in ``layout``, reference split or None): SPLIT16 / HALF16 (feature planes + Gaussian table, and with
    ``ref_feat`` the reference features' planes, which the tensor-core kernels read in place of ``ref_feat``), PIXC
    (features + Gaussians, pixel-major), TILED32 (features only) or the NCHW maps.  The maps are read as given: fp16 /
    bf16 for HALF16, fp32 for every other layout."""
    feat = nghbr_feat.detach()
    if layout == _lib.SRC_NCHW:
        return feat.contiguous(), None
    if layout == _lib.SRC_TILED32:
        return ops.repack_tiled32(feat), None
    fn = {_lib.SRC_PIXC: ops.repack_pixc, _lib.SRC_SPLIT16: ops.repack_split16, _lib.SRC_HALF16: ops.repack_half16}[layout]
    src = fn(feat, None if nghbr_gmms is None else nghbr_gmms.detach())
    return src, (fn(ref_feat.detach()) if ref_feat is not None and layout in ops.PACKED_LAYOUTS else None)


def _cached(kind, tensors, make):
    hit = _cache.get(kind, tensors)
    return hit if hit is not None else _cache.put(kind, tensors, make())


def _f32(x):
    """x as an fp32 tensor: x itself when it is fp32 (the same object, so that caches keyed on it still hit), else a
    detached upcast cached on x (once per forward)."""
    return x if x.dtype == torch.float32 else _cached("f32", (x,), lambda: x.detach().float())


_CACHE_KIND = {_lib.SRC_HALF16: "half16", _lib.SRC_SPLIT16: "split16", _lib.SRC_PIXC: "pixc", _lib.SRC_TILED32: "tiled32"}


def _packed_source(layout, nghbr_feat, nghbr_gmms, ref_feat):
    """``repack_source`` once per forward: the source maps and the reference split are each cached on the maps they are
    made from, so a change of the reference features alone repacks only them.  Returns (source, reference split)."""
    if layout != _lib.SRC_HALF16:
        nghbr_feat, ref_feat = _f32(nghbr_feat), _f32(ref_feat)
    if layout == _lib.SRC_NCHW:
        return repack_source(layout, nghbr_feat)
    gmms = None if nghbr_gmms is None or layout == _lib.SRC_TILED32 else _f32(nghbr_gmms)
    kind = _CACHE_KIND[layout]
    src = _cached(kind, (nghbr_feat,) if gmms is None else (nghbr_feat, gmms),
                  lambda: repack_source(layout, nghbr_feat, gmms)[0])
    if layout not in ops.PACKED_LAYOUTS:
        return src, None
    return src, _cached(kind + "ref", (ref_feat,), lambda: repack_source(layout, ref_feat)[0])


_geometry_grad = [False]


@contextlib.contextmanager
def geometry_grad(enabled: bool = True):
    """Inside the block, camera tensors that require grad (R / t, i.e. ``nghbr_poses``, ``intM``,
    ``unit_ray_array_2D``) get gradients from ``est_costvolume_CW``, ``est_costvolume_F``, ``plane_sweep_f`` (``MagnetF``)
    and ``MatchingPlan.cost``, as the reference's operators give them (DESIGN §3.11).  Off by default: outside the
    block the CW volume and ``MatchingPlan`` refuse such tensors.  A context manager, so that callers that cannot pass
    a keyword (``MAGNET.forward``, ``train_FNet.py``) run unchanged inside it."""
    prev = _geometry_grad[0]
    _geometry_grad[0] = bool(enabled)
    try:
        yield
    finally:
        _geometry_grad[0] = prev


def geometry_grad_enabled() -> bool:
    return _geometry_grad[0]


def camera_inputs(R, t, cam_intrins):
    """The caller's camera tensors, in the order the autograd Functions take them: R, t, intM, rays."""
    return R, t, cam_intrins['intM'], cam_intrins['unit_ray_array_2D']


def wants_camera_grad(cam_inputs) -> bool:
    """Camera gradients are computed only under geometry_grad() and when one of the camera tensors requires grad."""
    return geometry_grad_enabled() and wants_cw_grad(*cam_inputs)


def _detached(*xs):
    """The camera tensors as saved for backward: detached views, which share the version counter, so an in-place update
    of a pose between forward and backward raises as it does in autograd."""
    return tuple(None if x is None else x.detach() for x in xs)


def camera_grads(ctx, g_cams, g_rays, cam_inputs):
    """(grad_R, grad_t, grad_intM, grad_rays) from the kernel's (B*V,12) table and ray gradient, each in its input's
    dtype and on its input's device, None where not wanted (ctx.needs_input_grad of the last four inputs).
    cam_inputs: the saved (R, t, intM, rays)."""
    R, t, intM, rays = cam_inputs
    need = ctx.needs_input_grad[-4:]
    gR, gt, gK = ops.camera_chain(g_cams, intM.detach().to(g_cams.device), R.detach(), t.detach())
    out = [gR, gt, gK, None if g_rays is None else g_rays.reshape(rays.shape)]
    return tuple(None if not n or g is None else g.to(device=x.device, dtype=x.dtype)
                 for n, g, x in zip(need, out, cam_inputs))


def check_geometry_grad(**named) -> None:
    """Outside geometry_grad() the cost volume is differentiable in the feature maps and the depths only: raise instead
    of silently dropping the gradient of a camera tensor."""
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
    mask.  After a SPLIT16 / HALF16 forward the feature gradients run on the tensor cores on the same split buffers,
    otherwise on the CUDA cores; the depth gradient always on the CUDA cores.  The source Gaussians get no gradient (the
    mask is piecewise constant)."""

    @staticmethod
    def forward(ctx, depth, ref_feat, nghbr_feat, nghbr_gmms, run, spec, R=None, t=None, intM=None, rays=None):
        out, layout, variant, splits = run()
        ctx.save_for_backward(depth.detach(), ref_feat.detach(), nghbr_feat.detach(), nghbr_gmms.detach(),
                              *_detached(R, t, intM, rays))
        ctx.spec, ctx.fwd, ctx.splits = spec, (layout, variant), splits or (None, None)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        depth, ref_in, src_in, gmm, *cam_saved = ctx.saved_tensors
        rays, cams, V, kappa, karr = ctx.spec
        need_d, need_ref, need_src = ctx.needs_input_grad[:3]
        need_cam = any(ctx.needs_input_grad[6:])
        depth_src = dict(d_volume=depth if karr is None else None, ref_gmm=depth if karr is not None else None, k=karr)
        # the existing entry point computes the feature and depth gradients exactly as without camera gradients (the
        # camera kernel's own depth gradient can differ from it in the last bit, DESIGN §3.11); the camera entry point
        # adds the camera and ray gradients
        g_ref = g_src = g_d = None
        if need_ref or need_src or need_d:
            # the CUDA-core kernel reads fp32 NCHW maps: always after a non-HALF16 forward, for the depth gradient after one
            upcast = need_d or ctx.fwd[0] != _lib.SRC_HALF16
            ref, src = (ref_in.float(), src_in.float()) if upcast else (ref_in, src_in)
            g_ref, g_src, g_d = ops.cost_volume_bwd(
                ref, src, gmm.float(), rays, cams, grad_out.contiguous(), V=V, kappa=kappa, **depth_src,
                fwd_layout=ctx.fwd[0], fwd_variant=ctx.fwd[1], need_ref=need_ref, need_src=need_src,
                need_depth=need_d, ref_split=ctx.splits[0], src_split=ctx.splits[1])
            g_ref = None if g_ref is None else g_ref.to(ref_in.dtype)
            g_src = None if g_src is None else g_src.to(src_in.dtype)
        g_cam = (None,) * 4
        if need_cam:
            g_cams, g_rays, _ = ops.cost_volume_geom_bwd(
                ref_in.float(), src_in.float(), gmm.float(), rays, cams, grad_out.contiguous(), V=V, kappa=kappa,
                **depth_src, fwd_layout=ctx.fwd[0], fwd_variant=ctx.fwd[1], need_rays=ctx.needs_input_grad[9])
            g_cam = camera_grads(ctx, g_cams, g_rays, cam_saved)
        return (g_d, g_ref, g_src, None, None, None) + g_cam


def est_costvolume_CW(d_volume, ref_feat, nghbr_feat, ref_gmms, nghbr_gmms,
                      R, t, is_valid, cam_intrins, thres, variant=_lib.VARIANT_AUTO):
    """Consistency-weighted multi-view cost volume — drop-in for homography.est_costvolume_CW.

    d_volume (B,D,H,W); ref_feat (B,C,H,W); nghbr_feat (V*B,C,H,W) view-major; ref_gmms unused (as in
    the reference, SURVEY A.5 #7); nghbr_gmms (V*B,2,H,W) [mu, sigma]; R (B,V,3,3), t (B,V,3) device
    views; is_valid (B,V) int CPU or device; cam_intrins dict of 'intM' (B,3,3) and
    'unit_ray_array_2D' (B,3,H*W), CPU or device; thres int.  Returns (B,D,H,W) float32 on
    ref_feat.device, freshly allocated.  Differentiable, as the reference, in d_volume, ref_feat and nghbr_feat when
    grad mode is on and one of them requires grad; in R, t, intM and the rays too inside geometry_grad() (outside it the
    camera tensors must not require grad); detached otherwise.
    Any of the tensors may be fp16 / bf16 (torch.autocast): the volume is fp32, each gradient has its input's dtype."""
    device = ref_feat.device
    B = d_volume.shape[0]
    V = int(nghbr_feat.shape[0] / B)
    cam_in = camera_inputs(R, t, cam_intrins)
    if torch.is_grad_enabled() and not geometry_grad_enabled():
        check_geometry_grad(R=R, t=t, intM=cam_intrins['intM'], unit_ray_array_2D=cam_intrins['unit_ray_array_2D'])
    d_volume = d_volume.float()                            # differentiable upcast (a no-op for fp32)
    grad = wants_cw_grad(d_volume, ref_feat, nghbr_feat) or wants_camera_grad(cam_in)
    layout, fv = route(int(ref_feat.shape[1]), V, int(d_volume.shape[1]), variant, _lib.DEPTH_VOLUME, ref_feat.dtype,
                       nghbr_feat.dtype, differentiable=grad)
    _, rays_d = _device_intrinsics(cam_intrins, device)
    cams = _camera_table(cam_intrins, R, t, is_valid, device)

    def run():
        src, ref_split = _packed_source(layout, nghbr_feat, nghbr_gmms, ref_feat)
        ref = (ref_feat if layout == _lib.SRC_HALF16 else _f32(ref_feat)).detach()
        out = ops.cost_volume(ref, src, rays_d, cams, V=V, src_layout=layout, consistency=True,
                              src_gmm=_f32(nghbr_gmms).detach(), kappa=float(thres), d_volume=d_volume.detach(),
                              variant=fv, ref_split=ref_split)
        return out, layout, fv, (ref_split, src) if layout in ops.PACKED_LAYOUTS else None

    if grad:
        return _CostVolumeCW.apply(d_volume, ref_feat, nghbr_feat, nghbr_gmms, run,
                                   (rays_d, cams, V, float(thres), None), *cam_in)
    with torch.no_grad():
        return run()[0]


def _plane_list(d_center):
    """The D plane depths as host floats.  ``d_center`` is a constant of the training run (train_FNet.py:56-66): the
    device -> host read happens once per tensor, not once per step.  A sequence of floats is taken as it is; under
    torch.compile it is required (a tensor is refused rather than read in the compiled graph)."""
    if torch.compiler.is_compiling():
        return ops.k_array(d_center)                   # the list of floats; a tensor is refused
    if not isinstance(d_center, torch.Tensor):
        return [float(v) for v in d_center]
    return _cached("planes", (d_center,), lambda: d_center.detach().reshape(-1).cpu().tolist())


def _f_forward(ref_feat, nghbr_feat, planes, rays_d, cams, V, variant, softmax):
    """The F volume's forward: (volume, source layout, source maps, reference split)."""
    layout, fv = route(int(ref_feat.shape[1]), V, len(planes), variant, _lib.DEPTH_PLANES, ref_feat.dtype,
                       nghbr_feat.dtype)
    src, ref_split = _packed_source(layout, nghbr_feat, None, ref_feat)
    ref = (ref_feat if layout == _lib.SRC_HALF16 else _f32(ref_feat)).detach()
    out = ops.cost_volume(ref, src, rays_d, cams, V=V, src_layout=layout, consistency=False,
                          k=planes, planes=True, softmax=softmax, variant=fv, ref_split=ref_split)
    return out, layout, src, ref_split


class _CostVolumeF(torch.autograd.Function):
    """Plane-sweep volume (homography.py:10-75) — the probabilities (``softmax``) or the 1/V-averaged scores the fused
    F-Net loss reads — differentiable in both feature maps.  With ``tc_bwd`` the backward runs on the tensor cores
    after a SPLIT16 / HALF16 forward, on the forward's buffers; otherwise the CUDA-core kernel reads the fp32 NCHW
    maps."""

    @staticmethod
    def forward(ctx, ref_feat, nghbr_feat, planes, rays_d, cams, V, variant, softmax, tc_bwd,
                R=None, t=None, intM=None, rays=None):
        out, layout, src, ref_split = _f_forward(ref_feat, nghbr_feat, planes, rays_d, cams, V, variant, softmax)
        ctx.save_for_backward(ref_feat.detach(), nghbr_feat.detach(), out if softmax else None, rays_d, cams,
                              *_detached(R, t, intM, rays))
        ctx.layout = layout if tc_bwd else _lib.SRC_NCHW   # what the feature gradients read
        ctx.splits = (ref_split, src) if ctx.layout in ops.PACKED_LAYOUTS else (None, None)
        ctx.planes, ctx.V, ctx.softmax = planes, V, softmax
        return out

    @staticmethod
    def backward(ctx, grad_out):
        ref_feat, nghbr_feat, out, rays_d, cams, *cam_saved = ctx.saved_tensors
        need_cam = any(ctx.needs_input_grad[9:])
        g_ref = g_src = None
        if not need_cam or any(ctx.needs_input_grad[:2]):
            if ctx.layout == _lib.SRC_HALF16:              # the NCHW maps only supply the shapes
                ref, src = ref_feat, nghbr_feat
            else:
                ref, src = ref_feat.float(), nghbr_feat.float()
            g_ref, g_src = ops.cost_volume_f_bwd(ref, src, rays_d, cams, ctx.planes, ctx.V, out,
                                                 grad_out.contiguous(), softmax=ctx.softmax, ref_split=ctx.splits[0],
                                                 src_split=ctx.splits[1], split_layout=ctx.layout)
            g_ref, g_src = g_ref.to(ref_feat.dtype), g_src.to(nghbr_feat.dtype)
        g_cam = (None,) * 4
        if need_cam:
            g_cams, g_rays, _ = ops.cost_volume_geom_bwd(ref_feat.float(), nghbr_feat.float(), None, rays_d, cams,
                                                         grad_out.contiguous(), V=ctx.V, k=ctx.planes, planes=True,
                                                         softmax=ctx.softmax, prob=out,
                                                         need_rays=ctx.needs_input_grad[12])
            g_cam = camera_grads(ctx, g_cams, g_rays, cam_saved)
        return (g_ref, g_src) + (None,) * 7 + g_cam


def _f_volume(d_center, ref_feat, nghbr_feat, R, t, is_valid, cam_intrins, variant, softmax, tc_bwd):
    # the camera tensors take part only under geometry_grad(), where a d_center that requires grad is refused: the
    # planes are host constants
    cam_in = ()
    if geometry_grad_enabled():
        if torch.is_grad_enabled() and isinstance(d_center, torch.Tensor) and d_center.requires_grad:
            raise _lib.MagnetError("d_center requires grad, but the plane depths are constants of the F volume (detach it)")
        cam_in = camera_inputs(R, t, cam_intrins)
    device = ref_feat.device
    V = int(nghbr_feat.shape[0] / ref_feat.shape[0])
    planes = _plane_list(d_center)
    _, rays_d = _device_intrinsics(cam_intrins, device)
    cams = _camera_table(cam_intrins, R, t, is_valid, device)
    if torch.compiler.is_compiling() and not wants_cw_grad(ref_feat, nghbr_feat, *cam_in):
        return _f_forward(ref_feat, nghbr_feat, planes, rays_d, cams, V, variant, softmax)[0]   # traced inference
    if torch.compiler.is_compiling() and not cam_in:       # traced training: the op with a backward
        layout, fv = route(int(ref_feat.shape[1]), V, len(planes), variant, _lib.DEPTH_PLANES, ref_feat.dtype,
                           nghbr_feat.dtype)
        src, ref_split = _packed_source(layout, nghbr_feat, None, ref_feat)
        return ops._op("cost_volume_f")(ref_feat, nghbr_feat, src, ref_split, rays_d, cams, V, layout, fv, planes,
                                        softmax, tc_bwd)
    return _CostVolumeF.apply(ref_feat, nghbr_feat, planes, rays_d, cams, V, variant, softmax, tc_bwd, *cam_in)


def plane_sweep_f(d_center, ref_feat, nghbr_feat, R, t, is_valid, cam_intrins, softmax=True):
    """The F volume of est_costvolume_F (softmax=True) or its 1/V-averaged scores (softmax=False), with the
    tensor-core backward where the forward ran on the tensor cores (MagnetF's path; est_costvolume_F keeps the
    CUDA-core backward)."""
    return _f_volume(d_center, ref_feat, nghbr_feat, R, t, is_valid, cam_intrins, _lib.VARIANT_AUTO, softmax, True)


def est_costvolume_F(d_center, ref_feat, nghbr_feat, R, t, is_valid, cam_intrins, variant=_lib.VARIANT_AUTO):
    """Fronto-parallel plane-sweep volume with softmax over planes — drop-in (forward) for
    homography.est_costvolume_F.  d_center (1,D,1,1); the rest as in est_costvolume_CW."""
    return _f_volume(d_center, ref_feat, nghbr_feat, R, t, is_valid, cam_intrins, variant, True, False)
