"""Tensor-level wrappers over the C ABI (one Python call = one kernel launch) and the
``torch.autograd.Function`` wrappers the reference-facing modules use.

Everything here requires CUDA tensors and the built library; nothing falls back to PyTorch.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Optional, Sequence

import torch

from . import _lib
from ._lib import CostArgs, check, lib


def _stream(dev=None) -> int:
    """The current stream of the device the operands live on (not of whatever device happens to be current)."""
    return torch.cuda.current_stream(dev).cuda_stream


def _traced() -> bool:
    """Whether torch.compile is tracing the call.  A traced call goes through its registered op
    (``magnet_b200.library``), whose implementation is the eager call; an eager call goes to the C entry point directly,
    without the dispatcher (DESIGN §3.18)."""
    return torch.compiler.is_compiling()


def _op(name: str):
    return getattr(torch.ops.magnet_b200, name)


def _no_out_traced(out) -> None:
    if out is not None:
        raise _lib.MagnetError("out= writes into a caller buffer by address: under torch.compile the ops allocate "
                               "their outputs (pass out=None)")


def _launch(dev, name: str, *args) -> None:
    """Call the C entry point ``name`` with ``args`` and the current stream of ``dev``, with ``dev`` current; a
    failed status raises MagnetError."""
    with torch.cuda.device(dev):
        check(getattr(lib(), name)(*args, _stream(dev)), name)


def _same_device(*named):
    """All operands of one launch must live on one CUDA device; returns it."""
    dev = None
    for name, x in named:
        if x is None:
            continue
        if dev is None:
            dev = x.device
        elif x.device != dev:
            raise _lib.MagnetError(f"{name} is on {x.device}, expected {dev} (all operands of a launch share one device)")
    return dev


def _expect(name: str, x: torch.Tensor, shape) -> None:
    if tuple(x.shape) != tuple(shape):
        raise _lib.MagnetError(f"{name} must have shape {tuple(shape)}, got {tuple(x.shape)}")


def _need_cuda_f32(name: str, x: torch.Tensor, shape=None, contiguous: bool = True) -> torch.Tensor:
    """A CUDA float32 operand, of ``shape`` when given; made contiguous unless ``contiguous=False``."""
    x = _need_cuda(name, x)
    if x.dtype != torch.float32:
        raise _lib.MagnetError(f"{name} must be float32 (the reference path is fp32-only, homography.py:130)")
    if contiguous and not x.is_contiguous():
        x = x.contiguous()
    if shape is not None:
        _expect(name, x, shape)
    return x


def _need_preds(name: str, preds, shape=None) -> list:
    """Predictions ``name[i]`` (any iterable, consumed in order), each checked as ``_need_cuda_f32`` does."""
    return [_need_cuda_f32(f"{name}[{i}]", p, shape) for i, p in enumerate(preds)]


def _need_weights(named) -> list:
    """(name, weight, shape) triples -> the detached weights, each a CUDA float32 tensor of its shape."""
    return [_need_cuda_f32(nm, t.detach(), shp) for nm, t, shp in named]


def _need_cuda_u8_mask(name: str, m: torch.Tensor, shape, shape_text: str) -> torch.Tensor:
    """A CUDA uint8 mask of ``shape`` (``shape_text`` in the message), made contiguous."""
    if m.dtype != torch.uint8 or not m.is_cuda or tuple(m.shape) != tuple(shape):
        raise _lib.MagnetError(f"{name} must be a CUDA uint8 tensor of shape {shape_text}")
    return m.contiguous()


def _is_packed(buf, sizes=None) -> bool:
    """A packed buffer: a contiguous uint8 CUDA tensor, and, when ``sizes`` is given, of one of those byte counts."""
    return (isinstance(buf, torch.Tensor) and buf.is_cuda and buf.dtype == torch.uint8 and buf.is_contiguous()
            and (sizes is None or buf.numel() in sizes))


def _need_cuda(name: str, x: torch.Tensor) -> torch.Tensor:
    """An operand that only supplies a shape (any dtype, never read)."""
    if not isinstance(x, torch.Tensor):
        raise TypeError(f"{name} must be a torch.Tensor")
    if not x.is_cuda:
        raise _lib.MagnetError(f"{name} must be a CUDA tensor (magnet_b200 has no CPU path)")
    return x


# element types repack_half16 accepts
HALF_DTYPES = {torch.float16: _lib.DTYPE_F16, torch.bfloat16: _lib.DTYPE_BF16}
PACKED_LAYOUTS = (_lib.SRC_SPLIT16, _lib.SRC_HALF16)


def packed_bytes(layout: int, N: int, H: int, W: int) -> int:
    """Bytes of a SPLIT16 / HALF16 buffer of N images of H x W."""
    fn = lib().magnet_split16_bytes if layout == _lib.SRC_SPLIT16 else lib().magnet_half16_bytes
    return int(fn(N, H, W))


def _check_packed(name: str, buf, layout: int, N: int, H: int, W: int) -> None:
    """A SPLIT16 / HALF16 buffer of N images: uint8, contiguous, on the device, and exactly the layout's size (the
    kernels cannot tell the two kinds apart, so a buffer of the other kind is refused here, before any launch)."""
    what = "repack_split16" if layout == _lib.SRC_SPLIT16 else "repack_half16"
    if not _is_packed(buf):
        raise _lib.MagnetError(f"{name} must be a contiguous uint8 CUDA buffer from {what}")
    nbytes = packed_bytes(layout, N, H, W)
    if buf.numel() != nbytes:
        raise _lib.MagnetError(f"{name} must be a {what} buffer of {N} images of {H}x{W} ({nbytes} bytes), got "
                               f"{buf.numel()} bytes")


def k_array(k: Sequence[float]):
    """Python / numpy / tensor sequence -> host float[D] (rounded to fp32 like torch does for
    tensor * python-scalar, MAGNET.py:155).  While torch.compile traces: the list of Python floats the registered ops
    take instead (they round it the same way), and a tensor is refused, because reading it would put a device-to-host
    copy in the compiled graph."""
    if _traced():
        if isinstance(k, torch.Tensor):
            raise _lib.MagnetError("under torch.compile the hypotheses / plane depths must be a sequence of Python "
                                   "floats, not a tensor (read it to the host once, outside the compiled function)")
        return [float(v) for v in k]
    if isinstance(k, torch.Tensor):
        k = k.detach().cpu().flatten().tolist()
    vals = [float(v) for v in k]
    if len(vals) > _lib.MAGNET_MAX_PLANES:
        raise _lib.MagnetError(f"at most {_lib.MAGNET_MAX_PLANES} hypotheses per call, got {len(vals)}")
    return (C.c_float * len(vals))(*vals)


def pack_cameras(intM: torch.Tensor, R: torch.Tensor, t: torch.Tensor, is_valid: torch.Tensor) -> torch.Tensor:
    """(B,3,3) intrinsics, (B,V,3,3) / (B,V,3) pose views (any strides), (B,V) int32 validity — all on the
    device — -> (B*V, 16) float32 camera-constant table (struct magnet_camera)."""
    if _traced():
        return _op("pack_cameras")(intM, R, t, is_valid)
    intM = _need_cuda_f32("intM", intM)
    R = _need_cuda_f32("R", R, contiguous=False)
    t = _need_cuda_f32("t", t, contiguous=False)
    B, V = R.shape[0], R.shape[1]
    if is_valid.dtype != torch.int32 or not is_valid.is_cuda:
        is_valid = is_valid.to(device=intM.device, dtype=torch.int32)
    is_valid = is_valid.contiguous()
    cams = torch.empty(B * V, 16, device=intM.device, dtype=torch.float32)
    rs, ts = R.stride(), t.stride()
    dev = _same_device(("intM", intM), ("R", R), ("t", t), ("is_valid", is_valid))
    _launch(dev, "magnet_pack_cameras_f32", intM.data_ptr(), R.data_ptr(), rs[0], rs[1], rs[2], rs[3], t.data_ptr(),
            ts[0], ts[1], ts[2], is_valid.data_ptr(), B, V, cams.data_ptr())
    return cams


def _repack_operands(x: torch.Tensor, gmm: Optional[torch.Tensor], out: Optional[torch.Tensor], shape,
                     dtype=torch.uint8):
    """The operands of a repack of x (N,C,H,W) besides x: the optional Gaussians (N,2,H,W), checked, and the output,
    ``out`` if it holds a buffer of ``shape`` / ``dtype`` on x's device, else a new one.  Returns (gmm, out)."""
    N, _, H, W = x.shape
    if gmm is not None:
        gmm = _need_cuda_f32("gmm", gmm)
        if tuple(gmm.shape) != (N, 2, H, W):
            raise _lib.MagnetError(f"gmm must be (N,2,H,W) = {(N, 2, H, W)}, got {tuple(gmm.shape)}")
    if out is None:
        return gmm, torch.empty(shape, device=x.device, dtype=dtype)
    nbytes = math.prod(shape) * dtype.itemsize
    if out.numel() * out.element_size() < nbytes or out.device != x.device:
        raise _lib.MagnetError(f"out must hold {nbytes} bytes on {x.device}")
    return gmm, out


def _ptr(x: Optional[torch.Tensor]):
    return None if x is None else x.data_ptr()


def repack_tiled32(x: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """(N,C,H,W) -> TILED32 (N, H, ceil(W/32), C/4, 32, 4): the source-feature layout the tap-sharing
    kernel gathers from (channel quads of a pixel 512 B apart, 32 neighbouring pixels contiguous)."""
    if _traced():
        _no_out_traced(out)
        return _op("repack_tiled32")(x)
    x = _need_cuda_f32("x", x)
    N, Cc, H, W = x.shape
    if out is None:
        out = torch.empty(N, H, (W + 31) // 32, Cc // 4, 32, 4, device=x.device, dtype=torch.float32)
    _launch(x.device, "magnet_repack_tiled32_f32", x.data_ptr(), out.data_ptr(), N, Cc, H, W)
    return out


def repack_pixc(x: torch.Tensor, gmm: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """(N,C,H,W) features [+ (N,2,H,W) Gaussians] -> PIXC (N, H, W, C+4): pixel-major, per pixel the C channels then
    (mu, sigma, 0, 0) — the layout the TMA-staged CUDA-core kernel fetches its windows from.  C in {16, 32, 64}."""
    if _traced():
        _no_out_traced(out)
        return _op("repack_pixc")(x, gmm)
    x = _need_cuda_f32("x", x)
    N, Cc, H, W = x.shape
    gmm, out = _repack_operands(x, gmm, out, (N, H, W, Cc + 4), torch.float32)
    _launch(x.device, "magnet_repack_pixc_f32", x.data_ptr(), _ptr(gmm), out.data_ptr(), N, Cc, H, W)
    return out


def repack_split16(x: torch.Tensor, gmm: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """(N,64,H,W) features [+ (N,2,H,W) Gaussians] -> SPLIT16 buffer (uint8): header with the power-of-two scale s, fp16
    planes (N,2,H,W,64) with x*s = hi + lo, table (N,H,W,4) = (mu, sigma, 0, 0) — what the tensor-core kernel's TMA boxes
    fetch (reference features: gmm=None)."""
    if _traced():
        _no_out_traced(out)
        return _op("repack_split16")(x, gmm)
    x = _need_cuda_f32("x", x)
    N, Cc, H, W = x.shape
    gmm, out = _repack_operands(x, gmm, out, (int(lib().magnet_split16_bytes(N, H, W)),))
    _launch(x.device, "magnet_repack_split16_f32", x.data_ptr(), _ptr(gmm), out.data_ptr(), N, Cc, H, W)
    return out


def repack_half16(x: torch.Tensor, gmm: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """(N,64,H,W) fp16 / bf16 features [+ (N,2,H,W) fp32 Gaussians] -> HALF16 buffer (uint8): the header and table of
    ``repack_split16(x.float(), gmm)`` around ONE fp16 plane (N,1,H,W,64) = its hi plane (its lo plane is zero for
    every element above the threshold of DESIGN §3.7).  Read by the tensor-core kernels with ``src_layout=SRC_HALF16``."""
    if _traced():
        _no_out_traced(out)
        return _op("repack_half16")(x, gmm)
    x = _need_cuda("x", x)
    if x.dtype not in HALF_DTYPES:
        raise _lib.MagnetError(f"x must be float16 or bfloat16 (repack_split16 takes float32), got {x.dtype}")
    if x.dim() != 4:
        raise _lib.MagnetError(f"x must be (N,64,H,W), got {tuple(x.shape)}")
    x = x.contiguous()
    N, Cc, H, W = x.shape
    gmm, out = _repack_operands(x, gmm, out, (int(lib().magnet_half16_bytes(N, H, W)),))
    _same_device(("x", x), ("gmm", gmm))
    _launch(x.device, "magnet_repack_half16", x.data_ptr(), HALF_DTYPES[x.dtype], _ptr(gmm), out.data_ptr(), N, Cc, H, W)
    return out


def sample_depths(gmm: torch.Tensor, k, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Sampler alone (MAGNET.py:154-156): gmm (B,2,H,W) -> d_volume (B,D,H,W)."""
    if _traced():
        _no_out_traced(out)
        return _op("sample_depths")(gmm, k_array(k))
    gmm = _need_cuda_f32("gmm", gmm)
    karr = k if isinstance(k, C.Array) else k_array(k)
    B, _, H, W = gmm.shape
    D = len(karr)
    if out is None:
        out = torch.empty(B, D, H, W, device=gmm.device, dtype=torch.float32)
    _launch(gmm.device, "magnet_sample_depths_f32", gmm.data_ptr(), C.cast(karr, C.c_void_p), B, D, H * W,
            out.data_ptr())
    return out


def _cost_args(ref_feat: torch.Tensor, V: int, rays, cams, *, d_volume=None, ref_gmm=None, k=None, planes=False):
    """The CostArgs every cost-volume entry point shares, for ref_feat (B,C,H,W) and V views: ``rays`` and ``cams``
    checked against (B, V, H, W), the shape fields filled, and the depth source — ``d_volume`` (B,D,H,W), or
    ``ref_gmm`` (B,2,H,W) + ``k``, or ``k`` with ``planes=True``.  Returns (args, shape of the depth gradient or None
    for the constant planes, the checked operands by name for the device check).  The args keep the buffers they
    point into alive."""
    rays = _need_cuda_f32("rays", rays)
    cams = _need_cuda_f32("cams", cams)
    B, Cc, H, W = ref_feat.shape
    _expect("rays", rays, (B, 3, H * W))
    if cams.numel() != B * V * 16:
        raise _lib.MagnetError(f"cams must hold B*V = {B * V} camera records of 16 floats, got {tuple(cams.shape)}")
    a = CostArgs()
    a.B, a.V, a.C, a.H, a.W = B, V, Cc, H, W
    a.rays, a.cams = rays.data_ptr(), cams.data_ptr()
    karr = gd_shape = None
    if d_volume is not None:
        d_volume = _need_cuda_f32("d_volume", d_volume)
        if d_volume.dim() != 4 or d_volume.shape[0] != B or tuple(d_volume.shape[2:]) != (H, W):
            raise _lib.MagnetError(f"d_volume must be (B,D,H,W) = ({B},D,{H},{W}), got {tuple(d_volume.shape)}")
        a.depth_mode, a.D, a.d_volume = _lib.DEPTH_VOLUME, d_volume.shape[1], d_volume.data_ptr()
        gd_shape = tuple(d_volume.shape)
    else:
        karr = k if isinstance(k, C.Array) else k_array(k)
        a.D, a.k_host = len(karr), C.cast(karr, C.c_void_p)
        if planes:
            a.depth_mode = _lib.DEPTH_PLANES
        else:
            ref_gmm = _need_cuda_f32("ref_gmm", ref_gmm, (B, 2, H, W))
            a.depth_mode, a.ref_gmm = _lib.DEPTH_GAUSS, ref_gmm.data_ptr()
            gd_shape = (B, 2, H, W)
    a._keep = (rays, cams, d_volume, ref_gmm, karr)
    return a, gd_shape, (("rays", rays), ("cams", cams), ("d_volume", d_volume), ("ref_gmm", ref_gmm))


def check_src_index(src_index, B: int, V: int, n_src: int, *, check_range: bool = True) -> torch.Tensor:
    """The frame table of an indexed cost volume, checked: an int32 / int64 tensor of shape (B, V) whose entries all
    lie in [0, n_src), the views with is_valid == 0 included (fill those with any frame of the set).  A CUDA table is
    read back for the range check (one synchronisation; ``check_range=False`` skips it for a table checked before).
    Returns the table as contiguous int32 on its device."""
    if not isinstance(src_index, torch.Tensor):
        raise TypeError("src_index must be a torch.Tensor")
    if src_index.dtype not in (torch.int32, torch.int64):
        raise _lib.MagnetError(f"src_index must be an int32 or int64 tensor, got {src_index.dtype}")
    if tuple(src_index.shape) != (B, V):
        raise _lib.MagnetError(f"src_index must have shape (B, V) = {(B, V)}, got {tuple(src_index.shape)}")
    if n_src < 1:
        raise _lib.MagnetError(f"an indexed cost volume needs at least one source image, got n_src={n_src}")
    if check_range and src_index.numel():
        lo, hi = (int(v) for v in torch.aminmax(src_index))
        if lo < 0 or hi >= n_src:
            raise _lib.MagnetError(f"src_index entries must lie in [0, {n_src}) (the source images), got [{lo}, {hi}]")
    return src_index.to(torch.int32).contiguous()


# element types magnet_check_src_index reads
INDEX_DTYPES = {torch.int32: _lib.INDEX_I32, torch.int64: _lib.INDEX_I64}


def check_src_index_device(src_index: torch.Tensor, n_src: int):
    """The range check of a (B, V) int32 / int64 frame table on its device, without reading it back: one launch of
    magnet_check_src_index.  Returns (table, bad): the contiguous int32 (B, V) table with every entry outside
    [0, n_src) replaced by 0, which the indexed cost volume may read, and a (B,) int32 flag, nonzero for each row that
    held such an entry (views with is_valid == 0 count too, as in ``check_src_index``).  An int64 entry is compared in
    64 bits, so 2**31 is out of range rather than wrapped.  This is the check of the traced indexed path
    (DESIGN §3.18); eager calls check on the host and never launch it."""
    if _traced():
        return _op("check_src_index")(src_index, int(n_src))
    src_index = _need_cuda("src_index", src_index)
    if src_index.dtype not in INDEX_DTYPES:
        raise _lib.MagnetError(f"src_index must be an int32 or int64 tensor, got {src_index.dtype}")
    if src_index.dim() != 2:
        raise _lib.MagnetError(f"src_index must have shape (B, V), got {tuple(src_index.shape)}")
    if n_src < 1:
        raise _lib.MagnetError(f"an indexed cost volume needs at least one source image, got n_src={n_src}")
    src_index = src_index.contiguous()
    B, V = src_index.shape
    table = torch.empty((B, V), device=src_index.device, dtype=torch.int32)
    bad = torch.empty((B,), device=src_index.device, dtype=torch.int32)
    _launch(src_index.device, "magnet_check_src_index", src_index.data_ptr(), INDEX_DTYPES[src_index.dtype], B, V,
            int(n_src), table.data_ptr(), bad.data_ptr())
    return table, bad


def source_images(src_layout: int, src_feat, C: int, H: int, W: int) -> int:
    """Images in a source operand of ``src_layout`` for C channels at H x W: the leading dimension of an NCHW / TILED32 /
    PIXC tensor, or what the size of a SPLIT16 / HALF16 buffer holds (which must be a whole number of images)."""
    if src_layout in PACKED_LAYOUTS:
        if not isinstance(src_feat, torch.Tensor):
            raise TypeError("src_feat must be a torch.Tensor")
        one = packed_bytes(src_layout, 1, H, W)
        per = packed_bytes(src_layout, 2, H, W) - one
        n = (int(src_feat.numel()) - one) // per + 1      # int(): a symbolic size (a traced op's fake) is specialised
        _check_packed("src_feat", src_feat, src_layout, max(n, 1), H, W)
        return n
    shape = {_lib.SRC_NCHW: (C, H, W), _lib.SRC_TILED32: (H, (W + 31) // 32, C // 4, 32, 4),
             _lib.SRC_PIXC: (H, W, C + 4)}.get(src_layout)
    if shape is None:
        raise _lib.MagnetError(f"unknown src_layout {src_layout}")
    if src_feat.dim() != 1 + len(shape) or tuple(src_feat.shape[1:]) != shape or src_feat.shape[0] < 1:
        raise _lib.MagnetError(f"src_feat must have shape (n_src, *{shape}), got {tuple(src_feat.shape)}")
    return int(src_feat.shape[0])


def cost_volume(ref_feat: torch.Tensor, src_feat: torch.Tensor, rays: torch.Tensor, cams: torch.Tensor, *,
                V: int, src_layout: int, consistency: bool, src_gmm: Optional[torch.Tensor] = None,
                kappa: float = 5.0, d_volume: Optional[torch.Tensor] = None,
                ref_gmm: Optional[torch.Tensor] = None, k=None, planes: bool = False, softmax: bool = False,
                variant: int = _lib.VARIANT_AUTO, out: Optional[torch.Tensor] = None,
                ref_split: Optional[torch.Tensor] = None, src_index: Optional[torch.Tensor] = None,
                n_src: Optional[int] = None, check_index: bool = True) -> torch.Tensor:
    """One launch of magnet_cost_volume_f32.  Depth source: ``d_volume`` (drop-in), or ``ref_gmm`` + ``k``
    (fused sampler), or ``k`` with ``planes=True`` (fronto-parallel planes).  With ``src_layout=SRC_SPLIT16`` both
    ``src_feat`` and ``ref_split`` are ``repack_split16`` buffers (``ref_feat`` then only supplies the shape); with
    ``SRC_HALF16`` both are ``repack_half16`` buffers and ``ref_feat`` (any dtype) only supplies the shape.

    With ``src_index`` (B, V) (``check_src_index``) it is one launch of magnet_cost_volume_indexed_f32 instead:
    ``src_feat`` (and ``src_gmm``) then hold any number of source images, each packed once, and view (b, v) reads image
    ``src_index[b, v]``; ``n_src``, when given, must be the number of images they hold.  ``check_index=False`` skips the
    range check of the table (the caller has checked it).  None: the view-major operands of V*B images.
    Under torch.compile the view-major form is the registered op ``magnet_b200::cost_volume`` and the indexed form
    ``magnet_b200::cost_volume_indexed``, which checks the table on the device (``check_src_index_device``) whatever
    ``check_index`` says: a sample with an entry outside [0, n_src) gets a NaN volume instead of an exception, the
    others are unaffected (DESIGN §3.18).  A table on the CPU is copied to the device once, in the graph."""
    if _traced():
        _no_out_traced(out)
        args = (ref_feat, src_feat, rays, cams, int(V), int(src_layout), bool(consistency), src_gmm, float(kappa),
                d_volume, ref_gmm, None if k is None else k_array(k), bool(planes), bool(softmax), int(variant),
                ref_split)
        if src_index is None:
            return _op("cost_volume")(*args)
        return _op("cost_volume_indexed")(*args, src_index.to(ref_feat.device), None if n_src is None else int(n_src))
    ref_feat = _need_cuda("ref_feat", ref_feat) if src_layout == _lib.SRC_HALF16 else _need_cuda_f32("ref_feat", ref_feat)
    if src_layout not in PACKED_LAYOUTS:                   # the packed buffers are checked below, by their size
        src_feat = _need_cuda_f32("src_feat", src_feat)
    if ref_feat.dim() != 4:
        raise _lib.MagnetError(f"ref_feat must be (B,C,H,W), got {tuple(ref_feat.shape)}")
    B, Cc, H, W = ref_feat.shape
    if V <= 0:
        raise _lib.MagnetError(f"V must be positive, got {V}")
    n_img = V * B
    if src_index is not None:
        n_img = source_images(src_layout, src_feat, Cc, H, W)
        if n_src is not None and n_src != n_img:
            raise _lib.MagnetError(f"n_src={n_src} does not match src_feat, which holds {n_img} source images")
        src_index = check_src_index(src_index, B, V, n_img, check_range=check_index)
    # every operand against (B, V, D, C, H, W): a mismatch would read out of bounds, the reference raises instead
    src_shape = {_lib.SRC_NCHW: (n_img, Cc, H, W), _lib.SRC_TILED32: (n_img, H, (W + 31) // 32, Cc // 4, 32, 4),
                 _lib.SRC_PIXC: (n_img, H, W, Cc + 4)}.get(src_layout)
    if src_layout in PACKED_LAYOUTS:
        _check_packed("src_feat", src_feat, src_layout, n_img, H, W)
        _check_packed("ref_split", ref_split, src_layout, B, H, W)
    elif src_shape is None:
        raise _lib.MagnetError(f"unknown src_layout {src_layout}")
    else:
        _expect("src_feat", src_feat, src_shape)
    a, _, named = _cost_args(ref_feat, V, rays, cams, d_volume=d_volume, ref_gmm=ref_gmm, k=k, planes=planes)
    dev = _same_device(("ref_feat", ref_feat), ("src_feat", src_feat), ("src_gmm", src_gmm), *named, ("out", out),
                       ("ref_split", ref_split), ("src_index", src_index))
    a.src_layout = src_layout
    a.consistency = 1 if consistency else 0
    a.softmax = 1 if softmax else 0
    a.variant = variant
    a.kappa = float(kappa)
    a.ref_feat = ref_split.data_ptr() if src_layout in PACKED_LAYOUTS else ref_feat.data_ptr()
    a.src_feat = src_feat.data_ptr()
    if consistency and src_layout not in (_lib.SRC_PIXC, *PACKED_LAYOUTS):   # those carry the source Gaussians inside src_feat
        src_gmm = _need_cuda_f32("src_gmm", src_gmm, (n_img, 2, H, W))
        a.src_gmm = src_gmm.data_ptr()
    if out is None:
        out = torch.empty(B, a.D, H, W, device=ref_feat.device, dtype=torch.float32)
    else:
        out = _need_cuda_f32("out", out, (B, a.D, H, W))
    a.out = out.data_ptr()
    if src_index is None:
        _launch(dev, "magnet_cost_volume_f32", C.byref(a))
    else:
        _launch(dev, "magnet_cost_volume_indexed_f32", C.byref(a), src_index.data_ptr(), n_img)
    return out


def cost_volume_f_bwd(ref_feat, src_feat_nchw, rays, cams, planes, V, prob, grad_out, softmax=True,
                      ref_split=None, src_split=None, split_layout=_lib.SRC_SPLIT16):
    """Gradients of the plane-sweep volume w.r.t. (ref_feat, src_feat) — one magnet_cost_volume_f_bwd_f32 call.
    src_feat_nchw (V*B,C,H,W) view-major; prob = forward output (read only when ``softmax``); grad_out = gradient w.r.t.
    the forward output (the probabilities, or the 1/V-averaged scores with ``softmax=False``).  Returns (grad_ref,
    grad_src) in NCHW.  With ``ref_split`` / ``src_split`` — the repack_split16 buffers the forward read (C == 64,
    V <= 16) — the tensor-core kernel computes both gradients and the NCHW maps only supply the shapes; without them
    the CUDA-core kernel reads the NCHW maps (C in {8, 16, 32, 64}).  ``split_layout=SRC_HALF16``: the buffers are
    repack_half16 buffers, and the NCHW maps (any dtype) only supply the shapes.  The gradients are float32."""
    split = ref_split is not None or src_split is not None
    if split and split_layout not in PACKED_LAYOUTS:
        raise _lib.MagnetError(f"split_layout must be SRC_SPLIT16 or SRC_HALF16, got {split_layout}")
    shape_only = split and split_layout == _lib.SRC_HALF16
    ref_feat = _need_cuda("ref_feat", ref_feat) if shape_only else _need_cuda_f32("ref_feat", ref_feat)
    src = _need_cuda("src_feat", src_feat_nchw) if shape_only else _need_cuda_f32("src_feat", src_feat_nchw)
    grad_out = _need_cuda_f32("grad_out", grad_out)
    B, Cc, H, W = ref_feat.shape
    _expect("src_feat", src, (V * B, Cc, H, W))
    a, _, named = _cost_args(ref_feat, V, rays, cams, k=planes, planes=True)
    _expect("grad_out", grad_out, (B, a.D, H, W))
    if softmax:
        prob = _need_cuda_f32("prob", prob, (B, a.D, H, W))
    if split:
        for nm, buf, n in (("src_split", src_split, V * B), ("ref_split", ref_split, B)):
            _check_packed(nm, buf, split_layout, n, H, W)
    dev = _same_device(("ref_feat", ref_feat), ("src_feat", src), *named, ("prob", prob if softmax else None),
                       ("grad_out", grad_out), ("ref_split", ref_split), ("src_split", src_split))
    a.consistency, a.softmax = 0, 1 if softmax else 0
    a.src_layout = split_layout if split else _lib.SRC_NCHW
    a.ref_feat, a.src_feat = (ref_split.data_ptr(), src_split.data_ptr()) if split else (ref_feat.data_ptr(), src.data_ptr())
    work = torch.empty_like(grad_out)
    g_ref = torch.empty(ref_feat.shape, device=ref_feat.device, dtype=torch.float32)
    g_src = torch.zeros(src.shape, device=src.device, dtype=torch.float32)
    bw = _lib.CostFBwdArgs()
    bw.fwd = C.pointer(a)
    bw.prob = prob.data_ptr() if softmax else None
    bw.grad_out, bw.workspace = grad_out.data_ptr(), work.data_ptr()
    bw.grad_ref, bw.grad_src = g_ref.data_ptr(), g_src.data_ptr()
    _launch(dev, "magnet_cost_volume_f_bwd_f32", C.byref(bw))
    return g_ref, g_src


def cost_volume_bwd(ref_feat, src_feat, src_gmm, rays, cams, grad_out, *, V: int, kappa: float, consistency=True,
                    d_volume=None, ref_gmm=None, k=None, fwd_layout=_lib.SRC_NCHW, fwd_variant=_lib.VARIANT_DIRECT,
                    need_ref=True, need_src=True, need_depth=True, ref_split=None, src_split=None):
    """Gradients of the cost volume with per-pixel depths — one magnet_cost_volume_bwd_f32 call.
    ref_feat (B,C,H,W), src_feat (V*B,C,H,W) view-major and src_gmm (V*B,2,H,W) are NCHW; the depth source is
    ``d_volume`` (B,D,H,W) or ``ref_gmm`` (B,2,H,W) + ``k``, as in the forward.  ``fwd_layout`` / ``fwd_variant`` name
    the forward kernel (SRC_SPLIT16 with AUTO / MMA: tensor cores; VARIANT_DIRECT): its consistency mask is applied.
    After a SPLIT16 forward, ``ref_split`` / ``src_split`` are the repack_split16 buffers it read: both feature gradients
    then come from the tensor-core kernel on them (the NCHW maps serve the depth gradient only); without them the
    CUDA-core kernel computes every gradient with the tensor-core forward's mask (the cross-check).  After a HALF16
    forward (``fwd_layout=SRC_HALF16``) the buffers are repack_half16 buffers, and without ``need_depth`` the NCHW maps
    (any dtype) only supply the shapes; the depth gradient reads them, so they must then be float32.
    Returns (grad_ref, grad_src, grad_depth), each None when not requested; grad_depth is (B,D,H,W) w.r.t. d_volume or
    (B,2,H,W) w.r.t. ref_gmm.  The gradients are float32."""
    shape_only = fwd_layout == _lib.SRC_HALF16 and not need_depth and (ref_split is not None or src_split is not None)
    ref_feat = _need_cuda("ref_feat", ref_feat) if shape_only else _need_cuda_f32("ref_feat", ref_feat)
    src = _need_cuda("src_feat", src_feat) if shape_only else _need_cuda_f32("src_feat", src_feat)
    grad_out = _need_cuda_f32("grad_out", grad_out)
    B, Cc, H, W = ref_feat.shape
    _expect("src_feat", src, (V * B, Cc, H, W))
    a, gd_shape, named = _cost_args(ref_feat, V, rays, cams, d_volume=d_volume, ref_gmm=ref_gmm, k=k)
    a.src_layout, a.variant, a.consistency, a.softmax, a.kappa = fwd_layout, fwd_variant, 1 if consistency else 0, 0, float(kappa)
    _expect("grad_out", grad_out, (B, a.D, H, W))
    if fwd_layout in PACKED_LAYOUTS and (ref_split is not None or src_split is not None):
        for nm, buf, nimg in (("src_split", src_split, V * B), ("ref_split", ref_split, B)):
            _check_packed(nm, buf, fwd_layout, nimg, H, W)
        a.ref_feat, a.src_feat = ref_split.data_ptr(), src_split.data_ptr()
    bw = _lib.CostBwdArgs()
    bw.fwd = C.pointer(a)
    if not shape_only:                             # the NCHW maps are read (CUDA-core kernel)
        bw.ref_feat, bw.src_feat = ref_feat.data_ptr(), src.data_ptr()
    if consistency:
        src_gmm = _need_cuda_f32("src_gmm", src_gmm, (V * B, 2, H, W))
        bw.src_gmm = src_gmm.data_ptr()
    dev = _same_device(("ref_feat", ref_feat), ("src_feat", src), ("src_gmm", src_gmm if consistency else None),
                       *named, ("grad_out", grad_out), ("ref_split", ref_split), ("src_split", src_split))
    work = torch.empty_like(grad_out)
    g_ref = torch.empty(ref_feat.shape, device=dev, dtype=torch.float32) if need_ref else None
    g_src = torch.zeros(src.shape, device=dev, dtype=torch.float32) if need_src else None
    g_d = torch.empty(gd_shape, device=dev, dtype=torch.float32) if need_depth else None
    bw.grad_out, bw.workspace = grad_out.data_ptr(), work.data_ptr()
    bw.grad_ref, bw.grad_src, bw.grad_depth = _ptr(g_ref), _ptr(g_src), _ptr(g_d)
    _launch(dev, "magnet_cost_volume_bwd_f32", C.byref(bw))
    return g_ref, g_src, g_d


def geom_workspace_bytes(B: int, V: int, H: int, W: int) -> int:
    """Bytes of the workspace of cost_volume_geom_bwd (per-block partials of the camera gradients)."""
    return int(lib().magnet_cost_geom_workspace_bytes(B, V, H, W))


def cost_volume_geom_bwd(ref_feat, src_feat, src_gmm, rays, cams, grad_out, *, V: int, kappa: float = 0.0,
                         consistency=True, d_volume=None, ref_gmm=None, k=None, planes=False, softmax=False, prob=None,
                         fwd_layout=_lib.SRC_NCHW, fwd_variant=_lib.VARIANT_DIRECT, need_rays=True, need_depth=False):
    """Camera gradients of either cost volume — one magnet_cost_volume_geom_bwd_f32 call.  ref_feat (B,C,H,W) and
    src_feat (V*B,C,H,W) are the NCHW fp32 maps; the depth source is ``d_volume``, ``ref_gmm`` + ``k``, or ``k`` with
    ``planes=True`` (the F volume: no consistency, ``softmax`` with the forward output ``prob``).  ``fwd_layout`` /
    ``fwd_variant`` name the CW forward kernel, whose mask is applied.  Returns (grad_cams (B*V,12): d/d(K R) row-major
    then d/d(K t); grad_rays (B,3,H*W) or None; grad_depth or None), float32."""
    ref_feat = _need_cuda_f32("ref_feat", ref_feat)
    src = _need_cuda_f32("src_feat", src_feat)
    grad_out = _need_cuda_f32("grad_out", grad_out)
    B, Cc, H, W = ref_feat.shape
    _expect("src_feat", src, (V * B, Cc, H, W))
    a, gd_shape, named = _cost_args(ref_feat, V, rays, cams, d_volume=d_volume, ref_gmm=ref_gmm, k=k, planes=planes)
    a.src_layout, a.variant, a.kappa = fwd_layout, fwd_variant, float(kappa)
    a.consistency, a.softmax = 1 if consistency and not planes else 0, 1 if softmax else 0
    if need_depth and gd_shape is None:
        raise _lib.MagnetError("the plane depths of the F volume are constants: no depth gradient")
    _expect("grad_out", grad_out, (B, a.D, H, W))
    bw = _lib.CostGeomBwdArgs()
    bw.fwd = C.pointer(a)
    bw.ref_feat, bw.src_feat = ref_feat.data_ptr(), src.data_ptr()
    if a.consistency:
        src_gmm = _need_cuda_f32("src_gmm", src_gmm, (V * B, 2, H, W))
        bw.src_gmm = src_gmm.data_ptr()
    if softmax:
        prob = _need_cuda_f32("prob", prob, (B, a.D, H, W))
        bw.prob = prob.data_ptr()
    dev = _same_device(("ref_feat", ref_feat), ("src_feat", src), ("src_gmm", src_gmm if a.consistency else None),
                       *named, ("grad_out", grad_out), ("prob", prob if softmax else None))
    score = torch.empty_like(grad_out)
    work = torch.empty(geom_workspace_bytes(B, V, H, W), device=dev, dtype=torch.uint8)
    g_cams = torch.empty(B * V, 12, device=dev, dtype=torch.float32)
    g_rays = torch.empty(B, 3, H * W, device=dev, dtype=torch.float32) if need_rays else None
    g_d = torch.empty(gd_shape, device=dev, dtype=torch.float32) if need_depth else None
    bw.score, bw.workspace, bw.grad_out, bw.grad_cams = score.data_ptr(), work.data_ptr(), grad_out.data_ptr(), g_cams.data_ptr()
    bw.grad_rays, bw.grad_depth = _ptr(g_rays), _ptr(g_d)
    _launch(dev, "magnet_cost_volume_geom_bwd_f32", C.byref(bw))
    return g_cams, g_rays, g_d


def camera_chain(grad_cams, intM, R, t):
    """d/dA and d/da of the camera table (grad_cams (B*V,12), A = K R, a = K t) -> (grad_R (B,V,3,3), grad_t (B,V,3),
    grad_K (B,3,3)) by the chain rule of the reference's grouping (K R) Ray and K t: grad_R = K^T grad_A, grad_t =
    K^T grad_a, grad_K = sum_v (grad_A R^T + grad_a t^T).  Small batched matmuls in the dtype of grad_cams."""
    B, V = R.shape[:2]
    g = grad_cams.reshape(B, V, 12)
    gA, ga = g[..., :9].reshape(B, V, 3, 3), g[..., 9:]
    K = intM.to(g).unsqueeze(1)
    R, t = R.to(g), t.to(g)
    grad_R = K.transpose(-1, -2) @ gA
    grad_t = (K.transpose(-1, -2) @ ga.unsqueeze(-1)).squeeze(-1)
    grad_K = (gA @ R.transpose(-1, -2) + ga.unsqueeze(-1) * t.unsqueeze(-2)).sum(1)
    return grad_R, grad_t, grad_K


def cost_launch_info(B, V, D, Cc, H, W, variant=_lib.VARIANT_AUTO, device=None):
    """(grid CTAs, threads per CTA, dynamic smem bytes) the cost kernel would use for these sizes on ``device`` (a CUDA
    device; None: the current one).  The persistent kernels size their grid by that device's SM count."""
    if device is not None:
        with torch.cuda.device(device):
            return cost_launch_info(B, V, D, Cc, H, W, variant)
    a = CostArgs()
    a.B, a.V, a.D, a.C, a.H, a.W = B, V, D, Cc, H, W
    layout = {_lib.VARIANT_TMA: _lib.SRC_PIXC, _lib.VARIANT_MMA: _lib.SRC_SPLIT16}.get(variant, _lib.SRC_TILED32)
    a.depth_mode, a.src_layout, a.consistency, a.variant = _lib.DEPTH_PLANES, layout, 0, variant
    one = C.c_void_p(0x1000)                       # never dereferenced: validated for non-NULL / alignment only
    a.ref_feat = a.src_feat = a.rays = a.cams = a.out = a.k_host = one
    g, b, s = C.c_int(), C.c_int(), C.c_int()
    check(lib().magnet_cost_launch_info(C.byref(a), C.byref(g), C.byref(b), C.byref(s)), "magnet_cost_launch_info")
    return g.value, b.value, s.value


class GaussianUpdate(torch.autograd.Function):
    """mu' = mu0 + mu1*sigma0 ; sigma' = (elu(sigma1) + 1 + 1e-10)*sigma0  (MAGNET.py:60,65-69).
    Differentiable w.r.t. the G-Net output only; ``ref_gmm`` is detached in the reference (MAGNET.py:168)."""

    @staticmethod
    def forward(ctx, d_output: torch.Tensor, ref_gmm: torch.Tensor) -> torch.Tensor:
        d_output = _need_cuda_f32("d_output", d_output)
        ref_gmm = _need_cuda_f32("ref_gmm", ref_gmm.detach())
        B, _, H, W = d_output.shape
        _expect("ref_gmm", ref_gmm, d_output.shape)     # after the unpack, which refuses a d_output of another rank
        out = torch.empty_like(d_output)
        dev = _same_device(("d_output", d_output), ("ref_gmm", ref_gmm))
        _launch(dev, "magnet_gaussian_update_fwd_f32", d_output.data_ptr(), ref_gmm.data_ptr(), B, H * W, out.data_ptr())
        ctx.save_for_backward(d_output, ref_gmm)
        return out

    @staticmethod
    def backward(ctx, grad_out: torch.Tensor):
        d_output, ref_gmm = ctx.saved_tensors
        return gaussian_update_bwd(grad_out, d_output, ref_gmm), None


def gaussian_update_bwd(grad_out, d_output, ref_gmm) -> torch.Tensor:
    """The gradient of ``gaussian_update`` w.r.t. d_output: one magnet_gaussian_update_bwd_f32 launch."""
    grad_out = _need_cuda_f32("grad_out", grad_out)
    d_output, ref_gmm = _need_cuda_f32("d_output", d_output), _need_cuda_f32("ref_gmm", ref_gmm)
    B, _, H, W = d_output.shape
    gin = torch.empty_like(d_output)
    _launch(d_output.device, "magnet_gaussian_update_bwd_f32", grad_out.data_ptr(), d_output.data_ptr(),
            ref_gmm.data_ptr(), B, H * W, gin.data_ptr())
    return gin


def gaussian_update(d_output: torch.Tensor, ref_gmm: torch.Tensor) -> torch.Tensor:
    if _traced():                                  # the op has a backward (magnet_b200.library)
        return _op("gaussian_update")(d_output, ref_gmm.detach())
    return GaussianUpdate.apply(d_output, ref_gmm)


def gnet_weights_bytes(D: int) -> int:
    """Bytes of the packed G-Net weights for D cost channels (0 outside 1..MAGNET_MAX_PLANES)."""
    return int(lib().magnet_gnet_weights_bytes(int(D)))


def _check_cost_channels(D: int) -> None:
    if not 1 <= D <= _lib.MAGNET_MAX_PLANES:
        raise _lib.MagnetError(f"the fused G-Net head takes 1 to {_lib.MAGNET_MAX_PLANES} cost channels, got {D}")


def _gnet_convs(gnet, D: int):
    convs = gnet_head_layers(gnet, D)
    if convs is None:
        raise _lib.MagnetError(f"not a G-Net head with the reference's structure and at least {D} cost channels")
    return convs


def pack_gnet_weights(gnet, D: int) -> torch.Tensor:
    """The weights of a ``GNET`` (or its ``gnet`` Sequential) in the fused head's layout, for D cost channels: the
    cost slice W0[:, :D] of the first convolution, the two 128x128 layers and the 128->2 layer, split into fp16 hi/lo
    with one power-of-two scale per layer.  The head must have the structure ``gnet_head_layers`` recognises.  Read
    from the module at each call (nothing is cached).  Two launches."""
    c0, c1, c2, c3 = _gnet_convs(gnet, D)
    _check_cost_channels(D)
    ws = [t.detach() for t in (c0.weight[:, :D], c1.weight, c1.bias, c2.weight, c2.bias, c3.weight, c3.bias)]
    if _traced():
        return _op("pack_gnet_weights")(ws, int(D))
    return _pack_gnet(ws, D)


def _pack_gnet(ws, D: int) -> torch.Tensor:
    """``pack_gnet_weights`` of the detached tensors W0[:, :D], W1, b1, W2, b2, W3, b3."""
    nbytes = gnet_weights_bytes(D)
    ts = [_need_cuda_f32(nm, t) for nm, t in zip(("W0", "W1", "b1", "W2", "b2", "W3", "b3"), ws)]
    dev = _same_device(*((f"weight {i}", t) for i, t in enumerate(ts)))
    out = torch.empty(nbytes, device=dev, dtype=torch.uint8)
    _launch(dev, "magnet_gnet_pack_weights_f32", *(t.data_ptr() for t in ts), int(D), out.data_ptr())
    return out


def gnet_update(cost: torch.Tensor, invariant: torch.Tensor, packed: torch.Tensor, prev_gmm: torch.Tensor,
                out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """One inference iteration of the G-Net head and the Gaussian update in one fused kernel: cost (B,D,H,W),
    invariant (B,128,H,W) = ``GNET.invariant_part(x_d3, D)``, packed = ``pack_gnet_weights(g_net, D)``, prev_gmm
    (B,2,H,W) -> the updated (B,2,H,W) Gaussian.  Not differentiable (forward only)."""
    if _traced():
        _no_out_traced(out)
        return _op("gnet_update")(cost, invariant, packed, prev_gmm)
    cost = _need_cuda_f32("cost", cost)
    if cost.dim() != 4:
        raise _lib.MagnetError(f"cost must be (B,D,H,W), got {tuple(cost.shape)}")
    B, D, H, W = cost.shape
    invariant = _need_cuda_f32("invariant", invariant, (B, _lib.MAGNET_HIDDEN_CHANNELS, H, W))
    prev_gmm = _need_cuda_f32("prev_gmm", prev_gmm, (B, 2, H, W))
    _check_cost_channels(D)
    nbytes = gnet_weights_bytes(D)
    if not _is_packed(packed, (nbytes,)):
        raise _lib.MagnetError(f"packed must be a pack_gnet_weights buffer for D = {D} ({nbytes} bytes)")
    if out is None:
        out = torch.empty(B, 2, H, W, device=cost.device, dtype=torch.float32)
    else:
        out = _need_cuda_f32("out", out, (B, 2, H, W))
    dev = _same_device(("cost", cost), ("invariant", invariant), ("packed", packed), ("prev_gmm", prev_gmm), ("out", out))
    scratch = torch.empty(_lib.MAGNET_GNET_SCRATCH_BYTES // 4, device=dev, dtype=torch.int32)
    a = _lib.GnetArgs(B=B, D=D, H=H, W=W, cost=cost.data_ptr(), invariant=invariant.data_ptr(),
                      packed_weights=packed.data_ptr(), prev_gmm=prev_gmm.data_ptr(), scratch=scratch.data_ptr(),
                      out=out.data_ptr())
    _launch(dev, "magnet_gnet_update_f32", C.byref(a))
    return out


class GnetHeadTrain(torch.autograd.Function):
    """One iteration of the G-Net head and the Gaussian update, differentiable in the head's weights, the invariant and
    prev_gmm (DESIGN §3.10): the inference kernel's arithmetic plus stores of the hidden maps, and a backward of one
    tensor-core chain kernel and fixed-order weight-gradient GEMMs.  No gradient into the cost volume.  The weights are
    packed at every call (nothing is cached: they change at every optimizer step)."""

    @staticmethod
    def forward(ctx, cost, invariant, w0, w1, b1, w2, b2, w3, b3, prev_gmm):
        out, packed, saved, cost, prev_gmm = gnet_train_fwd(cost, invariant, (w0, w1, b1, w2, b2, w3, b3), prev_gmm)
        ctx.save_for_backward(cost, prev_gmm, packed, saved)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        cost, prev_gmm, packed, saved = ctx.saved_tensors
        need = ctx.needs_input_grad
        g_inv, *g, g_prev = gnet_bwd(grad_out, cost, prev_gmm, packed, saved, need[2:10])
        return (None, g_inv if need[1] else None, *g, g_prev)


def gnet_weight_shapes(D: int):
    """(name, shape) of the fused head's trained tensors W0[:, :D], W1, b1, W2, b2, W3, b3."""
    hid = _lib.MAGNET_HIDDEN_CHANNELS
    return (("W0", (hid, D, 3, 3)), ("W1", (hid, hid, 1, 1)), ("b1", (hid,)), ("W2", (hid, hid, 1, 1)), ("b2", (hid,)),
            ("W3", (2, hid, 1, 1)), ("b3", (2,)))


def gnet_train_fwd(cost, invariant, weights, prev_gmm):
    """The forward of ``GnetHeadTrain``: the weights W0[:, :D], W1, b1, W2, b2, W3, b3 packed for training, then the
    training forward (two launches).  Returns (out (B,2,H,W), packed weights, saved hidden maps, and the checked cost
    and prev_gmm the backward reads)."""
    cost = _need_cuda_f32("cost", cost.detach())
    if cost.dim() != 4:
        raise _lib.MagnetError(f"cost must be (B,D,H,W), got {tuple(cost.shape)}")
    B, D, H, W = cost.shape
    invariant = _need_cuda_f32("invariant", invariant.detach(), (B, _lib.MAGNET_HIDDEN_CHANNELS, H, W))
    prev_gmm = _need_cuda_f32("prev_gmm", prev_gmm.detach(), (B, 2, H, W))
    _check_cost_channels(D)
    nbytes = int(lib().magnet_gnet_train_weights_bytes(D))
    shapes = gnet_weight_shapes(D)
    ws = _need_weights([(nm, t, shp) for (nm, shp), t in zip(shapes, weights)])
    dev = _same_device(("cost", cost), ("invariant", invariant), ("prev_gmm", prev_gmm),
                       *((nm, t) for (nm, _), t in zip(shapes, ws)))
    packed = torch.empty(nbytes, device=dev, dtype=torch.uint8)
    saved = torch.empty(int(lib().magnet_gnet_saved_bytes(B, H, W)) // 4, device=dev, dtype=torch.float32)
    out = torch.empty(B, 2, H, W, device=dev, dtype=torch.float32)
    scratch = torch.empty(_lib.MAGNET_GNET_SCRATCH_BYTES // 4, device=dev, dtype=torch.int32)
    a = _lib.GnetTrainArgs(B=B, D=D, H=H, W=W, cost=cost.data_ptr(), invariant=invariant.data_ptr(),
                           packed_weights=packed.data_ptr(), prev_gmm=prev_gmm.data_ptr(), scratch=scratch.data_ptr(),
                           out=out.data_ptr(), saved=saved.data_ptr())
    _launch(dev, "magnet_gnet_pack_train_weights_f32", *(t.data_ptr() for t in ws), D, packed.data_ptr())
    _launch(dev, "magnet_gnet_train_fwd_f32", C.byref(a))
    return out, packed, saved, cost, prev_gmm


def gnet_bwd(grad_out, cost, prev_gmm, packed, saved, need):
    """The backward of ``GnetHeadTrain`` (one magnet_gnet_bwd_f32 call): -> [grad of the invariant, of W0[:, :D], W1, b1,
    W2, b2, W3, b3, of prev_gmm].  ``need``: 8 flags, whether the gradient of each weight and of prev_gmm is written
    (None where not); the invariant's gradient is always written."""
    B, D, H, W = cost.shape
    dev = cost.device
    grad_out = _need_cuda_f32("grad_out", grad_out)
    new = lambda shape: torch.empty(shape, device=dev, dtype=torch.float32)
    g_inv = new((B, _lib.MAGNET_HIDDEN_CHANNELS, H, W))
    g = [new(shape) if n else None for (_, shape), n in zip(gnet_weight_shapes(D), need[:7])]
    g_prev = new((B, 2, H, W)) if need[7] else None
    ws = torch.empty(int(lib().magnet_gnet_bwd_workspace_bytes(B, D, H, W)), device=dev, dtype=torch.uint8)
    a = _lib.GnetTrainArgs(B=B, D=D, H=H, W=W, cost=cost.data_ptr(), packed_weights=packed.data_ptr(),
                           prev_gmm=prev_gmm.data_ptr(), saved=saved.data_ptr(), grad_out=grad_out.data_ptr(),
                           workspace=ws.data_ptr(), grad_invariant=g_inv.data_ptr(), grad_w0_cost=_ptr(g[0]),
                           grad_w1=_ptr(g[1]), grad_b1=_ptr(g[2]), grad_w2=_ptr(g[3]), grad_b2=_ptr(g[4]),
                           grad_w3=_ptr(g[5]), grad_b3=_ptr(g[6]), grad_prev=_ptr(g_prev))
    _launch(dev, "magnet_gnet_bwd_f32", C.byref(a))
    return [g_inv, *g, g_prev]


def gnet_head_train(cost, invariant, gnet, prev_gmm):
    """``GnetHeadTrain`` on the weights of a ``GNET`` (or its ``gnet`` Sequential): the cost slice W0[:, :D] of the first
    convolution (autograd scatters its gradient into the full weight), the two 128x128 layers and the 128->2 layer.
    The head must have the structure ``gnet_head_layers`` recognises.  Validates like ``gnet_update``."""
    if cost.dim() != 4:
        raise _lib.MagnetError(f"cost must be (B,D,H,W), got {tuple(cost.shape)}")
    D = cost.shape[1]
    c0, c1, c2, c3 = _gnet_convs(gnet, D)
    ws = (c0.weight[:, :D], c1.weight, c1.bias, c2.weight, c2.bias, c3.weight, c3.bias)
    if _traced():
        return _op("gnet_train_fwd")(cost, invariant, *ws, prev_gmm)[0]
    return GnetHeadTrain.apply(cost, invariant, *ws, prev_gmm)


class ConvexUpsample(torch.autograd.Function):
    """upsample_depth_via_mask (MAGNET.py:15-27) as one kernel each way; differentiable in depth and mask."""

    @staticmethod
    def forward(ctx, depth: torch.Tensor, up_mask: torch.Tensor, k: int) -> torch.Tensor:
        depth = _need_cuda_f32("depth", depth)
        up_mask = _need_cuda_f32("up_mask", up_mask)
        B, CH, H, W = depth.shape
        if up_mask.shape != (B, 9 * k * k, H, W):
            raise _lib.MagnetError(f"up_mask must be (B, 9*k*k, H, W) = {(B, 9 * k * k, H, W)}, got {tuple(up_mask.shape)}")
        out = torch.empty(B, CH, k * H, k * W, device=depth.device, dtype=torch.float32)
        dev = _same_device(("depth", depth), ("up_mask", up_mask))
        _launch(dev, "magnet_convex_upsample_fwd_f32", depth.data_ptr(), up_mask.data_ptr(), B, CH, H, W, k,
                out.data_ptr())
        ctx.save_for_backward(depth, up_mask)
        ctx.k = k
        return out

    @staticmethod
    def backward(ctx, grad_out: torch.Tensor):
        depth, up_mask = ctx.saved_tensors
        return (*convex_upsample_bwd(grad_out, depth, up_mask, ctx.k), None)


def convex_upsample_bwd(grad_out, depth, up_mask, k: int):
    """The gradients of ``convex_upsample`` w.r.t. (depth, up_mask): one magnet_convex_upsample_bwd_f32 launch."""
    grad_out = _need_cuda_f32("grad_out", grad_out)
    depth, up_mask = _need_cuda_f32("depth", depth), _need_cuda_f32("up_mask", up_mask)
    B, CH, H, W = depth.shape
    g_depth = torch.zeros_like(depth)
    g_mask = torch.empty_like(up_mask)
    _launch(depth.device, "magnet_convex_upsample_bwd_f32", grad_out.data_ptr(), depth.data_ptr(),
            up_mask.data_ptr(), B, CH, H, W, k, g_depth.data_ptr(), g_mask.data_ptr())
    return g_depth, g_mask


def convex_upsample(depth: torch.Tensor, up_mask: torch.Tensor, k: int) -> torch.Tensor:
    if _traced():                                  # the op has a backward (magnet_b200.library)
        return _op("convex_upsample")(depth, up_mask, int(k))
    return ConvexUpsample.apply(depth, up_mask, k)


def mask_weights_bytes(k: int = 4) -> int:
    """Bytes of the packed mask-head weights for upsampling factor k (0 for any k but 4)."""
    return int(lib().magnet_mask_weights_bytes(int(k)))


def _is_conv(c, cin, cout, ksize: int) -> bool:
    """A biased Conv2d cout <- cin (cin None: any) with a ksize x ksize kernel, stride 1, 'same' zero padding."""
    pad = ksize // 2
    return (isinstance(c, torch.nn.Conv2d) and c.bias is not None and (cin is None or c.in_channels == cin)
            and c.out_channels == cout and c.kernel_size == (ksize, ksize) and c.padding == (pad, pad)
            and c.stride == (1, 1) and c.dilation == (1, 1) and c.groups == 1 and c.padding_mode == "zeros")


def _conv_chain(seq, *couts):
    """The convolutions of Conv(*,128,3), then ReLU, Conv(128,cout,1) for each of ``couts`` (every hidden one 128
    wide), or None."""
    hid = _lib.MAGNET_HIDDEN_CHANNELS
    if not isinstance(seq, torch.nn.Sequential) or len(seq) != 2 * len(couts) + 1:
        return None
    if not all(isinstance(seq[i], torch.nn.ReLU) for i in range(1, len(seq), 2)):
        return None
    convs = [seq[i] for i in range(0, len(seq), 2)]
    if not (_is_conv(convs[0], None, hid, 3) and all(_is_conv(c, hid, cout, 1) for c, cout in zip(convs[1:], couts))):
        return None
    return convs


def gnet_head_layers(gnet, D: int):
    """The four convolutions of a ``GNET`` (or its ``gnet`` Sequential) with the reference's structure (MAGNET.py:53-60):
    Conv(*,128,3), ReLU, Conv(128,128,1), ReLU, Conv(128,128,1), ReLU, Conv(128,2,1), every convolution with a bias,
    the first with at least D input channels (the cost channels come first).  None otherwise."""
    hid = _lib.MAGNET_HIDDEN_CHANNELS
    convs = _conv_chain(gnet.gnet if hasattr(gnet, "gnet") else gnet, hid, hid, 2)
    return None if convs is None or convs[0].in_channels < D else convs


def mask_head_layers(mask_head):
    """The four convolutions of a mask head with the reference's structure (MAGNET.py:111-118): Conv(*,128,3), ReLU,
    Conv(128,128,1), ReLU, Conv(128,128,1), ReLU, Conv(128,144,1), every convolution with a bias.  None otherwise."""
    hid = _lib.MAGNET_HIDDEN_CHANNELS
    return _conv_chain(mask_head, hid, hid, 9 * 4 * 4)


def _mask_convs(mask_head):
    convs = mask_head_layers(mask_head)
    if convs is None:
        raise _lib.MagnetError("not a mask head with the reference's structure (Conv(*,128,3), ReLU, Conv(128,128,1), "
                               "ReLU, Conv(128,128,1), ReLU, Conv(128,144,1))")
    return convs


def _check_k4(k, head: str = "mask head") -> None:
    if int(k) != 4:
        raise _lib.MagnetError(f"the fused {head} takes k = 4 only (144 mask channels), got {k}")


def _need_hidden(name: str, x: torch.Tensor) -> torch.Tensor:
    """A (B,128,H,W) hidden map: a first convolution's output before its ReLU, checked as ``_need_cuda_f32`` does."""
    x = _need_cuda_f32(name, x)
    if x.dim() != 4 or x.shape[1] != _lib.MAGNET_HIDDEN_CHANNELS:
        raise _lib.MagnetError(f"{name} must be (B,{_lib.MAGNET_HIDDEN_CHANNELS},H,W), got {tuple(x.shape)}")
    return x


def _pred_list(preds) -> list:
    return [preds] if isinstance(preds, torch.Tensor) else list(preds)


def pack_mask_weights(mask_head) -> torch.Tensor:
    """The weights of the mask head's last three layers in the fused kernel's layout (``mask_upsample``): the two
    128x128 layers and the 128->144 layer, split into fp16 hi/lo with one power-of-two scale per layer, and the fp32
    biases.  The first (3x3) layer stays outside (``MagnetHead.mask_pre``).  Read from the module at each call (nothing
    is cached).  Two launches."""
    _, c1, c2, c3 = _mask_convs(mask_head)
    ws = [t.detach() for t in (c1.weight, c1.bias, c2.weight, c2.bias, c3.weight, c3.bias)]
    if _traced():
        return _op("pack_mask_weights")(ws)
    return _pack_mask(ws)


def _pack_mask(ws) -> torch.Tensor:
    """``pack_mask_weights`` of the detached tensors W1, b1, W2, b2, W3, b3."""
    ts = [_need_cuda_f32(nm, t) for nm, t in zip(("W1", "b1", "W2", "b2", "W3", "b3"), ws)]
    dev = _same_device(*((f"weight {i}", t) for i, t in enumerate(ts)))
    out = torch.empty(mask_weights_bytes(4), device=dev, dtype=torch.uint8)
    _launch(dev, "magnet_mask_pack_weights_f32", *(t.data_ptr() for t in ts), out.data_ptr())
    return out


def mask_upsample(pre0: torch.Tensor, packed: torch.Tensor, preds, k: int = 4) -> list:
    """The mask head after its first convolution and the learned upsampling of every prediction, in one kernel per 8
    predictions: pre0 (B,128,H,W) = the first convolution's output before its ReLU (``MagnetHead.mask_pre``), packed =
    ``pack_mask_weights(mask_head)``, preds = quarter-resolution (B,2,H,W) [mu, sigma] tensors -> a list of
    (B,2,k*H,k*W) tensors, as ``convex_upsample(pred, mask_head(x_d3), k)`` gives them.  The 144-channel mask is never
    written.  k = 4 only.  Not differentiable (forward only): training runs the mask head, the upsampling and the
    loss through ``mask_head_loss``, which has a backward."""
    preds = _pred_list(preds)
    if _traced():
        return _op("mask_upsample")(pre0, packed, preds, int(k))
    if not preds:
        raise _lib.MagnetError("mask_upsample needs at least one prediction")
    _check_k4(k)
    pre0 = _need_hidden("pre0", pre0)
    B, _, H, W = pre0.shape
    nbytes = mask_weights_bytes(4)
    if not _is_packed(packed, (nbytes,)):
        raise _lib.MagnetError(f"packed must be a pack_mask_weights buffer ({nbytes} bytes)")
    preds = _need_preds("preds", preds, (B, 2, H, W))
    dev = _same_device(("pre0", pre0), ("packed", packed), *((f"preds[{i}]", p) for i, p in enumerate(preds)))
    outs = [torch.empty(B, 2, 4 * H, 4 * W, device=dev, dtype=torch.float32) for _ in preds]
    n = _lib.MAGNET_MASK_MAX_PRED
    for c in range(0, len(preds), n):
        ps, os_ = preds[c:c + n], outs[c:c + n]
        pp = (C.c_void_p * len(ps))(*[p.data_ptr() for p in ps])
        op = (C.c_void_p * len(os_))(*[o.data_ptr() for o in os_])
        a = _lib.MaskUpsampleArgs(P=len(ps), B=B, H=H, W=W, k=4, pre0=pre0.data_ptr(), packed_weights=packed.data_ptr(),
                                  pred=C.cast(pp, C.POINTER(C.c_void_p)), out=C.cast(op, C.POINTER(C.c_void_p)))
        _launch(dev, "magnet_mask_upsample_f32", C.byref(a))
    return outs


def dnet_head_layers(depth_head, mask_head=None):
    """The convolutions of D-Net's heads with the reference's structure (D_dense_depth.py:148-160): depth_head =
    Conv(*,128,3), ReLU, Conv(128,128,1), ReLU, Conv(128,2,1), and, when given, mask_head = the same with a last
    Conv(128,144,1) (k = 4), every convolution with a bias.  -> (depth convs, mask convs or None), or None."""
    hid = _lib.MAGNET_HIDDEN_CHANNELS
    d = _conv_chain(depth_head, hid, 2)
    if d is None:
        return None
    if mask_head is None:
        return d, None
    m = _conv_chain(mask_head, hid, 9 * 4 * 4)
    return None if m is None else (d, m)


def dnet_weights_bytes(k: int = 4) -> int:
    """Bytes of the packed D-Net weights: k = 0 the depth head alone, k = 4 both heads (0 for any other k)."""
    return int(lib().magnet_dnet_weights_bytes(int(k)))


def pack_dnet_weights(depth_head, mask_head=None) -> torch.Tensor:
    """The 1x1 layers of D-Net's depth head (and, when given, its mask head) in the fused kernels' layout
    (``dnet_depth``, ``dnet_upsample``): the 128x128 layers and the 128->144 layer split into fp16 hi/lo with one
    power-of-two scale per layer, the 128->2 layer and every bias in fp32.  The 3x3 layers stay outside (cuDNN).  Read
    from the modules at each call (nothing is cached).  Two launches."""
    layers = dnet_head_layers(depth_head, mask_head)
    if layers is None:
        raise _lib.MagnetError("not D-Net heads with the reference's structure (Conv(*,128,3), ReLU, Conv(128,128,1), "
                               "ReLU, Conv(128,2,1); mask head: the same ending in Conv(128,144,1))")
    return _pack_dnet_layers(layers)


def _pack_dnet_layers(layers) -> torch.Tensor:
    """``pack_dnet_weights`` of the heads' convolutions as ``dnet_head_layers`` returns them."""
    (_, d1, d2), m = layers
    k = 0 if m is None else 4
    ws = [d1.weight, d1.bias, d2.weight, d2.bias] + ([] if m is None else [m[1].weight, m[1].bias, m[2].weight, m[2].bias])
    ws = [t.detach() for t in ws]
    if _traced():
        return _op("pack_dnet_weights")(ws, k)
    return _pack_dnet(ws, k)


def _pack_dnet(ws, k: int) -> torch.Tensor:
    """``pack_dnet_weights`` of the detached tensors depth W1, b1, W2, b2 and, for k = 4, mask W1, b1, W3, b3."""
    names = ["depth W1", "depth b1", "depth W2", "depth b2", "mask W1", "mask b1", "mask W3", "mask b3"][:len(ws)]
    ts = [_need_cuda_f32(nm, t) for nm, t in zip(names, ws)]
    dev = _same_device(*zip(names, ts))
    out = torch.empty(dnet_weights_bytes(k), device=dev, dtype=torch.uint8)
    ptrs = [t.data_ptr() for t in ts] + [None] * (8 - len(ts))
    _launch(dev, "magnet_dnet_pack_weights_f32", *ptrs, k, out.data_ptr())
    return out


def _check_dnet_packed(packed, k: int) -> None:
    nbytes = dnet_weights_bytes(k)
    if not _is_packed(packed, (nbytes,) if k == 4 else (nbytes, dnet_weights_bytes(4))):
        what = "with the mask head " if k == 4 else ""
        raise _lib.MagnetError(f"packed must be a pack_dnet_weights buffer {what}({nbytes} bytes"
                               + (")" if k == 4 else f" or {dnet_weights_bytes(4)})"))


def dnet_depth(pre_d: torch.Tensor, packed: torch.Tensor, sigma: bool) -> torch.Tensor:
    """D-Net's depth head after its first convolution in one kernel: pre_d (B,128,H,W) = that convolution's output
    before its ReLU, packed = ``pack_dnet_weights(depth_head[, mask_head])`` -> (B,2,H,W): with ``sigma`` [mu, sigma] as
    activation_G_magnet gives it (DNET.py:62-67, MaGNet's mono_gmms), else the raw [mu, v] that ``dnet_upsample``
    reads.  Forward only."""
    if _traced():
        return _op("dnet_depth")(pre_d, packed, bool(sigma))
    pre_d = _need_hidden("pre_d", pre_d)
    _check_dnet_packed(packed, 0)
    B, _, H, W = pre_d.shape
    dev = _same_device(("pre_d", pre_d), ("packed", packed))
    out = torch.empty(B, 2, H, W, device=dev, dtype=torch.float32)
    _launch(dev, "magnet_dnet_depth_f32", pre_d.data_ptr(), packed.data_ptr(), B, H, W, int(bool(sigma)), out.data_ptr())
    return out


def dnet_upsample(pre_m: torch.Tensor, packed: torch.Tensor, raw: torch.Tensor, k: int = 4) -> torch.Tensor:
    """D-Net's mask head after its first convolution, the learned upsampling of the raw prediction and activation_G in
    one kernel: pre_m (B,128,H,W) = the mask head's first convolution before its ReLU, packed = ``pack_dnet_weights(
    depth_head, mask_head)``, raw = ``dnet_depth(..., sigma=False)`` -> (B,2,4H,4W) [mu, var], what DNET(args)
    returns (DNET.py:56-60).  The 144-channel mask is never written.  k = 4 only.  Forward only."""
    if _traced():
        return _op("dnet_upsample")(pre_m, packed, raw, int(k))
    _check_k4(k, "D-Net mask head")
    pre_m = _need_hidden("pre_m", pre_m)
    _check_dnet_packed(packed, 4)
    B, _, H, W = pre_m.shape
    raw = _need_cuda_f32("raw", raw, (B, 2, H, W))
    dev = _same_device(("pre_m", pre_m), ("packed", packed), ("raw", raw))
    out = torch.empty(B, 2, 4 * H, 4 * W, device=dev, dtype=torch.float32)
    _launch(dev, "magnet_dnet_upsample_f32", pre_m.data_ptr(), packed.data_ptr(), raw.data_ptr(), B, H, W, 4,
            out.data_ptr())
    return out


class MaskLossTrain(torch.autograd.Function):
    """The mask head after its first convolution, the learned upsampling and MagnetLoss 'gaussian' (utils/losses.py:
    34-50) of training in one forward kernel, differentiable in pre0, W1, b1, W2, b2, W3, b3 and every prediction
    (DESIGN §3.13): the forward also forms the loss's gradient with respect to the 144 logits and the predictions while
    they are on chip, so the mask is never written and is never read back per prediction (the logits' gradient is
    written once, for the backward); the backward is one tensor-core chain
    kernel and fixed-order weight-gradient GEMMs.  Inputs after b3: gt (B,1,4H,4W), the uint8 gt mask, k (4), gamma,
    the number of supervised pixels, then the P predictions (B,2,H,W).  The weights are packed at every call.

    Memory: the forward keeps h0, h1, h2 and the 144-channel gradient of the logits for the backward (528 channels per
    pixel when a layer or pre0 needs a gradient; none otherwise) and the unit-scale prediction gradients (2 per
    prediction); the backward adds d_h2 and d_h1 (256 channels).  The module path keeps about the same 528 channels
    (the three hidden maps and the mask), so this is no memory saving."""

    @staticmethod
    def forward(ctx, pre0, w1, b1, w2, b2, w3, b3, gt, gt_mask_u8, k, gamma, count, *preds):
        _check_k4(k)
        need = ctx.needs_input_grad
        save_maps, pred_grad = any(need[:7]), any(need[12:])
        P = len(preds)
        gammas = loss_weights(gamma, P)
        partial, packed, saved = mask_train_fwd(pre0, (w1, b1, w2, b2, w3, b3), preds, gt, gt_mask_u8, save_maps,
                                                pred_grad, [g / float(count) for g in gammas])
        ctx.save_for_backward(packed, saved)
        ctx.shape = (P, *pre0.shape[:1], *pre0.shape[2:])
        # as magnet_loss sums its terms: per prediction the float64 sum of the partials, in fp32 over count, weighted
        terms = partial.view(-1, P).sum(0, dtype=torch.float64).to(torch.float32) / float(count)
        loss = 0.0
        for i in range(P):
            loss = loss + gammas[i] * terms[i]
        return loss

    @staticmethod
    def backward(ctx, grad_loss):
        packed, saved = ctx.saved_tensors
        need = ctx.needs_input_grad
        g_pre0, *g = mask_bwd(grad_loss, packed, saved, ctx.shape, need[:7], need[12:])
        return (g_pre0, *g[:6], None, None, None, None, None, *g[6:])


MASK_WEIGHT_NAMES = ("W1", "b1", "W2", "b2", "W3", "b3")


def mask_weight_shapes():
    """(name, shape) of the fused mask head's trained tensors W1, b1, W2, b2, W3, b3."""
    hid, nout = _lib.MAGNET_HIDDEN_CHANNELS, 9 * 4 * 4
    return tuple(zip(MASK_WEIGHT_NAMES, ((hid, hid, 1, 1), (hid,), (hid, hid, 1, 1), (hid,), (nout, hid, 1, 1), (nout,))))


def loss_weights(gamma: float, P: int) -> list:
    """MagnetLoss's weight gamma^(P-i-1) of prediction i (utils/losses.py:50), as Python floats."""
    return [gamma ** (P - i - 1) for i in range(P)]


def mask_saved_floats(P: int, B: int, H: int, W: int, save_maps: bool) -> int:
    """Floats of the `saved` buffer of the fused mask-loss forward: the prediction gradients, then the maps only when a
    layer gradient needs them."""
    return int(lib().magnet_mask_saved_bytes(P, B, H, W)) // 4 if save_maps else 2 * P * B * H * W


def mask_train_fwd(pre0, weights, preds, gt, gt_mask_u8, save_maps: bool, pred_grad: bool, scales):
    """The forward of ``MaskLossTrain``: the weights W1, b1, W2, b2, W3, b3 packed for training, then the fused forward
    (two launches).  ``scales``: the P prediction scales gamma_p / count, a list of host floats, or a (P,) float32 device
    tensor that the kernel reads when it runs (magnet_mask_train_fwd_dev_f32).  Returns (loss partials
    [tiles x P], packed weights, saved)."""
    P = len(preds)
    if not 1 <= P <= _lib.MAGNET_MASK_MAX_PRED:
        raise _lib.MagnetError(f"the fused mask-head loss takes 1 to {_lib.MAGNET_MASK_MAX_PRED} predictions, got {P}")
    pre0 = _need_hidden("pre0", pre0.detach())
    B, _, H, W = pre0.shape
    shapes = mask_weight_shapes()
    ws = _need_weights([(nm, t, shp) for (nm, shp), t in zip(shapes, weights)])
    ps = _need_preds("preds", (p.detach() for p in preds), (B, 2, H, W))
    gt = _need_cuda_f32("gt", gt.detach(), (B, 1, 4 * H, 4 * W))
    gt_mask_u8 = _need_cuda_u8_mask("gt_mask", gt_mask_u8, (B, 1, 4 * H, 4 * W), "(B,1,4H,4W)")
    dev = _same_device(("pre0", pre0), ("gt", gt), ("gt_mask", gt_mask_u8),
                       *((nm, t) for (nm, _), t in zip(shapes, ws)), *((f"preds[{i}]", p) for i, p in enumerate(ps)))
    on_device = isinstance(scales, torch.Tensor)
    if on_device:
        scales = _need_cuda_f32("scales", scales, (P,))
        _same_device(("pre0", pre0), ("scales", scales))
        host_scale = None
    else:
        host_scale = (C.c_float * P)(*scales)
    pp = (C.c_void_p * P)(*[p.data_ptr() for p in ps])
    packed = torch.empty(int(lib().magnet_mask_train_weights_bytes(4)), device=dev, dtype=torch.uint8)
    partial = torch.empty(int(lib().magnet_mask_train_partials(B, H, W)) * P, device=dev, dtype=torch.float32)
    saved = torch.empty(mask_saved_floats(P, B, H, W, save_maps), device=dev, dtype=torch.float32)
    a = _lib.MaskTrainArgs(P=P, B=B, H=H, W=W, k=4, pre0=pre0.data_ptr(), packed_weights=packed.data_ptr(),
                           pred=C.cast(pp, C.POINTER(C.c_void_p)), gt=gt.data_ptr(), gt_mask=gt_mask_u8.data_ptr(),
                           pred_scale=None if on_device else C.cast(host_scale, C.POINTER(C.c_float)),
                           save_maps=int(save_maps), pred_grad=int(pred_grad), partial=partial.data_ptr(),
                           saved=saved.data_ptr())
    _launch(dev, "magnet_mask_pack_train_weights_f32", *(t.data_ptr() for t in ws), packed.data_ptr())
    if on_device:
        _launch(dev, "magnet_mask_train_fwd_dev_f32", C.byref(a), scales.data_ptr())
    else:
        _launch(dev, "magnet_mask_train_fwd_f32", C.byref(a))
    return partial, packed, saved


def mask_bwd(grad_loss, packed, saved, shape, need_layers, need_preds):
    """The backward of ``MaskLossTrain`` (one magnet_mask_bwd_f32 call) for (P, B, H, W) = ``shape``: -> [grad of pre0,
    of W1, b1, W2, b2, W3, b3, then of each prediction].  ``need_layers``: 7 flags (pre0 and the six tensors),
    ``need_preds``: P flags; a gradient not needed is None.  The upstream gradient stays on the device."""
    P, B, H, W = shape
    dev = saved.device
    new = lambda shp: torch.empty(shp, device=dev, dtype=torch.float32)
    g_pre0 = new((B, _lib.MAGNET_HIDDEN_CHANNELS, H, W)) if need_layers[0] else None
    g = [new(shp) if n else None for (_, shp), n in zip(mask_weight_shapes(), need_layers[1:7])]
    g_preds = [new((B, 2, H, W)) if need_preds[i] else None for i in range(P)]
    grad_scale = grad_loss.detach().to(device=dev, dtype=torch.float32).reshape(1).contiguous()
    nws = int(lib().magnet_mask_bwd_workspace_bytes(B, H, W)) if any(need_layers) else 256
    ws = torch.empty(nws, device=dev, dtype=torch.uint8)
    gp = (C.c_void_p * P)(*[_ptr(t) for t in g_preds])
    a = _lib.MaskTrainArgs(P=P, B=B, H=H, W=W, k=4, packed_weights=packed.data_ptr(), saved=saved.data_ptr(),
                           grad_scale=grad_scale.data_ptr(), workspace=ws.data_ptr(), grad_pre0=_ptr(g_pre0),
                           grad_w1=_ptr(g[0]), grad_b1=_ptr(g[1]), grad_w2=_ptr(g[2]), grad_b2=_ptr(g[3]),
                           grad_w3=_ptr(g[4]), grad_b3=_ptr(g[5]), grad_pred=C.cast(gp, C.POINTER(C.c_void_p)))
    _launch(dev, "magnet_mask_bwd_f32", C.byref(a))
    return [g_pre0, *g, *g_preds]


def device_scales(num: torch.Tensor, count: torch.Tensor) -> torch.Tensor:
    """num / count on the device, as the host forms float(num / float(count)): a float64 division rounded once to
    float32; 0 where count is 0, so that an empty mask gives exactly zero gradients."""
    count = count.to(torch.float64)
    q = num.to(torch.float64) / torch.where(count > 0, count, torch.ones_like(count))
    return torch.where(count > 0, q, torch.zeros_like(q)).to(torch.float32)


def loss_term(partial_sum: torch.Tensor, count: torch.Tensor) -> torch.Tensor:
    """The float64 sum of a loss's partials over the device count of supervised pixels, with the arithmetic of the eager
    ``partial_sum.to(float32) / float(count)``: torch divides a CUDA tensor by a host scalar as a product with the scalar's
    fp32 reciprocal.  NaN for a count of 0 (0 * inf), as a mean over an empty selection."""
    return partial_sum.to(torch.float32) * torch.reciprocal(count.to(torch.float32))


def mask_head_loss(pre0, mask_head, preds, gt, gt_mask, k: int = 4, gamma: float = 0.8):
    """MagnetLoss 'gaussian' of the predictions upsampled by the mask of ``mask_head``, from pre0 = the mask head's first
    convolution before its ReLU (``MagnetHead.mask_pre``): ``magnet_loss(preds, mask_head(x_d3), gt, gt_mask, k, gamma)``
    through ``MaskLossTrain``, differentiable in pre0, the last three layers' weights and biases and every prediction.
    k = 4 and 1 to MAGNET_MASK_MAX_PRED predictions; gt_mask bool / uint8.  Validates like ``mask_upsample`` and
    ``UpsampleNLL``; reads the number of supervised pixels with one host read, as ``magnet_loss``."""
    _, c1, c2, c3 = _mask_convs(mask_head)
    preds = _pred_list(preds)
    if not preds:
        raise _lib.MagnetError("mask_head_loss needs at least one prediction")
    _check_k4(k)
    gtm = gt_mask.to(torch.uint8)
    ws = (c1.weight, c1.bias, c2.weight, c2.bias, c3.weight, c3.bias)
    if _traced():                          # the count stays on the device; an empty mask gives a NaN loss
        grad = torch.is_grad_enabled()
        save_maps = grad and any(t.requires_grad for t in (pre0, *ws))
        pred_grad = grad and any(p.requires_grad for p in preds)
        return _op("mask_train_fwd")(pre0, *ws, gt, gtm, gtm.sum(), preds, float(gamma), save_maps, pred_grad)[0]
    count = int(gtm.sum().item())          # one host read per step, as magnet_loss
    if count == 0:
        raise _lib.MagnetError("gt_mask selects no pixel")
    return MaskLossTrain.apply(pre0, *ws, gt, gtm, 4, gamma, count, *preds)


class UpsampleNLL(torch.autograd.Function):
    """mean over the supervised pixels of the Gaussian NLL of ONE convex-upsampled prediction — upsample_depth_via_mask
    (MAGNET.py:15-27) + the per-prediction term of MagnetLoss (utils/losses.py:39-49) in one kernel each way; the
    (B,2,kH,kW) prediction never reaches HBM.  Differentiable in depth (B,2,H,W) and up_mask (B,9k^2,H,W).
    With ``dnet``: DnetLoss (utils/losses.py:13-22) instead, ``depth`` being D-Net's raw depth-head output [mu, v],
    upsampled and passed through activation_G (DNET.py:56-60) inside the kernel (DESIGN §3.19)."""

    @staticmethod
    def forward(ctx, depth, up_mask, gt, gt_mask_u8, k, count, dnet=False):
        depth = _need_cuda_f32("raw" if dnet else "depth", depth)
        up_mask = _need_cuda_f32("up_mask", up_mask)
        gt = _need_cuda_f32("gt", gt)
        partial, gt_mask_u8 = upsample_nll_fwd(depth, up_mask, gt, gt_mask_u8, k, dnet)
        ctx.save_for_backward(depth, up_mask, gt, gt_mask_u8)
        ctx.k, ctx.count, ctx.dnet = k, float(count), dnet
        return partial.sum(dtype=torch.float64).to(torch.float32) / ctx.count

    @staticmethod
    def backward(ctx, grad_out):
        depth, up_mask, gt, gtm = ctx.saved_tensors
        grads = upsample_nll_bwd(depth, up_mask, gt, gtm, ctx.k, float(grad_out) / ctx.count, ctx.dnet)
        return (*grads, None, None, None, None, None)


# the entry points (forward, backward, backward with a device scale) of the two upsample + NLL loss forms: MagnetLoss
# of an upsampled [mu, sigma] and, with dnet=True, DnetLoss of the upsampled raw [mu, v] through activation_G
_NLL_ENTRY = {False: ("magnet_upsample_nll_fwd_f32", "magnet_upsample_nll_bwd_f32", "magnet_upsample_nll_bwd_dev_f32"),
              True: ("magnet_dnet_nll_fwd_f32", "magnet_dnet_nll_bwd_f32", "magnet_dnet_nll_bwd_dev_f32")}


def upsample_nll_fwd(depth, up_mask, gt, gt_mask_u8, k: int, dnet: bool = False):
    """The forward kernel of ``UpsampleNLL`` (DnetLoss's with ``dnet``; ``depth`` is then D-Net's raw [mu, v]) on
    checked fp32 operands: -> (per-CTA NLL partial sums, the checked mask)."""
    name = "raw" if dnet else "depth"
    depth, up_mask, gt = _need_cuda_f32(name, depth), _need_cuda_f32("up_mask", up_mask), _need_cuda_f32("gt", gt)
    B, CH, H, W = depth.shape
    if CH != 2:
        raise _lib.MagnetError(f"{name} must be (B,2,H,W) [mu, {'v' if dnet else 'sigma'}], got {tuple(depth.shape)}")
    _expect("up_mask", up_mask, (B, 9 * k * k, H, W))
    _expect("gt", gt, (B, 1, k * H, k * W))
    gt_mask_u8 = _need_cuda_u8_mask("gt_mask", gt_mask_u8, (B, 1, k * H, k * W), "(B,1,k*H,k*W)")
    dev = _same_device((name, depth), ("up_mask", up_mask), ("gt", gt), ("gt_mask", gt_mask_u8))
    partial = torch.empty(lib().magnet_upsample_nll_partials(B, H, W, k), device=dev, dtype=torch.float32)
    _launch(dev, _NLL_ENTRY[bool(dnet)][0], depth.data_ptr(), up_mask.data_ptr(), gt.data_ptr(),
            gt_mask_u8.data_ptr(), B, H, W, k, partial.data_ptr())
    return partial, gt_mask_u8


def upsample_nll_bwd(depth, up_mask, gt, gt_mask_u8, k: int, scale, dnet: bool = False):
    """The gradients of ``UpsampleNLL`` (DnetLoss's with ``dnet``) w.r.t. (depth, up_mask) at ``scale`` = upstream
    gradient / count: a host float (magnet_upsample_nll_bwd_f32 / magnet_dnet_nll_bwd_f32), or a 1-element float32
    device tensor the kernel reads when it runs (the _dev_f32 entry points)."""
    name = "raw" if dnet else "depth"
    depth, up_mask, gt = _need_cuda_f32(name, depth), _need_cuda_f32("up_mask", up_mask), _need_cuda_f32("gt", gt)
    B, _, H, W = depth.shape
    # the kernel reads the mask by address: a traced caller's mask may be strided (a permuted or channels-last bool)
    gt_mask_u8 = _need_cuda_u8_mask("gt_mask", gt_mask_u8, (B, 1, k * H, k * W), "(B,1,k*H,k*W)")
    g_depth = torch.zeros_like(depth)
    g_mask = torch.empty_like(up_mask)
    _, host, on_device = _NLL_ENTRY[bool(dnet)]
    if isinstance(scale, torch.Tensor):
        scale = _need_cuda_f32("scale", scale.reshape(1))
        _launch(depth.device, on_device, depth.data_ptr(), up_mask.data_ptr(), gt.data_ptr(),
                gt_mask_u8.data_ptr(), scale.data_ptr(), B, H, W, k, g_depth.data_ptr(), g_mask.data_ptr())
    else:
        _launch(depth.device, host, depth.data_ptr(), up_mask.data_ptr(), gt.data_ptr(),
                gt_mask_u8.data_ptr(), scale, B, H, W, k, g_depth.data_ptr(), g_mask.data_ptr())
    return g_depth, g_mask


def dnet_loss(raw, up_mask, gt, gt_mask, k: int = 4):
    """DnetLoss 'gaussian' (utils/losses.py:13-22) of ``DNET(args)``'s output, from the heads' outputs BEFORE the
    upsampling: raw (B,2,h,w) = the depth head's [mu, v], up_mask (B,9k^2,h,w) = the mask head's logits, gt / gt_mask
    (B,1,kh,kw), gt_mask bool / uint8; any k >= 1.  Through ``UpsampleNLL`` with ``dnet``; fp32 operands.  Eager reads the number of
    supervised pixels with one host read and raises on an empty mask; under torch.compile the count stays on the device
    and an empty mask gives a NaN loss and zero gradients."""
    if int(k) < 1:
        raise _lib.MagnetError(f"the upsampling ratio k must be >= 1, got {k}")
    gtm = gt_mask.to(torch.uint8)
    if _traced():
        return _op("dnet_nll_fwd")(raw, up_mask, gt, gtm, int(k), gtm.sum())
    count = int(gtm.sum().item())          # one host read per step; the reference's boolean indexing syncs 3x
    if count == 0:
        raise _lib.MagnetError("gt_mask selects no pixel")
    return UpsampleNLL.apply(raw, up_mask, gt, gtm, int(k), count, True)


def magnet_loss(pred_list, up_mask, gt, gt_mask, k: int, gamma: float = 0.8):
    """MagnetLoss 'gaussian' (utils/losses.py:34-50) on the QUARTER-RESOLUTION predictions of the matching loop and the
    shared upsampling mask: sum_i gamma^(n-i-1) * mean NLL(upsample(pred_i)), each term one fused kernel (f-2).
    pred_list: the (B,2,H,W) Gaussians pred_1..pred_n; gt (B,1,kH,kW); gt_mask bool / uint8 of the same shape.
    Under torch.compile the count stays on the device and an empty mask gives a NaN loss (eager raises)."""
    gtm = gt_mask.to(torch.uint8)
    n = len(pred_list)
    if _traced():
        count = gtm.sum()
        loss = 0.0
        for i, pred in enumerate(pred_list):
            loss = loss + _op("upsample_nll_fwd")(pred, up_mask, gt, gtm, int(k), count, gamma ** (n - i - 1))
        return loss
    count = int(gtm.sum().item())          # one host read per step; the reference's boolean indexing syncs 3x per term
    if count == 0:
        raise _lib.MagnetError("gt_mask selects no pixel")
    loss = 0.0
    for i, pred in enumerate(pred_list):
        loss = loss + gamma ** (n - i - 1) * UpsampleNLL.apply(pred, up_mask, gt, gtm, k, count, False)
    return loss


class FnetL1Loss(torch.autograd.Function):
    """train_FNet.py:96-108 — soft-argmin over the planes of the 1/V-averaged scores, then the mean over the supervised
    pixels of |pred - gt| — one kernel each way; the probability volume and the prediction never reach memory.
    Differentiable in the scores.  ``count`` is the number of supervised pixels (int, or a 0-dim device tensor)."""

    @staticmethod
    def forward(ctx, scores, planes, gt, mask_u8, count):
        scores = _need_cuda_f32("scores", scores)
        gt = _need_cuda_f32("gt", gt)
        if scores.dim() != 4:
            raise _lib.MagnetError(f"scores must be (B,D,H,W), got {tuple(scores.shape)}")
        partial, karr, scores, gt, mask_u8 = fnet_l1_fwd(scores, planes, gt, mask_u8)
        ctx.save_for_backward(scores, gt, mask_u8)
        ctx.karr, ctx.count = karr, count
        return partial.sum(dtype=torch.float64).to(torch.float32) / count

    @staticmethod
    def backward(ctx, grad_out):
        scores, gt, mask_u8 = ctx.saved_tensors
        # the upstream gradient stays on the device (no host read: the step can be captured in a CUDA graph)
        if isinstance(ctx.count, torch.Tensor):
            gs, scale = (grad_out / ctx.count).to(torch.float32), 1.0
        else:
            gs, scale = grad_out.to(torch.float32), 1.0 / float(ctx.count)
        return fnet_l1_bwd(scores, ctx.karr, gt, mask_u8, scale, gs), None, None, None, None


def fnet_l1_fwd(scores, planes, gt, mask_u8):
    """The forward kernel of ``FnetL1Loss``: -> (per-CTA L1 partial sums, the host plane array, and the checked scores,
    gt and mask the backward reads)."""
    scores = _need_cuda_f32("scores", scores)
    gt = _need_cuda_f32("gt", gt)
    if scores.dim() != 4:
        raise _lib.MagnetError(f"scores must be (B,D,H,W), got {tuple(scores.shape)}")
    B, D, H, W = scores.shape
    karr = planes if isinstance(planes, C.Array) else k_array(planes)
    if len(karr) != D:
        raise _lib.MagnetError(f"{len(karr)} plane depths for {D} score planes")
    _expect("gt", gt, (B, 1, H, W))
    mask_u8 = _need_cuda_u8_mask("mask", mask_u8, (B, 1, H, W), "(B,1,H,W)")
    dev = _same_device(("scores", scores), ("gt", gt), ("mask", mask_u8))
    partial = torch.empty(lib().magnet_fnet_l1_partials(B, H, W), device=dev, dtype=torch.float32)
    _launch(dev, "magnet_fnet_l1_fwd_f32", scores.data_ptr(), C.cast(karr, C.c_void_p), gt.data_ptr(),
            mask_u8.data_ptr(), B, D, H, W, partial.data_ptr())
    return partial, karr, scores, gt, mask_u8


def fnet_l1_bwd(scores, planes, gt, mask_u8, scale: float, grad_scale: torch.Tensor) -> torch.Tensor:
    """The gradient of ``FnetL1Loss`` w.r.t. the scores: one magnet_fnet_l1_bwd_f32 launch with the host ``scale`` and
    the 1-element device ``grad_scale`` (read when the kernel runs)."""
    scores = _need_cuda_f32("scores", scores)
    B, D, H, W = scores.shape
    karr = planes if isinstance(planes, C.Array) else k_array(planes)
    gs = grad_scale.to(torch.float32).reshape(1).contiguous()
    g = torch.empty_like(scores)
    _launch(scores.device, "magnet_fnet_l1_bwd_f32", scores.data_ptr(), C.cast(karr, C.c_void_p), gt.data_ptr(),
            mask_u8.data_ptr(), scale, gs.data_ptr(), B, D, H, W, g.data_ptr())
    return g


def fnet_l1_loss(scores, planes, gt_q, mask_q, count=None):
    """F-Net's L1 loss (train_FNet.py:96-108) on the 1/V-averaged plane-sweep scores (B,D,H,W): softmax over the D
    planes, soft-argmin depth with the plane depths ``planes``, mean |pred - gt_q| where ``mask_q`` (B,1,H,W) is set.
    ``count`` = number of supervised pixels; by default it is read from the mask (one host read, which also rejects an
    empty mask — pass it explicitly to capture the step in a CUDA graph).  Under torch.compile the count is formed on
    the device (``count`` must then be None) and an empty mask gives a NaN loss."""
    mask_u8 = mask_q.to(torch.uint8)
    if _traced():
        if count is not None:
            raise _lib.MagnetError("under torch.compile fnet_l1_loss counts the mask on the device (pass count=None)")
        return _op("fnet_l1_fwd")(scores, k_array(planes), gt_q, mask_u8, mask_u8.sum())
    if count is None:
        count = int(mask_u8.sum().item())
        if count == 0:
            raise _lib.MagnetError("mask_q selects no pixel")
    return FnetL1Loss.apply(scores, planes, gt_q, mask_u8, count)


def plane_depth(volume: torch.Tensor, planes, *, scores: bool) -> torch.Tensor:
    """F-Net's soft-argmin depth map sum_j prob_j d_j (train_FNet.py:96 / :180) of a (B,D,h,w) plane volume ->
    (B,1,h,w) float32, one kernel.  ``scores=True``: ``volume`` is the 1/V-averaged scores of
    ``plane_sweep_f(softmax=False)``; the softmax over the planes is fused in and the prediction is bit for bit the one
    ``fnet_l1_loss`` supervises.  ``scores=False``: ``volume`` is the probability volume of ``est_costvolume_F`` /
    ``MAGNET_F.forward``.  ``planes``: the D plane depths, a sequence of floats or the (1,D,1,1) ``d_center`` tensor
    (read to the host once per tensor; under torch.compile it must be the sequence of floats).  Half-precision volumes
    (torch.autocast) are upcast."""
    if isinstance(volume, torch.Tensor) and volume.dtype in (torch.float16, torch.bfloat16):
        volume = volume.float()
    if _traced():
        return _op("plane_depth")(volume, k_array(planes), bool(scores))
    volume = _need_cuda_f32("volume", volume)
    if volume.dim() != 4:
        raise _lib.MagnetError(f"volume must be (B,D,H,W), got {tuple(volume.shape)}")
    B, D, H, W = volume.shape
    if isinstance(planes, torch.Tensor):
        from .homography import _plane_list
        planes = _plane_list(planes)
    karr = planes if isinstance(planes, C.Array) else k_array(planes)
    if len(karr) != D:
        raise _lib.MagnetError(f"{len(karr)} plane depths for {D} planes of the volume")
    out = torch.empty(B, 1, H, W, device=volume.device, dtype=torch.float32)
    _launch(volume.device, "magnet_plane_depth_f32", volume.data_ptr(), C.cast(karr, C.c_void_p), B, D, H, W,
            int(bool(scores)), out.data_ptr())
    return out


def relative_poses(ext_ref: torch.Tensor, ext_nghbr: torch.Tensor):
    """data_preprocess (utils/utils.py:72-98) on the device: ext_ref (B,4,4), ext_nghbr (V,B,4,4) ->
    (nghbr_poses (B,V,4,4), is_valid (B,V) int32)."""
    if _traced():
        return tuple(_op("relative_poses")(ext_ref, ext_nghbr))
    ext_ref = _need_cuda_f32("ext_ref", ext_ref)
    ext_nghbr = _need_cuda_f32("ext_nghbr", ext_nghbr)
    V, B = ext_nghbr.shape[0], ext_nghbr.shape[1]
    poses = torch.empty(B, V, 4, 4, device=ext_ref.device, dtype=torch.float32)
    valid = torch.empty(B, V, device=ext_ref.device, dtype=torch.int32)
    dev = _same_device(("ext_ref", ext_ref), ("ext_nghbr", ext_nghbr))
    _launch(dev, "magnet_relative_poses_f32", ext_ref.data_ptr(), ext_nghbr.data_ptr(), B, V, poses.data_ptr(),
            valid.data_ptr())
    return poses, valid


def camera_rays(raw_intrinsics: torch.Tensor, H: int, W: int):
    """get_cam_intrinsics (data/dataloader_scannet.py:113-153, data/dataloader_kitti.py:94-127) on the device:
    raw_intrinsics (B,8) float64 [fx, fy, cx, cy, img_W, img_H, left_margin, top_margin] (a (B,6) tensor
    [fx, fy, cx, cy, raw_W, raw_H] is accepted as the ScanNet case: no crop) -> cam_intrins dict
    {'intM' (B,3,3), 'unit_ray_array_2D' (B,3,H*W)} (device)."""
    if _traced():
        intM, rays = _op("camera_rays")(raw_intrinsics, int(H), int(W))
        return {"intM": intM, "unit_ray_array_2D": rays}
    if not raw_intrinsics.is_cuda or raw_intrinsics.dtype != torch.float64 or raw_intrinsics.dim() != 2 \
            or raw_intrinsics.shape[1] not in (6, 8):
        raise _lib.MagnetError("raw_intrinsics must be a CUDA float64 tensor (B,8) (or (B,6) without crop margins)")
    if raw_intrinsics.shape[1] == 6:
        raw_intrinsics = torch.cat([raw_intrinsics, torch.zeros_like(raw_intrinsics[:, :2])], dim=1)
    raw_intrinsics = raw_intrinsics.contiguous()
    B = raw_intrinsics.shape[0]
    intM = torch.empty(B, 3, 3, device=raw_intrinsics.device, dtype=torch.float32)
    rays = torch.empty(B, 3, H * W, device=raw_intrinsics.device, dtype=torch.float32)
    _launch(raw_intrinsics.device, "magnet_camera_rays_f32", raw_intrinsics.data_ptr(), B, H, W, intM.data_ptr(),
            rays.data_ptr())
    return {"intM": intM, "unit_ray_array_2D": rays}


# validate() (test_MaGNet.py:62-68): the KITTI evaluation crops as fractions of the GT size -> (row0, row1, col0, col1)
_CROPS = {"garg": (0.40810811, 0.99189189, 0.03594771, 0.96405229),
          "eigen": (0.3324324, 0.91351351, 0.0359477, 0.96405229)}
METRIC_KEYS = ("a1", "a2", "a3", "abs_diff", "abs_rel", "sq_rel", "rmse", "log_10", "irmse", "rmse_log", "silog", "nll")


def crop_box(crop, H: int, W: int):
    """Evaluation box [row0, row1) x [col0, col1) of an H x W GT: the whole image for ``crop=None``, else the 'garg' /
    'eigen' crop bounds, computed with Python floats and int() exactly as validate() slices its eval_mask."""
    if crop is None:
        return 0, H, 0, W
    if crop not in _CROPS:
        raise _lib.MagnetError(f"crop must be None, 'garg' or 'eigen', got {crop!r}")
    r0, r1, c0, c1 = _CROPS[crop]
    r0, r1, c0, c1 = int(r0 * H), int(r1 * H), int(c0 * W), int(c1 * W)
    return r0, max(r0, r1), c0, max(c0, c1)


def depth_metrics(pred_or_list, gt: torch.Tensor, *, min_depth: float, max_depth: float, crop=None,
                  up_mask: Optional[torch.Tensor] = None, k: Optional[int] = None, nearest: bool = False,
                  variance: bool = False) -> torch.Tensor:
    """Per-image depth metrics of validate() (test_MaGNet.py:52-79) + utils.compute_depth_errors, on the device.

    pred_or_list: one prediction or a list of up to 8 sharing ``gt`` (B,1,H,W) (raw GT; values above max_depth count
    as 0).  Each prediction is the full-resolution (B,2,H,W) [mu, sigma], or, with ``up_mask`` (B,9k^2,H/k,W/k) and
    ``k``, the quarter-resolution (B,2,H/k,W/k) Gaussians, upsampled inside the kernel (upsample_depth_via_mask).
    With ``nearest=True`` (F-Net's validate(), train_FNet.py:165-193) each prediction is a (B,1,h,w) depth map with
    h <= H, w <= W, upsampled inside the kernel as F.interpolate(..., size=(H, W), mode='nearest'); there is no
    variance and the nll column is 0.0, as compute_depth_errors(..., var=None) gives it.
    With ``variance=True`` (D-Net's validate(), test_DNet.py:22-73) each prediction is the full-resolution (B,2,H,W)
    [mu, var] that D-Net returns: channel 1 is the variance itself, clamped at 1e-6, not squared.  It does not combine
    with ``nearest`` or ``up_mask`` / ``k``.
    crop: None, 'garg' or 'eigen'.  Returns a (P,B,13) float64 device tensor: the number of valid pixels, then the
    metrics in METRIC_KEYS order (NaN for an image without a valid pixel; nll 0.0 there in the nearest form).  Two
    kernel launches, no host sync."""
    preds = _pred_list(pred_or_list)
    if _traced():
        return _op("depth_metrics")(preds, gt, float(min_depth), float(max_depth), crop, up_mask,
                                    None if k is None else int(k), bool(nearest), bool(variance))
    if not 1 <= len(preds) <= _lib.MAGNET_METRICS_MAX_PRED:
        raise _lib.MagnetError(f"1 to {_lib.MAGNET_METRICS_MAX_PRED} predictions per call, got {len(preds)}")
    if nearest and (up_mask is not None or k is not None):
        raise _lib.MagnetError("nearest=True takes (B,1,h,w) depth maps: it does not combine with up_mask / k")
    if variance and (nearest or up_mask is not None or k is not None):
        raise _lib.MagnetError("variance=True takes full-resolution (B,2,H,W) [mu, var]: it does not combine with "
                               "nearest or up_mask / k")
    gt = _need_cuda_f32("gt", gt)
    if gt.dim() != 4 or gt.shape[1] != 1:
        raise _lib.MagnetError(f"gt must be (B,1,H,W), got {tuple(gt.shape)}")
    B, _, H, W = gt.shape
    if nearest:
        return _depth_metrics_nearest(preds, gt, min_depth, max_depth, crop)
    if (up_mask is None) != (k is None):
        raise _lib.MagnetError("up_mask and k go together (the fused-upsampling form needs both)")
    if up_mask is not None:
        k = int(k)
        if k < 1 or H % k or W % k:
            raise _lib.MagnetError(f"k = {k} must be >= 1 and divide the GT size {H}x{W}")
        up_mask = _need_cuda_f32("up_mask", up_mask, (B, 9 * k * k, H // k, W // k))
        pshape = (B, 2, H // k, W // k)
    else:
        pshape = (B, 2, H, W)
    preds = _need_preds("pred", preds, pshape)
    dev = _same_device(("gt", gt), ("up_mask", up_mask), *((f"pred[{i}]", p) for i, p in enumerate(preds)))
    r0, r1, c0, c1 = crop_box(crop, H, W)
    ptrs = (C.c_void_p * len(preds))(*[p.data_ptr() for p in preds])
    a = _lib.DepthMetricsArgs(P=len(preds), B=B, H=H, W=W, k=k or 0, row0=r0, row1=r1, col0=c0, col1=c1,
                              min_depth=float(min_depth), max_depth=float(max_depth),
                              pred=C.cast(ptrs, C.POINTER(C.c_void_p)), up_mask=up_mask.data_ptr() if k else None,
                              gt=gt.data_ptr())
    fn = "magnet_depth_metrics_var_f32" if variance else "magnet_depth_metrics_f32"
    return _run_depth_metrics(dev, a, "magnet_depth_metrics_workspace", fn)


def _run_depth_metrics(dev, a, workspace_fn: str, fn: str) -> torch.Tensor:
    """The workspace and the (P,B,13) output of the checked metrics arguments ``a``, then the launch of ``fn``."""
    n = getattr(lib(), workspace_fn)(C.byref(a))
    if n < 0:
        check(int(n), workspace_fn)
    workspace = torch.empty(int(n), device=dev, dtype=torch.float64)
    out = torch.empty(a.P, a.B, _lib.MAGNET_METRICS_COLS, device=dev, dtype=torch.float64)
    a.workspace, a.out = workspace.data_ptr(), out.data_ptr()
    _launch(dev, fn, C.byref(a))
    return out


def _depth_metrics_nearest(preds, gt, min_depth, max_depth, crop):
    """The nearest form of ``depth_metrics``: ``preds`` (B,1,h,w) each, ``gt`` the checked (B,1,H,W) GT."""
    B, _, H, W = gt.shape
    preds = _need_preds("pred", preds)
    pshape = tuple(preds[0].shape)
    if len(pshape) != 4 or pshape[:2] != (B, 1) or not (1 <= pshape[2] <= H and 1 <= pshape[3] <= W):
        raise _lib.MagnetError(f"pred[0] must be (B,1,h,w) with B = {B}, h <= {H}, w <= {W}, got {pshape}")
    for i, p in enumerate(preds):
        _expect(f"pred[{i}]", p, pshape)
    dev = _same_device(("gt", gt), *((f"pred[{i}]", p) for i, p in enumerate(preds)))
    r0, r1, c0, c1 = crop_box(crop, H, W)
    ptrs = (C.c_void_p * len(preds))(*[p.data_ptr() for p in preds])
    a = _lib.DepthMetricsNearestArgs(P=len(preds), B=B, H=H, W=W, h=pshape[2], w=pshape[3], row0=r0, row1=r1, col0=c0,
                                     col1=c1, min_depth=float(min_depth), max_depth=float(max_depth),
                                     pred=C.cast(ptrs, C.POINTER(C.c_void_p)), gt=gt.data_ptr())
    return _run_depth_metrics(dev, a, "magnet_depth_metrics_nearest_workspace", "magnet_depth_metrics_nearest_f32")
