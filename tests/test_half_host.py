"""Host side of the half-precision path, without a GPU: the dispatch rule (HALF16 or upcast), the new header constants
and bytes formula, and the argument checks of magnet_repack_half16 and of the entry points on HALF16 buffers."""
import ctypes as C

import pytest
import torch

from magnet_b200 import _lib
from magnet_b200.homography import MMA_MIN_PLANES, differentiable_layout, route, wants_half16

F16, BF16, F32 = torch.float16, torch.bfloat16, torch.float32


@pytest.mark.parametrize("ref,src,C_,V,D,variant,want", [
    (BF16, BF16, 64, 2, 64, _lib.VARIANT_AUTO, True),
    (F16, F16, 64, 16, MMA_MIN_PLANES, _lib.VARIANT_AUTO, True),
    (F16, F16, 64, 2, 5, _lib.VARIANT_MMA, True),           # variant MMA: any D
    (F16, F16, 64, 2, 5, _lib.VARIANT_AUTO, False),         # the shipped N_s = 5: gather kernel on the upcast maps
    (F16, F16, 64, 2, MMA_MIN_PLANES - 1, _lib.VARIANT_AUTO, False),
    (BF16, BF16, 32, 2, 64, _lib.VARIANT_AUTO, False),      # C != 64
    (BF16, BF16, 64, 17, 64, _lib.VARIANT_AUTO, False),     # V > 16
    (BF16, BF16, 64, 2, 64, _lib.VARIANT_DIRECT, False),
    (BF16, BF16, 64, 2, 64, _lib.VARIANT_CELLS, False),
    (BF16, BF16, 64, 2, 64, _lib.VARIANT_TMA, False),
    (F16, BF16, 64, 2, 64, _lib.VARIANT_AUTO, False),       # mixed dtypes
    (F32, BF16, 64, 2, 64, _lib.VARIANT_AUTO, False),
    (F32, F32, 64, 2, 64, _lib.VARIANT_AUTO, False),        # fp32: today's SPLIT16 path
])
def test_dispatch_rule(ref, src, C_, V, D, variant, want):
    assert wants_half16(ref, src, C_, V, variant, D) is want
    layout, kernel = route(C_, V, D, variant, _lib.DEPTH_VOLUME, ref, src)
    assert (layout == _lib.SRC_HALF16) is want and kernel == variant


def test_route_differentiable_layout_with_half_maps():
    def layout(D, dtype):
        return route(64, 2, D, _lib.VARIANT_AUTO, _lib.DEPTH_VOLUME, dtype, dtype, differentiable=True)
    assert layout(64, F16) == (_lib.SRC_HALF16, _lib.VARIANT_AUTO)
    assert layout(64, F32) == (_lib.SRC_SPLIT16, _lib.VARIANT_AUTO)
    assert layout(5, F16) == (_lib.SRC_NCHW, _lib.VARIANT_DIRECT)
    assert differentiable_layout(64, 2, 64, _lib.VARIANT_AUTO, half=True) == _lib.SRC_HALF16
    assert differentiable_layout(64, 2, 64, _lib.VARIANT_AUTO, half=False) == _lib.SRC_SPLIT16
    assert differentiable_layout(64, 2, 5, _lib.VARIANT_AUTO, half=True) == _lib.SRC_NCHW


def test_constants_and_bytes_formula():
    L = _lib.lib()
    assert (_lib.SRC_SPLIT16, _lib.SRC_HALF16, _lib.DTYPE_F16, _lib.DTYPE_BF16) == (3, 4, 0, 1)
    assert L.magnet_abi_version() == _lib.MAGNET_ABI_VERSION == 4
    for N, H, W in ((1, 1, 1), (2, 3, 5), (6, 120, 160), (4, 88, 304)):
        assert L.magnet_half16_bytes(N, H, W) == 256 + N * H * W * 128 + N * H * (W + 1) * 16
        assert L.magnet_split16_bytes(N, H, W) - L.magnet_half16_bytes(N, H, W) == N * H * W * 128
    assert L.magnet_half16_bytes(0, 3, 5) == 0 and L.magnet_half16_bytes(2, -1, 5) == 0


def test_repack_half16_abi_validation_without_gpu():
    L = _lib.lib()
    buf = (C.c_double * 64)()
    p = C.cast(buf, C.c_void_p).value
    p = (p + 15) // 16 * 16 if p % 16 else p

    def run(src=p, dtype=_lib.DTYPE_F16, gmm=None, dst=p, N=2, C_=64, H=4, W=4):
        return L.magnet_repack_half16(src, dtype, gmm, dst, N, C_, H, W, None)

    assert run(src=None) == _lib.ERR_NULL
    assert run(dst=None) == _lib.ERR_NULL
    for bad in (dict(N=0), dict(H=0), dict(W=-1), dict(C_=0), dict(N=70000)):
        assert run(**bad) == _lib.ERR_SHAPE, bad
    for bad in (dict(C_=32), dict(C_=65), dict(dtype=2), dict(dtype=-1)):
        assert run(**bad) == _lib.ERR_UNSUPPORTED, bad
    assert run(src=p + 2) == _lib.ERR_ALIGN
    assert run(dst=p + 8, dtype=_lib.DTYPE_BF16) == _lib.ERR_ALIGN


def test_cost_entry_points_check_half16_arguments_without_gpu():
    """HALF16 takes SPLIT16's rules: C == 64, V <= 16, variant AUTO or MMA, 16-byte aligned buffers.  Every case below is
    refused before anything reaches the device."""
    L = _lib.lib()
    one = 0x1000

    def args(**kw):
        a = _lib.CostArgs()
        a.B, a.V, a.D, a.C, a.H, a.W = 1, 2, 64, 64, 8, 8
        a.depth_mode, a.src_layout, a.consistency, a.variant, a.kappa = _lib.DEPTH_PLANES, _lib.SRC_HALF16, 0, 0, 5.0
        a.ref_feat = a.src_feat = a.rays = a.cams = a.out = a.k_host = one
        for k, v in kw.items():
            setattr(a, k, v)
        return a

    for bad, status in ((dict(C=32), _lib.ERR_UNSUPPORTED), (dict(V=17), _lib.ERR_UNSUPPORTED),
                        (dict(variant=_lib.VARIANT_DIRECT), _lib.ERR_UNSUPPORTED),
                        (dict(variant=_lib.VARIANT_TMA), _lib.ERR_UNSUPPORTED),
                        (dict(src_feat=one + 4), _lib.ERR_ALIGN), (dict(ref_feat=one + 8), _lib.ERR_ALIGN),
                        (dict(ref_feat=None), _lib.ERR_NULL)):
        assert L.magnet_cost_volume_f32(C.byref(args(**bad)), None) == status, bad
    g, b, s = C.c_int(), C.c_int(), C.c_int()
    assert L.magnet_cost_launch_info(C.byref(args(C=16)), C.byref(g), C.byref(b), C.byref(s)) == _lib.ERR_UNSUPPORTED
    # the backward entry points: F volume with a HALF16 forward at an unsupported width, CW without a depth source
    fb = _lib.CostFBwdArgs()
    fa = args(C=32)
    fb.fwd = C.pointer(fa)
    fb.grad_out = fb.workspace = fb.grad_ref = fb.grad_src = one
    assert L.magnet_cost_volume_f_bwd_f32(C.byref(fb), None) == _lib.ERR_UNSUPPORTED
    cb = _lib.CostBwdArgs()
    ca = args(depth_mode=_lib.DEPTH_VOLUME, consistency=1, variant=_lib.VARIANT_DIRECT)
    ca.d_volume = one
    cb.fwd = C.pointer(ca)
    cb.grad_out = cb.workspace = one
    assert L.magnet_cost_volume_bwd_f32(C.byref(cb), None) == _lib.ERR_UNSUPPORTED


def test_python_layer_refuses_bad_half_input_without_gpu():
    from magnet_b200 import ops
    with pytest.raises(_lib.MagnetError):
        ops.repack_half16(torch.zeros(1, 64, 4, 4, dtype=torch.float16))      # CPU tensor
    with pytest.raises(TypeError):
        ops.repack_half16(None)
