"""CPU-side tests of the fused G-Net head (DESIGN §3.8): C-ABI argument checks (no launch), the packed-weight size, a
numpy restatement of its SPLIT16 numerics, and the dispatch rule of matching_loop on stand-in tensors."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn as nn

from magnet_b200 import _lib, ops
from magnet_b200.matcher import GNET, fused_gnet_applies


def test_gnet_entry_points_validate_without_launching():
    L = _lib.lib()
    buf = (C.c_float * 64)()
    p = C.cast(buf, C.c_void_p)
    assert L.magnet_gnet_update_f32(None, None) == _lib.ERR_NULL
    a = _lib.GnetArgs()
    assert L.magnet_gnet_update_f32(C.byref(a), None) == _lib.ERR_SHAPE
    a.B, a.D, a.H, a.W = 1, 8, 4, 4
    assert L.magnet_gnet_update_f32(C.byref(a), None) == _lib.ERR_NULL
    a.cost = a.invariant = a.packed_weights = a.prev_gmm = a.scratch = a.out = p
    a.D = _lib.MAGNET_MAX_PLANES + 1
    assert L.magnet_gnet_update_f32(C.byref(a), None) == _lib.ERR_UNSUPPORTED
    a.D = 8
    a.cost = C.c_void_p(C.addressof(buf) + 4)
    assert L.magnet_gnet_update_f32(C.byref(a), None) == _lib.ERR_ALIGN
    a.cost, a.packed_weights = p, C.c_void_p(C.addressof(buf) + 8)
    assert L.magnet_gnet_update_f32(C.byref(a), None) == _lib.ERR_ALIGN
    a.packed_weights, a.W = p, 0
    assert L.magnet_gnet_update_f32(C.byref(a), None) == _lib.ERR_SHAPE
    pack = L.magnet_gnet_pack_weights_f32
    assert pack(*([p] * 7), 8, None, None) == _lib.ERR_NULL
    assert pack(*([p] * 7), 0, p, None) == _lib.ERR_SHAPE
    assert pack(*([p] * 7), 257, p, None) == _lib.ERR_UNSUPPORTED
    assert pack(*([p] * 7), 8, C.c_void_p(C.addressof(buf) + 4), None) == _lib.ERR_ALIGN


def test_gnet_weights_bytes_formula():
    L = _lib.lib()
    # 4 KiB of header and fp32 vectors, W1 and W2 as 64 KiB of hi/lo fragments each, then per 16-channel chunk of the
    # cost volume the 9 taps x 128 outputs x 16 channels x (hi, lo) of W0
    for D in (1, 5, 16, 17, 64, 256):
        assert L.magnet_gnet_weights_bytes(D) == 4096 + 2 * 65536 + -(-D // 16) * 9 * 128 * 16 * 2 * 2
    assert L.magnet_gnet_weights_bytes(0) == 0
    assert L.magnet_gnet_weights_bytes(257) == 0


# ---- numpy restatement of the SPLIT16 numerics --------------------------------------------------------------------
def shift(m):
    """The SPLIT16 rule: power-of-two shift mapping the largest finite |x| into [2^14, 2^15); 0 for 0 / non-finite."""
    m = np.float32(m)
    if m == 0 or not np.isfinite(m) or m < np.finfo(np.float32).tiny:
        return 0
    return int(np.clip(14 - int(np.floor(np.log2(m))), -100, 100))


def split(x, sh):
    xs = (x.astype(np.float32) * np.float32(2.0 ** sh)).astype(np.float32)
    hi = xs.astype(np.float16)
    lo = (xs - hi.astype(np.float32)).astype(np.float16)
    return hi, lo


def gemm3(a, sa, w, sw):
    """a (M,K) with one shift per row, w (N,K) with one shift: three fp16 products in float64 (exact products, the
    tensor cores' fp32 accumulation is below the bound of DESIGN §3.8) and the exact descale."""
    ah, al = split(a, sa[:, None])
    wh, wl = split(w, sw)
    f = lambda u: u.astype(np.float64)
    acc = f(ah) @ f(wh).T + f(ah) @ f(wl).T + f(al) @ f(wh).T
    return acc * 2.0 ** (-sa[:, None].astype(np.float64)) * 2.0 ** (-sw)


@pytest.mark.parametrize("m", [1e-30, 1e-3, 0.7, 1.0, 3.0, 1e3, 6e4, 1e30])
def test_scale_rule(m):
    sh = shift(m)
    assert 2 ** 14 <= np.float64(np.float32(m)) * 2.0 ** sh < 2 ** 15 or abs(sh) == 100
    assert shift(0.0) == 0 and shift(np.inf) == 0 and shift(np.nan) == 0


def test_row_and_layer_scaling_are_exact():
    rng = np.random.default_rng(0)
    a = np.maximum(rng.standard_normal((16, 128)).astype(np.float32), 0) * np.float32(37.0)
    for sh in (-20, 0, 9, 30):
        xs = a * np.float32(2.0 ** sh)
        assert np.array_equal(xs / np.float32(2.0 ** sh), a)                 # a power of two commutes exactly
    # the row scale commutes with the GEMM: scaling a row by 2^s scales its outputs by exactly 2^s
    w = rng.standard_normal((128, 128)).astype(np.float32)
    y = a.astype(np.float64) @ w.T.astype(np.float64)
    assert np.array_equal(((a * np.float32(8.0)).astype(np.float64) @ w.T.astype(np.float64)), y * 8.0)


@pytest.mark.parametrize("scale", [1e-3, 1e-1, 1.0, 1e1, 1e3])
@pytest.mark.parametrize("K", [16 * 9, 64 * 9, 128, 256 * 9])
def test_three_product_gemm_error(scale, K):
    """The 3-product GEMM at G-Net shapes against float64: within 2^-20 of sum |a||w| per output."""
    rng = np.random.default_rng(K)
    a = (scale * rng.standard_normal((64, K))).astype(np.float32)
    a[a < 0] *= 0.1                                          # post-ReLU-like rows are skewed, not symmetric
    w = (rng.uniform(-1, 1, (128, K)) / np.sqrt(K)).astype(np.float32)
    sa = np.array([shift(np.abs(r).max()) for r in a])
    sw = shift(np.abs(w).max())
    got = gemm3(a, sa, w, sw)
    want = a.astype(np.float64) @ w.T.astype(np.float64)
    bound = np.abs(a).astype(np.float64) @ np.abs(w).T.astype(np.float64)
    assert np.all(np.abs(got - want) <= 2.0 ** -20 * bound)


# ---- dispatch rule ------------------------------------------------------------------------------------------------
def test_dispatch_rule_truth_table_with_head_width():
    g = GNET(ch_in=8 + 4)
    cv, inv = torch.zeros(1, 8, 4, 4), torch.zeros(1, 128, 4, 4)
    with torch.no_grad():
        assert fused_gnet_applies(g, cv, inv)
        assert not fused_gnet_applies(g.gnet, cv, inv)                  # the cat data flow
        assert not fused_gnet_applies(g, cv, None)
        assert not fused_gnet_applies(g, torch.zeros(1, 0, 4, 4), inv)  # D = 0
        assert not fused_gnet_applies(g, torch.zeros(1, 257, 4, 4), inv)
        assert not fused_gnet_applies(g, torch.zeros(1, 13, 4, 4), inv)  # D above the head's 12 input channels
        wide = GNET(ch_in=300)
        assert fused_gnet_applies(wide, torch.zeros(1, 256, 4, 4), inv)
        assert not fused_gnet_applies(wide, torch.zeros(1, 257, 4, 4), inv)
        assert not fused_gnet_applies(g, cv.half(), inv)
        g.half()
        assert not fused_gnet_applies(g, cv, inv)                       # weights not fp32
        g.float()
    assert not fused_gnet_applies(g, cv, inv)                           # grad mode on, trainable parameters
    for prm in g.parameters():
        prm.requires_grad_(False)
    assert fused_gnet_applies(g, cv, inv)                               # grad mode on, nothing requires grad
    assert not fused_gnet_applies(g, cv.clone().requires_grad_(True), inv)
    assert not fused_gnet_applies(g, cv, inv.clone().requires_grad_(True))
    with torch.no_grad():
        assert fused_gnet_applies(g, cv.clone().requires_grad_(True), inv)


def test_structure_recognition():
    g = GNET(ch_in=8 + 4)
    convs = ops.gnet_head_layers(g, 8)
    assert convs == [g.gnet[0], g.gnet[2], g.gnet[4], g.gnet[6]]
    assert ops.gnet_head_layers(g.gnet, 8) == convs                     # a GNET and its Sequential
    assert ops.gnet_head_layers(g, 12) == convs and ops.gnet_head_layers(g, 13) is None
    unpadded = GNET(ch_in=8 + 4)
    unpadded.gnet[0] = nn.Conv2d(12, 128, 3, padding=0)
    assert ops.gnet_head_layers(unpadded, 8) is None
    with torch.no_grad():
        assert not fused_gnet_applies(unpadded, torch.zeros(1, 8, 4, 4), torch.zeros(1, 128, 4, 4))
    # refused on the CPU, before any device check
    with pytest.raises(_lib.MagnetError, match="not a G-Net head"):
        ops.pack_gnet_weights(unpadded, 8)
    with pytest.raises(_lib.MagnetError, match="not a G-Net head"):
        ops.gnet_head_train(torch.zeros(1, 8, 4, 4), torch.zeros(1, 128, 4, 4), unpadded, torch.zeros(1, 2, 4, 4))
