"""CPU-side tests of the fused mask head and upsampling (DESIGN §3.12): C-ABI argument checks (no launch), the
packed-weight size, the dispatch rule of MagnetHead.forward, the kernel's mapping of n8 tiles to (tap, sub-pixel) and
the three-product error of the 144-column layer."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn as nn

from magnet_b200 import _lib, ops
from magnet_b200.matcher import MagnetHead, fused_mask_applies
from tests.head_ref import shift, split


def _args(P=1, B=1, H=4, W=4, k=4, ptr=None, preds=None, outs=None):
    n = max(P, 1)
    pp = (C.c_void_p * n)(*([ptr] * n if preds is None else preds))
    op = (C.c_void_p * n)(*([ptr] * n if outs is None else outs))
    a = _lib.MaskUpsampleArgs(P=P, B=B, H=H, W=W, k=k, pre0=ptr, packed_weights=ptr,
                              pred=C.cast(pp, C.POINTER(C.c_void_p)), out=C.cast(op, C.POINTER(C.c_void_p)))
    return a, (pp, op)


def test_mask_entry_points_validate_without_launching():
    L = _lib.lib()
    buf = (C.c_float * 64)()
    base = C.addressof(buf)
    base += (-base) % 16
    p, odd = base, base + 4
    run = lambda a: L.magnet_mask_upsample_f32(C.byref(a), None)
    assert L.magnet_mask_upsample_f32(None, None) == _lib.ERR_NULL
    for shape in ((1, 0, 4, 4), (1, 1, 0, 4), (1, 1, 4, 0)):
        a, keep = _args(*shape, ptr=p)
        assert run(a) == _lib.ERR_SHAPE
    a, keep = _args(B=2048, H=1024, W=1024, ptr=p)                       # B*H*W = 2^31
    assert run(a) == _lib.ERR_SHAPE
    for P, k in ((0, 4), (9, 4), (1, 2), (1, 8)):
        a, keep = _args(P=P, k=k, ptr=p)
        assert run(a) == _lib.ERR_UNSUPPORTED
    a, keep = _args(ptr=None)
    assert run(a) == _lib.ERR_NULL
    a, keep = _args(P=3, ptr=p, preds=[p, None, p])
    assert run(a) == _lib.ERR_NULL
    a, keep = _args(P=2, ptr=p, outs=[p, None])
    assert run(a) == _lib.ERR_NULL
    a, keep = _args(ptr=p)
    a.pre0 = odd
    assert run(a) == _lib.ERR_ALIGN
    a, keep = _args(ptr=p)
    a.packed_weights = odd
    assert run(a) == _lib.ERR_ALIGN
    a, keep = _args(P=2, ptr=p, preds=[p, odd])
    assert run(a) == _lib.ERR_ALIGN
    a, keep = _args(P=2, ptr=p, outs=[odd, p])
    assert run(a) == _lib.ERR_ALIGN
    pack = L.magnet_mask_pack_weights_f32
    assert pack(*([p] * 6), None, None) == _lib.ERR_NULL
    assert pack(None, *([p] * 6), None) == _lib.ERR_NULL
    assert pack(*([p] * 6), odd, None) == _lib.ERR_ALIGN


def test_mask_weights_bytes_formula():
    L = _lib.lib()
    # 4 KiB of header and fp32 vectors, W1 and W2 as 64 KiB of hi/lo fragments each, W3 as 8 K steps x 18 n8 tiles x
    # 32 lanes x 16 bytes
    assert L.magnet_mask_weights_bytes(4) == 4096 + 2 * 65536 + 8 * 18 * 32 * 16
    for k in (0, 1, 2, 3, 5, 8, -4):
        assert L.magnet_mask_weights_bytes(k) == 0
    assert ops.mask_weights_bytes(4) == 208896


# ---- dispatch rule ------------------------------------------------------------------------------------------------
def test_dispatch_rule_truth_table():
    mh = MagnetHead(dnet_fdim=8).mask_head
    pre0, preds = torch.zeros(1, 128, 4, 4), [torch.zeros(1, 2, 4, 4) for _ in range(3)]
    with torch.no_grad():
        assert fused_mask_applies(mh, pre0, preds, 4)
        assert fused_mask_applies(mh, None, preds, 4)
        assert fused_mask_applies(mh, pre0, preds[0], 4)
        assert not fused_mask_applies(mh, pre0, preds, 2)                # k != 4
        assert not fused_mask_applies(MagnetHead(dnet_fdim=8, downsample_ratio=2).mask_head, pre0, preds, 2)
        assert not fused_mask_applies(mh[:6], pre0, preds, 4)             # not the reference's structure
        swapped = nn.Sequential(*[nn.GELU() if i == 3 else m for i, m in enumerate(mh)])
        assert not fused_mask_applies(swapped, pre0, preds, 4)
        wide = MagnetHead(dnet_fdim=8).mask_head
        wide[0] = nn.Conv2d(8, 128, 5, padding=2)
        assert not fused_mask_applies(wide, pre0, preds, 4)
        assert not fused_mask_applies(mh, pre0.half(), preds, 4)
        assert not fused_mask_applies(mh, pre0, [preds[0], preds[1].double()], 4)
        mh.half()
        assert not fused_mask_applies(mh, pre0, preds, 4)                # weights not fp32
        mh.float()
        if torch.cuda.is_available():
            with torch.autocast("cuda"):
                assert not fused_mask_applies(mh, pre0, preds, 4)
    assert not fused_mask_applies(mh, pre0, preds, 4)                    # grad mode on, trainable parameters
    for prm in mh.parameters():
        prm.requires_grad_(False)
    assert fused_mask_applies(mh, pre0, preds, 4)                        # grad mode on, nothing requires grad
    assert not fused_mask_applies(mh, pre0, [preds[0], preds[1].clone().requires_grad_(True)], 4)
    assert not fused_mask_applies(mh, pre0.clone().requires_grad_(True), preds, 4)
    with torch.no_grad():
        assert fused_mask_applies(mh, pre0.clone().requires_grad_(True), preds, 4)


def test_fused_upsample_defaults_off():
    assert MagnetHead(dnet_fdim=8).fused_upsample is False
    assert MagnetHead(dnet_fdim=8, fused_upsample=True).fused_upsample is True


# ---- the kernel's mapping of the 144 channels -----------------------------------------------------------------------
def test_tile_mapping_matches_the_reference_view():
    """Channel c = 8 t + n of n8 tile t = 2 i + h is tap i of sub-pixel s = 8 h + n, (ky, kx) = divmod(s, 4), as the
    view (N, 1, 9, 4, 4, H, W) of upsample_depth_via_mask reads it; lane q of the MMA fragment holds columns n = 2q + e,
    so its sub-pixels lie on row ky = 2h + q // 2, columns kx = 2 (q % 2) + e."""
    N, H, W = 2, 3, 5
    mask = torch.arange(N * 144 * H * W, dtype=torch.float64).view(N, 144, H, W)
    v = mask.view(N, 1, 9, 4, 4, H, W)
    for t in range(18):
        i, h = divmod(t, 2)
        for n in range(8):
            ky, kx = divmod(8 * h + n, 4)
            assert torch.equal(mask[:, 8 * t + n], v[:, 0, i, ky, kx])
    for h in range(2):
        for q in range(4):
            for e in range(2):
                s = 8 * h + 2 * q + e
                assert divmod(s, 4) == (2 * h + q // 2, 2 * (q % 2) + e)
    # a warp's 16 pixels x 4 columns are 64 contiguous floats of each full-resolution row: whole 32-byte sectors
    cols = sorted(4 * x + 2 * (q % 2) + e for x in range(16) for q in range(4) for e in range(2) if q // 2 == 0)
    assert cols == list(range(64))


# ---- numpy restatement of the 144-column layer's SPLIT16 numerics (tests/head_ref.shift, split) --------------------
@pytest.mark.parametrize("scale", [1e-3, 1.0, 1e3])
def test_three_product_error_of_the_mask_layer(scale):
    """h2 (M,128) post-ReLU rows with one shift each, W3 (144,128) with one shift: hi*hi + hi*lo + lo*hi in float64
    (exact products), exact descale, + b3 in fp32 -> within 2^-20 of sum |h||w| of the float64 logits."""
    rng = np.random.default_rng(int(scale * 1000) + 1)
    h = np.maximum(scale * rng.standard_normal((64, 128)), 0).astype(np.float32)
    w = (rng.uniform(-1, 1, (144, 128)) / np.sqrt(128)).astype(np.float32)
    b = rng.uniform(-0.1, 0.1, 144).astype(np.float32)
    sa = np.array([shift(r.max()) for r in h])
    sw = shift(np.abs(w).max())
    ah, al = split(h, sa[:, None])
    wh, wl = split(w, sw)
    f = lambda u: u.astype(np.float64)
    acc = f(ah) @ f(wh).T + f(ah) @ f(wl).T + f(al) @ f(wh).T
    got = (acc * 2.0 ** (-sa[:, None].astype(np.float64)) * 2.0 ** (-sw)).astype(np.float32) + b
    want = f(h) @ f(w).T + f(b)
    bound = np.abs(f(h)) @ np.abs(f(w)).T
    assert np.all(np.abs(got - want) <= 2.0 ** -20 * bound + 2.0 ** -23 * np.abs(want))
