"""The SPLIT16 weight packs of the fused heads, byte for byte, against a numpy restatement of the format (DESIGN §3.16):
the G-Net pack for D from 1 to 256 and its training pack, the mask pack and its training pack, and the D-Net pack with
and without the mask head.  Weights: seeded random, all zero, all fp32-subnormal, scaled by 1e-36 (the shift clamps at
+100) and by 1e36 (the shift clamps at -100 and hi overflows), holding +-inf and NaN (which must not set the scale), and
one mix of those across the layers.  Bytes the pack does not own keep the buffer's fill.  The only freedom is a NaN
half: where the restatement's half is a NaN the device's must be one too."""
import ctypes as C

import numpy as np
import pytest
import torch

from magnet_b200 import _lib
from magnet_b200._lib import check, lib
from tests import head_ref as hr

HID = 128
FILL = 0xA5                                   # the buffer's bytes before the pack


# ---- the format ------------------------------------------------------------------------------------------------------
def _shift(w):
    """split16_shift of the largest finite |w|."""
    a = np.abs(np.asarray(w, np.float32))
    a = a[np.isfinite(a)]
    return hr.shift(a.max() if a.size else 0.0)


def _frags(bmat, sh):
    """B fragments of bmat (K, N) in MMA order: per (K step, n8 tile) 32 lanes x {hi b0, hi b1, lo b0, lo b1}, n = 8 tile
    + lane / 4, k = 16 step + 2 (lane % 4) + {0, 1, 8, 9}."""
    K, N = bmat.shape
    with np.errstate(over="ignore", invalid="ignore"):                # hi overflows, inf - inf
        hi, lo = hr.split(np.asarray(bmat, np.float32), sh)
    lane = np.arange(32)
    kidx = 2 * (lane % 4)[:, None] + np.array([0, 1, 8, 9])            # (32, 4)
    gidx = (lane // 4)[:, None]
    sel = lambda x: x.reshape(K // 16, 16, N // 8, 8).transpose(0, 2, 1, 3)[:, :, kidx, gidx]   # (steps, tiles, 32, 4)
    return np.concatenate([sel(hi), sel(lo)], -1).tobytes()


def _conv3x3(w0, D):
    """The 3x3 weights (128, D, 3, 3) as one (K, 128) matrix: K step cs 9 + tap, k = 16 cs + kk holds channel c = 16 cs
    + kk, zero for c >= D."""
    cs = -(-D // 16)
    w = np.zeros((HID, 16 * cs, 9), np.float32)
    w[:, :D] = w0.reshape(HID, D, 9)
    return w.reshape(HID, cs, 16, 9).transpose(1, 3, 2, 0).reshape(cs * 9 * 16, HID)


class _Pack:
    """The bytes of a pack, and which of them are fp16 fragments."""
    def __init__(self):
        self.buf = bytearray()
        self.frag = bytearray()

    def put(self, off, data, frag=False):
        if len(self.buf) < off + len(data):
            self.frag += bytes(off + len(data) - len(self.buf))
            self.buf += bytes([FILL]) * (off + len(data) - len(self.buf))
        self.buf[off:off + len(data)] = data
        self.frag[off:off + len(data)] = bytes([frag]) * len(data)

    def frags(self, off, bmat, sh):
        """B fragments of bmat at off -> the offset after them."""
        data = _frags(bmat, sh)
        self.put(off, data, frag=True)
        return off + len(data)

    def head(self, base, mats, vecs):
        """Header shifts of `mats` at base, fp32 vectors at base + 256, B fragments of the 1x1 layers from base + 4096;
        -> the shifts."""
        shifts = [_shift(m) for m in mats]
        self.put(base, np.array(shifts, np.int32).tobytes())
        self.put(base + 256, np.concatenate([np.ravel(v) for v in vecs]).astype(np.float32).tobytes())
        return shifts


def gnet_pack(w0, w1, b1, w2, b2, w3, b3, D, train=False):
    p = _Pack()
    s0, s1, s2 = p.head(0, [w0, w1, w2], [b1, b2, w3, b3])
    w1, w2 = w1.reshape(HID, HID), w2.reshape(HID, HID)
    off = p.frags(p.frags(p.frags(4096, w1.T, s1), w2.T, s2), _conv3x3(w0, D), s0)
    if train:                                   # W1^T, W2^T
        p.frags(p.frags(off, w1, s1), w2, s2)
    return p


def mask_pack(layers, base=0, train=False, p=None):
    """layers: [(W, b)] of the hidden 128 -> 128 layers, then the 128 -> 144 layer."""
    p = p or _Pack()
    mats = [w.reshape(w.shape[0], HID) for w, _ in layers]
    shifts = p.head(base, mats, [b for _, b in layers])
    off = base + 4096
    for m, sh in zip(mats, shifts):
        off = p.frags(off, m.T, sh)
    if train:                                   # W3^T (9 K steps of the 144 logits), W2^T, W1^T
        for m, sh in zip(mats[::-1], shifts[::-1]):
            off = p.frags(off, m, sh)
    return p


def dnet_pack(dw1, db1, dw2, db2, mask=None):
    p = _Pack()
    (s1,) = p.head(0, [dw1], [db1, dw2, db2])
    off = p.frags(4096, dw1.reshape(HID, HID).T, s1)
    if mask is not None:
        mask_pack(mask, base=off, p=p)
    return p


# ---- weights ---------------------------------------------------------------------------------------------------------
KINDS = ["random", "zero", "subnormal", "tiny", "huge", "nonfinite", "mixed"]


def _mat(rng, shape, kind, slot=0):
    if kind == "mixed":
        kind = KINDS[1 + slot % 5]
    w = rng.standard_normal(shape).astype(np.float32) * np.float32(0.1)
    if kind == "zero":
        return np.zeros(shape, np.float32)
    if kind == "subnormal":
        return (w * np.float32(1e-38)).astype(np.float32)              # |w| < 2^-126
    if kind == "tiny":
        return (w * np.float32(1e-35)).astype(np.float32)
    if kind == "huge":
        return (w * np.float32(1e37)).astype(np.float32)
    if kind == "nonfinite":
        f = w.reshape(-1)
        idx = rng.choice(f.size, 6, replace=False)
        f[idx] = [np.inf, -np.inf, np.nan, np.inf, np.nan, -np.nan]
    return w


def _vec(rng, n):
    return rng.standard_normal(n).astype(np.float32)


def _check(got, want):
    """Byte for byte, except that a NaN fragment half of the restatement only asks for a NaN half."""
    got = np.frombuffer(got, np.uint8)
    ref = np.frombuffer(bytes(want.buf), np.uint8)
    assert got.size == ref.size
    nan = np.isnan(ref.view(np.float16)) & (np.frombuffer(bytes(want.frag), np.uint8)[::2] != 0)
    assert np.isnan(got.view(np.float16)[nan]).all()
    bad = np.flatnonzero((got != ref) & ~np.repeat(nan, 2))
    assert bad.size == 0, f"{bad.size} bytes differ, first at offset {bad[0]}"


def _run(fn, nbytes, arrays, *args):
    """Pack on the device from the numpy arrays (None passes NULL) into a buffer holding FILL -> the bytes."""
    dev = torch.device("cuda:0")
    ts = [None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in arrays]
    out = torch.full((nbytes,), FILL, dtype=torch.uint8, device=dev)
    check(fn(*[None if t is None else t.data_ptr() for t in ts], *args, out.data_ptr(), None), "pack")
    torch.cuda.synchronize()
    return out.cpu().numpy().tobytes()


def _gnet_ws(rng, D, kind):
    return (_mat(rng, (HID, D, 3, 3), kind, 0), _mat(rng, (HID, HID, 1, 1), kind, 1), _vec(rng, HID),
            _mat(rng, (HID, HID, 1, 1), kind, 2), _vec(rng, HID), _mat(rng, (2, HID, 1, 1), kind, 3), _vec(rng, 2))


def _mask_layers(rng, kind, nhid):
    return ([(_mat(rng, (HID, HID, 1, 1), kind, i), _vec(rng, HID)) for i in range(nhid)]
            + [(_mat(rng, (144, HID, 1, 1), kind, nhid), _vec(rng, 144))])


# ---- tests -----------------------------------------------------------------------------------------------------------
def test_reference_sizes_match_the_library():
    L = lib()
    rng = np.random.default_rng(0)
    for D in (1, 15, 16, 17, 64, 256):
        ws = _gnet_ws(rng, D, "zero")
        assert len(gnet_pack(*ws, D).buf) == L.magnet_gnet_weights_bytes(D)
        assert len(gnet_pack(*ws, D, train=True).buf) == L.magnet_gnet_train_weights_bytes(D)
    layers = _mask_layers(rng, "zero", 2)
    assert len(mask_pack(layers).buf) == L.magnet_mask_weights_bytes(4)
    assert len(mask_pack(layers, train=True).buf) == L.magnet_mask_train_weights_bytes(4)
    d = (_mat(rng, (HID, HID, 1, 1), "zero"), _vec(rng, HID), _mat(rng, (2, HID, 1, 1), "zero"), _vec(rng, 2))
    assert len(dnet_pack(*d).buf) == L.magnet_dnet_weights_bytes(0)
    assert len(dnet_pack(*d, mask=_mask_layers(rng, "zero", 1)).buf) == L.magnet_dnet_weights_bytes(4)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("D", [1, 15, 16, 17, 64, 256])
def test_gnet_pack_bytes(cuda, D, kind):
    L = lib()
    ws = _gnet_ws(np.random.default_rng(D), D, kind)
    inf = _run(L.magnet_gnet_pack_weights_f32, L.magnet_gnet_weights_bytes(D), ws, D)
    _check(inf, gnet_pack(*ws, D))
    if D in (17, 64):
        train = _run(L.magnet_gnet_pack_train_weights_f32, L.magnet_gnet_train_weights_bytes(D), ws, D)
        _check(train, gnet_pack(*ws, D, train=True))
        assert train[:len(inf)] == inf


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_mask_pack_bytes(cuda, kind):
    L = lib()
    layers = _mask_layers(np.random.default_rng(1), kind, 2)
    arrays = [a for wb in layers for a in wb]
    inf = _run(L.magnet_mask_pack_weights_f32, L.magnet_mask_weights_bytes(4), arrays)
    _check(inf, mask_pack(layers))
    train = _run(L.magnet_mask_pack_train_weights_f32, L.magnet_mask_train_weights_bytes(4), arrays)
    _check(train, mask_pack(layers, train=True))
    assert train[:len(inf)] == inf


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_dnet_pack_bytes(cuda, kind):
    L = lib()
    rng = np.random.default_rng(2)
    d = (_mat(rng, (HID, HID, 1, 1), kind, 0), _vec(rng, HID), _mat(rng, (2, HID, 1, 1), kind, 1), _vec(rng, 2))
    m = _mask_layers(rng, kind, 1)
    k0 = _run(L.magnet_dnet_pack_weights_f32, L.magnet_dnet_weights_bytes(0), [*d, None, None, None, None], 0)
    _check(k0, dnet_pack(*d))
    k4 = _run(L.magnet_dnet_pack_weights_f32, L.magnet_dnet_weights_bytes(4), [*d, *[a for wb in m for a in wb]], 4)
    _check(k4, dnet_pack(*d, mask=m))
    assert k4[:len(k0)] == k0
