"""CPU-side tests of the differentiable fused G-Net head (DESIGN §3.10): C-ABI argument checks (no launch), the size
formulas, the fused_train dispatch rule on stand-in tensors and a numpy restatement of the 3xTF32 weight-gradient
GEMM against float64."""
import ctypes as C

import numpy as np
import pytest
import torch

from magnet_b200 import _lib
from magnet_b200.matcher import GNET, fused_gnet_trains


def _args(p):
    a = _lib.GnetTrainArgs()
    a.B, a.D, a.H, a.W = 1, 8, 4, 4
    for f in ("cost", "invariant", "packed_weights", "prev_gmm", "scratch", "out", "saved", "grad_out", "workspace",
              "grad_invariant"):
        setattr(a, f, p)
    return a


@pytest.mark.parametrize("fn", ["magnet_gnet_train_fwd_f32", "magnet_gnet_bwd_f32"])
def test_train_entry_points_validate_without_launching(fn):
    L = _lib.lib()
    f = getattr(L, fn)
    buf = (C.c_float * 64)()
    p = C.cast(buf, C.c_void_p)
    odd = C.c_void_p(C.addressof(buf) + 4)
    n0 = L.magnet_launch_count()
    assert f(None, None) == _lib.ERR_NULL
    a = _args(p)
    a.W = 0
    assert f(C.byref(a), None) == _lib.ERR_SHAPE
    a = _args(p)
    a.D = 0
    assert f(C.byref(a), None) == _lib.ERR_SHAPE
    a.D = _lib.MAGNET_MAX_PLANES + 1
    assert f(C.byref(a), None) == _lib.ERR_UNSUPPORTED
    a = _args(p)
    a.B, a.H, a.W = 1 << 10, 1 << 11, 1 << 10                              # B*H*W = 2^31 pixels
    assert f(C.byref(a), None) == _lib.ERR_SHAPE
    for field in ("cost", "packed_weights", "prev_gmm", "saved"):
        a = _args(p)
        setattr(a, field, None)
        assert f(C.byref(a), None) == _lib.ERR_NULL, field
    for field in ("cost", "packed_weights", "saved"):
        a = _args(p)
        setattr(a, field, odd)
        assert f(C.byref(a), None) == _lib.ERR_ALIGN, field
    own = ("invariant", "scratch", "out") if fn == "magnet_gnet_train_fwd_f32" else ("grad_out", "workspace", "grad_invariant")
    for field in own:
        a = _args(p)
        setattr(a, field, None)
        assert f(C.byref(a), None) == _lib.ERR_NULL, field
    a = _args(p)
    setattr(a, "invariant" if fn == "magnet_gnet_train_fwd_f32" else "workspace", odd)
    assert f(C.byref(a), None) == _lib.ERR_ALIGN
    assert L.magnet_launch_count() == n0                                   # nothing was launched


def test_train_pack_validates_without_launching():
    L = _lib.lib()
    buf = (C.c_float * 64)()
    p = C.cast(buf, C.c_void_p)
    pack = L.magnet_gnet_pack_train_weights_f32
    n0 = L.magnet_launch_count()
    assert pack(*([p] * 7), 8, None, None) == _lib.ERR_NULL
    assert pack(None, *([p] * 6), 8, p, None) == _lib.ERR_NULL
    assert pack(*([p] * 7), 0, p, None) == _lib.ERR_SHAPE
    assert pack(*([p] * 7), 257, p, None) == _lib.ERR_UNSUPPORTED
    assert pack(*([p] * 7), 8, C.c_void_p(C.addressof(buf) + 4), None) == _lib.ERR_ALIGN
    assert L.magnet_launch_count() == n0


def test_train_size_formulas():
    L = _lib.lib()
    for D in (1, 5, 16, 17, 64, 256):
        # the inference pack, then W1^T and W2^T as 64 KiB of hi/lo fragments each
        assert L.magnet_gnet_train_weights_bytes(D) == L.magnet_gnet_weights_bytes(D) + 2 * 65536
    assert L.magnet_gnet_train_weights_bytes(0) == 0 and L.magnet_gnet_train_weights_bytes(257) == 0
    for B, H, W in ((1, 1, 1), (3, 7, 9), (8, 120, 160)):
        # h0, h1, h2 (128 channels each) and the raw (mu1, sigma1), fp32
        assert L.magnet_gnet_saved_bytes(B, H, W) == (3 * 128 + 2) * B * H * W * 4
    assert L.magnet_gnet_saved_bytes(0, 4, 4) == 0
    a256 = lambda n: -(-n // 256) * 256
    for B, D, H, W in ((1, 1, 1, 1), (3, 17, 7, 9), (8, 64, 120, 160), (4, 256, 88, 304)):
        P = B * H * W
        chunks = -(-P // 1024)
        want = a256(2 * 128 * P * 4) + a256(2 * P * 4) + a256(chunks * 128 * (max(128, 9 * D) + 1) * 4)
        assert L.magnet_gnet_bwd_workspace_bytes(B, D, H, W) == want
    assert L.magnet_gnet_bwd_workspace_bytes(1, 0, 4, 4) == 0
    assert L.magnet_gnet_bwd_workspace_bytes(1, 257, 4, 4) == 0


# ---- dispatch rule ------------------------------------------------------------------------------------------------
def test_train_dispatch_rule_truth_table():
    g = GNET(ch_in=8 + 4)
    cv, inv = torch.zeros(1, 8, 4, 4), torch.zeros(1, 128, 4, 4)
    assert fused_gnet_trains(g, cv, inv)                                # grad mode on, trainable parameters
    with torch.no_grad():
        assert not fused_gnet_trains(g, cv, inv)
    assert not fused_gnet_trains(g, cv.clone().requires_grad_(True), inv)
    assert not fused_gnet_trains(g.gnet, cv, inv)                       # the cat data flow
    assert not fused_gnet_trains(g, cv, None)
    assert not fused_gnet_trains(g, torch.zeros(1, 0, 4, 4), inv)       # D = 0
    assert not fused_gnet_trains(g, torch.zeros(1, 257, 4, 4), inv)
    assert fused_gnet_trains(g, torch.zeros(1, 256, 4, 4), inv)
    assert not fused_gnet_trains(g, cv.half(), inv)
    # (CUDA autocast cannot be entered without a GPU: its case is in test_gpu_gnet_train)
    g.half()
    assert not fused_gnet_trains(g, cv, inv)                            # weights not fp32
    g.float()
    for prm in g.parameters():
        prm.requires_grad_(False)
    assert not fused_gnet_trains(g, cv, inv)                            # nothing to train
    assert fused_gnet_trains(g, cv, inv.clone().requires_grad_(True))   # the invariant still wants a gradient


# ---- numpy restatement of the weight-gradient GEMM ----------------------------------------------------------------
def tf32(x):
    """cvt.rna.tf32.f32: round to nearest, ties away from zero, to 10 explicit mantissa bits."""
    u = np.asarray(x, np.float32).view(np.uint32).astype(np.uint64)
    r = ((u + 0x1000) & 0xFFFFE000).astype(np.uint32)
    return r.view(np.float32)


def wgrad3(a, b, kc=1024, slab=32, ks=8):
    """out[m][n] = sum_p a[p][m] b[p][n] as the kernel evaluates it: x = hi + lo (tf32 each); per slab of 32 pixels a
    fresh fp32 accumulator takes, per k8 step, the three products lo*hi, hi*lo, hi*hi (each MMA's sum of exact products
    rounded once to fp32) and is added to the CTA's running fp32 sum; the per-chunk (kc pixels) sums are then added
    in order in fp32."""
    ah = tf32(a); al = tf32(a - ah)
    bh = tf32(b); bl = tf32(b - bh)
    f = lambda u: u.astype(np.float64)
    P = a.shape[0]
    r32 = lambda x: x.astype(np.float32)
    total = np.zeros((a.shape[1], b.shape[1]), np.float32)
    for c0 in range(0, P, kc):
        tot = np.zeros_like(total)
        for s0 in range(c0, min(P, c0 + kc), slab):
            acc = np.zeros_like(total)
            for k0 in range(s0, min(P, c0 + kc, s0 + slab), ks):
                s = slice(k0, min(P, c0 + kc, k0 + ks))
                for x, y in ((al, bh), (ah, bl), (ah, bh)):
                    acc = r32(f(acc) + f(x[s]).T @ f(y[s]))
            tot = r32(f(tot) + f(acc))
        total = r32(f(total) + f(tot))
    return total


@pytest.mark.parametrize("scale", [1e-3, 1.0, 1e3])
@pytest.mark.parametrize("P", [37, 1024, 3000])
def test_three_product_tf32_wgrad_error(scale, P):
    """Against float64 within the bound of DESIGN §3.10: |err| <= (3*2^-22 + (12 + kc/32 + n_chunks) * 2^-24)
    * sum_p |a||b| per output element."""
    rng = np.random.default_rng(P)
    a = (scale * rng.standard_normal((P, 24))).astype(np.float32)
    b = np.maximum(rng.standard_normal((P, 16)), 0).astype(np.float32) * np.float32(3.0)
    b[:, 0] = 1.0                                                        # a bias column
    got = wgrad3(a, b).astype(np.float64)
    want = a.astype(np.float64).T @ b.astype(np.float64)
    absum = np.abs(a).astype(np.float64).T @ np.abs(b).astype(np.float64)
    chunks = -(-P // 1024)
    bound = (3 * 2.0 ** -22 + (12 + 1024 / 32 + chunks) * 2.0 ** -24) * absum
    assert np.all(np.abs(got - want) <= bound)
    # and far inside it in practice: the relative error of the largest entry is fp32-level
    assert np.abs(got - want).max() <= 1e-5 * np.abs(want).max()
