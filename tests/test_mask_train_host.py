"""CPU-side tests of the fused mask-head training loss (DESIGN §3.13): C-ABI argument checks (no launch), the size
formulas, the dispatch rule of MagnetHead.train_loss, and a numpy restatement of the forward kernel's per-sub-pixel
order of operations against float64 autograd of the upsampling and the NLL."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn as nn

from magnet_b200 import _lib
from magnet_b200.matcher import MagnetHead, fused_mask_trains
from tests.mask_train_ref import loss64, subpixel_grads


def _aligned():
    buf = (C.c_float * 64)()
    base = C.addressof(buf)
    base += (-base) % 16
    return buf, base


def _args(p, P=1, B=1, H=4, W=4, k=4, preds=None):
    n = max(P, 1)
    pp = (C.c_void_p * n)(*([p] * n if preds is None else preds))
    sc = (C.c_float * n)(*([1.0] * n))
    a = _lib.MaskTrainArgs(P=P, B=B, H=H, W=W, k=k, pre0=p, packed_weights=p, pred=C.cast(pp, C.POINTER(C.c_void_p)),
                           gt=p, gt_mask=p, pred_scale=C.cast(sc, C.POINTER(C.c_float)), partial=p, saved=p,
                           grad_scale=p, workspace=p)
    return a, (pp, sc)


def test_mask_train_entry_points_validate_without_launching():
    L = _lib.lib()
    buf, p = _aligned()
    odd = p + 4
    for run in (lambda a: L.magnet_mask_train_fwd_f32(C.byref(a), None),
                lambda a: L.magnet_mask_bwd_f32(C.byref(a), None)):
        for shape in ((1, 0, 4, 4), (1, 1, 0, 4), (1, 1, 4, 0)):
            a, keep = _args(p, *shape)
            assert run(a) == _lib.ERR_SHAPE
        a, keep = _args(p, B=2048, H=1024, W=1024)                   # B*H*W = 2^31
        assert run(a) == _lib.ERR_SHAPE
        for P, k in ((0, 4), (9, 4), (1, 2), (1, 8)):
            a, keep = _args(p, P=P, k=k)
            assert run(a) == _lib.ERR_UNSUPPORTED
        for field in ("packed_weights", "saved"):
            a, keep = _args(p)
            setattr(a, field, None)
            assert run(a) == _lib.ERR_NULL
            setattr(a, field, odd)
            assert run(a) == _lib.ERR_ALIGN
    assert L.magnet_mask_train_fwd_f32(None, None) == _lib.ERR_NULL
    assert L.magnet_mask_bwd_f32(None, None) == _lib.ERR_NULL
    fwd = lambda a: L.magnet_mask_train_fwd_f32(C.byref(a), None)
    for field in ("pre0", "gt", "gt_mask", "partial", "pred_scale", "pred"):
        a, keep = _args(p)
        setattr(a, field, None)
        assert fwd(a) == _lib.ERR_NULL
    a, keep = _args(p, P=3, preds=[p, None, p])
    assert fwd(a) == _lib.ERR_NULL
    a, keep = _args(p)
    a.pre0 = odd
    assert fwd(a) == _lib.ERR_ALIGN
    a, keep = _args(p, P=2, preds=[p, odd])
    assert fwd(a) == _lib.ERR_ALIGN
    bwd = lambda a: L.magnet_mask_bwd_f32(C.byref(a), None)
    for field in ("grad_scale", "workspace"):
        a, keep = _args(p)
        setattr(a, field, None)
        assert bwd(a) == _lib.ERR_NULL
    a, keep = _args(p)
    a.workspace = odd
    assert bwd(a) == _lib.ERR_ALIGN
    pack = L.magnet_mask_pack_train_weights_f32
    assert pack(*([p] * 6), None, None) == _lib.ERR_NULL
    assert pack(None, *([p] * 6), None) == _lib.ERR_NULL
    assert pack(*([p] * 6), odd, None) == _lib.ERR_ALIGN


def test_size_formulas():
    L = _lib.lib()
    # the inference pack, then W3^T (9 K steps x 16 n8 tiles), W2^T and W1^T (8 x 16 each), 32 lanes x 16 bytes
    assert L.magnet_mask_train_weights_bytes(4) == L.magnet_mask_weights_bytes(4) + (9 + 8 + 8) * 16 * 32 * 16
    for k in (0, 2, 8):
        assert L.magnet_mask_train_weights_bytes(k) == 0
    # h0, h1, h2, the 144 logit gradients and P prediction gradients, per pixel
    for P, B, H, W in ((1, 1, 1, 1), (3, 8, 120, 160), (8, 4, 88, 304)):
        assert L.magnet_mask_saved_bytes(P, B, H, W) == (3 * 128 + 144 + 2 * P) * B * H * W * 4
        assert L.magnet_mask_train_partials(B, H, W) == B * -(-H // 8) * -(-W // 16)
        map_ = B * H * W * 4
        chunks = -(-B * H * W // 1024)
        assert L.magnet_mask_bwd_workspace_bytes(B, H, W) == -(-2 * 128 * map_ // 256) * 256 + chunks * 128 * 129 * 4
    assert L.magnet_mask_saved_bytes(0, 1, 4, 4) == 0 and L.magnet_mask_saved_bytes(9, 1, 4, 4) == 0
    assert L.magnet_mask_saved_bytes(1, 0, 4, 4) == 0 and L.magnet_mask_bwd_workspace_bytes(1, 4, 0) == 0
    assert L.magnet_mask_train_partials(0, 4, 4) == _lib.ERR_SHAPE


def test_dispatch_rule_truth_table():
    mh = MagnetHead(dnet_fdim=8).mask_head
    pre0, preds = torch.zeros(1, 128, 4, 4), [torch.zeros(1, 2, 4, 4) for _ in range(3)]
    gt = torch.zeros(1, 1, 16, 16)
    assert fused_mask_trains(mh, pre0, preds, 4, gt)                    # grad mode on, trainable parameters
    assert fused_mask_trains(mh, None, preds, 4)
    assert fused_mask_trains(mh, pre0, preds[0], 4)
    assert not fused_mask_trains(mh, pre0, preds, 2)                    # k != 4
    assert not fused_mask_trains(mh, pre0, [], 4)
    assert not fused_mask_trains(mh, pre0, preds * 3, 4)                # 9 predictions
    assert fused_mask_trains(mh, pre0, (preds * 3)[:8], 4)
    assert not fused_mask_trains(mh[:6], pre0, preds, 4)                # not the reference's structure
    swapped = nn.Sequential(*[nn.GELU() if i == 3 else m for i, m in enumerate(mh)])
    assert not fused_mask_trains(swapped, pre0, preds, 4)
    assert not fused_mask_trains(mh, pre0.half(), preds, 4)
    assert not fused_mask_trains(mh, pre0, [preds[0], preds[1].double()], 4)
    assert not fused_mask_trains(mh, pre0, preds, 4, gt.half())
    with torch.no_grad():
        assert not fused_mask_trains(mh, pre0, preds, 4)                # nothing to differentiate
    mh.half()
    assert not fused_mask_trains(mh, pre0, preds, 4)                    # weights not fp32
    mh.float()
    if torch.cuda.is_available():
        with torch.autocast("cuda"):
            assert not fused_mask_trains(mh, pre0, preds, 4)
    for prm in mh.parameters():
        prm.requires_grad_(False)
    assert not fused_mask_trains(mh, pre0, preds, 4)                    # nothing requires grad
    assert fused_mask_trains(mh, pre0, [preds[0], preds[1].clone().requires_grad_(True)], 4)
    assert fused_mask_trains(mh, pre0.clone().requires_grad_(True), preds, 4)


# ---- numpy restatement of the forward kernel's per-sub-pixel arithmetic ---------------------------------------------
@pytest.mark.parametrize("case", ["interior", "border", "clamp"])
@pytest.mark.parametrize("P", [1, 3])
def test_subpixel_order_of_operations_against_float64(case, P):
    """One supervised sub-pixel: the kernel's fp32 d_logits and neighbourhood gradients against float64 autograd of
    softmax -> convex combination -> NLL, within 2^-18 of the scale of the terms (sum over predictions of
    |scale| sum_i w_i (|g_mu a_i| + |g_sigma c_i|) / var-normalised), and the clamp's cut of the sigma gradient."""
    rng = np.random.default_rng(P * 10 + len(case))
    logits = rng.standard_normal(9).astype(np.float32)
    taps = [np.stack([1 + rng.random(9), 0.1 + 0.5 * rng.random(9)], 1).astype(np.float32) for _ in range(P)]
    if case == "clamp":
        taps[0][:, 1] = 1e-6
    valid = np.ones(9, bool)
    if case == "border":
        valid[[0, 3, 6]] = False                                        # left column outside the image
        for t in taps:
            t[~valid] = 0
    gt = np.float32(1.4)
    gammas = [0.8 ** (P - i - 1) for i in range(P)]
    count = 37
    scales = [np.float32(g / count) for g in gammas]
    dl, pg = subpixel_grads(logits, taps, valid, gt, scales)

    lg = torch.tensor(logits, dtype=torch.float64, requires_grad=True)
    tt = [torch.tensor(t, dtype=torch.float64, requires_grad=True) for t in taps]
    w = torch.softmax(lg, 0)
    vm = torch.tensor(valid, dtype=torch.float64)
    loss = 0.0
    for i, t in enumerate(tt):
        mu, sg = (w * vm * t[:, 0]).sum(), (w * vm * t[:, 1]).sum()
        var = torch.where(sg * sg < 1e-10, torch.full_like(sg, 1e-10), sg * sg)
        loss = loss + gammas[i] / count * ((mu - float(gt)) ** 2 / (2 * var) + 0.5 * torch.log(var))
    grads = torch.autograd.grad(loss, [lg] + tt)
    want_dl = grads[0].numpy()
    scale = float(np.abs(want_dl).max()) + max(float(g.abs().max()) for g in grads[1:])
    assert np.all(np.abs(dl - want_dl) <= 2.0 ** -18 * scale)
    for (g_mu, g_sg), want in zip(pg, grads[1:]):
        want = want.numpy()
        assert np.all(np.abs(g_mu - want[:, 0]) <= 2.0 ** -18 * scale)
        assert np.all(np.abs(g_sg - want[:, 1]) <= 2.0 ** -18 * scale)
    if case == "clamp":
        assert np.all(pg[0][1] == 0)                                    # no sigma gradient where var clamps


def test_float64_reference_is_the_module_chain():
    """loss64 restates mask_head(pre0 path) -> upsample_depth_via_mask -> MagnetLoss: compared with the reference's
    view-based upsampling written out, on CPU in float64."""
    torch.manual_seed(0)
    B, H, W = 2, 3, 5
    mh = MagnetHead(dnet_fdim=8).mask_head.double()
    pre0 = torch.randn(B, 128, H, W, dtype=torch.float64)
    preds = [torch.rand(B, 2, H, W, dtype=torch.float64) + 0.5 for _ in range(2)]
    gt = torch.rand(B, 1, 4 * H, 4 * W, dtype=torch.float64) + 1
    gtm = torch.rand(B, 1, 4 * H, 4 * W) < 0.5
    ws = [mh[2].weight, mh[2].bias, mh[4].weight, mh[4].bias, mh[6].weight, mh[6].bias]
    got, _ = loss64(pre0, ws, preds, gt, gtm)
    mask = mh[6](mh[5](mh[4](mh[3](mh[2](torch.relu(pre0))))))
    want = 0.0
    for i, p in enumerate(preds):
        m = mask.view(B, 1, 9, 4, 4, H, W).softmax(2)
        u = torch.nn.functional.unfold(p, [3, 3], padding=1).view(B, 2, 9, 1, 1, H, W)
        up = (m * u).sum(2).permute(0, 1, 4, 2, 5, 3).reshape(B, 2, 4 * H, 4 * W)
        mu, sg = up[:, :1], up[:, 1:]
        var = sg ** 2
        var[var < 1e-10] = 1e-10
        nll = (mu - gt) ** 2 / (2 * var) + 0.5 * torch.log(var)
        want = want + 0.8 ** (1 - i) * nll[gtm].mean()
    assert torch.allclose(got, want, rtol=1e-12)
