"""The float64 restatements of tests/aux_ref.py against float64 autograd of the ATen port (oracle/torch_ref.py) and of
the loss expressions (utils/losses.py:34-50, train_FNet.py:96-108), at 1e-12 of each output's bound, on shrunk copies of
the shapes tests/test_gpu_aux_f64.py runs on the device.  CPU only."""
import numpy as np
import pytest
import torch

from oracle import magnet_oracle as mo
from oracle import torch_ref
from tests import aux_ref as ar

REL = 1e-12


def _close(got, want, bound, what):
    got, want, bound = (torch.as_tensor(x, dtype=torch.float64) for x in (got, want, bound))
    assert got.shape == want.shape, (what, got.shape, want.shape)
    err = (got - want).abs()
    assert torch.isfinite(got).all(), what
    assert (err <= REL * bound).all(), (what, float((err / bound.clamp_min(1e-300)).max()))


UPSAMPLE = [dict(B=2, H=1, W=1, k=1, CH=1), dict(B=1, H=1, W=9, k=8, CH=2), dict(B=3, H=7, W=1, k=2, CH=1),
            dict(B=2, H=5, W=7, k=4, CH=2, spread=60.0), dict(B=2, H=6, W=6, k=4, CH=1),
            dict(B=2, H=4, W=5, k=8, CH=1, spread=60.0), dict(B=2, H=6, W=8, k=4, CH=2, neg=True)]


@pytest.mark.parametrize("case", UPSAMPLE, ids=lambda c: "_".join(f"{k}{v}" for k, v in c.items()))
def test_convex_upsample(case):
    k = case["k"]
    preds, lg, _, _, _ = ar.upsample_inputs(**case, seed=3)
    depth = preds[0].double().requires_grad_()
    mask = lg.double().requires_grad_()
    out = torch_ref.convex_upsample(depth, mask, k)
    gout = torch.randn(out.shape, generator=torch.Generator().manual_seed(4), dtype=torch.float64)
    out.backward(gout)
    want, bound = ar.convex_upsample(depth, mask, k)
    _close(want, out.detach(), bound, "out")
    gd, bd, gm, bm = ar.convex_upsample_bwd(gout, depth, mask, k)
    _close(gd, depth.grad, bd, "grad_depth")
    _close(gm, mask.grad, bm, "grad_mask")
    assert (bound >= want.abs()).all() and (bd >= gd.abs()).all()


def _nll_autograd(preds, mask, gt, gtm, k, gamma):
    """MagnetLoss 'gaussian' (utils/losses.py:34-50) in float64 on torch_ref.convex_upsample of every prediction."""
    loss = 0.0
    n = len(preds)
    for i, p in enumerate(preds):
        up = torch_ref.convex_upsample(p, mask, k)
        mu, sg = up[:, 0:1][gtm], up[:, 1:2][gtm]
        var = torch.square(sg)
        var = torch.where(var < 1e-10, torch.full_like(var, 1e-10), var)
        nll = torch.square(mu - gt[gtm]) / (2 * var) + 0.5 * torch.log(var)
        loss = loss + gamma ** (n - i - 1) * nll.mean()
    return loss


NLL = [dict(B=2, H=1, W=1, k=1, n=1), dict(B=1, H=1, W=9, k=4, n=2, mask="sparse", neg=True),
       dict(B=3, H=7, W=1, k=8, n=1, tiny=2), dict(B=2, H=5, W=7, k=4, n=3, mask="last", spread=60.0),
       dict(B=2, H=6, W=6, k=4, n=4, empty=True, tiny=3, neg=True), dict(B=2, H=5, W=6, k=2, n=2, mask="sparse",
                                                                      tiny=2)]


@pytest.mark.parametrize("case", NLL, ids=lambda c: "_".join(f"{k}{v}" for k, v in c.items()))
def test_upsample_nll(case):
    k = case["k"]
    preds, lg, gt, gtm, clamped = ar.upsample_inputs(**case, seed=5)
    preds = [p.double().requires_grad_() for p in preds]
    mask = lg.double().requires_grad_()
    loss = _nll_autograd(preds, mask, gt.double(), gtm, k, 0.8)
    loss.backward()
    r = ar.upsample_nll(preds, mask, gt, gtm, k)
    assert abs(r["loss"] - float(loss.detach())) <= REL * r["loss_bound"]
    for i, p in enumerate(preds):
        _close(r["grad_preds"][i], p.grad, r["grad_preds_bound"][i], f"grad_pred{i}")
    _close(r["grad_mask"], mask.grad, r["grad_mask_bound"], "grad_mask")
    if case.get("tiny"):
        assert clamped.any()


@pytest.mark.parametrize("B,H,W", [(1, 1, 1), (3, 5, 7), (16, 3, 29)])
def test_gaussian_update(B, H, W):
    g = torch.Generator().manual_seed(B)
    dout = torch.randn(B, 2, H, W, generator=g, dtype=torch.float64)
    dout[:, 1] = 40.0 * torch.rand(B, H, W, generator=g, dtype=torch.float64) - 20.0
    dout[0, 1, 0, 0] = 0.0
    if W > 2:
        dout[0, 1, 0, 1:3] = torch.tensor([-110.0, -200.0])
    gmm0 = torch.rand(B, 2, H, W, generator=g, dtype=torch.float64) + 0.1
    gout = torch.randn(B, 2, H, W, generator=g, dtype=torch.float64)
    x = dout.clone().requires_grad_()
    out = torch_ref.gaussian_update(x, gmm0)
    out.backward(gout)
    want, bound, grad, gbound = ar.gaussian_update(dout, gmm0, gout)
    _close(want, out.detach(), bound, "out")
    _close(grad, x.grad, gbound, "grad")


FNET = [dict(B=2, D=1, H=3, W=5, scale=1.0), dict(B=1, D=2, H=4, W=4, scale=1e-2), dict(B=2, D=5, H=5, W=7, scale=1e2),
        dict(B=2, D=80, H=4, W=6, scale=1.0), dict(B=1, D=256, H=3, W=3, scale=10.0)]


@pytest.mark.parametrize("case", FNET, ids=lambda c: "_".join(f"{k}{v}" for k, v in c.items()))
def test_fnet_l1(case):
    scores, planes, gt, mask = ar.fnet_inputs(**case, seed=7)
    s = scores.double().requires_grad_()
    p = torch.softmax(s, 1)
    pred = (p * planes.double().view(1, -1, 1, 1)).sum(1, keepdim=True)
    loss = torch.abs(pred[mask] - gt.double()[mask]).mean()
    loss.backward()
    r = ar.fnet_l1(scores, planes, gt, mask)
    assert abs(r["loss"] - float(loss.detach())) <= REL * r["loss_bound"]
    _close(r["grad"], s.grad, r["grad_bound"], "grad")


def test_fnet_l1_exact_tie():
    """pred == gt: torch's abs backward gives sign(0) = 0, so does the restatement (and its bound is zero)."""
    scores = torch.zeros(1, 4, 1, 2)
    planes = torch.tensor([1.0, 2.0, 3.0, 4.0])
    gt = torch.tensor([2.5, 1.0]).view(1, 1, 1, 2)
    r = ar.fnet_l1(scores, planes, gt, torch.ones(1, 1, 1, 2, dtype=torch.bool))
    assert (r["grad"][..., 0] == 0).all() and (r["grad_bound"][..., 0] == 0).all()
    assert (r["grad"][..., 1] != 0).all()


def test_relative_poses_reference_and_gj_emulation():
    """The float64 product is np.linalg.inv's; the fp32 emulation of the kernel's pivoted Gauss-Jordan inverse meets
    the same tolerance the device test applies (and is finite on the axis turns, where the diagonal has zeros)."""
    er, en = ar.pose_inputs(6, 5, 1e3, seed=11, nan_ref=(2,), nan_nghbr=((1, 4),))
    want, absprod = ar.relative_poses(er, en)
    ref32, valid = mo.relative_poses(er, en)
    assert np.isnan(want[2]).all() and (valid[2] == 0).all() and valid[4, 1] == 0 and valid.sum() == 6 * 5 - 5 - 1
    for b in range(6):
        if b == 2:
            continue
        emu_inv = ar.gj_inverse_f32(er[b])
        assert np.isfinite(emu_inv).all()
        for v in range(5):
            if valid[b, v]:
                np.testing.assert_allclose(want[b, v], en[v, b].astype(np.float64) @ np.linalg.inv(er[b].astype(
                    np.float64)), rtol=0, atol=1e-9)
                emu = np.stack([[np.float32(sum(np.float64(en[v, b, i, q]) * emu_inv[q, j] for q in range(4)))
                                 for j in range(4)] for i in range(4)])
                tol = ar.pose_tolerance(want[b:b + 1, v:v + 1], ref32[b:b + 1, v:v + 1], absprod[b:b + 1, v:v + 1],
                                        8.0)[0, 0]
                assert (np.abs(emu - want[b, v]) <= tol).all(), (b, v)


def test_pack_cameras_reference():
    rng = np.random.default_rng(2)
    K = rng.uniform(-500, 500, (2, 3, 3))
    R, t = rng.normal(size=(2, 3, 3, 3)), rng.normal(size=(2, 3, 3))
    cams, bound = ar.pack_cameras(K, R, t, np.array([[1, 0, 1], [1, 1, 0]]))
    assert (cams[:, 0] == [1, 0, 1, 1, 1, 0]).all()
    np.testing.assert_allclose(cams[4, 4:13], (K[1] @ R[1, 1]).reshape(-1), rtol=1e-14)
    np.testing.assert_allclose(cams[4, 1:4], K[1] @ t[1, 1], rtol=1e-14)
    assert (bound[:, 1:13] >= np.abs(cams[:, 1:13])).all()


def test_sample_depths_two_roundings():
    """mu + sigma k in fp32 with the product rounded first: differs from a single-rounding fma on some elements."""
    rng = np.random.default_rng(3)
    gmm = rng.uniform(0.1, 10, (2, 2, 5, 7)).astype(np.float32)
    k = rng.normal(size=9).astype(np.float32)
    got = ar.sample_depths_f32(gmm, k)
    want = gmm[:, 0:1].astype(np.float64) + (gmm[:, 1:2].astype(np.float64) * k.reshape(1, -1, 1, 1)).astype(
        np.float32)
    assert (got == want.astype(np.float32)).all()
