"""The kernels every training step runs around the cost volumes, element by element, against the float64 restatements of
tests/aux_ref.py: convex upsampling (forward and both gradients, CH 1 and 2, k 1 to 8), the fused upsample + Gaussian
NLL of magnet_loss (loss and every gradient), the Gaussian update, the F-Net soft-argmin L1 loss, the relative poses,
the camera rays, the depth sampler and the camera table.

Tolerance: |got - ref| <= c u bound, u = 2^-24, c = C_TOL = 32 for every output (the bounds and their derivation are in
aux_ref's docstring); the worst err / (u bound) is printed per output.  The relative poses are held to POSE_FACTOR times
the error of the reference's own fp32 route; the rays, the intrinsics and the sampled depths must be bit-identical.

Ambiguity is removed by construction, never budgeted: sigma is drawn away from the 1e-10 clamp (|sigma| >= 0.05) except
in the deliberately clamped 3x3 blocks (1e-7), and every full-resolution pixel whose float64 d or sigma^2 - 1e-10 lies
within c u of its own bound leaves the mask; F-Net pixels whose |pred - gt| lies within c u of the bound of pred leave
the mask, except at the deliberate exact ties (where the gradient must be exactly zero)."""
import numpy as np
import pytest
import torch

from magnet_b200 import ops
from oracle import magnet_oracle as mo
from tests import aux_ref as ar

pytestmark = pytest.mark.gpu

C_TOL = 32.0
POSE_FACTOR = 8.0


def _close(got, want, bound, what):
    got = got.detach().to(torch.float64)
    want = torch.as_tensor(want, dtype=torch.float64, device=got.device)
    bound = torch.as_tensor(bound, dtype=torch.float64, device=got.device)
    assert got.shape == want.shape, (what, tuple(got.shape), tuple(want.shape))
    assert torch.isfinite(got).all(), f"{what}: non-finite output"
    tol = C_TOL * ar.U * bound
    err = (got - want).abs()
    bad = err > tol
    ratio = float(torch.where(tol > 0, err / torch.where(tol > 0, tol, torch.ones_like(tol)),
                              torch.where(err > 0, torch.full_like(err, float("inf")), torch.zeros_like(err))).max())
    print(f"{what}: max |err| / (u bound) = {ratio * C_TOL:.3g}")
    if bad.any():
        i = np.unravel_index(int(torch.argmax(torch.where(bad, err / tol.clamp_min(1e-300), torch.zeros_like(err)))),
                             bad.shape)
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements beyond c u bound; worst at {i}: got "
                             f"{float(got[i])!r}, want {float(want[i])!r}, tol {float(tol[i])!r}")


def _scalar(got, want, bound, what):
    err = abs(float(got) - want)
    print(f"{what}: |err| / (u bound) = {err / (ar.U * bound):.3g}")
    assert err <= C_TOL * ar.U * bound, (what, float(got), want, bound)


def _ids(c):
    return "_".join(f"{k}{v}" for k, v in c.items())


# ---------------------------------------------------------------------------------------------------------------------
# convex upsampling

UPSAMPLE = [dict(B=2, H=1, W=1, k=1, CH=1), dict(B=2, H=1, W=1, k=8, CH=2), dict(B=1, H=1, W=37, k=8, CH=2),
            dict(B=3, H=29, W=1, k=2, CH=1), dict(B=2, H=13, W=33, k=4, CH=2, spread=60.0),
            dict(B=2, H=13, W=33, k=1, CH=1), dict(B=2, H=32, W=32, k=4, CH=1),
            dict(B=2, H=13, W=33, k=8, CH=1, spread=60.0), dict(B=3, H=13, W=33, k=2, CH=2, neg=True),
            dict(B=8, H=120, W=160, k=4, CH=1), dict(B=4, H=88, W=304, k=4, CH=2)]


@pytest.mark.parametrize("case", UPSAMPLE, ids=_ids)
def test_convex_upsample(cuda, case):
    k = case["k"]
    preds, lg, _, _, _ = ar.upsample_inputs(**case, seed=21)
    depth = preds[0].to(cuda).requires_grad_()
    mask = lg.to(cuda).requires_grad_()
    out = ops.convex_upsample(depth, mask, k)
    gout = torch.randn(out.shape, generator=torch.Generator().manual_seed(22)).to(cuda)
    out.backward(gout)
    want, bound = ar.convex_upsample(depth, mask, k)
    _close(out, want, bound, "upsample out")
    gd, bd, gm, bm = ar.convex_upsample_bwd(gout, depth, mask, k)
    _close(depth.grad, gd, bd, "upsample grad_depth")
    _close(mask.grad, gm, bm, "upsample grad_mask")


# ---------------------------------------------------------------------------------------------------------------------
# fused upsample + NLL (magnet_loss)

NLL = [dict(B=2, H=1, W=1, k=1, n=1), dict(B=1, H=1, W=37, k=4, n=2, mask="sparse", neg=True),
       dict(B=3, H=29, W=1, k=8, n=1, tiny=2), dict(B=2, H=13, W=33, k=4, n=3, mask="last", spread=60.0),
       dict(B=2, H=32, W=32, k=4, n=4, empty=True, tiny=3, neg=True),
       dict(B=2, H=13, W=33, k=2, n=2, mask="sparse", tiny=2), dict(B=2, H=13, W=33, k=8, n=1, neg=True),
       dict(B=8, H=120, W=160, k=4, n=4, tiny=8, neg=True),
       dict(B=4, H=88, W=304, k=4, n=2, mask="sparse", empty=True, tiny=4),
       dict(B=4, H=88, W=304, k=4, n=1, mask="last", neg=True)]


@pytest.mark.parametrize("case", NLL, ids=_ids)
def test_magnet_loss(cuda, case):
    k = case["k"]
    preds, lg, gt, gtm, clamped = ar.upsample_inputs(**case, seed=31)
    preds = [p.to(cuda).requires_grad_() for p in preds]
    mask = lg.to(cuda).requires_grad_()
    gt, gtm, clamped = gt.to(cuda), gtm.to(cuda), clamped.to(cuda)
    amb = ar.upsample_nll(preds, mask, gt, gtm, k, c=C_TOL)["ambiguous"] & gtm
    gtm = gtm & ~amb
    print(f"{int(gtm.sum())} supervised pixels, {int(amb.sum())} ambiguous left out, "
          f"{int((clamped & gtm).sum())} clamped")
    if case.get("tiny"):
        assert (clamped & gtm).any()
    r = ar.upsample_nll(preds, mask, gt, gtm, k, c=C_TOL)
    loss = ops.magnet_loss(preds, mask, gt, gtm, k, gamma=0.8)
    loss.backward()
    _scalar(loss, r["loss"], r["loss_bound"], "nll loss")
    for i, p in enumerate(preds):
        _close(p.grad, r["grad_preds"][i], r["grad_preds_bound"][i], f"nll grad_pred{i}")
    _close(mask.grad, r["grad_mask"], r["grad_mask_bound"], "nll grad_mask")


# ---------------------------------------------------------------------------------------------------------------------
# Gaussian update

@pytest.mark.parametrize("B,H,W", [(1, 1, 1), (5, 37, 41), (16, 29, 13)])
def test_gaussian_update(cuda, B, H, W):
    g = torch.Generator().manual_seed(B * 7 + W)
    dout = torch.randn(B, 2, H, W, generator=g)
    dout[:, 1] = 40.0 * torch.rand(B, H, W, generator=g) - 20.0
    flat = dout[:, 1].reshape(-1).clone()
    special = torch.tensor([0.0, -0.0, -95.0, -103.5, -110.0, -200.0, 1e-30, -1e-30])[:flat.numel()]
    flat[:special.numel()] = special
    dout[:, 1] = flat.view(B, H, W)
    gmm0 = torch.cat([1.0 + 9.0 * torch.rand(B, 1, H, W, generator=g), 0.01 + 2.0 * torch.rand(B, 1, H, W, generator=g)],
                     1)
    gout = torch.randn(B, 2, H, W, generator=g)
    x = dout.to(cuda).requires_grad_()
    out = ops.gaussian_update(x, gmm0.to(cuda))
    out.backward(gout.to(cuda))
    want, bound, grad, gbound = ar.gaussian_update(dout, gmm0, gout)
    _close(out, want, bound, "update out")
    _close(x.grad, grad, gbound, "update grad")


# ---------------------------------------------------------------------------------------------------------------------
# F-Net soft-argmin L1

FNET = [dict(B=2, D=80, H=120, W=160, scale=1.0), dict(B=4, D=80, H=88, W=304, scale=10.0),
        dict(B=3, D=256, H=37, W=29, scale=1e2), dict(B=2, D=256, H=88, W=304, scale=1.0),
        dict(B=2, D=5, H=37, W=29, scale=1e-2), dict(B=1, D=2, H=13, W=11, scale=1.0),
        dict(B=2, D=1, H=9, W=15, scale=1.0)]


def _fnet_check(cuda, scores, planes, gt, mask, count_tensor):
    scores, gt, mask = scores.to(cuda), gt.to(cuda), mask.to(cuda)
    amb = ar.fnet_l1(scores, planes, gt, mask, c=C_TOL)["ambiguous"]
    mask = mask & ~amb
    r = ar.fnet_l1(scores, planes, gt, mask, c=C_TOL)
    s = scores.clone().requires_grad_()
    n = int(mask.sum())
    count = torch.tensor(n, device=cuda) if count_tensor else n
    loss = ops.fnet_l1_loss(s, planes.tolist(), gt, mask, count)
    loss.backward()
    print(f"{n} supervised pixels, {int(amb.sum())} ambiguous left out")
    _scalar(loss, r["loss"], r["loss_bound"], "fnet loss")
    _close(s.grad, r["grad"], r["grad_bound"], "fnet grad")
    return s.grad, r


@pytest.mark.parametrize("case", FNET, ids=_ids)
@pytest.mark.parametrize("count_tensor", [False, True], ids=["int", "tensor"])
def test_fnet_l1(cuda, case, count_tensor):
    scores, planes, gt, mask = ar.fnet_inputs(**case, seed=41)
    if case["D"] == 1:                     # an exact tie at every other pixel: pred = d_0 = gt
        gt.view(-1)[::2] = planes[0]
    grad, r = _fnet_check(cuda, scores, planes, gt, mask, count_tensor)
    tie = (r["pred"] == gt.to(cuda).double()).expand_as(grad)
    assert (grad[tie] == 0).all() and (case["D"] > 1 or tie.any())


def test_fnet_l1_exact_tie(cuda):
    """Equal scores over 4 planes 1..4: pred = 2.5 exactly in fp32 and float64; where gt = 2.5 the gradient is exactly
    zero (sign(0) = 0), elsewhere it is not."""
    g = torch.Generator().manual_seed(43)
    B, H, W = 2, 19, 27
    scores = torch.randn(B, 1, H, W, generator=g).expand(B, 4, H, W).contiguous()
    planes = torch.tensor([1.0, 2.0, 3.0, 4.0])
    gt = 0.5 + 4.0 * torch.rand(B, 1, H, W, generator=g)
    tie = torch.rand(B, 1, H, W, generator=g) < 0.5
    gt[tie] = 2.5
    mask = torch.ones(B, 1, H, W, dtype=torch.bool)
    grad, _ = _fnet_check(cuda, scores, planes, gt, mask, False)
    grad = grad.cpu()
    assert (grad[tie.expand_as(grad)] == 0).all()
    assert (grad[(~tie).expand_as(grad)] != 0).all()


# ---------------------------------------------------------------------------------------------------------------------
# camera preparation

@pytest.mark.parametrize("tmax", [1.0, 1e3])
def test_relative_poses(cuda, tmax):
    B, V = 12, 7                                              # 84 (b, v) threads: two blocks of 64
    er, en = ar.pose_inputs(B, V, tmax, seed=51, nan_ref=(3,), nan_nghbr=((2, 5), (6, 0)))
    poses, valid = ops.relative_poses(torch.from_numpy(er).to(cuda), torch.from_numpy(en).to(cuda))
    poses, valid = poses.cpu().numpy(), valid.cpu().numpy()
    ref32, valid32 = mo.relative_poses(er, en)
    assert (valid == valid32).all() and valid.sum() == B * V - V - 2
    assert (poses[valid == 0] == 0).all()
    want, absprod = ar.relative_poses(er, en)
    ok = valid == 1
    tol = ar.pose_tolerance(want, ref32, absprod, POSE_FACTOR)[ok]
    err = np.abs(poses[ok].astype(np.float64) - want[ok])
    print(f"relative poses |t| <= {tmax:g}: max err / tol = {float(np.max(err / tol)):.3g}, max err / fp32 route err = "
          f"{float(np.max(err / np.maximum(tol / POSE_FACTOR, 1e-300))):.3g}")
    assert (err <= tol).all()


def _raw_intrinsics(B, H, W, family, rng):
    raw = np.zeros((B, 8))
    for b in range(B):
        if family == "scannet":
            raw[b] = [rng.uniform(540, 600), rng.uniform(540, 600), rng.uniform(300, 340), rng.uniform(220, 260), 640,
                      480, 0, 0]
        elif family == "kitti":
            rw, rh = rng.integers(1224, 1250), rng.integers(360, 380)
            raw[b] = [rng.uniform(700, 730), rng.uniform(700, 730), rng.uniform(590, 620), rng.uniform(160, 190),
                      1216, 352, (rw - 1216) // 2, rh - 352]
        else:                             # arbitrary crops: non-power-of-two grid ratios, fractional margins
            iw, ih = rng.uniform(100, 2000), rng.uniform(100, 2000)
            raw[b] = [rng.uniform(50, 3000), rng.uniform(50, 3000), rng.uniform(0, iw), rng.uniform(0, ih), iw, ih,
                      rng.uniform(0, 40), rng.uniform(0, 40)]
    return raw


@pytest.mark.parametrize("B,H,W,family", [(1, 1, 1, "random"), (2, 1, 1, "scannet"), (3, 7, 13, "random"),
                                          (2, 120, 160, "scannet"), (3, 88, 304, "kitti"), (3, 352, 1216, "kitti"),
                                          (4, 37, 29, "random")])
def test_camera_rays_bit_exact(cuda, B, H, W, family):
    rng = np.random.default_rng(H * 1000 + W + B)
    raw = _raw_intrinsics(B, H, W, family, rng)
    if family == "random":
        # principal point exactly on a pixel centre (in fp64): the reference's ray is exactly 0 there, and only a
        # product rounded before the subtraction (no fma) reproduces it
        x0, y0 = W // 2, H // 2
        raw[0, 2], raw[0, 3] = (x0 + 0.5) * (raw[0, 4] / W), (y0 + 0.5) * (raw[0, 5] / H)
        raw[0, 6] = raw[0, 7] = 0.0
    intM_want, rays_want = mo.camera_rays(raw, H, W)
    if family == "random":
        assert rays_want[0, 0, x0] == 0.0 and rays_want[0, 1, y0 * W] == 0.0
    got = ops.camera_rays(torch.from_numpy(raw).to(cuda), H, W)
    assert np.array_equal(got["intM"].cpu().numpy(), intM_want)
    r = got["unit_ray_array_2D"].cpu().numpy()
    assert np.array_equal(r, rays_want), f"{int((r != rays_want).sum())} ray elements differ"


@pytest.mark.parametrize("B,D,H,W", [(3, 1, 1, 1), (8, 256, 37, 29), (2, 256, 13, 7), (5, 1, 120, 160)])
def test_sample_depths_bit_exact(cuda, B, D, H, W):
    g = torch.Generator().manual_seed(D + W)
    gmm = torch.cat([0.5 + 9.5 * torch.rand(B, 1, H, W, generator=g), 0.01 + 3 * torch.rand(B, 1, H, W, generator=g)],
                    1)
    gmm[-1, 1] = -gmm[-1, 1]
    k = (3.0 * torch.randn(D, generator=g)).tolist()
    got = ops.sample_depths(gmm.to(cuda), k).cpu().numpy()
    assert np.array_equal(got, ar.sample_depths_f32(gmm.numpy(), k))


@pytest.mark.parametrize("transposed", [False, True])
def test_pack_cameras(cuda, transposed):
    B, V = 9, 8                                              # 72 (b, v) threads: two blocks of 64
    er, en = ar.pose_inputs(B, V, 1e3, seed=61, nan_nghbr=((3, 2),))
    poses, valid = ops.relative_poses(torch.from_numpy(er).to(cuda), torch.from_numpy(en).to(cuda))
    rng = np.random.default_rng(62)
    K = np.zeros((B, 3, 3), np.float32)
    K[:, 0, 0], K[:, 1, 1] = rng.uniform(100, 800, B), rng.uniform(100, 800, B)
    K[:, 0, 2], K[:, 1, 2], K[:, 2, 2] = rng.uniform(50, 300, B), rng.uniform(50, 200, B), 1.0
    R = poses[..., :3, :3]
    if transposed:
        R = R.transpose(-1, -2)
    t = poses[..., :3, 3]
    assert not R.is_contiguous() and not t.is_contiguous()
    cams = ops.pack_cameras(torch.from_numpy(K).to(cuda), R, t, valid)
    want, bound = ar.pack_cameras(K, R.cpu().numpy(), t.cpu().numpy(), valid.cpu().numpy())
    cams = cams.cpu()
    assert torch.equal(cams[:, 0], torch.from_numpy(want[:, 0]).float()) and (cams[:, 13:] == 0).all()
    _close(cams[:, 1:13], want[:, 1:13], bound[:, 1:13], "pack_cameras")
