"""The fused mask-head training loss on the H100 (DESIGN §3.13): loss and gradients against float64 autograd of the
mask head, the upsampling and MagnetLoss and against the cuDNN module path, determinism, gradient masking, non-finite
input, and MagnetHead.train_loss with fused_upsample against the module path, including its fallbacks."""
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import magnet_b200
from magnet_b200 import ops
from magnet_b200.synthetic import make_inputs
from tests.mask_train_ref import loss64

pytestmark = pytest.mark.gpu

NAMES = ["pre0", "W1", "b1", "W2", "b2", "W3", "b3"]


def _mask_head(dev, seed=0):
    torch.manual_seed(seed)
    return magnet_b200.MagnetHead(dnet_fdim=16).mask_head.to(dev)


def _layers(mh):
    return [mh[2].weight, mh[2].bias, mh[4].weight, mh[4].bias, mh[6].weight, mh[6].bias]


def _inputs(B, P, H, W, dev, seed, scale=1.0, density=0.5):
    gen = torch.Generator(device=dev).manual_seed(seed)
    pre0 = scale * torch.randn(B, 128, H, W, device=dev, generator=gen)
    preds = [torch.cat([1 + torch.rand(B, 1, H, W, device=dev, generator=gen),
                        0.1 + 0.5 * torch.rand(B, 1, H, W, device=dev, generator=gen)], 1) for _ in range(P)]
    gt = 1 + torch.rand(B, 1, 4 * H, 4 * W, device=dev, generator=gen)
    gtm = torch.rand(B, 1, 4 * H, 4 * W, device=dev, generator=gen) < density
    return pre0, preds, gt, gtm


def unambiguous(mh, pre0, band=1e-5):
    """(B,1,H,W) bool: pixels whose h1 and h2 pre-activations all lie further than band * (largest of the layer) from
    zero, so that an fp32 evaluation takes the same side of every ReLU kink as float64 (h0 = ReLU(pre0) of an exact
    input needs no band)."""
    with torch.no_grad():
        z = F.conv2d(F.relu(pre0.double()), mh[2].weight.double(), mh[2].bias.double())
        ok = (z.abs() > band * z.abs().max()).all(1, keepdim=True)
        z = F.conv2d(F.relu(z), mh[4].weight.double(), mh[4].bias.double())
        ok &= (z.abs() > band * z.abs().max()).all(1, keepdim=True)
    return ok


def _supervise_unambiguous(mh, pre0, gtm):
    """The gt mask without the full-resolution pixels of ambiguous quarter-resolution pixels: their logits then carry no
    gradient, so the gradients compare the arithmetic, not the two sides of a kink."""
    ok = unambiguous(mh, pre0)
    return gtm & F.interpolate(ok.float(), scale_factor=4, mode="nearest").bool()


def _f64(mh, pre0, preds, gt, gtm, gamma, grad_out):
    ws = [t.detach().double().requires_grad_(True) for t in _layers(mh)]
    p0 = pre0.detach().double().requires_grad_(True)
    ps = [p.detach().double().requires_grad_(True) for p in preds]
    loss, bound = loss64(p0, ws, ps, gt.double(), gtm, gamma)
    gr = torch.autograd.grad(loss * grad_out, [p0] + ws + ps)
    return float(loss.detach()), bound, list(gr)


def _fused(mh, pre0, preds, gt, gtm, gamma, grad_out):
    for p in mh.parameters():
        p.grad = None
    p0 = pre0.detach().clone().requires_grad_(True)
    ps = [p.detach().clone().requires_grad_(True) for p in preds]
    loss = ops.mask_head_loss(p0, mh, ps, gt, gtm, 4, gamma)
    (loss * grad_out).backward()
    return loss.detach(), [p0.grad] + [t.grad for t in _layers(mh)] + [p.grad for p in ps]


def _module(mh, pre0, preds, gt, gtm, gamma, grad_out):
    for p in mh.parameters():
        p.grad = None
    p0 = pre0.detach().clone().requires_grad_(True)
    ps = [p.detach().clone().requires_grad_(True) for p in preds]
    mask = mh[6](mh[5](mh[4](mh[3](mh[2](F.relu(p0))))))
    loss = ops.magnet_loss(ps, mask, gt, gtm, 4, gamma)
    (loss * grad_out).backward()
    return loss.detach(), [p0.grad] + [t.grad for t in _layers(mh)] + [p.grad for p in ps]


def _errs(got, want):
    return [float((a.double() - b).abs().max()) for a, b in zip(got, want)]


def _check(mh, pre0, preds, gt, gtm, gamma=0.8, grad_out=1.0, compare_module=True, tol=1e-4):
    gtm = _supervise_unambiguous(mh, pre0, gtm)
    want_loss, bound, want = _f64(mh, pre0, preds, gt, gtm, gamma, grad_out)
    loss, got = _fused(mh, pre0, preds, gt, gtm, gamma, grad_out)
    assert abs(float(loss) - want_loss) <= 1e-5 * bound, (float(loss), want_loss, bound)
    names = NAMES + [f"pred{i}" for i in range(len(preds))]
    e_fused = _errs(got, want)
    worst = 0.0
    for n, e, w in zip(names, e_fused, want):
        m = float(w.abs().max())
        worst = max(worst, e / m if m > 0 else e)
        assert e <= tol * m, f"{n}: {e:.3e} vs max {m:.3e}"
    print(f"largest error / largest entry: {worst:.3e}")
    if compare_module:                                   # PyTorch's default flags: cuDNN convolutions in TF32
        assert torch.backends.cudnn.allow_tf32
        _, mod = _module(mh, pre0, preds, gt, gtm, gamma, grad_out)
        e_mod = _errs(mod, want)
        for n, a, b in zip(names, e_fused, e_mod):
            if n.startswith("b") or n.startswith("pred"):   # fp32 sums and no TF32 product in either path
                continue
            assert a <= b, f"{n}: fused {a:.3e} > module {b:.3e}"


GRIDS = [(1, 1), (1, 17), (8, 16), (13, 29)]


@pytest.mark.parametrize("P", [1, 3, 8])
@pytest.mark.parametrize("grid", GRIDS, ids=[f"{h}x{w}" for h, w in GRIDS])
def test_gradients_match_float64(cuda, grid, P):
    H, W = grid
    mh = _mask_head(cuda, seed=P)
    _check(mh, *_inputs(2, P, H, W, cuda, seed=H * W + P), compare_module=H * W > 100)


SHAPES = [(8, 120, 160), (4, 88, 304)]


@pytest.mark.parametrize("shape", SHAPES, ids=["cfg2", "cfg3"])
def test_gradients_at_production_shapes(cuda, shape):
    B, H, W = shape
    mh = _mask_head(cuda, seed=2)
    _check(mh, *_inputs(B, 3, H, W, cuda, seed=5))


def test_dense_sparse_and_empty_gt_masks(cuda):
    mh = _mask_head(cuda, seed=3)
    pre0, preds, gt, _ = _inputs(3, 3, 13, 29, cuda, seed=12)
    gen = torch.Generator(device=cuda).manual_seed(1)
    gtm = torch.zeros_like(gt, dtype=torch.bool)
    gtm[0] = True                                                   # dense
    gtm[1] = torch.rand(gt[1].shape, device=cuda, generator=gen) < 0.02   # sparse; image 2 empty
    _check(mh, pre0, preds, gt, gtm, compare_module=False)


def test_sigma_clamp_cuts_the_sigma_gradient(cuda):
    mh = _mask_head(cuda, seed=4)
    pre0, preds, gt, gtm = _inputs(2, 3, 8, 16, cuda, seed=13)
    preds[1][:, 1] = 1e-6                                           # sigma^2 < 1e-10 everywhere: var clamps
    preds[2][:, 1, :4] = 1e-6
    _check(mh, pre0, preds, gt, gtm, compare_module=False)


def test_upstream_gradient_other_than_one(cuda):
    mh = _mask_head(cuda, seed=5)
    _check(mh, *_inputs(2, 3, 13, 29, cuda, seed=14), grad_out=0.37)


def test_deterministic_and_masked(cuda):
    mh = _mask_head(cuda, seed=6)
    pre0, preds, gt, gtm = _inputs(2, 3, 24, 40, cuda, seed=15)
    runs = [_fused(mh, pre0, preds, gt, gtm, 0.8, 1.0) for _ in range(2)]
    assert torch.equal(runs[0][0], runs[1][0])
    for a, b in zip(runs[0][1][:7], runs[1][1][:7]):
        assert torch.equal(a, b)
    for a, b in zip(runs[0][1][7:], runs[1][1][7:]):                # prediction gradients: sums of atomic adds
        assert torch.allclose(a, b, rtol=1e-5, atol=1e-7 * float(b.abs().max()))
    # frozen layers and a frozen pre0 get no gradient; the rest are unchanged
    mh[2].weight.requires_grad_(False)
    mh[6].bias.requires_grad_(False)
    for p in mh.parameters():
        p.grad = None
    ps = [p.detach().clone().requires_grad_(i != 1) for i, p in enumerate(preds)]
    ops.mask_head_loss(pre0, mh, ps, gt, gtm).backward()
    assert mh[2].weight.grad is None and mh[6].bias.grad is None and ps[1].grad is None
    assert torch.equal(mh[4].weight.grad, runs[0][1][3]) and torch.equal(mh[6].weight.grad, runs[0][1][5])
    assert ps[0].grad is not None and ps[2].grad is not None
    # only the predictions: no saved maps, no chain, no GEMM
    for p in mh.parameters():
        p.requires_grad_(False)
    n0 = magnet_b200._lib.launch_count()
    ops.mask_head_loss(pre0, mh, ps, gt, gtm).backward()
    assert magnet_b200._lib.launch_count() - n0 == 3 + 2 + 1    # pack (3), memset + forward, one scale kernel
    for p in mh.parameters():
        p.requires_grad_(True)


def test_nan_in_pre0_gives_nan_loss(cuda):
    mh = _mask_head(cuda, seed=7)
    pre0, preds, gt, gtm = _inputs(1, 2, 8, 16, cuda, seed=16)
    gtm[:] = True
    pre0[0, 5, 3, 7] = float("nan")
    loss = ops.mask_head_loss(pre0, mh, preds, gt, gtm)
    mask = mh[6](mh[5](mh[4](mh[3](mh[2](F.relu(pre0))))))
    assert torch.isnan(loss) and torch.isnan(ops.magnet_loss(preds, mask, gt, gtm, 4))


# ---- MagnetHead.train_loss -----------------------------------------------------------------------------------------
def _scene(dev, B=2, H=24, W=40, D=16, k=4):
    inp = make_inputs(B=B, V=2, D=D, H=H, W=W, C=64, seed=31, depth="smooth").to(dev)
    x_d3 = torch.randn(B, 256, H, W, generator=torch.Generator().manual_seed(7)).to(dev)
    gt = F.interpolate(inp.ref_gmms[:, 0:1] * 1.03, scale_factor=k, mode="nearest")
    return inp, x_d3, gt, gt > 1e-3


def _head(fused, dev, **kw):
    torch.manual_seed(0)
    return magnet_b200.MagnetHead(n_samples=16, sampling_range=3, n_iter=3, thres=5, fused_upsample=fused, **kw).to(dev)


def _step_loss(head, scene, gamma=0.8):
    inp, x_d3, gt, gtm = scene
    return head.train_loss(inp.ref_feat, inp.nghbr_feat, inp.ref_gmms, inp.nghbr_gmms, x_d3, inp.nghbr_poses,
                           inp.is_valid, inp.cam_intrins, gt, gtm, gamma)


def _today(head, scene, gamma=0.8):
    inp, x_d3, gt, gtm = scene
    preds, mask = head.forward_quarter(inp.ref_feat, inp.nghbr_feat, inp.ref_gmms, inp.nghbr_gmms, x_d3, inp.nghbr_poses,
                                       inp.is_valid, inp.cam_intrins)
    return head.loss(preds, mask, gt, gtm, gamma)


def test_train_loss_matches_the_module_path(cuda):
    """Loss and every parameter gradient, W0, b0 and the G-Net head's included.  As in the G-Net head's training test,
    a whole step is compared in norm: where an fp32 pre-activation lies within rounding of a ReLU kink the two paths
    may take different sides of it (the element-wise numerics are checked per op above, away from the kinks)."""
    scene = _scene(cuda)
    grads = []
    flag = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        for fused in (True, False):
            head = _head(fused, cuda)
            loss = _step_loss(head, scene)
            assert type(loss.grad_fn).__name__.startswith("MaskLossTrain") == fused
            loss.backward()
            grads.append((float(loss.detach()), {n: p.grad.double() for n, p in head.named_parameters()}))
    finally:
        torch.backends.cudnn.allow_tf32 = flag
    (lf, gf), (lm, gm) = grads
    assert abs(lf - lm) <= 1e-5 * abs(lm)
    for n in gm:
        err = float((gf[n] - gm[n]).norm() / gm[n].norm())
        print(n, err)
        assert err <= 5e-2, (n, err)


def test_train_loss_without_fusion_is_todays_loss(cuda):
    scene = _scene(cuda)
    head = _head(False, cuda)
    assert torch.equal(_step_loss(head, scene), _today(head, scene))


def test_fallbacks_are_todays_bits(cuda):
    scene = _scene(cuda)
    head = _head(True, cuda)
    with torch.no_grad():                                            # nothing to differentiate
        assert torch.equal(_step_loss(head, scene), _today(head, scene))
    with torch.autocast("cuda", dtype=torch.bfloat16):
        assert torch.equal(_step_loss(head, scene), _today(head, scene))
    many = _head(True, cuda)
    many.n_iter = 9                                                  # P > MAGNET_MASK_MAX_PRED
    assert torch.equal(_step_loss(many, scene), _today(many, scene))
    other = _head(True, cuda)
    other.mask_head[3] = nn.GELU()                                   # not the reference's structure
    assert torch.equal(_step_loss(other, scene), _today(other, scene))
    torch.manual_seed(0)
    k2 = magnet_b200.MagnetHead(n_samples=16, n_iter=3, downsample_ratio=2, fused_upsample=True).to(cuda)
    scene2 = _scene(cuda, k=2)
    assert torch.equal(_step_loss(k2, scene2), _today(k2, scene2))   # k != 4
    half = _head(True, cuda)
    half.mask_head.half()                                            # fp16 weights (x_d3 cast on the way in)
    half.mask_head.register_forward_pre_hook(lambda m, a: (a[0].half(),))
    assert torch.equal(_step_loss(half, scene), _today(half, scene))


def _train(fused, steps, dev):
    scene = _scene(dev)
    head = _head(fused, dev)
    opt = torch.optim.AdamW(head.parameters(), lr=3.57e-4, weight_decay=1e-2)
    losses = []
    flag = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        for _ in range(steps):
            loss = _step_loss(head, scene)
            opt.zero_grad(set_to_none=True)
            loss.backward()
            opt.step()
            losses.append(float(loss.detach()))
    finally:
        torch.backends.cudnn.allow_tf32 = flag
    return losses


def test_adamw_steps_follow_the_module_path(cuda):
    fused, ref = _train(True, 25, cuda), _train(False, 25, cuda)
    assert fused[-1] < fused[0]
    print("final losses", fused[-1], ref[-1])
    # the loss crosses zero on the way, so the gap is measured against the run's largest |loss| (measured on an H100:
    # 1.1e-4 of it after 25 steps; the G-Net head's training test holds 1e-3)
    top = max(abs(b) for b in ref)
    for a, b in zip(fused, ref):
        assert abs(a - b) <= 1e-3 * top, (a, b)
