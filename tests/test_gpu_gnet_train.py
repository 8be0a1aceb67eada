"""The differentiable fused G-Net head on the H100 (DESIGN §3.10): gradients against a float64 autograd evaluation of
the head and update and against the cuDNN module path, forward identity with the inference kernel, determinism,
CUDA-graph replay, the fused_train dispatch of matching_loop and a few training steps of MagnetHead."""
import pytest
import torch
import torch.nn.functional as F

import magnet_b200
from magnet_b200 import ops
from magnet_b200.matcher import GNET, fused_gnet_trains, matching_loop
from magnet_b200.synthetic import make_inputs

pytestmark = pytest.mark.gpu


def _head(D, dev, seed=0):
    torch.manual_seed(seed)
    return GNET(ch_in=D + 16).to(dev).train()


def _params(g):
    s = g.gnet
    return [s[0].weight, s[2].weight, s[2].bias, s[4].weight, s[4].bias, s[6].weight, s[6].bias]


def _f64_grads(g, cost, inv, prev, grad_out):
    """Autograd through the head and the update in float64: gradients of sum(out * grad_out) w.r.t. inv, W0[:, :D],
    W1, b1, W2, b2, W3, b3."""
    D = cost.shape[1]
    ws = [p.detach().double().requires_grad_(True) for p in _params(g)]
    inv64 = inv.detach().double().requires_grad_(True)
    h = F.relu(F.conv2d(cost.double(), ws[0][:, :D], None, padding=1) + inv64)
    h = F.relu(F.conv2d(h, ws[1], ws[2]))
    h = F.relu(F.conv2d(h, ws[3], ws[4]))
    raw = F.conv2d(h, ws[5], ws[6])
    mu0, s0 = prev[:, :1].double(), prev[:, 1:].double()
    out = torch.cat([mu0 + raw[:, :1] * s0, (F.elu(raw[:, 1:]) + 1 + 1e-10) * s0], 1)
    gr = torch.autograd.grad(out, [inv64] + ws, grad_out.double())
    return [gr[0], gr[1][:, :D]] + list(gr[2:])


def _fused_grads(g, cost, inv, prev, grad_out):
    inv = inv.detach().clone().requires_grad_(True)
    for p in g.parameters():
        p.grad = None
    out = ops.gnet_head_train(cost, inv, g, prev)
    out.backward(grad_out)
    D = cost.shape[1]
    ps = _params(g)
    return out.detach(), [inv.grad, ps[0].grad[:, :D]] + [p.grad for p in ps[1:]]


def _module_grads(g, cost, inv, prev, grad_out):
    inv = inv.detach().clone().requires_grad_(True)
    for p in g.parameters():
        p.grad = None
    out = ops.gaussian_update(g.raw_from_parts(cost, inv), prev)
    out.backward(grad_out)
    D = cost.shape[1]
    ps = _params(g)
    return [inv.grad, ps[0].grad[:, :D]] + [p.grad for p in ps[1:]]


NAMES = ["inv", "W0c", "W1", "b1", "W2", "b2", "W3", "b3"]


def _errs(got, want):
    return [float((a.double() - b).abs().max()) for a, b in zip(got, want)]


def _inputs(B, D, H, W, dev, seed, cost_scale=1.0, inv_scale=0.3):
    gen = torch.Generator(device=dev).manual_seed(seed)
    cost = cost_scale * torch.randn(B, D, H, W, device=dev, generator=gen)
    inv = inv_scale * torch.randn(B, 128, H, W, device=dev, generator=gen)
    prev = torch.cat([1 + torch.rand(B, 1, H, W, device=dev, generator=gen),
                      0.1 + 0.5 * torch.rand(B, 1, H, W, device=dev, generator=gen)], 1)
    grad_out = torch.randn(B, 2, H, W, device=dev, generator=gen)
    return cost, inv, prev, grad_out


def unambiguous(g, cost, inv, band=1e-5):
    """(B,1,H,W) float mask of the pixels whose ReLU masks are the same in any evaluation within `band` relative error:
    no pre-activation of h0, h1, h2 within band * (largest |pre-activation| of its layer) of zero.  The gradients are
    discontinuous across a ReLU's kink, so a pixel where an fp32 evaluation may land on the other side of it would
    compare the two sides, not the arithmetic."""
    D = cost.shape[1]
    s = g.gnet
    with torch.no_grad():
        z = F.conv2d(cost.double(), s[0].weight[:, :D].double(), None, padding=1) + inv.double()
        ok = torch.ones_like(z[:, :1], dtype=torch.bool)
        for layer in (2, 4, None):
            ok &= (z.abs() > band * z.abs().max()).all(1, keepdim=True)
            if layer is None:
                break
            z = F.conv2d(F.relu(z), s[layer].weight.double(), s[layer].bias.double())
    return ok.float()


def _check_against_f64(g, cost, inv, prev, grad_out, compare_module=True):
    grad_out = grad_out * unambiguous(g, cost, inv)
    want = _f64_grads(g, cost, inv, prev, grad_out)
    _, got = _fused_grads(g, cost, inv, prev, grad_out)
    e_fused = _errs(got, want)
    for n, e, w in zip(NAMES, e_fused, want):
        assert e <= 1e-4 * float(w.abs().max()), f"{n}: {e:.3e} vs max {float(w.abs().max()):.3e}"
    if compare_module:                                   # PyTorch's default flags: cuDNN convolutions in TF32
        assert torch.backends.cudnn.allow_tf32
        e_mod = _errs(_module_grads(g, cost, inv, prev, grad_out), want)
        for n, a, b in zip(NAMES, e_fused, e_mod):
            if n.startswith("b"):      # bias gradients: plain fp32 reductions in both paths, no TF32 product to beat
                continue
            assert a <= b, f"{n}: fused {a:.3e} > module {b:.3e}"


GRIDS = [(7, 9), (24, 40)]


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("D", [1, 5, 16, 17, 64, 256])
@pytest.mark.parametrize("grid", GRIDS, ids=[f"{h}x{w}" for h, w in GRIDS])
def test_fused_head_gradients_match_float64(cuda, D, grid, B):
    H, W = grid
    g = _head(D, cuda, seed=D)
    _check_against_f64(g, *_inputs(B, D, H, W, cuda, seed=H * W + D + B))


# cfg2, cfg3 at D 64 and the shipped N_s = 5 at the cfg2 grid (test_gpu_gnet_head.SHAPES)
SHAPES = [(8, 64, 120, 160), (4, 64, 88, 304), (8, 5, 120, 160)]


@pytest.mark.parametrize("shape", SHAPES, ids=["cfg2", "cfg3", "ns5"])
def test_fused_head_gradients_at_production_shapes(cuda, shape):
    B, D, H, W = shape
    g = _head(D, cuda, seed=2)
    _check_against_f64(g, *_inputs(B, D, H, W, cuda, seed=5))


@pytest.mark.parametrize("cost_scale", [1e-3, 1.0, 1e3])
@pytest.mark.parametrize("inv_scale", [1e-3, 1.0, 1e3])
def test_fused_head_gradients_across_input_scales(cuda, cost_scale, inv_scale):
    g = _head(64, cuda, seed=1)
    _check_against_f64(g, *_inputs(3, 64, 24, 40, cuda, seed=11, cost_scale=cost_scale, inv_scale=inv_scale),
                       compare_module=False)


def test_gradient_from_the_fused_loss(cuda):
    B, D, H, W = 2, 16, 24, 40
    g = _head(D, cuda, seed=4)
    cost, inv, prev, _ = _inputs(B, D, H, W, cuda, seed=3)
    out = ops.gnet_head_train(cost, inv, g, prev).detach().requires_grad_(True)
    mask = torch.rand(B, 9 * 16, H, W, device=cuda)
    gt = 1.5 + torch.rand(B, 1, 4 * H, 4 * W, device=cuda)
    ops.magnet_loss([out], mask, gt, gt > 0, 4).backward()
    _check_against_f64(g, cost, inv, prev, out.grad)


def test_training_forward_is_the_inference_forward(cuda):
    for D, (H, W) in [(5, (7, 9)), (64, (24, 40)), (64, (120, 160))]:
        g = _head(D, cuda, seed=7)
        cost, inv, prev, _ = _inputs(2, D, H, W, cuda, seed=D)
        with torch.no_grad():
            want = ops.gnet_update(cost, inv, ops.pack_gnet_weights(g, D), prev)
        got = ops.gnet_head_train(cost, inv, g, prev)
        assert got.requires_grad and torch.equal(got.detach(), want)


def test_gradient_into_prev(cuda):
    B, D, H, W = 2, 8, 12, 20
    g = _head(D, cuda, seed=9)
    cost, inv, prev, grad_out = _inputs(B, D, H, W, cuda, seed=9)
    p = prev.clone().requires_grad_(True)
    ops.gnet_head_train(cost, inv, g, p).backward(grad_out)
    p64 = prev.double().requires_grad_(True)
    s = g.gnet
    h = F.relu(F.conv2d(cost.double(), s[0].weight[:, :D].double(), None, padding=1) + inv.double())
    h = F.relu(F.conv2d(h, s[2].weight.double(), s[2].bias.double()))
    h = F.relu(F.conv2d(h, s[4].weight.double(), s[4].bias.double()))
    raw = F.conv2d(h, s[6].weight.double(), s[6].bias.double()).detach()
    out = torch.cat([p64[:, :1] + raw[:, :1] * p64[:, 1:], (F.elu(raw[:, 1:]) + 1 + 1e-10) * p64[:, 1:]], 1)
    (want,) = torch.autograd.grad(out, [p64], grad_out.double())
    assert float((p.grad.double() - want).abs().max()) <= 1e-4 * float(want.abs().max())


def test_backward_is_deterministic_and_graph_capturable(cuda):
    B, D, H, W = 2, 64, 24, 40
    g = _head(D, cuda, seed=6)
    cost, inv, prev, grad_out = _inputs(B, D, H, W, cuda, seed=6)
    runs = [_fused_grads(g, cost, inv, prev, grad_out) for _ in range(2)]
    assert torch.equal(runs[0][0], runs[1][0])
    for a, b in zip(runs[0][1], runs[1][1]):
        assert torch.equal(a, b)

    static_inv = inv.clone().requires_grad_(True)

    def step():
        for p in g.parameters():
            p.grad = None
        static_inv.grad = None
        out = ops.gnet_head_train(cost, static_inv, g, prev)
        out.backward(grad_out)
        return out

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                                          # warm-up outside the capture
        step()
    torch.cuda.current_stream().wait_stream(s)
    for p in g.parameters():
        p.grad = None
    static_inv.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static_out = step()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(static_out.detach(), runs[0][0])
    ps = _params(g)
    for a, b in zip([static_inv.grad, ps[0].grad[:, :D]] + [p.grad for p in ps[1:]], runs[0][1]):
        assert torch.equal(a, b)


def _plan_inputs(dev, D=16, rg=False):
    inp = make_inputs(B=2, V=2, D=D, H=24, W=40, C=64, seed=21, depth="smooth")
    g = inp.to(dev)
    rf, sf = g.ref_feat, g.nghbr_feat
    if rg:
        rf, sf = rf.clone().requires_grad_(True), sf.clone().requires_grad_(True)
    plan = magnet_b200.MatchingPlan(rf, sf, g.nghbr_gmms, g.nghbr_poses, inp.is_valid, inp.cam_intrins, thres=inp.thres)
    x_d3 = torch.randn(2, 16, 24, 40, device=dev, generator=torch.Generator(device=dev).manual_seed(4))
    return inp, g, plan, x_d3


def _chain(plan, ref, x_d3, head, k, n, fused, detach=True):
    inv = head.invariant_part(x_d3, len(k))
    cur, out = ref, []
    for _ in range(n):
        cur = cur.detach().float()
        if detach:
            with torch.no_grad():
                cv = plan.cost(cur, k)
        else:
            cv = plan.cost(cur, k)
        cur = ops.gnet_head_train(cv, inv, head, cur) if fused else ops.gaussian_update(head.raw_from_parts(cv, inv).float(), cur)
        out.append(cur)
    return out


def test_matching_loop_fused_train_dispatch(cuda):
    inp, g, plan, x_d3 = _plan_inputs(cuda)
    head = _head(16, cuda, seed=3)
    k = inp.k.tolist()
    # trainable parameters: the fused path
    preds = matching_loop(plan, g.ref_gmms, x_d3, head, 2, k, fused_train=True)
    want = _chain(plan, g.ref_gmms, x_d3, head, k, 2, fused=True)
    for a, b in zip(preds[1:], want):
        assert torch.equal(a.detach(), b.detach()) and a.requires_grad
        assert type(a.grad_fn).__name__.startswith("GnetHeadTrain")
    # fused_train=False: unchanged (the module chain)
    preds = matching_loop(plan, g.ref_gmms, x_d3, head, 2, k)
    want = _chain(plan, g.ref_gmms, x_d3, head, k, 2, fused=False)
    for a, b in zip(preds[1:], want):
        assert torch.equal(a.detach(), b.detach())
    # detach_cost=False with feature maps that require grad: the module chain
    inp2, g2, plan2, _ = _plan_inputs(cuda, rg=True)
    preds = matching_loop(plan2, g2.ref_gmms, x_d3, head, 2, k, detach_cost=False, fused_train=True)
    want = _chain(plan2, g2.ref_gmms, x_d3, head, k, 2, fused=False, detach=False)
    for a, b in zip(preds[1:], want):
        assert torch.equal(a.detach(), b.detach())
    # autocast: the module chain
    with torch.autocast("cuda", dtype=torch.bfloat16):
        preds = matching_loop(plan, g.ref_gmms, x_d3, head, 2, k, fused_train=True)
        want = _chain(plan, g.ref_gmms, x_d3, head, k, 2, fused=False)
    for a, b in zip(preds[1:], want):
        assert torch.equal(a.detach(), b.detach())


def test_dispatch_rule_on_device_tensors(cuda):
    head = _head(8, cuda)
    cv, inv = torch.zeros(1, 8, 4, 4, device=cuda), torch.zeros(1, 128, 4, 4, device=cuda)
    assert fused_gnet_trains(head, cv, inv)
    with torch.no_grad():
        assert not fused_gnet_trains(head, cv, inv)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        assert not fused_gnet_trains(head, cv, inv)


def _train(fused, steps, dev, tf32=True):
    B, H, W, D = 2, 24, 40, 16
    inp = make_inputs(B=B, V=2, D=D, H=H, W=W, C=64, seed=31, depth="smooth").to(dev)
    x_d3 = torch.randn(B, 256, H, W, generator=torch.Generator().manual_seed(7)).to(dev)
    gt = torch.nn.functional.interpolate(inp.ref_gmms[:, 0:1] * 1.03, scale_factor=4, mode="nearest")
    mask = gt > 1e-3
    torch.manual_seed(0)
    head = magnet_b200.MagnetHead(n_samples=D, sampling_range=3, n_iter=3, thres=5, fused_train=fused).to(dev)
    opt = torch.optim.AdamW(head.parameters(), lr=3.57e-4, weight_decay=1e-2)
    losses, first = [], None
    flag = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = tf32
    try:
        for _ in range(steps):
            preds_q, up_mask = head.forward_quarter(inp.ref_feat, inp.nghbr_feat, inp.ref_gmms, inp.nghbr_gmms, x_d3,
                                                    inp.nghbr_poses, inp.is_valid, inp.cam_intrins)
            loss = head.loss(preds_q, up_mask, gt, mask)
            opt.zero_grad(set_to_none=True)
            loss.backward()
            if first is None:
                first = {n: p.grad.detach().clone() for n, p in head.named_parameters()}
            opt.step()
            losses.append(float(loss.detach()))
    finally:
        torch.backends.cudnn.allow_tf32 = flag
    return losses, first


def test_magnet_head_training_steps(cuda):
    losses, first = _train(True, 6, cuda)
    assert all(torch.isfinite(g).all() for g in first.values())
    assert losses[-1] < losses[0]
    ref_losses, ref = _train(False, 6, cuda, tf32=False)
    # The element-wise gradient numerics are checked per op above (away from ReLU kinks).  A whole step of three
    # iterations on 2 x 24 x 40 pixels cannot be compared element-wise: where an fp32 pre-activation lies within
    # rounding of zero the two paths may take different sides of the kink, and at this size one such pixel moves a
    # weight gradient by about a percent of its norm.  So the step is checked in norm and through the losses of six
    # AdamW steps, which must follow the module path's.
    for n, g in first.items():
        err = float((g - ref[n]).norm() / ref[n].norm())
        assert err <= 5e-2, (n, err)
    for a, b in zip(losses, ref_losses):
        assert abs(a - b) <= 1e-3 * abs(b), (a, b)
