"""D-Net's fused training loss on the H100 (ops.dnet_loss, DnetHead.loss, DESIGN §3.19):
  * the loss and the gradients into raw and the mask logits, element by element, against the float64 restatement of
    tests/dnet_loss_ref.py (|got - ref| <= c u bound, c = 32) at both training shapes and at small ragged grids for
    k = 2, 4, 8, with collapsed (v <= -20) and large positive v; pixels whose decisions lie inside their bounds leave the
    mask (dnet_loss_ref's docstring);
  * v <= -20 everywhere: var is exactly fp32(1e-10), the clamp never fires, and the gradient into v is not cut;
  * DnetHead.loss against the reference's Decoder heads + upsample_depth_via_mask + activation_G + DnetLoss
    (tests/golden/dnet_loss.npz: an ordinary case and a collapsed one), and against the module route (DnetHead.forward + DnetLoss with boolean indexing);
  * an empty mask raises eagerly; compiled, it gives a NaN loss and zero gradients;
  * compiled against eager (no graph break, a captured reduce-overhead step), and the loss bit-identical run to run."""
import copy
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from magnet_b200 import DnetHead, _lib, ops
from tests import aux_ref as ar
from tests import dnet_loss_ref as dr

pytestmark = pytest.mark.gpu

C_TOL = 32.0


def _close(got, want, bound, what):
    got = got.detach().to(torch.float64)
    want = torch.as_tensor(want, dtype=torch.float64, device=got.device)
    tol = C_TOL * ar.U * torch.as_tensor(bound, dtype=torch.float64, device=got.device)
    assert got.shape == want.shape, (what, tuple(got.shape), tuple(want.shape))
    assert torch.isfinite(got).all(), f"{what}: non-finite output"
    err = (got - want).abs()
    ratio = float((err / tol).max())
    print(f"{what}: max |err| / (c u bound) = {ratio:.3g}")
    bad = err > tol
    if bad.any():
        i = np.unravel_index(int(torch.argmax(torch.where(bad, err / tol, torch.zeros_like(err)))), bad.shape)
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} beyond c u bound; worst at {i}: got "
                             f"{float(got[i])!r}, want {float(want[i])!r}, tol {float(tol[i])!r}")


def _ids(c):
    return "_".join(f"{k}{v}" for k, v in c.items())


# ---------------------------------------------------------------------------------------------------------------------
# element by element against float64

CASES = [dict(B=16, H=104, W=136, k=4, deep=24, high=16),
         dict(B=16, H=88, W=176, k=4, mask="sparse", deep=24, high=16),
         dict(B=2, H=1, W=1, k=2), dict(B=1, H=1, W=37, k=8, high=2), dict(B=3, H=29, W=1, k=4),
         dict(B=2, H=13, W=33, k=2, deep=3, high=3), dict(B=2, H=13, W=33, k=8, mask="sparse", deep=2),
         dict(B=2, H=32, W=32, k=4, deep=4, high=4), dict(B=1, H=7, W=5, k=8, deep=1)]


@pytest.mark.parametrize("case", CASES, ids=_ids)
def test_loss_and_gradients_within_the_float64_bound(cuda, case):
    k = case["k"]
    raw, lg, gt, gtm, deep = dr.loss_inputs(**case, seed=61)
    raw, lg, gt, gtm, deep = raw.to(cuda), lg.to(cuda), gt.to(cuda), gtm.to(cuda), deep.to(cuda)
    amb = dr.dnet_nll(raw, lg, gt, gtm, k, c=C_TOL)["ambiguous"] & gtm
    gtm = gtm & ~amb
    r = dr.dnet_nll(raw, lg, gt, gtm, k, c=C_TOL, grad=1.5)
    print(f"{int(gtm.sum())} supervised, {int(amb.sum())} ambiguous left out, "
          f"{int((r['collapsed'] & gtm).sum())} collapsed")
    if case.get("deep") and case["H"] >= 3:
        assert (deep & gtm & r["collapsed"]).any()
    raw_l, lg_l = raw.clone().requires_grad_(), lg.clone().requires_grad_()
    loss = ops.dnet_loss(raw_l, lg_l, gt, gtm, k)
    (1.5 * loss).backward()
    err = abs(float(loss) - r["loss"])
    print(f"loss: |err| / (c u bound) = {err / (C_TOL * ar.U * r['loss_bound']):.3g}")
    assert err <= C_TOL * ar.U * r["loss_bound"], (float(loss), r["loss"])
    _close(raw_l.grad, r["grad_raw"], r["grad_raw_bound"], "grad_raw")
    _close(lg_l.grad, r["grad_mask"], r["grad_mask_bound"], "grad_mask")


def test_deep_negative_v_is_not_clamped(cuda):
    """raw v in [-120, -20] everywhere (expf underflows below -103): away from the border the upsampled v is <= -20, so
    var is exactly fp32(1e-10), which torch's own activation_G gives too and which the clamp var < 1e-10 leaves alone;
    the gradient into v is g_var e^v, not cut, and within the float64 bound."""
    g = torch.Generator().manual_seed(71)
    B, H, W, k = 2, 9, 11, 4
    mu = 1.0 + 9.0 * torch.rand(B, 1, H, W, generator=g)
    raw = torch.cat([mu, -20.0 - 100.0 * torch.rand(B, 1, H, W, generator=g)], 1).to(cuda)
    lg = (2.0 * torch.randn(B, 9 * k * k, H, W, generator=g)).to(cuda)
    gt = (1.0 + 9.0 * torch.rand(B, 1, k * H, k * W, generator=g)).to(cuda)
    v_up = ops.convex_upsample(raw, lg, k)[:, 1:2]
    deep = v_up <= -20                                  # all but border pixels, whose zero-padded taps pull v_up up
    assert float(deep.float().mean()) > 0.5
    var_torch = F.elu(v_up) + 1.0 + 1e-10               # activation_G in torch
    assert (var_torch[deep] == dr.VAR_MIN).all() and not (var_torch < 1e-10).any()
    r = dr.dnet_nll(raw, lg, gt, deep, k, c=C_TOL)
    assert r["collapsed"][deep].all()
    gtm = deep & ~r["ambiguous"]                        # only |d| within its bound can be ambiguous here
    r = dr.dnet_nll(raw, lg, gt, gtm, k, c=C_TOL)
    raw_l, lg_l = raw.clone().requires_grad_(), lg.clone().requires_grad_()
    loss = ops.dnet_loss(raw_l, lg_l, gt, gtm, k)
    loss.backward()
    assert abs(float(loss) - r["loss"]) <= C_TOL * ar.U * r["loss_bound"]
    _close(raw_l.grad, r["grad_raw"], r["grad_raw_bound"], "deep grad_raw")
    _close(lg_l.grad, r["grad_mask"], r["grad_mask_bound"], "deep grad_mask")
    assert (raw_l.grad[:, 1] != 0).any()


# ---------------------------------------------------------------------------------------------------------------------
# DnetHead.loss against the reference and against the module route

def _golden_head(cuda, case):
    head = DnetHead(in_dim=dr.GOLDEN["C"]).to(cuda)
    cpu = DnetHead(in_dim=dr.GOLDEN["C"])
    dr.seed_loss_heads(cpu.depth_head, cpu.mask_head, case)
    head.load_state_dict(cpu.state_dict())
    return head


def _golden(case):
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", "dnet_loss.npz"))
    return {k[len(case) + 1:]: z[k] for k in z.files if k.startswith(case + "_")}


def _golden_errors(z, loss, x, head):
    """|loss - reference| / |reference| and, per gradient (x_feat, each head parameter), max |got - reference| over
    max |reference|."""
    want = float(z["loss"])
    grads = {"g_x": x.grad, **{f"g_{n}": p.grad for n, p in head.named_parameters()}}
    errs = {}
    for name, got in grads.items():
        ref = torch.from_numpy(z[name]).to(got.device, torch.float64)
        got = (got[:, :dr.FIRST_IN] if name.endswith("0.weight") else got).double()
        errs[name] = float((got - ref).abs().max()) / float(ref.abs().max())
    return abs(float(loss) - want) / abs(want), errs


def _golden_step(cuda, case, z, dtype, fn=None):
    """One DnetHead.loss step (or ``fn(head, x, gt, gtm)``) of a golden case with the heads in ``dtype``; cuDNN without
    TF32.  With float64 heads DnetHead.loss casts their outputs to fp32 for the loss kernel, so the only fp32
    arithmetic left is the loss's own."""
    head = _golden_head(cuda, case).to(dtype)
    x, gt, _ = dr.golden_inputs()
    x = x.to(cuda, dtype).requires_grad_()
    gt, gtm = gt.to(cuda), torch.from_numpy(z["gt_mask"]).to(cuda)
    with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
        loss = head.loss(x, gt, gtm) if fn is None else fn(head, x, gt, gtm)
        loss.backward()
    return _golden_errors(z, loss, x, head)


def test_dnet_head_loss_matches_the_reference(cuda):
    """DnetHead.loss against the reference's Decoder heads + upsample_depth_via_mask + activation_G + DnetLoss on the
    ordinary golden case (moderate negative and large positive v, no collapsed pixel; tests/dnet_loss_ref.py).

    With the heads in float64 the only fp32 arithmetic is the reference's and the fused loss's: the loss within 2e-5
    relative and every gradient (x_feat, each head parameter) within 2e-5 of its maximum, as the MagnetLoss golden test.
    With fp32 heads on cuDNN (what training runs), the convolutions' own fp32 rounding on the GPU is 1.6e-5 of a
    maximum from float64 here (the reference's CPU convolutions: 4e-6), the same for any loss behind them; so each
    gradient is held to be no further from the reference than the module route's (the same heads, DnetHead.forward +
    DnetLoss in torch) plus 5e-6, and the loss to 2e-5."""
    z = _golden("ordinary")
    assert int(z["n_deep"]) == 0 and int(z["n_neg"]) > 0 and int(z["n_high"]) > 0
    loss_err, errs = _golden_step(cuda, "ordinary", z, torch.float64)
    print("float64 heads", f"{loss_err:.3g}", {k: f"{v:.2g}" for k, v in errs.items()})
    assert loss_err <= 2e-5 and max(errs.values()) <= 2e-5, (loss_err, errs)
    loss_err, errs = _golden_step(cuda, "ordinary", z, torch.float32)
    _, module = _golden_step(cuda, "ordinary", z, torch.float32, lambda h, x, g, m: _module_route_loss(h, x, g, m))
    print("fp32 heads", f"{loss_err:.3g}", {k: f"{v:.2g}/{module[k]:.2g}" for k, v in errs.items()})
    assert loss_err <= 2e-5, loss_err
    for name, err in errs.items():
        assert err <= module[name] + 5e-6, (name, err, module[name])


def test_dnet_head_loss_matches_the_reference_where_var_collapses(cuda):
    """The collapsed golden case: pixels with v_up <= -17.5 (var exactly 1e-10) next to ordinary and large positive
    ones.  The loss within 2e-5 relative; every gradient within 1e-4 of its maximum.  The collapsed pixels make up the
    whole loss and send gradients 1e10 times the others' into the heads, where they cancel: in the logits' softmax
    gradient (mu_i - mu_up of neighbouring pixels) and in the heads' backward.  On this input the reference's own fp32
    backward of the heads differs from a float64 one, on the same loss gradients, by 2.7e-5 of a maximum, so no fp32
    implementation can be held to 2e-5 of it; this case checks the collapsed regime, the ordinary one the rest."""
    z = _golden("collapsed")
    assert int(z["n_deep"]) > 0
    loss_err, errs = _golden_step(cuda, "collapsed", z, torch.float32)
    print("collapsed", f"{loss_err:.3g}", {k: f"{v:.2g}" for k, v in errs.items()})
    assert loss_err <= 2e-5 and max(errs.values()) <= 1e-4, (loss_err, errs)


def _module_route_loss(head, x, gt, gtm):
    """DnetHead.forward in train mode (module chain) + DnetLoss as a user writes it, with boolean indexing."""
    pred = head(x)
    mu, var = torch.split(pred, 1, dim=1)
    g, mu, var = gt[gtm], mu[gtm], var[gtm]
    var = torch.where(var < 1e-10, torch.full_like(var, 1e-10), var)
    return (torch.square(mu - g) / (2 * var) + 0.5 * torch.log(var)).mean()


@pytest.mark.parametrize("B,h,w", [(2, 26, 34), (3, 22, 44)])
def test_dnet_head_loss_matches_the_module_route(cuda, B, h, w):
    torch.manual_seed(B)
    head = DnetHead(in_dim=64).to(cuda).train()
    ref = copy.deepcopy(head)
    x = torch.relu(torch.randn(B, 64, h, w, device=cuda))
    gt = 1.0 + 9.0 * torch.rand(B, 1, 4 * h, 4 * w, device=cuda)
    gtm = torch.rand(B, 1, 4 * h, 4 * w, device=cuda) < 0.6
    x1, x2 = x.clone().requires_grad_(), x.clone().requires_grad_()
    with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
        loss = head.loss(x1, gt, gtm)
        loss.backward()
        want = _module_route_loss(ref, x2, gt, gtm)
        want.backward()
    assert abs(float(loss) - float(want)) <= 2e-5 * abs(float(want))
    pairs = [("x", x1.grad, x2.grad)] + [(n, p.grad, q.grad) for (n, p), (_, q) in
                                         zip(head.named_parameters(), ref.named_parameters())]
    for name, got, exp in pairs:
        err, scale = float((got - exp).abs().max()), float(exp.abs().max())
        assert err <= 1e-4 * scale, (name, err, scale)


def test_dnet_head_loss_under_autocast(cuda):
    """Under torch.autocast (fp16) the heads' convolutions run in half precision and their outputs are upcast once
    before the fp32 loss kernel: the loss is fp32, within 5e-3 of the fp32 step's (the heads' half-precision rounding),
    and it and every gradient (x_feat, each head parameter, all fp32) agree with the module route under the same
    autocast (DnetHead.forward, which upcasts before its upsampling, + DnetLoss in torch) to 1e-5 of the loss and 1e-3
    of each gradient's maximum (both routes run the same half-precision convolutions on gradients that differ in fp32
    rounding only)."""
    torch.manual_seed(11)
    head = DnetHead(in_dim=64).to(cuda)
    ref, full = copy.deepcopy(head), copy.deepcopy(head)
    x = torch.relu(torch.randn(2, 64, 26, 34, device=cuda))
    gt = 1.0 + 9.0 * torch.rand(2, 1, 104, 136, device=cuda)
    gtm = torch.rand(2, 1, 104, 136, device=cuda) < 0.6
    x1, x2 = x.clone().requires_grad_(), x.clone().requires_grad_()
    with torch.autocast("cuda", dtype=torch.float16):
        assert head.depth_head(x1).dtype == torch.float16                     # the heads do run in half precision
        loss = head.loss(x1, gt, gtm)
        want = _module_route_loss(ref, x2, gt, gtm)
    loss.backward()
    want.backward()
    with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
        fp32 = full.loss(x.clone().requires_grad_(), gt, gtm)
    assert loss.dtype == torch.float32
    assert abs(float(loss) - float(fp32)) <= 5e-3 * abs(float(fp32)), (float(loss), float(fp32))
    assert abs(float(loss) - float(want)) <= 1e-5 * abs(float(want)), (float(loss), float(want))
    pairs = [("x", x1.grad, x2.grad)] + [(n, p.grad, q.grad) for (n, p), (_, q) in
                                         zip(head.named_parameters(), ref.named_parameters())]
    errs = {}
    for name, got, exp in pairs:
        assert got.dtype == torch.float32 and torch.isfinite(got).all() and torch.isfinite(exp).all(), name
        errs[name] = float((got - exp).abs().max()) / float(exp.abs().max())
    print("autocast", {k: f"{v:.2g}" for k, v in errs.items()})
    assert max(errs.values()) <= 1e-3, errs


def test_empty_mask_raises_eagerly(cuda):
    head = DnetHead(in_dim=16).to(cuda)
    x = torch.rand(1, 16, 5, 6, device=cuda)
    with pytest.raises(_lib.MagnetError, match="no pixel"):
        head.loss(x, torch.rand(1, 1, 20, 24, device=cuda), torch.zeros(1, 1, 20, 24, dtype=torch.bool, device=cuda))


def test_loss_is_bit_identical_run_to_run(cuda):
    raw, lg, gt, gtm, _ = dr.loss_inputs(16, 104, 136, 4, deep=8, high=8, seed=81)
    raw, lg, gt, gtm = raw.to(cuda), lg.to(cuda), gt.to(cuda), gtm.to(cuda)
    first = ops.dnet_loss(raw, lg, gt, gtm, 4)
    for _ in range(3):
        assert torch.equal(ops.dnet_loss(raw, lg, gt, gtm, 4), first)


# ---------------------------------------------------------------------------------------------------------------------
# torch.compile and CUDA graphs

def _leaf_step(fn, raw, lg, gt, gtm):
    raw_l, lg_l = raw.clone().requires_grad_(), lg.clone().requires_grad_()
    loss = fn(raw_l, lg_l, gt, gtm)
    loss.backward()
    return loss.detach(), raw_l.grad, lg_l.grad


@pytest.mark.parametrize("k", [2, 4, 8])
def test_compiled_loss_equals_eager(cuda, k):
    """fullgraph: the loss is torch.equal to eager's and the mask gradient (written once per element) too; the raw
    gradient (accumulated with atomic adds) within 16 fp32 ulps of its maximum."""
    torch._dynamo.reset()
    raw, lg, gt, gtm, _ = dr.loss_inputs(4, 26, 34, k, deep=4, high=4, seed=90 + k)
    raw, lg, gt, gtm = raw.to(cuda), lg.to(cuda), gt.to(cuda), gtm.to(cuda)
    fn = lambda r, m, g, gm: ops.dnet_loss(r, m, g, gm, k)
    want = _leaf_step(fn, raw, lg, gt, gtm)
    got = _leaf_step(torch.compile(fn, fullgraph=True), raw, lg, gt, gtm)
    assert torch.equal(got[0], want[0]), (float(got[0]), float(want[0]))
    assert torch.equal(got[2], want[2])
    scale = float(want[1].abs().max())
    assert float((got[1] - want[1]).abs().max()) <= 16 * 2.0 ** -23 * scale


def test_dnet_head_loss_traces_without_graph_breaks(cuda):
    torch._dynamo.reset()
    head = DnetHead(in_dim=32).to(cuda)
    x = torch.rand(2, 32, 12, 16, device=cuda, requires_grad=True)
    gt, gtm = torch.rand(2, 1, 48, 64, device=cuda) + 1.0, torch.rand(2, 1, 48, 64, device=cuda) < 0.5
    e = torch._dynamo.explain(head.loss)(x, gt, gtm)
    assert e.graph_break_count == 0, [r.reason[:300] for r in e.break_reasons]
    loss = torch.compile(head.loss, fullgraph=True)(x, gt, gtm)
    loss.backward()
    assert torch.isfinite(loss) and x.grad is not None and head.depth_head[0].weight.grad is not None
    assert head.mask_head[0].weight.grad is not None


def _head_grads(head, x):
    return [x.grad] + [p.grad for p in head.parameters()]


def test_reduce_overhead_step_equals_eager(cuda):
    """Three DnetHead.loss steps under CUDA-graph trees with new inputs copied into static buffers: each loss within
    1e-6 relative of the eager step's, every cuDNN-side gradient within 1e-5 of its maximum, and no graph skipped."""
    with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
        _reduce_overhead_steps(cuda)


def _reduce_overhead_steps(cuda):
    from torch._dynamo.utils import counters
    torch._dynamo.reset()
    torch.manual_seed(5)
    head = DnetHead(in_dim=64).to(cuda)
    eager = copy.deepcopy(head)
    B, h, w = 4, 26, 34
    static = [torch.empty(B, 64, h, w, device=cuda), torch.empty(B, 1, 4 * h, 4 * w, device=cuda),
              torch.empty(B, 1, 4 * h, 4 * w, device=cuda, dtype=torch.bool)]
    compiled = torch.compile(head.loss, mode="reduce-overhead")
    counters.clear()
    for i in range(3):
        g = torch.Generator(device=cuda).manual_seed(100 + i)
        new = [torch.relu(torch.randn(B, 64, h, w, device=cuda, generator=g)),
               1.0 + 9.0 * torch.rand(B, 1, 4 * h, 4 * w, device=cuda, generator=g),
               torch.rand(B, 1, 4 * h, 4 * w, device=cuda, generator=g) < 0.6]
        for s, n in zip(static, new):
            s.copy_(n)
        for m in (head, eager):
            m.zero_grad(set_to_none=True)
        xs, xe = static[0].clone().requires_grad_(), new[0].clone().requires_grad_()
        got = compiled(xs, static[1], static[2])
        got.backward()
        want = eager.loss(xe, new[1], new[2])
        want.backward()
        assert abs(float(got) - float(want)) <= 1e-6 * abs(float(want)), (i, float(got), float(want))
        for a, b in zip(_head_grads(head, xs), _head_grads(eager, xe)):
            assert float((a - b).abs().max()) <= 1e-5 * float(b.abs().max()), i
    assert not counters["inductor"]["cudagraph_skips"], dict(counters["inductor"])


def test_compiled_empty_mask_gives_nan_and_zero_gradients(cuda):
    torch._dynamo.reset()
    raw, lg, gt, _, _ = dr.loss_inputs(2, 6, 7, 4, seed=3)
    raw, lg, gt = raw.to(cuda), lg.to(cuda), gt.to(cuda)
    none = torch.zeros_like(gt, dtype=torch.bool)
    loss, g_raw, g_mask = _leaf_step(torch.compile(lambda r, m, g, gm: ops.dnet_loss(r, m, g, gm, 4), fullgraph=True),
                                     raw, lg, gt, none)
    assert torch.isnan(loss)
    assert torch.equal(g_raw, torch.zeros_like(g_raw)) and torch.equal(g_mask, torch.zeros_like(g_mask))


def test_compiled_loss_reads_a_strided_mask(cuda):
    """A non-contiguous bool mask (a transposed one) gives the compiled loss and gradients of its contiguous copy: the
    kernels read the mask by address, so both ops take it through the same contiguous check."""
    torch._dynamo.reset()
    raw, lg, gt, gtm, _ = dr.loss_inputs(2, 12, 12, 4, mask="sparse", seed=7)
    raw, lg, gt = raw.to(cuda), lg.to(cuda), gt.to(cuda)
    strided = gtm.to(cuda).transpose(2, 3).contiguous().transpose(2, 3)
    assert not strided.is_contiguous() and torch.equal(strided, gtm.to(cuda))
    fn = torch.compile(lambda r, m, g, gm: ops.dnet_loss(r, m, g, gm, 4), fullgraph=True)
    got = _leaf_step(fn, raw, lg, gt, strided)
    want = _leaf_step(fn, raw, lg, gt, strided.contiguous())
    assert torch.equal(got[0], want[0]) and torch.equal(got[2], want[2])
    assert float((got[1] - want[1]).abs().max()) <= 16 * 2.0 ** -23 * float(want[1].abs().max())
