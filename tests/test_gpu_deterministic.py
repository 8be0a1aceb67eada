"""Reproducible training under torch.use_deterministic_algorithms (DESIGN §3.20).

- Every fixed-order (``_det``) entry point, through its Python wrapper with the flag on, gives bit-identical results
  over runs at the cfg2 and cfg3 training shapes: on the default stream, on a side stream, replayed from a CUDA graph
  and with unrelated kernels running on another stream.
- Its outputs equal the atomic path's where both write in a fixed order (the mask-logit gradients, the loss partials
  and saved maps) and agree with it to fp32 rounding where the atomic path adds in any order.
- The existing float64 checks of the upsampling backwards, the fused mask-loss forward and DnetLoss pass unchanged with
  the flag on, where the ``_det`` forms run (a subprocess).
- End to end, in a subprocess with CUBLAS_WORKSPACE_CONFIG: two steps from one seed give equal gradients for every
  parameter and input of the MaGNet head (module path, convex upsampling, fused_upsample, fused_train) and of
  DnetHead.loss, eager and under torch.compile's reduce-overhead mode.  The two training paths whose matching-volume
  backward has no deterministic form yet raise: F-Net training (MagnetF.loss) and fine-tuning a stand-in F-Net through
  the CW volume (detach_cost=False).
"""
import os
import subprocess
import sys

import pytest
import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import magnet_b200  # noqa: E402
from magnet_b200 import ops  # noqa: E402

SHAPES = {"cfg2": (8, 120, 160), "cfg3": (4, 88, 304)}      # quarter-resolution B, H, W of bench.py's workloads; k = 4
ENV = {**os.environ, "CUBLAS_WORKSPACE_CONFIG": ":4096:8"}


@pytest.fixture
def det_flag():
    saved = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(saved[0], warn_only=saved[1])


def _inputs(dev, B, H, W, seed=0):
    g = torch.Generator(device=dev).manual_seed(seed)
    rnd = lambda *s: torch.randn(*s, device=dev, generator=g)
    uni = lambda *s: torch.rand(*s, device=dev, generator=g)
    full = (B, 1, 4 * H, 4 * W)
    depth = torch.cat([0.5 + 5 * uni(B, 1, H, W), 0.05 + uni(B, 1, H, W)], 1)
    raw = torch.cat([0.5 + 5 * uni(B, 1, H, W), 2 * rnd(B, 1, H, W)], 1)
    return dict(depth=depth, raw=raw, up=3 * rnd(B, 144, H, W), gout=rnd(B, 2, 4 * H, 4 * W), gt=0.5 + 5 * uni(*full),
                gtm=(uni(*full) > 0.2).to(torch.uint8), pre0=rnd(B, 128, H, W),
                ws=[0.05 * rnd(*s) for _, s in ops.mask_weight_shapes()],
                preds=[depth + 0.1 * i for i in range(3)], scale=torch.full((1,), 1e-5, device=dev),
                scales=torch.tensor([0.64e-5, 0.8e-5, 1e-5], device=dev))


# name -> (call on the inputs returning its outputs, the outputs written in a fixed order on the atomic path too)
CALLS = {
    "convex_ch1": (lambda x: ops.convex_upsample_bwd(x["gout"][:, :1].contiguous(), x["depth"][:, :1].contiguous(),
                                                     x["up"], 4), (1,)),
    "convex_ch2": (lambda x: ops.convex_upsample_bwd(x["gout"], x["depth"], x["up"], 4), (1,)),
    "nll": (lambda x: ops.upsample_nll_bwd(x["depth"], x["up"], x["gt"], x["gtm"], 4, 1e-5), (1,)),
    "nll_dev": (lambda x: ops.upsample_nll_bwd(x["depth"], x["up"], x["gt"], x["gtm"], 4, x["scale"]), (1,)),
    "dnet": (lambda x: ops.upsample_nll_bwd(x["raw"], x["up"], x["gt"], x["gtm"], 4, 1e-5, True), (1,)),
    "dnet_dev": (lambda x: ops.upsample_nll_bwd(x["raw"], x["up"], x["gt"], x["gtm"], 4, x["scale"], True), (1,)),
    # (partials, saved): saved holds the 3 prediction gradients, then the maps
    "mask": (lambda x: ops.mask_train_fwd(x["pre0"], x["ws"], x["preds"], x["gt"], x["gtm"], True, True,
                                          [0.64e-5, 0.8e-5, 1e-5])[::2], (0,)),
    "mask_dev": (lambda x: ops.mask_train_fwd(x["pre0"], x["ws"], x["preds"], x["gt"], x["gtm"], True, True,
                                              x["scales"])[::2], (0,)),
}


def _clone(outs):
    return [t.clone() for t in outs]


def _runs(fn):
    """fn's outputs in each setting: the default stream, a side stream, a CUDA-graph replay and next to unrelated work."""
    cur = torch.cuda.current_stream()
    yield "default", _clone(fn())
    side = torch.cuda.Stream()
    side.wait_stream(cur)
    with torch.cuda.stream(side):
        out = _clone(fn())
    cur.wait_stream(side)
    yield "side stream", out
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = fn()
    for _ in range(2):
        graph.replay()
    torch.cuda.synchronize()
    yield "graph replay", _clone(captured)
    busy, other = torch.cuda.Stream(), torch.empty(1 << 26, device="cuda").fill_(1.0)
    busy.wait_stream(cur)
    with torch.cuda.stream(busy):
        for _ in range(50):
            other.mul_(1.0001).add_(1e-4)
    out = _clone(fn())
    cur.wait_stream(busy)
    torch.cuda.synchronize()
    yield "concurrent work", out


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CALLS))
@pytest.mark.parametrize("shape", list(SHAPES))
def test_det_entry_points_repeat_bit_for_bit(cuda, det_flag, name, shape):
    x = _inputs(cuda, *SHAPES[shape])
    fn = lambda: CALLS[name][0](x)
    first = None
    for setting, outs in _runs(fn):
        if first is None:
            first = outs
            assert all(torch.isfinite(t).all() for t in outs), name
            continue
        for i, (a, b) in enumerate(zip(first, outs)):
            assert torch.equal(a, b), (name, setting, i, (a - b).abs().max().item())


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CALLS))
def test_det_entry_points_agree_with_the_atomic_path(cuda, name):
    """The same rounded terms in another order: fixed-order outputs equal bit for bit, the sums within fp32 rounding of
    their largest partial sum."""
    x = _inputs(cuda, *SHAPES["cfg3"], seed=3)
    fn, exact = CALLS[name]
    assert not torch.are_deterministic_algorithms_enabled()
    atomic = _clone(fn(x))
    torch.use_deterministic_algorithms(True)
    try:
        det = _clone(fn(x))
    finally:
        torch.use_deterministic_algorithms(False)
    for i, (a, d) in enumerate(zip(atomic, det)):
        if name.startswith("mask") and i == 1:                  # saved: the maps after the prediction gradients
            n = 3 * x["depth"].numel()
            assert torch.equal(a[n:], d[n:]), name
            a, d = a[:n], d[:n]
        elif i in exact:
            assert torch.equal(a, d), (name, i)
            continue
        # at most 9*16 terms per element, each sum within 144 ulps of its magnitude in any order
        tol = 144 * 2.0 ** -23 * a.abs().max().item()
        assert (a - d).abs().max().item() <= tol, (name, i)


F64_TESTS = ["tests/test_gpu_aux_f64.py::test_convex_upsample", "tests/test_gpu_aux_f64.py::test_magnet_loss",
             "tests/test_gpu_mask_train.py::test_gradients_match_float64",
             "tests/test_gpu_mask_train.py::test_gradients_at_production_shapes",
             "tests/test_gpu_dnet_loss.py::test_loss_and_gradients_within_the_float64_bound"]


def _subprocess(args, timeout):
    """Run ``python args`` from the repository root; the process is killed if it outlives ``timeout`` seconds."""
    p = subprocess.Popen([sys.executable, *args], cwd=ROOT, env=ENV, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                         text=True)
    try:
        out, _ = p.communicate(timeout=timeout)
    finally:
        if p.poll() is None:
            p.kill()
            p.communicate()
    return p.returncode, out


@pytest.mark.gpu
def test_float64_checks_hold_with_the_flag_on(cuda):
    code = ("import sys, torch, pytest; torch.use_deterministic_algorithms(True); "
            f"sys.exit(pytest.main(['-q', '-p', 'no:cacheprovider', *{F64_TESTS!r}]))")
    rc, out = _subprocess(["-c", code], timeout=1500)
    assert rc == 0, out[-4000:]


# --- end to end ------------------------------------------------------------------------------------------------------

def _batch(dev, B, V, D, H, W, seed=1):
    from magnet_b200.synthetic import make_inputs
    inp = make_inputs(B=B, V=V, D=D, H=H, W=W, C=64, seed=seed)
    g = inp.to(dev)
    cam = {k: v.to(dev) for k, v in inp.cam_intrins.items()}
    gen = torch.Generator(device=dev).manual_seed(seed)
    x_d3 = torch.randn(B, 256, H, W, device=dev, generator=gen).requires_grad_(True)
    gt = nn.functional.interpolate(g.ref_gmms[:, :1] * 1.03, scale_factor=4, mode="nearest")
    gt = gt * (torch.rand(B, 1, 4 * H, 4 * W, device=dev, generator=gen) > 0.2)
    return (g.ref_feat, g.nghbr_feat, g.ref_gmms, g.nghbr_gmms, x_d3, g.nghbr_poses, inp.is_valid.to(dev), cam), gt


def _compiled(fn):
    return torch.compile(fn, mode="reduce-overhead")


def _head_step(case, dev):
    torch.manual_seed(0)
    fused = case in ("fused_upsample", "fused_train", "compiled_fused_upsample")
    head = magnet_b200.MagnetHead(n_samples=5, fused_train=case == "fused_train",
                                  fused_upsample=fused).to(dev).train()
    args, gt = _batch(dev, B=4, V=4, D=5, H=120, W=160)
    if case == "module":
        fn = lambda: head.loss(*head.forward_quarter(*args), gt, gt > 0)
    elif case == "full_res":                               # full-resolution predictions: convex_upsample's backward
        def fn():
            m = (gt > 0).float()
            loss = 0.0
            for p in head(*args):
                var = torch.square(p[:, 1:2]).clamp_min(1e-10)
                loss = loss + ((torch.square(p[:, :1] - gt) / (2 * var) + 0.5 * torch.log(var)) * m).sum() / m.sum()
            return loss
    elif case == "compiled_module":
        step = _compiled(lambda *a: head.loss(*head.forward_quarter(*a), gt, gt > 0))
        fn = lambda: step(*args)
    elif case == "compiled_fused_upsample":
        step = _compiled(lambda *a: head.train_loss(*a, gt, gt > 0))
        fn = lambda: step(*args)
    else:
        fn = lambda: head.train_loss(*args, gt, gt > 0)
    return fn, [("x_d3", args[4]), *head.named_parameters()]


def _dnet_step(dev, compiled):
    torch.manual_seed(0)
    head = magnet_b200.DnetHead(in_dim=64).to(dev).train()
    gen = torch.Generator(device=dev).manual_seed(2)
    x = torch.randn(4, 64, 104, 136, device=dev, generator=gen).requires_grad_(True)
    gt = 0.5 + 5 * torch.rand(4, 1, 416, 544, device=dev, generator=gen)
    gtm = torch.rand(4, 1, 416, 544, device=dev, generator=gen) > 0.3
    loss = lambda x_feat: head.loss(x_feat, gt, gtm)
    step = _compiled(loss) if compiled else loss
    return lambda: step(x), [("x_feat", x), *head.named_parameters()]


def _refused(what: str, step) -> None:
    """``step`` (forward + backward) must raise, naming the entry point ``what`` that has no deterministic form."""
    try:
        step()
    except RuntimeError as e:
        assert what in str(e), e
        print("refused:", str(e)[:200])
        return
    raise AssertionError(f"{what} ran under the deterministic flag")


def _grads(fn, named):
    for _, t in named:
        t.grad = None
    loss = fn()
    loss.backward()
    return loss.detach().clone(), {n: t.grad.clone() for n, t in named if t.grad is not None}


def _e2e(case: str) -> None:
    """Two steps of ``case`` under the flag; exits non-zero unless loss and every gradient repeat bit for bit."""
    torch.use_deterministic_algorithms(True)
    torch.backends.cudnn.benchmark = False
    dev = torch.device("cuda:0")
    from magnet_b200.synthetic import make_inputs
    if case == "fnet_refused":                             # the F volume's grad_src has no deterministic form
        f = nn.Sequential(nn.Conv2d(3, 64, 3, stride=4, padding=1))
        model = magnet_b200.MagnetF(f).to(dev).train()
        inp = make_inputs(B=1, V=2, D=8, H=30, W=40, C=64, seed=5)
        cam = {k: v.to(dev) for k, v in inp.cam_intrins.items()}
        imgs = torch.randn(3, 3, 120, 160, device=dev)
        planes = magnet_b200.sid_planes(1e-3, 10.0, 80).flatten().tolist()
        _refused("magnet_cost_volume_f_bwd_f32", lambda: model.loss(
            imgs[:1], imgs[1:], inp.to(dev).nghbr_poses, inp.is_valid.to(dev), cam, planes,
            5 * torch.rand(1, 1, 120, 160, device=dev), 1e-3, 10.0).backward())
        return
    if case == "cw_finetune_refused":                      # nor does the CW volume's: a trainable F-Net upstream
        B, V, H, W = 1, 2, 30, 40
        inp = make_inputs(B=B, V=V, D=5, H=H, W=W, C=64, seed=21)
        g = inp.to(dev)
        cam = {k: v.to(dev) for k, v in inp.cam_intrins.items()}
        fnet = nn.Conv2d(3, 64, 3, padding=1).to(dev)
        head = magnet_b200.MagnetHead(n_samples=5, n_iter=2, thres=inp.thres, detach_cost=False).to(dev).train()
        imgs = torch.randn(B * (V + 1), 3, H, W, device=dev)
        x_d3 = torch.randn(B, 256, H, W, device=dev)

        def step():
            feat = fnet(imgs)
            preds, _ = head.forward_quarter(feat[:B], feat[B:], g.ref_gmms, g.nghbr_gmms, x_d3, g.nghbr_poses,
                                            inp.is_valid.to(dev), cam)
            sum(p.square().mean() for p in preds).backward()
        _refused("magnet_cost_volume_bwd_f32", step)
        return
    compiled = case.startswith("compiled")
    fn, named = _dnet_step(dev, compiled) if case.endswith("dnet") else _head_step(case, dev)
    runs = [_grads(fn, named) for _ in range(3 if compiled else 2)]
    a, b = runs[-2], runs[-1]                              # compiled: the first call records the graphs
    assert torch.equal(a[0], b[0]), (case, a[0].item(), b[0].item())
    assert set(a[1]) == set(b[1]) and a[1], case
    bad = [n for n in a[1] if not torch.equal(a[1][n], b[1][n])]
    assert not bad, (case, bad)
    print(f"{case}: loss and {len(a[1])} gradients repeat bit for bit")


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["module", "full_res", "fused_upsample", "fused_train", "dnet", "compiled_module",
                                  "compiled_fused_upsample", "compiled_dnet", "fnet_refused", "cw_finetune_refused"])
def test_training_steps_repeat_bit_for_bit(cuda, case):
    rc, out = _subprocess([os.path.abspath(__file__), case], timeout=900)
    assert rc == 0, out[-4000:]


if __name__ == "__main__":
    _e2e(sys.argv[1])
