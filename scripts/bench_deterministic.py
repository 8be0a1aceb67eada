"""The cost of reproducible training (DESIGN §3.20): each backward that has a fixed-order (``_det``) form, and whole
training steps, with torch.use_deterministic_algorithms off (the atomic entry points) and on (the ``_det`` ones).

Kernels, at bench.py's cfg2 (ScanNet, quarter resolution B 8, 120x160) and cfg3 (KITTI, B 4, 88x304), k = 4:
  convex   ops.convex_upsample_bwd, 2 channels (MagnetHead.forward's full-resolution predictions in training);
  nll      ops.upsample_nll_bwd, MagnetLoss form, device scale (MagnetHead.loss under torch.compile);
  dnet     the same in the DnetLoss form (DnetHead.loss);
  mask     ops.mask_train_fwd with the prediction gradients, P = 3 (MagnetHead.train_loss with fused_upsample).
Steps (forward + backward, zero_grad included), B 4:
  head_module  MagnetHead.forward_quarter + loss, N_s 5, 120x160, V 4;
  head_fused   MagnetHead(fused_train, fused_upsample).train_loss, the same shape;
  dnet_loss    DnetHead.loss, 64 trunk channels, 104x136.
The matching volumes' backwards have no ``_det`` form (the package refuses them under the flag), so F-Net training and
fine-tuning through the CW volume are not measured.

Each timed window runs --steps calls of one mode between CUDA events; the modes alternate window by window for --repeats
windows and the median and range per mode are reported.  Beside the times: the workspace the ``_det`` form adds
(computed from the shape by the library) and the peak device memory of one call in each mode.  Under the flag torch
also fills every new allocation with NaN (torch.utils.deterministic.fill_uninitialized_memory), the ``_det`` workspaces
included.  The kernel rows are timed with that fill off, so that they compare the kernels alone; the step rows keep
torch's default (fill on under the flag), what a user's reproducible step pays.  Each JSON line records the setting as
"nan_fill", with the card and its power limit; writes nothing.

usage: python scripts/bench_deterministic.py [--steps K] [--warmup W] [--repeats R]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")

import torch  # noqa: E402
import torch.nn as nn  # noqa: E402
import torch.utils.deterministic  # noqa: E402

import magnet_b200  # noqa: E402
from magnet_b200 import _lib, ops  # noqa: E402

SHAPES = {"cfg2": (8, 120, 160), "cfg3": (4, 88, 304)}


def _card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=30).stdout.strip()
    name, power = [s.strip() for s in q.splitlines()[0].split(",")]
    return {"card": name, "power_limit": power}


def _kernel_cases(dev, B, H, W):
    g = torch.Generator(device=dev).manual_seed(0)
    rnd = lambda *s: torch.randn(*s, device=dev, generator=g)
    uni = lambda *s: torch.rand(*s, device=dev, generator=g)
    full = (B, 1, 4 * H, 4 * W)
    depth = torch.cat([0.5 + 5 * uni(B, 1, H, W), 0.05 + uni(B, 1, H, W)], 1)
    raw = torch.cat([depth[:, :1], 2 * rnd(B, 1, H, W)], 1)
    up, gout, gt, gtm = 3 * rnd(B, 144, H, W), rnd(B, 2, 4 * H, 4 * W), 0.5 + 5 * uni(*full), (uni(*full) > 0.2).to(torch.uint8)
    scale = torch.full((1,), 1e-6, device=dev)
    pre0, ws = rnd(B, 128, H, W), [0.05 * rnd(*s) for _, s in ops.mask_weight_shapes()]
    preds = [depth + 0.1 * i for i in range(3)]
    L = _lib.lib()
    nll_ws = int(L.magnet_upsample_nll_bwd_det_workspace_bytes(B, H, W, 4))
    return {
        "convex": (lambda: ops.convex_upsample_bwd(gout, depth, up, 4), 0),
        "nll": (lambda: ops.upsample_nll_bwd(depth, up, gt, gtm, 4, scale), nll_ws),
        "dnet": (lambda: ops.upsample_nll_bwd(raw, up, gt, gtm, 4, scale, True), nll_ws),
        "mask": (lambda: ops.mask_train_fwd(pre0, ws, preds, gt, gtm, False, True, [1e-6] * 3),
                 int(L.magnet_mask_train_det_workspace_bytes(3, B, H, W))),
    }


def _step_cases(dev):
    from magnet_b200.synthetic import make_inputs
    B, V, D, H, W = 4, 4, 5, 120, 160
    inp = make_inputs(B=B, V=V, D=D, H=H, W=W, C=64, seed=1)
    gi = inp.to(dev)
    cam = {k: v.to(dev) for k, v in inp.cam_intrins.items()}
    gen = torch.Generator(device=dev).manual_seed(1)
    x_d3 = torch.randn(B, 256, H, W, device=dev, generator=gen).requires_grad_(True)
    gt = nn.functional.interpolate(gi.ref_gmms[:, :1] * 1.03, scale_factor=4, mode="nearest")
    gt = gt * (torch.rand(B, 1, 4 * H, 4 * W, device=dev, generator=gen) > 0.2)
    args = (gi.ref_feat, gi.nghbr_feat, gi.ref_gmms, gi.nghbr_gmms, x_d3, gi.nghbr_poses, inp.is_valid.to(dev), cam)
    module = magnet_b200.MagnetHead(n_samples=D).to(dev).train()
    fused = magnet_b200.MagnetHead(n_samples=D, fused_train=True, fused_upsample=True).to(dev).train()
    dnet = magnet_b200.DnetHead(in_dim=64).to(dev).train()
    xf = torch.randn(B, 64, 104, 136, device=dev, generator=gen).requires_grad_(True)
    dgt = 0.5 + 5 * torch.rand(B, 1, 416, 544, device=dev, generator=gen)
    dgtm = torch.rand(B, 1, 416, 544, device=dev, generator=gen) > 0.3

    def step(model, loss_fn, leaf):
        def run():
            model.zero_grad(set_to_none=True)
            leaf.grad = None
            loss_fn().backward()
        return run
    return {
        "head_module": (step(module, lambda: module.loss(*module.forward_quarter(*args), gt, gt > 0), x_d3), None),
        "head_fused": (step(fused, lambda: fused.train_loss(*args, gt, gt > 0), x_d3), None),
        "dnet_loss": (step(dnet, lambda: dnet.loss(xf, dgt, dgtm), xf), None),
    }


def _window(fn, det, steps):
    torch.use_deterministic_algorithms(det)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / steps


def _peak(fn, det):
    torch.use_deterministic_algorithms(det)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 1e6


def measure(name, shape, fn, ws_bytes, args, card, nan_fill):
    torch.utils.deterministic.fill_uninitialized_memory = nan_fill
    for det in (False, True):
        torch.use_deterministic_algorithms(det)
        for _ in range(args.warmup):
            fn()
    times = {False: [], True: []}
    for _ in range(args.repeats):
        for det in (False, True):
            times[det].append(_window(fn, det, args.steps))
    rec = {"case": name, "shape": shape, **card, "steps": args.steps, "repeats": args.repeats, "nan_fill": nan_fill}
    for det, tag in ((False, "atomic"), (True, "det")):
        t = times[det]
        rec[f"{tag}_ms_median"] = round(statistics.median(t), 4)
        rec[f"{tag}_ms_range"] = [round(min(t), 4), round(max(t), 4)]
        rec[f"{tag}_peak_MB"] = round(_peak(fn, det), 1)
    rec["det_over_atomic"] = round(rec["det_ms_median"] / rec["atomic_ms_median"], 3)
    if ws_bytes is not None:
        rec["det_workspace_MB"] = round(ws_bytes / 1e6, 1)
    torch.use_deterministic_algorithms(False)
    print(json.dumps(rec), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=7)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_deterministic.py needs a CUDA device")
    dev = torch.device("cuda:0")
    card = _card()
    torch.backends.cudnn.benchmark = False              # cuDNN's algorithm choice is then the same in both modes
    for shape, (B, H, W) in SHAPES.items():
        for name, (fn, ws) in _kernel_cases(dev, B, H, W).items():
            measure(name, shape, fn, ws, args, card, nan_fill=False)
    for name, (fn, ws) in _step_cases(dev).items():
        measure(name, "B4", fn, ws, args, card, nan_fill=True)


if __name__ == "__main__":
    main()
