"""Training steps eager against torch.compile (default) and torch.compile(mode="reduce-overhead") of the loss function.

Each timed step is the loss function's forward followed by ``loss.backward()``, so the compiled backward is timed too;
the optimizer is not part of the step.  Before timing, the compiled losses and gradients are checked against eager's
(TF32 off, deterministic cuDNN, as in tests/test_gpu_compile_train.py); the timing runs with the backend settings the
script was started with, printed in the first line.  Eager, default and reduce-overhead alternate
within one call; each is timed with CUDA events over windows of ``--iters`` steps, every shape warmed up first, and the
median and range over ``--reps`` windows are printed with the card and its power limit read in the same call.

Workloads (cameras and validity on the device, inputs fixed across steps):
  head-module: MagnetHead.forward_quarter + loss (cuDNN G-Net and mask head, upsample-NLL kernels);
  head-fused:  MagnetHead(fused_train, fused_upsample).train_loss (fused G-Net and mask-loss kernels);
  at ScanNet B 4, V 4, 120x160, N_iter 3, N_s 5 and 64, and KITTI B 4, V 2, 88x304, N_s 5;
  fnet:        MagnetF.loss with a stand-in F-Net of three convolutions over 80 SID planes, ScanNet B 2 V 4 and KITTI
               B 4 V 2; the stand-in's own forward + backward is timed alone and reported as ``fnet_convs_ms``.

usage: python scripts/bench_compile_train.py [--reps R] [--iters N] [--only NAME]"""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import torch  # noqa: E402
import torch.nn as nn  # noqa: E402

import magnet_b200  # noqa: E402
from magnet_b200.synthetic import make_inputs  # noqa: E402
from bench_fnet import _power_limit_w  # noqa: E402


def _cam(intM, rays):
    return {"intM": intM, "unit_ray_array_2D": rays}


def _head_workload(dev, B, V, H, W, D, fused):
    torch.manual_seed(0)
    head = magnet_b200.MagnetHead(n_samples=D, fused_train=fused, fused_upsample=fused).to(dev).train()
    inp = make_inputs(B=B, V=V, D=D, H=H, W=W, C=64, seed=1)
    g = inp.to(dev)
    cam = {k: v.to(dev) for k, v in inp.cam_intrins.items()}
    x_d3 = torch.randn(B, 256, H, W, device=dev)
    gt = nn.functional.interpolate(g.ref_gmms[:, :1] * 1.03, scale_factor=4, mode="nearest")

    def loss_fn(ref, src, gmm, sgmm, x_d3, poses, valid, intM, rays, gt):
        if fused:
            return head.train_loss(ref, src, gmm, sgmm, x_d3, poses, valid, _cam(intM, rays), gt, gt > 1e-3)
        preds, mask = head.forward_quarter(ref, src, gmm, sgmm, x_d3, poses, valid, _cam(intM, rays))
        return head.loss(preds, mask, gt, gt > 1e-3)

    args = (g.ref_feat, g.nghbr_feat, g.ref_gmms, g.nghbr_gmms, x_d3, g.nghbr_poses, inp.is_valid.to(dev), cam["intM"],
            cam["unit_ray_array_2D"], gt)
    return head, loss_fn, args, None


def _fnet_workload(dev, B, V, H, W):
    torch.manual_seed(0)
    f = nn.Sequential(nn.Conv2d(3, 32, 3, padding=1), nn.ReLU(), nn.Conv2d(32, 64, 3, stride=4, padding=1), nn.ReLU(),
                      nn.Conv2d(64, 64, 3, padding=1))
    model = magnet_b200.MagnetF(f).to(dev).train()
    planes = magnet_b200.sid_planes(1e-3, 10.0, 80).flatten().tolist()
    inp = make_inputs(B=B, V=V, D=8, H=H, W=W, C=64, seed=5)
    g = inp.to(dev)
    cam = {k: v.to(dev) for k, v in inp.cam_intrins.items()}
    imgs = torch.randn((V + 1) * B, 3, 4 * H, 4 * W, device=dev)
    gt = 12.0 * torch.rand(B, 1, 4 * H, 4 * W, device=dev)

    def loss_fn(ref_img, nghbr_imgs, poses, valid, intM, rays, gt):
        return model.loss(ref_img, nghbr_imgs, poses, valid, _cam(intM, rays), planes, gt, 1e-3, 10.0)

    def convs_only(ref_img, nghbr_imgs, *_):
        return f(torch.cat((ref_img, nghbr_imgs), 0)).square().mean()

    args = (imgs[:B], imgs[B:], g.nghbr_poses, inp.is_valid.to(dev), cam["intM"], cam["unit_ray_array_2D"], gt)
    return model, loss_fn, args, convs_only


def _step(fn, params, args):
    for p in params:
        p.grad = None
    loss = fn(*args)
    loss.backward()
    return loss


def _check(fn, compiled, params, args):
    """Compiled loss against eager's, bit for bit, and the indices of the parameters whose gradients differ (bit for bit;
    the tests bound those differences)."""
    want = _step(fn, params, args).detach().clone()
    wg = [p.grad.clone() for p in params]
    got = _step(compiled, params, args).detach().clone()
    bad = [i for i, (p, w) in enumerate(zip(params, wg)) if not torch.equal(p.grad, w)]
    return bool(torch.equal(got, want)), bad


def _window_ms(fn, params, args, iters):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        _step(fn, params, args)
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / iters


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--only", default=None)
    a = ap.parse_args()
    from torch._dynamo.utils import counters
    dev = torch.device("cuda:0")
    # the equality check runs without TF32 and with deterministic cuDNN; the timing with torch's defaults, as training
    # runs them (cuDNN picks its algorithms in the warm-up)
    timing = {"tf32_matmul": torch.backends.cuda.matmul.allow_tf32, "tf32_cudnn": torch.backends.cudnn.allow_tf32,
              "cudnn_deterministic": torch.backends.cudnn.deterministic, "cudnn_benchmark": torch.backends.cudnn.benchmark}

    def backend(tf32_matmul, tf32_cudnn, cudnn_deterministic, cudnn_benchmark):
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32_matmul, tf32_cudnn
        torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = cudnn_deterministic, cudnn_benchmark

    card = {"gpu": torch.cuda.get_device_name(dev), "power_limit_w": _power_limit_w(), "timed_with": timing}
    print(json.dumps(card), flush=True)
    workloads = {}
    for D in (5, 64):
        for fused in (False, True):
            workloads[f"head-{'fused' if fused else 'module'}-scannet-ns{D}"] = lambda D=D, fused=fused: \
                _head_workload(dev, 4, 4, 120, 160, D, fused)
    for fused in (False, True):
        workloads[f"head-{'fused' if fused else 'module'}-kitti-ns5"] = lambda fused=fused: \
            _head_workload(dev, 4, 2, 88, 304, 5, fused)
    workloads["fnet-scannet"] = lambda: _fnet_workload(dev, 2, 4, 120, 160)
    workloads["fnet-kitti"] = lambda: _fnet_workload(dev, 4, 2, 88, 304)
    for name, make in workloads.items():
        if a.only and a.only not in name:
            continue
        model, fn, args, convs_only = make()
        params = [p for p in model.parameters() if p.requires_grad]
        torch._dynamo.reset()
        fns = {"eager": fn, "default": torch.compile(fn), "reduce-overhead": torch.compile(fn, mode="reduce-overhead")}
        counters.clear()
        backend(False, False, True, False)
        checks = {k: _check(fn, c, params, args) for k, c in fns.items() if k != "eager"}
        backend(**timing)
        for f in fns.values():                              # warm-up: compilation, capture, cuDNN's algorithm choice
            for _ in range(5):
                _step(f, params, args)
        if convs_only is not None:
            for _ in range(5):
                _step(convs_only, params, args)
        torch.cuda.synchronize()
        times = {k: [] for k in fns}
        conv_times = []
        for _ in range(a.reps):
            for k, f in fns.items():
                times[k].append(_window_ms(f, params, args, a.iters))
            if convs_only is not None:
                conv_times.append(_window_ms(convs_only, params, args, a.iters))
        row = {"workload": name, **{f"{k}_ms": round(statistics.median(t), 3) for k, t in times.items()},
               **{f"{k}_range_ms": [round(min(t), 3), round(max(t), 3)] for k, t in times.items()},
               "equal_to_eager": {k: {"loss": ok, "grads_differ": bad} for k, (ok, bad) in checks.items()},
               "cudagraph_skips": sum(counters["inductor"]["cudagraph_skips"].values())
               if isinstance(counters["inductor"]["cudagraph_skips"], dict) else counters["inductor"]["cudagraph_skips"]}
        if conv_times:
            row["fnet_convs_ms"] = round(statistics.median(conv_times), 3)
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
