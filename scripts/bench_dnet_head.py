"""D-Net's heads after the trunk: the module path (depth_head / mask_head on cuDNN with cudnn.benchmark on and PyTorch's
default TF32 flags, convex_upsample, torch's elu / sqrt) against the fused path (the 3x3 convolutions on cuDNN, the
pack, ops.dnet_depth / ops.dnet_upsample) on the same x_feat, in one process, alternating repeat by repeat:
  * MaGNet's D-Net pass (DnetHead(dnet=False): [mu, sigma] at the feature grid) at cfg2 (40 images, 120 x 160) and
    cfg3 (20 images, 88 x 304);
  * test_DNet's prediction (DnetHead(dnet=True): [mu, var] at 4x the grid) at B 1 and B 8 on 120 x 160 (480 x 640) and
    88 x 304 (352 x 1216);
  * test_DNet's evaluation of one B-1 image: the reference's way (the prediction copied to the host, validate()'s
    numpy metric block) against DnetHead + DepthMetrics.update(..., variance=True) and one host read.
CUDA events around `--loop` calls after warm-up, the median of `--samples` (>= 20) repeats.  Then each fused kernel
alone under torch.profiler, in a run of its own: device time, bytes and FLOPs from the shapes, and the share of the
H100 SXM data-sheet bound that binds (3.35 TB/s HBM3, 989 TFLOP/s dense fp16, three fp16 products per multiply-add).
Asserts at every timed size that the fused outputs are within 1e-4 of each channel's max of a float64 evaluation and
prints the largest such error.  One JSON line per measurement with the card name and its power limit; writes nothing.

usage: python scripts/bench_dnet_head.py [--samples N] [--warmup W] [--loop L]"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from bench_fnet import _power_limit_w  # noqa: E402
from bench_half import _median_pair  # noqa: E402

HBM_BPS, FP16_FLOPS = 3.35e12, 989e12
HID = 128
SHAPES = [  # (what, dnet, B, h, w)
    ("magnet_dnet_pass_cfg2", False, 40, 120, 160),
    ("magnet_dnet_pass_cfg3", False, 20, 88, 304),
    ("test_dnet_B1_480x640", True, 1, 120, 160),
    ("test_dnet_B8_480x640", True, 8, 120, 160),
    ("test_dnet_B1_352x1216", True, 1, 88, 304),
    ("test_dnet_B8_352x1216", True, 8, 88, 304),
]


def _f64(head, x, dnet):
    """The heads in float64 from the module's own 3x3 outputs (fp32 cuDNN, the fused path's input)."""
    d = lambda t: t.detach().double()
    dh, mh = head.depth_head, head.mask_head
    pre_d = F.conv2d(x, dh[0].weight, dh[0].bias, padding=1).double()
    depth = F.conv2d(F.relu(F.conv2d(F.relu(pre_d), d(dh[2].weight), d(dh[2].bias))), d(dh[4].weight), d(dh[4].bias))
    if not dnet:
        return torch.cat([depth[:, :1], torch.sqrt(F.elu(depth[:, 1:]) + 1.0 + 1e-10)], 1)
    pre_m = F.conv2d(x, mh[0].weight, mh[0].bias, padding=1).double()
    mask = F.conv2d(F.relu(F.conv2d(F.relu(pre_m), d(mh[2].weight), d(mh[2].bias))), d(mh[4].weight), d(mh[4].bias))
    N, C, H, W = depth.shape
    w = torch.softmax(mask.view(N, 1, 9, 4, 4, H, W), dim=2)
    nb = F.unfold(depth, [3, 3], padding=1).view(N, C, 9, 1, 1, H, W)
    up = (w * nb).sum(2).permute(0, 1, 4, 2, 5, 3).reshape(N, C, 4 * H, 4 * W)
    return torch.cat([up[:, :1], F.elu(up[:, 1:]) + 1.0 + 1e-10], 1)


def _module_path(head, x, dnet):
    """DnetHead's module chain (what it runs where fused_dnet_applies does not hold), called directly under no_grad."""
    depth = head.depth_head(x)
    if not dnet:
        return torch.cat([depth[:, :1], torch.sqrt(F.elu(depth[:, 1:]) + 1.0 + 1e-10)], 1), x
    from magnet_b200 import ops
    up = ops.convex_upsample(depth, head.mask_head(x), 4)
    return torch.cat([up[:, :1], F.elu(up[:, 1:]) + 1.0 + 1e-10], 1)


def _validate_numpy(out, gt, lo, hi):
    """test_DNet.validate's per-image block (test_DNet.py:40-71) with compute_depth_errors (utils.py:106-144)."""
    pred, var = torch.split(out, 1, dim=1)
    g = gt.cpu().permute(0, 2, 3, 1).numpy()[0, :, :, 0]
    p = pred.cpu().permute(0, 2, 3, 1).numpy()[0, :, :, 0]
    v = var.cpu().permute(0, 2, 3, 1).numpy()[0, :, :, 0]
    valid = np.logical_and(g > lo, g < hi)
    p[p < lo], p[p > hi] = lo, hi
    p[np.isinf(p)], p[np.isnan(p)] = hi, lo
    g, p, v = g[valid], p[valid], v[valid]
    th = np.maximum(g / p, p / g)
    err = np.log(p) - np.log(g)
    v[v < 1e-6] = 1e-6
    return [(th < 1.25).mean(), (th < 1.25 ** 2).mean(), (th < 1.25 ** 3).mean(), np.mean(np.abs(g - p)),
            np.mean(np.abs(g - p) / g), np.mean(((g - p) ** 2) / g), np.sqrt(((g - p) ** 2).mean()),
            (np.abs(np.log10(g) - np.log10(p))).mean(), np.sqrt(((1 / g - 1 / p) ** 2).mean()),
            np.sqrt(((np.log(g) - np.log(p)) ** 2).mean()), np.sqrt(np.mean(err ** 2) - np.mean(err) ** 2) * 100,
            np.mean(0.5 * (np.log(v) + np.log(2 * np.pi) + (np.square(g - p) / v)))]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=20, help="timed repeats per path (at least 20)")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--loop", type=int, default=10, help="calls per timed repeat")
    args = ap.parse_args()
    args.samples = max(20, args.samples)
    if not torch.cuda.is_available():
        raise SystemExit("bench_dnet_head.py needs a CUDA device: magnet_b200 has no CPU path")
    import magnet_b200
    from magnet_b200 import ops

    torch.backends.cudnn.benchmark = True                  # as bench.py and the reference's drivers set it
    dev = torch.device("cuda:0")
    card = {"card": torch.cuda.get_device_name(dev), "power_limit_w": _power_limit_w(0)}
    T = dict(steps=args.samples, warmup=args.warmup, loop=args.loop)
    gen = torch.Generator(device=dev).manual_seed(1)

    def heads(dnet):
        torch.manual_seed(0)
        return magnet_b200.DnetHead(dnet=dnet).to(dev).eval().requires_grad_(False)

    for what, dnet, B, h, w in SHAPES:
        fused = heads(dnet)
        x = torch.relu(torch.randn(B, 256, h, w, device=dev, generator=gen))
        first = (lambda o: o) if dnet else (lambda o: o[0])
        with torch.no_grad():
            torch.backends.cudnn.allow_tf32 = False        # the check reads fp32 3x3 outputs on both sides
            got = first(fused(x))
            want = _f64(fused, x, dnet)
            err = max(float((got[:, c].double() - want[:, c]).abs().max() / want[:, c].abs().max()) for c in range(2))
            assert err <= 1e-4, f"{what}: fused heads off by {err:.2e} of a channel's max"
            del want, got
            torch.backends.cudnn.allow_tf32 = True         # PyTorch's default for the timing
            m_ms, f_ms = _median_pair(lambda: _module_path(fused, x, dnet), lambda: fused(x), **T)
        print(json.dumps({"what": what, "dnet": dnet, "B": B, "h": h, "w": w, "module_ms": round(m_ms, 4),
                          "fused_ms": round(f_ms, 4), "speedup": round(m_ms / f_ms, 3),
                          "max_rel_err_f64": float(f"{err:.3g}"), **card, "samples": args.samples}), flush=True)

    # test_DNet evaluation of one image: host copy + numpy against the device metrics
    for h, w, hi in ((120, 160, 10.0), (88, 304, 80.0)):
        fused = heads(True)
        x = torch.relu(torch.randn(1, 256, h, w, device=dev, generator=gen))
        gt = hi * torch.rand(1, 1, 4 * h, 4 * w, device=dev, generator=gen)
        metrics = magnet_b200.DepthMetrics(1e-3, hi)
        with torch.no_grad():
            def ref_way():
                return _validate_numpy(fused(x), gt, 1e-3, hi)

            def device_way():
                metrics.update(fused(x), gt, variance=True)
                return metrics.images()                     # the one host read a running average needs
            m_ms, f_ms = _median_pair(ref_way, device_way, **T)
        print(json.dumps({"what": f"test_dnet_eval_{4 * h}x{4 * w}", "host_numpy_ms": round(m_ms, 4),
                          "device_ms": round(f_ms, 4), "speedup": round(m_ms / f_ms, 3), **card,
                          "samples": args.samples}), flush=True)

    # each fused kernel alone under the profiler
    for what, dnet, B, h, w in (SHAPES[0], SHAPES[3]):
        fused = heads(dnet)
        x = torch.relu(torch.randn(B, 256, h, w, device=dev, generator=gen))
        with torch.no_grad():
            packed = ops.pack_dnet_weights(fused.depth_head, fused.mask_head if dnet else None)
            pre_d, pre_m = fused._pre(fused.depth_head, x), fused._pre(fused.mask_head, x)
            raw = ops.dnet_depth(pre_d, packed, sigma=False)

            def run():
                ops.dnet_depth(pre_d, packed, sigma=not dnet)
                if dnet:
                    ops.dnet_upsample(pre_m, packed, raw)
            for _ in range(3):
                run()
            torch.cuda.synchronize()
            n = 20
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(n):
                    run()
                torch.cuda.synchronize()
        HW = h * w
        kernels = [("dnet_depth_kernel", B * HID * HW * 4 + B * 2 * HW * 4 + ops.dnet_weights_bytes(0),
                    3 * 2 * HID * HID * B * HW + 2 * 2 * HID * B * HW)]
        if dnet:
            kernels.append(("mask_upsample_kernel", B * HID * HW * 4 + B * 2 * HW * 4 + B * 2 * 16 * HW * 4
                            + ops.dnet_weights_bytes(4) - ops.dnet_weights_bytes(0),
                            3 * 2 * (HID * HID + 144 * HID) * B * HW))
        for name, nbytes, flops in kernels:
            evs = [ev for ev in prof.key_averages() if name in ev.key]
            assert len(evs) == 1 and evs[0].count == n, f"expected {n} {name} events"
            us = getattr(evs[0], "device_time_total", None)
            k_ms = (us if us is not None else evs[0].cuda_time_total) / n / 1e3
            t_bytes, t_flops = nbytes / HBM_BPS, flops / FP16_FLOPS
            print(json.dumps({"what": name, "shape": what, "kernel_ms": round(k_ms, 4), "bytes": nbytes,
                              "GB_per_s": round(nbytes / (k_ms * 1e-3) / 1e9, 1),
                              "TFLOP_per_s": round(flops / (k_ms * 1e-3) / 1e12, 1),
                              "bound": "fp16 tensor cores" if t_flops > t_bytes else "HBM",
                              "frac_of_bound": round(max(t_bytes, t_flops) / (k_ms * 1e-3), 3), **card,
                              "samples": n}), flush=True)


if __name__ == "__main__":
    main()
