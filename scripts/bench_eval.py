"""Depth-evaluation benchmark: scoring a prediction per image, the reference's way against ops.depth_metrics.

Shapes: 480x640 (ScanNet, min 1e-3, max 10, no crop) and 352x1216 (KITTI, min 1e-3, max 80, Garg crop), B = 1 and 8,
two forms: full resolution ((B,2,H,W) [mu, sigma]) and fused (quarter-resolution Gaussians + the k = 4 upsampling mask).
  host: what validate() does per image (test_MaGNet.py:52-79): device->host copies of GT, mu and sigma (a
        synchronising copy), then the numpy metric block (float32 means, utils.compute_depth_errors); the fused form
        first upsamples on the device (ops.convex_upsample), as the reference must.  Every image of the batch is scored.
  kernel: ops.depth_metrics (two launches), CUDA events around a loop of calls, median over repeats; and the same call
        captured in a CUDA graph and replayed (device time without the Python wrapper).
Prints one JSON line per (shape, B, form) with the card, its power limit and the host CPU; writes nothing.

usage: python scripts/bench_eval.py [--reps R] [--host-reps N]"""
import argparse
import json
import os
import platform
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_fnet import _power_limit_w  # noqa: E402


def _cpu_model():
    """The host CPU's model name; where /proc/cpuinfo has none, its vendor / family / model numbers and architecture."""
    info = {}
    try:
        with open("/proc/cpuinfo") as f:
            for line in f:
                if ":" in line:
                    key, val = (x.strip() for x in line.split(":", 1))
                    info.setdefault(key.lower(), val)
    except OSError:
        pass
    if info.get("model name"):
        return info["model name"]
    parts = [info.get("vendor_id"), info.get("cpu family") and "family " + info["cpu family"],
             info.get("model") and "model " + info["model"], platform.machine()]
    return " ".join(p for p in parts if p) or "not reported"


def host_block(gt, mu, sg, min_depth, max_depth, box):
    """The numpy metric block of validate() on one image, float32 means as there (the timing target); returns the
    metrics in ops.METRIC_KEYS order."""
    gt = gt.copy()
    gt[gt > max_depth] = 0
    valid = np.logical_and(gt > min_depth, gt < max_depth)
    r0, r1, c0, c1 = box
    crop = np.zeros(valid.shape)
    crop[r0:r1, c0:c1] = 1
    valid = np.logical_and(valid, crop)
    mu = mu.copy()
    mu[mu < min_depth] = min_depth
    mu[mu > max_depth] = max_depth
    mu[np.isinf(mu)] = max_depth
    mu[np.isnan(mu)] = min_depth
    var = np.square(sg)[valid]
    g, p = gt[valid], mu[valid]
    thresh = np.maximum(g / p, p / g)
    out = [(thresh < 1.25).mean(), (thresh < 1.25 ** 2).mean(), (thresh < 1.25 ** 3).mean(), np.mean(np.abs(g - p)),
           np.mean(np.abs(g - p) / g), np.mean(((g - p) ** 2) / g), np.sqrt(((g - p) ** 2).mean())]
    out.append(np.abs(np.log10(g) - np.log10(p)).mean())
    out.append(np.sqrt(((1 / g - 1 / p) ** 2).mean()))
    out.append(np.sqrt(((np.log(g) - np.log(p)) ** 2).mean()))
    err = np.log(p) - np.log(g)
    out.append(np.sqrt(np.mean(err ** 2) - np.mean(err) ** 2) * 100)
    var[var < 1e-6] = 1e-6
    out.append(np.mean(0.5 * (np.log(var) + np.log(2 * np.pi) + (np.square(g - p) / var))))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=31, help="timed repeats of the kernel loop")
    ap.add_argument("--loop", type=int, default=20, help="calls per timed kernel repeat")
    ap.add_argument("--host-reps", type=int, default=5, help="timed repeats of the host path")
    args = ap.parse_args()
    import magnet_b200  # noqa: F401
    from magnet_b200 import ops
    dev = torch.device("cuda:0")
    card, power = torch.cuda.get_device_name(dev), _power_limit_w(0)
    cpu = {"cpu_model": _cpu_model(), "cpu_count": os.cpu_count(), "numpy": np.__version__}
    k = 4
    for (H, W, crop, lo, hi) in ((480, 640, None, 1e-3, 10.0), (352, 1216, "garg", 1e-3, 80.0)):
        box = ops.crop_box(crop, H, W)
        for B in (1, 8):
            g = torch.Generator(device=dev).manual_seed(H + B)
            gt = torch.rand(B, 1, H, W, device=dev, generator=g) * (0.9 * hi)
            depth_q = torch.rand(B, 2, H // k, W // k, device=dev, generator=g) * (0.9 * hi) + 0.1
            mask = torch.randn(B, 9 * k * k, H // k, W // k, device=dev, generator=g)
            full = ops.convex_upsample(depth_q, mask, k)
            for form in ("full", "fused"):
                kw = dict(min_depth=lo, max_depth=hi, crop=crop)
                if form == "fused":
                    def kernel():
                        return ops.depth_metrics(depth_q, gt, up_mask=mask, k=k, **kw)

                    def to_full():
                        return ops.convex_upsample(depth_q, mask, k)
                else:
                    def kernel():
                        return ops.depth_metrics(full, gt, **kw)

                    def to_full():
                        return full

                # host path: device -> host copies (synchronising) + the numpy block per image
                def host():
                    pr = to_full()
                    gt_h = gt.detach().cpu().numpy()
                    mu_h = pr[:, 0].detach().cpu().numpy()
                    sg_h = pr[:, 1].detach().cpu().numpy()
                    return [host_block(gt_h[b, 0], mu_h[b], sg_h[b], lo, hi, box) for b in range(B)]

                host()
                host_ms = []
                for _ in range(args.host_reps):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    host()
                    host_ms.append((time.perf_counter() - t0) * 1e3)
                for _ in range(3):
                    kernel()
                torch.cuda.synchronize()
                ker_ms = []
                for _ in range(args.reps):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(args.loop):
                        kernel()
                    e1.record()
                    e1.synchronize()
                    ker_ms.append(e0.elapsed_time(e1) / args.loop)
                # the same call captured in a CUDA graph: device time without the Python wrapper's overhead
                gr = torch.cuda.CUDAGraph()
                st = torch.cuda.Stream()
                st.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(st):
                    kernel()
                torch.cuda.current_stream().wait_stream(st)
                with torch.cuda.graph(gr):
                    kernel()
                gr.replay()
                graph_ms = []
                for _ in range(args.reps):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(args.loop):
                        gr.replay()
                    e1.record()
                    e1.synchronize()
                    graph_ms.append(e0.elapsed_time(e1) / args.loop)
                # the two agree: kernel rows against the host block on image 0 (float32 means there)
                ref = host()[0]
                got = kernel()[0, 0, 1:].cpu().numpy()
                agree = float(np.max(np.abs(got - np.array(ref, dtype=np.float64)) / np.maximum(np.abs(got), 1e-30)))
                print(json.dumps({
                    "shape": [H, W], "crop": crop, "B": B, "form": form,
                    "host_ms_per_image": round(statistics.median(host_ms) / B, 4),
                    "kernel_ms_per_call": round(statistics.median(ker_ms), 5),
                    "kernel_us_per_image": round(statistics.median(ker_ms) / B * 1e3, 3),
                    "graph_us_per_call": round(statistics.median(graph_ms) * 1e3, 2),
                    "speedup": round(statistics.median(host_ms) / statistics.median(ker_ms), 1),
                    "max_rel_diff_vs_host": agree, "card": card, "power_limit_w": power, **cpu}), flush=True)


if __name__ == "__main__":
    main()
