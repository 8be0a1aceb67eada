"""F-Net evaluation benchmark: scoring F-Net's depth per image, the reference's way against plane_depth +
depth_metrics(nearest=True).

Shapes: 480x640 (ScanNet, min 1e-3, max 10, no crop) and 352x1216 (KITTI, min 1e-3, max 80, Garg crop) with the volume
at quarter resolution and 80 SID planes, B = 1 and 8.
  host: what train_FNet.py validate() does per batch (:178-193) from the probability volume: torch.sum(prob * d_center)
        and F.interpolate(mode='nearest') on the device, device->host copies of GT and prediction (a synchronising
        copy), then the numpy metric block with var=None (float32 means, utils.compute_depth_errors).  Every image of the
        batch is scored.
  kernel: ops.plane_depth on the scores (softmax fused in) + ops.depth_metrics(nearest=True), three launches; CUDA
        events around a loop of calls, median over repeats; and the same calls captured in a CUDA graph and replayed.
Prints one JSON line per (shape, B) with the card, its power limit and the host CPU, all read in the same run; writes
nothing.

usage: python scripts/bench_fnet_eval.py [--reps R] [--loop L] [--host-reps N]"""
import argparse
import json
import os
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from bench_eval import _cpu_model  # noqa: E402
from bench_fnet import _power_limit_w  # noqa: E402


def host_block(gt, pred, min_depth, max_depth, box):
    """The numpy metric block of train_FNet.py validate() on one image (var=None: nll 0.0), float32 means as there;
    returns the metrics in ops.METRIC_KEYS order."""
    gt = gt.copy()
    gt[gt > max_depth] = 0
    valid = np.logical_and(gt > min_depth, gt < max_depth)
    r0, r1, c0, c1 = box
    crop = np.zeros(valid.shape)
    crop[r0:r1, c0:c1] = 1
    valid = np.logical_and(valid, crop)
    pred = pred.copy()
    pred[pred < min_depth] = min_depth
    pred[pred > max_depth] = max_depth
    pred[np.isinf(pred)] = max_depth
    pred[np.isnan(pred)] = min_depth
    g, p = gt[valid], pred[valid]
    thresh = np.maximum(g / p, p / g)
    out = [(thresh < 1.25).mean(), (thresh < 1.25 ** 2).mean(), (thresh < 1.25 ** 3).mean(), np.mean(np.abs(g - p)),
           np.mean(np.abs(g - p) / g), np.mean(((g - p) ** 2) / g), np.sqrt(((g - p) ** 2).mean())]
    out.append(np.abs(np.log10(g) - np.log10(p)).mean())
    out.append(np.sqrt(((1 / g - 1 / p) ** 2).mean()))
    out.append(np.sqrt(((np.log(g) - np.log(p)) ** 2).mean()))
    err = np.log(p) - np.log(g)
    out.append(np.sqrt(np.mean(err ** 2) - np.mean(err) ** 2) * 100)
    out.append(0.0)
    return out


def _median_ms(fn, reps, loop):
    times = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(loop):
            fn()
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1) / loop)
    return statistics.median(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=31, help="timed repeats of the kernel loop")
    ap.add_argument("--loop", type=int, default=20, help="calls per timed kernel repeat")
    ap.add_argument("--host-reps", type=int, default=5, help="timed repeats of the host path")
    args = ap.parse_args()
    import magnet_b200
    from magnet_b200 import ops
    dev = torch.device("cuda:0")
    card, power = torch.cuda.get_device_name(dev), _power_limit_w(0)
    cpu = {"cpu_model": _cpu_model(), "cpu_count": os.cpu_count(), "numpy": np.__version__}
    D = 80
    for (H, W, crop, lo, hi) in ((480, 640, None, 1e-3, 10.0), (352, 1216, "garg", 1e-3, 80.0)):
        box = ops.crop_box(crop, H, W)
        d_center = magnet_b200.sid_planes(lo, hi, D, device=dev)
        planes = d_center.reshape(-1).tolist()
        for B in (1, 8):
            g = torch.Generator(device=dev).manual_seed(H + B)
            gt = torch.rand(B, 1, H, W, device=dev, generator=g) * (0.9 * hi)
            scores = torch.randn(B, D, H // 4, W // 4, device=dev, generator=g) * 3.0
            prob = torch.softmax(scores, dim=1)

            def kernel():
                pred = ops.plane_depth(scores, planes, scores=True)
                return ops.depth_metrics(pred, gt, min_depth=lo, max_depth=hi, crop=crop, nearest=True)

            # host path: the reference's validate() from the probability volume, every image of the batch
            def host():
                pred = torch.sum(prob * d_center, dim=1, keepdim=True)
                pred = F.interpolate(pred, size=[H, W], mode="nearest").cpu().numpy()
                gt_h = gt.cpu().numpy()
                return [host_block(gt_h[b, 0], pred[b, 0], lo, hi, box) for b in range(B)]

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
            ker_ms = _median_ms(kernel, args.reps, args.loop)
            plane_ms = _median_ms(lambda: ops.plane_depth(scores, planes, scores=True), args.reps, args.loop)
            gr = torch.cuda.CUDAGraph()
            st = torch.cuda.Stream()
            st.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(st):
                kernel()
            torch.cuda.current_stream().wait_stream(st)
            with torch.cuda.graph(gr):
                kernel()
            gr.replay()
            graph_ms = _median_ms(gr.replay, args.reps, args.loop)
            # the two agree on image 0 (float32 means on the host; the predictions differ in the last bits)
            ref = np.array(host()[0], dtype=np.float64)
            got = kernel()[0, 0, 1:].cpu().numpy()
            agree = float(np.max(np.abs(got - ref)[3:] / np.maximum(np.abs(got[3:]), 1e-30)))
            print(json.dumps({
                "shape": [H, W], "volume": [D, H // 4, W // 4], "crop": crop, "B": B,
                "host_ms_per_image": round(statistics.median(host_ms) / B, 4),
                "kernel_ms_per_call": round(ker_ms, 5),
                "kernel_us_per_image": round(ker_ms / B * 1e3, 3),
                "plane_depth_us_per_call": round(plane_ms * 1e3, 2),
                "graph_us_per_call": round(graph_ms * 1e3, 2),
                "speedup": round(statistics.median(host_ms) / ker_ms, 1),
                "max_rel_diff_vs_host": agree, "a_diff_vs_host": float(np.max(np.abs(got - ref)[:3])),
                "card": card, "power_limit_w": power, **cpu}), flush=True)


if __name__ == "__main__":
    main()
