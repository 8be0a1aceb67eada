"""Sequence evaluation: the frame-table path (MAGNET.forward_frames / FrameCache, DESIGN §3.17) against the per-sample
data flow of test_MaGNet, on a synthetic ScanNet-like sequence: the reference loader's neighbour rule with its
end-of-sequence fallback, a generated camera trajectory, relative poses from ops.relative_poses and intrinsics from
synthetic.quarter_res_camera.

  1. Head only, batched: B = 8 consecutive references at 120x160 with V = 4 and at 88x304 with V = 2, N_s = 5 and
     D = 64 hypotheses, on the same per-frame backbone outputs: MagnetHead on the view-major gathered maps (what
     MAGNET.forward hands it) against MagnetHead with the frame table (what forward_frames hands it).  Median of
     alternating CUDA-event repeats; then, in a run of its own under torch.profiler, the device time of the source
     repack (every kernel whose name holds "repack" or "absmax") and of the whole head; the repack bytes from shapes.
  2. Evaluation loop at batch 1: FrameCache against per-sample MAGNET.forward over the same sequence, with STAND-IN
     backbones built here from plain convolutions (EfficientNet-B5 / PSM-Net are not used): backbone image passes per
     sample from a forward hook, the stand-in's own time per image, samples/s (median over alternating repeats).

Both paths' predictions are compared bit for bit.  One JSON line per measurement with the card name and its power
limit; writes nothing.

usage: python scripts/bench_sequence.py [--repeats R] [--warmup W] [--loop L] [--refs N]"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402
import torch.nn as nn  # noqa: E402

from bench_fnet import _power_limit_w  # noqa: E402
from bench_half import _median_pair  # noqa: E402

import magnet_b200  # noqa: E402
from magnet_b200 import FrameCache, MagnetHead, homography, ops, _lib  # noqa: E402
from magnet_b200.synthetic import quarter_res_camera, scannet_sequence, trajectory  # noqa: E402

HEAD_SHAPES = [("scannet", 120, 160, 4), ("kitti", 88, 304, 2)]   # (family, h, w, V); B = 8


def _sequence_batch(n_refs, V, first, B, dev, family, h, w, seed=0):
    """B consecutive references from `first` of a sequence of n_refs, their neighbours by the loader's rule, relative
    poses from a generated trajectory, the intrinsics.  Returns (frame ids, ref ids, nghbr ids, poses, valid, intr)."""
    refs, nghbrs = scannet_sequence(n_refs, window_radius=20 if V == 4 else 10, n_views=V)
    refs, nghbrs = refs[first:first + B], nghbrs[first:first + B]
    ids = sorted(set(refs) | set(f for row in nghbrs for f in row))
    ext = {f: torch.from_numpy(e).to(dev) for f, e in trajectory(ids, seed).items()}
    poses, valid = ops.relative_poses(torch.stack([ext[r] for r in refs]),
                                      torch.stack([torch.stack([ext[row[v]] for row in nghbrs]) for v in range(V)]))
    K, rays = quarter_res_camera(h, w, family)
    intr = {"intM": torch.from_numpy(K)[None].repeat(B, 1, 1), "unit_ray_array_2D": torch.from_numpy(rays)[None].repeat(B, 1, 1)}
    return ids, refs, nghbrs, poses, valid.cpu(), intr


def _repack_bytes(layout, N, C, h, w):
    """Bytes the source repack of N maps reads and writes, from shapes (fp32 maps and Gaussians)."""
    feat, gmm = N * C * h * w * 4, N * 2 * h * w * 4
    if layout == _lib.SRC_TILED32:
        return feat + N * h * ((w + 31) // 32) * 32 * C * 4
    if layout == _lib.SRC_PIXC:
        return feat + gmm + N * h * w * (C + 4) * 4
    if layout in ops.PACKED_LAYOUTS:                     # absmax pass + repack pass
        return 2 * feat + gmm + ops.packed_bytes(layout, N, h, w)
    return 0


def _device_times(fn):
    """(repack device ms, all kernels' device ms) of one call of fn under torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    rep = tot = 0.0
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        us = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
        tot += us
        if "repack" in e.name or "absmax" in e.name:
            rep += us
    return rep / 1e3, tot / 1e3


def bench_head(args, dev, card):
    for family, h, w, V in HEAD_SHAPES:
        for ns in (5, 64):
            B = 8
            ids, refs, nghbrs, poses, valid, intr = _sequence_batch(16, V, 4, B, dev, family, h, w)
            pos = {f: i for i, f in enumerate(ids)}
            S = len(ids)
            g = torch.Generator(device=dev).manual_seed(1)
            feat = torch.randn(S, 64, h, w, device=dev, generator=g)
            mu = 1.0 + 3.0 * torch.rand(S, 1, h, w, device=dev, generator=g)
            gm = torch.cat([mu, 0.1 * mu], 1)
            x_d3 = torch.randn(S, 256, h, w, device=dev, generator=g)
            ref = torch.tensor([pos[r] for r in refs], device=dev)
            table = torch.tensor([[pos[f] for f in row] for row in nghbrs], dtype=torch.int32)
            gather = table.t().reshape(-1).to(dev)
            torch.manual_seed(2)
            head = MagnetHead(n_samples=ns, n_iter=3).to(dev).eval()
            rf, rg, rx = feat[ref], gm[ref], x_d3[ref]
            nf, ng = feat[gather].contiguous(), gm[gather].contiguous()
            with torch.no_grad():
                run_g = lambda: head(rf, nf, rg, ng, rx, poses, valid, intr)
                run_i = lambda: head(rf, feat, rg, gm, rx, poses, valid, intr, src_index=table)
                a, b = run_g(), run_i()
                same = all(torch.equal(x, y) for x, y in zip(a, b))
                ms_g, ms_i = _median_pair(run_g, run_i, args.repeats, args.warmup, args.loop)
                rep_g, tot_g = _device_times(run_g)
                rep_i, tot_i = _device_times(run_i)
            layout, _ = homography.route(64, V, ns, _lib.VARIANT_AUTO, _lib.DEPTH_GAUSS, torch.float32, torch.float32)
            U = int(torch.unique(table).numel())
            print(json.dumps(dict(
                what="head_batched", family=family, h=h, w=w, B=B, V=V, n_samples=ns, layout=int(layout),
                source_maps_gathered=V * B, source_frames_indexed=U, outputs_bit_identical=same,
                head_ms_gathered=round(ms_g, 4), head_ms_indexed=round(ms_i, 4),
                head_device_ms_gathered=round(tot_g, 4), head_device_ms_indexed=round(tot_i, 4),
                repack_device_ms_gathered=round(rep_g, 4), repack_device_ms_indexed=round(rep_i, 4),
                repack_bytes_gathered=_repack_bytes(layout, V * B, 64, h, w),
                repack_bytes_indexed=_repack_bytes(layout, U, 64, h, w), **card)), flush=True)


class StandInD(nn.Module):
    """STAND-IN for D-Net (not EfficientNet-B5): plain convolutions to (mono Gaussian, x_d3) at 1/4 resolution."""

    def __init__(self):
        super().__init__()
        self.t = nn.Sequential(nn.Conv2d(3, 64, 4, stride=4), nn.ReLU(), nn.Conv2d(64, 256, 3, padding=1), nn.ReLU(),
                               nn.Conv2d(256, 256, 3, padding=1), nn.ReLU())
        self.g = nn.Conv2d(256, 2, 1)

    def forward(self, x):
        f = self.t(x)
        g = self.g(f)
        return torch.cat([2.5 + 0.5 * torch.tanh(g[:, :1]), 0.2 + 0.05 * torch.sigmoid(g[:, 1:])], 1), f


def bench_loop(args, dev, card):
    torch.manual_seed(3)
    f_net = nn.Sequential(nn.Conv2d(3, 64, 4, stride=4), nn.ReLU(), nn.Conv2d(64, 64, 3, padding=1))
    model = magnet_b200.MAGNET(StandInD(), f_net, n_samples=5, test_iter=3).to(dev).eval()
    passes = [0]
    hook = model.d_net.register_forward_hook(lambda m, i, o: passes.__setitem__(0, passes[0] + i[0].shape[0]))
    n = args.refs
    refs, nghbrs = scannet_sequence(n)
    ids = sorted(set(refs) | set(f for row in nghbrs for f in row))
    g = torch.Generator(device=dev).manual_seed(4)
    imgs = {f: torch.rand(3, 480, 640, device=dev, generator=g) for f in ids}
    ext = {f: torch.from_numpy(e).to(dev) for f, e in trajectory(ids, 0).items()}
    K, rays = quarter_res_camera(120, 160)
    intr = {"intM": torch.from_numpy(K)[None], "unit_ray_array_2D": torch.from_numpy(rays)[None]}
    samples = []
    for r, row in zip(refs, nghbrs):
        poses, valid = ops.relative_poses(ext[r][None], torch.stack([ext[f] for f in row])[:, None])
        samples.append((r, row, imgs[r][None], torch.stack([imgs[f] for f in row]), poses, valid.cpu()))
    cache = FrameCache(model, capacity=32)

    def per_sample():
        return [model(ri, ni, p, v, intr, mode="test")[-1] for _, _, ri, ni, p, v in samples]

    def cached():
        cache.clear()
        return [cache(ri, ni, p, v, intr, [r], [row], mode="test")[-1] for r, row, ri, ni, p, v in samples]

    with torch.no_grad():
        passes[0] = 0
        a = per_sample()
        p_fwd = passes[0]
        passes[0] = 0
        b = cached()
        p_cache = passes[0]
        same = all(torch.equal(x, y) for x, y in zip(a, b))
        x1 = torch.rand(1, 3, 480, 640, device=dev)
        backbone = lambda: (model.d_net(x1), model.f_net(x1))
        _, ms_img = _median_pair(backbone, backbone, args.repeats, args.warmup, args.loop)
        times = ([], [])
        for i in range(args.warmup_loops + args.loop_repeats):
            for t, fn in zip(times, (per_sample, cached)):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()
                torch.cuda.synchronize()
                if i >= args.warmup_loops:
                    t.append(time.perf_counter() - t0)
    hook.remove()
    med = [sorted(t)[len(t) // 2] for t in times]
    print(json.dumps(dict(
        what="eval_loop_batch1", backbones="stand-in (plain convolutions, not EfficientNet-B5 / PSM-Net)",
        images="480x640", grid="120x160", V=4, n_samples=5, samples=n, distinct_frames=len(ids),
        backbone_passes_per_sample_forward=p_fwd / n, backbone_passes_per_sample_cache=p_cache / n,
        standin_backbone_ms_per_image=round(ms_img, 4),
        samples_per_s_forward=round(n / med[0], 2), samples_per_s_cache=round(n / med[1], 2),
        outputs_bit_identical_cudnn_batch_dependent=same, **card)), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=21)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--loop", type=int, default=5)
    ap.add_argument("--refs", type=int, default=40, help="references of the batch-1 loop")
    ap.add_argument("--loop-repeats", type=int, default=5)
    ap.add_argument("--warmup-loops", type=int, default=1)
    ap.add_argument("--only", choices=["head", "loop"], default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sequence.py needs a CUDA device: magnet_b200 has no CPU path")
    dev = torch.device("cuda:0")
    card = {"card": torch.cuda.get_device_name(dev), "power_limit_w": _power_limit_w(0)}
    if args.only in (None, "head"):
        bench_head(args, dev, card)
    if args.only in (None, "loop"):
        bench_loop(args, dev, card)


if __name__ == "__main__":
    main()
