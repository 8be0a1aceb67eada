"""Sequence evaluation at batch 1 with the head under CUDA graphs (DESIGN §3.17, §3.18): the loop of test_MaGNet over a
synthetic ScanNet-like sequence (the reference loader's neighbour rule, a generated trajectory, relative poses from
ops.relative_poses), with STAND-IN backbones built here from plain convolutions (EfficientNet-B5 / PSM-Net are not used).

Two FrameCaches over the same model: the eager one, and one whose head is
``torch.compile(model.forward_sources, mode="reduce-overhead")``.  Each timed repeat runs the whole sequence through one
of them, the two alternating repeat by repeat; CUDA events around each repeat.  Reported per case: median and range of
samples/s and ms per sample, the outputs compared bit for bit, and the parts of a sample timed on their own: the
stand-in backbones (images per sample, time per image) and the head alone on one sample's arguments (eager call
against graph replay).  Each part runs back to back with itself, so the parts overlap otherwise than in the loop and
do not add up to it.

Cases: 120x160 with V = 4 at N_s = 5 (TILED32 volume) and N_s = 64 (SPLIT16), 88x304 with V = 2 at both.  One more line
records whether the traced plan's volume changes when the table leaves frames unused (SPLIT16 scale over all frames).
One JSON line per measurement with the card, its power limit, its SM clock and clock limit; writes nothing.

usage: python scripts/bench_sequence_compile.py [--refs N] [--repeats R] [--warmup W]"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402
import torch.nn as nn  # noqa: E402

import magnet_b200  # noqa: E402
from magnet_b200 import FrameCache, homography, ops, _lib  # noqa: E402
from magnet_b200.synthetic import quarter_res_camera, scannet_sequence, trajectory  # noqa: E402

CASES = [("scannet", 120, 160, 4, 5), ("scannet", 120, 160, 4, 64), ("kitti", 88, 304, 2, 5), ("kitti", 88, 304, 2, 64)]


def _card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    name, power, sm, sm_max = [s.strip() for s in q.splitlines()[0].split(",")]
    return {"card": name, "power_limit": power, "sm_clock_idle": sm, "sm_clock_max": sm_max}


def _sm_clock():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=clocks.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=30).stdout.strip()
    return q.splitlines()[0].strip()


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


def _samples(dev, n, family, h, w, V):
    refs, nghbrs = scannet_sequence(n, window_radius=20 if V == 4 else 10, n_views=V)
    ids = sorted(set(refs) | set(f for row in nghbrs for f in row))
    g = torch.Generator(device=dev).manual_seed(4)
    imgs = {f: torch.rand(3, 4 * h, 4 * w, device=dev, generator=g) for f in ids}
    ext = {f: torch.from_numpy(e).to(dev) for f, e in trajectory(ids, 0).items()}
    K, rays = quarter_res_camera(h, w, family)
    intr = {"intM": torch.from_numpy(K)[None].to(dev), "unit_ray_array_2D": torch.from_numpy(rays)[None].to(dev)}
    out = []
    for r, row in zip(refs, nghbrs):
        poses, valid = ops.relative_poses(ext[r][None], torch.stack([ext[f] for f in row])[:, None])
        out.append((r, row, imgs[r][None], torch.stack([imgs[f] for f in row]), poses, valid, intr))
    return out, len(ids)


def _events_ms(fn, repeats, warmup, loop=1):
    times = []
    for i in range(warmup + repeats):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(loop):
            fn()
        e.record()
        torch.cuda.synchronize()
        if i >= warmup:
            times.append(s.elapsed_time(e) / loop)
    return sorted(times)[len(times) // 2]


def bench_case(args, dev, card, family, h, w, V, ns):
    torch.manual_seed(3)
    f_net = nn.Sequential(nn.Conv2d(3, 64, 4, stride=4), nn.ReLU(), nn.Conv2d(64, 64, 3, padding=1))
    model = magnet_b200.MAGNET(StandInD(), f_net, n_samples=ns, test_iter=3, fused_upsample=True).to(dev).eval()
    samples, n_frames = _samples(dev, args.refs, family, h, w, V)
    n = len(samples)
    torch._dynamo.reset()
    compiled_head = torch.compile(model.forward_sources, mode="reduce-overhead")
    eager, compiled = FrameCache(model, capacity=32), FrameCache(model, capacity=32, head=compiled_head)

    def run(cache, keep=False):
        cache.clear()
        out = []
        for r, row, ri, ni, p, v, intr in samples:
            pred = cache(ri, ni, p, v, intr, [r], [row], mode="test")[-1]
            if keep:
                out.append(pred.clone())
        return out

    with torch.no_grad():
        a = run(eager, True)
        images = eager.backbone_images                     # one pass over the sequence (the cache starts empty)
        b = run(compiled, True)                            # the first pass records the graphs
        same = all(torch.equal(x, y) for x, y in zip(a, b))
        times = ([], [])
        for i in range(args.warmup + args.repeats):
            for t, cache in zip(times, (eager, compiled)):
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                run(cache)
                e.record()
                torch.cuda.synchronize()
                if i >= args.warmup:
                    t.append(s.elapsed_time(e))
        clock = _sm_clock()
        # the parts on their own: the backbones per image, the head alone (eager call / graph replay)
        x1 = samples[0][2]
        ms_img = _events_ms(lambda: (model.d_net(x1), model.f_net(x1)), 21, 5, 5)
        r, row, ri, ni, p, v, intr = samples[-1]
        compiled(ri, ni, p, v, intr, [r], [row], mode="test")
        ref = compiled._frames[r]
        src = [compiled._frames[f] for f in dict.fromkeys(row)]
        table = torch.arange(V, dtype=torch.int32)[None]
        hargs = (ref[2][None], ref[0][None], ref[1][None], torch.stack([f[2] for f in src]),
                 torch.stack([f[0] for f in src]))
        dtable = table.to(dev)
        head_eager = _events_ms(lambda: model.forward_sources(*hargs, table, p, v, intr, "test"), 21, 5, 5)
        head_graph = _events_ms(lambda: compiled_head(*hargs, dtable, p, v, intr, "test"), 21, 5, 5)
    layout, _ = homography.route(64, V, ns, _lib.VARIANT_AUTO, _lib.DEPTH_GAUSS, torch.float32, torch.float32)
    ms = [[t / n for t in ts] for ts in times]
    med = [sorted(m)[len(m) // 2] for m in ms]
    img_per_sample = images / n
    print(json.dumps(dict(
        what="eval_loop_batch1_compiled_head", family=family, grid=f"{h}x{w}", images=f"{4 * h}x{4 * w}", V=V,
        n_samples=ns, layout=int(layout), samples=n, distinct_frames=n_frames, repeats=args.repeats,
        backbones="stand-in (plain convolutions, not EfficientNet-B5 / PSM-Net)",
        ms_per_sample_eager=round(med[0], 4), ms_per_sample_eager_range=[round(min(ms[0]), 4), round(max(ms[0]), 4)],
        ms_per_sample_compiled=round(med[1], 4),
        ms_per_sample_compiled_range=[round(min(ms[1]), 4), round(max(ms[1]), 4)],
        samples_per_s_eager=round(1e3 / med[0], 1), samples_per_s_compiled=round(1e3 / med[1], 1),
        backbone_images_per_sample=round(img_per_sample, 3), standin_backbone_ms_per_image=round(ms_img, 4),
        head_ms_eager=round(head_eager, 4), head_ms_graph_replay=round(head_graph, 4),
        outputs_bit_identical=same, sm_clock_after=clock, **card)), flush=True)


def bench_unused_frames(dev, card):
    """A SPLIT16 plan whose table leaves frames unused: the traced plan packs all S frames (its scale from all of them),
    the eager plan only the named ones.  Reports whether any bit of the volume and the predictions changes."""
    B, V, S, h, w = 2, 4, 9, 120, 160
    g = torch.Generator(device=dev).manual_seed(5)
    frames = torch.randn(S, 64, h, w, device=dev, generator=g)
    frames[0] *= 40.0                                   # an unused frame with the largest magnitude sets the traced scale
    mu = 1.5 + 2.0 * torch.rand(S, 1, h, w, device=dev, generator=g)
    gm = torch.cat([mu, 0.1 * mu], 1)
    ref = torch.randn(B, 64, h, w, device=dev, generator=g)
    rg = gm[:B].clone()
    x_d3 = torch.randn(B, 256, h, w, device=dev, generator=g)
    K, rays = quarter_res_camera(h, w)
    ang = 0.01 * torch.arange(B * V, dtype=torch.float32).view(B, V)
    poses = torch.eye(4).repeat(B, V, 1, 1)
    poses[:, :, 0, 3], poses[:, :, 1, 3] = 0.05 + ang, 0.02 - ang
    intr = {"intM": torch.from_numpy(K)[None].repeat(B, 1, 1).to(dev),
            "unit_ray_array_2D": torch.from_numpy(rays)[None].repeat(B, 1, 1).to(dev)}
    valid = torch.ones(B, V, dtype=torch.int32, device=dev)
    table = torch.tensor([[1, 3, 5, 7], [3, 5, 7, 2]], dtype=torch.int32)
    torch.manual_seed(2)
    head = magnet_b200.MagnetHead(n_samples=64, n_iter=3).to(dev).eval()
    args = (ref, frames, rg, gm, x_d3, poses.to(dev), valid, intr)
    torch._dynamo.reset()
    with torch.no_grad():
        want = head(*args, src_index=table)
        got = torch.compile(head, fullgraph=True)(*args, src_index=table)
        plan_e = magnet_b200.MatchingPlan(ref, frames, gm, poses.to(dev), valid, intr, src_index=table)
        k = head.k_list
        vol_e = plan_e.cost(rg, k)
        vol_t = torch.compile(lambda *a: magnet_b200.MatchingPlan(*a, src_index=table.to(dev)).cost(rg, k),
                              fullgraph=True)(ref, frames, gm, poses.to(dev), valid, intr)
    diff = [float((a - b).abs().max()) for a, b in zip(got, want)]
    print(json.dumps(dict(
        what="unused_frames_split16", B=B, V=V, S=S, named_frames=int(torch.unique(table).numel()), grid=f"{h}x{w}",
        volume_bit_identical=bool(torch.equal(vol_t, vol_e)),
        volume_max_abs_diff=float((vol_t - vol_e).abs().max()),
        predictions_bit_identical=all(torch.equal(a, b) for a, b in zip(got, want)), predictions_max_abs_diff=diff,
        **card)), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--refs", type=int, default=40, help="references of the batch-1 loop")
    ap.add_argument("--repeats", type=int, default=7, help="timed repeats of the whole loop per arm")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--only", choices=[f"{c[1]}x{c[2]}-ns{c[4]}" for c in CASES] + ["unused"], default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sequence_compile.py needs a CUDA device: magnet_b200 has no CPU path")
    dev = torch.device("cuda:0")
    card = _card()
    for family, h, w, V, ns in CASES:
        if args.only in (None, f"{h}x{w}-ns{ns}"):
            bench_case(args, dev, card, family, h, w, V, ns)
    if args.only in (None, "unused"):
        bench_unused_frames(dev, card)


if __name__ == "__main__":
    main()
