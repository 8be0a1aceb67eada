"""Cost of the camera gradients (magnet_cost_volume_geom_bwd_f32, DESIGN §3.11) next to today's backward.

Arms, alternated in every repeat on the same inputs (CUDA events, median of --repeats repeats of --calls calls each):
  cfg2 / cfg3, VOLUME and GAUSS, after the production SPLIT16 forward:
    bwd       today's backward: feature gradients on the tensor cores, depth gradient on the CUDA cores;
    bwd+cam   the same call plus the camera and ray gradients (what the autograd path runs under geometry_grad());
    cam       the camera and ray gradients alone;
  the ScanNet and KITTI F-Net training shapes (scripts/bench_fnet.py):
    f         MagnetF's matching side: plane_sweep_f(softmax=False) forward + backward into both feature maps;
    f+pose    the same with nghbr_poses requiring grad under geometry_grad().
grad_depth of bwd and bwd+cam is asserted equal at the timed size.  The card's name and power limit are read in the
same call.  Prints one JSON line.

usage: python scripts/bench_geom_grad.py [--repeats N] [--calls K]"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import magnet_b200  # noqa: E402
from magnet_b200 import _lib, ops  # noqa: E402
from magnet_b200.homography import plane_sweep_f  # noqa: E402
from magnet_b200.synthetic import make_inputs  # noqa: E402

CFGS = {"cfg2": dict(B=8, V=4, H=120, W=160, family="scannet"), "cfg3": dict(B=4, V=4, H=88, W=304, family="kitti")}
FNET = {"scannet": dict(B=2, V=4, H=120, W=160, family="scannet", max_depth=10.0),
        "kitti": dict(B=4, V=2, H=88, W=304, family="kitti", max_depth=80.0)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()


def timed(arms, repeats, calls):
    """{name: median ms per call}; the arms alternate within every repeat."""
    for fn in arms.values():
        fn()
    torch.cuda.synchronize()
    ms = {k: [] for k in arms}
    for _ in range(repeats):
        for k, fn in arms.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(calls):
                fn()
            b.record()
            b.synchronize()
            ms[k].append(a.elapsed_time(b) / calls)
    return {k: round(statistics.median(v), 4) for k, v in ms.items()}


def cw_case(cfg, mode, repeats, calls):
    sh = CFGS[cfg]
    inp = make_inputs(B=sh["B"], V=sh["V"], D=64, H=sh["H"], W=sh["W"], C=64, seed=7, family=sh["family"])
    dev = torch.device("cuda")
    g = inp.to(dev)
    V = sh["V"]
    cams = ops.pack_cameras(inp.cam_intrins['intM'].to(dev), g.R, g.t, inp.is_valid.to(dev, torch.int32))
    rays = inp.cam_intrins['unit_ray_array_2D'].to(dev).contiguous()
    k = inp.k.tolist()
    src_split = ops.repack_split16(g.nghbr_feat, g.nghbr_gmms)
    ref_split = ops.repack_split16(g.ref_feat)
    depth = dict(d_volume=ops.sample_depths(g.ref_gmms, k)) if mode == "volume" else dict(ref_gmm=g.ref_gmms, k=k)
    gout = torch.randn(sh["B"], 64, sh["H"], sh["W"], device=dev)
    common = dict(V=V, kappa=float(inp.thres), fwd_layout=_lib.SRC_SPLIT16, fwd_variant=_lib.VARIANT_AUTO, **depth)

    def bwd():
        return ops.cost_volume_bwd(g.ref_feat, g.nghbr_feat, g.nghbr_gmms, rays, cams, gout, ref_split=ref_split,
                                   src_split=src_split, **common)

    def cam():
        return ops.cost_volume_geom_bwd(g.ref_feat, g.nghbr_feat, g.nghbr_gmms, rays, cams, gout, **common)

    def both():
        return bwd(), cam()

    (_, _, gd0) = bwd()
    ((_, _, gd1), (gc, _, _)) = both()
    assert torch.equal(gd0, gd1) and bool(torch.isfinite(gc).all())
    return timed({"bwd": bwd, "bwd+cam": both, "cam": cam}, repeats, calls)


def f_case(name, repeats, calls):
    sh = FNET[name]
    inp = make_inputs(B=sh["B"], V=sh["V"], D=64, H=sh["H"], W=sh["W"], C=64, seed=3, family=sh["family"])
    dev = torch.device("cuda")
    g = inp.to(dev)
    d_center = magnet_b200.sid_planes(1e-3, sh["max_depth"], 80, dev)     # train_FNet.py's 80 SID planes
    ref = g.ref_feat.clone().requires_grad_(True)
    src = g.nghbr_feat.clone().requires_grad_(True)
    poses = g.nghbr_poses.clone().requires_grad_(True)
    gout = torch.randn(sh["B"], 80, sh["H"], sh["W"], device=dev)

    def run(with_pose):
        p = poses if with_pose else poses.detach()
        with magnet_b200.geometry_grad(with_pose):
            s = plane_sweep_f(d_center, ref, src, p[:, :, :3, :3], p[:, :, :3, 3], inp.is_valid, inp.cam_intrins,
                              softmax=False)
        (s * gout).sum().backward()
        ref.grad = src.grad = poses.grad = None

    return timed({"f": lambda: run(False), "f+pose": lambda: run(True)}, repeats, calls)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=21)
    ap.add_argument("--calls", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_geom_grad.py measures the GPU: no CUDA device"
    res = {"card": card()}
    for cfg in CFGS:
        for mode in ("volume", "gauss"):
            res[f"{cfg}_{mode}"] = cw_case(cfg, mode, args.repeats, args.calls)
    for name in FNET:
        res[f"fnet_{name}"] = f_case(name, args.repeats, args.calls)
    res["card_after"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
