"""Kernel-only timing of the cost kernel for quick A/B runs on the GPU.
usage: [MAGNET_B200_LIB=...] python scripts/kbench.py [cfg2|cfg3] [variant] [reps] [gauss|volume]   (volume = drop-in d_volume mode)"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import magnet_b200
from magnet_b200 import _lib, ops
from magnet_b200.synthetic import make_config
cfg = sys.argv[1] if len(sys.argv) > 1 else "cfg2"
variant = {"auto": 0, "direct": 1, "cells": 2, "noreuse": 3, "tma": 4, "mma": 5}[(sys.argv[2] if len(sys.argv) > 2 and sys.argv[2] else "auto")]
reps = int(sys.argv[3]) if len(sys.argv) > 3 else 30
mode = sys.argv[4] if len(sys.argv) > 4 else "gauss"
inp = make_config(cfg, seed=1)
g = inp.to("cuda")
plan = magnet_b200.MatchingPlan(g.ref_feat, g.nghbr_feat, g.nghbr_gmms, g.nghbr_poses, inp.is_valid, inp.cam_intrins, thres=5)
k = ops.k_array(inp.k.tolist())
out = torch.empty(inp.B, inp.D, *inp.ref_feat.shape[2:], device="cuda")
flush = torch.empty(64 * 1024 * 1024, device="cuda")     # 256 MB > L2
dvol = ops.sample_depths(g.ref_gmms, k) if mode == "volume" else None


def launch():
    if dvol is None:
        plan.cost(g.ref_gmms, k, out=out, variant=variant)
    else:
        layout = {4: _lib.SRC_PIXC, 5: _lib.SRC_SPLIT16}.get(variant, _lib.SRC_TILED32)
        src = plan._source(layout)
        ops.cost_volume(plan.ref_feat, src, plan.rays, plan.cams, V=plan.V, src_layout=layout, consistency=True,
                        src_gmm=plan.src_gmm, kappa=plan.kappa, d_volume=dvol, out=out, variant=variant,
                        ref_split=plan._ref_split if layout == _lib.SRC_SPLIT16 else None)


for _ in range(3):
    launch()
ts = []
for _ in range(reps):
    flush.zero_()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); launch(); e1.record()
    torch.cuda.synchronize(); ts.append(e0.elapsed_time(e1))
ts.sort()
print("%s lib=%s mode=%s variant=%s: median %.4f ms  min %.4f ms" % (cfg, os.path.basename(os.environ.get("MAGNET_B200_LIB", "default")),
      mode, variant, ts[len(ts) // 2], ts[0]))
