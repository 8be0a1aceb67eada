"""CW-volume training benchmark at the cfg2 / cfg3 shapes (C = 64, D = 64): the backward kernels alone on the same
upstream gradient, alternating — feature gradients on the tensor cores (the forward's split buffers) against the
CUDA-core kernel (NCHW maps, the same mask), and the depth gradient alone — plus forward + backward of the drop-in
est_costvolume_CW with ref_feat, nghbr_feat and d_volume requiring grad.  Prints one JSON line with the card and its
power limit; writes nothing.

usage: python scripts/bench_cw_grad.py --config {cfg2,cfg3} [--steps K] [--warmup W]"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from bench_fnet import _power_limit_w  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="cfg2", choices=["cfg2", "cfg3"])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import magnet_b200
    from magnet_b200 import _lib, ops
    from magnet_b200.synthetic import make_config
    dev = torch.device("cuda:0")
    inp = make_config(args.config, seed=0)
    g = inp.to(dev)
    intr = {k: v.to(dev) for k, v in inp.cam_intrins.items()}
    valid = inp.is_valid.to(dev)
    dv = g.depth_volume().requires_grad_(True)
    ref, src = g.ref_feat.clone().requires_grad_(True), g.nghbr_feat.clone().requires_grad_(True)
    gout = torch.randn(inp.B, inp.D, *g.ref_feat.shape[2:], device=dev)

    def drop_in():
        out = magnet_b200.est_costvolume_CW(dv, ref, src, g.ref_gmms, g.nghbr_gmms, g.R, g.t, valid, intr, inp.thres)
        return torch.autograd.grad(out, (dv, ref, src), gout)

    cams = ops.pack_cameras(intr['intM'], g.R, g.t, valid.to(torch.int32))
    rays = intr['unit_ray_array_2D'].contiguous()
    rs, sp = ops.repack_split16(g.ref_feat), ops.repack_split16(g.nghbr_feat, g.nghbr_gmms)
    kw = dict(V=inp.V, kappa=float(inp.thres), d_volume=g.depth_volume(), fwd_layout=_lib.SRC_SPLIT16,
              fwd_variant=_lib.VARIANT_AUTO)

    def bwd(**extra):
        return lambda: ops.cost_volume_bwd(g.ref_feat, g.nghbr_feat, g.nghbr_gmms, rays, cams, gout, **kw, **extra)

    arms = {"tensor_core_feature_bwd": bwd(ref_split=rs, src_split=sp, need_depth=False),
            "cuda_core_feature_bwd": bwd(need_depth=False),
            "depth_grad_only": bwd(need_ref=False, need_src=False),
            "drop_in_fwd_plus_bwd": drop_in}
    times = {k: [] for k in arms}
    for i in range(args.warmup + args.steps):
        for name, fn in arms.items():                  # alternating arms: clock and thermal drift hit both alike
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            fn()
            e.record()
            torch.cuda.synchronize()
            if i >= args.warmup:
                times[name].append(s.elapsed_time(e))
    med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
    a, b = arms["tensor_core_feature_bwd"](), arms["cuda_core_feature_bwd"]()
    agree = max(float((x - y).norm() / y.norm()) for x, y in zip(a[:2], b[:2]))
    print(json.dumps({"config": args.config, "steps": args.steps, "median_ms": med,
                      "feature_grad_rel_diff_tc_vs_cuda_core": agree, "card": torch.cuda.get_device_name(dev),
                      "power_limit_w": _power_limit_w(0)}))


if __name__ == "__main__":
    main()
