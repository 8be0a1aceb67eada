"""Half-precision feature maps: SPLIT16 (fp32 maps, hi / lo planes, three products) against HALF16 (fp16 / bf16 maps, one
plane, one product) on the same bf16-rounded features, so that both compute the same volume (asserted with
array_equal at the timed size).  In one process, alternating the two forms repeat by repeat:
  * the cost kernel alone, GAUSS (fused sampler) and VOLUME (drop-in) mode, consistency on;
  * the repack of the source maps (with their Gaussians) and of the reference maps;
  * the CW feature backward (tensor-core kernel, no depth gradient);
  * MagnetF's matching side (plane-sweep scores + fused L1 loss + backward into both maps) at the F-Net training shapes
    of bench_fnet.py, fp32 features against bf16 features.
CUDA events around `--loop` launches after warm-up, the median of `--steps` (>= 20) repeats.  Prints one JSON line per
measurement with the card name and its power limit; writes nothing.

usage: python scripts/bench_half.py --config {cfg2,cfg3} [--steps K] [--warmup W] [--loop L] [--no-fnet]"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from bench_fnet import FNET_SHAPES, _power_limit_w  # noqa: E402


def _median_pair(fa, fb, steps, warmup, loop):
    """Median ms per call of fa and fb, alternating repeat by repeat (clock and thermal drift hit both alike)."""
    times = ([], [])
    for i in range(warmup + steps):
        for t, fn in zip(times, (fa, fb)):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(loop):
                fn()
            e.record()
            torch.cuda.synchronize()
            if i >= warmup:
                t.append(s.elapsed_time(e) / loop)
    return tuple(sorted(t)[len(t) // 2] for t in times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="cfg2", choices=["cfg2", "cfg3"])
    ap.add_argument("--steps", type=int, default=20, help="timed repeats per form (at least 20)")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--loop", type=int, default=10, help="launches per timed repeat")
    ap.add_argument("--no-fnet", action="store_true", help="skip the MagnetF matching side")
    args = ap.parse_args()
    args.steps = max(20, args.steps)
    if not torch.cuda.is_available():
        raise SystemExit("bench_half.py needs a CUDA device: magnet_b200 has no CPU path")
    import magnet_b200
    from magnet_b200 import _lib, homography as hg, ops
    from magnet_b200.synthetic import make_config, make_inputs

    dev = torch.device("cuda:0")
    card = {"card": torch.cuda.get_device_name(dev), "power_limit_w": _power_limit_w(0)}
    T = dict(steps=args.steps, warmup=args.warmup, loop=args.loop)

    def emit(what, split_ms, half_ms, loop=args.loop, **extra):
        print(json.dumps({"config": args.config, "what": what, "split16_ms": split_ms, "half16_ms": half_ms,
                          "speedup": split_ms / half_ms, "steps": args.steps, "loop": loop, **extra, **card}),
              flush=True)

    inp = make_config(args.config, seed=0)
    g = inp.to(dev)
    B, V, D = inp.B, inp.V, inp.D
    ref_h, src_h = g.ref_feat.to(torch.bfloat16), g.nghbr_feat.to(torch.bfloat16)
    ref32, src32 = ref_h.float(), src_h.float()                # the same values: both forms compute one volume
    intr = {k: v.to(dev) for k, v in inp.cam_intrins.items()}
    cams = ops.pack_cameras(intr['intM'], g.R, g.t, inp.is_valid.to(dev, torch.int32))
    rays = intr['unit_ray_array_2D'].contiguous()
    k = inp.k.tolist()
    karr = ops.k_array(k)
    dvol = ops.sample_depths(g.ref_gmms, karr)
    shape = dict(B=B, V=V, D=D, C=64, H=g.ref_feat.shape[2], W=g.ref_feat.shape[3])

    # ---- repacks (into preallocated buffers) ----
    s_src, s_ref = ops.repack_split16(src32, g.nghbr_gmms), ops.repack_split16(ref32)
    h_src, h_ref = ops.repack_half16(src_h, g.nghbr_gmms), ops.repack_half16(ref_h)
    ms = _median_pair(lambda: ops.repack_split16(src32, g.nghbr_gmms, out=s_src),
                      lambda: ops.repack_half16(src_h, g.nghbr_gmms, out=h_src), **T)
    emit("repack_source", *ms, shape=shape)
    ms = _median_pair(lambda: ops.repack_split16(ref32, out=s_ref), lambda: ops.repack_half16(ref_h, out=h_ref), **T)
    emit("repack_reference", *ms, shape=shape)

    # ---- the cost kernel alone, both depth modes ----
    for mode, depth in (("gauss", dict(ref_gmm=g.ref_gmms, k=karr)), ("volume", dict(d_volume=dvol))):
        out_s = torch.empty(B, D, *g.ref_feat.shape[2:], device=dev)
        out_h = torch.empty_like(out_s)
        kw = dict(V=V, consistency=True, kappa=float(inp.thres), **depth)
        fs = lambda: ops.cost_volume(ref32, s_src, rays, cams, src_layout=_lib.SRC_SPLIT16, ref_split=s_ref, out=out_s, **kw)
        fh = lambda: ops.cost_volume(ref_h, h_src, rays, cams, src_layout=_lib.SRC_HALF16, ref_split=h_ref, out=out_h, **kw)
        fs(), fh()
        torch.cuda.synchronize()
        assert torch.equal(out_s, out_h), f"{mode}: HALF16 and SPLIT16 volumes differ"
        ms = _median_pair(fs, fh, **T)
        assert torch.equal(out_s, out_h)
        emit(f"cost_kernel_{mode}", *ms, shape=shape, array_equal=True)

    # ---- CW feature backward on the tensor cores (depth gradient excluded: CUDA-core kernel, same for both) ----
    gout = torch.randn(B, D, *g.ref_feat.shape[2:], device=dev)
    kw = dict(V=V, kappa=float(inp.thres), d_volume=dvol, fwd_variant=_lib.VARIANT_AUTO, need_depth=False)
    bs = lambda: ops.cost_volume_bwd(ref32, src32, g.nghbr_gmms, rays, cams, gout, fwd_layout=_lib.SRC_SPLIT16,
                                     ref_split=s_ref, src_split=s_src, **kw)
    bh = lambda: ops.cost_volume_bwd(ref_h, src_h, g.nghbr_gmms, rays, cams, gout, fwd_layout=_lib.SRC_HALF16,
                                     ref_split=h_ref, src_split=h_src, **kw)
    ms = _median_pair(bs, bh, **T)
    a, b = bs(), bh()
    rel = max(float((x - y).norm() / y.norm()) for x, y in zip(a[:2], b[:2]))
    emit("cw_feature_backward", *ms, shape=shape, grad_rel_diff=rel)

    # ---- MagnetF's matching side at the F-Net training shapes ----
    if args.no_fnet:
        return
    hg.prep_cache(False)                # features change every training step: both forms repack inside the step
    for name, sh in FNET_SHAPES.items():
        Bf, Vf, H, W, maxd, mind = sh["B"], sh["V"], sh["H"], sh["W"], sh["max_depth"], 1e-3
        fi = make_inputs(B=Bf, V=Vf, D=8, H=H, W=W, C=64, seed=1, depth="smooth", family=sh["family"]).to(dev)
        fr_h, fs_h = fi.ref_feat.to(torch.bfloat16), fi.nghbr_feat.to(torch.bfloat16)
        d_center = magnet_b200.sid_planes(mind, maxd, 80, device=dev)
        gen = torch.Generator(device=dev).manual_seed(2)
        gt = 0.3 + 1.1 * maxd * torch.rand(Bf, 1, H, W, device=dev, generator=gen)
        gt = torch.where(gt > maxd, torch.zeros_like(gt), gt)
        planes = hg._plane_list(d_center)
        count = int((gt > mind).sum())

        def step(r0, s0):
            def fn():
                r, s = r0.detach().clone().requires_grad_(True), s0.detach().clone().requires_grad_(True)
                scores = hg.plane_sweep_f(d_center, r, s, fi.R, fi.t, fi.is_valid, fi.cam_intrins, softmax=False)
                ops.fnet_l1_loss(scores, planes, gt, gt > mind, count=count).backward()
                return scores.detach()
            return fn

        f32, f16 = step(fr_h.float(), fs_h.float()), step(fr_h, fs_h)
        assert torch.equal(f32(), f16()), f"MagnetF {name}: HALF16 and SPLIT16 scores differ"
        ms = _median_pair(f32, f16, steps=args.steps, warmup=args.warmup, loop=1)
        emit(f"magnetf_matching_{name}", *ms, loop=1, shape={"B": Bf, "V": Vf, "D": 80, "C": 64, "H": H, "W": W},
             array_equal=True)
    hg.prep_cache(True)


if __name__ == "__main__":
    main()
