"""F-Net training benchmark: the matching side of one F-Net training step (train_FNet.py:95-114) at the training
shapes of train_scripts/fnet/*.txt, native (MagnetF's path) against drop-in (est_costvolume_F + the training script's
ATen loss), plus each volume backward kernel alone.  Prints one JSON line; writes nothing.

usage: python scripts/bench_fnet.py --fnet {scannet,kitti} [--steps K] [--warmup W]"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402


# F-Net training shapes (train_scripts/fnet/*.txt): batch, source views, dpv size, max_depth; 80 SID planes from 1e-3
FNET_SHAPES = {"scannet": dict(B=2, V=4, H=120, W=160, max_depth=10.0, family="scannet"),
               "kitti": dict(B=4, V=2, H=88, W=304, max_depth=80.0, family="kitti")}


def _power_limit_w(index=0):
    """The card's enforced power limit in watts (read only), or None."""
    try:
        import pynvml
        pynvml.nvmlInit()
        return pynvml.nvmlDeviceGetEnforcedPowerLimit(pynvml.nvmlDeviceGetHandleByIndex(index)) / 1000.0
    except Exception:
        try:
            import subprocess
            out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                                 capture_output=True, text=True, timeout=20).stdout.strip()
            return float(out.splitlines()[0])
        except Exception:
            return None


def run_fnet_arm(args):
    """The matching side of one F-Net training step (train_FNet.py:95-114) — split16 repack + scores + loss forward +
    backward into both feature maps — two ways in the same call, alternating step by step:
      native:  MagnetF's path (plane-sweep scores, fused soft-argmin L1 loss, tensor-core volume backward);
      drop-in: est_costvolume_F + the training script's ATen loss + the CUDA-core volume backward.
    PSMNet itself is not timed.  Also times each volume backward kernel alone and reports how far apart the two arms'
    gradients are."""
    import magnet_b200
    from magnet_b200 import homography as hg, ops
    from magnet_b200.synthetic import make_inputs
    import torch.nn.functional as F
    sh = FNET_SHAPES[args.fnet]
    dev = torch.device("cuda", 0)
    B, V, H, W, maxd, mind = sh["B"], sh["V"], sh["H"], sh["W"], sh["max_depth"], 1e-3
    inp = make_inputs(B=B, V=V, D=8, H=H, W=W, C=64, seed=1, depth="smooth", family=sh["family"])
    g = inp.to(dev)
    d_center = magnet_b200.sid_planes(mind, maxd, 80, device=dev)
    gen = torch.Generator(device=dev).manual_seed(2)
    gt_full = 0.3 + 1.1 * maxd * torch.rand(B, 1, 4 * H, 4 * W, device=dev, generator=gen)   # some above max_depth
    hg.prep_cache(False)            # features change every training step: both arms repack inside the step

    def native():
        r, s = g.ref_feat.clone().requires_grad_(True), g.nghbr_feat.clone().requires_grad_(True)
        scores = hg.plane_sweep_f(d_center, r, s, g.R, g.t, inp.is_valid, inp.cam_intrins, softmax=False)
        gt = F.interpolate(torch.where(gt_full > maxd, torch.zeros_like(gt_full), gt_full), size=[H, W], mode="nearest")
        loss = ops.fnet_l1_loss(scores, hg._plane_list(d_center), gt, gt > mind)
        loss.backward()
        return r.grad, s.grad

    def drop_in():
        r, s = g.ref_feat.clone().requires_grad_(True), g.nghbr_feat.clone().requires_grad_(True)
        vol = magnet_b200.est_costvolume_F(d_center, r, s, g.R, g.t, inp.is_valid, inp.cam_intrins)
        pred = torch.sum(vol * d_center, dim=1, keepdim=True)
        gt = gt_full.clone()
        gt[gt > maxd] = 0.0
        gt = F.interpolate(gt, size=[H, W], mode="nearest")
        mask = gt > mind
        loss = torch.mean(torch.abs(pred[mask] - gt[mask]))
        loss.backward()
        return r.grad, s.grad

    def timed(fn):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b), out

    reps = max(20, args.steps)
    for _ in range(max(3, args.warmup)):
        native(), drop_in()
    t_nat, t_drop = [], []
    for _ in range(reps):
        ms, g_nat = timed(native)
        t_nat.append(ms)
        ms, g_drop = timed(drop_in)
        t_drop.append(ms)
    agree = max(float((a - b).abs().max()) / max(float(b.abs().max()), 1e-30) for a, b in zip(g_nat, g_drop))

    # the two volume backward kernels alone, on the same upstream gradient of the scores
    cams = ops.pack_cameras(inp.cam_intrins['intM'].to(dev), g.R, g.t, inp.is_valid.to(dev, torch.int32))
    rays = inp.cam_intrins['unit_ray_array_2D'].to(dev).contiguous()
    planes = hg._plane_list(d_center)
    rs, ss = ops.repack_split16(g.ref_feat), ops.repack_split16(g.nghbr_feat)
    gout = torch.randn(B, 80, H, W, device=dev, generator=gen) * 1e-3
    tc = lambda: ops.cost_volume_f_bwd(g.ref_feat, g.nghbr_feat, rays, cams, planes, V, None, gout, softmax=False,
                                       ref_split=rs, src_split=ss)
    cc = lambda: ops.cost_volume_f_bwd(g.ref_feat, g.nghbr_feat, rays, cams, planes, V, None, gout, softmax=False)
    for _ in range(3):
        tc(), cc()
    k_tc, k_cc = [], []
    for _ in range(reps):
        k_tc.append(timed(tc)[0])
        k_cc.append(timed(cc)[0])
    med = lambda xs: sorted(xs)[len(xs) // 2]
    line = {
        "metric": f"fnet_train_step_{args.fnet}", "unit": "ms", "value": med(t_nat),
        "shape": {"B": B, "V": V, "D": 80, "C": 64, "H": H, "W": W, "min_depth": mind, "max_depth": maxd},
        "native_ms": med(t_nat), "drop_in_ms": med(t_drop), "speedup": med(t_drop) / med(t_nat),
        "bwd_kernel_tensor_core_ms": med(k_tc), "bwd_kernel_cuda_core_ms": med(k_cc),
        "grad_max_rel_diff": agree, "repeats": reps,
        "card": torch.cuda.get_device_name(dev), "power_limit_w": _power_limit_w(0),
    }
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--fnet", default="scannet", choices=sorted(FNET_SHAPES))
    ap.add_argument("--steps", type=int, default=20, help="timed repeats per arm (at least 20)")
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fnet.py needs a CUDA device: magnet_b200 has no CPU path")
    run_fnet_arm(args)


if __name__ == "__main__":
    main()
