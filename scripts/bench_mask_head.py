"""The mask head and learned upsampling of inference: the module path (mask_head(x_d3) on cuDNN, cudnn.benchmark on,
PyTorch's default TF32 flags, then one convex_upsample per prediction) against the fused path (MagnetHead.mask_pre on
cuDNN + ops.mask_upsample, one kernel) on the same x_d3 and 3 predictions.  In one process, alternating repeat by repeat:
  * the mask head and the 3 upsamplings alone;
  * whole MagnetHead.forward calls under no_grad with fused_upsample False and True, at N_s = 5 and D = 64 hypotheses.
CUDA events around `--loop` calls after warm-up, the median of `--samples` (>= 20) repeats.  Then the fused kernel alone
under torch.profiler: its device time, bytes per second and share of the H100 SXM data-sheet bound (3.35 TB/s HBM3,
989 TFLOP/s dense fp16, three fp16 products per multiply-add), naming the bound.  Asserts at the timed size that the
fused outputs are within 1e-4 of each channel's max of a float64 evaluation.  Prints one JSON line per measurement with
the card name and its power limit; writes nothing.

usage: python scripts/bench_mask_head.py --config {cfg2,cfg3} [--samples N] [--warmup W] [--loop L]"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from bench_fnet import _power_limit_w  # noqa: E402
from bench_half import _median_pair  # noqa: E402

HBM_BPS, FP16_FLOPS = 3.35e12, 989e12
HID = 128


def _f64_upsample(depth, mask, k=4):
    """upsample_depth_via_mask in float64."""
    N, C, H, W = depth.shape
    w = torch.softmax(mask.view(N, 1, 9, k, k, H, W), dim=2)
    nb = F.unfold(depth, [3, 3], padding=1).view(N, C, 9, 1, 1, H, W)
    return (w * nb).sum(2).permute(0, 1, 4, 2, 5, 3).reshape(N, C, k * H, k * W)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="cfg2", choices=["cfg2", "cfg3"])
    ap.add_argument("--samples", type=int, default=20, help="timed repeats per path (at least 20)")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--loop", type=int, default=10, help="calls per timed repeat")
    args = ap.parse_args()
    args.samples = max(20, args.samples)
    if not torch.cuda.is_available():
        raise SystemExit("bench_mask_head.py needs a CUDA device: magnet_b200 has no CPU path")
    import magnet_b200
    from magnet_b200 import ops
    from magnet_b200.synthetic import make_config

    torch.backends.cudnn.benchmark = True                  # as bench.py and the reference's drivers set it
    dev = torch.device("cuda:0")
    card = {"card": torch.cuda.get_device_name(dev), "power_limit_w": _power_limit_w(0)}
    T = dict(steps=args.samples, warmup=args.warmup, loop=args.loop)
    inp = make_config(args.config)
    g = inp.to(dev)
    B, _, H, W = g.ref_feat.shape
    shape = dict(B=B, H=H, W=W)

    def emit(what, module_ms, fused_ms, **extra):
        print(json.dumps({"config": args.config, "what": what, "module_ms": round(module_ms, 4),
                          "fused_ms": round(fused_ms, 4), "speedup": round(module_ms / fused_ms, 3),
                          **extra, **shape, **card, "samples": args.samples}), flush=True)

    torch.manual_seed(0)
    head = magnet_b200.MagnetHead(n_samples=5).to(dev).eval()
    gen = torch.Generator(device=dev).manual_seed(1)
    x_d3 = torch.randn(B, 256, H, W, device=dev, generator=gen)
    preds = [torch.cat([1.0 + torch.rand(B, 1, H, W, device=dev, generator=gen),
                        0.1 + torch.rand(B, 1, H, W, device=dev, generator=gen)], 1) for _ in range(3)]
    mh = head.mask_head
    with torch.no_grad():
        def module():
            mask = mh(x_d3)
            return [ops.convex_upsample(p, mask, 4) for p in preds]

        def fused():
            return ops.mask_upsample(head.mask_pre(x_d3), ops.pack_mask_weights(mh), preds, 4)

        # accuracy at the timed size: the fused outputs against float64 from the same pre0
        pre0 = head.mask_pre(x_d3)
        got = ops.mask_upsample(pre0, ops.pack_mask_weights(mh), preds, 4)
        h = F.relu(pre0.double())
        for i in (2, 4):
            h = F.relu(F.conv2d(h, mh[i].weight.double(), mh[i].bias.double()))
        mask64 = F.conv2d(h, mh[6].weight.double(), mh[6].bias.double())
        err = 0.0
        for p, o in zip(preds, got):
            want = _f64_upsample(p.double(), mask64)
            for c in range(2):
                e = float((o[:, c].double() - want[:, c]).abs().max() / want[:, c].abs().max())
                assert e <= 1e-4, f"fused mask head off by {e:.2e} of channel {c}'s max"
                err = max(err, e)
        del h, mask64, want
        m_ms, f_ms = _median_pair(module, fused, **T)
    emit("mask_head_and_3_upsamplings", m_ms, f_ms, max_rel_err_f64=float(f"{err:.3g}"))

    # the fused kernel alone under the profiler
    packed = ops.pack_mask_weights(mh)
    with torch.no_grad():
        for _ in range(3):
            ops.mask_upsample(pre0, packed, preds, 4)
        torch.cuda.synchronize()
        n = 20
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(n):
                ops.mask_upsample(pre0, packed, preds, 4)
            torch.cuda.synchronize()
    evs = [ev for ev in prof.key_averages() if "mask_upsample_kernel" in ev.key]
    assert len(evs) == 1 and evs[0].count == n, f"expected {n} mask_upsample_kernel events"
    us = getattr(evs[0], "device_time_total", None)
    k_ms = (us if us is not None else evs[0].cuda_time_total) / n / 1e3      # mean device time per launch
    HW, P = H * W, len(preds)
    nbytes = B * HID * HW * 4 + P * B * 2 * HW * 4 + P * B * 2 * 16 * HW * 4 + ops.mask_weights_bytes(4)
    flops = 3 * 2 * (2 * HID * HID + 144 * HID) * B * HW
    t_bytes, t_flops = nbytes / HBM_BPS, flops / FP16_FLOPS
    print(json.dumps({"config": args.config, "what": "mask_upsample_kernel", "kernel_ms": round(k_ms, 4), "P": P,
                      "bytes": nbytes, "GB_per_s": round(nbytes / (k_ms * 1e-3) / 1e9, 1),
                      "TFLOP_per_s": round(flops / (k_ms * 1e-3) / 1e12, 1),
                      "bound": "fp16 tensor cores" if t_flops > t_bytes else "HBM",
                      "frac_of_bound": round(max(t_bytes, t_flops) / (k_ms * 1e-3), 3),
                      **shape, **card, "samples": n}), flush=True)

    # whole MagnetHead.forward, fused_upsample off / on
    x_d3h = torch.randn(B, 256, H, W, device=dev, generator=gen)
    for ns in (5, 64):
        torch.manual_seed(0)
        hd = magnet_b200.MagnetHead(n_samples=ns, thres=inp.thres).to(dev).eval()
        hf = magnet_b200.MagnetHead(n_samples=ns, thres=inp.thres, fused_upsample=True).to(dev).eval()
        hf.load_state_dict(hd.state_dict())
        fwd_args = (g.ref_feat, g.nghbr_feat, g.ref_gmms, g.nghbr_gmms, x_d3h, g.nghbr_poses, inp.is_valid,
                    inp.cam_intrins)
        with torch.no_grad():
            m_ms, f_ms = _median_pair(lambda: hd(*fwd_args), lambda: hf(*fwd_args), steps=args.samples,
                                      warmup=args.warmup, loop=max(1, args.loop // 5))
        emit("MagnetHead_forward_no_grad", m_ms, f_ms, n_samples=ns)


if __name__ == "__main__":
    main()
