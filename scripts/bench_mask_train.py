"""The mask head of training: the module path (mask_head(x_d3) on cuDNN, cudnn.benchmark on, PyTorch's default TF32
flags, then ops.magnet_loss over 3 predictions) against the fused path (MagnetHead.mask_pre on cuDNN +
ops.mask_head_loss), forward + backward into the mask head's parameters, x_d3 and the predictions, on the same inputs.
In one process, alternating repeat by repeat, CUDA events around `--loop` steps after warm-up, the median of `--samples`
(>= 20) repeats.  Then each new kernel alone under torch.profiler: its mean device time and its share of the H100 SXM
data-sheet bound (3.35 TB/s HBM3, 989 TFLOP/s dense fp16 with three products per multiply-add; the weight-gradient
GEMMs' three TF32 products counted against 494 TFLOP/s dense TF32), naming the bound.  Last, unless
`--no-train-head`, the median device time per step of examples/train_head.py (batch 4, 120x160, 20 steps) at N_s 64
and 5, without and with --fused-mask.  Prints one JSON line per measurement with the card name and its power limit;
writes nothing.

usage: python scripts/bench_mask_train.py --config {cfg2,cfg3} [--samples N] [--warmup W] [--loop L] [--no-train-head]"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from bench_fnet import _power_limit_w  # noqa: E402
from bench_half import _median_pair  # noqa: E402

HBM_BPS, FP16_FLOPS, TF32_FLOPS = 3.35e12, 989e12, 494e12
HID, NOUT = 128, 144


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="cfg2", choices=["cfg2", "cfg3"])
    ap.add_argument("--samples", type=int, default=20, help="timed repeats per path (at least 20)")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--loop", type=int, default=5, help="steps per timed repeat")
    ap.add_argument("--no-train-head", action="store_true", help="skip the examples/train_head.py step times")
    args = ap.parse_args()
    args.samples = max(20, args.samples)
    if not torch.cuda.is_available():
        raise SystemExit("bench_mask_train.py needs a CUDA device: magnet_b200 has no CPU path")
    import magnet_b200
    from magnet_b200 import ops
    from magnet_b200.synthetic import make_config

    torch.backends.cudnn.benchmark = True
    dev = torch.device("cuda:0")
    card = {"card": torch.cuda.get_device_name(dev), "power_limit_w": _power_limit_w(0)}
    inp = make_config(args.config)
    B, _, H, W = inp.ref_feat.shape
    shape = dict(B=B, H=H, W=W, P=3)
    torch.manual_seed(0)
    head = magnet_b200.MagnetHead(n_samples=5).to(dev).train()
    mh = head.mask_head
    gen = torch.Generator(device=dev).manual_seed(1)
    x_d3 = torch.randn(B, 256, H, W, device=dev, generator=gen).requires_grad_(True)
    preds = [torch.cat([1.0 + torch.rand(B, 1, H, W, device=dev, generator=gen),
                        0.1 + torch.rand(B, 1, H, W, device=dev, generator=gen)], 1).requires_grad_(True)
             for _ in range(3)]
    gt = 1.0 + torch.rand(B, 1, 4 * H, 4 * W, device=dev, generator=gen)
    gtm = torch.rand(B, 1, 4 * H, 4 * W, device=dev, generator=gen) < 0.7

    def module():
        ops.magnet_loss(preds, mh(x_d3), gt, gtm, 4).backward()

    def fused():
        ops.mask_head_loss(head.mask_pre(x_d3), mh, preds, gt, gtm, 4).backward()

    m_ms, f_ms = _median_pair(module, fused, steps=args.samples, warmup=args.warmup, loop=args.loop)
    print(json.dumps({"config": args.config, "what": "mask_head_loss_fwd_bwd", "module_ms": round(m_ms, 4),
                      "fused_ms": round(f_ms, 4), "speedup": round(m_ms / f_ms, 3), **shape, **card,
                      "samples": args.samples}), flush=True)

    # each kernel of the fused path under the profiler
    pre0 = head.mask_pre(x_d3).detach().requires_grad_(True)
    step = lambda: ops.mask_head_loss(pre0, mh, preds, gt, gtm, 4).backward()
    for _ in range(3):
        step()
    torch.cuda.synchronize()
    n = 10
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            step()
        torch.cuda.synchronize()
    HW, P, map_ = H * W, 3, B * H * W
    # bytes each kernel must move at least and the products it issues
    model = {
        "mask_train_fwd_kernel": ((HID + 2 * P) * map_ * 4 + 16 * map_ * 5 + (3 * HID + NOUT) * map_ * 4,
                                  3 * 2 * (2 * HID * HID + NOUT * HID) * map_, FP16_FLOPS),
        "mask_bwd_chain_kernel": ((NOUT + 3 * HID) * map_ * 4 + 3 * HID * map_ * 4,
                                  3 * 2 * (NOUT * HID + 2 * HID * HID) * map_, FP16_FLOPS),
        "gnet_wgrad_kernel": ((2 * (NOUT + 3 * HID)) * map_ * 4, 3 * 2 * (NOUT * HID + 2 * HID * HID) * map_,
                              TF32_FLOPS),
    }
    for ev in prof.key_averages():
        name = next((k for k in list(model) + ["gnet_wgrad_reduce_kernel", "scale_grads_kernel", "head_scale", "head_pack"]
                     if k in ev.key), None)
        if name is None:
            continue
        us = getattr(ev, "device_time_total", None)
        k_ms = (us if us is not None else ev.cuda_time_total) / n / 1e3       # device time per step
        line = {"config": args.config, "what": ev.key[:60], "kernel_ms_per_step": round(k_ms, 4),
                "launches_per_step": ev.count // n}
        if name in model:
            nbytes, flops, peak = model[name]
            t_b, t_f = nbytes / HBM_BPS, flops / peak
            line.update(bytes=nbytes, bound="tensor cores" if t_f > t_b else "HBM",
                        frac_of_bound=round(max(t_b, t_f) / (k_ms * 1e-3), 3))
        print(json.dumps({**line, **shape, **card, "samples": n}), flush=True)

    # whole training steps of the example, module mask head against --fused-mask
    if args.no_train_head:
        return
    example = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "examples", "train_head.py")
    for hyp in (64, 5):
        for flags in ([], ["--fused-mask"]):
            out = subprocess.run([sys.executable, example, "--steps", "20", "--hypotheses", str(hyp), *flags],
                                 capture_output=True, text=True, check=True).stdout.strip().splitlines()[-1]
            r = json.loads(out)
            print(json.dumps({"what": "train_head_step", "hypotheses": hyp, "fused_mask": bool(flags),
                              "step_ms_median": round(r["rank0_step_ms_median"], 3), "loss_path": r["loss_path"],
                              "B": r["global_batch"], "steps": 20, **card}), flush=True)


if __name__ == "__main__":
    main()
