"""The G-Net head of inference: the module path (cuDNN convolutions + ReLUs + the update kernel, cudnn.benchmark on,
PyTorch's default TF32 flags) against the fused head (one kernel) on the same cost volume, invariant and Gaussian.
In one process, alternating the two repeat by repeat:
  * one iteration (head + update), at D = 64 and at the shipped N_s = 5;
  * the whole matching_loop of 3 iterations with a GNET (cost volumes included) under no_grad, against the same loop
    written out with the module path.
CUDA events around `--loop` calls after warm-up, the median of `--samples` (>= 20) repeats.  Asserts at the timed size
that the raw head outputs (mu1, elu(sigma1) + 1 + 1e-10) of the fused head and of the module path with TF32 off agree
within 1e-4 of each channel's max.  Prints one JSON line per measurement with the card name and its power limit;
writes nothing.

usage: python scripts/bench_gnet.py --config {cfg2,cfg3} [--samples N] [--warmup W] [--loop L]"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from bench_fnet import _power_limit_w  # noqa: E402
from bench_half import _median_pair  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="cfg2", choices=["cfg2", "cfg3"])
    ap.add_argument("--samples", type=int, default=20, help="timed repeats per path (at least 20)")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--loop", type=int, default=10, help="calls per timed repeat")
    args = ap.parse_args()
    args.samples = max(20, args.samples)
    if not torch.cuda.is_available():
        raise SystemExit("bench_gnet.py needs a CUDA device: magnet_b200 has no CPU path")
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

    def emit(what, module_ms, fused_ms, **extra):
        print(json.dumps({"config": args.config, "what": what, "module_ms": round(module_ms, 4),
                          "fused_ms": round(fused_ms, 4), "speedup": round(module_ms / fused_ms, 3),
                          **extra, **card, "samples": args.samples}), flush=True)

    for D in (64, 5):
        torch.manual_seed(0)
        head = magnet_b200.GNET(ch_in=256 + D).to(dev).eval()
        gen = torch.Generator(device=dev).manual_seed(1)
        cost = torch.randn(B, D, H, W, device=dev, generator=gen)
        x_d3 = torch.randn(B, 256, H, W, device=dev, generator=gen)
        with torch.no_grad():
            inv = head.invariant_part(x_d3, D)
            packed = ops.pack_gnet_weights(head, D)
            prev = g.ref_gmms
            module = lambda: ops.gaussian_update(head.raw_from_parts(cost, inv), prev)   # noqa: E731
            fused = lambda: ops.gnet_update(cost, inv, packed, prev)                     # noqa: E731
            # agreement on the raw head output (prev = (0, 1): mu' = mu1), with the module path in fp32: under the
            # default TF32 flags its own error is larger than the bar
            unit = torch.cat([torch.zeros_like(prev[:, :1]), torch.ones_like(prev[:, 1:])], 1)
            tf32 = torch.backends.cudnn.allow_tf32
            torch.backends.cudnn.allow_tf32 = False
            a = ops.gaussian_update(head.raw_from_parts(cost, inv), unit)
            torch.backends.cudnn.allow_tf32 = tf32
            b = ops.gnet_update(cost, inv, packed, unit)
            for c in range(2):
                assert float((a[:, c] - b[:, c]).abs().max()) <= 1e-4 * float(a[:, c].abs().max()), \
                    f"fused head disagrees with the fp32 module path (channel {c})"
            m_ms, f_ms = _median_pair(module, fused, **T)
        emit("iteration", m_ms, f_ms, D=D, B=B, H=H, W=W)

    # the whole loop with the cost volumes (D = 64 hypotheses of the config)
    D = len(inp.k)
    torch.manual_seed(0)
    head = magnet_b200.GNET(ch_in=256 + D).to(dev).eval()
    x_d3 = torch.randn(B, 256, H, W, device=dev)
    karr = inp.k.tolist()
    plan = magnet_b200.MatchingPlan(g.ref_feat, g.nghbr_feat, g.nghbr_gmms, g.nghbr_poses, inp.is_valid,
                                    inp.cam_intrins, thres=inp.thres)

    def loop_fused():
        with torch.no_grad():
            return magnet_b200.matching_loop(plan, g.ref_gmms, x_d3, head, 3, karr)[-1]

    def loop_module():                                     # matching_loop's module path, written out
        with torch.no_grad():
            inv, cur = head.invariant_part(x_d3, D), g.ref_gmms
            for _ in range(3):
                cur = ops.gaussian_update(head.raw_from_parts(plan.cost(cur, karr), inv), cur)
            return cur

    m_ms, f_ms = _median_pair(loop_module, loop_fused, steps=args.samples, warmup=args.warmup, loop=max(1, args.loop // 5))
    emit("matching_loop_3_iterations", m_ms, f_ms, D=D, B=B, H=H, W=W)


if __name__ == "__main__":
    main()
