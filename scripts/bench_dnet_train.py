"""D-Net's training step after the trunk (DESIGN §3.19): the two heads + the learned upsampling + activation_G + DnetLoss,
forward + backward (into both heads' parameters and x_feat), at train_DNet's shapes: ScanNet B 16, 104x136 -> 416x544
and KITTI Eigen B 16, 88x176 -> 352x704, 256 trunk channels.

Routes, on the same module and inputs:
  module   DnetHead.forward in train mode (the module chain: cuDNN heads, ops.convex_upsample, torch's elu) + DnetLoss
           written from its formula with boolean indexing, as a user writes it today;
  fused    DnetHead.loss (cuDNN heads + ops.dnet_loss), eager;
  graphs   DnetHead.loss under torch.compile(mode="reduce-overhead") with the inputs in static buffers.
cuDNN with its default flags (cudnn.benchmark on, TF32 allowed), as train_DNet.py sets them.  Each timed window runs
--steps steps of one route (zero_grad, loss, backward) between CUDA events; the routes alternate window by window for
--repeats windows and the median and range per route are reported.  The loss of each route is printed beside it.
Then, in a separate run, torch.profiler lists the device time of each kernel of one module and one fused step.  Bytes
are computed from the shapes: the full-resolution maps the module route writes, and what the fused kernels read and
write.  One JSON line per measurement with the card, its power limit and its SM clock limit; writes nothing unless
--trace-dir is given.

usage: python scripts/bench_dnet_train.py [--steps K] [--warmup W] [--repeats R] [--only scannet|kitti]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from magnet_b200 import DnetHead  # noqa: E402

CASES = {"scannet": (16, 104, 136), "kitti": (16, 88, 176)}


def _card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=30).stdout.strip()
    name, power, sm_max = [s.strip() for s in q.splitlines()[0].split(",")]
    return {"card": name, "power_limit": power, "sm_clock_max": sm_max}


def module_loss(head, x, gt, gtm):
    """DnetHead.forward (module chain in training) + DnetLoss from its formula (utils/losses.py:13-22)."""
    pred = head(x)
    mu, var = torch.split(pred, 1, dim=1)
    g, mu, var = gt[gtm], mu[gtm], var[gtm]
    var = torch.where(var < 1e-10, torch.full_like(var, 1e-10), var)
    return (torch.square(mu - g) / (2 * var) + 0.5 * torch.log(var)).mean()


def _bytes(B, h, w, k=4):
    hw, full = h * w, h * w * k * k
    return {
        # the module route: the (B,2,kh,kw) upsampled prediction, elu + 1 + 1e-10 and the cat, each a full-res map
        "module_full_res_map_MB": B * 2 * full * 4 / 1e6,
        # the fused forward reads raw, the 9k^2 logits, gt and its mask once; the backward reads them again and writes
        # the logits' gradient and the raw gradient (atomics)
        "fused_fwd_MB": B * (2 * hw * 4 + 9 * k * k * hw * 4 + full * 5) / 1e6,
        "fused_bwd_MB": B * (2 * hw * 4 * 2 + 9 * k * k * hw * 4 * 2 + full * 5) / 1e6,
    }


def _inputs(dev, B, h, w, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    x = torch.relu(torch.randn(B, 256, h, w, device=dev, generator=g))
    gt = 0.5 + 9.5 * torch.rand(B, 1, 4 * h, 4 * w, device=dev, generator=g)
    gtm = torch.rand(B, 1, 4 * h, 4 * w, device=dev, generator=g) < 0.8
    return x, gt, gtm


def _step(head, fn, x, gt, gtm):
    head.zero_grad(set_to_none=False)
    xg = x.detach().requires_grad_()
    loss = fn(xg, gt, gtm)
    loss.backward()
    return loss


def _window(head, fn, args, steps):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(steps):
        loss = _step(head, fn, *args)
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / steps, float(loss)


def run_case(name, args, card):
    dev = torch.device("cuda:0")
    B, h, w = CASES[name]
    torch.manual_seed(0)
    head = DnetHead(in_dim=256).to(dev).train()
    inp = _inputs(dev, B, h, w, 1)
    static = [t.clone() for t in inp]
    compiled = torch.compile(head.loss, mode="reduce-overhead")
    routes = {"module": (lambda x, g, m: module_loss(head, x, g, m), inp),
              "fused": (head.loss, inp),
              "graphs": (compiled, static)}
    for fn, a in routes.values():
        for _ in range(args.warmup):
            _step(head, fn, *a)
    torch.cuda.synchronize()
    times = {r: [] for r in routes}
    losses = {}
    for _ in range(args.repeats):
        for r, (fn, a) in routes.items():
            ms, losses[r] = _window(head, fn, a, args.steps)
            times[r].append(ms)
    for r in routes:
        t = times[r]
        print(json.dumps({"case": name, "B": B, "grid": [h, w], "full_res": [4 * h, 4 * w], "route": r,
                          "ms_per_step_median": round(statistics.median(t), 4), "ms_min": round(min(t), 4),
                          "ms_max": round(max(t), 4), "steps": args.steps, "repeats": args.repeats,
                          "loss": losses[r], **_bytes(B, h, w), **card}), flush=True)
    m = statistics.median(times["module"])
    print(json.dumps({"case": name, "speedup_fused_vs_module": round(m / statistics.median(times["fused"]), 3),
                      "speedup_graphs_vs_module": round(m / statistics.median(times["graphs"]), 3), **card}),
          flush=True)
    _profile(name, head, routes, args)


def _profile(name, head, routes, args):
    """Device time per kernel of one step of the module and the fused route (a separate, profiled run)."""
    from torch.profiler import ProfilerActivity, profile
    for r in ("module", "fused"):
        fn, a = routes[r]
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                _step(head, fn, *a)
            torch.cuda.synchronize()
        rows = []
        for ev in prof.key_averages():
            t = getattr(ev, "device_time_total", None)
            if t is None:
                t = ev.cuda_time_total
            if t > 0:
                rows.append((ev.key[:90], round(t / 3 / 1e3, 4), ev.count // 3))
        rows.sort(key=lambda x: -x[1])
        total = sum(x[1] for x in rows)
        print(json.dumps({"case": name, "route": r, "profile": "device ms per step by kernel",
                          "device_ms_total": round(total, 4), "kernels": rows[:14]}), flush=True)
        if args.trace_dir:
            os.makedirs(args.trace_dir, exist_ok=True)
            prof.export_chrome_trace(os.path.join(args.trace_dir, f"dnet_train_{name}_{r}.json"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--only", choices=sorted(CASES), default=None)
    ap.add_argument("--trace-dir", default=None, help="write the profiler traces here (default: none)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_dnet_train.py needs a CUDA device")
    torch.backends.cudnn.enabled = True
    torch.backends.cudnn.benchmark = True
    card = _card()
    for name in ([args.only] if args.only else CASES):
        run_case(name, args, card)


if __name__ == "__main__":
    main()
