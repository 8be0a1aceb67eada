"""Evaluation steps eager against torch.compile(mode="reduce-overhead") (CUDA-graph trees over the registered ops).

Workloads, 480x640 GT (ScanNet, quarter resolution 120x160, V = 4, C = 64, min 1e-3, max 10):
  head:  MagnetHead(fused_upsample=True, N_s) + DepthMetrics.update of its N_iter predictions, B = 1 and 8;
  dnet:  DnetHead + DepthMetrics.update(variance=True), B = 1;
  fnet:  MagnetF(identity F-Net).predict over 80 SID planes + DepthMetrics.update(nearest=True), B = 1.
Each step is timed with CUDA events around a loop of calls; eager and compiled alternate, and the median over repeats is
reported with the card and its power limit read in the same run.  Cameras and validity are on the device (a CUDA graph
has no host inputs); the compiled step is called on the same tensors each time.  ``cudagraph_skips`` counts the graphs
CUDA-graph trees declined to capture (0: every graph replays).

``--parent DIR`` also times the eager head step of the package in DIR (the previous revision, built) alternately with
this one's, to show what the traced-call branch costs an eager call.

usage: python scripts/bench_compile.py [--reps R] [--iters N] [--n-samples S] [--parent DIR]"""
import argparse
import importlib.util
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import torch  # noqa: E402
import torch.nn as nn  # noqa: E402

from bench_fnet import _power_limit_w  # noqa: E402

H, W = 120, 160


def _load_package(tree: str, name: str):
    """The magnet_b200 package of another source tree, imported under ``name``."""
    pkg = os.path.join(tree, "magnet_b200")
    spec = importlib.util.spec_from_file_location(name, os.path.join(pkg, "__init__.py"), submodule_search_locations=[pkg])
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    spec.loader.exec_module(mod)
    return mod


def _head_step(pkg, dev, B, n_samples):
    """(step, args) of the MaGNet head and the metrics update at batch B, built from package ``pkg``."""
    from magnet_b200.synthetic import make_inputs
    torch.manual_seed(0)
    head = pkg.MagnetHead(n_samples=n_samples, fused_upsample=True).to(dev).eval()
    metrics = pkg.DepthMetrics(1e-3, 10.0)
    inp = make_inputs(B=B, V=4, D=n_samples, H=H, W=W, C=64, seed=1)
    g = inp.to(dev)
    cam = {k: v.to(dev) for k, v in inp.cam_intrins.items()}
    x_d3 = torch.randn(B, 256, H, W, device=dev)
    gt = 0.5 + 8 * torch.rand(B, 1, 4 * H, 4 * W, device=dev)

    def step(ref_feat, nghbr_feat, ref_gmms, nghbr_gmms, x_d3, poses, valid, intM, rays, gt):
        preds = head(ref_feat, nghbr_feat, ref_gmms, nghbr_gmms, x_d3, poses, valid,
                     {"intM": intM, "unit_ray_array_2D": rays})
        return metrics.update(preds, gt)

    return step, (g.ref_feat, g.nghbr_feat, g.ref_gmms, g.nghbr_gmms, x_d3, g.nghbr_poses, inp.is_valid.to(dev),
                  cam["intM"], cam["unit_ray_array_2D"], gt)


def _dnet_step(pkg, dev):
    torch.manual_seed(0)
    head = pkg.DnetHead().to(dev).eval()
    metrics = pkg.DepthMetrics(1e-3, 10.0)

    def step(x, gt):
        return metrics.update(head(x), gt, variance=True)

    return step, (torch.randn(1, 256, H, W, device=dev), 0.5 + 8 * torch.rand(1, 1, 4 * H, 4 * W, device=dev))


def _fnet_step(pkg, dev):
    from magnet_b200.synthetic import make_inputs
    model = pkg.MagnetF(nn.Identity())
    metrics = pkg.DepthMetrics(1e-3, 10.0)
    planes = pkg.sid_planes(1e-3, 10.0, 80).flatten().tolist()
    inp = make_inputs(B=1, V=4, D=8, H=H, W=W, C=64, seed=2)
    g = inp.to(dev)
    cam = {k: v.to(dev) for k, v in inp.cam_intrins.items()}

    def step(ref, nghbr, poses, valid, intM, rays, gt):
        pred = model.predict(ref, nghbr, poses, valid, {"intM": intM, "unit_ray_array_2D": rays}, planes)
        return metrics.update(pred, gt, nearest=True)

    return step, (g.ref_feat, g.nghbr_feat, g.nghbr_poses, inp.is_valid.to(dev), cam["intM"],
                  cam["unit_ray_array_2D"], 0.5 + 8 * torch.rand(1, 1, 4 * H, 4 * W, device=dev))


def _ms_per_call(fn, args, iters):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn(*args)
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / iters


def _alternate(fns, args, reps, iters):
    """Median ms per call of each of ``fns`` (name -> callable), timed in alternation."""
    for fn in fns.values():                            # warm-up: compilation, capture, cuDNN's algorithm choice
        for _ in range(5):
            fn(*args)
    torch.cuda.synchronize()
    times = {name: [] for name in fns}
    for _ in range(reps):
        for name, fn in fns.items():
            times[name].append(_ms_per_call(fn, args, iters))
    return {name: statistics.median(t) for name, t in times.items()}, {name: (min(t), max(t)) for name, t in times.items()}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--n-samples", type=int, default=5)
    ap.add_argument("--parent", default=None, help="a built source tree of the previous revision (eager before/after)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_compile.py needs a CUDA device")
    import magnet_b200
    from torch._dynamo.utils import counters

    dev = torch.device("cuda:0")
    card = {"card": torch.cuda.get_device_name(dev), "power_limit_w": _power_limit_w(0)}
    torch.backends.cudnn.benchmark = False
    with torch.no_grad():
        work = [(f"head B={B} N_s={args.n_samples} + metrics", lambda B=B: _head_step(magnet_b200, dev, B, args.n_samples))
                for B in (1, 8)]
        work += [("dnet B=1 + metrics(variance)", lambda: _dnet_step(magnet_b200, dev)),
                 ("fnet predict B=1 + metrics(nearest)", lambda: _fnet_step(magnet_b200, dev))]
        for name, make in work:
            torch._dynamo.reset()
            counters.clear()
            eager, a = make()
            compiled_step, _ = make()
            compiled = torch.compile(compiled_step, mode="reduce-overhead")
            med, rng = _alternate({"eager": eager, "compiled": compiled}, a, args.reps, args.iters)
            print(json.dumps({"workload": name, "eager_ms": round(med["eager"], 4), "compiled_ms": round(med["compiled"], 4),
                              "speedup": round(med["eager"] / med["compiled"], 3),
                              "eager_range_ms": [round(x, 4) for x in rng["eager"]],
                              "compiled_range_ms": [round(x, 4) for x in rng["compiled"]],
                              "cudagraph_skips": int(counters["inductor"]["cudagraph_skips"]),
                              "reps": args.reps, "iters": args.iters, **card}), flush=True)
        if args.parent:
            parent = _load_package(os.path.abspath(args.parent), "magnet_b200_parent")
            for B in (1, 8):
                fns, a = {}, None
                for tag, pkg in (("parent", parent), ("change", magnet_b200)):
                    fns[tag], a = _head_step(pkg, dev, B, args.n_samples)
                med, rng = _alternate(fns, a, args.reps, args.iters)
                print(json.dumps({"workload": f"eager head B={B} N_s={args.n_samples} + metrics, parent vs change",
                                  "parent_ms": round(med["parent"], 4), "change_ms": round(med["change"], 4),
                                  "parent_range_ms": [round(x, 4) for x in rng["parent"]],
                                  "change_range_ms": [round(x, 4) for x in rng["change"]],
                                  "reps": args.reps, "iters": args.iters, **card}), flush=True)


if __name__ == "__main__":
    main()
