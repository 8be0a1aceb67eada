"""The SPLIT16 / HALF16 producer (ops.repack_split16 / ops.repack_half16) against the HBM roofline, at the bench.py
workloads: for the source maps (with their Gaussians) and the reference maps of each config,
  * the whole call: `--loop` calls captured in one CUDA graph (device time, no host overhead), CUDA events around
    replays, the median of `--steps` (>= 20) repeats;
  * each part of it (the header memset, where a build still has one, absmax_kernel, split16_repack_kernel): device time
    per call from torch.profiler (CUDA activities) over `--loop` calls, in a run of its own;
  * GB/s of each part against the bytes it moves, and of the call against its algorithmic bytes (the map and the
    Gaussians read once, planes and table written once), as a share of MEASURED_PEAKS.json's HBM bandwidth when the
    file exists, of the H100 SXM data sheet's 3.35 TB/s otherwise.
`--step` also replays the headline step of bench.py from a CUDA graph under the profiler and reports each kernel's
device time per step, their sum and the replay time under the same profiler (CUDA events): the difference is time
between kernels.  The step time with the profiler off is reported beside it.
Prints one JSON line per measurement with the card, its power limit and its SM clock limit; writes nothing.

usage: python scripts/bench_repack.py [--config cfg2 cfg3] [--steps K] [--warmup W] [--loop L] [--half] [--step]"""
import argparse
import json
import os
import sys
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import torch  # noqa: E402

from bench import N_ITER, measured_peak  # noqa: E402
from bench_fnet import _power_limit_w  # noqa: E402

PARTS = (("memset", ("memset",)), ("absmax_kernel", ("absmax_kernel",)),
         ("split16_repack_kernel", ("split16_repack_kernel",)))


def _sm_max_mhz():
    try:
        import pynvml
        pynvml.nvmlInit()
        return pynvml.nvmlDeviceGetMaxClockInfo(pynvml.nvmlDeviceGetHandleByIndex(0), pynvml.NVML_CLOCK_SM)
    except Exception:
        return None


def _graph(fn, calls, dev):
    """fn called `calls` times, captured in one CUDA graph."""
    graph = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side), torch.cuda.graph(graph, stream=side):
        for _ in range(calls):
            fn()
    torch.cuda.current_stream().wait_stream(side)
    return graph


def _median_ms(fn, steps, warmup, loop):
    t = []
    for i in range(warmup + steps):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(loop):
            fn()
        e.record()
        torch.cuda.synchronize()
        if i >= warmup:
            t.append(s.elapsed_time(e) / loop)
    return sorted(t)[len(t) // 2]


def _kernel_us(fn, calls):
    """Device time per call of every CUDA activity fn launches, by name (torch.profiler, CUDA activities), and the
    time per call of the profiled region (CUDA events)."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(calls):
            fn()
        e.record()
        torch.cuda.synchronize()
    out = defaultdict(float)
    for ev in prof.key_averages():
        us = getattr(ev, "device_time_total", None)
        if us is None:
            us = ev.cuda_time_total
        if us > 0:
            out[ev.key] += us / calls
    return dict(out), s.elapsed_time(e) / calls


def _part_us(per_name):
    got = {}
    for part, keys in PARTS:
        hits = [us for name, us in per_name.items() if any(k in name.lower() for k in keys)]
        got[part] = sum(hits) if hits else None
    return got


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", nargs="+", default=["cfg2", "cfg3"], choices=["cfg2", "cfg3"])
    ap.add_argument("--steps", type=int, default=30, help="timed repeats of the whole call (at least 20)")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--loop", type=int, default=20, help="calls per timed repeat / per profiled run")
    ap.add_argument("--half", action="store_true", help="also the HALF16 producer on the bf16-rounded maps")
    ap.add_argument("--step", action="store_true", help="also the kernels of bench.py's headline step")
    args = ap.parse_args()
    args.steps = max(20, args.steps)
    if not torch.cuda.is_available():
        raise SystemExit("bench_repack.py needs a CUDA device: magnet_b200 has no CPU path")
    from magnet_b200 import _lib, ops
    from magnet_b200.synthetic import make_config

    dev = torch.device("cuda:0")
    peak, peak_src = measured_peak()
    card = {"card": torch.cuda.get_device_name(dev), "power_limit_w": _power_limit_w(0), "sm_max_mhz": _sm_max_mhz(),
            "lib": os.path.basename(str(_lib.LIB_PATH)), "peak_gbs": peak, "peak_source": peak_src}

    for cfg in args.config:
        inp = make_config(cfg, seed=0)
        g = inp.to(dev)
        maps = [("source", g.nghbr_feat, g.nghbr_gmms), ("reference", g.ref_feat, None)]
        forms = [("split16", ops.repack_split16, lambda x: x, 2)]
        if args.half:
            forms.append(("half16", ops.repack_half16, lambda x: x.to(torch.bfloat16), 1))
        for form, repack, cast, planes in forms:
            for which, feat, gmm in maps:
                x = cast(feat).contiguous()
                N, C, H, W = x.shape
                buf = repack(x, gmm)
                call = lambda: repack(x, gmm, out=buf)                        # noqa: E731
                read = x.numel() * x.element_size()
                gbytes = 0 if gmm is None else gmm.numel() * 4
                written = N * H * W * 128 * planes + N * H * (W + 1) * 16
                moved = {"memset": None, "absmax_kernel": read, "split16_repack_kernel": read + gbytes + written}
                graph = _graph(call, args.loop, dev)
                ms = _median_ms(graph.replay, args.steps, args.warmup, 1) / args.loop
                per_name, _ = _kernel_us(call, args.loop)
                parts = {}
                for part, us in _part_us(per_name).items():
                    if us is None:
                        continue
                    row = {"us": round(us, 2)}
                    if moved[part]:
                        row["bytes"] = moved[part]
                        row["gbs"] = round(moved[part] / (us * 1e-6) / 1e9, 1)
                        row["frac_of_peak"] = round(moved[part] / (us * 1e-6) / 1e9 / peak, 3)
                    parts[part] = row
                algo = read + gbytes + written + 256
                print(json.dumps({"config": cfg, "form": form, "map": which, "shape": [N, C, H, W],
                                  "call_ms": round(ms, 4), "call_algorithmic_bytes": algo,
                                  "call_gbs": round(algo / (ms * 1e-3) / 1e9, 1),
                                  "call_frac_of_peak": round(algo / (ms * 1e-3) / 1e9 / peak, 3),
                                  "roofline_ms": round(algo / (peak * 1e9) * 1e3, 4), "parts": parts,
                                  "steps": args.steps, "loop": args.loop, **card}), flush=True)
                del buf, graph
        if args.step:
            _step_profile(cfg, inp, g, dev, args, card)
        del g
        torch.cuda.empty_cache()


def _step_profile(cfg, inp, g, dev, args, card):
    """bench.py's headline step (both repacks, camera table, N_ITER x (cost kernel + update)), captured in a CUDA graph:
    each kernel's device time per replay against the replay's time."""
    from magnet_b200 import _lib, ops
    B, V = inp.B, inp.V
    H, W = g.ref_feat.shape[2:]
    karr = ops.k_array([float(v) for v in inp.k.tolist()])
    gen = torch.Generator().manual_seed(5)
    raw = (torch.randn(B, 2, H, W, generator=gen) * 0.1).to(dev)
    intM, rays = inp.cam_intrins["intM"].to(dev), inp.cam_intrins["unit_ray_array_2D"].to(dev).contiguous()
    valid = inp.is_valid.to(dev)
    src = torch.empty(ops.packed_bytes(_lib.SRC_SPLIT16, V * B, H, W), device=dev, dtype=torch.uint8)
    ref = torch.empty(ops.packed_bytes(_lib.SRC_SPLIT16, B, H, W), device=dev, dtype=torch.uint8)
    cv = torch.empty(B, inp.D, H, W, device=dev)

    def step():
        ops.repack_split16(g.nghbr_feat, g.nghbr_gmms, out=src)
        ops.repack_split16(g.ref_feat, out=ref)
        cams = ops.pack_cameras(intM, g.R, g.t, valid)
        pred = g.ref_gmms
        for _ in range(N_ITER):
            ops.cost_volume(g.ref_feat, src, rays, cams, V=V, src_layout=_lib.SRC_SPLIT16, consistency=True,
                            src_gmm=g.nghbr_gmms, kappa=float(inp.thres), ref_gmm=pred, k=karr, out=cv, ref_split=ref)
            pred = ops.gaussian_update(raw, pred)
        return pred

    with torch.no_grad():
        for _ in range(3):
            step()
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side), torch.cuda.graph(graph, stream=side):
            step()
        torch.cuda.current_stream().wait_stream(side)
        ms = _median_ms(graph.replay, args.steps, args.warmup, args.loop)
        per_name, prof_ms = _kernel_us(graph.replay, args.loop)
    kernels = {k: round(v, 2) for k, v in sorted(per_name.items(), key=lambda kv: -kv[1])}
    busy = sum(per_name.values()) / 1e3
    print(json.dumps({"config": cfg, "what": "headline_step_graph", "step_ms": round(ms, 4),
                      "profiled_step_ms": round(prof_ms, 4), "kernels_ms": round(busy, 4),
                      "between_kernels_ms": round(prof_ms - busy, 4),
                      "us_per_step": kernels, "steps": args.steps, "loop": args.loop, **card}), flush=True)


if __name__ == "__main__":
    main()
