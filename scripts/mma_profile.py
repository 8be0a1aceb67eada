"""Stage profile of the tensor-core cost kernel: where a CTA's cycles go, measured inside the kernel.

Builds libmagnet_b200_<tag>.so with -DMAGNET_MMA_PROFILE (thread 0 of every CTA reads clock64() at the barriers that
separate the stages of a work item), runs cfg2 and cfg3 in GAUSS and VOLUME modes and prints each stage's share of the
CTA cycles, the cycles per (tile, view) pass and the SM clock (CTA cycles over the kernel's CUDA-event time).
usage: python scripts/mma_profile.py [--tag mmaprof] [--no-build] [--reps 20]"""
import argparse, ctypes as C, os, subprocess, sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ap = argparse.ArgumentParser()
ap.add_argument("--tag", default="mmaprof")
ap.add_argument("--no-build", action="store_true", help="use an existing libmagnet_b200_<tag>.so as it is")
ap.add_argument("--reps", type=int, default=20)
args = ap.parse_args()
LIBFILE = os.path.join(ROOT, "magnet_b200", f"libmagnet_b200_{args.tag}.so")
os.environ["MAGNET_B200_LIB"] = LIBFILE                    # read when magnet_b200._lib is imported
sys.path.insert(0, ROOT)
from magnet_b200 import build as _build                    # noqa: E402

if not args.no_build:
    _build.build(defines=("MAGNET_MMA_PROFILE",), tag=args.tag)

import numpy as np, torch                                  # noqa: E402
import magnet_b200                                         # noqa: E402
from magnet_b200 import _lib, ops                          # noqa: E402
from magnet_b200.synthetic import make_config              # noqa: E402

L = _lib.lib()
if not hasattr(L, "magnet_mma_debug_buffer"):
    sys.exit(f"{LIBFILE} is not a MAGNET_MMA_PROFILE build")
# "box" is the first view's box of an item; the boxes of the other views are computed while a view's copies land, so
# they count in "TMA wait + box"
STAGES = ["item setup", "box", "TMA wait + box", "MMA + G", "phase C", "epilogue + fetch"]
try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
except OSError as e:
    q = f"nvidia-smi unavailable ({e})"
print(f"lib {os.path.basename(LIBFILE)}; card: {q}")


def profile(cfg, mode):
    inp = make_config(cfg, seed=1)
    g = inp.to("cuda")
    plan = magnet_b200.MatchingPlan(g.ref_feat, g.nghbr_feat, g.nghbr_gmms, g.nghbr_poses, inp.is_valid, inp.cam_intrins,
                                    thres=5)
    k = ops.k_array(inp.k.tolist())
    out = torch.empty(inp.B, inp.D, *inp.ref_feat.shape[2:], device="cuda")
    dvol = ops.sample_depths(g.ref_gmms, k) if mode == "volume" else None

    def launch():
        if dvol is None:
            plan.cost(g.ref_gmms, k, out=out, variant=_lib.VARIANT_MMA)
        else:
            src = plan._source(_lib.SRC_SPLIT16)
            ops.cost_volume(plan.ref_feat, src, plan.rays, plan.cams, V=plan.V, src_layout=_lib.SRC_SPLIT16,
                            consistency=True, src_gmm=plan.src_gmm, kappa=plan.kappa, d_volume=dvol, out=out,
                            variant=_lib.VARIANT_MMA, ref_split=plan._ref_split)

    for _ in range(3):
        launch()
    torch.cuda.synchronize()
    buf = torch.zeros(8, dtype=torch.int64, device="cuda")
    L.magnet_mma_debug_buffer(C.c_void_p(buf.data_ptr()))
    try:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.reps):
            launch()
        e1.record()
        torch.cuda.synchronize()
    finally:
        L.magnet_mma_debug_buffer(C.c_void_p(0))
    ms = e0.elapsed_time(e1) / args.reps
    t = buf.cpu().numpy().astype(np.float64)
    ctas = t[7] / args.reps
    cyc = t[:len(STAGES)] / args.reps                      # per launch, summed over CTAs
    total = cyc.sum()
    H, W = inp.ref_feat.shape[2:]
    passes = ((H + 7) // 8) * ((W + 7) // 8) * ((inp.D + 63) // 64) * int(inp.is_valid.sum())   # valid (b, v) pairs
    clock = total / ctas / (ms * 1e-3)                     # a persistent CTA lives for the whole launch
    print(f"\n{cfg} {mode}: {ms:.4f} ms/launch (profile build), {int(ctas)} CTAs, SM clock ~{clock / 1e9:.2f} GHz, "
          f"{total / passes:.0f} CTA cycles per (tile, view) pass")
    for name, c in zip(STAGES, cyc):
        print(f"  {name:<18} {100 * c / total:5.1f} %   {c / passes:7.0f} cycles / pass")


for cfg in ("cfg2", "cfg3"):
    for mode in ("gauss", "volume"):
        profile(cfg, mode)
