"""BASELINE.json configs[4]: stress sweep views x hypotheses at the 640x480 (120x160) grid on 1..8 GPUs (weak scaling:
every rank owns its own batch of 8, no data-path collective): per point the cost-kernel time (CUDA events, L2 flushed
between launches, MAX over ranks), algorithmic HBM GB/s and fraction of the measured roofline, for the tensor-core kernel
(fused sampler and drop-in d_volume mode), the global-gather kernel and the TMA-staged CUDA-core kernel (fused sampler).

    python scripts/sweep.py out.md
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 scripts/sweep.py out.md
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import magnet_b200  # noqa: E402
from bench import algorithmic_bytes, measured_peak  # noqa: E402
from magnet_b200 import _lib, dist as md, ops  # noqa: E402
from magnet_b200.synthetic import make_inputs  # noqa: E402

rank, local_rank, world = md.env_world()
torch.cuda.set_device(local_rank)
dev = torch.device("cuda", local_rank)
md.init_process_group("nccl", device_id=dev)
peak, src = measured_peak()
B, H, W, C = 8, 120, 160, 64
flush = torch.empty(64 * 1024 * 1024, device=dev)
VS = [int(v) for v in os.environ.get("SWEEP_V", "2,4,8").split(",")]
DS = [int(d) for d in os.environ.get("SWEEP_D", "32,64,128,256").split(",")]


def median_ms(fn, reps=11):
    for _ in range(3):
        fn()
    ts = []
    for _ in range(reps):
        flush.zero_()
        md.barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(md.max_over_ranks(e0.elapsed_time(e1), device=dev))
    return sorted(ts)[len(ts) // 2]


rows = []
for V in VS:
    for D in DS:
        inp = make_inputs(B=B, V=V, D=D, H=H, W=W, C=C, seed=1, depth="smooth")   # same work on every rank (weak scaling)
        g = inp.to(dev)
        plan = magnet_b200.MatchingPlan(g.ref_feat, g.nghbr_feat, g.nghbr_gmms, g.nghbr_poses, inp.is_valid,
                                        inp.cam_intrins, thres=5)
        k = ops.k_array(inp.k.tolist())
        out = torch.empty(B, D, H, W, device=dev)
        dvol = ops.sample_depths(g.ref_gmms, k)
        spl = plan._source(_lib.SRC_SPLIT16)
        ms_m = median_ms(lambda: plan.cost(g.ref_gmms, k, out=out, variant=_lib.VARIANT_MMA))
        ms_d = median_ms(lambda: ops.cost_volume(plan.ref_feat, spl, plan.rays, plan.cams, V=V, src_layout=_lib.SRC_SPLIT16,
                                                 consistency=True, kappa=5.0, d_volume=dvol, out=out, ref_split=plan._ref_split))
        ms_g = median_ms(lambda: plan.cost(g.ref_gmms, k, out=out, variant=_lib.VARIANT_CELLS))
        ms_t = median_ms(lambda: plan.cost(g.ref_gmms, k, out=out, variant=_lib.VARIANT_TMA))
        ab = algorithmic_bytes(B, V, D, C, H * W, fused=True)
        abd = algorithmic_bytes(B, V, D, C, H * W, fused=False)
        rows.append((V, D, ab / 1e6, ms_m, ab / ms_m / 1e6 / peak, ms_d, abd / ms_d / 1e6 / peak, ms_g, ab / ms_g / 1e6 / peak,
                     ms_t, ab / ms_t / 1e6 / peak, world * B / (3 * ms_m * 1e-3)))
        if rank == 0:
            print(rows[-1], flush=True)
        del plan, g, out, dvol, spl
        torch.cuda.empty_cache()
if rank == 0:
    md_lines = [f"# stress sweep (BASELINE.json configs[4]) on {world} x H100: B=8 per GPU, 120x160 grid (640x480), C=64",
                f"peak = {peak:.0f} GB/s ({src}); kernel ms = median of 11 launches, L2 flushed, max over the {world} ranks; frac = "
                "algorithmic bytes / kernel time / peak (per GPU); frames/s = all ranks' frames / (3 iterations x tensor-core kernel)\n",
                "| views | hyp. | algorithmic MB | tensor-core kernel ms | frac | drop-in ms | frac | gather kernel ms | frac | TMA CUDA-core kernel ms | frac | frames/s (kernel only) |",
                "|---:|---:|---:|---:|---:|---:|---:|---:|---:|---:|---:|---:|"]
    for r in rows:
        md_lines.append("| %d | %d | %.1f | %.3f | %.3f | %.3f | %.3f | %.3f | %.3f | %.3f | %.3f | %.0f |" % r)
    open(sys.argv[1] if len(sys.argv) > 1 else "sweep.md", "w").write("\n".join(md_lines) + "\n")
md.shutdown()
