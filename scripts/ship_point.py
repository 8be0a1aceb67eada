"""The reference's SHIPPED operating point (test_scripts/magnet/scannet.txt:8-14: N_s = 5 samples, 3 iterations, 4 source
views; KITTI: 2 views) — a launch-latency regime (SURVEY §7 hard part 4): the whole matching loop of one frame is ~10
short kernels.  Reports, for batch 1: per-kernel device times, the eager loop time and the CUDA-graph-replayed loop time.
usage: python scripts/ship_point.py [out.md]"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import magnet_b200  # noqa: E402
from magnet_b200 import _lib, ops  # noqa: E402
from magnet_b200.synthetic import make_inputs  # noqa: E402

dev = torch.device("cuda")
rows = []
for name, kw in (("scannet 640x480, V=4, N_s=5", dict(B=1, V=4, D=5, H=120, W=160, C=64, family="scannet")),
                 ("kitti 1216x352, V=2, N_s=5", dict(B=1, V=2, D=5, H=88, W=304, C=64, family="kitti")),
                 ("scannet 640x480, V=4, N_s=5, batch 8", dict(B=8, V=4, D=5, H=120, W=160, C=64, family="scannet"))):
    inp = make_inputs(seed=3, depth="smooth", **kw)
    g = inp.to(dev)
    B, V, D = inp.B, inp.V, inp.D
    H, W = inp.ref_feat.shape[2:]
    k = ops.k_array(magnet_b200.depth_sampling(3, 5))
    raw = torch.randn(B, 2, H, W, device=dev) * 0.1
    intM_d, rays_d = inp.cam_intrins['intM'].to(dev), inp.cam_intrins['unit_ray_array_2D'].to(dev).contiguous()
    valid_d = inp.is_valid.to(dev)
    res = {}
    for vname, variant, layout in (("tensor-core", _lib.VARIANT_MMA, _lib.SRC_SPLIT16), ("gather", _lib.VARIANT_CELLS, _lib.SRC_TILED32),
                                   ("tma", _lib.VARIANT_TMA, _lib.SRC_PIXC)):
        ref_split = None
        if layout == _lib.SRC_SPLIT16:
            src = torch.empty(int(_lib.lib().magnet_split16_bytes(V * B, H, W)), device=dev, dtype=torch.uint8)
            ref_split = torch.empty(int(_lib.lib().magnet_split16_bytes(B, H, W)), device=dev, dtype=torch.uint8)
        elif layout == _lib.SRC_PIXC:
            src = torch.empty(V * B, H, W, 68, device=dev)
        else:
            src = torch.empty(V * B, H, (W + 31) // 32, 16, 32, 4, device=dev)
        cv = torch.empty(B, D, H, W, device=dev)

        def frame():
            if layout == _lib.SRC_SPLIT16:
                ops.repack_split16(g.nghbr_feat, g.nghbr_gmms, out=src)
                ops.repack_split16(g.ref_feat, out=ref_split)
            elif layout == _lib.SRC_PIXC:
                ops.repack_pixc(g.nghbr_feat, g.nghbr_gmms, out=src)
            else:
                ops.repack_tiled32(g.nghbr_feat, out=src)
            cams = ops.pack_cameras(intM_d, g.R, g.t, valid_d)
            pred = g.ref_gmms
            for _ in range(3):
                ops.cost_volume(g.ref_feat, src, rays_d, cams, V=V, src_layout=layout, consistency=True, src_gmm=g.nghbr_gmms,
                                kappa=5.0, ref_gmm=pred, k=k, out=cv, variant=variant, ref_split=ref_split)
                pred = ops.gaussian_update(raw, pred)
            return pred

        def timeit(fn, n):
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(n):
                fn()
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) / n

        with torch.no_grad():
            for _ in range(5):
                frame()
            eager = timeit(frame, 200)
            graph = torch.cuda.CUDAGraph()
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                with torch.cuda.graph(graph, stream=side):
                    frame()
            torch.cuda.current_stream().wait_stream(side)
            for _ in range(5):
                graph.replay()
            replay = timeit(graph.replay, 500)
            # the cost kernel alone
            cams = ops.pack_cameras(intM_d, g.R, g.t, valid_d)
            kern = timeit(lambda: ops.cost_volume(g.ref_feat, src, rays_d, cams, V=V, src_layout=layout, consistency=True,
                                                  src_gmm=g.nghbr_gmms, kappa=5.0, ref_gmm=g.ref_gmms, k=k, out=cv,
                                                  variant=variant, ref_split=ref_split), 300)
        res[vname] = (eager, replay, kern)
    rows.append((name, B, res))
    print(name, res, flush=True)
lines = ["# shipped operating point (N_s = 5, 3 iterations): launch-latency regime, 1 x H100",
         "One frame = repack (tensor-core: max|x| + split of source and reference features, 4 launches) + camera table + 3 x "
         "(fused cost kernel + update kernel) = 8 (11) launches.  eager = Python/ctypes "
         "launches back to back; graph = the same 8 kernels replayed from one CUDA graph; cost kernel = that kernel alone "
         "(back-to-back launches, so launch overhead included).\n",
         "| workload | kernel | eager ms/frame-batch | graph ms/frame-batch | cost kernel ms | frames/s (graph) |", "|---|---|---:|---:|---:|---:|"]
for name, B, res in rows:
    for vname, (eager, replay, kern) in res.items():
        lines.append("| %s | %s | %.4f | %.4f | %.4f | %.0f |" % (name, vname, eager, replay, kern, B * 1e3 / replay))
open(sys.argv[1] if len(sys.argv) > 1 else "ship_point.md", "w").write("\n".join(lines) + "\n")
