"""Runs the tensor-core cost kernel of a MAGNET_MMA_DEBUG build (selected by MAGNET_B200_LIB) over the window-box cases
of test_gpu_mma_box.py and prints, per case, the kernel's two counters as one JSON line: hypotheses whose cell origin
fell outside their window box, and tile rows whose box took the exact per-hypothesis pass."""
import ctypes as C
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import magnet_b200  # noqa: E402
from magnet_b200 import _lib, ops  # noqa: E402
from magnet_b200.homography import plane_sweep_f  # noqa: E402
from magnet_b200.synthetic import make_config, make_inputs  # noqa: E402

COUNTERS = 16 + 64 * 256                                   # MMA_DBG_OUTSIDE in csrc/cost_mma.cu
L = _lib.lib()
assert hasattr(L, "magnet_mma_debug_buffer"), "not a MAGNET_MMA_DEBUG build"
dev = torch.device("cuda:0")
buf = torch.zeros(COUNTERS + 2, dtype=torch.float32, device=dev)


def counted(fn):
    buf.zero_()
    L.magnet_mma_debug_buffer(C.c_void_p(buf.data_ptr()))
    try:
        fn()
        torch.cuda.synchronize()
    finally:
        L.magnet_mma_debug_buffer(C.c_void_p(0))
    out, exact = buf[COUNTERS:].view(torch.int32).tolist()
    return [out, exact]


def both_modes(inp):
    g = inp.to(dev)
    plan = magnet_b200.MatchingPlan(g.ref_feat, g.nghbr_feat, g.nghbr_gmms, g.nghbr_poses, inp.is_valid, inp.cam_intrins,
                                    thres=inp.thres)
    k = inp.k.tolist()
    dvol = ops.sample_depths(g.ref_gmms, k)
    gauss = counted(lambda: plan.cost(g.ref_gmms, k, variant=_lib.VARIANT_MMA))
    volume = counted(lambda: magnet_b200.est_costvolume_CW(dvol, g.ref_feat, g.nghbr_feat, g.ref_gmms, g.nghbr_gmms, g.R,
                                                           g.t, inp.is_valid, inp.cam_intrins, inp.thres,
                                                           variant=_lib.VARIANT_MMA))
    return gauss, volume


res = {}
rng = np.random.default_rng(4048)                          # the shapes of test_mma_kernel_fuzz_against_direct_kernel
for it in range(24):
    B, V = int(rng.integers(1, 3)), int(rng.integers(1, 7))
    D = int(rng.choice([1, 3, 5, 17, 33, 64, 65, 150])) if it % 3 else int(rng.integers(1, 70))
    H, W = int(rng.integers(5, 41)), int(rng.integers(5, 71))
    depth = "random" if it % 4 == 0 else "smooth"
    family = "kitti" if it % 5 == 0 else "scannet"
    kw = dict(rot_deg=float(rng.uniform(1, 14)), trans=float(rng.uniform(0.05, 0.7))) if it % 2 else {}
    invalid = [(0, int(rng.integers(0, V)))] if V > 1 and it % 3 == 0 else ()
    rng.integers(-3, 4)
    inp = make_inputs(B=B, V=V, D=D, H=H, W=W, C=64, seed=3000 + it, depth=depth, family=family, invalid=invalid, **kw)
    res[f"fuzz{it}/gauss"], res[f"fuzz{it}/volume"] = both_modes(inp)
for cfg in ("cfg2", "cfg3"):
    res[f"{cfg}/gauss"], res[f"{cfg}/volume"] = both_modes(make_config(cfg, seed=1))

# SID planes from 1e-3 with the source cameras behind the reference centre (t_z < 0): z <= 0 at the nearest planes
inp = make_inputs(B=2, V=2, D=8, H=40, W=64, C=64, seed=17, depth="smooth")
inp.nghbr_poses[:, :, 2, 3] = -0.3
g = inp.to(dev)
d_center = magnet_b200.sid_planes(1e-3, 10.0, 80, device=dev)
res["sid_planes"] = counted(lambda: plane_sweep_f(d_center, g.ref_feat, g.nghbr_feat, g.R, g.t, inp.is_valid,
                                                  inp.cam_intrins, softmax=False))
print(json.dumps(res))
