"""Runs the tensor-core cost kernel of a MAGNET_MMA_DEBUG build (selected by MAGNET_B200_LIB) on HALF16 buffers over the
fuzz shapes and feature scales of test_mma_kernel_fuzz_against_direct_kernel, both depth modes, and prints per case the kernel's two
counters as one JSON line: hypotheses whose cell origin fell outside their window box, and tile rows whose box took
the exact per-hypothesis pass."""
import ctypes as C
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import magnet_b200  # noqa: E402
from magnet_b200 import _lib, ops  # noqa: E402
from magnet_b200.synthetic import make_inputs  # noqa: E402

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
    return buf[COUNTERS:].view(torch.int32).tolist()


res = {}
rng = np.random.default_rng(4048)
for it in range(24):
    B, V = int(rng.integers(1, 3)), int(rng.integers(1, 7))
    D = int(rng.choice([1, 3, 5, 17, 33, 64, 65, 150])) if it % 3 else int(rng.integers(1, 70))
    H, W = int(rng.integers(5, 41)), int(rng.integers(5, 71))
    depth = "random" if it % 4 == 0 else "smooth"
    family = "kitti" if it % 5 == 0 else "scannet"
    kw = dict(rot_deg=float(rng.uniform(1, 14)), trans=float(rng.uniform(0.05, 0.7))) if it % 2 else {}
    invalid = [(0, int(rng.integers(0, V)))] if V > 1 and it % 3 == 0 else ()
    inp = make_inputs(B=B, V=V, D=D, H=H, W=W, C=64, seed=3000 + it, depth=depth, family=family, invalid=invalid, **kw)
    scale = float(10.0 ** rng.integers(-3, 4))             # feature scales from 1e-3 to 1e3, as the fuzz test
    inp.ref_feat.mul_(scale)
    inp.nghbr_feat.mul_(1.0 / scale if it % 2 else scale)
    g = inp.to(dev)
    ref, src = g.ref_feat.to(torch.bfloat16), g.nghbr_feat.to(torch.bfloat16)
    plan = magnet_b200.MatchingPlan(ref, src, g.nghbr_gmms, g.nghbr_poses, inp.is_valid, inp.cam_intrins, thres=inp.thres)
    k = inp.k.tolist()
    dvol = ops.sample_depths(g.ref_gmms, k)
    res[f"fuzz{it}/gauss"] = counted(lambda: plan.cost(g.ref_gmms, k, variant=_lib.VARIANT_MMA))
    res[f"fuzz{it}/volume"] = counted(lambda: magnet_b200.est_costvolume_CW(
        dvol, ref, src, g.ref_gmms, g.nghbr_gmms, g.R, g.t, inp.is_valid, inp.cam_intrins, inp.thres,
        variant=_lib.VARIANT_MMA))
print(json.dumps(res))
