"""Generate tests/golden/cw_train.npz by running the UNMODIFIED reference (a checkout of baegwangbin/MaGNet) on CPU:
    MAGNET_REFERENCE=<path of the checkout> python tests/golden/make_cw_golden.py

One backward pass through est_costvolume_CW (homography.py:79-161) on the seeded case CW_CASE (one invalid view), with
ref_feat, nghbr_feat and d_volume requiring grad: (out * gout).sum().backward() with a seeded gout.  Stores
gout and the three gradients.  Inputs are rebuilt from the seed (the file carries their sha256, as the files of
make_golden.py).
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from make_golden import _import_reference  # noqa: E402
from tests.util import input_digest  # noqa: E402

CW_CASE = dict(B=2, V=3, D=8, H=12, W=16, C=64, seed=91, depth="random", invalid=[(1, 2)])


def cw_gout(B, D, H, W, seed=92):
    return torch.from_numpy(np.random.default_rng(seed).standard_normal((B, D, H, W)).astype(np.float32))


def main():
    _import_reference()
    import models.submodules.homography as refh
    from magnet_b200.synthetic import make_inputs
    torch.set_num_threads(1)
    inp = make_inputs(**CW_CASE)
    dv = inp.depth_volume().clone().requires_grad_(True)
    ref, src = inp.ref_feat.clone().requires_grad_(True), inp.nghbr_feat.clone().requires_grad_(True)
    out = refh.est_costvolume_CW(dv, ref, src, inp.ref_gmms, inp.nghbr_gmms, inp.R, inp.t, inp.is_valid,
                                 inp.cam_intrins, inp.thres)
    gout = cw_gout(inp.B, inp.D, CW_CASE["H"], CW_CASE["W"])
    (out * gout).sum().backward()
    np.savez_compressed(os.path.join(HERE, "cw_train.npz"), digest=np.array(input_digest(inp)),
                        kwargs=np.array(repr(CW_CASE)), gout=gout.numpy(),
                        g_ref=ref.grad.numpy(), g_src=src.grad.numpy(), g_depth=dv.grad.numpy())
    print("cw_train written: |g_depth| max", float(dv.grad.abs().max()))


if __name__ == "__main__":
    main()
