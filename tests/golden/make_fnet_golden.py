"""Generate tests/golden/fnet_train.npz by running the UNMODIFIED reference (a checkout of baegwangbin/MaGNet) on CPU:
    MAGNET_REFERENCE=<path of the checkout> python tests/golden/make_fnet_golden.py

One F-Net training step on the case of tests/fnet_ref.py: est_costvolume_F (homography.py:10-47) -> the loss of
train_FNet.py:88,96-104 -> backward(); stores the loss and the gradients w.r.t. both feature maps, with the ground truth
and the plane depths.  Inputs are rebuilt from the seed (the file carries their sha256, as the files of make_golden.py).
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


def main():
    _import_reference()
    import models.submodules.homography as refh
    from magnet_b200.synthetic import make_inputs
    from tests.fnet_ref import FNET_CASE, FNET_MAX_DEPTH, FNET_MIN_DEPTH, FNET_PLANES, fnet_gt, fnet_l1_loss, sid_centres
    torch.set_num_threads(1)          # the softmax of the F volume reduces in a thread-count dependent order
    inp = make_inputs(**FNET_CASE)
    d_center = sid_centres(FNET_MIN_DEPTH, FNET_MAX_DEPTH, FNET_PLANES)
    gt = fnet_gt(FNET_CASE["B"], FNET_CASE["H"], FNET_CASE["W"])
    ref, src = inp.ref_feat.clone().requires_grad_(True), inp.nghbr_feat.clone().requires_grad_(True)
    vol = refh.est_costvolume_F(d_center, ref, src, inp.R, inp.t, inp.is_valid, inp.cam_intrins)
    loss = fnet_l1_loss(vol, d_center, gt, FNET_MIN_DEPTH, FNET_MAX_DEPTH)
    loss.backward()
    np.savez_compressed(os.path.join(HERE, "fnet_train.npz"), digest=np.array(input_digest(inp)),
                        kwargs=np.array(repr(FNET_CASE)), gt_dmap=gt.numpy(), planes=d_center.numpy().reshape(-1),
                        loss=np.float32(loss.item()), g_ref=ref.grad.numpy(), g_src=src.grad.numpy())
    print("fnet_train written: loss", loss.item())


if __name__ == "__main__":
    main()
