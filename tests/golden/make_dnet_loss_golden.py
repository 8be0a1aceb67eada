"""Generate tests/golden/dnet_loss.npz from the UNMODIFIED reference's D-Net heads and DnetLoss on the CPU:
    MAGNET_REFERENCE=<path of the checkout> python tests/golden/make_dnet_loss_golden.py

For each case of tests.dnet_loss_ref.GOLDEN_CASES the reference's Decoder(2, 4, True, True, dnet=True) is built (it
constructs offline; only the Encoder needs torch.hub), its depth_head / mask_head get the parameters of
tests.dnet_loss_ref.seed_loss_heads (tests.dnet_ref.seed_heads, then the depth head's v row scaled by the case's gain),
and on the seeded x_feat of tests.dnet_loss_ref.golden_inputs it runs depth_head, mask_head, upsample_depth_via_mask,
DNET.activation_G and DnetLoss (utils/losses.py:13-22) over the case's pixels (dnet_loss_ref.golden_mask), then
autograd.  Stored per case, as <case>_<key>: the loss, the gradient into x_feat and into every head parameter (by
name; of the two 3x3 convolutions' weights only input channels 0..FIRST_IN-1, which keeps the file small: the other
channels are the same computation, and g_x has all of them), the gt mask, how many supervised pixels have v_up <= -17.5,
v_up < 0 and v_up >= 20, and the sha256 of the seeded inputs and parameters; the tests rebuild the inputs from the seed.
"""
import argparse
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from make_golden import _import_reference  # noqa: E402
from tests.dnet_loss_ref import (COLLAPSE, FIRST_IN, GOLDEN_CASES, golden_inputs, golden_mask,  # noqa: E402
                                 seed_loss_heads)
from tests.dnet_ref import digest, state_digest  # noqa: E402


def main():
    _import_reference()
    from models.DNET import DNET
    from models.submodules.D_dense_depth import Decoder, upsample_depth_via_mask
    from utils.losses import DnetLoss
    torch.set_num_threads(1)
    out = {}
    for case in GOLDEN_CASES:
        dec = Decoder(2, 4, True, True, True)
        seed_loss_heads(dec.depth_head, dec.mask_head, case)
        x, gt, gtm = golden_inputs()
        with torch.no_grad():
            v = upsample_depth_via_mask(dec.depth_head(x), dec.mask_head(x), 4)[:, 1:2]
        gtm = golden_mask(case, gtm, v)
        xg = x.clone().requires_grad_()
        pred = DNET.activation_G(None, upsample_depth_via_mask(dec.depth_head(xg), dec.mask_head(xg), 4))
        loss = DnetLoss(argparse.Namespace(loss_fn="gaussian"))(pred, gt, gtm)
        loss.backward()
        c = {"loss": loss.detach().numpy(), "g_x": xg.grad.numpy(), "gt_mask": gtm.numpy(),
             "n_deep": np.array(int((gtm & (v <= COLLAPSE)).sum())), "n_neg": np.array(int((gtm & (v < 0)).sum())),
             "n_high": np.array(int((gtm & (v >= 20)).sum())),
             "digest": np.array(digest(x.numpy(), gt.numpy(), state_digest(dec.depth_head, dec.mask_head)))}
        for prefix, head in (("depth_head", dec.depth_head), ("mask_head", dec.mask_head)):
            for name, p in head.named_parameters():
                c[f"g_{prefix}.{name}"] = p.grad[:, :FIRST_IN].numpy() if name == "0.weight" else p.grad.numpy()
        print(f"{case}: loss {float(loss.detach()):.6g}, supervised {int(gtm.sum())}, v_up <= -17.5: "
              f"{int(c['n_deep'])}, < 0: {int(c['n_neg'])}, >= 20: {int(c['n_high'])}")
        out.update({f"{case}_{k}": a for k, a in c.items()})
    np.savez_compressed(os.path.join(HERE, "dnet_loss.npz"), **out)


if __name__ == "__main__":
    main()
