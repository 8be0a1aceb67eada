"""Generate tests/golden/dnet_head.npz from the UNMODIFIED reference's D-Net heads on the CPU:
    MAGNET_REFERENCE=<path of the checkout> python tests/golden/make_dnet_golden.py

For every case of tests/dnet_ref.HEAD_CASES the reference's Decoder(2, 4, True, True, dnet) is built (it constructs
offline; only the Encoder needs torch.hub), its depth_head / mask_head get the seeded parameters of
tests.dnet_ref.seed_heads, and on the seeded x_feat it runs
  dnet=True:  depth_head, mask_head, upsample_depth_via_mask, DNET.activation_G       -> (B,2,4h,4w) [mu, var]
  dnet=False: depth_head, DNET.activation_G_magnet                                      -> (B,2,h,w) [mu, sigma]
(the activations called unbound: they do not use self).  Stored: both outputs and the sha256 of the seeded inputs and
parameters; the tests rebuild the inputs from the seed.
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
from tests.dnet_ref import HEAD_CASES, digest, head_input, seed_heads, state_digest  # noqa: E402


def main():
    _import_reference()
    from models.DNET import DNET
    from models.submodules.D_dense_depth import Decoder, upsample_depth_via_mask
    torch.set_num_threads(1)
    out = {}
    for name in HEAD_CASES:
        x = head_input(name)
        with torch.no_grad():
            dec = Decoder(2, 4, True, True, True)
            seed_heads(dec.depth_head, dec.mask_head, HEAD_CASES[name]["seed"])
            depth = dec.depth_head(x)
            up = upsample_depth_via_mask(depth, dec.mask_head(x), 4)
            full = DNET.activation_G(None, up)
            mono, feat = DNET.activation_G_magnet(None, (dec.depth_head(x), x))
        assert feat is x
        out[f"{name}_dnet"] = full.numpy()
        out[f"{name}_magnet"] = mono.numpy()
        out[f"{name}_digest"] = np.array(digest(x.numpy(), state_digest(dec.depth_head, dec.mask_head)))
        print(name, tuple(full.shape), tuple(mono.shape))
    np.savez_compressed(os.path.join(HERE, "dnet_head.npz"), **out)


if __name__ == "__main__":
    main()
