"""Generate tests/golden/dnet_metrics.npz by running the UNMODIFIED reference's D-Net evaluation on the CPU:
    MAGNET_REFERENCE=<path of the checkout> python tests/golden/make_dnet_metrics_golden.py

For every case of tests/dnet_ref.METRIC_CASES the reference's test_DNet.validate (test_DNet.py:22-73) runs with a stub
model that returns the stored [mu, var] map of the image (what DNET(args) returns) and a plain list of batch-1 items as
the loader.  validate() itself copies the prediction to the host, masks it and calls utils.compute_depth_errors with the
variance.  Stored per case: the per-image dicts (validate on a one-image loader; n = the number of pixels
compute_depth_errors received), the running average over all images, and the sha256 of the seeded inputs.  Inputs are
not stored: tests rebuild them from the seed.
"""
import argparse
import os
import sys
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from make_golden import _import_reference  # noqa: E402
from tests.depth_metrics_ref import KEYS, inputs_digest  # noqa: E402
from tests.dnet_ref import METRIC_CASES, metric_inputs  # noqa: E402


class _StubModel:
    """Returns the stored [mu, var] of image i; the image tensor carries i."""

    def __init__(self, pred):
        self.pred = pred

    def __call__(self, img):
        i = int(img.reshape(-1)[0])
        return self.pred[i:i + 1].clone()


def main():
    _import_reference()
    import test_DNet as td
    td.tqdm = lambda it, **kw: it
    counts = []
    original = td.utils.compute_depth_errors

    def counting(gt, pred, var=None):
        counts.append(gt.size)
        return original(gt, pred, var)

    td.utils.compute_depth_errors = counting
    out = {}
    for name, kw in METRIC_CASES.items():
        inp = metric_inputs(name)
        args = argparse.Namespace(dataset_name="nyu" if kw["crop"] is None else "kitti_eigen",
                                  min_depth=kw["min_depth"], max_depth=kw["max_depth"],
                                  garg_crop=kw["crop"] == "garg", eigen_crop=kw["crop"] == "eigen")

        def loader(idx):
            return [{"img": torch.full((1, 3, 4, 4), float(i)), "depth": torch.from_numpy(inp["gt"][i:i + 1]).clone()}
                    for i in idx]

        model = _StubModel(torch.from_numpy(inp["pred"]))
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", RuntimeWarning)     # log of the planted negative / infinite values
            per_image, counts[:] = [], []
            for i in range(kw["n"]):
                d = td.validate(model, args, loader([i]), "cpu")
                per_image.append([float(d[key]) for key in KEYS])
            n = list(counts)
            avg = td.validate(model, args, loader(range(kw["n"])), "cpu")
        out[f"{name}_rows"] = np.array(per_image, dtype=np.float64)
        out[f"{name}_n"] = np.array(n, dtype=np.int64)
        out[f"{name}_avg"] = np.array([float(avg[key]) for key in KEYS], dtype=np.float64)
        out[f"{name}_digest"] = np.array(inputs_digest(inp))
        print(f"{name}: n = {n}, nll per image {out[f'{name}_rows'][:, KEYS.index('nll')]}")
    out["keys"] = np.array(KEYS)
    np.savez_compressed(os.path.join(HERE, "dnet_metrics.npz"), **out)


if __name__ == "__main__":
    main()
