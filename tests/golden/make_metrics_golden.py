"""Generate tests/golden/depth_metrics.npz by running the UNMODIFIED reference's evaluation on CPU:
    MAGNET_REFERENCE=<path of the checkout> python tests/golden/make_metrics_golden.py

For every case of tests/depth_metrics_ref.CASES the reference's test_MaGNet.validate (test_MaGNet.py:27-81) runs with
  - a stub model that returns the stored prediction of the batch (for the '_up' cases: the reference's
    upsample_depth_via_mask, MAGNET.py:15-27, of the quarter-resolution Gaussians and mask logits);
  - a plain list of batch-1 items as the loader;
  - utils.data_preprocess replaced by a stub (poses do not matter here, and under numpy 2 its np.linalg.inv of a torch
    tensor returns a tensor that torch.from_numpy rejects).
Stored per case: the per-image dicts (validate on a one-image loader; n = the number of pixels
utils.compute_depth_errors received), the running average over all images (validate on the whole loader), and the
sha256 of the seeded inputs.  Inputs are not stored: tests rebuild them from the seed.
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
from tests.depth_metrics_ref import CASES, KEYS, case_inputs, inputs_digest  # noqa: E402


class _StubModel:
    """Returns [stored prediction of image i]; the image tensor carries i."""

    def __init__(self, preds):
        self.preds = preds

    def __call__(self, ref_img, nghbr_imgs, nghbr_poses, is_valid, cam_intrins, mode="test"):
        return [self.preds[int(ref_img.reshape(-1)[0])].clone()]


def _stub_preprocess(data_array, cur_batch_size):
    ref = data_array[0]
    return ref, [{"img": ref["img"]}], torch.zeros(cur_batch_size, 1, 4, 4), torch.ones(cur_batch_size, 1)


def main():
    _import_reference()
    import warnings
    import test_MaGNet as tm
    from models.MAGNET import upsample_depth_via_mask
    tm.utils.data_preprocess = _stub_preprocess
    tm.tqdm = lambda it, **kw: it
    counts = []
    original = tm.utils.compute_depth_errors

    def counting(gt, pred, var=None):
        counts.append(gt.size)
        return original(gt, pred, var)

    tm.utils.compute_depth_errors = counting
    torch.set_num_threads(1)
    out = {}
    for name, kw in CASES.items():
        inp = case_inputs(name)
        if "k" in kw:
            preds = upsample_depth_via_mask(torch.from_numpy(inp["depth"]), torch.from_numpy(inp["logits"]), kw["k"])
        else:
            preds = torch.from_numpy(inp["pred"])
        preds = [preds[i:i + 1].contiguous() for i in range(kw["n"])]
        args = argparse.Namespace(dataset_name="scannet" if kw["crop"] is None else "kitti_eigen",
                                  min_depth=kw["min_depth"], max_depth=kw["max_depth"],
                                  garg_crop=kw["crop"] == "garg", eigen_crop=kw["crop"] == "eigen")

        def loader(idx):
            return [([{"img": torch.full((1, 3, 1, 1), float(i)), "gt_dmap": torch.from_numpy(inp["gt"][i:i + 1]).clone()}],
                     None) for i in idx]

        model = _StubModel(preds)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", RuntimeWarning)     # the empty image's mean of an empty slice
            per_image, counts[:] = [], []
            for i in range(kw["n"]):
                d = tm.validate(model, args, loader([i]), "cpu")
                per_image.append([float(d[key]) for key in KEYS])
            n = list(counts)
            avg = tm.validate(model, args, loader(range(kw["n"])), "cpu")
        out[f"{name}_rows"] = np.array(per_image, dtype=np.float64)
        out[f"{name}_n"] = np.array(n, dtype=np.int64)
        out[f"{name}_avg"] = np.array([float(avg[key]) for key in KEYS], dtype=np.float64)
        out[f"{name}_digest"] = np.array(inputs_digest(inp))
        print(f"{name}: n = {n}, rmse per image {out[f'{name}_rows'][:, KEYS.index('rmse')]}")
    out["keys"] = np.array(KEYS)
    np.savez_compressed(os.path.join(HERE, "depth_metrics.npz"), **out)


if __name__ == "__main__":
    main()
