"""Generate tests/golden/fnet_metrics.npz by running the UNMODIFIED reference's F-Net evaluation on CPU:
    MAGNET_REFERENCE=<path of the checkout> python tests/golden/make_fnet_metrics_golden.py

For every case of tests/fnet_metrics_ref.CASES the reference's train_FNet.validate (train_FNet.py:165-195) runs with
  - a stub model that returns the stored probability volume of the image: torch.softmax of the seeded scores over the
    planes on the CPU, which is what MAGNET_F.forward returns (homography.py:45-46);
  - a plain list of batch-1 items as the loader;
  - utils.data_preprocess replaced by a stub (poses do not matter here).
validate() itself forms torch.sum(prob * d_center), upsamples it with F.interpolate(mode='nearest') to the image size
and runs the numpy metric block with var=None.  Stored per case: the per-image dicts (validate on a one-image loader;
n = the number of pixels utils.compute_depth_errors received), the running average over all images (validate on the
whole loader), and the sha256 of the seeded inputs.  Inputs are not stored: tests rebuild them from the seed.
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
from tests.depth_metrics_ref import KEYS, inputs_digest  # noqa: E402
from tests.fnet_metrics_ref import CASES, case_inputs  # noqa: E402


class _StubModel:
    """Returns the stored probability volume of image i; the image tensor carries i."""

    def __init__(self, prob):
        self.prob = prob

    def __call__(self, ref_img, nghbr_imgs, nghbr_poses, is_valid, cam_intrins, d_center):
        i = int(ref_img.reshape(-1)[0])
        return self.prob[i:i + 1].clone()


def _stub_preprocess(data_array, cur_batch_size):
    ref = data_array[0]
    return ref, [{"img": ref["img"]}], torch.zeros(cur_batch_size, 1, 4, 4), torch.ones(cur_batch_size, 1)


def main():
    _import_reference()
    import warnings
    import train_FNet as tf
    tf.utils.data_preprocess = _stub_preprocess
    tf.tqdm = lambda it, **kw: it
    counts = []
    original = tf.utils.compute_depth_errors

    def counting(gt, pred, var=None):
        counts.append(gt.size)
        return original(gt, pred, var)

    tf.utils.compute_depth_errors = counting
    torch.set_num_threads(1)          # the CPU softmax and sum reduce in a thread-count dependent order
    out = {}
    for name, kw in CASES.items():
        inp = case_inputs(name)
        prob = torch.softmax(torch.from_numpy(inp["scores"]), dim=1)
        d_center = torch.from_numpy(inp["planes"]).view(1, -1, 1, 1)
        args = argparse.Namespace(dataset_name="scannet" if kw["crop"] is None else "kitti_eigen",
                                  min_depth=kw["min_depth"], max_depth=kw["max_depth"],
                                  garg_crop=kw["crop"] == "garg", eigen_crop=kw["crop"] == "eigen")

        def loader(idx):
            return [([{"img": torch.full((1, 3, kw["H"], kw["W"]), float(i)),
                       "gt_dmap": torch.from_numpy(inp["gt"][i:i + 1]).clone()}], None) for i in idx]

        model = _StubModel(prob)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", RuntimeWarning)     # the empty image's mean of an empty slice
            per_image, counts[:] = [], []
            for i in range(kw["n"]):
                d = tf.validate(model, args, loader([i]), "cpu", d_center)
                per_image.append([float(d[key]) for key in KEYS])
            n = list(counts)
            avg = tf.validate(model, args, loader(range(kw["n"])), "cpu", d_center)
        out[f"{name}_rows"] = np.array(per_image, dtype=np.float64)
        out[f"{name}_n"] = np.array(n, dtype=np.int64)
        out[f"{name}_avg"] = np.array([float(avg[key]) for key in KEYS], dtype=np.float64)
        out[f"{name}_digest"] = np.array(inputs_digest(inp))
        print(f"{name}: n = {n}, rmse per image {out[f'{name}_rows'][:, KEYS.index('rmse')]}")
    out["keys"] = np.array(KEYS)
    np.savez_compressed(os.path.join(HERE, "fnet_metrics.npz"), **out)


if __name__ == "__main__":
    main()
