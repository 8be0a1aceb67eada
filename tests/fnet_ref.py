"""F-Net training case shared by tests/golden/make_fnet_golden.py (which freezes the reference's outputs for it in
tests/golden/fnet_train.npz) and the tests: the inputs, and the loss expression of train_FNet.py:95-108 in ATen."""
import numpy as np
import torch
import torch.nn.functional as F

# 80 SID planes from min_depth = 1e-3 (train_scripts/fnet/*.txt), an invalid view, H and W not multiples of 8
FNET_CASE = dict(B=2, V=2, D=8, H=12, W=20, C=64, seed=81, depth="smooth", invalid=[(0, 1)])
FNET_MIN_DEPTH, FNET_MAX_DEPTH, FNET_PLANES = 1e-3, 8.0, 80


def fnet_gt(B, H, W, seed=82):
    """Ground truth at twice the volume's resolution: values above max_depth (zeroed by the loss) and zeros (masked)."""
    rng = np.random.default_rng(seed)
    gt = rng.uniform(0.3, 11.0, (B, 1, 2 * H, 2 * W)).astype(np.float32)
    gt[rng.random(gt.shape) < 0.2] = 0.0
    return torch.from_numpy(gt)


def sid_centres(min_depth, max_depth, n):
    """train_FNet.py:56-66."""
    idx = np.arange(n + 1)
    gamma = 1 - min_depth
    bounds = np.exp(np.log(max_depth + gamma) * idx / n) - gamma
    return torch.from_numpy(((bounds[:-1] + bounds[1:]) / 2).astype(np.float32)).view(1, n, 1, 1)


def fnet_l1_loss(cost_volume, d_center, gt_dmap, min_depth, max_depth):
    """train_FNet.py:88,96-104 verbatim on a probability volume (gt_dmap is not modified)."""
    gt_dmap = gt_dmap.clone()
    gt_dmap[gt_dmap > max_depth] = 0.0
    pred_dmap = torch.sum(cost_volume * d_center, dim=1, keepdim=True)
    gt_dmap = F.interpolate(gt_dmap, size=[pred_dmap.shape[2], pred_dmap.shape[3]], mode='nearest')
    gt_dmap_mask = gt_dmap > min_depth
    l1 = torch.abs(pred_dmap[gt_dmap_mask] - gt_dmap[gt_dmap_mask])
    return torch.mean(l1)
