"""numpy restatement of F-Net's evaluation (train_FNet.py validate(), :165-193) as ops.plane_depth +
ops.depth_metrics(nearest=True) compute it (DESIGN §3.14): the soft-argmin depth in float64, ATen's nearest source
index, and the metric rows of tests/depth_metrics_ref.py with nll = 0.0 (compute_depth_errors(..., var=None)).  Also
the seeded inputs of tests/golden/fnet_metrics.npz (tests/golden/make_fnet_metrics_golden.py) and the comparison of
rows whose predictions differ by at most the soft-argmin bound.
"""
from __future__ import annotations

import numpy as np

from tests.depth_metrics_ref import KEYS, eval_mask, image_sums, row_from_sums
from tests.fnet_ref import sid_centres

NLL = KEYS.index("nll")
THRESHOLDS = (1.25, 1.25 ** 2, 1.25 ** 3)


def soft_argmin64(volume, planes, scores: bool):
    """(B,D,h,w) volume -> (B,1,h,w) float64 sum_j prob_j d_j; ``scores``: softmax over the planes first, in float64.
    A row with a NaN or an infinite maximum gives NaN, as torch.softmax."""
    v = np.asarray(volume, dtype=np.float64)
    d = np.asarray(planes, dtype=np.float64).reshape(1, -1, 1, 1)
    with np.errstate(all="ignore"):
        if scores:
            e = np.exp(v - v.max(axis=1, keepdims=True))
            v = e / e.sum(axis=1, keepdims=True)
        return (v * d).sum(axis=1, keepdims=True)


def soft_argmin_bound(planes) -> float:
    """How far the float32 soft-argmin of D planes may lie from the float64 one: (D + 8) 2^-24 max_j |d_j|."""
    planes = np.asarray(planes, dtype=np.float64).reshape(-1)
    return (planes.size + 8) * 2.0 ** -24 * float(np.abs(planes).max())


def nearest_index(out_size: int, in_size: int):
    """ATen's nearest source index for F.interpolate(size=...): min(floor(i * s), in - 1) with s = (float)in / out
    rounded to float32 and the product in float32."""
    s = np.float32(in_size) / np.float32(out_size)
    i = np.arange(out_size, dtype=np.float32)
    return np.minimum(np.floor(i * s).astype(np.int64), in_size - 1)


def nearest_upsample(pred, H: int, W: int):
    """(B,C,h,w) -> (B,C,H,W), F.interpolate(..., size=(H, W), mode='nearest')."""
    pred = np.asarray(pred)
    return pred[:, :, nearest_index(H, pred.shape[2])][:, :, :, nearest_index(W, pred.shape[3])]


def metric_rows_nearest(pred, gt, min_depth, max_depth, crop=None):
    """pred (B,1,h,w) float32 depth maps, gt (B,1,H,W) -> (B,13) float64 rows as ops.depth_metrics(nearest=True):
    float32 terms, float64 sums, nll 0.0."""
    gt = np.asarray(gt)
    full = nearest_upsample(np.asarray(pred, dtype=np.float32), gt.shape[2], gt.shape[3])
    rows = np.stack([row_from_sums(image_sums(gt[b, 0], full[b, 0], np.ones_like(full[b, 0]), min_depth, max_depth,
                                              crop)) for b in range(gt.shape[0])])
    rows[:, 1 + NLL] = 0.0
    return rows


def threshold_allowance(p64, gt, min_depth, max_depth, crop, bound):
    """(B,3) numbers of valid pixels whose ratio max(gt/p, p/gt) can cross 1.25, 1.25^2, 1.25^3 when the prediction
    moves by up to ``bound`` from its float64 value p64 (B,1,h,w): the only pixels a1-a3 may count differently."""
    gt = np.asarray(gt, dtype=np.float32)
    H, W = gt.shape[2:]
    full = nearest_upsample(p64, H, W)
    lo32, hi32 = np.float32(min_depth), np.float32(max_depth)
    out = []
    for b in range(gt.shape[0]):
        g = gt[b, 0].copy()
        g[g > hi32] = 0
        valid = (g > lo32) & (g < hi32) & eval_mask(H, W, crop)
        gv, p = g[valid].astype(np.float64), full[b, 0][valid]
        finite = np.isfinite(p)                                  # NaN becomes min_depth exactly on both sides
        pl, ph = np.clip(p - bound, min_depth, max_depth), np.clip(p + bound, min_depth, max_depth)
        with np.errstate(all="ignore"):
            r_lo, r_hi = np.maximum(gv / pl, pl / gv), np.maximum(gv / ph, ph / gv)
        r_max = np.maximum(r_lo, r_hi)
        r_min = np.where((gv >= pl) & (gv <= ph), 1.0, np.minimum(r_lo, r_hi))
        out.append([int((finite & (r_min <= t * (1 + 1e-6)) & (r_max >= t * (1 - 1e-6))).sum()) for t in THRESHOLDS])
    return np.array(out)


def assert_rows_match(rows, want_n, want, allowance, rtol=1e-4):
    """rows (B,13) as ops.depth_metrics(nearest=True) returns them, against (B,) counts and (B,12) metrics in KEYS
    order computed from predictions within the soft-argmin bound: n exact; a1-a3 off by at most ``allowance`` (B,3)
    pixels; nll exactly 0.0; the rest within rtol (NaN where NaN)."""
    rows, want = np.asarray(rows), np.asarray(want)
    np.testing.assert_array_equal(rows[:, 0], want_n)
    n = np.maximum(rows[:, :1], 1)
    off = np.abs(rows[:, 1:4] - want[:, :3]) * n
    assert (np.nan_to_num(off, nan=0.0) <= allowance + 1e-6 * n).all(), (off, allowance)
    np.testing.assert_array_equal(np.isnan(rows[:, 1:4]), np.isnan(want[:, :3]))
    assert (rows[:, 1 + NLL] == 0.0).all() and (want[:, NLL] == 0.0).all()
    np.testing.assert_allclose(rows[:, 4:1 + NLL], want[:, 3:NLL], rtol=rtol, atol=0, equal_nan=True)


# ---- seeded golden inputs ------------------------------------------------------------------------------------------

PLANES = 80
CASES = {
    # name: kwargs; h x w is the volume's grid, H x W the GT's; images are scored one per batch (batch-1 loaders)
    "scannet": dict(seed=91, n=3, h=12, w=16, H=48, W=64, min_depth=1e-3, max_depth=10.0, crop=None),
    "kitti_garg": dict(seed=92, n=2, h=22, w=76, H=88, W=304, min_depth=1e-3, max_depth=80.0, crop="garg"),
    "kitti_eigen": dict(seed=93, n=2, h=22, w=76, H=88, W=304, min_depth=1e-3, max_depth=80.0, crop="eigen"),
    "ratio": dict(seed=94, n=2, h=15, w=20, H=50, W=70, min_depth=1e-3, max_depth=10.0, crop=None),
    "empty": dict(seed=95, n=2, h=12, w=16, H=48, W=64, min_depth=1e-3, max_depth=10.0, crop=None, empty=1),
}


def case_planes(name):
    kw = CASES[name]
    return sid_centres(kw["min_depth"], kw["max_depth"], PLANES).numpy().reshape(-1)


def case_inputs(name):
    """Seeded inputs of one golden case: scores (n,80,h,w) peaked near a per-pixel depth, GT (n,1,H,W) scattered
    around the same depth (zeros, values above max_depth), planted rows; numpy float32.  The probability volume the
    reference's validate() sees is torch.softmax(scores, 1) on the CPU."""
    kw = CASES[name]
    rng = np.random.default_rng(kw["seed"])
    n, h, w, H, W, hi = kw["n"], kw["h"], kw["w"], kw["H"], kw["W"], kw["max_depth"]
    f32 = np.float32
    planes = case_planes(name)
    t = rng.uniform(0.5, 0.9 * hi, (n, h, w))
    scores = -0.5 * ((np.log(planes)[None, :, None, None] - np.log(t)[:, None]) / 0.3) ** 2
    scores = (scores + rng.normal(0.0, 1.5, scores.shape)).astype(f32)
    gt = (nearest_upsample(t[:, None], H, W) * np.exp(rng.normal(0.0, 0.25, (n, 1, H, W)))).astype(f32)
    gt[rng.random(gt.shape) < 0.2] = 0                                       # no GT
    gt[rng.random(gt.shape) < 0.02] = f32(1.5 * hi)                          # above max_depth
    for i in range(n):                                                       # planted rows
        ys, xs = rng.integers(0, h, 4), rng.integers(0, w, 4)
        scores[i, :, ys[0], xs[0]] = -np.inf                                 # NaN prediction -> min_depth
        scores[i, rng.integers(0, PLANES), ys[1], xs[1]] = np.inf            # NaN as well
        scores[i, rng.integers(0, PLANES), ys[2], xs[2]] = np.nan
        scores[i, PLANES // 2, ys[3], xs[3]] = f32(1e4)                      # one plane takes all the mass
    if "empty" in kw:
        gt[kw["empty"]] = 0                                                  # no valid pixel: NaN metrics, nll 0.0
    return {"scores": scores, "gt": gt, "planes": planes}

