"""numpy restatement of the depth evaluation of validate() (test_MaGNet.py:52-79, utils/utils.py:106-144) as
ops.depth_metrics computes it (DESIGN §3.6): float32 per-pixel terms in numpy's operation order, float64 sums, every
image of the batch.  Also the seeded inputs of tests/golden/depth_metrics.npz (tests/golden/make_metrics_golden.py).
"""
from __future__ import annotations

import hashlib

import numpy as np

KEYS = ("a1", "a2", "a3", "abs_diff", "abs_rel", "sq_rel", "rmse", "log_10", "irmse", "rmse_log", "silog", "nll")
LOG_KEYS = ("log_10", "rmse_log", "silog", "nll")      # built on logf / log10f, whose last bit differs between libms


def eval_mask(H, W, crop):
    """validate()'s eval_mask, with the reference's own expressions."""
    m = np.zeros((H, W), dtype=bool)
    if crop is None:
        m[:] = True
    elif crop == "garg":
        m[int(0.40810811 * H):int(0.99189189 * H), int(0.03594771 * W):int(0.96405229 * W)] = True
    elif crop == "eigen":
        m[int(0.3324324 * H):int(0.91351351 * H), int(0.0359477 * W):int(0.96405229 * W)] = True
    else:
        raise ValueError(crop)
    return m


def image_sums(gt, mu, sg, min_depth, max_depth, crop):
    """The 13 float64 sums of one (H,W) image: n, the three threshold counts, then the float32 terms of
    compute_depth_errors summed in float64 (the squared log error once: rmse_log and silog share it)."""
    lo, hi = np.float32(min_depth), np.float32(max_depth)          # numpy 2: a Python float next to float32 is float32
    gt, mu, sg = (np.array(a, dtype=np.float32) for a in (gt, mu, sg))
    gt[gt > hi] = 0
    valid = (gt > lo) & (gt < hi) & eval_mask(*gt.shape, crop)
    mu[mu < lo] = lo
    mu[mu > hi] = hi
    mu[np.isinf(mu)] = hi
    mu[np.isnan(mu)] = lo
    var = np.square(sg)
    g, p, v = gt[valid], mu[valid], var[valid]
    v[v < np.float32(1e-6)] = np.float32(1e-6)
    with np.errstate(all="ignore"):
        thresh = np.maximum(g / p, p / g)
        d = g - p
        d2 = d ** 2
        lg, lp = np.log(g), np.log(p)
        terms = [np.ones_like(g), thresh < 1.25, thresh < 1.25 ** 2, thresh < 1.25 ** 3, np.abs(d), np.abs(d) / g,
                 d2 / g, d2, (lg - lp) ** 2, lp - lg, np.abs(np.log10(g) - np.log10(p)), (1 / g - 1 / p) ** 2,
                 0.5 * (np.log(v) + np.log(2 * np.pi) + (np.square(d) / v))]
    return np.array([np.sum(t, dtype=np.float64) for t in terms])


def row_from_sums(S):
    """(13,) sums -> (13,) row: n, then the metrics in KEYS order (NaN when n == 0)."""
    with np.errstate(all="ignore"):
        n = S[0]
        mean = S / n
        return np.array([n, mean[1], mean[2], mean[3], mean[4], mean[5], mean[6], np.sqrt(mean[7]), mean[10],
                         np.sqrt(mean[11]), np.sqrt(mean[8]), np.sqrt(mean[8] - mean[9] ** 2) * 100, mean[12]])


def metric_rows(pred, gt, min_depth, max_depth, crop=None):
    """pred (B,2,H,W) full-resolution [mu, sigma], gt (B,1,H,W) -> (B,13) float64 rows, as ops.depth_metrics."""
    pred, gt = np.asarray(pred), np.asarray(gt)
    return np.stack([row_from_sums(image_sums(gt[b, 0], pred[b, 0], pred[b, 1], min_depth, max_depth, crop))
                     for b in range(gt.shape[0])])


def convex_upsample(depth, logits, k):
    """upsample_depth_via_mask (MAGNET.py:15-27) in float32 numpy: depth (B,C,h,w), logits (B,9k^2,h,w)."""
    B, Cc, h, w = depth.shape
    m = logits.reshape(B, 1, 9, k, k, h, w).astype(np.float32)
    m = np.exp(m - m.max(axis=2, keepdims=True))
    m = m / m.sum(axis=2, keepdims=True)
    pad = np.pad(depth, ((0, 0), (0, 0), (1, 1), (1, 1)))
    nb = np.stack([pad[:, :, i // 3:i // 3 + h, i % 3:i % 3 + w] for i in range(9)], axis=2)   # (B,C,9,h,w)
    up = (m * nb[:, :, :, None, None]).sum(axis=2, dtype=np.float32)                          # (B,C,k,k,h,w)
    return up.transpose(0, 1, 4, 2, 5, 3).reshape(B, Cc, k * h, k * w)


# ---- seeded golden inputs ------------------------------------------------------------------------------------------

CASES = {
    # name: (kwargs); images are scored one per batch, as the reference's test loaders do (batch 1)
    "scannet": dict(seed=71, n=3, H=48, W=64, min_depth=1e-3, max_depth=10.0, crop=None),
    "kitti_garg": dict(seed=72, n=3, H=88, W=304, min_depth=1e-3, max_depth=80.0, crop="garg", nan_sigma=2),
    "kitti_eigen": dict(seed=73, n=3, H=88, W=304, min_depth=1e-3, max_depth=80.0, crop="eigen"),
    "scannet_empty": dict(seed=74, n=2, H=16, W=24, min_depth=1e-3, max_depth=10.0, crop=None, empty=1),
    "scannet_up": dict(seed=75, n=3, H=48, W=64, min_depth=1e-3, max_depth=10.0, crop=None, k=4),
    "kitti_garg_up": dict(seed=76, n=2, H=88, W=304, min_depth=1e-3, max_depth=80.0, crop="garg", k=4),
}


def _special_pixels(gt, mu, sg, rng, lo, hi):
    """Plant the edge cases of validate() at random positions of one full-resolution image."""
    flat_g, flat_m, flat_s = gt.reshape(-1), mu.reshape(-1), sg.reshape(-1)
    idx = rng.permutation(flat_g.size)
    f32 = np.float32
    plants = [
        # (gt, mu, sigma); None keeps the drawn value
        (f32(5.0), f32(4.0), None), (f32(4.0), f32(5.0), None),               # gt/pred == 1.25 exactly
        (f32(6.25), f32(4.0), None), (f32(4.0), f32(6.25), None),             # 1.5625
        (f32(7.8125), f32(4.0), None), (f32(4.0), f32(7.8125), None),         # 1.953125
        (None, f32(np.nan), None), (None, f32(np.inf), None), (None, f32(-np.inf), None),
        (None, f32(lo) * f32(0.1), None), (None, f32(-3.0), None), (None, f32(hi) * f32(2.0), None),
        (None, f32(lo), None), (None, f32(hi), None),
        (None, None, f32(1e-4)), (None, None, f32(0.0)), (None, None, f32(-0.5)), (None, None, f32(9e-4)),
        (f32(hi), None, None), (f32(hi) * f32(1.5), None, None), (np.nextafter(f32(hi), f32(0)), None, None),
        (f32(lo), None, None), (np.nextafter(f32(lo), f32(1)), None, None), (f32(lo) * f32(0.5), None, None),
        (f32(0.0), None, None),
    ]
    reps = max(1, flat_g.size // 400)
    j = 0
    for _ in range(reps):
        for g, m, s in plants:
            p = idx[j]
            j += 1
            if g is not None:
                flat_g[p] = g
            if m is not None:
                flat_m[p] = m
            if s is not None:
                flat_s[p] = s


def case_inputs(name):
    """Seeded inputs of one golden case: dict with gt (n,1,H,W) and either pred (n,2,H,W) or the quarter-resolution
    depth (n,2,H/k,W/k) + logits (n,9k^2,H/k,W/k); numpy float32."""
    kw = CASES[name]
    rng = np.random.default_rng(kw["seed"])
    n, H, W, lo, hi = kw["n"], kw["H"], kw["W"], kw["min_depth"], kw["max_depth"]
    f32 = np.float32
    gt = rng.uniform(0.5, 0.9 * hi, (n, 1, H, W)).astype(f32)
    gt[rng.random(gt.shape) < 0.2] = 0                                       # no GT
    out = {"gt": gt}
    if "k" in kw:
        k = kw["k"]
        h, w = H // k, W // k
        depth = np.empty((n, 2, h, w), dtype=f32)
        depth[:, 0] = rng.uniform(0.5, 0.9 * hi, (n, h, w))
        depth[:, 1] = np.abs(rng.normal(0.0, 0.1 * hi, (n, h, w))) + 1e-3
        sel = rng.random((n, h, w))
        depth[:, 0][sel < 0.03] = f32(lo) * f32(0.1)                          # below min after upsampling too
        depth[:, 0][sel > 0.97] = f32(hi) * f32(1.5)                          # above max
        depth[:, 1][(sel > 0.5) & (sel < 0.52)] = f32(2e-4)                   # var clamp
        out["depth"] = depth
        out["logits"] = (2.0 * rng.standard_normal((n, 9 * k * k, h, w))).astype(f32)
        gt[:, 0, 0, :8] = hi                                                  # GT at max_depth
        gt[:, 0, 1, :8] = 1.5 * hi                                            # GT above it
    else:
        pred = np.empty((n, 2, H, W), dtype=f32)
        pred[:, 0] = gt[:, 0] * np.exp(rng.normal(0.1, 0.3, (n, H, W)))
        pred[:, 0][gt[:, 0] == 0] = rng.uniform(0.5, 0.9 * hi, int((gt[:, 0] == 0).sum()))
        pred[:, 1] = np.abs(rng.normal(0.0, 0.1, (n, H, W))) * pred[:, 0] + 1e-2
        for i in range(n):
            _special_pixels(gt[i, 0], pred[i, 0], pred[i, 1], rng, lo, hi)
        if "nan_sigma" in kw:
            pred[kw["nan_sigma"], 1, int(0.7 * H), W // 2:W // 2 + 5] = np.nan    # NaN sigma: that image's nll is NaN
        if "empty" in kw:
            gt[kw["empty"]] = 0                                               # no valid pixel: NaN metrics
        out["pred"] = pred
    return out


def inputs_digest(inp) -> str:
    h = hashlib.sha256()
    for key in sorted(inp):
        h.update(key.encode())
        h.update(np.ascontiguousarray(inp[key]).tobytes())
    return h.hexdigest()
