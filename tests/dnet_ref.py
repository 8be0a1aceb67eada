"""float64 restatement, with per-element rounding bounds, of D-Net's fused heads (dnet_depth_kernel and
mask_upsample_kernel<1, true>, DESIGN §3.15): the depth head after its 3x3 convolution, activation_G_magnet, the mask
head with one hidden layer, the learned upsampling of the raw prediction and activation_G.

Conventions as tests/head_ref.py and tests/aux_ref.py: torch tensors in, float64 out, bounds in units of u = 2^-24,
gate |got - ref| <= c u bound with one c.  Built on head_ref.layer (SPLIT16 128 -> 128 / 128 -> 144 layers), G-Net's
128 -> 2 bound (35 (|W2||h1| + |b2|): 32 sequential FMAs, two quad adds, the bias) and aux_ref.convex_upsample's
softmax-weight bound, plus:
  upsampling of a computed raw:  sum_i w_i B_raw_i on top (the raw's own error, carried through the convex weights)
  elu(v) + 1 + 1e-10:            max(1, e^v) B_v (first order; elu' <= max(1, e^v)) + 2 (|elu(v)| + 1) (expm1f's ulp
                                 and the two fp32 adds, which round at the size of |elu| + 1)
  sqrt(var):                     B_var / (2 sqrt(var)) (half the relative bound) + sqrt(var) (sqrtf's rounding)
"""
import hashlib

import numpy as np
import torch

from tests import aux_ref as ar
from tests import head_ref as hr
from tests.depth_metrics_ref import eval_mask, row_from_sums


def _d(x):
    return x.detach().to(torch.float64)


def activation_g(v, bv):
    """var = elu(v) + 1 + 1e-10 and its bound, from v (float64) with bound bv."""
    e = torch.where(v > 0, v, torch.expm1(v))
    de = torch.where(v > 0, torch.ones_like(v), torch.exp(v)).clamp(min=1.0)
    return e + 1.0 + 1e-10, de * bv + 2 * (e.abs() + 1.0)


def depth_forward(pre_d, ws):
    """pre_d (B, 128, H, W) before its ReLU, ws = (W1, b1, W2 (2, 128), b2) -> dict of raw (B, 2, H, W), sigma (the
    second channel after activation_G_magnet) and their bounds."""
    w1, b1, w2, b2 = ws
    h0 = torch.relu(_d(pre_d))
    h1, bh1 = hr.layer(w1, b1, h0, torch.zeros_like(h0))
    w2m = hr._mat(w2)
    raw = hr._mm(w2m, h1) + _d(b2).view(1, 2, 1, 1)
    braw = hr._mm(w2m.abs(), bh1) + 35 * (hr._mm(w2m.abs(), h1) + _d(b2).abs().view(1, 2, 1, 1))
    var, bvar = activation_g(raw[:, 1:2], braw[:, 1:2])
    sg = var.sqrt()
    return {"raw": raw, "raw_bound": braw, "sigma": sg, "sigma_bound": bvar / (2 * sg) + sg}


def upsample_forward(pre_m, ws, raw, raw_bound, k=4):
    """pre_m (B, 128, H, W) before its ReLU, ws = (W1, b1, W3 (144, 128), b3), raw (B, 2, H, W) float64 and its bound
    -> (out (B, 2, kH, kW) [mu, var], its bound)."""
    w1, b1, w3, b3 = ws
    g0 = torch.relu(_d(pre_m))
    g1, bg1 = hr.layer(w1, b1, g0, torch.zeros_like(g0))
    lg, blg = hr.layer(w3, b3, g1, bg1, relu=False)
    B, _, H, W = lg.shape
    w, _ = ar.softmax9(lg, k)
    bl = blg.view(B, 9, k, k, H, W)
    dw = w * (bl + (w * bl).sum(1, keepdim=True))
    up, bup = ar.convex_upsample(raw, lg, k)
    nb = ar.neighbours(raw)[:, :, :, None, None].abs()
    nbb = ar.neighbours(raw_bound)[:, :, :, None, None]
    bup = bup + ar.full_res((dw[:, None] * nb).sum(2)) + ar.full_res((w[:, None] * nbb).sum(2))
    var, bvar = activation_g(up[:, 1:2], bup[:, 1:2])
    return torch.cat([up[:, :1], var], 1), torch.cat([bup[:, :1], bvar], 1)


def ratio(got, want, bound):
    """max |got - want| / (u bound) (the gate is <= 32)."""
    err = (_d(got) - want).abs() / (ar.U * bound)
    return float(err.max())


# ---- seeded heads and inputs of tests/golden/dnet_head.npz (tests/golden/make_dnet_golden.py) ------------------------

HEAD_CASES = {
    # name: seed, B, in_dim, h, w
    "small": dict(seed=31, B=2, C=256, h=6, w=10),
    "odd": dict(seed=32, B=1, C=256, h=5, w=19),
}


def seed_heads(depth_head, mask_head, seed):
    """Overwrite the parameters of the two heads (the reference's Decoder or DnetHead: same names and shapes) with
    seeded values, in state-dict order: weights ~ N(0, 1/fan_in) x 2, biases ~ U(-0.2, 0.2)."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for head in (depth_head, mask_head):
            for name, p in head.named_parameters():
                if name.endswith("weight"):
                    fan = p[0].numel()
                    p.copy_(torch.randn(p.shape, generator=g, dtype=torch.float64).mul(2.0 / fan ** 0.5).to(p.dtype))
                else:
                    p.copy_((torch.rand(p.shape, generator=g, dtype=torch.float64) * 0.4 - 0.2).to(p.dtype))


def head_input(name):
    """Seeded x_feat (B, C, h, w) float32 of a golden case: ReLU'd decoder-like features."""
    kw = HEAD_CASES[name]
    g = torch.Generator().manual_seed(kw["seed"] + 1000)
    return torch.relu(torch.randn(kw["B"], kw["C"], kw["h"], kw["w"], generator=g))


def digest(*arrays) -> str:
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(np.asarray(a)).tobytes())
    return h.hexdigest()


def state_digest(depth_head, mask_head) -> str:
    return digest(*[p.detach().cpu().numpy() for h in (depth_head, mask_head) for _, p in h.named_parameters()])


# ---- the variance form of the depth metrics (test_DNet.py validate(), :22-73) ------------------------------------------

def image_sums_var(gt, mu, var, min_depth, max_depth, crop):
    """The 13 float64 sums of one image as ops.depth_metrics(variance=True) forms them: depth_metrics_ref.image_sums
    with var = channel 1 itself (clamped at 1e-6 on the float32 value), not sigma^2."""
    lo, hi = np.float32(min_depth), np.float32(max_depth)
    gt, mu, var = (np.array(a, dtype=np.float32) for a in (gt, mu, var))
    gt[gt > hi] = 0
    valid = (gt > lo) & (gt < hi) & eval_mask(*gt.shape, crop)
    mu[mu < lo] = lo
    mu[mu > hi] = hi
    mu[np.isinf(mu)] = hi
    mu[np.isnan(mu)] = lo
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


def metric_rows_var(pred, gt, min_depth, max_depth, crop=None):
    """pred (B,2,H,W) [mu, var], gt (B,1,H,W) -> (B,13) float64 rows."""
    pred, gt = np.asarray(pred), np.asarray(gt)
    return np.stack([row_from_sums(image_sums_var(gt[b, 0], pred[b, 0], pred[b, 1], min_depth, max_depth, crop))
                     for b in range(gt.shape[0])])


METRIC_CASES = {
    # name: images (scored one per batch, as test_DNet's loaders), GT size, depth range, crop
    "nyu": dict(seed=41, n=3, H=48, W=64, min_depth=1e-3, max_depth=10.0, crop=None),
    "kitti_garg": dict(seed=42, n=2, H=88, W=304, min_depth=1e-3, max_depth=80.0, crop="garg"),
}


def metric_inputs(name):
    """Seeded [mu, var] predictions (n,2,H,W) and GT (n,1,H,W), numpy float32: GT with holes and values above
    max_depth; predictions around the GT with non-finite and out-of-range mu, variances below 1e-6, zero, negative,
    infinite and NaN."""
    kw = METRIC_CASES[name]
    rng = np.random.default_rng(kw["seed"])
    n, H, W, hi = kw["n"], kw["H"], kw["W"], kw["max_depth"]
    f32 = np.float32
    t = rng.uniform(0.5, 0.9 * hi, (n, 1, H, W))
    gt = (t * np.exp(rng.normal(0.0, 0.1, t.shape))).astype(f32)
    gt[rng.random(gt.shape) < 0.2] = 0
    gt[rng.random(gt.shape) < 0.02] = f32(1.5 * hi)
    mu = t * np.exp(rng.normal(0.0, 0.2, t.shape))
    var = np.exp(rng.normal(-2.0, 2.0, t.shape)) * mu ** 2
    pred = np.concatenate([mu, var], 1).astype(f32)
    sel = rng.random((n, H, W))
    pred[:, 0][sel < 0.01] = np.nan
    pred[:, 0][(sel > 0.01) & (sel < 0.02)] = np.inf
    pred[:, 0][(sel > 0.02) & (sel < 0.03)] = -np.inf
    pred[:, 0][(sel > 0.03) & (sel < 0.05)] = f32(2 * hi)                   # above max_depth
    pred[:, 0][(sel > 0.05) & (sel < 0.07)] = f32(1e-5)                     # below min_depth
    pred[:, 1][(sel > 0.1) & (sel < 0.12)] = f32(3e-7)                      # var clamp
    pred[:, 1][(sel > 0.12) & (sel < 0.13)] = 0.0
    pred[:, 1][(sel > 0.13) & (sel < 0.14)] = f32(-1.0)                     # clamped as well
    pred[n - 1, 1, H // 2, W // 2] = np.inf                                 # nll inf for that image
    if n > 2:
        pred[1, 1, H // 3, W // 3] = np.nan                                 # nll NaN for that image
    return {"pred": pred, "gt": gt}
