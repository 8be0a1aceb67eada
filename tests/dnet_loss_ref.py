"""float64 restatement, with per-element rounding bounds, of D-Net's fused training loss (ops.dnet_loss: the convex
upsampling of the raw [mu, v], activation_G and DnetLoss, upsample_nll_fwd / bwd_kernel<DNET>, DESIGN §3.19), and the
seeded inputs of its tests and golden file.

Conventions as tests/aux_ref.py (its docstring derives the softmax-weight and upsampling bounds reused here): torch
tensors in, float64 out, bounds in units of u = 2^-24, gate |got - ref| <= c u bound with one c.  Per supervised
full-resolution pixel, with the upsampled mu, v and their bounds B_mu, B_v:
    d = mu - gt                          B_d   = B_mu + |d|
    e = elu(v) = v (v > 0) or expm1(v)   elu'  = 1 (v > 0) or e^v
    var = e + 1 + 1e-10                  B_var = max(1, elu') B_v + 2 (|e| + 1)   (expm1f's ulp and the two fp32 adds,
                                                 which round at the size of |e| + 1)
  collapsed, v < -17.5: e^v < 2^-25, expm1f(v) rounds to -1 and var is exactly fp32(1e-10) (B_var = 0).  The clamp
  var[var < 1e-10] = 1e-10 never fires for a non-NaN v (var >= fp32(1e-10), DESIGN §3.19); nothing here models it.
    nll = d^2 / (2 var) + log(var) / 2   B_nll = |d| / var B_d + (d^2 / (2 var^2) + 1 / (2 var)) B_var + d^2 / (2 var)
                                                 + |log var| / 2
    loss bound = [sum (B_nll + 7 |nll|) + 3 |sum nll|] / count + |loss|          (as aux_ref.upsample_nll, one term)
Backward, s = upstream gradient / count:
    g_mu  = s d / var                    E_mu  = s [B_d / var + |d| B_var / var^2 + |d| / var]
    g_var = s (1 / (2 var) - d^2 / (2 var^2))
                                         E_var = s [B_var / (2 var^2) + |d| B_d / var^2 + d^2 B_var / var^3 + 1 / (2 var)
                                                    + d^2 / (2 var^2)]      (the two terms cancel: absolute values)
    g_v   = g_var elu'(v)                E_v   = E_var elu' + |g_var| (elu' (B_v + 2) + TINY/u) + |g_v| + TINY/u
where expf underflows (v < -103) elu' is subnormal or zero and its error absolute: TINY = 2^-126, as the Gaussian
update's bound in aux_ref.  Then t_i = g_v v_i + g_mu mu_i and the scatter into raw exactly as aux_ref.upsample_nll.

A first-order bound needs the perturbation small against the value, and no decision may sit inside its own bound:
``dnet_nll`` reports as ambiguous the pixels where |d| <= c u B_d (the sign of g_mu), |v| <= c u B_v (elu's branch),
|v + 17.5| <= c u B_v (the collapsed regime) or c u B_var > var / 4 (var below fp32's resolution of e^v + 1, i.e.
-17.5 < v < about -10); the tests take them out of the mask.
"""
import numpy as np
import torch

from tests import aux_ref as ar

U, TINY = ar.U, ar.TINY
COLLAPSE = -17.5                                  # below: expm1f(v) == -1 and var == fp32(1e-10)
VAR_MIN = float(np.float32(1e-10))                # activation_G's + 1e-10 and the clamp, both fp32


def _d(x):
    return x.detach().to(torch.float64)


def dnet_nll(raw, mask, gt, gtm, k, c=32.0, grad=1.0):
    """ops.dnet_loss and its gradients at upstream gradient ``grad``.  raw (B, 2, H, W) [mu, v]; mask (B, 9k^2, H, W);
    gt (B, 1, kH, kW); gtm bool.  -> dict: loss, loss_bound, grad_raw, grad_raw_bound, grad_mask, grad_mask_bound,
    ambiguous (B, 1, kH, kW) bool, collapsed (B, 1, kH, kW) bool (v_up < -17.5), var (B, 1, kH, kW)."""
    B, _, H, W = raw.shape
    sel = ar.quarter_res(gtm.to(torch.float64).reshape(B, 1, H * k, W * k), k)[:, 0]      # (B, k, k, H, W)
    gtq = ar.quarter_res(_d(gt), k)[:, 0]
    count = float(sel.sum())
    nq = ar.term_counts(B, H, W, k, gt.device)
    w, wr, nb, mu, v, bmu, bv = ar._upsampled_gaussian(raw, mask, k)
    d = mu - gtq
    bd = bmu + d.abs()
    pos = v > 0
    e = torch.where(pos, v, torch.expm1(v))
    de = torch.where(pos, torch.ones_like(v), torch.exp(v))
    col = v < COLLAPSE
    var = torch.where(col, torch.full_like(v, VAR_MIN), e + 1.0 + VAR_MIN)
    bvar = torch.where(col, torch.zeros_like(v), de.clamp(min=1.0) * bv + 2 * (e.abs() + 1.0))
    amb = (d.abs() <= c * U * bd) | (v.abs() <= c * U * bv) | ((v - COLLAPSE).abs() <= c * U * bv) | \
        (c * U * bvar > var / 4)
    nll = d * d / (2 * var) + 0.5 * torch.log(var)
    bnll = d.abs() / var * bd + (d * d / (2 * var * var) + 1 / (2 * var)) * bvar + d * d / (2 * var) + \
        0.5 * torch.log(var).abs()
    s_nll = float((nll * sel).sum())
    loss = s_nll / count
    loss_b = (float(((bnll + 7 * nll.abs()) * sel).sum()) + 3 * abs(s_nll)) / count + abs(loss)
    s = grad / count
    on = sel > 0
    zero = torch.zeros_like(d)
    g_mu = torch.where(on, s * d / var, zero)
    e_mu = torch.where(on, abs(s) * (bd / var + d.abs() * bvar / var ** 2 + d.abs() / var), zero)
    g_var = s * (1 / (2 * var) - d * d / (2 * var * var))
    e_var = abs(s) * (bvar / (2 * var ** 2) + d.abs() * bd / var ** 2 + d * d * bvar / var ** 3 + 1 / (2 * var)
                      + d * d / (2 * var * var))
    g_v = torch.where(on, g_var * de, zero)
    e_v = torch.where(on, e_var * de + g_var.abs() * (de * (bv + 2) + TINY / U) + g_v.abs() + TINY / U, zero)
    g_mu_, g_v_, e_mu_, e_v_ = (x[:, None] for x in (g_mu, g_v, e_mu, e_v))
    t = g_v_ * nb[:, 1] + g_mu_ * nb[:, 0]
    ta = g_v_.abs() * nb[:, 1].abs() + g_mu_.abs() * nb[:, 0].abs()
    et = e_v_ * nb[:, 1].abs() + e_mu_ * nb[:, 0].abs()
    gm, bm = ar._mask_grad(w, wr, t, ta, et)
    gd, bdp = [], []
    for gg, ee in ((g_mu_, e_mu_), (g_v_, e_v_)):
        gd.append(ar.scatter9((gg * w).sum((2, 3))[:, None])[:, 0])
        bdp.append(ar.scatter9((gg.abs() * wr + ee * w).sum((2, 3))[:, None])[:, 0] + nq[:, 0] *
                   ar.scatter9((gg.abs() * w).sum((2, 3))[:, None])[:, 0] + TINY / U)
    full = lambda a: ar.full_res(a[:, None].to(torch.float64))
    return dict(loss=loss, loss_bound=loss_b, grad_raw=torch.stack(gd, 1), grad_raw_bound=torch.stack(bdp, 1),
                grad_mask=gm.reshape(B, 9 * k * k, H, W), grad_mask_bound=bm.reshape(B, 9 * k * k, H, W),
                ambiguous=full(amb) > 0, collapsed=full(col) > 0, var=full(var))


# ---- seeded inputs -----------------------------------------------------------------------------------------------------

def loss_inputs(B, H, W, k, mask="dense", deep=0, high=0, seed=0):
    """Quarter-resolution raw [mu, v] (mu in [1, 10], v ~ N(0, 1.5^2)), logits N(0, 2^2), gt in [1, 10] and its mask
    ("dense" or "sparse", ~5 %).  ``deep`` 3x3 blocks of v in [-50, -20] around interior centres (their centre's k^2
    upsampled pixels are in the collapsed regime for certain: v_up <= -20) and ``high`` pixels of v in [50, 500] (elu
    is the identity there).  The last pixel is always supervised.  -> raw, logits, gt, gtm (bool), the deep centres'
    full-resolution mask."""
    g = torch.Generator().manual_seed(seed)
    mu = 1.0 + 9.0 * torch.rand(B, 1, H, W, generator=g)
    v = 1.5 * torch.randn(B, 1, H, W, generator=g)
    cen = torch.zeros(B, 1, H, W, dtype=torch.bool)
    for _ in range(deep if H >= 3 and W >= 3 else 0):        # interior centres: no zero-padded tap
        cen[torch.randint(B, (1,), generator=g), 0, torch.randint(1, H - 1, (1,), generator=g),
            torch.randint(1, W - 1, (1,), generator=g)] = True
    block = torch.nn.functional.max_pool2d(cen.float(), 3, 1, 1) > 0
    v = torch.where(block, -20.0 - 30.0 * torch.rand(v.shape, generator=g), v)
    for _ in range(high):
        v[torch.randint(B, (1,), generator=g), 0, torch.randint(H, (1,), generator=g),
          torch.randint(W, (1,), generator=g)] = 50.0 + 450.0 * float(torch.rand(1, generator=g))
    lg = 2.0 * torch.randn(B, 9 * k * k, H, W, generator=g)
    gt = 1.0 + 9.0 * torch.rand(B, 1, H * k, W * k, generator=g)
    if mask == "dense":
        gtm = torch.ones(B, 1, H * k, W * k, dtype=torch.bool)
    else:
        gtm = torch.rand(B, 1, H * k, W * k, generator=g) < 0.05
    deep_full = torch.nn.functional.interpolate(cen.float(), scale_factor=k, mode="nearest") > 0
    gtm |= deep_full
    gtm[-1, 0, -1, -1] = True
    return torch.cat([mu, v], 1).contiguous(), lg.contiguous(), gt, gtm, deep_full


# ---- the golden cases (tests/golden/make_dnet_loss_golden.py -> tests/golden/dnet_loss.npz) --------------------------

GOLDEN = dict(seed=51, B=2, C=256, h=6, w=10)
# Two cases on the same seeded heads and x_feat, apart in the depth head's v gain and in the supervised pixels:
#   ordinary   v gain 8 (raw v roughly +-20), supervised where v_up > -3: moderate negative v (elu on its exp side)
#              and large positive v (v_up >= 20, elu the identity), no collapsed pixel; every pixel carries weight;
#   collapsed  v gain 30 (raw v roughly +-60), supervised outside BAND: collapsed pixels (v_up <= -17.5, var exactly
#              1e-10) next to ordinary and large positive ones; their 1e10-scale gradients dominate the case.
# BAND = (-17.5, -3) is left out of both.  There var = e^v + 1e-10 and one ulp of expm1f (6e-8 absolute near -1)
# moves var by 6e-8 / e^v relative: 1.2e-6 at v = -3, 6e-5 at -10, the whole of var near -17; and nll grows as 1/var,
# so those pixels dominate a loss.  Supervising them would compare the CPU's and CUDA's expm1f, not the kernel.  -3
# keeps one ulp's effect more than 16 times under the 2e-5 of the comparison.
GOLDEN_CASES = {"ordinary": dict(v_gain=8.0), "collapsed": dict(v_gain=30.0)}
BAND = (COLLAPSE, -3.0)
FIRST_IN = 16           # input channels of the two 3x3 convolutions' weight gradients the golden file keeps


def seed_loss_heads(depth_head, mask_head, case):
    """tests.dnet_ref.seed_heads with the golden seed, then the depth head's v row (output channel 1 of its last
    convolution) times the case's v gain."""
    from tests.dnet_ref import seed_heads
    seed_heads(depth_head, mask_head, GOLDEN["seed"])
    with torch.no_grad():
        depth_head[4].weight[1].mul_(GOLDEN_CASES[case]["v_gain"])
        depth_head[4].bias[1].mul_(GOLDEN_CASES[case]["v_gain"])


def golden_mask(case, gtm, v_up):
    """The supervised pixels of a golden case: the seeded ~70 % mask ``gtm`` without BAND, and for the ordinary case
    without anything at or below its upper end."""
    keep = v_up > BAND[1] if case == "ordinary" else ~((v_up > BAND[0]) & (v_up < BAND[1]))
    return gtm & keep


def golden_inputs():
    """Seeded x_feat (B, C, h, w) float32 (ReLU'd), gt (B, 1, 4h, 4w) in [1, 10] and a ~70 % mask before a case's
    pixels are chosen (``golden_mask``)."""
    kw = GOLDEN
    g = torch.Generator().manual_seed(kw["seed"] + 1000)
    x = torch.relu(torch.randn(kw["B"], kw["C"], kw["h"], kw["w"], generator=g))
    gt = 1.0 + 9.0 * torch.rand(kw["B"], 1, 4 * kw["h"], 4 * kw["w"], generator=g)
    gtm = torch.rand(gt.shape, generator=g) < 0.7
    return x, gt, gtm
