"""Float64 references of the fused mask-head training loss (DESIGN §3.13): autograd of mask_head (after its first
convolution) -> upsample_depth_via_mask -> MagnetLoss 'gaussian' in torch float64; the training forward with a
per-element rounding bound on every output (``train_forward``); and a numpy restatement of the kernels' order of
operations for one full-resolution sub-pixel (the NLL's derivative, the clamp cut and the logits' gradient
d = sum_p w (t_p - <w, t_p>)).

Bounds follow tests/aux_ref.py and tests/head_ref.py (units of u = 2^-24, gate |got - ref| <= c u bound):
    h1, h2, logits    head_ref.layer, SPLIT16, from the exact h0 = ReLU(pre0)
    loss, d_logits,   aux_ref.upsample_nll on the float64 logits, with the logits' bound B_l carried into the softmax
    prediction grads  weights as |dw_i| <= w_i (B_l_i + sum_j w_j B_l_j) on top of their own error; the loss partials
                      are 8 sequential adds per thread, a 5-level shuffle tree and 8 warps in order (19 levels where
                      aux_ref counts 7): 12 sum_p gamma_p / count sum |nll_p| more
    d_h2              SPLIT16 from the kernel's d_logits (144 deep: 9 K steps, 27 MMAs), masked by its saved h2
    d_h1, grad_pre0   head_ref.grad_layer from the kernel's d_h2, d_h1 and saved h1, h0
    dW, db            head_ref.wgrad from the kernel's saved operands, plus the flush of subnormal operands: at input
                      scales where the softmax weights underflow, d_logits holds subnormals, which the tensor cores'
                      3xTF32 products take as zero (|err| <= 2^-126 |other operand| per product):
                      2 TINY/u (sum_p |b_n| + sum_p |a_m|)
An upstream gradient g != 1 multiplies each output once: bound |g| B + |g out|."""
import contextlib

import numpy as np
import torch
import torch.nn.functional as F

from tests import aux_ref as ar
from tests import head_ref as hr


def upsample64(depth, mask, k=4):
    """upsample_depth_via_mask (MAGNET.py:15-27) in float64."""
    N, C, H, W = depth.shape
    m = mask.view(N, 1, 9, k, k, H, W).softmax(2)
    u = F.unfold(depth, 3, padding=1).view(N, C, 9, 1, 1, H, W)
    return (m * u).sum(2).permute(0, 1, 4, 2, 5, 3).reshape(N, C, k * H, k * W)


def loss64(pre0, weights, preds, gt, gt_mask, gamma=0.8):
    """The loss of mask_head_loss in float64: weights = [W1, b1, W2, b2, W3, b3] (any float tensors); returns the loss
    and the bound sum_p gamma_p mean |nll_p| of its rounding."""
    w1, b1, w2, b2, w3, b3 = weights
    h = F.relu(pre0)
    h = F.relu(F.conv2d(h, w1, b1))
    h = F.relu(F.conv2d(h, w2, b2))
    mask = F.conv2d(h, w3, b3)
    sel = gt_mask.bool()
    n = len(preds)
    loss, scale = 0.0, 0.0
    for i, p in enumerate(preds):
        up = upsample64(p, mask)
        mu, sg = up[:, :1][sel], up[:, 1:][sel]
        sq = sg * sg
        var = torch.where(sq < 1e-10, torch.full_like(sq, 1e-10), sq)     # var[var < 1e-10] = 1e-10 (losses.py:45)
        nll = (mu - gt[sel]) ** 2 / (2 * var) + 0.5 * torch.log(var)
        loss = loss + gamma ** (n - i - 1) * nll.mean()
        scale = scale + gamma ** (n - i - 1) * float(nll.detach().abs().mean())
    return loss, scale


def subpixel_grads(logits, taps, valid, gt, scales):
    """The forward kernel's arithmetic at one supervised sub-pixel, in float32 numpy, in its order: softmax of the 9
    logits, per prediction p the convex combination of its taps (9 x [mu, sigma]; invalid taps skipped), the NLL's
    derivative scaled by scales[p], t_i = g_sigma c_i + g_mu a_i, and the logits' gradient summed over the predictions
    in order.  Returns (d_logits (9,), [(g_mu * w, g_sigma * w) per prediction])."""
    f = np.float32
    lg = logits.astype(f)
    e = np.exp(lg - lg.max()).astype(f)
    w = (e * (f(1) / e.sum(dtype=f))).astype(f)
    dl = np.zeros(9, f)
    pgrads = []
    for p, s in enumerate(scales):
        a, c = taps[p][:, 0].astype(f), taps[p][:, 1].astype(f)
        mu = f(sum(w[i] * a[i] for i in range(9) if valid[i]))
        sg = f(sum(w[i] * c[i] for i in range(9) if valid[i]))
        var = max(f(sg * sg), f(1e-10))
        d = f(mu - f(gt))
        g_mu = f(f(s) * d / var)
        g_sg = f(0) if sg * sg < f(1e-10) else f(f(s) * (f(1) / sg - d * d / (var * sg)))
        t = np.array([g_sg * c[i] + g_mu * a[i] if valid[i] else 0 for i in range(9)], f)
        dl = (dl + w * (t - f(np.dot(w, t)))).astype(f)
        pgrads.append((g_mu * w * valid, g_sg * w * valid))
    return dl, pgrads


@contextlib.contextmanager
def _logit_error(blg):
    """aux_ref's softmax weights with the first-order error of logits bounded by blg (B, 144, H, W) added to theirs:
    every bound aux_ref.upsample_nll derives from the weights then carries the logits' rounding."""
    orig = ar.softmax9

    def softmax9(mask, k):
        w, wr = orig(mask, k)
        B, _, H, W = mask.shape
        bl = blg.view(B, 9, k, k, H, W)
        return w, wr + w * (bl + (w * bl).sum(1, keepdim=True))

    ar.softmax9 = softmax9
    try:
        yield
    finally:
        ar.softmax9 = orig


def train_forward(pre0, ws, preds, gt, gtm, gamma=0.8):
    """The training forward in float64 with bounds: ws = (W1, b1, W2, b2, W3, b3).  -> aux_ref.upsample_nll's dict
    (loss, loss_bound, grad_mask = d_logits, grad_preds at unit upstream gradient, their bounds, ambiguous) plus h1,
    h2 and their bounds."""
    w1, b1, w2, b2, w3, b3 = ws
    h0 = F.relu(hr._d(pre0))
    h1, bh1 = hr.layer(w1, b1, h0, torch.zeros_like(h0))
    h2, bh2 = hr.layer(w2, b2, h1, bh1)
    lg, blg = hr.layer(w3, b3, h2, bh2, relu=False)
    with _logit_error(blg):
        r = ar.upsample_nll(preds, lg, gt, gtm, 4, gamma)
    _, absl = loss64(hr._d(pre0), [hr._d(t) for t in ws], [hr._d(p) for p in preds], hr._d(gt),
                     gtm, gamma)
    r["loss_bound"] = r["loss_bound"] + 12 * absl
    r.update(h1=h1, h1_bound=bh1, h2=h2, h2_bound=bh2)
    return r


def logit_grad_layer(w3, d, h2):
    """d_h2 = (W3^T d_logits) [h2 > 0] from the kernel's d_logits (B, 144, H, W) and saved h2: SPLIT16 with 144-deep
    rows (27 MMAs) -> value, bound."""
    wt = hr._mat(w3).t()
    d = hr._d(d)
    m = (hr._d(h2) > 0).to(torch.float64)
    aw, ad = wt.abs(), d.abs()
    ia = hr.inv_scale(ad.amax(1, keepdim=True))
    iw = hr.inv_scale(aw.max())
    bound = hr.split16(hr._mm(aw, ad), aw.sum(1).view(1, -1, 1, 1), ia, ad.sum(1, keepdim=True), iw, 3 * 9)
    return hr._mm(wt, d) * m, bound * m


def scaled(value, bound, g):
    """An output multiplied once by the upstream gradient g (one fp32 rounding)."""
    return g * value, abs(g) * bound + (g * value).abs()


def wgrad(a, b):
    """head_ref.wgrad with the absolute term of subnormal operands flushed by the tensor cores -> dW, bound, db, bound."""
    dw, bw, db, bb = hr.wgrad(a, b)
    sa, sb = hr._d(a).abs().sum((0, 2, 3)), hr._d(b).abs().sum((0, 2, 3))
    return dw, bw + 2 * ar.TINY / ar.U * (sa[:, None] + sb[None, :]), db, bb
