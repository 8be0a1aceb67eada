"""float64 restatements, each with a per-element rounding bound, of the fused heads on the tensor cores: the G-Net head
(gnet_head_kernel, DESIGN §3.8), its backward (gnet_bwd_chain_kernel + gnet_wgrad_kernel, §3.10) and the mask head with
the learned upsampling (mask_upsample_kernel, §3.12).  Also the numpy helpers that emulate their arithmetic.

Conventions as tests/aux_ref.py: torch tensors in (any device), float64 out; a bound is in units of u = 2^-24 and is the
same expression evaluated on absolute values; the gate is |got - ref| <= c u bound with one c.  Fixed constants (one
rounding per fp32 operation, expf's ulps) are left to c; what grows with the data or the shape is carried explicitly.

SPLIT16 product term (``split16``).  A GEMM output y = sum_k a_k w_k, with a scaled by the power of two s_a and w by
s_w, split x s = hi + lo (fp16 each), three products hi hi + hi lo + lo hi on mma.sync with fp32 accumulation, exact
descale:
    12 sum |a_k||w_k|         the two split residuals and the dropped lo lo, 3 2^-22 of each product
  + n_mma sum |a_k||w_k|      one fp32 accumulation (not IEEE) per mma.sync the output goes through
  + sum |w_k| / s_a + sum |a_k| / s_w
                              lo rounded to an fp16 subnormal: 2^-25 absolute in scaled units, doubled (2 2^-25 / s =
                              1 u / s) because the kernel takes s from its own fp32 values, which may sit one binade up.
The scales restate split16_shift exactly (largest value into [2^14, 2^15), clamped to +-100, 0 for zero, subnormal or
non-finite maxima): per pixel for the hidden activations (largest ReLU'd value over the 128 channels) and for the
backward gradients (largest |x|), per layer for the weights, and one per call for the cost volume, from the largest
finite |cost| of the whole batch.  So a small image in a batch with a large one gets the large image's scale and a floor
sum |W0| / s_c far above its own signal: that is the design (§3.8), and the bound states it.
MMAs per output: 3 x 9 x ceil(D/16) for the 3x3 conv, 3 x 8 for every 128-deep layer (128 -> 128 forward and backward,
128 -> 144).

Propagation.  Each layer's bound is |W| B_in + its own rounding; ReLU is 1-Lipschitz, so no pixel near a kink is left
out.  The bias add after the exact descale is one fp32 rounding (|W||a| + |b|).  The 128 -> 2 layer is 32 sequential
fp32 FMAs per lane, two quad adds and the bias: 35 (|W3||h2| + |b3|).  The update adds aux_ref.gaussian_update's own
bound to the first-order terms |s0| B_mu1 and elu'(s1) |s0| B_s1.  The mask head's softmax carries
|dw_i| <= w_i (B_l_i + sum_j w_j B_l_j) of the logit bounds B_l on top of aux_ref.convex_upsample's bound.

Backward stages, each from the kernel's own fp32 input to that stage (so a stage's bound is its own rounding only) and
with the ReLU masks of the kernel's saved activations (h > 0, exact: no kink ambiguity):
    d_raw, grad_prev    from the saved raw: aux_ref.gaussian_update's gradient bound; d_s0 = g_mu mu1 + g_sg (elu + 1
                        + 1e-10) with bound |g_mu mu1| + |g_sg| (|elu|~ + 1 + 1e-10)
    d_h2 = W3^T d_raw   two fp32 operations: 2 |W3|^T |d_raw|
    d_h1, d_h0          split16 with per-pixel scales from max |d| and the layer's weight scale, 24 MMAs
    dW = sum_p a_p b_p^T (3xTF32, §3.10): (3 2^-22 + (12 + 32 + n_chunks) 2^-24) sum |a||b| = (24 + 32 + n_chunks) u
                        sum |a||b|, n_chunks = ceil(B H W / 1024); dW0 with b = the zero-padded 3x3 unfold of the cost
    db = sum_p a_p      128 sequential fp32 adds per thread, 3 shuffle adds, n_chunks partials: (131 + n_chunks) sum |a|
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from tests import aux_ref as ar

U = ar.U
HID = 128
KC = 1024                      # pixels per weight-gradient chunk (WG_KC)
MMA_HIDDEN = 3 * 8             # 128-deep layers: 8 K steps x 3 products


def _d(x):
    return x.detach().to(torch.float64)


# ---------------------------------------------------------------------------------------------------------------------
# numpy helpers: the SPLIT16 and 3xTF32 arithmetic of the kernels

def shift(m):
    """split16_shift of one fp32 maximum."""
    m = np.float32(m)
    if m == 0 or not np.isfinite(m) or m < np.finfo(np.float32).tiny:
        return 0
    return int(np.clip(14 - int(np.floor(np.log2(m))), -100, 100))


def split(x, sh):
    """x 2^sh = hi + lo, fp16 each (subnormals as the hardware rounds them), from the fp32 scaled value."""
    xs = (x.astype(np.float32) * np.float32(2.0 ** sh)).astype(np.float32)
    hi = xs.astype(np.float16)
    lo = (xs - hi.astype(np.float32)).astype(np.float16)
    return hi, lo


def tf32(x):
    """cvt.rna.tf32.f32: round to nearest, ties away from zero, to 10 explicit mantissa bits."""
    u = np.asarray(x, np.float32).view(np.uint32).astype(np.uint64)
    r = ((u + 0x1000) & 0xFFFFE000).astype(np.uint32)
    return r.view(np.float32)


def wgrad3(a, b, kc=KC, slab=32, ks=8):
    """out[m][n] = sum_p a[p][m] b[p][n] as the kernel evaluates it: x = hi + lo (tf32 each); per slab of 32 pixels a
    fresh fp32 accumulator takes, per k8 step, the three products lo*hi, hi*lo, hi*hi (each MMA's sum of exact products
    rounded once to fp32) and is added to the CTA's running fp32 sum; the per-chunk (kc pixels) sums are then added
    in order in fp32.  slab = kc is one accumulator per chunk."""
    ah = tf32(a); al = tf32(a - ah)
    bh = tf32(b); bl = tf32(b - bh)
    f = lambda u: u.astype(np.float64)
    P = a.shape[0]
    r32 = lambda x: x.astype(np.float32)
    total = np.zeros((a.shape[1], b.shape[1]), np.float32)
    for c0 in range(0, P, kc):
        tot = np.zeros_like(total)
        for s0 in range(c0, min(P, c0 + kc), slab):
            acc = np.zeros_like(total)
            for k0 in range(s0, min(P, c0 + kc, s0 + slab), ks):
                s = slice(k0, min(P, c0 + kc, k0 + ks))
                for x, y in ((al, bh), (ah, bl), (ah, bh)):
                    acc = r32(f(acc) + f(x[s]).T @ f(y[s]))
            tot = r32(f(tot) + f(acc))
        total = r32(f(total) + f(tot))
    return total


def split16_gemm(a, w, kblocks, row_shift="pixel", drop_lohi=False):
    """y[m][n] = sum_k a[m][k] w[n][k] as mma3 evaluates it: a (M, K) fp32 with a shift per row (``row_shift``:
    "pixel"; "all" for one shift for every row, as the cost volume has; the mutants "row16", one shift per 16 rows
    from the largest of the block, and "g", row g's shift for rows g and g + 8 of every 16), w (N, K) fp32 with one
    shift; per K block of 16 (``kblocks``, in the kernel's order) three MMAs lo_a hi_w, hi_a lo_w, hi_a hi_w, each an
    exact sum of products rounded once to fp32; exact descale.  ``drop_lohi`` leaves out lo_a hi_w.  -> fp32 (M, N)."""
    a = np.asarray(a, np.float32)
    w = np.asarray(w, np.float32)
    amax = np.abs(a).max(1)
    if row_shift == "all":
        amax = np.full_like(amax, amax.max())
    elif row_shift == "row16":
        amax = np.repeat(amax.reshape(-1, 16).max(1), 16)
    elif row_shift == "g":
        amax = np.repeat(amax.reshape(-1, 2, 8)[:, :1], 2, axis=1).reshape(-1)
    sa = np.array([shift(m) for m in amax])
    sw = shift(np.abs(w).max())
    ah, al = split(a, sa[:, None])
    wh, wl = split(w, sw)
    f = lambda u: u.astype(np.float64)
    acc = np.zeros((a.shape[0], w.shape[0]), np.float32)
    prods = ((ah, wl), (ah, wh)) if drop_lohi else ((al, wh), (ah, wl), (ah, wh))
    for kb in kblocks:
        for x, y in prods:
            acc = (f(acc) + f(x[:, kb]) @ f(y[:, kb]).T).astype(np.float32)
    d = np.float32(2.0) ** (-sa[:, None].astype(np.float32))
    return (acc * d * np.float32(2.0 ** -sw)).astype(np.float32)


def ladder(n, parity=0, step=3):
    """Per-pixel scales 2^(-step j) over a 16-pixel row, j = t (or 15 - t for odd ``parity``): 2^0 ... 2^-45, pixels
    g and g + 8 of the MMA fragment 2^-24 apart, the order reversed between neighbouring tiles."""
    t = np.arange(n) % 16
    j = np.where((np.arange(n) // 16 + parity) % 2 == 0, t, 15 - t)
    return 2.0 ** (-step * j)


# ---------------------------------------------------------------------------------------------------------------------
# scales and the SPLIT16 term

def inv_scale(m):
    """1 / 2^split16_shift(m) for a tensor of maxima (their fp32 values); 0 where m is 0 (no split error at all)."""
    m32 = _d(m).to(torch.float32).to(torch.float64)
    _, ex = torch.frexp(m32)
    sh = (15 - ex).clamp(-100, 100)                      # floor(log2 m) = ex - 1
    sh = torch.where((m32 >= 2.0 ** -126) & torch.isfinite(m32), sh, torch.zeros_like(sh))
    return torch.where(m32 == 0, torch.zeros_like(m32), 2.0 ** (-sh.to(torch.float64)))


def finite_absmax(x):
    a = _d(x).abs()
    return a[torch.isfinite(a)].max() if torch.isfinite(a).any() else torch.zeros((), dtype=torch.float64)


def split16(absprod, wsum, ia, asum, iw, n_mma):
    """The SPLIT16 term: (12 + n_mma) sum |a||w| + sum |w| / s_a + sum |a| / s_w (u); ia = 1 / s_a, iw = 1 / s_w."""
    return (12 + n_mma) * absprod + wsum * ia + asum * iw


def _mm(w, x):
    """1x1 layer: (O, C) x (B, C, H, W) -> (B, O, H, W)."""
    return torch.einsum("oc,bchw->bohw", w, x)


def _mat(w):
    return _d(w).reshape(w.shape[0], -1)


def layer(w, b, x, bx, n_mma=MMA_HIDDEN, relu=True):
    """One 1x1 SPLIT16 layer y = W x + b (then ReLU) on x (B, C, H, W) >= 0 with bound bx, per-pixel activation scale
    from max_c x.  -> y, bound."""
    w, x = _mat(w), _d(x)
    aw, ax = w.abs(), x.abs()
    y = _mm(w, x)
    ab = torch.zeros(w.shape[0], dtype=torch.float64, device=w.device) if b is None else _d(b).abs()
    if b is not None:
        y = y + _d(b).view(1, -1, 1, 1)
    absprod = _mm(aw, ax)
    ia = inv_scale(ax.amax(1, keepdim=True))
    iw = inv_scale(aw.max())
    own = split16(absprod, aw.sum(1).view(1, -1, 1, 1), ia, ax.sum(1, keepdim=True), iw, n_mma)
    bound = _mm(aw, _d(bx)) + own + absprod + ab.view(1, -1, 1, 1)
    return (F.relu(y) if relu else y), bound


# ---------------------------------------------------------------------------------------------------------------------
# G-Net head forward

def gnet_forward(cost, inv, ws, prev):
    """cost (B, D, H, W), invariant (B, 128, H, W), ws = (W0[:, :D] (128, D, 3, 3), W1, b1, W2, b2, W3, b3), prev
    (B, 2, H, W) -> dict of h0, h1, h2, raw, out and their bounds (h0_bound, ...)."""
    w0, w1, b1, w2, b2, w3, b3 = ws
    c, w0 = _d(cost), _d(w0)
    D = c.shape[1]
    r = {}
    y0 = F.conv2d(c, w0, padding=1)
    absprod = F.conv2d(c.abs(), w0.abs(), padding=1)
    ic = inv_scale(finite_absmax(c))
    iw0 = inv_scale(w0.abs().max())
    wsum = F.conv2d(torch.ones_like(c), w0.abs(), padding=1)        # in-image taps only: the padding is exact zeros
    asum = F.conv2d(c.abs(), torch.ones(1, D, 3, 3, dtype=torch.float64, device=c.device), padding=1)
    b_pre = split16(absprod, wsum, ic, asum, iw0, 27 * math.ceil(D / 16)) + absprod + _d(inv).abs()
    r["h0"], r["h0_bound"] = F.relu(y0 + _d(inv)), b_pre
    r["h1"], r["h1_bound"] = layer(w1, b1, r["h0"], r["h0_bound"])
    r["h2"], r["h2_bound"] = layer(w2, b2, r["h1"], r["h1_bound"])
    w3m = _mat(w3)
    raw = _mm(w3m, r["h2"]) + _d(b3).view(1, 2, 1, 1)
    r["raw"] = raw
    r["raw_bound"] = _mm(w3m.abs(), r["h2_bound"]) + 35 * (_mm(w3m.abs(), r["h2"]) + _d(b3).abs().view(1, 2, 1, 1))
    out, ob = ar.gaussian_update(raw, prev)
    s0, s1 = _d(prev[:, 1:2]).abs(), raw[:, 1:2]
    delu = torch.where(s1 > 0, torch.ones_like(s1), torch.exp(s1))
    r["out"] = out
    r["out_bound"] = ob + torch.cat([s0 * r["raw_bound"][:, 0:1], delu * s0 * r["raw_bound"][:, 1:2]], 1)
    return r


# ---------------------------------------------------------------------------------------------------------------------
# mask head forward

def mask_forward(pre0, ws, preds, k=4):
    """pre0 (B, 128, H, W) before its ReLU, ws = (W1, b1, W2, b2, W3 (144, 128), b3), preds: list of (B, 2, H, W) ->
    (logits, their bound, [(out, bound) per prediction])."""
    w1, b1, w2, b2, w3, b3 = ws
    h0 = F.relu(_d(pre0))
    h1, bh1 = layer(w1, b1, h0, torch.zeros_like(h0))
    h2, bh2 = layer(w2, b2, h1, bh1)
    lg, blg = layer(w3, b3, h2, bh2, relu=False)
    B, _, H, W = lg.shape
    w, _ = ar.softmax9(lg, k)
    bl = blg.view(B, 9, k, k, H, W)
    dw = w * (bl + (w * bl).sum(1, keepdim=True))
    outs = []
    for p in preds:
        out, bound = ar.convex_upsample(p, lg, k)
        nb = ar.neighbours(p)[:, :, :, None, None].abs()           # (B, 2, 9, 1, 1, H, W)
        outs.append((out, bound + ar.full_res((dw[:, None] * nb).sum(2))))
    return lg, blg, outs


# ---------------------------------------------------------------------------------------------------------------------
# G-Net head backward, stage by stage

def update_bwd(raw, prev, grad_out):
    """From the saved raw (mu1, sigma1): d_raw, its bound, grad_prev, its bound."""
    _, _, d_raw, b_raw = ar.gaussian_update(raw, prev, grad_out)
    mu1, s1 = _d(raw[:, 0:1]), _d(raw[:, 1:2])
    g_mu, g_sg = _d(grad_out[:, 0:1]), _d(grad_out[:, 1:2])
    e = torch.exp(s1)
    neg = s1 <= 0
    elu = torch.where(neg, e - 1.0, s1)
    gp = torch.cat([g_mu, g_mu * mu1 + g_sg * (elu + 1.0 + 1e-10)], 1)
    bp = torch.cat([g_mu.abs(), (g_mu * mu1).abs() + g_sg.abs() * (torch.where(neg, e + 1.0, s1) + 1.0 + 1e-10)], 1)
    return d_raw, b_raw, gp, bp


def w3t(w3, d_raw, h2):
    """d_h2 = (W3^T d_raw) [h2 > 0] from the kernel's d_raw and saved h2 -> value, bound."""
    w = _mat(w3)
    m = (_d(h2) > 0).to(torch.float64)
    return _mm(w.t(), _d(d_raw)) * m, 2 * _mm(w.abs().t(), _d(d_raw).abs()) * m


def grad_layer(w, d, h):
    """(W^T d) [h > 0] on the tensor cores from the kernel's d (B, 128, H, W) and saved h -> value, bound."""
    wt = _mat(w).t()
    d = _d(d)
    m = (_d(h) > 0).to(torch.float64)
    aw, ad = wt.abs(), d.abs()
    ia = inv_scale(ad.amax(1, keepdim=True))
    iw = inv_scale(aw.max())
    bound = split16(_mm(aw, ad), aw.sum(1).view(1, -1, 1, 1), ia, ad.sum(1, keepdim=True), iw, MMA_HIDDEN)
    return _mm(wt, d) * m, bound * m


def n_chunks(B, H, W):
    return -(-B * H * W // KC)


def wgrad(a, b):
    """dW = sum over pixels of a (B, M, H, W) b (B, N, H, W)^T and db = sum a -> dW, its bound, db, its bound."""
    B, _, H, W = a.shape
    n = n_chunks(B, H, W)
    a, b = _d(a), _d(b)
    dw = torch.einsum("bmhw,bnhw->mn", a, b)
    bw = (24 + 32 + n) * torch.einsum("bmhw,bnhw->mn", a.abs(), b.abs())
    return dw, bw, a.sum((0, 2, 3)), (131 + n) * a.abs().sum((0, 2, 3))


def unfold3(cost):
    """(B, D, H, W) -> (B, 9 D, H W): column 9 c + tap holds cost[c] at the pixel's 3x3 neighbour tap (zero outside)."""
    return F.unfold(_d(cost), 3, padding=1)


def wgrad0(grad_inv, cost):
    """dW0[o][c][tap] = sum_p d_h0[p, o] cost[c](p + tap) -> (128, D, 3, 3) value, bound."""
    B, D, H, W = cost.shape
    a = _d(grad_inv).reshape(B, HID, H * W)
    u = unfold3(cost)
    n = n_chunks(B, H, W)
    dw = torch.einsum("bmp,bnp->mn", a, u)
    bw = (24 + 32 + n) * torch.einsum("bmp,bnp->mn", a.abs(), u.abs())
    return dw.view(HID, D, 3, 3), bw.view(HID, D, 3, 3)
