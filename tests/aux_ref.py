"""float64 restatements, each with a per-element rounding bound, of the small kernels every training step runs around the
cost volumes: convex upsampling (forward, both gradients), the fused upsample + Gaussian NLL (MagnetLoss), the Gaussian
update (forward, backward), the F-Net soft-argmin L1 loss (forward, backward), the relative poses and the camera table.

Every function takes torch tensors (any device) and computes in float64.  A bound is in units of u = 2^-24: the gate is
|got - ref| <= c u bound with one c for every output (tests/test_gpu_aux_f64.py).  A bound is the same expression as the
output evaluated on the absolute value of every factor, times the relative error each factor can carry, plus the
first-order propagation of the rounding of the upstream quantities it is computed from.  Fixed constants of a few u
(expf's 2 ulp, one rounding per operation, the 9-term chains of the upsampling) are left to c; what grows with the data
or the shape is carried explicitly:

Softmax weights (convex upsampling, NLL, F-Net).  The kernels form w_i = expf(l_i - m) / sum_j expf(l_j - m), m = max l.
The difference l_i - m is rounded before expf: an absolute error of u |l_i - m| in the exponent is a relative error of
u |l_i - m| in w_i.  So each weight carries rho_i = |l_i - m| + 1 (in u; the + 1 stands for expf, the sum of 9 and the
division, about 13 u together).  Logits spread over +-60 make this term dominate.  Where expf underflows (l_i - m
< -87) the weight is subnormal or zero and its error is absolute: every w_i rho_i below stands for w_i rho_i + TINY/u,
TINY = 2^-126, and every output bound gets TINY/u more for the subnormal rounding of its last product.

Convex upsampling, CH channels, 3x3 neighbourhood v_i (zero outside the image):
    out        = sum_i w_i v_i                              bound  sum_i w_i |v_i| rho_i
    t_i        = sum_c g_c v_ci,   |t|_i = sum_c |g_c| |v_ci|
    grad_mask  = w_i (t_i - sum_j w_j t_j)                  bound  w_i [rho_i (|t|_i + sum_j w_j |t|_j) + sum_j w_j rho_j |t|_j]
    grad_depth = sum over the (pixel, tap) pairs reading q of g w_i, accumulated with atomicAdd in any order: n_q terms
                 (n_q = k^2 x the in-image neighbours of q, up to 9 k^2), so the sum's own rounding is at most n_q u
                 sum |g| w_i                                bound  sum |g| w_i (rho_i + n_q)
The mask-gradient bound carries w_i (|t|_i + sum_j w_j |t|_j) because t_i - sum_j w_j t_j cancels.

Fused upsample + NLL (ops.magnet_loss; utils/losses.py:34-50).  Per supervised full-resolution pixel, with the upsampled
mu, sigma and their bounds B_mu, B_sg from above:
    d = mu - gt                         B_d   = B_mu + |d|
    var = max(sigma^2, 1e-10)           B_var = 2 |sigma| B_sg + var        (var alone where clamped)
    nll = d^2 / (2 var) + log(var) / 2  B_nll = |d| / var B_d + (d^2 / (2 var^2) + 1 / (2 var)) B_var + d^2 / (2 var) + |log var| / 2
The kernel sums 128 pixels per CTA in a 7-level tree (7 u sum |nll|), the caller adds the partials in float64, rounds to
fp32 and divides by the count; magnet_loss weighs prediction i of n by gamma^(n-i-1) and adds the terms in fp32:
    loss bound = sum_i gamma_i / count [sum (B_nll + 7 |nll|) + 3 |sum nll|] + n |loss|
Backward, s = gamma_i / count:
    g_mu = s d / var                    E_mu = s [B_d / var + 2 |d| B_sg / (var |sigma|) + |d| / var]
    g_sg = s (1/sigma - d^2 / (var sigma)), zero where sigma^2 < 1e-10 (losses.py:45 cuts the gradient there)
                                        E_sg = s [2 |d| B_d / |sigma|^3 + (1 / sigma^2 + 3 d^2 / sigma^4) B_sg
                                                  + 1 / |sigma| + d^2 / |sigma|^3]
(the two terms of g_sg cancel where d^2 ~ sigma^2, so its bound uses their absolute values).  Then t_i = g_sg sigma_i +
g_mu mu_i with E_t_i = |sigma_i| E_sg + |mu_i| E_mu added to the convex-upsampling mask bound above (plus
sum_j w_j E_t_j), and the depth gradients get sum w_i E_mu (resp. E_sg) on top.  The mask gradients of the n
predictions are added by autograd in fp32: (n - 1) sum_i |grad_mask_i| more.
No discrete decision may sit inside its own bound: ``upsample_nll`` reports the pixels where |d| or |sigma^2 - 1e-10| is
within c u of its bound, and the tests take them out of the mask.

Gaussian update (MAGNET.py:60,65-69): mu' = mu0 + mu1 s0, sigma' = (elu(s1) + 1 + 1e-10) s0 with elu = expf(s1) - 1 on
the negative side, which cancels against the + 1:
    mu' bound |mu0| + |mu1 s0|;   sigma' bound (|elu|~ + 1 + 1e-10) |s0|,  |elu|~ = s1 (s1 > 0) or e^s1 + 1
    d_mu1 = g_mu s0 bound |g_mu s0|;  d_s1 = g_sg elu'(s1) s0 bound |g_sg| (elu'(s1) + TINY/u) |s0| + TINY/u |s0|
where expf underflows (s1 < -103) its result and the product are subnormal: TINY = 2^-126 is their absolute error.

F-Net soft-argmin L1 (train_FNet.py:96-108), D planes d_j, p = softmax(s): z and num run sequentially over D, so
    pred = sum_j p_j d_j                E_pred = sum_j p_j |d_j| (rho_j + D) + |pred| (sum_j p_j rho_j + D)
    loss = mean over the mask of |pred - gt|: bound [sum (E_pred + |pred - gt| + 7 |pred - gt|) + 3 |sum|] / count
    grad s_j = p_j (d_j - pred) sign(pred - gt) / count
                                        bound |coef| p_j [(rho_j + D) |d_j - pred| + E_pred]
(d_j - pred cancels: the rounding of pred enters absolutely).  sign(0) = 0: at an exact tie the gradient is exactly zero.

Relative poses (utils/utils.py:72-98): nghbr_pose = ext_nghbr inv(ext_ref).  A condition-number bound is useless at
KITTI translations (|t| ~ 1e3 makes kappa ~ 1e3 while the rotation block stays accurate), so the tolerance is relative
to the reference's own fp32 route (``np.linalg.inv`` of the fp32 matrix, fp32 matmul): per block of the pose (rotation
3x3, translation column, bottom row), the kernel's error may be at most a stated factor times the larger of that route's
error in the block and u max_block (|N| |inv(ext_ref)|).

Camera table (homography.py:98-102): A = K R, a = K t as 3-term fma chains: bound (|K| |R|)_ij and (|K| |t|)_i."""
import numpy as np
import torch
import torch.nn.functional as F

U = 2.0 ** -24
TINY = 2.0 ** -126
NLL_CLAMP = 1e-10


def _d(x):
    return x.detach().to(torch.float64)


# ---------------------------------------------------------------------------------------------------------------------
# convex upsampling

def softmax9(mask, k):
    """(B, 9k^2, H, W) logits -> weights w and the bound of their error w rho + TINY/u (u), both (B, 9, k, k, H, W):
    channel (i k + ky) k + kx holds tap i of sub-pixel (ky, kx) (MAGNET.py:22)."""
    B, _, H, W = mask.shape
    lg = _d(mask).view(B, 9, k, k, H, W)
    w = torch.softmax(lg, 1)
    rho = (lg - lg.max(1, keepdim=True).values).abs() + 1.0
    return w, w * rho + TINY / U


def neighbours(x):
    """(B, C, H, W) -> (B, C, 9, H, W): the zero-padded 3x3 neighbourhood, tap i = 3 (dy + 1) + (dx + 1)."""
    H, W = x.shape[-2:]
    p = F.pad(_d(x), (1, 1, 1, 1))
    return torch.stack([p[..., dy:dy + H, dx:dx + W] for dy in range(3) for dx in range(3)], 2)


def scatter9(c):
    """(B, C, 9, H, W) values at the centre pixel per tap -> (B, C, H, W) summed at the pixel each tap reads."""
    B, C, _, H, W = c.shape
    out = torch.zeros(B, C, H + 2, W + 2, dtype=c.dtype, device=c.device)
    for i in range(9):
        dy, dx = divmod(i, 3)
        out[..., dy:dy + H, dx:dx + W] += c[:, :, i]
    return out[..., 1:H + 1, 1:W + 1]


def full_res(a):
    """(B, C, k, k, H, W) -> (B, C, kH, kW)."""
    B, C, k, _, H, W = a.shape
    return a.permute(0, 1, 4, 2, 5, 3).reshape(B, C, H * k, W * k)


def quarter_res(a, k):
    """(B, C, kH, kW) -> (B, C, k, k, H, W)."""
    B, C, Hk, Wk = a.shape
    return a.reshape(B, C, Hk // k, k, Wk // k, k).permute(0, 1, 3, 5, 2, 4)


def term_counts(B, H, W, k, device):
    """(B, 1, H, W): how many (full-resolution pixel, tap) pairs read each low-resolution pixel."""
    return scatter9(torch.full((B, 1, 9, H, W), float(k * k), dtype=torch.float64, device=device))


def convex_upsample(depth, mask, k):
    """-> out (B, CH, kH, kW), bound."""
    w, wr = softmax9(mask, k)
    nb = neighbours(depth)[:, :, :, None, None]
    out = (w[:, None] * nb).sum(2)
    bound = (wr[:, None] * nb.abs()).sum(2) + TINY / U
    return full_res(out), full_res(bound)


def _mask_grad(w, wr, t, ta, et=None):
    """w (t - sum_j w_j t_j) and its bound; t, ta (= |t|), et (the propagated error of t) shaped like w."""
    dot = (w * t).sum(1, keepdim=True)
    g = w * (t - dot)
    bound = wr * (ta + (w * ta).sum(1, keepdim=True)) + w * (wr * ta).sum(1, keepdim=True) + TINY / U
    if et is not None:
        bound = bound + w * (et + (w * et).sum(1, keepdim=True))
    return g, bound


def convex_upsample_bwd(gout, depth, mask, k):
    """-> grad_depth (B, CH, H, W), its bound, grad_mask (B, 9k^2, H, W), its bound."""
    B, CH, H, W = depth.shape
    w, wr = softmax9(mask, k)
    nb = neighbours(depth)[:, :, :, None, None]             # (B, CH, 9, 1, 1, H, W)
    g = quarter_res(_d(gout), k)[:, :, None]               # (B, CH, 1, k, k, H, W)
    t = (g * nb).sum(1)
    ta = (g.abs() * nb.abs()).sum(1)
    gm, bm = _mask_grad(w, wr, t, ta)
    ga = g.abs()
    gd = scatter9((g * w[:, None]).sum((3, 4)))
    bd = scatter9((ga * wr[:, None]).sum((3, 4))) + term_counts(B, H, W, k, depth.device) * \
        scatter9((ga * w[:, None]).sum((3, 4))) + TINY / U
    return gd, bd, gm.reshape(B, 9 * k * k, H, W), bm.reshape(B, 9 * k * k, H, W)


# ---------------------------------------------------------------------------------------------------------------------
# fused upsample + Gaussian NLL

def _upsampled_gaussian(pred, mask, k):
    """-> w, its error bound (softmax9), neighbours (B, 2, 9, 1, 1, H, W), mu, sigma, B_mu, B_sg (B, k, k, H, W)."""
    w, wr = softmax9(mask, k)
    nb = neighbours(pred)[:, :, :, None, None]
    mu, sg = (w * nb[:, 0]).sum(1), (w * nb[:, 1]).sum(1)
    bmu = (wr * nb[:, 0].abs()).sum(1)
    bsg = (wr * nb[:, 1].abs()).sum(1)
    return w, wr, nb, mu, sg, bmu, bsg


def upsample_nll(preds, mask, gt, gtm, k, gamma=0.8, c=32.0):
    """magnet_loss and its gradients.  preds: list of (B, 2, H, W); mask (B, 9k^2, H, W); gt (B, 1, kH, kW); gtm bool.
    -> dict: loss, loss_bound, grad_preds / grad_preds_bound (lists), grad_mask, grad_mask_bound, ambiguous (B, 1, kH,
    kW) bool: the pixels where d or sigma^2 - 1e-10 lies within c u of its bound, for any prediction."""
    B, _, H, W = preds[0].shape
    n = len(preds)
    sel = quarter_res(gtm.to(torch.float64).reshape(B, 1, H * k, W * k), k)[:, 0]      # (B, k, k, H, W)
    gtq = quarter_res(_d(gt), k)[:, 0]
    count = float(sel.sum())
    nq = term_counts(B, H, W, k, gt.device)
    loss = loss_b = 0.0
    grads, gbounds = [], []
    gmask = torch.zeros(B, 9, k, k, H, W, dtype=torch.float64, device=sel.device)
    gmask_b = torch.zeros_like(gmask)
    gmask_abs = torch.zeros_like(gmask)
    amb = torch.zeros_like(sel, dtype=torch.bool)
    for i, pred in enumerate(preds):
        gam = gamma ** (n - i - 1)
        w, wr, nb, mu, sg, bmu, bsg = _upsampled_gaussian(pred, mask, k)
        d = mu - gtq
        bd = bmu + d.abs()
        clamped = sg * sg < NLL_CLAMP
        var = torch.where(clamped, torch.full_like(sg, NLL_CLAMP), sg * sg)
        bvar = torch.where(clamped, var, 2 * sg.abs() * bsg + var)
        amb |= (d.abs() <= c * U * bd) | ((sg * sg - NLL_CLAMP).abs() <= c * U * (2 * sg.abs() * bsg + sg * sg))
        nll = d * d / (2 * var) + 0.5 * torch.log(var)
        bnll = d.abs() / var * bd + (d * d / (2 * var * var) + 1 / (2 * var)) * bvar + d * d / (2 * var) + \
            0.5 * torch.log(var).abs()
        s_nll = float((nll * sel).sum())
        term = s_nll / count
        loss = loss + gam * term
        loss_b = loss_b + gam / count * (float(((bnll + 7 * nll.abs()) * sel).sum()) + 3 * abs(s_nll))
        # backward of gam * term
        s = gam / count
        sga = sg.abs()
        g_mu = torch.where(sel > 0, s * d / var, torch.zeros_like(d))
        e_mu = s * (bd / var + torch.where(clamped, 0.0, 2 * d.abs() * bsg / (var * sga)) + d.abs() / var)
        g_sg = s * (1 / sg - d * d / (var * sg))
        e_sg = s * (2 * d.abs() * bd / sga ** 3 + (1 / sg ** 2 + 3 * d * d / sg ** 4) * bsg + 1 / sga + d * d / sga ** 3)
        off = clamped | (sel == 0)
        g_sg = torch.where(off, torch.zeros_like(g_sg), g_sg)
        e_sg = torch.where(off, torch.zeros_like(e_sg), e_sg)
        e_mu = torch.where(sel > 0, e_mu, torch.zeros_like(e_mu))
        g_mu_, g_sg_, e_mu_, e_sg_ = (x[:, None] for x in (g_mu, g_sg, e_mu, e_sg))
        t = g_sg_ * nb[:, 1] + g_mu_ * nb[:, 0]
        ta = g_sg_.abs() * nb[:, 1].abs() + g_mu_.abs() * nb[:, 0].abs()
        et = e_sg_ * nb[:, 1].abs() + e_mu_ * nb[:, 0].abs()
        gm, bm = _mask_grad(w, wr, t, ta, et)
        gmask += gm
        gmask_b += bm
        gmask_abs += gm.abs()
        gd, bdp = [], []
        for gg, ee in ((g_mu_, e_mu_), (g_sg_, e_sg_)):
            gd.append(scatter9((gg * w).sum((2, 3))[:, None])[:, 0])
            bdp.append(scatter9((gg.abs() * wr + ee * w).sum((2, 3))[:, None])[:, 0] + nq[:, 0] *
                       scatter9((gg.abs() * w).sum((2, 3))[:, None])[:, 0] + TINY / U)
        grads.append(torch.stack(gd, 1))
        gbounds.append(torch.stack(bdp, 1))
    gmask_b = gmask_b + (n - 1) * gmask_abs
    return dict(loss=loss, loss_bound=loss_b + n * abs(loss), grad_preds=grads, grad_preds_bound=gbounds,
                grad_mask=gmask.reshape(B, 9 * k * k, H, W), grad_mask_bound=gmask_b.reshape(B, 9 * k * k, H, W),
                ambiguous=full_res(amb[:, None].to(torch.float64)) > 0)


# ---------------------------------------------------------------------------------------------------------------------
# Gaussian update

def gaussian_update(dout, gmm0, gout=None):
    """-> out (B, 2, H, W), bound[, grad_dout, bound]."""
    mu1, s1 = _d(dout[:, 0:1]), _d(dout[:, 1:2])
    mu0, s0 = _d(gmm0[:, 0:1]), _d(gmm0[:, 1:2])
    e = torch.exp(s1)
    neg = s1 <= 0
    elu = torch.where(neg, e - 1.0, s1)
    out = torch.cat([mu0 + mu1 * s0, (elu + 1.0 + 1e-10) * s0], 1)
    bound = torch.cat([mu0.abs() + (mu1 * s0).abs(), (torch.where(neg, e + 1.0, s1) + 1.0 + 1e-10) * s0.abs()], 1)
    if gout is None:
        return out, bound
    g_mu, g_sg = _d(gout[:, 0:1]), _d(gout[:, 1:2])
    delu = torch.where(neg, e, torch.ones_like(e))
    grad = torch.cat([g_mu * s0, g_sg * delu * s0], 1)
    gbound = torch.cat([(g_mu * s0).abs(), (g_sg.abs() * (delu + TINY / U) + TINY / U) * s0.abs()], 1)
    return out, bound, grad, gbound


# ---------------------------------------------------------------------------------------------------------------------
# F-Net soft-argmin L1

def fnet_l1(scores, planes, gt, mask, c=32.0):
    """scores (B, D, H, W), planes (D,) (their fp32 values), gt (B, 1, H, W), mask bool (B, 1, H, W) -> dict: loss,
    loss_bound, grad (B, D, H, W), grad_bound, ambiguous (B, 1, H, W): supervised pixels whose |pred - gt| is within
    c u of the rounding bound of pred (the sign of the gradient is then not determined)."""
    s = _d(scores)
    D = s.shape[1]
    dj = _d(torch.as_tensor(planes, dtype=torch.float32)).to(s.device).view(1, D, 1, 1)
    g = _d(gt)
    sel = mask.to(torch.float64)
    count = float(sel.sum())
    p = torch.softmax(s, 1)
    rho = (s - s.max(1, keepdim=True).values).abs() + 1.0
    pred = (p * dj).sum(1, keepdim=True)
    e_pred = (p * dj.abs() * (rho + D)).sum(1, keepdim=True) + pred.abs() * ((p * rho).sum(1, keepdim=True) + D)
    l1 = (pred - g).abs() * sel
    s_l1 = float(l1.sum())
    loss = s_l1 / count
    loss_b = (float((e_pred * sel).sum()) + 8 * s_l1 + 3 * s_l1) / count
    coef = torch.sign(pred - g) * sel / count
    grad = p * (dj - pred) * coef
    gbound = coef.abs() * ((p * (rho + D) + TINY / U) * (dj - pred).abs() + p * e_pred + TINY / U)
    amb = (sel > 0) & ((pred - g).abs() <= c * U * e_pred) & (pred != g)
    return dict(loss=loss, loss_bound=loss_b + abs(loss), grad=grad, grad_bound=gbound, pred=pred, ambiguous=amb)


# ---------------------------------------------------------------------------------------------------------------------
# camera preparation

def relative_poses(ext_ref, ext_nghbr):
    """float64 numpy: ext_ref (B, 4, 4), ext_nghbr (V, B, 4, 4) -> poses (B, V, 4, 4) = ext_nghbr inv(ext_ref) and
    the abs-value product |ext_nghbr| |inv(ext_ref)| (NaN where an input has a NaN)."""
    er = np.asarray(ext_ref, np.float64)
    en = np.asarray(ext_nghbr, np.float64)
    V, B = en.shape[:2]
    poses = np.full((B, V, 4, 4), np.nan)
    absprod = np.full((B, V, 4, 4), np.nan)
    for b in range(B):
        if np.isnan(er[b]).any():
            continue
        inv = np.linalg.inv(er[b])
        for v in range(V):
            poses[b, v] = en[v, b] @ inv
            absprod[b, v] = np.abs(en[v, b]) @ np.abs(inv)
    return poses, absprod


POSE_BLOCKS = ((slice(0, 3), slice(0, 3)), (slice(0, 3), slice(3, 4)), (slice(3, 4), slice(0, 4)))


def pose_tolerance(want, ref32, absprod, factor):
    """Per (b, v) and block of the pose (rotation, translation, bottom row): factor x max(the fp32 route's largest error
    in the block, u x the block's largest |N| |inv|).  Arrays (B, V, 4, 4); -> tolerance of the same shape."""
    tol = np.zeros_like(want)
    err32 = np.abs(ref32.astype(np.float64) - want)
    for rs, cs in POSE_BLOCKS:
        e = np.max(err32[:, :, rs, cs], axis=(2, 3))
        a = U * np.max(absprod[:, :, rs, cs], axis=(2, 3))
        tol[:, :, rs, cs] = factor * np.maximum(e, a)[:, :, None, None]
    return tol


def pack_cameras(intM, R, t, valid):
    """float64 numpy (B, 3, 3), (B, V, 3, 3), (B, V, 3), (B, V) -> camera table (B V, 16) and its bound (u)."""
    K, R, t = (np.asarray(x, np.float64) for x in (intM, R, t))
    B, V = R.shape[:2]
    cams = np.zeros((B * V, 16))
    bound = np.zeros((B * V, 16))
    cams[:, 0] = (np.asarray(valid).reshape(-1) == 1).astype(np.float64)
    cams[:, 1:4] = np.einsum("bij,bvj->bvi", K, t).reshape(B * V, 3)
    cams[:, 4:13] = np.einsum("bij,bvjk->bvik", K, R).reshape(B * V, 9)
    bound[:, 1:4] = np.einsum("bij,bvj->bvi", np.abs(K), np.abs(t)).reshape(B * V, 3)
    bound[:, 4:13] = np.einsum("bij,bvjk->bvik", np.abs(K), np.abs(R)).reshape(B * V, 9)
    return cams, bound


def gj_inverse_f32(a):
    """relative_poses_kernel's 4x4 Gauss-Jordan inverse with partial pivoting (the first row of largest |a_rc|),
    emulated in fp32 (an fma rounded once through float64)."""
    m = np.concatenate([np.asarray(a, np.float32), np.eye(4, dtype=np.float32)], 1)
    for c in range(4):
        piv = c + int(np.argmax(np.abs(m[c:, c])))
        m[[c, piv]] = m[[piv, c]]
        m[c] = m[c] * (np.float32(1.0) / m[c, c])
        for r in range(4):
            if r != c:
                m[r] = (-np.float64(m[r, c]) * m[c].astype(np.float64) + m[r]).astype(np.float32)
    return m[:, 4:]


def sample_depths_f32(gmm, k):
    """MAGNET.py:155 in fp32, operation by operation: mu + (sigma * k_j), both rounded (never an fma)."""
    g = np.asarray(gmm, np.float32)
    kk = np.asarray(k, np.float32).reshape(1, -1, 1, 1)
    return (g[:, 0:1] + (g[:, 1:2] * kk).astype(np.float32)).astype(np.float32)


# ---------------------------------------------------------------------------------------------------------------------
# inputs shared by tests/test_aux_ref_cpu.py and tests/test_gpu_aux_f64.py (CPU float32 tensors)

def upsample_inputs(B, H, W, k, CH=2, n=1, spread=None, mask="dense", tiny=0, neg=False, empty=False, seed=0):
    """Quarter-resolution predictions (n of them, (B, CH, H, W): mu in [1, 10], sigma in [0.05, 2], the last image's
    sigma negated when ``neg``, a 3x3 block of sigma = 1e-7 around ``tiny`` random centres so that their k^2 upsampled
    pixels are clamped for certain), logits N(0, 2^2) or U(-spread, spread), gt in [1, 10] and its mask: "dense",
    "sparse" (~5 %, KITTI-like) or "last" (only the last 128-pixel CTA of every full-resolution row); ``empty`` leaves
    image 0 without a supervised pixel.  -> preds, mask, gt, gtm (bool), the clamped centres' mask (B, 1, kH, kW)."""
    g = torch.Generator().manual_seed(seed)
    preds = []
    cen = torch.zeros(B, 1, H, W, dtype=torch.bool)
    for _ in range(tiny):                  # never in the image ``empty`` leaves unsupervised
        cen[torch.randint(int(empty), B, (1,), generator=g), 0, torch.randint(H, (1,), generator=g),
            torch.randint(W, (1,), generator=g)] = True
    block = F.max_pool2d(cen.float(), 3, 1, 1) > 0
    for _ in range(n):
        mu = 1.0 + 9.0 * torch.rand(B, 1, H, W, generator=g)
        sg = 0.05 + 1.95 * torch.rand(B, CH - 1, H, W, generator=g)
        if neg:
            sg[-1] = -sg[-1]
        if CH == 2:
            sg = torch.where(block, torch.full_like(sg, 1e-7), sg)
        preds.append(torch.cat([mu, sg], 1)[:, :CH].contiguous())
    if spread is None:
        lg = 2.0 * torch.randn(B, 9 * k * k, H, W, generator=g)
    else:
        lg = spread * (2.0 * torch.rand(B, 9 * k * k, H, W, generator=g) - 1.0)
    gt = 1.0 + 9.0 * torch.rand(B, 1, H * k, W * k, generator=g)
    if mask == "dense":
        gtm = torch.ones(B, 1, H * k, W * k, dtype=torch.bool)
    elif mask == "sparse":
        gtm = torch.rand(B, 1, H * k, W * k, generator=g) < 0.05
    else:
        gtm = torch.zeros(B, 1, H * k, W * k, dtype=torch.bool)
        gtm[..., 128 * ((W * k - 1) // 128):] = True
    clamped = F.interpolate(cen.float(), scale_factor=k, mode="nearest") > 0
    gtm |= clamped
    if empty:
        gtm[0] = False
        clamped[0] = False
    gtm[-1, 0, -1, -1] = True
    return preds, lg.contiguous(), gt, gtm, clamped


def fnet_inputs(B, D, H, W, scale, seed=0):
    """Scores N(0, scale^2), sorted plane depths in [0.5, 10] (fp32), gt in [0.5, 10], a ~80 % mask."""
    g = torch.Generator().manual_seed(seed)
    scores = scale * torch.randn(B, D, H, W, generator=g)
    planes = torch.sort(0.5 + 9.5 * torch.rand(D, generator=g)).values
    gt = 0.5 + 9.5 * torch.rand(B, 1, H, W, generator=g)
    mask = torch.rand(B, 1, H, W, generator=g) < 0.8
    mask[0, 0, 0, 0] = True
    return scores, planes, gt, mask


def rigid(R, t):
    e = np.eye(4)
    e[:3, :3], e[:3, 3] = R, t
    return e


def axis_turns():
    """The 90, 180 and 270 degree turns about x, y and z: rotations with zero diagonal entries, where the inverse needs
    its pivot search."""
    out = []
    for ax in range(3):
        for q in (1, 2, 3):
            c, s = [1.0, 0.0, -1.0, 0.0][q], [0.0, 1.0, 0.0, -1.0][q]
            i, j = [(1, 2), (0, 2), (0, 1)][ax]
            R = np.eye(3)
            R[i, i], R[i, j], R[j, i], R[j, j] = c, -s, s, c
            out.append(R)
    return out


def pose_inputs(B, V, tmax, seed=0, nan_ref=(), nan_nghbr=()):
    """ext_ref (B, 4, 4), ext_nghbr (V, B, 4, 4) fp32 world-to-camera extrinsics: random rotations and the axis turns,
    translations up to ``tmax``; NaN in ext_ref[b] for b in nan_ref and in ext_nghbr[v, b] for (v, b) in nan_nghbr."""
    from scipy.spatial.transform import Rotation
    rng = np.random.default_rng(seed)
    turns = axis_turns()
    rots = list(Rotation.random(B * (V + 1), random_state=seed).as_matrix())
    mats = []
    for i in range(B * (V + 1)):
        R = turns[i % len(turns)] if i % 2 == 0 else rots[i]
        if i % 6 == 3:
            R = turns[(i // 6) % len(turns)] @ rots[i]
        mats.append(rigid(R, rng.uniform(-tmax, tmax, 3)))
    ext_ref = np.stack(mats[:B]).astype(np.float32)
    ext_nghbr = np.stack(mats[B:]).reshape(V, B, 4, 4).astype(np.float32)
    for b in nan_ref:
        ext_ref[b, 1, 2] = np.nan
    for v, b in nan_nghbr:
        ext_nghbr[v, b, 0, 3] = np.nan
    return ext_ref, ext_nghbr
