"""CPU oracle for MaGNet's multi-view matching hot path — TEST INFRASTRUCTURE ONLY.

This module is the checker, never the product: only ``tests/``,
``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline leg may import it.
``magnet_b200`` never imports anything under ``oracle/``.

It is an independent numpy restatement (no torch ops) of the reference algorithm,
element by element in the reference's fp32 operation order (SURVEY Appendix A.2):

  * sampler ............ models/MAGNET.py:154-156
  * cost volume (CW) ... models/submodules/homography.py:79-161
  * bilinear sampling .. torch ``F.grid_sample(mode='bilinear', padding_mode='zeros',
                         align_corners=False)`` as called at homography.py:70,150-152;
                         semantics from ATen/native/GridSampler.h (grid_sampler_unnormalize,
                         within_bounds_2d) of torch 2.11 — third-party dependency of the
                         reference (requirements.txt:1 pins torch==1.6.0; the bilinear /
                         zeros / align_corners=False semantics are identical in both)
  * cost volume (F) .... models/submodules/homography.py:10-75
  * Gaussian update .... models/MAGNET.py:58-70  (+ analytic backward)
  * convex upsampling .. models/MAGNET.py:15-27
  * offsets k_j ........ models/MAGNET.py:120-128 (via magnet_b200.sampling, same formula)

PIN STATUS: the reference ships no tests, golden vectors or fixtures for this path
(SURVEY §4, §8c).  The pin is therefore (i) outputs of the reference's own functions,
run on an unmodified checkout of the reference and frozen under tests/golden/
by tests/golden/make_golden.py, and (ii) the analytic known-answer tests of SURVEY B.1.
``tests/test_oracle_golden.py`` checks this oracle against both.

Passing ``dtype=np.float64`` evaluates the same formulas in double precision; the
difference between the two runs is what classifies consistency-mask flips (a hard
``<`` threshold, homography.py:157-158) in the parity tests.
"""
from __future__ import annotations

import numpy as np

__all__ = [
    "relative_poses", "camera_rays",
    "depth_sampler", "camera_terms", "bilinear_zeros", "cost_volume_cw", "cost_volume_f",
    "gaussian_update", "gaussian_update_backward", "convex_upsample", "softmax",
]


def depth_sampler(mu, sigma, k, dtype=np.float32):
    """d[b,j] = mu[b] + sigma[b]*k_j — separate multiply and add (MAGNET.py:155), k rounded
    to the working dtype first.  mu, sigma: (B,H,W) -> (B,D,H,W)."""
    mu = np.asarray(mu, dtype=dtype)
    sigma = np.asarray(sigma, dtype=dtype)
    k = np.asarray(k, dtype=np.float64).astype(np.float32).astype(dtype)
    prod = (sigma[:, None] * k[None, :, None, None]).astype(dtype)
    return (mu[:, None] + prod).astype(dtype)


def camera_terms(intM, R, t, rays, dtype=np.float32):
    """Per (b,v) projection terms of homography.py:98-102.

    intM (3,3), R (3,3), t (3,), rays (3,HW) ->
      a  = K t          (3,)     'term1_pix'
      q  = (K R) rays   (3,HW)   'term2_pix'
      tz = t[2], rz = R[2,:] rays (HW,)  — the z rows of 'term1_cam'/'term2_cam'
    The identity-matrix products at :98-100 are exact no-ops (SURVEY A.5 #8)."""
    K = np.asarray(intM, dtype=dtype)
    R = np.asarray(R, dtype=dtype)
    t = np.asarray(t, dtype=dtype)
    rays = np.asarray(rays, dtype=dtype)
    a = (K @ t).astype(dtype)
    A = (K @ R).astype(dtype)
    q = (A @ rays).astype(dtype)
    rz = (R @ rays).astype(dtype)[2]
    return a, q, t[2], rz


def _project(a, q, d, H, W, dtype):
    """Pixel coordinates -> clamped normalised grid coordinates (homography.py:131-148).
    a (3,), q (3,HW), d (D,HW).  Returns gx, gy (D,HW)."""
    one_em10 = dtype(1e-10)
    P0 = (a[0] + (q[0][None] * d).astype(dtype)).astype(dtype)
    P1 = (a[1] + (q[1][None] * d).astype(dtype)).astype(dtype)
    P2 = (a[2] + (q[2][None] * d).astype(dtype)).astype(dtype)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        Zp = (P2 + one_em10).astype(dtype)
        u = (P0 / Zp).astype(dtype)
        w = (P1 / Zp).astype(dtype)
        uc, vc = dtype(W / 2.0), dtype(H / 2.0)
        gx = ((u - uc).astype(dtype) / uc).astype(dtype)
        gy = ((w - vc).astype(dtype) / vc).astype(dtype)
    ten = dtype(10.0)
    gx = np.where(gx > ten, ten, gx)
    gx = np.where(gx < -ten, -ten, gx)
    gy = np.where(gy > ten, ten, gy)
    gy = np.where(gy < -ten, -ten, gy)
    return gx.astype(dtype), gy.astype(dtype)


def _unnormalize(g, size, dtype):
    # grid_sampler_unnormalize, align_corners=False: ((coord + 1) * size - 1) / 2
    return ((((g + dtype(1.0)).astype(dtype) * dtype(size)).astype(dtype) - dtype(1.0)).astype(dtype)
            / dtype(2.0)).astype(dtype)


def bilinear_zeros(src, gx, gy, dtype=np.float32):
    """grid_sample(bilinear, zeros, align_corners=False) of src (C,H,W) at normalised
    coordinates gx, gy (any shape S) -> (C, *S).  Taps outside the image contribute
    nothing (within_bounds_2d); accumulation order nw, ne, sw, se.  Non-finite
    coordinates are treated as out of bounds (CUDA kernel behaviour)."""
    src = np.asarray(src, dtype=dtype)
    C, H, W = src.shape
    ix = _unnormalize(gx, W, dtype)
    iy = _unnormalize(gy, H, dtype)
    finite = np.isfinite(ix) & np.isfinite(iy)
    ixs = np.where(finite, ix, dtype(-5.0))
    iys = np.where(finite, iy, dtype(-5.0))
    x0f = np.floor(ixs)
    y0f = np.floor(iys)
    x1f = x0f + dtype(1.0)
    y1f = y0f + dtype(1.0)
    w_nw = ((x1f - ixs) * (y1f - iys)).astype(dtype)
    w_ne = ((ixs - x0f) * (y1f - iys)).astype(dtype)
    w_sw = ((x1f - ixs) * (iys - y0f)).astype(dtype)
    w_se = ((ixs - x0f) * (iys - y0f)).astype(dtype)
    x0 = x0f.astype(np.int64)
    y0 = y0f.astype(np.int64)
    out = np.zeros((C,) + ix.shape, dtype=dtype)
    for (yy, xx, ww) in ((y0, x0, w_nw), (y0, x0 + 1, w_ne), (y0 + 1, x0, w_sw), (y0 + 1, x0 + 1, w_se)):
        inb = (xx >= 0) & (xx < W) & (yy >= 0) & (yy < H) & finite
        val = src[:, np.clip(yy, 0, H - 1), np.clip(xx, 0, W - 1)]
        out = (out + np.where(inb[None], (val * ww[None]).astype(dtype), dtype(0.0))).astype(dtype)
    return out


def cost_volume_cw(d_volume, ref_feat, nghbr_feat, nghbr_gmms, R, t, is_valid, intM, rays, thres,
                   dtype=np.float32, return_margin=False):
    """est_costvolume_CW (homography.py:79-121) + _compute_cost_CW (:124-161).

    d_volume (B,D,H,W); ref_feat (B,C,H,W); nghbr_feat (V*B,C,H,W) view-major;
    nghbr_gmms (V*B,2,H,W) [mu,sigma]; R (B,V,3,3); t (B,V,3); is_valid (B,V) int;
    intM (B,3,3); rays (B,3,HW); thres int.  -> (B,D,H,W) fp32.

    Per-view products and the accumulation over views are fp64 (the ``.double()`` at :158),
    the sum is rounded to fp32 on store (:118) and divided by float(V) over ALL views (:120).
    With return_margin=True also returns min over views of | |z-mu~| - kappa*sigma~ | scaled by
    max(|z|, kappa*sigma~, 1e-30): how close each output is to a consistency-mask flip."""
    d_volume = np.asarray(d_volume)
    B, D, H, W = d_volume.shape
    HW = H * W
    V = np.asarray(nghbr_feat).shape[0] // B
    out = np.zeros((B, D, H, W), dtype=np.float32)
    margin = np.full((B, D, H, W), np.inf, dtype=np.float64)
    kappa = dtype(float(thres))
    for b in range(B):
        ref = np.asarray(ref_feat[b], dtype=dtype)                    # (C,H,W)
        d = np.asarray(d_volume[b], dtype=dtype).reshape(D, HW)
        acc = np.zeros((D, H, W), dtype=np.float64)
        for v in range(V):
            if int(is_valid[b][v]) != 1:
                continue
            a, q, tz, rz = camera_terms(intM[b], R[b][v], t[b][v], rays[b], dtype)
            gx, gy = _project(a, q, d, H, W, dtype)
            z = (tz + (rz[None] * d).astype(dtype)).astype(dtype).reshape(D, H, W)
            gx = gx.reshape(D, H, W)
            gy = gy.reshape(D, H, W)
            idx = v * B + b
            fwarp = bilinear_zeros(nghbr_feat[idx], gx, gy, dtype)     # (C,D,H,W)
            mu_w = bilinear_zeros(np.asarray(nghbr_gmms[idx])[0:1], gx, gy, dtype)[0]
            sg_w = bilinear_zeros(np.asarray(nghbr_gmms[idx])[1:2], gx, gy, dtype)[0]
            prod = (ref[:, None] * fwarp).astype(dtype)
            feat_cost = prod.sum(axis=0, dtype=dtype)                  # (D,H,W)
            with np.errstate(invalid="ignore"):
                diff = np.abs((z - mu_w).astype(dtype))
                thr = (sg_w * kappa).astype(dtype)
                m = diff < thr
            acc += feat_cost.astype(np.float64) * m.astype(np.float64)
            if return_margin:
                with np.errstate(invalid="ignore"):
                    scale = np.maximum(np.maximum(np.abs(z), np.abs(thr)), 1e-30).astype(np.float64)
                    mg = np.abs(diff.astype(np.float64) - thr.astype(np.float64)) / scale
                mg = np.where(np.isfinite(mg), mg, 0.0)
                margin[b] = np.minimum(margin[b], mg)
        out[b] = acc.astype(np.float32)
    out = (out / np.float32(V)).astype(np.float32)
    if return_margin:
        return out, margin
    return out


def softmax(x, axis):
    x = np.asarray(x)
    m = x.max(axis=axis, keepdims=True)
    e = np.exp(x - m)
    return (e / e.sum(axis=axis, keepdims=True)).astype(x.dtype)


def cost_volume_f(d_center, ref_feat, nghbr_feat, R, t, is_valid, intM, rays, dtype=np.float32,
                  apply_softmax=True):
    """est_costvolume_F (homography.py:10-47) + _compute_cost_F (:50-75): one shared depth per
    plane, no consistency test, fp32 accumulation over views, /V, softmax over planes."""
    ref_feat = np.asarray(ref_feat)
    B, C, H, W = ref_feat.shape
    HW = H * W
    dc = np.asarray(d_center, dtype=dtype).reshape(-1)
    D = dc.shape[0]
    V = np.asarray(nghbr_feat).shape[0] // B
    out = np.zeros((B, D, H, W), dtype=dtype)
    dfull = np.broadcast_to(dc[:, None], (D, HW)).astype(dtype)
    for b in range(B):
        ref = np.asarray(ref_feat[b], dtype=dtype)
        acc = np.zeros((D, H, W), dtype=dtype)
        for v in range(V):
            if int(is_valid[b][v]) != 1:
                continue
            a, q, _, _ = camera_terms(intM[b], R[b][v], t[b][v], rays[b], dtype)
            gx, gy = _project(a, q, dfull, H, W, dtype)
            fwarp = bilinear_zeros(nghbr_feat[v * B + b], gx.reshape(D, H, W), gy.reshape(D, H, W), dtype)
            acc = (acc + (ref[:, None] * fwarp).astype(dtype).sum(axis=0, dtype=dtype)).astype(dtype)
        out[b] = acc
    out = (out / dtype(V)).astype(dtype)
    if apply_softmax:
        out = softmax(out, axis=1)
    return out


def gaussian_update(d_output, ref_gmm, dtype=np.float32):
    """GNET.forward's update equations (MAGNET.py:60,65-69).
    d_output (B,2,H,W) = (mu_1, sigma_1); ref_gmm (B,2,H,W) = (mu_0, sigma_0)."""
    d_output = np.asarray(d_output, dtype=dtype)
    ref_gmm = np.asarray(ref_gmm, dtype=dtype)
    mu1, s1 = d_output[:, 0], d_output[:, 1]
    mu0, s0 = ref_gmm[:, 0], ref_gmm[:, 1]
    mu_new = (mu0 + (mu1 * s0).astype(dtype)).astype(dtype)
    with np.errstate(over="ignore"):
        elu = np.where(s1 > 0, s1, np.expm1(np.minimum(s1, dtype(0.0))).astype(dtype))
    sig_new = ((((elu + dtype(1.0)).astype(dtype) + dtype(1e-10)).astype(dtype)) * s0).astype(dtype)
    return np.stack([mu_new, sig_new], axis=1)


def gaussian_update_backward(grad_out, d_output, ref_gmm, dtype=np.float32):
    """d(loss)/d(d_output) for gaussian_update: dmu1 = g_mu*sigma0,
    dsigma1 = g_sigma*sigma0*(sigma1>0 ? 1 : exp(sigma1))  (SURVEY §8 a6)."""
    g = np.asarray(grad_out, dtype=dtype)
    d_output = np.asarray(d_output, dtype=dtype)
    s0 = np.asarray(ref_gmm, dtype=dtype)[:, 1]
    s1 = d_output[:, 1]
    dmu1 = (g[:, 0] * s0).astype(dtype)
    delu = np.where(s1 > 0, dtype(1.0), np.exp(np.minimum(s1, dtype(0.0))).astype(dtype))
    ds1 = ((g[:, 1] * delu).astype(dtype) * s0).astype(dtype)
    return np.stack([dmu1, ds1], axis=1)


def convex_upsample(depth, up_mask, k, dtype=np.float32):
    """upsample_depth_via_mask (MAGNET.py:15-27): softmax over the 9 neighbours of a learned
    mask, weighted sum of the zero-padded 3x3 neighbourhood, pixel-shuffle by k."""
    depth = np.asarray(depth, dtype=dtype)
    up_mask = np.asarray(up_mask, dtype=dtype)
    N, C, H, W = depth.shape
    m = softmax(up_mask.reshape(N, 1, 9, k, k, H, W), axis=2)
    pad = np.zeros((N, C, H + 2, W + 2), dtype=dtype)
    pad[:, :, 1:-1, 1:-1] = depth
    nb = np.stack([pad[:, :, dy:dy + H, dx:dx + W] for dy in range(3) for dx in range(3)], axis=2)
    up = (m * nb.reshape(N, C, 9, 1, 1, H, W)).sum(axis=2, dtype=dtype)   # (N,C,k,k,H,W)
    up = up.transpose(0, 1, 4, 2, 5, 3)                                    # (N,C,H,k,W,k)
    return up.reshape(N, C, k * H, k * W).astype(dtype)


def relative_poses(ext_ref, ext_nghbr):
    """data_preprocess (utils/utils.py:72-98): ext_ref (B,4,4), ext_nghbr (V,B,4,4) fp32 ->
    nghbr_poses (B,V,4,4) = ext_nghbr . inv(ext_ref) and is_valid (B,V); NaN in either extrinsic or in the
    product invalidates the view (its pose stays zero)."""
    ext_ref = np.asarray(ext_ref, dtype=np.float32)
    ext_nghbr = np.asarray(ext_nghbr, dtype=np.float32)
    V, B = ext_nghbr.shape[:2]
    poses = np.zeros((B, V, 4, 4), dtype=np.float32)
    valid = np.ones((B, V), dtype=np.int32)
    for b in range(B):
        if np.isnan(ext_ref[b]).any():
            valid[b, :] = 0
            continue
        inv = np.linalg.inv(ext_ref[b])
        for v in range(V):
            if np.isnan(ext_nghbr[v, b]).any():
                valid[b, v] = 0
                continue
            pose = (ext_nghbr[v, b] @ inv).astype(np.float32)
            if np.isnan(pose).any():
                valid[b, v] = 0
            else:
                poses[b, v] = pose
    return poses, valid


def camera_rays(raw, H, W):
    """get_ray_array + get_cam_intrinsics (data/dataloader_scannet.py:113-153; crop-margin variant
    data/dataloader_kitti.py:94-127): raw (B,8) float64 = fx, fy, cx, cy of the raw image, img_W, img_H (the cropped image
    the grid spans), left_margin, top_margin ((B,6) = no crop: ScanNet) -> intM (B,3,3) fp32 of the H x W grid, rays
    (B,3,H*W) fp32 through the pixel centres (x+0.5, y+0.5); everything in fp64 until the final cast, operation by
    operation as in the numpy originals (with zero margins the KITTI expressions reduce exactly to the ScanNet ones)."""
    raw = np.asarray(raw, dtype=np.float64)
    if raw.shape[1] == 6:
        raw = np.concatenate([raw, np.zeros((raw.shape[0], 2))], axis=1)
    B = raw.shape[0]
    intM = np.zeros((B, 3, 3), dtype=np.float64)
    rays = np.ones((B, H, W, 3), dtype=np.float64)
    xs = np.arange(W, dtype=np.float64) + 0.5
    ys = np.arange(H, dtype=np.float64) + 0.5
    for b in range(B):
        fx, fy, cx, cy, iw, ih, left, top = raw[b]
        intM[b, 2, 2] = 1.0
        intM[b, 0, 0] = fx * (W / iw)
        intM[b, 1, 1] = fy * (H / ih)
        intM[b, 0, 2] = (cx - left) * (W / iw)
        intM[b, 1, 2] = (cy - top) * (H / ih)
        rays[b, :, :, 0] = (((xs * (iw / W)) - cx) + left)[None, :] / fx
        rays[b, :, :, 1] = (((ys * (ih / H)) - cy) + top)[:, None] / fy
    rays2d = np.reshape(np.transpose(rays, (0, 3, 1, 2)), (B, 3, H * W))
    return intM.astype(np.float32), rays2d.astype(np.float32)


def gaussian_nll(pred_list, gt, mask, gamma=0.8):
    """MagnetLoss 'gaussian' (utils/losses.py:34-50): sum_i gamma^(n-i-1) mean_{mask}[(mu-gt)^2 / (2 var) + 0.5 log var],
    var = max(sigma^2, 1e-10).  pred_list: (B,2,H,W) arrays at the resolution of gt (B,1,H,W); mask bool (B,1,H,W).
    fp32 operations in the reference's order."""
    gt = np.asarray(gt, dtype=np.float32)
    mask = np.asarray(mask, dtype=bool)
    g = gt[mask]
    n = len(pred_list)
    loss = np.float32(0.0)
    for i, pred in enumerate(pred_list):
        pred = np.asarray(pred, dtype=np.float32)
        mu, sigma = pred[:, 0:1][mask], pred[:, 1:2][mask]
        var = np.square(sigma)
        var[var < 1e-10] = 1e-10
        nll = (np.square(mu - g) / (np.float32(2) * var)) + (np.float32(0.5) * np.log(var))
        loss = np.float32(loss + np.float32(gamma ** (n - i - 1)) * np.mean(nll, dtype=np.float32))
    return loss

