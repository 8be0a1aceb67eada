"""numpy restatement, in float64, of the gradient of the CW volume w.r.t. the depth hypotheses (homography.py:124-161):

    grad_d[b,j,p] = 1/V sum_v g m (dcost/dix du/dd + dcost/diy dv/dd),  du/dd = (q0 Zp - P0 q2) / Zp^2  (v likewise)

with cost the bilinear interpolant of the four tap dot products <ref_p, src_t> (zero outside the image), m the
consistency mask and zero through a coordinate clamped at +-10 (the reference's masked assignment)."""
import numpy as np


def grad_depth_cw(d_volume, ref, src, gmm, R, t, valid, intM, rays, thres, gout):
    """All arrays float64 numpy; returns (grad_d (B,D,H,W), margin (B,D,H,W), edge (B,D,H,W), reached): the distance of
    every element to a mask flip (relative) and to a cell edge (pixels), minimised over the valid views, and how many
    (view, hypothesis, pixel) samples hit the +-10 clamp, had a tap outside the image, had every tap outside."""
    B, D, H, W = d_volume.shape
    V = src.shape[0] // B
    C = ref.shape[1]
    gd = np.zeros((B, D, H, W))
    margin = np.full((B, D, H, W), np.inf)
    edge = np.full((B, D, H, W), np.inf)
    reached = {"clamped": 0, "tap_outside": 0, "all_outside": 0}
    for b in range(B):
        d = d_volume[b].reshape(D, -1)
        refb = ref[b].reshape(C, -1)
        for v in range(V):
            if valid[b, v] != 1:
                continue
            K = intM[b]
            q = K @ R[b, v] @ rays[b]                     # (3, HW)
            a = K @ t[b, v]
            P = a[:, None, None] + q[:, None, :] * d[None]  # (3, D, HW)
            Zp = P[2] + 1e-10
            u, w = P[0] / Zp, P[1] / Zp
            gx, gy = (u - W / 2.0) / (W / 2.0), (w - H / 2.0) / (H / 2.0)
            dudd = np.where(np.abs(gx) > 10, 0.0, (q[0][None] * Zp - P[0] * q[2][None]) / Zp ** 2)
            dvdd = np.where(np.abs(gy) > 10, 0.0, (q[1][None] * Zp - P[1] * q[2][None]) / Zp ** 2)
            reached["clamped"] += int(((np.abs(gx) > 10) | (np.abs(gy) > 10)).sum())
            gx, gy = np.clip(gx, -10, 10), np.clip(gy, -10, 10)
            ix, iy = ((gx + 1) * W - 1) / 2, ((gy + 1) * H - 1) / 2
            x0, y0 = np.floor(ix), np.floor(iy)
            fx, fy = ix - x0, iy - y0
            edge[b] = np.minimum(edge[b], np.minimum(np.minimum(fx, 1 - fx), np.minimum(fy, 1 - fy)).reshape(D, H, W))
            s = src[v * B + b].reshape(C, -1)
            gm = gmm[v * B + b].reshape(2, -1)
            f, mu, sg, n_in = {}, 0.0, 0.0, 0
            for dx in (0, 1):
                for dy in (0, 1):
                    xi, yi = (x0 + dx).astype(np.int64), (y0 + dy).astype(np.int64)
                    inb = (xi >= 0) & (xi < W) & (yi >= 0) & (yi < H)
                    n_in = n_in + inb
                    idx = np.where(inb, yi * W + xi, 0)
                    dot = (refb[:, None, :] * s[:, idx]).sum(0)
                    f[dx, dy] = np.where(inb, dot, 0.0)
                    wgt = (fx if dx else 1 - fx) * (fy if dy else 1 - fy)
                    mu = mu + np.where(inb, gm[0][idx], 0.0) * wgt
                    sg = sg + np.where(inb, gm[1][idx], 0.0) * wgt
            reached["tap_outside"] += int((n_in < 4).sum())
            reached["all_outside"] += int((n_in == 0).sum())
            z = P[2]
            gap, thr = np.abs(z - mu), sg * thres
            m = gap < thr
            scale = np.maximum(np.maximum(np.abs(z), np.abs(thr)), 1e-30)
            margin[b] = np.minimum(margin[b], (np.abs(gap - thr) / scale).reshape(D, H, W))
            dcdx = (f[1, 0] - f[0, 0]) * (1 - fy) + (f[1, 1] - f[0, 1]) * fy
            dcdy = (f[0, 1] - f[0, 0]) * (1 - fx) + (f[1, 1] - f[1, 0]) * fx
            g = gout[b].reshape(D, -1)
            gd[b] += (g * m * (dcdx * dudd + dcdy * dvdd)).reshape(D, H, W)
    return gd / V, margin, edge, reached
