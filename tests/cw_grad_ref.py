"""numpy restatements, in float64, of both cost volumes and of every gradient the backward kernels write, each with a
companion bound (the same sum over the absolute value of every factor) and the maps of the places where fp32 rounding
can change a discrete decision (consistency mask, bilinear cell, projection near z = 0).

CW volume (homography.py:124-161, DESIGN §3.5), per batch element b, hypothesis j, pixel p and valid view v:

    cost_v = sum_t w_t f_t,   f_t = <ref[b,:,p], src_v[:, tap_t]>   (zero outside the image)
    out    = 1/V sum_v m_v cost_v                      (m_v: |z - mu~| < kappa sigma~, or 1 without consistency)
    gs     = gout / V
    grad_ref[b,c,p]   = sum_{v,j,t} gs m_v w_t src_v[c, tap_t]
    grad_src[v,c,tap] = sum_{p,j: tap_t = tap} gs m_v w_t ref[b,c,p]
    grad_d[b,j,p]     = sum_v gs m_v (dcost/dix du/dd + dcost/diy dv/dd),  du/dd = (q0 - u q2) / Zp
    GAUSS mode (d_j = mu + sigma k_j): grad_mu = sum_j grad_d_j, grad_sigma = sum_j k_j grad_d_j

F volume (homography.py:10-75): the same sum with one plane depth per hypothesis, m = 1, scores = out, optionally a
softmax over the planes; its backward takes the score gradient gs = p (g - sum_j p g) / V (softmax) or g / V.

Sample positions (``pos``):
  "f64"    — the reference's formulas in float64 (the CPU comparison with float64 autograd);
  "direct" — the DIRECT forward's fp32 operation sequence (oracle ``_project`` / ``_unnormalize``, q = A r as the fma
             chain of the kernels): tap set, mask and weights are the kernel's;
  "mma"    — the sequence of ``project()`` (cells_common.cuh), whose reciprocal (rcp + one Newton step) is not
             reproducible here: the bounds then carry a position-error term |g| |d cost / d ix| delta with
             delta = (A + 8) u |ix + 0.5| (DESIGN §3.1).  The F volume and every tap-sharing kernel use these positions.
Everything downstream of the positions (dot products, products with g, sums over j, t, v) is float64.  The geometry is
numpy; the contractions gather each tap's source vector and scatter into its cell (never the all-pairs matrix
<ref_p, src_s>) in torch float64 on the device the caller names (the GPU tests pass theirs), one hypothesis chunk of one
view at a time, so the reference runs at the production shapes."""
import numpy as np
import torch

from oracle import magnet_oracle as mo

U = 2.0 ** -24
# the tensor-core forward's box bound (DESIGN §3.1): beyond it the kernel takes its exact fallback, and a position's
# rounding error may reach a cell edge
AMP_LIMIT = 2.0 ** 16


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


# ---------------------------------------------------------------------------------------------------------------------
# Full reference: geometry (positions, taps, weights, masks, ambiguity maps), then values and gradients.

def _fma32(a, b, c):
    """fp32 fma: the product of two fp32 values is exact in float64, one rounding of the sum to fp32 (a double
    rounding through float64 can differ from the hardware only when the sum sits on an fp32 midpoint)."""
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(np.float32)


def cameras_f64(intM, R, t, valid):
    """(B*V, 16) camera table (struct magnet_camera: valid, a = K t, A = K R row-major) in float64, for "f64"."""
    B, V = R.shape[:2]
    cams = np.zeros((B * V, 16))
    for b in range(B):
        for v in range(V):
            cams[b * V + v, 0] = 1.0 if int(valid[b, v]) == 1 else 0.0
            cams[b * V + v, 1:4] = intM[b] @ t[b, v]
            cams[b * V + v, 4:13] = (intM[b] @ R[b, v]).reshape(-1)
    return cams


def gauss_depths(gmm, k, pos):
    """d_j = mu + sigma k_j: fp32 multiply, then add (MAGNET.py:155), or float64 for "f64".  gmm (B,2,H,W)."""
    if pos == "f64":
        return gmm[:, 0:1] + gmm[:, 1:2] * np.asarray(k, np.float64).reshape(1, -1, 1, 1)
    kk = np.asarray(k, np.float64).astype(np.float32).reshape(1, -1, 1, 1)
    g = np.asarray(gmm, np.float32)
    return (g[:, 0:1] + (g[:, 1:2] * kk).astype(np.float32)).astype(np.float32)


class View:
    """One (b, v) pair: per tap t (00, 01, 10, 11 = (dy, dx)) the flat source index, in-image flag and weight, plus
    the depth derivatives of the position and the ambiguity maps.  Arrays are (D, HW)."""


def _view(cam, rays, d, H, W, pos, src_gmm, kappa, consistency):
    HW = H * W
    g = View()
    a, A = cam[1:4], cam[4:13]
    if pos == "f64":
        a = np.asarray(a, np.float64)
        q = np.asarray(A, np.float64).reshape(3, 3) @ np.asarray(rays, np.float64)
        d = np.asarray(d, np.float64)
        P = a[:, None, None] + q[:, None, :] * d[None]
        Zp = P[2] + 1e-10
        with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
            u, w = P[0] / Zp, P[1] / Zp
            gx, gy = (u - W / 2.0) / (W / 2.0), (w - H / 2.0) / (H / 2.0)
        clamped = (np.abs(gx) > 10) | (np.abs(gy) > 10)
        gx, gy = np.clip(gx, -10, 10), np.clip(gy, -10, 10)
        ix, iy = ((gx + 1) * W - 1) / 2, ((gy + 1) * H - 1) / 2
        z = P[2]
    else:
        a32, A32 = np.asarray(a, np.float32), np.asarray(A, np.float32)
        r = np.asarray(rays, np.float32)
        q = np.stack([_fma32(A32[3 * i + 2], r[2], _fma32(A32[3 * i + 1], r[1], (A32[3 * i] * r[0]).astype(np.float32)))
                      for i in range(3)])
        d = np.asarray(d, np.float32)
        with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
            z32 = (a32[2] + (q[2][None] * d).astype(np.float32)).astype(np.float32)
            if pos == "direct":
                gx, gy = mo._project(a32, q, d, H, W, np.float32)
                ix, iy = mo._unnormalize(gx, W, np.float32), mo._unnormalize(gy, H, np.float32)
            else:                                  # project(): fma(q0, d, a0) * rcp(z + 1e-10) - 0.5, clamp_coord
                Zp32 = (z32 + np.float32(1e-10)).astype(np.float32)
                rc = (1.0 / Zp32.astype(np.float64)).astype(np.float32)
                ix = _fma32(_fma32(q[0][None], d, a32[0]), rc, -0.5)
                iy = _fma32(_fma32(q[1][None], d, a32[1]), rc, -0.5)
        P = np.asarray(a32, np.float64)[:, None, None] + q.astype(np.float64)[:, None, :] * d.astype(np.float64)[None]
        Zp = P[2] + 1e-10
        with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
            u, w = P[0] / Zp, P[1] / Zp
            clamped = (np.abs((u - W / 2.0) / (W / 2.0)) > 10) | (np.abs((w - H / 2.0) / (H / 2.0)) > 10)
        ix, iy = ix.astype(np.float64), iy.astype(np.float64)
        z = P[2]
        q = q.astype(np.float64)
    finite = np.isfinite(ix) & np.isfinite(iy)
    ixs, iys = np.where(finite, ix, -5.0), np.where(finite, iy, -5.0)
    if pos == "mma":                              # clamp_coord: only moves positions whose taps are all outside
        ixs, iys = np.clip(ixs, -2.0, W + 1.0), np.clip(iys, -2.0, H + 1.0)
    x0, y0 = np.floor(ixs), np.floor(iys)
    g.x0, g.y0 = x0, y0
    fx, fy = ixs - x0, iys - y0
    g.wx, g.wy = (1.0 - fx, fx), (1.0 - fy, fy)
    g.idx, g.inb, g.w = {}, {}, {}
    n_in = 0
    for dy in (0, 1):
        for dx in (0, 1):
            xi, yi = x0.astype(np.int64) + dx, y0.astype(np.int64) + dy
            inb = (xi >= 0) & (xi < W) & (yi >= 0) & (yi < H) & finite
            g.inb[dy, dx] = inb
            g.idx[dy, dx] = np.where(inb, yi * W + xi, 0)
            g.w[dy, dx] = np.where(inb, g.wx[dx] * g.wy[dy], 0.0)
            n_in = n_in + inb
    g.any_in = n_in > 0
    g.clamped, g.tap_outside, g.all_outside, g.behind = clamped, n_in < 4, n_in == 0, z < 0
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        az = np.abs(z)
        g.amp = np.abs(q[2][None] * d) / az + 2e-3 / az                   # DESIGN §3.1
        g.amp_bad = ~((g.amp + 8.0) * (max(W, H) + 3.0) <= AMP_LIMIT)
        # du/dd, dv/dd and their cancellation-free bounds (|q0| + |u q2|) / |Zp|
        g.dudd = np.where(clamped, 0.0, (q[0][None] - u * q[2][None]) / Zp)
        g.dvdd = np.where(clamped, 0.0, (q[1][None] - w * q[2][None]) / Zp)
        g.Du = np.where(clamped, 0.0, (np.abs(q[0][None]) + np.abs(u * q[2][None])) / np.abs(Zp))
        g.Dv = np.where(clamped, 0.0, (np.abs(q[1][None]) + np.abs(w * q[2][None])) / np.abs(Zp))
    # position error of project() in units of u: delta = (A + 8) u |ix + 0.5| (capped: no inf * 0 in the bounds)
    g.ex = np.where(g.any_in, np.minimum((g.amp + 8.0) * np.abs(ixs + 0.5), 1e30), 0.0)
    g.ey = np.where(g.any_in, np.minimum((g.amp + 8.0) * np.abs(iys + 0.5), 1e30), 0.0)
    g.ex, g.ey = np.where(np.isnan(g.ex), 1e30, g.ex), np.where(np.isnan(g.ey), 1e30, g.ey)
    # distance to a cell edge that changes the tap set: edges at -1..W (x) / -1..H (y), for positions near the image
    ex_ = np.abs(ix - np.round(ix))
    ey_ = np.abs(iy - np.round(iy))
    near = finite & (ix > -2.0) & (ix < W + 1.0) & (iy > -2.0) & (iy < H + 1.0)
    ex_ = np.where((np.round(ix) >= -1) & (np.round(ix) <= W), ex_, np.inf)
    ey_ = np.where((np.round(iy) >= -1) & (np.round(iy) <= H), ey_, np.inf)
    g.edge = np.where(near, np.minimum(ex_, ey_), np.inf)
    # consistency mask and its relative margin
    if consistency:
        gm = np.asarray(src_gmm, np.float64).reshape(2, HW)
        mu = sum(np.where(g.inb[t], gm[0][g.idx[t]], 0.0) * g.wx[t[1]] * g.wy[t[0]] for t in g.idx)
        sg = sum(np.where(g.inb[t], gm[1][g.idx[t]], 0.0) * g.wx[t[1]] * g.wy[t[0]] for t in g.idx)
        gap, thr = np.abs(z - mu), sg * kappa
        with np.errstate(invalid="ignore"):
            g.m = (gap < thr) & g.any_in
            mg = np.abs(gap - thr) / np.maximum(np.maximum(np.abs(z), np.abs(thr)), 1e-30)
        g.margin = np.where(g.any_in & np.isfinite(mg), mg, np.where(g.any_in, 0.0, np.inf))
    else:
        g.m = g.any_in.copy()
        g.margin = np.full(g.m.shape, np.inf)
    return g


class Reference:
    """The reference for one call: ``Reference(...)`` walks the geometry of every valid (b, v) pair once and keeps
    only the ambiguity and ``reached`` maps; ``forward()`` the volume and its bound; ``backward(gs, gs_abs)`` the
    gradients for a score gradient gs (= gout / V for the CW volume) and its bound.  Each call recomputes the geometry
    (numpy, O(D HW) per view) in hypothesis chunks, so no more than one chunk of one view is alive at a time.

    The contractions are gathers and scatters in torch float64 on ``device``: f_t = <ref_p, src[idx_t]> from the
    gathered tap vectors, grad_ref the weighted sum of gathered source vectors, grad_src an ``index_add_`` into the
    tap's cell; each bound is the same expression over absolute values.  They equal the all-pairs contraction
    <ref_p, src_s> up to the float64 summation order (tests/test_cw_grad_cpu.py holds them to it).

    depth (B,D,H,W) hypothesis depths (fp32 for "direct" / "mma"); ref (B,C,H,W); src (V*B,C,H,W) view-major;
    src_gmm (V*B,2,H,W) or None; cams (B*V,16) the kernel's camera table (b-major); rays (B,3,HW)."""

    CHUNK = 1 << 25                            # elements of one gathered (C, chunk, HW) block: 256 MB in float64

    def __init__(self, depth, ref, src, src_gmm, cams, rays, kappa, *, pos="direct", consistency=True, device="cpu"):
        self.depth = np.asarray(depth)
        self.B, self.D, self.H, self.W = self.depth.shape
        self.HW = self.H * self.W
        self.C = ref.shape[1]
        self.V = src.shape[0] // self.B
        self.dev = torch.device(device)
        self.ref = self._t(np.asarray(ref, np.float64).reshape(self.B, self.C, self.HW))
        self.src = self._t(np.asarray(src, np.float64).reshape(self.V * self.B, self.C, self.HW))
        self.cams, self.rays = np.asarray(cams), np.asarray(rays)
        self.src_gmm, self.kappa, self.consistency = src_gmm, kappa, consistency
        self.pos = pos
        self.pos_err = pos == "mma"            # bounds carry the position-error term by default on mma positions
        self.valid = [(b, v) for b in range(self.B) for v in range(self.V) if self.cams[b * self.V + v][0] == 1.0]
        self.nj = max(1, min(self.D, self.CHUNK // (self.C * self.HW), (1 << 20) // self.HW))
        self._memo = {}
        shp = (self.B, self.D, self.HW)
        self.margin, self.edge, self.delta = np.full(shp, np.inf), np.full(shp, np.inf), np.zeros(shp)
        self.amp_bad = np.zeros(shp, bool)
        self.reached = {k: np.zeros(shp, bool) for k in ("clamped", "tap_outside", "all_outside", "behind")}
        # box of the cell origins of every (valid view, 64-hypothesis chunk, pixel): the tensor-core window
        nk = -(-self.D // 64)
        self.origins = np.stack([np.full((self.B, self.V, nk, self.HW), s * np.inf) for s in (1, -1, 1, -1)])
        for b, v, j0, j1, g in self._chunks():
            sl = (b, slice(j0, j1))
            self.margin[sl] = np.minimum(self.margin[sl], g.margin)
            self.edge[sl] = np.minimum(self.edge[sl], g.edge)
            self.delta[sl] = np.maximum(self.delta[sl], U * np.maximum(g.ex, g.ey))
            self.amp_bad[sl] |= g.amp_bad & g.any_in
            for k in self.reached:
                self.reached[k][sl] |= getattr(g, k)
            for k in range(j0 // 64, (j1 - 1) // 64 + 1):
                s = slice(max(j0, 64 * k) - j0, min(j1, 64 * k + 64) - j0)
                o = self.origins[:, b, v, k]
                o[0], o[1] = np.minimum(o[0], g.x0[s].min(0)), np.maximum(o[1], g.x0[s].max(0))
                o[2], o[3] = np.minimum(o[2], g.y0[s].min(0)), np.maximum(o[3], g.y0[s].max(0))

    def _t(self, x):
        return torch.tensor(np.asarray(x), device=self.dev)

    def _chunks(self):
        """(b, v, j0, j1, View of hypotheses j0..j1-1) for every valid (b, v) pair."""
        for b, v in self.valid:
            gm = None if self.src_gmm is None else self.src_gmm[v * self.B + b]
            d = self.depth[b].reshape(self.D, self.HW)
            for j0 in range(0, self.D, self.nj):
                j1 = min(self.D, j0 + self.nj)
                yield b, v, j0, j1, _view(self.cams[b * self.V + v], self.rays[b], d[j0:j1], self.H, self.W, self.pos,
                                          gm, self.kappa, self.consistency)

    def _taps(self, b, v, g):
        """Per tap t: f_t = <ref_p, src[idx_t]> and <|ref_p|, |src[idx_t]|> (chunk, HW), zero outside the image."""
        r, s = self.ref[b], self.src[v * self.B + b]
        f, fa = {}, {}
        for t in g.idx:
            S = s[:, self._t(g.idx[t])]                              # (C, chunk, HW) gathered tap vectors
            inb = self._t(g.inb[t])
            f[t] = torch.where(inb, (S * r[:, None]).sum(0), 0.0)
            fa[t] = torch.where(inb, (S.abs() * r.abs()[:, None]).sum(0), 0.0)
        return f, fa

    def _feature_grads(self, b, v, g, coef, coef_abs, out):
        """grad_ref[b] += sum_{j,t} coef_t src[idx_t], grad_src[v B + b][idx_t] += ref coef_t, and their bounds from
        coef_abs.  coef / coef_abs: per tap (chunk, HW), zero outside the image; out: (gref, grefb, gsrc, gsrcb)."""
        gref, grefb, gsrc, gsrcb = out
        r, s, i = self.ref[b], self.src[v * self.B + b], v * self.B + b
        for t in g.idx:
            idx = self._t(g.idx[t])
            S = s[:, idx]
            gref[b] += (S * coef[t][None]).sum(1)
            grefb[b] += (S.abs() * coef_abs[t][None]).sum(1)
            gsrc[i].index_add_(1, idx.reshape(-1), (r[:, None] * coef[t][None]).reshape(self.C, -1))
            gsrcb[i].index_add_(1, idx.reshape(-1), (r.abs()[:, None] * coef_abs[t][None]).reshape(self.C, -1))

    def ambiguous(self, margin_tol=1e-3, edge_tol=1e-3):
        """(B,D,H,W): hypotheses near a mask flip, near a cell edge (or within 4 position errors of one, on mma
        positions), or beyond the projection bound."""
        edge_tol = np.maximum(edge_tol, 4.0 * self.delta) if self.pos_err else edge_tol
        amb = (self.margin <= margin_tol) | (self.edge <= edge_tol) | self.amp_bad
        return amb.reshape(self.B, self.D, self.H, self.W)

    def _wabs(self, g, t, pos_err):
        """Bound of the weight of tap t, plus the position error (|dw_t/dix| = wy_t, |dw_t/diy| = wx_t) in units of u
        when ``pos_err``."""
        w = g.wx[t[1]] * g.wy[t[0]]
        if pos_err:
            w = w + g.ex * g.wy[t[0]] + g.ey * g.wx[t[1]]
        return np.where(g.inb[t], w, 0.0)

    def forward(self, pos_err=None):
        """(out, bound, terms, margins): the volume 1/V sum_v m_v cost_v, its bound, the per-view terms cost_v / V
        (V,B,D,H,W, whatever the mask) and the per-view margins (V,B,D,H,W).  ``pos_err``: add the position-error
        term (default: on mma positions) — for a forward kernel whose positions come from project()."""
        pos_err = self.pos_err if pos_err is None else pos_err
        if ("fwd", pos_err) not in self._memo:
            self._memo["fwd", pos_err] = self._forward(pos_err)
        return self._memo["fwd", pos_err]

    def _forward(self, pos_err):
        B, D, HW, V, T = self.B, self.D, self.HW, self.V, self._t
        z = lambda *s: torch.zeros(s, dtype=torch.float64, device=self.dev)
        out, bound, terms = z(B, D, HW), z(B, D, HW), z(V, B, D, HW)
        vmargin = torch.full((V, B, D, HW), np.inf, dtype=torch.float64, device=self.dev)
        for b, v, j0, j1, g in self._chunks():
            f, fa = self._taps(b, v, g)
            cost = sum(T(g.w[t]) * f[t] for t in f)
            cabs = sum(T(self._wabs(g, t, pos_err)) * fa[t] for t in f)
            m, margin = T(g.m), T(g.margin)
            out[b, j0:j1] += torch.where(m, cost, 0.0) / V
            bound[b, j0:j1] += torch.where(m | (margin <= 1e-3), cabs, 0.0) / V
            terms[v, b, j0:j1] = cost / V
            vmargin[v, b, j0:j1] = margin
        sh = (B, D, self.H, self.W)
        return tuple(x.reshape(s).cpu().numpy() for x, s in ((out, sh), (bound, sh), (terms, (V,) + sh),
                                                               (vmargin, (V,) + sh)))

    def backward(self, gs, gs_abs=None, pos_err=None):
        """gs (B,D,H,W): the score gradient (gout / V for the CW volume).  Returns a dict of float64 arrays: ref,
        src (V*B,C,H,W), d (B,D,H,W) and their bounds ref_b, src_b, d_b (in units of u: tolerance c u bound)."""
        B, D, HW, V, C, T = self.B, self.D, self.HW, self.V, self.C, self._t
        pos_err = self.pos_err if pos_err is None else pos_err
        gs = np.asarray(gs, np.float64).reshape(B, D, HW)
        gs_abs = T(np.abs(gs) if gs_abs is None else np.asarray(gs_abs, np.float64).reshape(B, D, HW))
        gs = T(gs)
        z = lambda *s: torch.zeros(s, dtype=torch.float64, device=self.dev)
        feat = (z(B, C, HW), z(B, C, HW), z(V * B, C, HW), z(V * B, C, HW))
        gd, gdb = z(B, D, HW), z(B, D, HW)
        for b, v, j0, j1, g in self._chunks():
            m = T(g.m)
            gm, gma = torch.where(m, gs[b, j0:j1], 0.0), torch.where(m, gs_abs[b, j0:j1], 0.0)
            self._feature_grads(b, v, g, {t: gm * T(g.w[t]) for t in g.idx},
                                {t: gma * T(self._wabs(g, t, pos_err)) for t in g.idx}, feat)
            f, fa = self._taps(b, v, g)
            (wy0, wy1), (wx0, wx1) = map(T, g.wy), map(T, g.wx)
            dcdx = (f[0, 1] - f[0, 0]) * wy0 + (f[1, 1] - f[1, 0]) * wy1
            dcdy = (f[1, 0] - f[0, 0]) * wx0 + (f[1, 1] - f[0, 1]) * wx1
            DX = (fa[0, 1] + fa[0, 0]) * wy0 + (fa[1, 1] + fa[1, 0]) * wy1
            DY = (fa[1, 0] + fa[0, 0]) * wx0 + (fa[1, 1] + fa[0, 1]) * wx1
            FA = fa[0, 0] + fa[0, 1] + fa[1, 0] + fa[1, 1]
            Du, Dv = T(g.Du), T(g.Dv)
            gd[b, j0:j1] += torch.where(gm != 0, gm * (dcdx * T(g.dudd) + dcdy * T(g.dvdd)), 0.0)
            pe = FA * (T(g.ey) * Du + T(g.ex) * Dv) if pos_err else 0.0
            gdb[b, j0:j1] += torch.where(gma != 0, gma * (DX * Du + DY * Dv + pe), 0.0)
        sh = (self.H, self.W)
        n = lambda x, s: x.reshape(s + sh).cpu().numpy()
        gref, grefb, gsrc, gsrcb = feat
        return dict(ref=n(gref, (B, C)), ref_b=n(grefb, (B, C)), src=n(gsrc, (V * B, C)), src_b=n(gsrcb, (V * B, C)),
                    d=n(gd, (B, D)), d_b=n(gdb, (B, D)))


def gauss_chain(gd, gd_b, k):
    """(grad_mu, grad_sigma) = (sum_j grad_d_j, sum_j k_j grad_d_j) (B,2,H,W) and their bound."""
    kk = np.asarray(k, np.float64).astype(np.float32).astype(np.float64).reshape(1, -1, 1, 1)
    val = np.stack([gd.sum(1), (kk * gd).sum(1)], axis=1)
    bnd = np.stack([gd_b.sum(1), (np.abs(kk) * gd_b).sum(1)], axis=1)
    return val, bnd


def softmax_score_grad(prob, gout, V):
    """Score gradient of the F volume's softmax, g_s = p (g - sum_j p g) / V, and its bound p (|g| + sum_j p |g|) / V.
    prob, gout (B,D,H,W)."""
    prob, gout = np.asarray(prob, np.float64), np.asarray(gout, np.float64)
    dot = (prob * gout).sum(1, keepdims=True)
    adot = (prob * np.abs(gout)).sum(1, keepdims=True)
    return prob * (gout - dot) / V, prob * (np.abs(gout) + adot) / V
