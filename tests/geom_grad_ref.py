"""numpy restatement, in float64, of the camera gradients of both cost volumes (DESIGN §3.11), with the companion bound
(the same sums over the absolute value of every factor), built on the geometry of ``tests/cw_grad_ref.Reference``.

For a valid (b, v), hypothesis j and pixel p, with q = A r_p, P = a + q d, Zp = P2 + 1e-10, u = P0 / Zp, w = P1 / Zp:

    gx = gs m dcost/dix,  gy = gs m dcost/diy   (zero on an axis the +-10 clamp held, and where no tap is inside)
    g_P = (gx / Zp, gy / Zp, -(gx u + gy w) / Zp)
    grad_a[b,v] = sum_{p,j} g_P,   grad_A[b,v] = sum_p (sum_j g_P d_j) r_p^T,   grad_ray[b,:,p] = sum_v A_v^T sum_j g_P d_j

Positions and taps are the Reference's ("f64": the reference's formulas; "direct" / "mma": the kernels' fp32
positions).  P, u, w and Zp are float64 from the camera table and the rays the kernel reads (fp32 values; for "direct"
and "mma" q is the kernels' fma chain).  The bound of each output is the same sum with |.| on every factor, where
|dcost/dix| is bounded by the absolute dot products (plus, on "mma" positions, the position-error term of DESIGN §3.1),
|u| by (|a0| + |q0 d|) / |Zp| (the cancellation in P0) and every term carries the factor 1 + A (the cancellation in Zp,
A the projection amplification of DESIGN §3.1)."""
import numpy as np

from tests.cw_grad_ref import _fma32


def _q(cam, rays, pos):
    A = np.asarray(cam[4:13])
    if pos == "f64":
        return np.asarray(A, np.float64).reshape(3, 3) @ np.asarray(rays, np.float64)
    A32, r = np.asarray(A, np.float32), np.asarray(rays, np.float32)
    return np.stack([_fma32(A32[3 * i + 2], r[2], _fma32(A32[3 * i + 1], r[1], (A32[3 * i] * r[0]).astype(np.float32)))
                     for i in range(3)]).astype(np.float64)


def camera_grads(rf, depth, cams, rays, gs, gs_abs=None, pos_err=None):
    """rf: a cw_grad_ref.Reference; depth (B,D,H,W) the hypothesis depths it was built with (per-pixel, or the plane
    depths broadcast); cams (B*V,16) its camera table; rays (B,3,HW); gs (B,D,H,W) the score gradient (gout / V, or
    the softmax's).  Returns a dict of float64 arrays: cams (B*V,12) = d/dA row-major then d/da, rays (B,3,HW), and
    their bounds cams_b, rays_b (in units of u: tolerance c u bound)."""
    B, D, HW, V, H, W = rf.B, rf.D, rf.HW, rf.V, rf.H, rf.W
    pos_err = rf.pos_err if pos_err is None else pos_err
    gs = np.asarray(gs, np.float64).reshape(B, D, HW)
    gs_abs = np.abs(gs) if gs_abs is None else np.asarray(gs_abs, np.float64).reshape(B, D, HW)
    depth = np.broadcast_to(np.asarray(depth, np.float64), (B, D, H, W)).reshape(B, D, HW)
    gc, gcb = np.zeros((B * V, 12)), np.zeros((B * V, 12))
    gr, grb = np.zeros((B, 3, HW)), np.zeros((B, 3, HW))
    p = np.broadcast_to(np.arange(HW)[None, :], (D, HW))
    for (b, v), g in rf.views.items():
        cam = np.asarray(cams[b * V + v], np.float64)
        a, A = cam[1:4], cam[4:13].reshape(3, 3)
        r = np.asarray(rays[b], np.float64)
        q = _q(cams[b * V + v], rays[b], rf.pos)
        d = depth[b]
        P = a[:, None, None] + q[:, None, :] * d[None]
        Pa = np.abs(a)[:, None, None] + np.abs(q[:, None, :] * d[None])
        dot, dabs = rf._dot(b, v)
        f = {t: np.where(g.inb[t], dot[p, g.idx[t]], 0.0) for t in g.w}
        fa = {t: np.where(g.inb[t], dabs[p, g.idx[t]], 0.0) for t in g.w}
        (wy0, wy1), (wx0, wx1) = g.wy, g.wx
        dcdx = (f[0, 1] - f[0, 0]) * wy0 + (f[1, 1] - f[1, 0]) * wy1
        dcdy = (f[1, 0] - f[0, 0]) * wx0 + (f[1, 1] - f[0, 1]) * wx1
        DX = (fa[0, 1] + fa[0, 0]) * wy0 + (fa[1, 1] + fa[1, 0]) * wy1
        DY = (fa[1, 0] + fa[0, 0]) * wx0 + (fa[1, 1] + fa[0, 1]) * wx1
        if pos_err:
            FA = fa[0, 0] + fa[0, 1] + fa[1, 0] + fa[1, 1]
            DX, DY = DX + FA * g.ey, DY + FA * g.ex
        with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
            Zp = P[2] + 1e-10
            u, w = P[0] / Zp, P[1] / Zp
            clx = ~(np.abs((u - W / 2.0) / (W / 2.0)) <= 10)
            cly = ~(np.abs((w - H / 2.0) / (H / 2.0)) <= 10)
            live = g.m & (gs_abs[b] != 0)
            gm, gma = np.where(live, gs[b], 0.0), np.where(live, gs_abs[b], 0.0)
            gx = np.where(clx | ~live, 0.0, gm * dcdx)
            gy = np.where(cly | ~live, 0.0, gm * dcdy)
            GX = np.where(clx | ~live, 0.0, gma * DX)
            GY = np.where(cly | ~live, 0.0, gma * DY)
            iz = np.where(live, 1.0 / Zp, 0.0)
            aiz = np.where(live, (1.0 + np.minimum(g.amp, 1e30)) / np.abs(Zp), 0.0)
            gP = np.stack([gx * iz, gy * iz, -(gx * u + gy * w) * iz])
            GP = np.stack([GX * aiz, GY * aiz, (GX * Pa[0] + GY * Pa[1]) * aiz / np.abs(Zp)])
            GP = np.where(live[None], GP, 0.0)
        gP = np.where(live[None], gP, 0.0)
        h, hb = (gP * d[None]).sum(1), (GP * np.abs(d)[None]).sum(1)            # (3, HW)
        gc[b * V + v, :9] = (h @ r.T).reshape(-1)
        gc[b * V + v, 9:] = gP.sum((1, 2))
        gcb[b * V + v, :9] = (hb @ np.abs(r).T).reshape(-1)
        gcb[b * V + v, 9:] = GP.sum((1, 2))
        gr[b] += A.T @ h
        grb[b] += np.abs(A).T @ hb
    return dict(cams=gc, cams_b=gcb, rays=gr, rays_b=grb)


def chain(g_cams, intM, R, t):
    """d/dA, d/da (B*V,12) -> (grad_R, grad_t, grad_K) for A = K R, a = K t, in numpy float64."""
    B, V = R.shape[:2]
    g = np.asarray(g_cams, np.float64).reshape(B, V, 12)
    gA, ga = g[..., :9].reshape(B, V, 3, 3), g[..., 9:]
    K = np.asarray(intM, np.float64)[:, None]
    gR = np.swapaxes(K, -1, -2) @ gA
    gt = (np.swapaxes(K, -1, -2) @ ga[..., None])[..., 0]
    gK = (gA @ np.swapaxes(R, -1, -2) + ga[..., :, None] * t[..., None, :]).sum(1)
    return gR, gt, gK
