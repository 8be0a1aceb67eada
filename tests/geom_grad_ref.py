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
import torch

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
    their bounds cams_b, rays_b (in units of u: tolerance c u bound).  Computed in torch float64 on rf's device, over
    rf's hypothesis chunks, from its gathered tap dot products."""
    B, D, HW, V, H, W, T = rf.B, rf.D, rf.HW, rf.V, rf.H, rf.W, rf._t
    pos_err = rf.pos_err if pos_err is None else pos_err
    gs = np.asarray(gs, np.float64).reshape(B, D, HW)
    gs_abs = T(np.abs(gs) if gs_abs is None else np.asarray(gs_abs, np.float64).reshape(B, D, HW))
    gs = T(gs)
    depth = np.broadcast_to(np.asarray(depth, np.float64), (B, D, H, W)).reshape(B, D, HW)
    z = lambda *s: torch.zeros(s, dtype=torch.float64, device=rf.dev)
    gc, gcb, gr, grb = z(B * V, 12), z(B * V, 12), z(B, 3, HW), z(B, 3, HW)
    for b, v, j0, j1, g in rf._chunks():
        cam = np.asarray(cams[b * V + v], np.float64)
        a, A = T(cam[1:4]), T(cam[4:13].reshape(3, 3))
        r = T(np.asarray(rays[b], np.float64))
        q = T(_q(cams[b * V + v], rays[b], rf.pos))
        d = T(depth[b, j0:j1])
        P = a[:, None, None] + q[:, None, :] * d[None]
        Pa = a.abs()[:, None, None] + (q[:, None, :] * d[None]).abs()
        f, fa = rf._taps(b, v, g)
        (wy0, wy1), (wx0, wx1) = map(T, g.wy), map(T, g.wx)
        dcdx = (f[0, 1] - f[0, 0]) * wy0 + (f[1, 1] - f[1, 0]) * wy1
        dcdy = (f[1, 0] - f[0, 0]) * wx0 + (f[1, 1] - f[0, 1]) * wx1
        DX = (fa[0, 1] + fa[0, 0]) * wy0 + (fa[1, 1] + fa[1, 0]) * wy1
        DY = (fa[1, 0] + fa[0, 0]) * wx0 + (fa[1, 1] + fa[0, 1]) * wx1
        if pos_err:
            FA = fa[0, 0] + fa[0, 1] + fa[1, 0] + fa[1, 1]
            DX, DY = DX + FA * T(g.ey), DY + FA * T(g.ex)
        Zp = P[2] + 1e-10
        u, w = P[0] / Zp, P[1] / Zp
        clx = ~(((u - W / 2.0) / (W / 2.0)).abs() <= 10)
        cly = ~(((w - H / 2.0) / (H / 2.0)).abs() <= 10)
        live = T(g.m) & (gs_abs[b, j0:j1] != 0)
        gm, gma = torch.where(live, gs[b, j0:j1], 0.0), torch.where(live, gs_abs[b, j0:j1], 0.0)
        gx = torch.where(clx | ~live, 0.0, gm * dcdx)
        gy = torch.where(cly | ~live, 0.0, gm * dcdy)
        GX = torch.where(clx | ~live, 0.0, gma * DX)
        GY = torch.where(cly | ~live, 0.0, gma * DY)
        iz = torch.where(live, 1.0 / Zp, 0.0)
        aiz = torch.where(live, (1.0 + T(np.minimum(g.amp, 1e30))) / Zp.abs(), 0.0)
        gP = torch.where(live[None], torch.stack([gx * iz, gy * iz, -(gx * u + gy * w) * iz]), 0.0)
        GP = torch.where(live[None], torch.stack([GX * aiz, GY * aiz, (GX * Pa[0] + GY * Pa[1]) * aiz / Zp.abs()]),
                         0.0)
        h, hb = (gP * d[None]).sum(1), (GP * d.abs()[None]).sum(1)            # (3, HW)
        gc[b * V + v, :9] += (h @ r.T).reshape(-1)
        gc[b * V + v, 9:] += gP.sum((1, 2))
        gcb[b * V + v, :9] += (hb @ r.abs().T).reshape(-1)
        gcb[b * V + v, 9:] += GP.sum((1, 2))
        gr[b] += A.T @ h
        grb[b] += A.abs().T @ hb
    return {k: x.cpu().numpy() for k, x in dict(cams=gc, cams_b=gcb, rays=gr, rays_b=grb).items()}


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
