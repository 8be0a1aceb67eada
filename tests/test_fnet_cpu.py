"""F-Net training without a GPU: the ATen port against the reference's frozen training step (tests/golden/fnet_train.npz),
a numpy restatement of the tensor-core volume backward (csrc/cost_f_bwd_mma.cu) against autograd, and the C ABI of the
F-Net entry points (argument validation only)."""
import ctypes as C

import numpy as np
import pytest
import torch

from magnet_b200 import _lib
from magnet_b200._lib import CostArgs
from oracle import torch_ref
from tests.fnet_ref import FNET_MAX_DEPTH, FNET_MIN_DEPTH, fnet_l1_loss
from tests.test_split16_numerics import split16
from tests.util import golden_inputs


def test_torch_port_reproduces_reference_fnet_step():
    """est_costvolume_F -> train_FNet.py loss -> backward, ATen port vs the reference's own step, bit for bit."""
    z, inp = golden_inputs("fnet_train")
    threads = torch.get_num_threads()
    torch.set_num_threads(1)          # as the fixture was made: the softmax reduces in a thread-count dependent order
    try:
        d_center = torch.from_numpy(z["planes"]).view(1, -1, 1, 1)
        ref, src = inp.ref_feat.clone().requires_grad_(True), inp.nghbr_feat.clone().requires_grad_(True)
        vol = torch_ref.cost_volume_f(d_center, ref, src, inp.R, inp.t, inp.is_valid, inp.cam_intrins)
        loss = fnet_l1_loss(vol, d_center, torch.from_numpy(z["gt_dmap"]), FNET_MIN_DEPTH, FNET_MAX_DEPTH)
        loss.backward()
    finally:
        torch.set_num_threads(threads)
    assert np.float32(loss.item()) == z["loss"]
    assert np.array_equal(ref.grad.numpy(), z["g_ref"]) and np.array_equal(src.grad.numpy(), z["g_src"])
    assert (z["gt_dmap"] > FNET_MAX_DEPTH).any() and (z["gt_dmap"] == 0).any()
    assert not inp.is_valid.all() and float(z["planes"][0]) < 0.02


# ---------------------------------------------------------------------------------------------------------------
# numpy restatement of the tensor-core backward (DESIGN §3.4)
# ---------------------------------------------------------------------------------------------------------------
BSEG = 16                             # 8-cell segments per sub-window


def _item_scale(bound):
    """Power of two that maps the item's bound max_p sum_j |g| into [2^14, 2^15) (1 for 0)."""
    if bound == 0 or not np.isfinite(bound):
        return 1.0
    e = int(np.floor(np.log2(bound)))
    return float(2.0 ** max(-100, min(100, 14 - e)))


def _split(x, s):
    v = (np.asarray(x, np.float64) * s).astype(np.float32)
    hi = v.astype(np.float16)
    lo = (v - hi.astype(np.float32)).astype(np.float16)
    return hi.astype(np.float64), lo.astype(np.float64)


def mma_backward(ref, src, g, planes, K, R, t, valid, rays):
    """ref (B,64,H,W), src (V*B,64,H,W), g (B,D,H,W) = dL/dscore / V.  Returns (g_ref, g_src) as the kernel forms them:
    per (batch element, 8x8 tile) the coefficient matrix Gc of each view and sub-window, one scale per item, fp16 hi/lo
    operands, three products (no lo*lo), exact accumulation."""
    B, Cc, H, W = ref.shape
    V = src.shape[0] // B
    D = len(planes)
    rh, rl, sr = split16(ref)
    sh, sl, ss = split16(src)
    rh, rl, sh, sl = (a.astype(np.float64) for a in (rh, rl, sh, sl))
    g_ref = np.zeros((B, Cc, H, W))
    g_src = np.zeros((V * B, Cc, H, W))
    nsplit = 0
    for b in range(B):
        for ty0 in range(0, H, 8):
            for tx0 in range(0, W, 8):
                ys, xs = np.meshgrid(np.arange(ty0, ty0 + 8), np.arange(tx0, tx0 + 8), indexing="ij")
                ys, xs = ys.reshape(-1), xs.reshape(-1)
                live = (ys < H) & (xs < W)
                n = np.minimum(ys, H - 1) * W + np.minimum(xs, W - 1)
                gp = np.where(live[:, None], g[b].reshape(D, -1)[:, n].T, 0.0)              # (64, D)
                s_g = _item_scale(np.abs(gp).sum(1).max())
                acc1 = np.zeros((64, Cc))
                for v in range(V):
                    if valid[b, v] != 1:
                        continue
                    a = K[b] @ t[b, v]
                    q = (K[b] @ R[b, v]) @ rays[b][:, n]                                      # (3, 64)
                    P = a[:, None, None] + q[:, :, None] * planes[None, None, :]             # (3, 64, D)
                    ix = P[0] / (P[2] + 1e-10) - 0.5
                    iy = P[1] / (P[2] + 1e-10) - 0.5
                    ix = np.clip(np.nan_to_num(ix, nan=-2.0), -2.0, W + 1.0)
                    iy = np.clip(np.nan_to_num(iy, nan=-2.0), -2.0, H + 1.0)
                    x0, y0 = np.floor(ix).astype(int), np.floor(iy).astype(int)
                    use = live[:, None] & (gp != 0) & (x0 >= -1) & (x0 < W) & (y0 >= -1) & (y0 < H)
                    if not use.any():
                        continue
                    wx0, wx1, wy0, wy1 = x0[use].min(), x0[use].max(), y0[use].min(), y0[use].max()
                    nseg_all, rows_all = (wx1 - wx0 + 2 + 7) >> 3, wy1 - wy0 + 2
                    nsw = min(nseg_all, BSEG // 2)
                    rmax = rows_all if nseg_all * rows_all <= BSEG else max(2, BSEG // nsw)
                    stepx, stepy = 8 * nsw - 1, rmax - 1
                    sxi_all, syi_all = (x0 - wx0) // stepx, (y0 - wy0) // stepy
                    for syi in range((wy1 - wy0) // stepy + 1):
                        for sxi in range((wx1 - wx0) // stepx + 1):
                            sel = use & (sxi_all == sxi) & (syi_all == syi)
                            if not sel.any():
                                continue
                            nsplit += 1
                            sx, sy = wx0 + sxi * stepx, wy0 + syi * stepy
                            rows = min(stepy, wy1 - sy + 1) + 1
                            nseg = (min(stepx, wx1 - sx + 1) + 1 + 7) >> 3
                            pitch = nseg * 8
                            assert nseg * rows <= BSEG
                            gc = np.zeros((64, rows * pitch), np.float32)                  # fp32, like red.shared.add
                            pi, ji = np.nonzero(sel)
                            fx = (ix[pi, ji] - x0[pi, ji]).astype(np.float32)
                            fy = (iy[pi, ji] - y0[pi, ji]).astype(np.float32)
                            li = (y0[pi, ji] - sy) * pitch + (x0[pi, ji] - sx)
                            gg = gp[pi, ji].astype(np.float32)
                            for off, w in ((0, (1 - fx) * (1 - fy)), (1, fx * (1 - fy)), (pitch, (1 - fx) * fy),
                                           (pitch + 1, fx * fy)):
                                np.add.at(gc, (pi, li + off), gg * w)
                            assert np.abs(gc).sum(1).max() <= np.abs(gp).sum(1).max() * (1 + 1e-5)
                            gh, gl = _split(gc, s_g)
                            cy = sy + np.arange(rows * pitch) // pitch
                            cx = sx + np.arange(rows * pitch) % pitch
                            inside = (cx >= 0) & (cx < W) & (cy >= 0) & (cy < H)
                            cn = np.clip(cy, 0, H - 1) * W + np.clip(cx, 0, W - 1)
                            vb = v * B + b
                            Sh = np.where(inside[:, None], sh[vb].reshape(Cc, -1)[:, cn].T, 0.0)   # zero fill (TMA)
                            Sl = np.where(inside[:, None], sl[vb].reshape(Cc, -1)[:, cn].T, 0.0)
                            acc1 += gl @ Sh + gh @ Sl + gh @ Sh                                     # GEMM 1
                            Rh = np.where(live[:, None], rh[b].reshape(Cc, -1)[:, n].T, 0.0)
                            Rl = np.where(live[:, None], rl[b].reshape(Cc, -1)[:, n].T, 0.0)
                            acc2 = (gl.T @ Rh + gh.T @ Rl + gh.T @ Rh) / (s_g * sr)                # GEMM 2
                            for k in np.nonzero(inside)[0]:
                                g_src[vb, :, cy[k], cx[k]] += acc2[k]
                for k in np.nonzero(live)[0]:
                    g_ref[b, :, ys[k], xs[k]] = acc1[k] / (s_g * ss)
    return g_ref, g_src, nsplit


def test_numpy_restatement_of_tensor_core_backward_matches_autograd():
    from magnet_b200.synthetic import make_inputs
    inp = make_inputs(B=1, V=2, D=8, H=12, W=20, C=64, seed=91, depth="smooth")
    planes = np.asarray(torch_ref_planes(), np.float32)
    D = len(planes)
    rng = np.random.default_rng(5)
    gout = (rng.standard_normal((1, D, 12, 20)) * 10.0 ** rng.uniform(-3, 3, (1, D, 12, 20))).astype(np.float32)
    ref, src = inp.ref_feat.clone().double().requires_grad_(True), inp.nghbr_feat.clone().double().requires_grad_(True)
    d_center = torch.from_numpy(planes).double().view(1, -1, 1, 1)
    cam = {k: v.double() for k, v in inp.cam_intrins.items()}
    dtype = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)           # the port's temporaries (sampling grid, sums) in fp64 too
    try:
        scores = torch_ref.cost_volume_f(d_center, ref, src, inp.R.double(), inp.t.double(), inp.is_valid, cam,
                                         apply_softmax=False)
        (scores * torch.from_numpy(gout).double()).sum().backward()
    finally:
        torch.set_default_dtype(dtype)
    got_ref, got_src, nsplit = mma_backward(inp.ref_feat.numpy(), inp.nghbr_feat.numpy(), gout / 2.0, planes,
                                            inp.cam_intrins['intM'].numpy().astype(np.float64), inp.R.numpy().astype(np.float64),
                                            inp.t.numpy().astype(np.float64), inp.is_valid.numpy(),
                                            inp.cam_intrins['unit_ray_array_2D'].numpy().astype(np.float64))
    assert nsplit > 6 * 2                              # at least one (tile, view) was cut into sub-windows
    for got, want in ((got_ref, ref.grad.numpy()), (got_src, src.grad.numpy())):
        assert np.abs(got - want).max() <= 1e-5 * np.abs(want).max()


def torch_ref_planes():
    """80 SID planes from 1e-3 (the F-Net training distribution)."""
    from tests.fnet_ref import sid_centres
    return sid_centres(1e-3, 10.0, 80).reshape(-1).numpy()


# ---------------------------------------------------------------------------------------------------------------
# C ABI v4
# ---------------------------------------------------------------------------------------------------------------
def test_fnet_entry_points_validate_without_gpu():
    L = _lib.lib()
    assert L.magnet_abi_version() == _lib.MAGNET_ABI_VERSION == 4
    for name in ("magnet_fnet_l1_partials", "magnet_fnet_l1_fwd_f32", "magnet_fnet_l1_bwd_f32"):
        assert name in _lib.EXPORTS and hasattr(L, name)
    assert L.magnet_fnet_l1_partials(2, 120, 160) == 2 * 150
    assert L.magnet_fnet_l1_partials(0, 120, 160) == _lib.ERR_SHAPE
    buf = (C.c_float * 64)()
    p = C.cast(buf, C.c_void_p)
    assert L.magnet_fnet_l1_fwd_f32(None, p, p, p, 1, 8, 4, 4, p, None) == _lib.ERR_NULL
    assert L.magnet_fnet_l1_fwd_f32(p, p, p, p, 1, 8, 4, 4, None, None) == _lib.ERR_NULL
    assert L.magnet_fnet_l1_fwd_f32(p, p, p, p, 1, 0, 4, 4, p, None) == _lib.ERR_SHAPE
    assert L.magnet_fnet_l1_fwd_f32(p, p, p, p, 1, _lib.MAGNET_MAX_PLANES + 1, 4, 4, p, None) == _lib.ERR_UNSUPPORTED
    assert L.magnet_fnet_l1_bwd_f32(p, None, p, p, 1.0, None, 1, 8, 4, 4, p, None) == _lib.ERR_NULL
    assert L.magnet_fnet_l1_bwd_f32(p, p, p, p, 1.0, None, 1, 8, -4, 4, p, None) == _lib.ERR_SHAPE


def _bwd_args(L, C_, V, D, layout=_lib.SRC_SPLIT16, variant=_lib.VARIANT_AUTO):
    buf = (C.c_float * 64)()
    p = C.cast(buf, C.c_void_p)
    a = CostArgs()
    a.B, a.V, a.D, a.C, a.H, a.W = 1, V, D, C_, 8, 8
    a.depth_mode, a.src_layout, a.variant = _lib.DEPTH_PLANES, layout, variant
    a.ref_feat = a.src_feat = a.rays = a.cams = a.k_host = p
    bw = _lib.CostFBwdArgs()
    bw.fwd = C.pointer(a)
    bw.grad_out = bw.workspace = bw.grad_ref = bw.grad_src = p
    return L.magnet_cost_volume_f_bwd_f32(C.byref(bw), None), buf


def test_split16_volume_backward_validation_without_gpu():
    L = _lib.lib()
    assert _bwd_args(L, 32, 2, 80)[0] == _lib.ERR_UNSUPPORTED                   # tensor-core backward: C == 64 only
    assert _bwd_args(L, 64, 17, 80)[0] == _lib.ERR_UNSUPPORTED                  # V <= 16
    assert _bwd_args(L, 64, 2, _lib.MAGNET_MAX_PLANES + 1)[0] == _lib.ERR_UNSUPPORTED
    assert _bwd_args(L, 64, 2, 80, variant=_lib.VARIANT_CELLS)[0] == _lib.ERR_UNSUPPORTED
    assert _bwd_args(L, 64, 2, 80, layout=_lib.SRC_PIXC)[0] == _lib.ERR_UNSUPPORTED   # NCHW or SPLIT16 only
    assert _bwd_args(L, 12, 2, 80, layout=_lib.SRC_NCHW)[0] == _lib.ERR_UNSUPPORTED   # CUDA-core kernel: C in {8,...,64}


def test_fnet_python_entry_points_without_gpu():
    import magnet_b200
    from magnet_b200 import ops
    d = magnet_b200.sid_planes(1e-3, 10.0)
    assert d.shape == (1, 80, 1, 1) and d.dtype == torch.float32
    from tests.fnet_ref import sid_centres
    assert torch.equal(d, sid_centres(1e-3, 10.0, 80))
    with pytest.raises(_lib.MagnetError):
        ops.fnet_l1_loss(torch.zeros(1, 4, 2, 2), [1.0, 2.0, 3.0, 4.0], torch.zeros(1, 1, 2, 2), torch.ones(1, 1, 2, 2))
    with pytest.raises(_lib.MagnetError):           # empty mask, rejected before any launch
        ops.fnet_l1_loss(torch.zeros(1, 4, 2, 2), [1.0, 2.0, 3.0, 4.0], torch.zeros(1, 1, 2, 2), torch.zeros(1, 1, 2, 2))
    m = magnet_b200.MagnetF(torch.nn.Conv2d(3, 64, 1))
    assert set(m.state_dict()) == {"f_net.weight", "f_net.bias"}
