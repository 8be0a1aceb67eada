"""Autograd of the CW volume without a GPU: the ATen port against the reference's frozen backward, a float64 numpy
restatement of the depth gradient against autograd of the port, the gather / scatter contractions of
tests/cw_grad_ref.py (on the CPU here) against a dense all-pairs restatement, the new C export's argument checks and the
Python wrapper's refusal to drop a camera gradient."""
import ctypes as C

import numpy as np
import pytest
import torch

from magnet_b200 import _lib
from magnet_b200._lib import CostArgs
from oracle import torch_ref
from tests.cw_grad_ref import grad_depth_cw
from tests.util import golden_inputs


def _port_grads(inp, gout, dtype=torch.float32):
    dv = inp.depth_volume().to(dtype).clone().requires_grad_(True)
    ref = inp.ref_feat.to(dtype).clone().requires_grad_(True)
    src = inp.nghbr_feat.to(dtype).clone().requires_grad_(True)
    cast = (lambda x: x.to(dtype))
    out = torch_ref.cost_volume_cw(dv, ref, src, cast(inp.ref_gmms), cast(inp.nghbr_gmms), cast(inp.R), cast(inp.t),
                                   inp.is_valid, {k: cast(v) for k, v in inp.cam_intrins.items()}, inp.thres)
    (out * gout.to(out.dtype)).sum().backward()
    return dv.grad, ref.grad, src.grad


def test_torch_port_reproduces_reference_cw_backward():
    z, inp = golden_inputs("cw_train")
    threads = torch.get_num_threads()
    torch.set_num_threads(1)
    try:
        gd, gr, gs = _port_grads(inp, torch.from_numpy(z["gout"]))
    finally:
        torch.set_num_threads(threads)
    assert torch.equal(gr, torch.from_numpy(z["g_ref"]))
    assert torch.equal(gs, torch.from_numpy(z["g_src"]))
    assert torch.equal(gd, torch.from_numpy(z["g_depth"]))


def test_numpy_depth_gradient_matches_autograd_float64():
    from magnet_b200.synthetic import make_inputs
    # wide baseline and depths behind the camera: samples left the image (zero padding) and hit the +-10 clamp
    inp = make_inputs(B=2, V=3, D=6, H=10, W=14, C=8, seed=17, depth="random", invalid=[(0, 1)])
    dv = inp.depth_volume().double().numpy().copy()
    dv[:, 0] = -dv[:, 0]
    dv[:, 1] *= 0.02
    gout = torch.from_numpy(np.random.default_rng(4).standard_normal(dv.shape))
    d_t = torch.from_numpy(dv).requires_grad_(True)
    default = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)                  # the port's temporaries (grid, accumulators) in float64
    try:
        out = torch_ref.cost_volume_cw(d_t, inp.ref_feat.double(), inp.nghbr_feat.double(), inp.ref_gmms.double(),
                                       inp.nghbr_gmms.double(), inp.R.double(), inp.t.double(), inp.is_valid,
                                       {k: v.double() for k, v in inp.cam_intrins.items()}, inp.thres)
    finally:
        torch.set_default_dtype(default)
    (out.double() * gout).sum().backward()
    want = d_t.grad.numpy()
    got, margin, edge, reached = grad_depth_cw(dv, inp.ref_feat.double().numpy(), inp.nghbr_feat.double().numpy(),
                                      inp.nghbr_gmms.double().numpy(), inp.R.double().numpy(), inp.t.double().numpy(),
                                      inp.is_valid.numpy(), inp.cam_intrins['intM'].double().numpy(),
                                      inp.cam_intrins['unit_ray_array_2D'].double().numpy(), inp.thres, gout.numpy())
    # the chosen depths reach the +-10 clamp, taps outside the image (zero padding) and a sample with every tap outside
    assert reached["clamped"] > 0 and reached["tap_outside"] > 0 and reached["all_outside"] > 0, reached
    # elements at a mask flip or on a cell edge (where the bilinear derivative jumps) are excluded
    keep = (margin > 1e-9) & (edge > 1e-9)
    assert keep.mean() > 0.95 and np.abs(want).max() > 0
    scale = np.abs(want).max()
    err = np.abs(got - want)[keep].max() / scale
    assert err < 1e-9, err


def _within(got, want, bound, rel, what):
    err = np.abs(np.asarray(got, np.float64) - np.asarray(want, np.float64))
    bad = err > rel * bound
    assert not bad.any(), (what, int(bad.sum()), float(np.max(err / np.maximum(bound, 1e-300))))
    assert np.abs(want).max() > 0, what


def _f64_autograd(fn, leaves, gout):
    default = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)                  # the port's temporaries (grid, accumulators) in float64
    try:
        out = fn(*leaves)
    finally:
        torch.set_default_dtype(default)
    (out * gout).sum().backward()
    return out.detach().numpy(), [x.grad.numpy() for x in leaves]


@pytest.mark.parametrize("C_", [1, 3, 8, 13])
def test_float64_reference_matches_autograd(C_):
    """tests/cw_grad_ref.Reference with float64 positions against float64 autograd of the ATen port: every output of
    the CW volume (VOLUME and GAUSS depths, consistency on and off) and of the F volume (softmax on and off), within
    1e-12 of each element's bound, after the upstream gradient was zeroed at the (rare) hypotheses that sit on a mask
    flip, a cell edge or z ~ 0.  The inputs reach the +-10 clamp, taps outside the image, samples with every tap
    outside, depths behind the source camera and an invalid view."""
    from magnet_b200.synthetic import make_inputs
    from tests.cw_grad_ref import Reference, cameras_f64, gauss_chain, softmax_score_grad
    inp = make_inputs(B=2, V=3, D=6, H=10, W=14, C=C_, seed=17 + C_, depth="random", invalid=[(0, 1)])
    B, V, H, W = 2, 3, 10, 14
    f64 = {k: v.double() for k, v in inp.cam_intrins.items()}
    R, t = inp.R.double(), inp.t.double()
    cams = cameras_f64(f64['intM'].numpy(), R.numpy(), t.numpy(), inp.is_valid.numpy())
    rays = f64['unit_ray_array_2D'].numpy()
    ref, src, sgmm = inp.ref_feat.double(), inp.nghbr_feat.double(), inp.nghbr_gmms.double()
    rng = np.random.default_rng(C_)
    k = [-40.0, -9.0, -2.0, 0.0, 1.5, 4.0]                  # GAUSS: behind the camera, near z = 0, the clamp
    dv = inp.depth_volume().double().numpy().copy()
    dv[:, 0] = -dv[:, 0]
    dv[:, 1] *= 0.02
    assert int(inp.is_valid.min()) == 0
    for mode in ("volume", "gauss"):
        gmm = inp.ref_gmms.double().numpy()
        depth = dv if mode == "volume" else gmm[:, 0:1] + gmm[:, 1:2] * np.asarray(k).reshape(1, -1, 1, 1)
        for cw in (True, False):
            thres = inp.thres if cw else 1e30
            rf = Reference(depth, ref.numpy(), src.numpy(), sgmm.numpy(), cams, rays, float(thres), pos="f64",
                           consistency=cw)
            amb = rf.ambiguous(1e-9, 1e-9)
            keep = ~amb
            for name in ("clamped", "tap_outside", "all_outside", "behind"):
                assert (rf.reached[name].reshape(amb.shape) & keep).any(), (mode, cw, name)
            assert amb.mean() < 0.05, amb.mean()
            gout = np.where(amb, 0.0, rng.standard_normal(amb.shape))
            want_out, want_b, _, _ = rf.forward()
            g = rf.backward(gout / V)
            lf = [torch.from_numpy(depth).requires_grad_(True) if mode == "volume"
                  else torch.from_numpy(gmm).requires_grad_(True),
                  ref.clone().requires_grad_(True), src.clone().requires_grad_(True)]

            def fn(d_or_gmm, r, s):
                d = d_or_gmm if mode == "volume" else torch.cat([d_or_gmm[:, 0:1] + d_or_gmm[:, 1:2] * kj for kj in k], 1)
                return torch_ref.cost_volume_cw(d, r, s, None, sgmm, R, t, inp.is_valid, f64, thres)
            out, (gd, gr, gs) = _f64_autograd(fn, lf, torch.from_numpy(gout))
            tag = f"{mode} cw={cw}"
            flip = (rf.margin <= 1e-9).reshape(amb.shape)
            _within(np.where(flip, 0, out), np.where(flip, 0, want_out), want_b, 1e-12, tag + " out")
            _within(gr, g["ref"], g["ref_b"], 1e-12, tag + " ref")
            _within(gs, g["src"], g["src_b"], 1e-12, tag + " src")
            if mode == "volume":
                _within(gd, g["d"], g["d_b"], 1e-12, tag + " depth")
            else:
                val, bnd = gauss_chain(g["d"], g["d_b"], k)
                _within(gd, val, bnd, 1e-12, tag + " (mu, sigma)")
    planes = np.array([0.002, 0.05, 0.5, 1.5, 3.0, 8.0])        # the smallest planes reach the clamp
    depth = np.broadcast_to(planes.reshape(1, -1, 1, 1), (B, 6, H, W))
    rf = Reference(depth, ref.numpy(), src.numpy(), None, cams, rays, 0.0, pos="f64", consistency=False)
    for name in ("clamped", "tap_outside", "all_outside"):
        assert rf.reached[name].any(), name
    amb = rf.ambiguous(1e-9, 1e-9)
    score, score_b, _, _ = rf.forward()
    for softmax in (True, False):
        gout = np.where(amb, 0.0, rng.standard_normal(amb.shape))
        out, (gr, gs) = _f64_autograd(
            lambda r, s: torch_ref.cost_volume_f(torch.from_numpy(planes).view(1, -1, 1, 1), r, s, R, t, inp.is_valid,
                                                 f64, apply_softmax=softmax),
            [ref.clone().requires_grad_(True), src.clone().requires_grad_(True)], torch.from_numpy(gout))
        if softmax:
            e = np.exp(score - score.max(1, keepdims=True))
            prob = e / e.sum(1, keepdims=True)
            _within(out, prob, prob * (1 + score_b), 1e-12, "F prob")
            gsc, gsc_b = softmax_score_grad(prob, gout, V)
        else:
            _within(out, score, score_b, 1e-12, "F score")
            gsc, gsc_b = gout / V, np.abs(gout) / V
        g = rf.backward(gsc, gsc_b)
        _within(gr, g["ref"], g["ref_b"], 1e-12, f"F softmax={softmax} ref")
        _within(gs, g["src"], g["src_b"], 1e-12, f"F softmax={softmax} src")


def _dense_reference():
    """tests/cw_grad_ref.Reference with its two contractions restated over all (reference pixel p, source pixel s)
    pairs: the dense matrix <ref_p, src_s> read through each tap's one-hot (chunk, p, s) selector, and the coefficient
    matrix sum_{j,t} coef_t [idx_t = s] applied to the whole maps."""
    from tests.cw_grad_ref import Reference

    def onehot(rf, g, t):
        idx, inb = rf._t(g.idx[t]), rf._t(g.inb[t])
        return torch.zeros(idx.shape + (rf.HW,), dtype=torch.float64).scatter_(2, idx[..., None], inb[..., None].double())

    class Dense(Reference):
        def _taps(self, b, v, g):
            r, s = self.ref[b], self.src[v * self.B + b]
            dot, dabs = torch.einsum("cp,cs->ps", r, s), torch.einsum("cp,cs->ps", r.abs(), s.abs())
            O = {t: onehot(self, g, t) for t in g.idx}
            return ({t: torch.einsum("jps,ps->jp", O[t], dot) for t in O},
                    {t: torch.einsum("jps,ps->jp", O[t], dabs) for t in O})

        def _feature_grads(self, b, v, g, coef, coef_abs, out):
            r, s, i = self.ref[b], self.src[v * self.B + b], v * self.B + b
            M = sum(torch.einsum("jps,jp->ps", onehot(self, g, t), coef[t]) for t in g.idx)
            Ma = sum(torch.einsum("jps,jp->ps", onehot(self, g, t), coef_abs[t]) for t in g.idx)
            out[0][b] += s @ M.T
            out[1][b] += s.abs() @ Ma.T
            out[2][i] += r @ M
            out[3][i] += r.abs() @ Ma
    return Dense


@pytest.mark.parametrize("case", ["c1_cw_direct", "c64_volume_mma_invalid", "planes_softmax_f64"])
def test_gather_contractions_equal_all_pairs(case):
    """The reference's gathers and scatters against the dense all-pairs restatement: forward, backward and camera
    gradients to 1e-12 of each bound, on positions "direct", "mma" and "f64", with consistency on and off."""
    from magnet_b200.synthetic import make_inputs
    from tests.cw_grad_ref import Reference, cameras_f64, softmax_score_grad
    from tests.geom_grad_ref import camera_grads
    C_, pos, kind, invalid = {"c1_cw_direct": (1, "direct", "cw", []),
                              "c64_volume_mma_invalid": (64, "mma", "volume", [(1, 2)]),
                              "planes_softmax_f64": (5, "f64", "planes", [])}[case]
    B, V, D, H, W = 2, 3, 6, 7, 11
    inp = make_inputs(B=B, V=V, D=D, H=H, W=W, C=C_, seed=C_, depth="random", invalid=invalid)
    cams = cameras_f64(inp.cam_intrins['intM'].double().numpy(), inp.R.double().numpy(), inp.t.double().numpy(),
                       inp.is_valid.numpy())
    rays = inp.cam_intrins['unit_ray_array_2D'].numpy()
    if pos != "f64":                                       # the kernels' fp32 camera table and depths
        cams, depth = cams.astype(np.float32), inp.depth_volume().numpy().copy()
        depth[:, 1] *= np.float32(0.02)
    else:
        depth = np.broadcast_to(np.array([0.002, 0.05, 0.5, 1.5, 3.0, 8.0]).reshape(1, -1, 1, 1), (B, D, H, W))
    cw = kind == "cw"
    args = (depth, inp.ref_feat.numpy(), inp.nghbr_feat.numpy(), inp.nghbr_gmms.numpy() if cw else None, cams, rays,
            float(inp.thres))
    chunked = type("Chunked", (Reference,), {"CHUNK": 4 * C_ * H * W})     # hypothesis chunks of 4 and 2
    rfs = [cls(*args, pos=pos, consistency=cw) for cls in (chunked, _dense_reference())]
    assert rfs[0].nj == 4 and rfs[1].nj == D and rfs[0].reached["tap_outside"].any()
    rng = np.random.default_rng(C_)
    gout = rng.standard_normal((B, D, H, W))
    if kind == "planes":
        score = rfs[0].forward()[0]
        e = np.exp(score - score.max(1, keepdims=True))
        gs, gs_abs = softmax_score_grad(e / e.sum(1, keepdims=True), gout, V)
    else:
        gs, gs_abs = gout / V, None
    got, want = [(rf.forward(), rf.backward(gs, gs_abs), camera_grads(rf, depth, cams, rays, gs, gs_abs))
                 for rf in rfs]
    for k, (a, b) in enumerate(zip(got[0][:3], want[0][:3])):
        _within(a, b, want[0][1], 1e-12, f"forward {k}")
    np.testing.assert_array_equal(got[0][3], want[0][3])
    for out in ("ref", "src", "d"):
        _within(got[1][out], want[1][out], want[1][out + "_b"], 1e-12, out)
        _within(got[1][out + "_b"], want[1][out + "_b"], want[1][out + "_b"], 1e-12, out + " bound")
    for out in ("cams", "rays"):
        _within(got[2][out], want[2][out], want[2][out + "_b"], 1e-12, out)
        _within(got[2][out + "_b"], want[2][out + "_b"], want[2][out + "_b"], 1e-12, out + " bound")


def _args(L, *, C_=64, V=2, D=8, layout=_lib.SRC_NCHW, variant=_lib.VARIANT_DIRECT, mode=_lib.DEPTH_VOLUME,
          null=(), softmax=0, consistency=1):
    buf = (C.c_float * 64)()
    p = C.cast(buf, C.c_void_p)
    a = CostArgs()
    a.B, a.V, a.D, a.C, a.H, a.W = 1, V, D, C_, 8, 8
    a.depth_mode, a.src_layout, a.variant, a.softmax, a.consistency = mode, layout, variant, softmax, consistency
    a.rays = a.cams = a.d_volume = a.ref_gmm = a.k_host = p
    bw = _lib.CostBwdArgs()
    bw.fwd = C.pointer(a)
    bw.ref_feat = bw.src_feat = bw.src_gmm = bw.grad_out = bw.workspace = bw.grad_ref = bw.grad_src = bw.grad_depth = p
    for name in null:
        setattr(a if name in ("rays", "cams", "d_volume", "ref_gmm", "k_host") else bw, name, None)
    return L.magnet_cost_volume_bwd_f32(C.byref(bw), None), buf


def test_cw_backward_export_validates_without_gpu():
    L = _lib.lib()
    assert "magnet_cost_volume_bwd_f32" in _lib.EXPORTS and hasattr(L, "magnet_cost_volume_bwd_f32")
    assert L.magnet_cost_volume_bwd_f32(None, None) == _lib.ERR_NULL
    for name in ("ref_feat", "src_feat", "src_gmm", "grad_out", "workspace", "rays", "cams", "d_volume"):
        assert _args(L, null=(name,))[0] == _lib.ERR_NULL, name
    assert _args(L, mode=_lib.DEPTH_GAUSS, null=("k_host",))[0] == _lib.ERR_NULL
    assert _args(L, mode=_lib.DEPTH_GAUSS, null=("ref_gmm",))[0] == _lib.ERR_NULL
    assert _args(L, D=0)[0] == _lib.ERR_SHAPE
    assert _args(L, D=_lib.MAGNET_MAX_PLANES + 1)[0] == _lib.ERR_UNSUPPORTED
    assert _args(L, mode=_lib.DEPTH_PLANES)[0] == _lib.ERR_UNSUPPORTED
    assert _args(L, softmax=1)[0] == _lib.ERR_UNSUPPORTED
    assert _args(L, C_=65)[0] == _lib.ERR_UNSUPPORTED                        # CUDA-core kernel: C <= 64
    assert _args(L, variant=_lib.VARIANT_CELLS)[0] == _lib.ERR_UNSUPPORTED    # no backward reproduces that mask
    assert _args(L, layout=_lib.SRC_PIXC, variant=_lib.VARIANT_TMA)[0] == _lib.ERR_UNSUPPORTED
    assert _args(L, layout=_lib.SRC_SPLIT16, variant=_lib.VARIANT_DIRECT)[0] == _lib.ERR_UNSUPPORTED
    assert _args(L, layout=_lib.SRC_SPLIT16, variant=_lib.VARIANT_MMA, C_=32)[0] == _lib.ERR_UNSUPPORTED
    assert _args(L, layout=_lib.SRC_SPLIT16, variant=_lib.VARIANT_MMA, V=17)[0] == _lib.ERR_UNSUPPORTED


def test_wrapper_raises_on_camera_gradients_without_gpu():
    import magnet_b200
    from magnet_b200.synthetic import make_inputs
    inp = make_inputs(B=1, V=2, D=4, H=6, W=8, C=8, seed=1, depth="smooth")
    dv = inp.depth_volume()
    cases = {"R": (inp.R.clone().requires_grad_(True), inp.t, inp.cam_intrins),
             "t": (inp.R, inp.t.clone().requires_grad_(True), inp.cam_intrins),
             "intM": (inp.R, inp.t, dict(inp.cam_intrins, intM=inp.cam_intrins['intM'].clone().requires_grad_(True)))}
    for name, (R, t, intr) in cases.items():
        with pytest.raises(_lib.MagnetError, match=f"{name} requires grad"):
            magnet_b200.est_costvolume_CW(dv, inp.ref_feat, inp.nghbr_feat, inp.ref_gmms, inp.nghbr_gmms, R, t,
                                          inp.is_valid, intr, inp.thres)
    with pytest.raises(_lib.MagnetError, match="nghbr_poses requires grad"):
        magnet_b200.MatchingPlan(inp.ref_feat, inp.nghbr_feat, inp.nghbr_gmms,
                                 inp.nghbr_poses.clone().requires_grad_(True), inp.is_valid, inp.cam_intrins)
    assert magnet_b200.MagnetHead(dnet_fdim=8).detach_cost is True
