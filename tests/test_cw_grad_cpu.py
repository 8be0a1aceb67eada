"""Autograd of the CW volume without a GPU: the ATen port against the reference's frozen backward, a float64 numpy
restatement of the depth gradient against autograd of the port, the new C export's argument checks and the Python
wrapper's refusal to drop a camera gradient."""
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
