"""Camera gradients without a GPU: the float64 restatement of tests/geom_grad_ref.py against float64 autograd of the
ATen port (R, t, intM and the rays as leaves), the chain rule of ops.camera_chain, the argument checks and workspace
formula of magnet_cost_volume_geom_bwd_f32, and the geometry_grad() switch."""
import ctypes as C

import numpy as np
import pytest
import torch

import magnet_b200
from magnet_b200 import _lib, ops
from magnet_b200._lib import CostArgs, CostGeomBwdArgs
from magnet_b200.synthetic import make_inputs
from oracle import torch_ref
from tests.cw_grad_ref import Reference, cameras_f64, gauss_depths, softmax_score_grad
from tests.geom_grad_ref import camera_grads, chain


def _f64_port(kind, inp, depth, gout, consistency=True, softmax=True):
    """float64 autograd of the port with the camera tensors as leaves -> (out, grad_R, grad_t, grad_K, grad_rays)."""
    R = inp.R.double().clone().requires_grad_(True)
    t = inp.t.double().clone().requires_grad_(True)
    K = inp.cam_intrins['intM'].double().clone().requires_grad_(True)
    rays = inp.cam_intrins['unit_ray_array_2D'].double().clone().requires_grad_(True)
    intr = {'intM': K, 'unit_ray_array_2D': rays}
    default = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)                  # the port's temporaries (grid, accumulators) in float64
    try:
        if kind == "cw":
            gm = inp.nghbr_gmms.double()
            thres = inp.thres if consistency else 1e30      # kappa = 1e30: every sample with a tap inside is kept
            out = torch_ref.cost_volume_cw(torch.from_numpy(depth), inp.ref_feat.double(), inp.nghbr_feat.double(),
                                           inp.ref_gmms.double(), gm, R, t, inp.is_valid, intr, thres)
        else:
            out = torch_ref.cost_volume_f(torch.from_numpy(depth), inp.ref_feat.double(), inp.nghbr_feat.double(), R, t,
                                          inp.is_valid, intr, apply_softmax=softmax)
    finally:
        torch.set_default_dtype(default)
    (out * torch.from_numpy(gout)).sum().backward()
    return out.detach().numpy(), R.grad.numpy(), t.grad.numpy(), K.grad.numpy(), rays.grad.numpy()


CASES = {
    "cw_volume": dict(kind="cw", mode="volume"),
    "cw_volume_nocw": dict(kind="cw", mode="volume", consistency=False),
    "cw_gauss": dict(kind="cw", mode="gauss", invalid=[(1, 2)]),
    "cw_gauss_nocw": dict(kind="cw", mode="gauss", consistency=False),
    "f_softmax": dict(kind="f", softmax=True),
    "f_scores": dict(kind="f", softmax=False, invalid=[(0, 0)]),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_restatement_matches_float64_autograd(name):
    spec = dict(mode="volume", consistency=True, softmax=True, invalid=[])
    spec.update(CASES[name])
    B, V, D, H, W, Cc = 2, 3, 6, 9, 12, 5
    inp = make_inputs(B=B, V=V, D=D, H=H, W=W, C=Cc, seed=len(name), depth="random", invalid=spec["invalid"])
    rng = np.random.default_rng(len(name))
    if spec["kind"] == "cw":
        if spec["mode"] == "gauss":
            k = np.linspace(-2.0, 2.0, D)
            depth = gauss_depths(inp.ref_gmms.double().numpy(), k, "f64")
        else:
            depth = inp.depth_volume().double().numpy().copy()
            depth[:, 0] *= 0.02                            # samples that leave the image and hit the +-10 clamp
    else:
        depth = np.linspace(0.8, 5.0, D).reshape(1, D, 1, 1)
    gout = rng.standard_normal((B, D, H, W))
    out, gR, gt, gK, grays = _f64_port(spec["kind"], inp, depth, gout, spec["consistency"], spec["softmax"])
    cams = cameras_f64(inp.cam_intrins['intM'].double().numpy(), inp.R.double().numpy(), inp.t.double().numpy(),
                       inp.is_valid.numpy())
    rays = inp.cam_intrins['unit_ray_array_2D'].double().numpy()
    vol = np.broadcast_to(depth, (B, D, H, W))
    cw = spec["kind"] == "cw" and spec["consistency"]
    rf = Reference(vol, inp.ref_feat.double().numpy(), inp.nghbr_feat.double().numpy(),
                   inp.nghbr_gmms.double().numpy() if cw else None, cams, rays, float(inp.thres), pos="f64",
                   consistency=cw)
    if spec["kind"] == "f" and spec["softmax"]:
        gs, _ = softmax_score_grad(out, gout, V)
    else:
        gs = gout / V
    got = camera_grads(rf, vol, cams, rays, gs)
    wR, wt, wK = chain(got["cams"], inp.cam_intrins['intM'].double().numpy(), inp.R.double().numpy(),
                       inp.t.double().numpy())
    for what, a, b in (("R", wR, gR), ("t", wt, gt), ("K", wK, gK), ("rays", got["rays"], grays)):
        scale = max(np.abs(b).max(), 1e-300)
        assert np.abs(a - b).max() <= 1e-12 * scale, (what, np.abs(a - b).max(), scale)
    # the bound covers the value, and the views without a valid flag get nothing
    assert (np.abs(got["cams"]) <= got["cams_b"] * (1 + 1e-12)).all()
    for b_, v_ in spec["invalid"]:
        assert not got["cams"][b_ * V + v_].any()
    assert np.abs(gR).max() > 0 and np.abs(grays).max() > 0


def test_camera_chain_matches_float64_autograd():
    rng = np.random.default_rng(5)
    B, V = 2, 3
    K = torch.from_numpy(rng.standard_normal((B, 3, 3))).requires_grad_(True)
    R = torch.from_numpy(rng.standard_normal((B, V, 3, 3))).requires_grad_(True)
    t = torch.from_numpy(rng.standard_normal((B, V, 3))).requires_grad_(True)
    A = K.unsqueeze(1) @ R
    a = (K.unsqueeze(1) @ t.unsqueeze(-1)).squeeze(-1)
    g = torch.from_numpy(rng.standard_normal((B * V, 12)))
    (A.reshape(B * V, 9) * g[:, :9]).sum().add((a.reshape(B * V, 3) * g[:, 9:]).sum()).backward()
    gR, gt, gK = ops.camera_chain(g, K.detach(), R.detach(), t.detach())
    for got, want in ((gR, R.grad), (gt, t.grad), (gK, K.grad)):
        assert torch.allclose(got, want, rtol=1e-13, atol=1e-13)
    nR, nt, nK = chain(g.numpy(), K.detach().numpy(), R.detach().numpy(), t.detach().numpy())
    assert np.allclose(nR, R.grad.numpy(), rtol=1e-13, atol=1e-13) and np.allclose(nK, K.grad.numpy(), rtol=1e-13, atol=1e-13)


# ---------------------------------------------------------------------------------------------------------------------
# C ABI: argument checks happen before any CUDA call, so they run without a device.

def test_geom_workspace_formula():
    L = _lib.lib()
    for B, V, H, W in ((1, 1, 1, 1), (8, 4, 120, 160), (4, 4, 88, 304), (3, 5, 7, 33)):
        assert L.magnet_cost_geom_workspace_bytes(B, V, H, W) == B * V * 12 * ((H * W + 31) // 32) * 4
    for bad in ((0, 1, 1, 1), (1, 0, 1, 1), (1, 1, 0, 1), (1, 1, 1, -2)):
        assert L.magnet_cost_geom_workspace_bytes(*bad) == 0


def _args(**over):
    one = 0x1000
    a = CostArgs()
    a.B, a.V, a.D, a.C, a.H, a.W = 1, 2, 8, 16, 6, 7
    a.depth_mode, a.src_layout, a.consistency, a.softmax, a.variant, a.kappa = (
        _lib.DEPTH_VOLUME, _lib.SRC_NCHW, 1, 0, _lib.VARIANT_DIRECT, 5.0)
    a.ref_feat = a.src_feat = a.src_gmm = a.rays = a.cams = a.d_volume = a.ref_gmm = a.out = one
    karr = (C.c_float * 8)(*range(8))
    a.k_host = C.cast(karr, C.c_void_p)
    b = CostGeomBwdArgs()
    b.ref_feat = b.src_feat = b.src_gmm = b.grad_out = b.prob = b.score = b.grad_cams = b.grad_rays = one
    b.workspace = one
    for k, v in over.items():
        setattr(a if hasattr(a, k) and k not in ("ref_feat", "src_feat", "src_gmm") else b, k, v)
    b.fwd = C.pointer(a)
    return a, b, karr


@pytest.mark.parametrize("over,status", [
    (dict(B=0), _lib.ERR_SHAPE),
    (dict(H=-1), _lib.ERR_SHAPE),
    (dict(D=257), _lib.ERR_UNSUPPORTED),
    (dict(C=65), _lib.ERR_UNSUPPORTED),
    (dict(rays=None), _lib.ERR_NULL),
    (dict(cams=None), _lib.ERR_NULL),
    (dict(ref_feat=None), _lib.ERR_NULL),
    (dict(src_feat=None), _lib.ERR_NULL),
    (dict(grad_out=None), _lib.ERR_NULL),
    (dict(score=None), _lib.ERR_NULL),
    (dict(workspace=None), _lib.ERR_NULL),
    (dict(grad_cams=None), _lib.ERR_NULL),
    (dict(d_volume=None), _lib.ERR_NULL),
    (dict(src_gmm=None), _lib.ERR_NULL),
    (dict(depth_mode=7), _lib.ERR_UNSUPPORTED),
    (dict(softmax=1), _lib.ERR_UNSUPPORTED),                      # a CW volume has no softmax
    (dict(variant=_lib.VARIANT_CELLS), _lib.ERR_UNSUPPORTED),     # the tap-sharing kernels' masks are not reproduced
    (dict(variant=_lib.VARIANT_TMA, src_layout=_lib.SRC_PIXC), _lib.ERR_UNSUPPORTED),
    (dict(variant=_lib.VARIANT_AUTO), _lib.ERR_UNSUPPORTED),     # NCHW forward with AUTO: not the DIRECT kernel
    (dict(src_layout=_lib.SRC_SPLIT16, variant=_lib.VARIANT_MMA), _lib.ERR_UNSUPPORTED),   # needs C == 64
    (dict(workspace=0x1004), _lib.ERR_ALIGN),
    # the F volume
    (dict(depth_mode=_lib.DEPTH_PLANES, consistency=1), _lib.ERR_UNSUPPORTED),
    (dict(depth_mode=_lib.DEPTH_PLANES, consistency=0, grad_depth=0x1000), _lib.ERR_UNSUPPORTED),
    (dict(depth_mode=_lib.DEPTH_PLANES, consistency=0, softmax=1, prob=None), _lib.ERR_NULL),
    (dict(depth_mode=_lib.DEPTH_PLANES, consistency=0, k_host=None), _lib.ERR_NULL),
    (dict(depth_mode=_lib.DEPTH_GAUSS, ref_gmm=None), _lib.ERR_NULL),
])
def test_geom_bwd_rejects_bad_arguments(over, status):
    a, b, karr = _args(**over)
    assert _lib.lib().magnet_cost_volume_geom_bwd_f32(C.byref(b), None) == status
    assert _lib.lib().magnet_cost_volume_geom_bwd_f32(None, None) == _lib.ERR_NULL


def test_geom_bwd_exported():
    assert "magnet_cost_volume_geom_bwd_f32" in _lib.EXPORTS and "magnet_cost_geom_workspace_bytes" in _lib.EXPORTS
    assert _lib.lib().magnet_abi_version() == 4


# ---------------------------------------------------------------------------------------------------------------------
# The switch

def _cpu_inputs():
    inp = make_inputs(B=1, V=2, D=4, H=5, W=6, C=4, seed=1)
    return inp


def test_switch_off_keeps_the_refusals():
    inp = _cpu_inputs()
    poses = inp.nghbr_poses.clone().requires_grad_(True)
    assert not magnet_b200.homography.geometry_grad_enabled()
    with pytest.raises(_lib.MagnetError, match="nghbr_poses requires grad"):
        magnet_b200.MatchingPlan(inp.ref_feat, inp.nghbr_feat, inp.nghbr_gmms, poses, inp.is_valid, inp.cam_intrins)
    with pytest.raises(_lib.MagnetError, match="R requires grad"):
        magnet_b200.est_costvolume_CW(inp.depth_volume(), inp.ref_feat, inp.nghbr_feat, inp.ref_gmms, inp.nghbr_gmms,
                                      poses[:, :, :3, :3], poses[:, :, :3, 3], inp.is_valid, inp.cam_intrins, inp.thres)
    with magnet_b200.geometry_grad():
        assert magnet_b200.homography.geometry_grad_enabled()
        with magnet_b200.geometry_grad(False):
            assert not magnet_b200.homography.geometry_grad_enabled()
        assert magnet_b200.homography.geometry_grad_enabled()
    assert not magnet_b200.homography.geometry_grad_enabled()


def test_switch_restored_after_an_exception():
    with pytest.raises(KeyError):
        with magnet_b200.geometry_grad():
            raise KeyError("x")
    assert not magnet_b200.homography.geometry_grad_enabled()


def test_switch_refuses_a_d_center_that_requires_grad():
    inp = _cpu_inputs()
    dc = torch.linspace(1.0, 4.0, 4).view(1, -1, 1, 1).requires_grad_(True)
    with magnet_b200.geometry_grad(), pytest.raises(_lib.MagnetError, match="d_center requires grad"):
        magnet_b200.est_costvolume_F(dc, inp.ref_feat, inp.nghbr_feat, inp.R, inp.t, inp.is_valid, inp.cam_intrins)
