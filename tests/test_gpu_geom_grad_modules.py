"""Camera gradients through the public entry points and modules under geometry_grad(), against the reference's data flow
on the ATen port (autograd, independent of the kernels): at full size (cfg2 / cfg3, both depth modes), through
MagnetF.loss and MagnetHead(detach_cost=False), and the pose refinement of examples/refine_pose.py.

The full-size comparison is norm-wise: |got - want| <= 1e-4 |want| per tensor (Frobenius; about 1.5e-5 on an H100);
element-wise agreement is
gated in test_gpu_geom_grad.py.  The upstream gradient is zeroed where cw_threshold_margin <= 1e-3 (a mask flip) and
where a sample lies within 1e-3 px of a cell edge, where dcost/dix jumps: without the latter, the few samples per
hundred thousand whose fp32 and float64 positions straddle an edge move the sums by up to 1e-2 (measured at cfg3)."""
import importlib.util
import os

import numpy as np
import pytest
import torch

import magnet_b200
from magnet_b200.synthetic import make_inputs
from oracle import torch_ref
from tests.fnet_ref import fnet_l1_loss

pytestmark = pytest.mark.gpu

CFGS = {"cfg2": dict(B=8, V=4, H=120, W=160, family="scannet"), "cfg3": dict(B=4, V=4, H=88, W=304, family="kitti")}


def _norm_close(got, want, rel, what):
    got, want = got.detach().double().cpu(), want.detach().double().cpu()
    ratio = float((got - want).norm() / want.norm())
    print(f"{what}: |got - want| / |want| = {ratio:.3g}")
    assert float(want.norm()) > 0 and ratio <= rel, (what, ratio)


def _leaves(inp, dev):
    return (inp.nghbr_poses.to(dev).clone().requires_grad_(True), inp.cam_intrins['intM'].clone().requires_grad_(True),
            inp.cam_intrins['unit_ray_array_2D'].clone().requires_grad_(True))


def _edge_distance(dvol, g, inp, dev):
    """(B,D,H,W) float64: distance of every sample position (ix, iy) = P / P2 - 0.5 to the nearest cell edge, minimised
    over the valid views.  At an edge dcost/dix jumps, so an fp32 position on the other side of it changes the term."""
    B, D, H, W = dvol.shape
    V = g.nghbr_poses.shape[1]
    out = torch.full((B, D, H * W), float("inf"), dtype=torch.float64, device=dev)
    for b in range(B):
        K = inp.cam_intrins['intM'][b].double().to(dev)
        rays = inp.cam_intrins['unit_ray_array_2D'][b].double().to(dev)
        for v in range(V):
            if int(inp.is_valid[b, v]) != 1:
                continue
            R, t = g.nghbr_poses[b, v, :3, :3].double(), g.nghbr_poses[b, v, :3, 3].double()
            P = (K @ t)[:, None, None] + (K @ R @ rays)[:, None, :] * dvol[b].reshape(1, D, -1)
            ix, iy = P[0] / P[2] - 0.5, P[1] / P[2] - 0.5
            e = torch.minimum((ix - ix.round()).abs(), (iy - iy.round()).abs())
            out[b] = torch.minimum(out[b], torch.nan_to_num(e, nan=0.0))
    return out.reshape(B, D, H, W)


@pytest.mark.parametrize("mode", ["volume", "gauss"])
@pytest.mark.parametrize("cfg", sorted(CFGS))
def test_full_size_public_api_against_float64_port(cfg, mode, cuda):
    sh = CFGS[cfg]
    B, V, H, W, D = sh["B"], sh["V"], sh["H"], sh["W"], 64
    inp = make_inputs(B=B, V=V, D=D, H=H, W=W, C=64, seed=31, family=sh["family"])
    g = inp.to(cuda)
    k = inp.k.tolist()
    dvol = torch_ref.sample_depth_candidates(g.ref_gmms.double(), k)            # float64 hypotheses
    # the upstream gradient, zeroed near a mask flip
    margin = torch_ref.cw_threshold_margin(dvol.float(), g.nghbr_gmms, g.R, g.t, inp.is_valid,
                                           {kk: v.to(cuda) for kk, v in inp.cam_intrins.items()}, inp.thres)
    gout = torch.randn(B, D, H, W, device=cuda, generator=torch.Generator(cuda).manual_seed(1))
    gout = torch.where((margin <= 1e-3) | (_edge_distance(dvol, g, inp, cuda) <= 1e-3), torch.zeros_like(gout), gout)
    # public API
    poses, intM, rays = _leaves(inp, cuda)
    intr = {'intM': intM, 'unit_ray_array_2D': rays}
    with magnet_b200.geometry_grad():
        if mode == "volume":
            out = magnet_b200.est_costvolume_CW(dvol.float(), g.ref_feat, g.nghbr_feat, g.ref_gmms, g.nghbr_gmms,
                                                poses[:, :, :3, :3], poses[:, :, :3, 3], inp.is_valid, intr, inp.thres)
        else:
            plan = magnet_b200.MatchingPlan(g.ref_feat, g.nghbr_feat, g.nghbr_gmms, poses, inp.is_valid, intr,
                                            thres=inp.thres)
            out = plan.cost(g.ref_gmms, k)
    (out * gout).sum().backward()
    # float64 autograd of the port, one batch element at a time (its D-fold repeats are large)
    wp = torch.zeros(B, V, 4, 4, dtype=torch.float64, device=cuda)
    wK = torch.zeros(B, 3, 3, dtype=torch.float64)
    wr = torch.zeros(B, 3, H * W, dtype=torch.float64)
    default = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        for b in range(B):
            src_idx = [v * B + b for v in range(V)]
            p = inp.nghbr_poses[b:b + 1].to(cuda).double().requires_grad_(True)
            K = inp.cam_intrins['intM'][b:b + 1].double().to(cuda).requires_grad_(True)
            r = inp.cam_intrins['unit_ray_array_2D'][b:b + 1].double().to(cuda).requires_grad_(True)
            o = torch_ref.cost_volume_cw(dvol[b:b + 1], g.ref_feat[b:b + 1].double(), g.nghbr_feat[src_idx].double(),
                                         None, g.nghbr_gmms[src_idx].double(), p[:, :, :3, :3], p[:, :, :3, 3],
                                         inp.is_valid[b:b + 1], {'intM': K, 'unit_ray_array_2D': r}, inp.thres)
            (o * gout[b:b + 1].double()).sum().backward()
            wp[b], wK[b], wr[b] = p.grad[0], K.grad[0].cpu(), r.grad[0].cpu()
            del o, p, K, r
    finally:
        torch.set_default_dtype(default)
    assert float(poses.grad[:, :, 3].abs().max()) == 0
    _norm_close(poses.grad[:, :, :3, :3], wp[:, :, :3, :3], 1e-4, f"{cfg} {mode} R")
    _norm_close(poses.grad[:, :, :3, 3], wp[:, :, :3, 3], 1e-4, f"{cfg} {mode} t")
    _norm_close(intM.grad, wK, 1e-4, f"{cfg} {mode} intM")
    _norm_close(rays.grad, wr, 1e-4, f"{cfg} {mode} rays")


def test_magnetf_loss_pose_gradients_against_port(cuda):
    """MagnetF.loss under the switch (fused L1 loss on the plane-sweep scores) against train_FNet.py's loss on the
    port's probability volume, float64 autograd."""
    B, V, H, W = 2, 2, 12, 20
    inp = make_inputs(B=B, V=V, D=32, H=H, W=W, C=64, seed=13)
    g = inp.to(cuda)
    d_center = magnet_b200.sid_planes(1e-3, 10.0, 32, cuda)
    gt = torch.rand(B, 1, 4 * H, 4 * W, device=cuda, generator=torch.Generator(cuda).manual_seed(2)) * 8.0 + 0.5
    model = magnet_b200.MagnetF(torch.nn.Identity())            # the "images" are the feature maps
    poses, intM, rays = _leaves(inp, cuda)
    with magnet_b200.geometry_grad():
        loss = model.loss(g.ref_feat, g.nghbr_feat, poses, inp.is_valid, {'intM': intM, 'unit_ray_array_2D': rays},
                          d_center, gt, 1e-3, 10.0)
    loss.backward()
    p = inp.nghbr_poses.to(cuda).double().requires_grad_(True)
    K = inp.cam_intrins['intM'].double().to(cuda).requires_grad_(True)
    r = inp.cam_intrins['unit_ray_array_2D'].double().to(cuda).requires_grad_(True)
    default = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        vol = torch_ref.cost_volume_f(d_center.double(), g.ref_feat.double(), g.nghbr_feat.double(), p[:, :, :3, :3],
                                      p[:, :, :3, 3], inp.is_valid, {'intM': K, 'unit_ray_array_2D': r})
        want = fnet_l1_loss(vol, d_center.double(), gt.double(), 1e-3, 10.0)
    finally:
        torch.set_default_dtype(default)
    want.backward()
    assert abs(float(loss) - float(want)) <= 1e-4 * abs(float(want))
    _norm_close(poses.grad[:, :, :3, :3], p.grad[:, :, :3, :3], 1e-3, "MagnetF R")
    _norm_close(poses.grad[:, :, :3, 3], p.grad[:, :, :3, 3], 1e-3, "MagnetF t")
    _norm_close(intM.grad, K.grad, 1e-3, "MagnetF intM")
    _norm_close(rays.grad, r.grad, 1e-3, "MagnetF rays")


@pytest.fixture
def deterministic_cudnn():
    saved = torch.backends.cudnn.deterministic
    torch.backends.cudnn.deterministic = True
    yield
    torch.backends.cudnn.deterministic = saved


def test_magnet_head_detach_cost_false_pose_gradients(cuda, deterministic_cudnn):
    """MagnetHead(detach_cost=False).forward_quarter under the switch against the same data flow on the port (fp32,
    as in test_gpu_cw_grad); with the default detach_cost=True the poses get nothing, as in the reference."""
    torch.manual_seed(0)
    B, V, H, W = 1, 2, 16, 24
    inp = make_inputs(B=B, V=V, D=5, H=H, W=W, C=16, seed=21, depth="smooth")
    g = inp.to(cuda)
    head = magnet_b200.MagnetHead(n_samples=5, n_iter=2, thres=inp.thres, dnet_fdim=8, detach_cost=False).to(cuda)
    x_d3 = torch.randn(B, 8, H, W, device=cuda)
    poses = g.nghbr_poses.clone().requires_grad_(True)
    with magnet_b200.geometry_grad():
        preds, _ = head.forward_quarter(g.ref_feat, g.nghbr_feat, g.ref_gmms, g.nghbr_gmms, x_d3, poses,
                                        inp.is_valid, inp.cam_intrins)
    sum(p.square().mean() for p in preds).backward()
    got = poses.grad.clone()
    p = g.nghbr_poses.clone().requires_grad_(True)
    intr = {k: v.to(cuda) for k, v in inp.cam_intrins.items()}
    cur, loss = g.ref_gmms, 0.0
    for _ in range(2):
        dv = torch_ref.sample_depth_candidates(cur.detach(), head.k_list)
        cv = torch_ref.cost_volume_cw(dv, g.ref_feat, g.nghbr_feat, g.ref_gmms, g.nghbr_gmms, p[:, :, :3, :3],
                                      p[:, :, :3, 3], inp.is_valid, intr, inp.thres)
        cur = torch_ref.gaussian_update(head.g_net.gnet(torch.cat([cv, x_d3], dim=1)), cur.detach())
        loss = loss + cur.square().mean()
    loss.backward()
    _norm_close(got, p.grad, 1e-3, "MagnetHead poses")
    head.detach_cost = True
    poses2 = g.nghbr_poses.clone().requires_grad_(True)
    with magnet_b200.geometry_grad():
        preds, _ = head.forward_quarter(g.ref_feat, g.nghbr_feat, g.ref_gmms, g.nghbr_gmms, x_d3, poses2,
                                        inp.is_valid, inp.cam_intrins)
    sum(p.square().mean() for p in preds).backward()
    assert poses2.grad is None


def test_refine_pose_example_follows_the_rehearsal(cuda):
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "examples", "refine_pose.py")
    spec = importlib.util.spec_from_file_location("refine_pose", path)
    ex = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ex)
    cpu = np.array(ex.refine("port", 40))
    gpu = np.array(ex.refine("magnet", 40, device=cuda))
    print("cpu", cpu[::5], "\ngpu", gpu[::5])
    assert abs(gpu[0]) == pytest.approx(0.6, abs=1e-5)
    assert abs(gpu[-1]) <= 0.02 and abs(cpu[-1]) <= 0.02          # 0.6 px -> below 0.02 px
    assert np.abs(gpu - cpu).max() <= 5e-3                         # the same trajectory
