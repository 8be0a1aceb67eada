"""Camera gradients on the GPU (magnet_cost_volume_geom_bwd_f32), element by element against the float64 restatement of
tests/geom_grad_ref.py (contracted from gathered tap dot products in torch float64 on the test's GPU, up to the cfg2,
cfg3 and F-Net shapes), and through the public entry points under geometry_grad().

Tolerance: |got - ref| <= c u bound with u = 2^-24, bound the float64 sum of absolute contributions (geom_grad_ref) and
c = D + C + V + nblk / 32 + 64 (DESIGN §3.11: the longest fp32 chain any term passes through: the channel dot product,
the sum over the hypotheses, the 3 + 2 block levels, the nblk / 32 blocks per lane and 5 lane levels of the fixed-order
reduction, the V-term ray sum, plus a few roundings of the position arithmetic).  Ambiguity is removed as in
test_gpu_grad_f64: the score gradient is zeroed where the float64 mask margin is <= 1e-3, where a position lies within
1e-3 px (or 4 position errors) of a cell edge, or where A is beyond the §3.1 limit.  For a softmax volume the
probability is zeroed there instead, which zeroes the score gradient the kernel derives."""
import numpy as np
import pytest
import torch

import magnet_b200
from magnet_b200 import _lib, ops
from magnet_b200.homography import plane_sweep_f
from magnet_b200.synthetic import make_inputs
from tests.cw_grad_ref import U, Reference, gauss_depths, softmax_score_grad
from tests.geom_grad_ref import camera_grads

pytestmark = pytest.mark.gpu


def _c(D, C, V, HW):
    return D + C + V + ((HW + 31) // 32) / 32.0 + 64.0


def _close(got, want, bound, c, what):
    got = got.detach().double().cpu().numpy()
    assert got.shape == want.shape, (what, got.shape, want.shape)
    assert np.isfinite(got).all(), what
    tol = c * U * bound
    err = np.abs(got - want)
    ratio = float(np.max(np.where(tol > 0, err / np.where(tol > 0, tol, 1.0), np.where(err > 0, np.inf, 0.0))))
    print(f"{what}: max |err| / (c u bound) = {ratio:.3g}")
    assert ratio <= 1.0, (what, ratio)


# (C, D, V, H, W, depth mode, forward kernel, consistency, softmax, family[, B = 2])
CASES = {
    "c1_direct": (1, 5, 2, 9, 13, "volume", "direct", True, False, "scannet"),
    "c8_gauss_direct": (8, 32, 4, 10, 14, "gauss", "direct", True, False, "scannet"),
    "c33_nocw": (33, 64, 2, 7, 37, "volume", "direct", False, False, "kitti"),
    "c64_split16": (64, 64, 4, 12, 16, "volume", "split16", True, False, "scannet"),
    "c64_gauss_split16": (64, 40, 3, 9, 20, "gauss", "split16", True, False, "kitti"),
    "c64_half16_v8": (64, 32, 8, 8, 9, "volume", "half16", True, False, "scannet"),
    "c16_d256_v1": (16, 256, 1, 5, 9, "volume", "direct", True, False, "scannet"),
    "planes_c8_softmax": (8, 32, 2, 11, 15, "planes", None, False, True, "scannet"),
    "planes_c64_scores_v4": (64, 64, 4, 12, 20, "planes", None, False, False, "kitti"),
    "planes_c33_sid_softmax": (33, 5, 8, 6, 33, "planes", None, False, True, "scannet"),
    # production shapes: the cfg2 / cfg3 matching step, where each lane of the fixed-order reduction adds nblk / 32 > 1
    # blocks.  On the DIRECT kernel's positions, which the reference reproduces: on project() positions the bound of
    # every term carries the position error (A + 8) u |ix + 0.5| of some 100 px, and the sum of 10^6 terms of random
    # sign per (b, v) then lies far inside c u bound, so a wrong reduction would pass
    "cfg2_gauss_direct": (64, 64, 4, 120, 160, "gauss", "direct", True, False, "scannet", 8),
    "cfg3_volume_direct": (64, 64, 4, 88, 304, "volume", "direct", True, False, "kitti", 4),
}


class Case:
    def __init__(self, name, cuda):
        Cc, D, V, H, W, mode, fwd, cw, softmax, family, *batch = CASES[name]
        B = batch[0] if batch else 2
        self.__dict__.update(B=B, C=Cc, D=D, V=V, H=H, W=W, mode=mode, fwd=fwd, cw=cw, softmax=softmax,
                             production=bool(batch))
        seed = sum(map(ord, name))
        # the production cases also have a batch element without a valid view
        self.invalid = ([(1, V - 1)] if V > 1 else []) + ([(2, v) for v in range(V)] if B > 2 else [])
        inp = make_inputs(B=B, V=V, D=D, H=H, W=W, C=Cc, seed=seed, family=family, depth="smooth",
                          invalid=self.invalid)
        if self.production:                                # view 0 of batch element 0 moves sideways: the +-10 clamp
            inp.nghbr_poses[0, 0, :3, 3] = torch.tensor([0.3, 0.05, 0.01])
        rng = np.random.default_rng(seed)
        self.inp, self.dev = inp, cuda
        g = inp.to(cuda)
        self.g = g
        intr = {k: v.to(cuda) for k, v in inp.cam_intrins.items()}
        self.cams = ops.pack_cameras(intr['intM'], g.R, g.t, inp.is_valid.to(cuda, torch.int32))
        self.rays = intr['unit_ray_array_2D'].contiguous()
        gmm = inp.ref_gmms.numpy()
        self.k = None
        if mode == "gauss":
            self.k = np.linspace(-2.5, 2.5, D).astype(np.float32).tolist()
            if self.production:                            # behind the source cameras, and beyond the +-10 clamp
                self.k = [-40.0, -9.98] + self.k[2:]
            depth = gauss_depths(gmm, self.k, "direct")
        elif mode == "planes":
            if name.endswith("sid_softmax"):               # SID planes reaching behind a source camera
                planes = np.array([-1.0, 0.05, 0.7, 2.0, 6.0], np.float32)
            else:
                planes = np.linspace(0.6, 6.0, D).astype(np.float32)
            self.k = planes.tolist()
            depth = np.broadcast_to(planes.reshape(1, D, 1, 1), (B, D, H, W)).astype(np.float32)
        else:
            depth = (gmm[:, :1] + gmm[:, 1:] * np.linspace(-2.5, 2.5, D).reshape(1, D, 1, 1)).astype(np.float32)
            depth[0, 0] = -depth[0, 0]                    # behind the source cameras
            if D > 1:
                depth[0, 1] *= np.float32(0.002)          # beyond the +-10 clamp
        self.depth = depth
        self.d_volume = torch.from_numpy(depth).to(cuda)
        pos = "direct" if fwd == "direct" else "mma"
        self.rf = Reference(depth, inp.ref_feat.numpy(), inp.nghbr_feat.numpy(),
                            inp.nghbr_gmms.numpy() if cw else None, self.cams.cpu().numpy(),
                            inp.cam_intrins['unit_ray_array_2D'].numpy(), float(inp.thres), pos=pos, consistency=cw,
                            device=cuda)
        amb = self.rf.ambiguous()
        gout = rng.standard_normal(amb.shape).astype(np.float32)
        if softmax:
            sc = rng.standard_normal(amb.shape)
            prob = np.exp(sc - sc.max(1, keepdims=True))
            prob = (prob / prob.sum(1, keepdims=True)).astype(np.float32)
            self.prob = np.where(amb, np.float32(0), prob).astype(np.float32)
            self.gout = gout
            self.gs, self.gs_abs = softmax_score_grad(self.prob, gout, V)
        else:
            self.prob = None
            self.gout = np.where(amb, np.float32(0), gout).astype(np.float32)
            self.gs, self.gs_abs = self.gout.astype(np.float64) / V, None
        self.want = camera_grads(self.rf, depth, self.cams.cpu().numpy(), inp.cam_intrins['unit_ray_array_2D'].numpy(),
                                 self.gs, self.gs_abs)

    def call(self, need_depth=False, grad_out=None):
        g = self.g
        layout, variant = {"direct": (_lib.SRC_NCHW, _lib.VARIANT_DIRECT), "split16": (_lib.SRC_SPLIT16, _lib.VARIANT_AUTO),
                           "half16": (_lib.SRC_HALF16, _lib.VARIANT_AUTO), None: (_lib.SRC_NCHW, _lib.VARIANT_AUTO)}[self.fwd]
        kw = dict(V=self.V, kappa=float(self.inp.thres), consistency=self.cw, fwd_layout=layout, fwd_variant=variant,
                  need_depth=need_depth)
        if self.mode == "volume":
            kw["d_volume"] = self.d_volume
        elif self.mode == "gauss":
            kw.update(ref_gmm=g.ref_gmms, k=self.k)
        else:
            kw.update(k=self.k, planes=True, softmax=self.softmax,
                      prob=None if self.prob is None else torch.from_numpy(self.prob).to(self.dev))
        go = torch.from_numpy(self.gout).to(self.dev) if grad_out is None else grad_out
        return ops.cost_volume_geom_bwd(g.ref_feat, g.nghbr_feat, g.nghbr_gmms, self.rays, self.cams, go, **kw)


@pytest.mark.parametrize("name", sorted(CASES))
def test_camera_gradients_elementwise(name, cuda):
    cs = Case(name, cuda)
    amb = cs.rf.ambiguous()
    print(f"{name}: zeroed {amb.mean():.4f}")
    c = _c(cs.D, cs.C, cs.V, cs.H * cs.W)
    if cs.production:
        # each lane of geom_reduce_kernel adds several blocks; the planted edges are compared; the gate is sharp: most
        # valid camera-table entries and ray elements exceed their tolerance, so a zeroed output or a missing block
        # partial of that size is rejected
        assert (cs.H * cs.W + 31) // 32 > 32 and amb.mean() <= 0.025, amb.mean()
        for k in ("behind", "clamped", "tap_outside"):
            assert (cs.rf.reached[k].reshape(amb.shape) & ~amb).any(), k
        valid = cs.inp.is_valid.numpy().reshape(-1) == 1
        for out, sel in (("cams", valid), ("rays", cs.want["rays_b"] > 0)):
            sharp = (np.abs(cs.want[out]) > c * U * cs.want[out + "_b"])[sel]
            print(f"{name} {out}: {sharp.mean():.3f} of the elements exceed c u bound")
            assert sharp.mean() > 0.75, (out, sharp.mean())
    g_cams, g_rays, _ = cs.call()
    torch.cuda.synchronize()
    _close(g_cams, cs.want["cams"], cs.want["cams_b"], c, f"{name} cams")
    _close(g_rays, cs.want["rays"], cs.want["rays_b"], c, f"{name} rays")
    assert np.abs(cs.want["cams"]).max() > 0
    for b, v in cs.invalid:                                # invalid views get exactly zero
        assert not g_cams[b * cs.V + v].any()
    # determinism: no atomics
    g2, r2, _ = cs.call()
    assert torch.equal(g_cams, g2) and torch.equal(g_rays, r2)


@pytest.mark.parametrize("name", ["c8_gauss_direct", "c64_split16", "c33_nocw"])
def test_depth_gradient_of_camera_pass(name, cuda):
    """The grad_depth a camera launch writes agrees with the non-camera kernel's to the last bits (the two
    instantiations may contract the products of the depth derivative differently); the autograd path keeps taking it
    from the non-camera kernel."""
    cs = Case(name, cuda)
    g = cs.g
    _, _, gd = cs.call(need_depth=True)
    layout = _lib.SRC_SPLIT16 if cs.fwd == "split16" else _lib.SRC_NCHW
    variant = _lib.VARIANT_AUTO if cs.fwd == "split16" else _lib.VARIANT_DIRECT
    kw = dict(d_volume=torch.from_numpy(cs.depth).to(cuda)) if cs.mode == "volume" else dict(ref_gmm=g.ref_gmms, k=cs.k)
    _, _, gd0 = ops.cost_volume_bwd(g.ref_feat, g.nghbr_feat, g.nghbr_gmms, cs.rays, cs.cams,
                                    torch.from_numpy(cs.gout).to(cuda), V=cs.V, kappa=float(cs.inp.thres),
                                    consistency=cs.cw, fwd_layout=layout, fwd_variant=variant, need_ref=False,
                                    need_src=False, **kw)
    assert torch.allclose(gd, gd0, rtol=1e-5, atol=1e-6 * float(gd0.abs().max()))


def test_cuda_graph_replay(cuda):
    cs = Case("c64_split16", cuda)
    go = torch.from_numpy(cs.gout).to(cuda)
    cs.call(grad_out=go)                                   # warm-up outside the capture
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        gc, gr, _ = cs.call(grad_out=go)
    go.copy_(go * -0.5 + 0.25)
    graph.replay()
    torch.cuda.synchronize()
    ec, er, _ = cs.call(grad_out=go)
    assert torch.equal(gc, ec) and torch.equal(gr, er)


# ---------------------------------------------------------------------------------------------------------------------
# Public entry points

def _leaves(inp, cuda):
    poses = inp.nghbr_poses.to(cuda).clone().requires_grad_(True)
    intM = inp.cam_intrins['intM'].clone().requires_grad_(True)              # CPU, as in test_MaGNet.py
    rays = inp.cam_intrins['unit_ray_array_2D'].clone().requires_grad_(True)
    return poses, intM, rays


@pytest.mark.parametrize("variant", [_lib.VARIANT_DIRECT, _lib.VARIANT_AUTO])
def test_est_costvolume_cw_camera_gradients(variant, cuda):
    """R / t (views of nghbr_poses), intM and the rays get the chain of the ops-level camera gradients; grad_depth and
    the CUDA-core grad_ref are bit-identical with and without camera gradients, grad_src within its atomics' rounding."""
    inp = make_inputs(B=2, V=3, D=64, H=12, W=16, C=64, seed=11, invalid=[(1, 1)])
    g = inp.to(cuda)
    dvol = inp.depth_volume().to(cuda)
    gout = torch.from_numpy(np.random.default_rng(3).standard_normal(dvol.shape).astype(np.float32)).to(cuda)

    def run(with_cams):
        d = dvol.clone().requires_grad_(True)
        ref = g.ref_feat.clone().requires_grad_(True)
        src = g.nghbr_feat.clone().requires_grad_(True)
        poses, intM, rays = _leaves(inp, cuda)
        if not with_cams:
            poses, intM, rays = poses.detach(), intM.detach(), rays.detach()
        with magnet_b200.geometry_grad():
            out = magnet_b200.est_costvolume_CW(d, ref, src, g.ref_gmms, g.nghbr_gmms, poses[:, :, :3, :3],
                                                poses[:, :, :3, 3], inp.is_valid,
                                                {'intM': intM, 'unit_ray_array_2D': rays}, inp.thres, variant=variant)
        (out * gout).sum().backward()
        torch.cuda.synchronize()
        return out.detach(), d.grad, ref.grad, src.grad, poses, intM, rays

    o0, d0, r0, s0, _, _, _ = run(False)
    o1, d1, r1, s1, poses, intM, rays = run(True)
    assert torch.equal(o0, o1) and torch.equal(d0, d1)
    if variant == _lib.VARIANT_DIRECT:
        assert torch.equal(r0, r1)
    assert torch.allclose(s0, s1, rtol=1e-5, atol=1e-5 * float(s0.abs().max()))
    assert intM.grad.device.type == "cpu" and rays.grad.device.type == "cpu" and poses.grad.device == d1.device
    # the same gradients from one ops call on the forward's kernel
    layout = _lib.SRC_SPLIT16 if variant == _lib.VARIANT_AUTO else _lib.SRC_NCHW
    cams = ops.pack_cameras(inp.cam_intrins['intM'].to(cuda), g.R, g.t, inp.is_valid.to(cuda, torch.int32))
    gc, gr, _ = ops.cost_volume_geom_bwd(g.ref_feat, g.nghbr_feat, g.nghbr_gmms,
                                         inp.cam_intrins['unit_ray_array_2D'].to(cuda), cams, gout, V=3,
                                         kappa=float(inp.thres), d_volume=dvol, fwd_layout=layout, fwd_variant=variant)
    gR, gt, gK = ops.camera_chain(gc, inp.cam_intrins['intM'].to(cuda), g.R, g.t)
    assert torch.equal(poses.grad[:, :, :3, :3], gR) and torch.equal(poses.grad[:, :, :3, 3], gt)
    assert not poses.grad[:, :, 3].any()
    assert torch.equal(intM.grad, gK.cpu()) and torch.equal(rays.grad, gr.cpu())


def test_no_camera_grad_issues_todays_launches(cuda):
    inp = make_inputs(B=1, V=2, D=8, H=6, W=9, C=8, seed=2)
    g = inp.to(cuda)

    def launches(switch):
        magnet_b200.clear_cache()                          # both arms prepare their inputs
        d = inp.depth_volume().to(cuda).requires_grad_(True)
        before = _lib.launch_count()
        with magnet_b200.geometry_grad(switch):
            out = magnet_b200.est_costvolume_CW(d, g.ref_feat, g.nghbr_feat, g.ref_gmms, g.nghbr_gmms, g.R, g.t,
                                                inp.is_valid, inp.cam_intrins, inp.thres)
            out.sum().backward()
            dc = torch.linspace(1.0, 5.0, 8).view(1, -1, 1, 1)
            ref = g.ref_feat.clone().requires_grad_(True)
            plane_sweep_f(dc, ref, g.nghbr_feat, g.R, g.t, inp.is_valid, inp.cam_intrins, softmax=False).sum().backward()
        torch.cuda.synchronize()
        return _lib.launch_count() - before, d.grad, ref.grad

    n0, d0, r0 = launches(False)
    n1, d1, r1 = launches(True)
    assert n0 == n1 and torch.equal(d0, d1) and torch.equal(r0, r1)


@pytest.mark.parametrize("softmax", [False, True])
def test_plane_sweep_pose_gradients(softmax, cuda):
    """plane_sweep_f (MagnetF's path) and est_costvolume_F give the pose gradients of one ops call."""
    inp = make_inputs(B=2, V=2, D=48, H=12, W=16, C=64, seed=5)
    g = inp.to(cuda)
    dc = torch.linspace(0.8, 5.0, 48).view(1, -1, 1, 1)
    gout = torch.from_numpy(np.random.default_rng(8).standard_normal((2, 48, 12, 16)).astype(np.float32)).to(cuda)
    for fn in (lambda *a: plane_sweep_f(*a, softmax=softmax),) + ((magnet_b200.est_costvolume_F,) if softmax else ()):
        poses, intM, rays = _leaves(inp, cuda)
        with magnet_b200.geometry_grad():
            out = fn(dc, g.ref_feat, g.nghbr_feat, poses[:, :, :3, :3], poses[:, :, :3, 3], inp.is_valid,
                     {'intM': intM, 'unit_ray_array_2D': rays})
        (out * gout).sum().backward()
        cams = ops.pack_cameras(inp.cam_intrins['intM'].to(cuda), g.R, g.t, inp.is_valid.to(cuda, torch.int32))
        gc, gr, _ = ops.cost_volume_geom_bwd(g.ref_feat, g.nghbr_feat, None,
                                             inp.cam_intrins['unit_ray_array_2D'].to(cuda), cams, gout, V=2,
                                             k=dc.reshape(-1).tolist(), planes=True, softmax=softmax,
                                             prob=out.detach() if softmax else None)
        gR, gt, gK = ops.camera_chain(gc, inp.cam_intrins['intM'].to(cuda), g.R, g.t)
        assert torch.equal(poses.grad[:, :, :3, :3], gR) and torch.equal(poses.grad[:, :, :3, 3], gt)
        assert torch.equal(intM.grad, gK.cpu()) and torch.equal(rays.grad, gr.cpu())
        assert gR.abs().max() > 0


def test_matching_plan_detach_cost_false(cuda):
    """MatchingPlan.cost under the switch: nghbr_poses gets the pose gradient of one ops call (GAUSS mode)."""
    inp = make_inputs(B=1, V=3, D=5, H=10, W=12, C=16, seed=9)
    g = inp.to(cuda)
    poses, intM, rays = _leaves(inp, cuda)
    k = inp.k.tolist()
    gout = torch.from_numpy(np.random.default_rng(1).standard_normal((1, 5, 10, 12)).astype(np.float32)).to(cuda)
    with magnet_b200.geometry_grad():
        plan = magnet_b200.MatchingPlan(g.ref_feat, g.nghbr_feat, g.nghbr_gmms, poses, inp.is_valid,
                                        {'intM': intM, 'unit_ray_array_2D': rays}, thres=inp.thres)
        (plan.cost(g.ref_gmms, k) * gout).sum().backward()
    gc, gr, _ = ops.cost_volume_geom_bwd(g.ref_feat, g.nghbr_feat, g.nghbr_gmms,
                                         inp.cam_intrins['unit_ray_array_2D'].to(cuda), plan.cams, gout, V=3,
                                         kappa=float(inp.thres), ref_gmm=g.ref_gmms, k=k)
    gR, gt, gK = ops.camera_chain(gc, inp.cam_intrins['intM'].to(cuda), g.R, g.t)
    assert torch.equal(poses.grad[:, :, :3, :3], gR) and torch.equal(poses.grad[:, :, :3, 3], gt)
    assert torch.equal(rays.grad, gr.cpu()) and gR.abs().max() > 0
