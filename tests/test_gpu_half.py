"""Half-precision feature maps on the H100: the HALF16 repack, the tensor-core forward bit for bit against the fp32 path
on the upcast maps, the gradients against the float64 reference and through autograd, torch.autocast end to end,
graph replay, the buffer checks and the window-box counters of a debug build (DESIGN §3.7)."""
import json
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch
import torch.nn as nn

import magnet_b200
from magnet_b200 import _lib, ops
from magnet_b200 import build as _build
from magnet_b200 import homography as hg
from magnet_b200.homography import plane_sweep_f
from magnet_b200.synthetic import make_config, make_inputs
from tests import test_gpu_grad_f64 as gf

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DTYPES = [torch.bfloat16, torch.float16]
DT_IDS = ["bf16", "fp16"]


def _halve(inp, dt):
    """The inputs with half-precision feature maps (the fp32 path then runs on their exact upcast)."""
    inp.ref_feat, inp.nghbr_feat = inp.ref_feat.to(dt), inp.nghbr_feat.to(dt)
    return inp


class _Repacks:
    """Counts the HALF16 and SPLIT16 repacks issued inside a ``with`` block (every prep cache cleared on entry), so that
    a test sees which layout an entry point actually took."""

    def __enter__(self):
        self.n = {"half16": 0, "split16": 0}
        self._orig = (ops.repack_half16, ops.repack_split16)
        hg.clear_cache()

        def wrap(kind, fn):
            def counted(*a, **kw):
                self.n[kind] += 1
                return fn(*a, **kw)
            return counted

        ops.repack_half16, ops.repack_split16 = wrap("half16", self._orig[0]), wrap("split16", self._orig[1])
        return self

    def __exit__(self, *exc):
        ops.repack_half16, ops.repack_split16 = self._orig
        hg.clear_cache()


def _took(rp, half, what):
    """The layout an entry point took: HALF16 (and no fp32 split) for half maps, SPLIT16 (and no HALF16) for fp32."""
    if half:
        assert rp.n["half16"] > 0 and rp.n["split16"] == 0, (what, rp.n)
    else:
        assert rp.n["half16"] == 0 and rp.n["split16"] > 0, (what, rp.n)


def _eq(got, want, what):
    assert got.dtype == torch.float32, (what, got.dtype)
    assert np.array_equal(got.cpu().numpy(), want.cpu().numpy()), (what, float((got - want).abs().max()))


def _all_forwards(g, inp, dt, variant=_lib.VARIANT_AUTO, f=True):
    """(name, half result, fp32 result) of every entry point: est_costvolume_CW (VOLUME), MatchingPlan.cost (GAUSS),
    est_costvolume_F and plane_sweep_f with softmax on and off (PLANES)."""
    ref32, src32 = g.ref_feat.float(), g.nghbr_feat.float()
    k = inp.k.tolist()
    dvol = ops.sample_depths(g.ref_gmms, k)
    out = []
    dc = torch.linspace(0.5, 8.0, max(inp.D, 32), device=g.ref_feat.device).view(1, -1, 1, 1)
    calls = [lambda r, s: magnet_b200.est_costvolume_CW(dvol, r, s, g.ref_gmms, g.nghbr_gmms, g.R, g.t, inp.is_valid,
                                                        inp.cam_intrins, inp.thres, variant=variant),
             lambda r, s: magnet_b200.MatchingPlan(r, s, g.nghbr_gmms, g.nghbr_poses, inp.is_valid, inp.cam_intrins,
                                                   thres=inp.thres).cost(g.ref_gmms, k, variant=variant)]
    if f:
        calls.append(lambda r, s: magnet_b200.est_costvolume_F(dc, r, s, g.R, g.t, inp.is_valid, inp.cam_intrins))
        calls += [lambda r, s, sm=sm: plane_sweep_f(dc, r, s, g.R, g.t, inp.is_valid, inp.cam_intrins, softmax=sm)
                  for sm in (True, False)]
    with torch.no_grad():
        for name, (r, s) in (("half", (g.ref_feat, g.nghbr_feat)), ("f32", (ref32, src32))):
            res = []
            for i, call in enumerate(calls):
                with _Repacks() as rp:
                    res.append(call(r, s))
                _took(rp, name == "half", f"{name}/entry point {i}")
            out.append(res)
    names = ["CW/volume", "plan/gauss", "F", "sweep/softmax", "sweep/scores"]
    return [(n, a, b) for n, a, b in zip(names, out[0], out[1])]


@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("H,W", [(16, 24), (7, 9)])          # vectorised and ragged H * W
def test_repack_equals_hi_plane_of_the_fp32_split(cuda, dt, H, W):
    N = 3
    x = (torch.randn(N, 64, H, W, device=cuda) * 5).to(dt)
    x[0, 0, 0, 0] = float("inf")                             # does not set the scale
    gmm = torch.rand(N, 2, H, W, device=cuda) + 0.1
    h = ops.repack_half16(x, gmm)
    s = ops.repack_split16(x.float(), gmm)
    assert h.numel() == lib_bytes(_lib.SRC_HALF16, N, H, W)
    assert torch.equal(h[:12], s[:12])                       # scale, 1 / scale, absmax bits
    plane = N * H * W * 128
    hi = s[256:256 + 2 * plane].view(N, 2, H * W * 128)[:, 0].reshape(-1)
    lo = s[256:256 + 2 * plane].view(N, 2, H * W * 128)[:, 1].reshape(-1)
    assert torch.equal(h[256:256 + plane], hi)
    finite = torch.isfinite(x.float()).permute(0, 2, 3, 1).reshape(-1)
    assert not lo.view(torch.float16)[finite].float().any()   # exact map: zero lo plane
    assert torch.equal(h[256 + plane:], s[256 + 2 * plane:])  # the (mu, sigma) table


def lib_bytes(layout, N, H, W):
    return ops.packed_bytes(layout, N, H, W)


@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("cfg", ["cfg2", "cfg3"])
def test_forward_bit_identity_full_configs(cuda, dt, cfg):
    inp = _halve(make_config(cfg, seed=1), dt)
    inp.k = torch.linspace(-2.5, 2.5, 64)                    # >= MMA_MIN_PLANES: the tensor-core kernel
    g = inp.to(cuda)
    for name, a, b in _all_forwards(g, inp, dt):
        _eq(a, b, f"{cfg}/{name}")


@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
def test_forward_bit_identity_fuzz(cuda, dt):
    """The shapes and generator settings of test_mma_kernel_fuzz_against_direct_kernel, variant MMA."""
    rng = np.random.default_rng(4048)
    for it in range(24):
        B, V = int(rng.integers(1, 3)), int(rng.integers(1, 7))
        D = int(rng.choice([1, 3, 5, 17, 33, 64, 65, 150])) if it % 3 else int(rng.integers(1, 70))
        H, W = int(rng.integers(5, 41)), int(rng.integers(5, 71))
        depth = "random" if it % 4 == 0 else "smooth"
        family = "kitti" if it % 5 == 0 else "scannet"
        kw = dict(rot_deg=float(rng.uniform(1, 14)), trans=float(rng.uniform(0.05, 0.7))) if it % 2 else {}
        invalid = [(0, int(rng.integers(0, V)))] if V > 1 and it % 3 == 0 else ()
        inp = make_inputs(B=B, V=V, D=D, H=H, W=W, C=64, seed=3000 + it, depth=depth, family=family, invalid=invalid, **kw)
        scale = float(10.0 ** rng.integers(-3, 4))
        inp.ref_feat.mul_(scale)
        inp.nghbr_feat.mul_(1.0 / scale if it % 2 else scale)
        g = _halve(inp, dt).to(cuda)
        for name, a, b in _all_forwards(g, inp, dt, variant=_lib.VARIANT_MMA, f=it % 4 == 1):
            _eq(a, b, f"fuzz{it}/{name}")


@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
def test_forward_bit_identity_sid_planes_behind_camera(cuda, dt):
    inp = make_inputs(B=2, V=2, D=8, H=40, W=64, C=64, seed=17, depth="smooth")
    inp.nghbr_poses[:, :, 2, 3] = -0.3
    g = _halve(inp, dt).to(cuda)
    dc = magnet_b200.sid_planes(1e-3, 10.0, 80, device=cuda)
    for sm in (True, False):
        with _Repacks() as rp:
            a = plane_sweep_f(dc, g.ref_feat, g.nghbr_feat, g.R, g.t, inp.is_valid, inp.cam_intrins, softmax=sm)
        _took(rp, True, "sid")
        b = plane_sweep_f(dc, g.ref_feat.float(), g.nghbr_feat.float(), g.R, g.t, inp.is_valid, inp.cam_intrins,
                          softmax=sm)
        _eq(a, b, f"sid/softmax={sm}")


@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
def test_volume_mode_without_consistency_at_ops_level(cuda, dt):
    """<VOLUME, false, 1> issues n128 for warpgroup 1 where the fp32 kernel issues n64 (DESIGN §3.7): same volume."""
    inp = make_inputs(B=2, V=3, D=64, H=24, W=72, C=64, seed=8, depth="random", trans=0.5)
    g = _halve(inp, dt).to(cuda)
    plan = magnet_b200.MatchingPlan(g.ref_feat.float(), g.nghbr_feat.float(), g.nghbr_gmms, g.nghbr_poses,
                                    inp.is_valid, inp.cam_intrins)
    dvol = ops.sample_depths(g.ref_gmms, inp.k.tolist())
    kw = dict(V=3, consistency=False, d_volume=dvol, variant=_lib.VARIANT_MMA)
    a = ops.cost_volume(g.ref_feat, ops.repack_half16(g.nghbr_feat), plan.rays, plan.cams, src_layout=_lib.SRC_HALF16,
                        ref_split=ops.repack_half16(g.ref_feat), **kw)
    b = ops.cost_volume(g.ref_feat.float(), ops.repack_split16(g.nghbr_feat.float()), plan.rays, plan.cams,
                        src_layout=_lib.SRC_SPLIT16, ref_split=ops.repack_split16(g.ref_feat.float()), **kw)
    _eq(a, b, "volume/no consistency")


# ------------------------------------------------------------------------------------------------------------------
# gradients: the float64 reference of tests/cw_grad_ref.py on the upcast maps, contracted on the GPU (cases of
# test_gpu_grad_f64 with unit feature scales, so that the half maps are the rounded fp32 ones, up to cfg2)
def _half_case(name, cuda, dt):
    orig = gf.make_inputs

    def rounded(**kw):
        return _halve_back(orig(**kw), dt)

    gf.make_inputs = rounded
    try:
        return gf.Case(name, cuda)
    finally:
        gf.make_inputs = orig


def _halve_back(inp, dt):
    inp.ref_feat, inp.nghbr_feat = inp.ref_feat.to(dt).float(), inp.nghbr_feat.to(dt).float()
    return inp


def _ulp(x, dt):
    """Spacing of dtype dt at |x| (the subnormal step below its smallest normal)."""
    fi = torch.finfo(dt)
    e = torch.floor(torch.log2(x.abs().clamp_min(fi.smallest_normal)))
    return torch.exp2(e - (fi.bits - 1 - (8 if dt == torch.bfloat16 else 5)))


@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("name", ["tc_d32", "gauss_c64_tc", "cfg2_gauss"])
def test_cw_gradients_half16(cuda, dt, name):
    cs = _half_case(name, cuda, dt)
    g, inp = cs.g, cs.inp
    ref_h, src_h = torch.from_numpy(cs.ref).to(cuda).to(dt), torch.from_numpy(cs.src).to(cuda).to(dt)
    gout = torch.from_numpy(cs.gout).to(cuda)
    kw = dict(V=cs.V, kappa=float(inp.thres), fwd_layout=_lib.SRC_HALF16, fwd_variant=_lib.VARIANT_AUTO,
              need_depth=False, ref_split=ops.repack_half16(ref_h), src_split=ops.repack_half16(src_h, g.nghbr_gmms))
    if cs.mode == "gauss":
        kw.update(ref_gmm=g.ref_gmms, k=cs.k)
    else:
        kw.update(d_volume=torch.from_numpy(cs.depth_vol).to(cuda))
    gr, gs, _ = ops.cost_volume_bwd(ref_h, src_h, g.nghbr_gmms, cs.rays, cs.cams, gout, **kw)
    assert gr.dtype == gs.dtype == torch.float32
    cs.check_grads(None, gr, gs, f"{name}/{dt} ops", tc_features=True)
    # through autograd: the input's dtype, within one ulp of it of a result inside the float64 bound (the fp32 results
    # themselves vary from run to run by up to ~u bound: grad_src is summed with atomics, DESIGN §3.5); the depth
    # gradient equals the fp32 path's bit for bit (CUDA-core kernel on the same upcast maps)
    res = {}
    for tag, (r0, s0) in (("half", (ref_h, src_h)), ("f32", (ref_h.float(), src_h.float()))):
        d, _, _ = cs.leaves()
        r, s = r0.clone().requires_grad_(), s0.clone().requires_grad_()
        if cs.mode == "gauss":
            plan = magnet_b200.MatchingPlan(r, s, g.nghbr_gmms, g.nghbr_poses, inp.is_valid, inp.cam_intrins,
                                            thres=inp.thres)
            out = plan.cost(d, cs.k)
        else:
            out = magnet_b200.est_costvolume_CW(d, r, s, g.ref_gmms, g.nghbr_gmms, g.R, g.t, inp.is_valid,
                                                inp.cam_intrins, inp.thres)
        (out * gout).sum().backward()
        res[tag] = (out.detach(), d.grad, r.grad, s.grad)
    out_h, gd_h, gr_h, gs_h = res["half"]
    _eq(out_h, res["f32"][0], f"{name} forward")
    assert gr_h.dtype == gs_h.dtype == dt
    w = cs.want
    for got, key, floor in ((gr_h, "ref", cs.floors[0]), (gs_h, "src", cs.floors[1])):
        want = torch.from_numpy(w[key]).to(cuda)
        tol = torch.from_numpy(gf.C_TOL * gf.U * w[key + "_b"] + floor).to(cuda) + _ulp(want, dt).double()
        err = (got.double() - want).abs()
        assert (err <= tol).all(), (key, float((err / tol).max()))
    assert torch.equal(gd_h, res["f32"][1]), "depth gradient"


@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("softmax", [True, False])
def test_f_gradients_half16(cuda, dt, softmax):
    """The F volume's feature gradients on HALF16 buffers (SID planes from 1e-3) against the float64 reference, as
    test_f_volume_against_float64 holds the SPLIT16 ones."""
    orig = gf.make_inputs
    gf.make_inputs = lambda **kw: _halve_back(orig(**kw), dt)
    try:
        fc = gf.FCase("f64_tc_sid", cuda)
    finally:
        gf.make_inputs = orig
    g, inp, V = fc.g, fc.inp, fc.V
    intr = {k: v.to(cuda) for k, v in inp.cam_intrins.items()}
    cams = ops.pack_cameras(intr['intM'], g.R, g.t, inp.is_valid.to(cuda, torch.int32))
    rays = intr['unit_ray_array_2D'].contiguous()
    ref_h, src_h = g.ref_feat.to(dt), g.nghbr_feat.to(dt)
    rs, ss = ops.repack_half16(ref_h), ops.repack_half16(src_h)
    planes = fc.planes.reshape(-1).tolist()
    out = ops.cost_volume(ref_h, ss, rays, cams, V=V, src_layout=_lib.SRC_HALF16, consistency=False, k=planes,
                          planes=True, softmax=softmax, ref_split=rs)
    gout = torch.from_numpy(fc.gout).to(cuda)
    gr, gs = ops.cost_volume_f_bwd(ref_h, src_h, rays, cams, planes, V, out, gout, softmax=softmax, ref_split=rs,
                                   src_split=ss, split_layout=_lib.SRC_HALF16)
    assert gr.dtype == gs.dtype == torch.float32
    if softmax:
        gsc, gsc_b = gf.softmax_score_grad(gf._np(out), fc.gout, V)
    else:
        gsc, gsc_b = fc.gout.astype(np.float64) / V, np.abs(fc.gout.astype(np.float64)) / V
    want = fc.rf.backward(gsc, gsc_b)
    f_ref, f_src = gf._tc_floors(gsc_b, inp.ref_feat.numpy(), inp.nghbr_feat.numpy(), V)
    gf._close(gr, want["ref"], want["ref_b"], f"half16 softmax={softmax} ref", f_ref)
    gf._close(gs, want["src"], want["src_b"], f"half16 softmax={softmax} src", f_src)


# ------------------------------------------------------------------------------------------------------------------
# torch.autocast end to end, small conv stand-ins for the backbones
class _Stand(nn.Module):
    """F-Net / D-Net stand-in: a 1x1 convolution of the features (half under autocast)."""

    def __init__(self, cin, cout):
        super().__init__()
        self.conv = nn.Conv2d(cin, cout, 1)

    def forward(self, x):
        return self.conv(x)


@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("n_samples", [32, 5])                # HALF16, and the gather kernel on the upcast maps
def test_autocast_magnet_head_step(cuda, dt, n_samples, monkeypatch):
    torch.manual_seed(0)
    inp = make_inputs(B=2, V=3, D=n_samples, H=24, W=32, C=64, seed=44, depth="smooth").to(cuda)
    fnet = _Stand(64, 64).to(cuda)
    dnet = _Stand(64, 16).to(cuda)
    head = magnet_b200.MagnetHead(n_samples=n_samples, dnet_fdim=16, detach_cost=False).to(cuda)
    seen = []
    orig = magnet_b200.MatchingPlan.cost

    def rec(plan, gmm, k, out=None, variant=_lib.VARIANT_AUTO):
        v = orig(plan, gmm, k, out=out, variant=variant)
        seen.append((plan, gmm.detach().clone(), v.detach().clone()))
        return v

    monkeypatch.setattr(magnet_b200.MatchingPlan, "cost", rec)
    B = inp.B
    with torch.autocast("cuda", dtype=dt):
        feat = fnet(torch.cat([inp.ref_feat, inp.nghbr_feat]))
        x_d3 = dnet(inp.ref_feat)
        assert feat.dtype == dt and x_d3.dtype == dt
        preds, mask = head.forward_quarter(feat[:B], feat[B:], inp.ref_gmms.to(dt), inp.nghbr_gmms.to(dt), x_d3,
                                           inp.nghbr_poses, inp.is_valid, inp.cam_intrins)
        gt = torch.rand(B, 1, 96, 128, device=cuda) * 5 + 0.5
        loss = head.loss(preds, mask, gt, gt > 1.0)
    assert all(p.dtype == torch.float32 for p in preds) and mask.dtype == torch.float32 and loss.dtype == torch.float32
    loss.backward()
    for prm in fnet.parameters():
        assert prm.grad is not None and prm.grad.dtype == torch.float32 and torch.isfinite(prm.grad).all()
    monkeypatch.setattr(magnet_b200.MatchingPlan, "cost", orig)
    assert len(seen) == head.n_iter
    # the fp32 plan on the upcast features, differentiable as well (the same kernel: DIRECT when D < MMA_MIN_PLANES)
    f32 = magnet_b200.MatchingPlan(feat[:B].detach().float().requires_grad_(), feat[B:].detach().float().requires_grad_(),
                                   inp.nghbr_gmms.to(dt).float(), inp.nghbr_poses, inp.is_valid, inp.cam_intrins,
                                   thres=head.thres)
    for plan, gmm, vol in seen:
        # the layout taken: HALF16 buffers at 32 hypotheses, the DIRECT kernel's upcast NCHW maps at the shipped 5
        assert list(plan._packed) == [_lib.SRC_HALF16 if n_samples >= 32 else _lib.SRC_NCHW], list(plan._packed)
        _eq(vol, f32.cost(gmm, head.k_list).detach(), "G-Net input")


@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
def test_autocast_magnet_f_step(cuda, dt):
    torch.manual_seed(1)
    inp = make_inputs(B=2, V=2, D=8, H=24, W=32, C=64, seed=45, depth="smooth").to(cuda)
    fnet = nn.Conv2d(3, 64, 3, padding=1).to(cuda)
    mf = magnet_b200.MagnetF(fnet)
    imgs = torch.rand(inp.B * 3, 3, 24, 32, device=cuda)
    ref_img, nghbr_imgs = imgs[:inp.B], imgs[inp.B:]
    dc = magnet_b200.sid_planes(0.5, 10.0, 64, device=cuda)
    gt = torch.rand(inp.B, 1, 24, 32, device=cuda) * 8 + 0.5
    with torch.autocast("cuda", dtype=dt), _Repacks() as rp:
        loss = mf.loss(ref_img, nghbr_imgs, inp.nghbr_poses, inp.is_valid, inp.cam_intrins, dc, gt, 0.5, 10.0)
        ref_f, src_f = mf._features(ref_img, nghbr_imgs)
        vol = mf(ref_img, nghbr_imgs, inp.nghbr_poses, inp.is_valid, inp.cam_intrins, dc)
    _took(rp, True, "MagnetF")
    assert ref_f.dtype == dt and loss.dtype == torch.float32
    loss.backward()
    assert fnet.weight.grad.dtype == torch.float32 and torch.isfinite(fnet.weight.grad).all()
    want = plane_sweep_f(dc, ref_f.detach().float(), src_f.detach().float(), inp.R, inp.t, inp.is_valid,
                         inp.cam_intrins, softmax=True)
    _eq(vol.detach(), want, "MagnetF volume")


@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
def test_install_under_autocast(cuda, dt):
    mod = types.ModuleType("homography")
    magnet_b200.install(mod)
    inp = make_inputs(B=1, V=2, D=64, H=16, W=24, C=64, seed=46, depth="smooth").to(cuda)
    conv = nn.Conv2d(64, 64, 1).to(cuda)
    dvol = ops.sample_depths(inp.ref_gmms, inp.k.tolist())
    dc = torch.linspace(0.5, 6.0, 48, device=cuda).view(1, -1, 1, 1)
    with torch.autocast("cuda", dtype=dt), _Repacks() as rp:
        f = conv(torch.cat([inp.ref_feat, inp.nghbr_feat]))
        cw = mod.est_costvolume_CW(dvol.to(dt), f[:1], f[1:], inp.ref_gmms, inp.nghbr_gmms.to(dt), inp.R, inp.t,
                                   inp.is_valid, inp.cam_intrins, 5)
        fv = mod.est_costvolume_F(dc, f[:1], f[1:], inp.R, inp.t, inp.is_valid, inp.cam_intrins)
    _took(rp, True, "install")
    f32 = f.detach().float()
    with torch.no_grad():
        _eq(cw, magnet_b200.est_costvolume_CW(dvol.to(dt).float(), f32[:1], f32[1:], inp.ref_gmms,
                                              inp.nghbr_gmms.to(dt).float(), inp.R, inp.t, inp.is_valid,
                                              inp.cam_intrins, 5), "install CW")
        _eq(fv, magnet_b200.est_costvolume_F(dc, f32[:1], f32[1:], inp.R, inp.t, inp.is_valid, inp.cam_intrins),
            "install F")


class _DNet(nn.Module):
    """D-Net stand-in: imgs -> ((N,2,h,w) positive [mu, sigma], (N,16,h,w) x_d3), as DNET.py:62-67."""

    def __init__(self):
        super().__init__()
        self.g, self.x = nn.Conv2d(3, 2, 1), nn.Conv2d(3, 16, 1)

    def forward(self, imgs):
        y = self.g(imgs)
        return torch.cat([y[:, :1].abs() + 1.0, y[:, 1:].abs() + 0.1], 1), self.x(imgs)


@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
def test_autocast_magnet_forward(cuda, dt):
    """MAGNET.forward under autocast: half backbone outputs, HALF16 matching, fp32 predictions equal to the head's on
    the upcast features and Gaussians."""
    torch.manual_seed(2)
    inp = make_inputs(B=2, V=2, D=32, H=16, W=24, C=64, seed=47, depth="smooth").to(cuda)
    model = magnet_b200.MAGNET(_DNet().to(cuda), nn.Conv2d(3, 64, 1).to(cuda), n_samples=32, train_iter=2, test_iter=2,
                               dnet_fdim=16).to(cuda)
    B = inp.B
    ref_img, nghbr_imgs = torch.rand(B, 3, 16, 24, device=cuda), torch.rand(2 * B, 3, 16, 24, device=cuda)
    with torch.autocast("cuda", dtype=dt), torch.no_grad():
        with _Repacks() as rp:
            preds = model(ref_img, nghbr_imgs, inp.nghbr_poses, inp.is_valid, inp.cam_intrins, mode="test")
        _took(rp, True, "MAGNET.forward")
        imgs = torch.cat((ref_img, nghbr_imgs))
        gm, x_d3 = model.d_net(imgs)
        feat = model.f_net(imgs)
        assert gm.dtype == feat.dtype == dt
        want = model.head(feat[:B].float(), feat[B:].float(), gm[:B].float(), gm[B:].float(), x_d3[:B],
                          inp.nghbr_poses, inp.is_valid, inp.cam_intrins)
    assert len(preds) == 2
    for p, w in zip(preds, want):
        assert p.shape == (B, 2, 64, 96)
        _eq(p, w, "MAGNET prediction")


@pytest.mark.parametrize("dt", DTYPES, ids=DT_IDS)
def test_depth_metrics_update_under_autocast(cuda, dt):
    torch.manual_seed(3)
    B, h, w, k = 2, 12, 16, 4
    preds = [torch.rand(B, 2, h, w, device=cuda) * 5 + 0.2 for _ in range(2)]
    mask = torch.randn(B, 9 * k * k, h, w, device=cuda)
    gt = torch.rand(B, 1, k * h, k * w, device=cuda) * 9
    m_h, m_f = magnet_b200.DepthMetrics(0.1, 8.0), magnet_b200.DepthMetrics(0.1, 8.0)
    with torch.autocast("cuda", dtype=dt):
        rows_h = m_h.update([p.to(dt) for p in preds], gt, up_mask=mask.to(dt), k=k)
    rows_f = m_f.update([p.to(dt).float() for p in preds], gt, up_mask=mask.to(dt).float(), k=k)
    assert rows_h.dtype == torch.float64
    assert np.array_equal(rows_h.cpu().numpy(), rows_f.cpu().numpy(), equal_nan=True)
    assert m_h.value(all_predictions=True) == m_f.value(all_predictions=True)


# ------------------------------------------------------------------------------------------------------------------
def test_half16_forward_backward_is_graph_replayable(cuda):
    inp = make_inputs(B=2, V=3, D=64, H=24, W=40, C=64, seed=93, depth="smooth").to(cuda)
    ref, src = inp.ref_feat.to(torch.bfloat16), inp.nghbr_feat.to(torch.bfloat16)
    plan = magnet_b200.MatchingPlan(inp.ref_feat, inp.nghbr_feat, inp.nghbr_gmms, inp.nghbr_poses, inp.is_valid,
                                    inp.cam_intrins)
    rs, ss = ops.repack_half16(ref), ops.repack_half16(src)
    planes = ops.k_array(torch.linspace(0.5, 6.0, 64).tolist())
    vol = torch.empty(2, 64, 24, 40, device=cuda)
    gout = torch.randn(2, 64, 24, 40, device=cuda)

    def step():
        ops.cost_volume(ref, ss, plan.rays, plan.cams, V=3, src_layout=_lib.SRC_HALF16, consistency=False, k=planes,
                        planes=True, out=vol, ref_split=rs)
        return ops.cost_volume_f_bwd(ref, src, plan.rays, plan.cams, planes, 3, None, gout, softmax=False,
                                     ref_split=rs, src_split=ss, split_layout=_lib.SRC_HALF16)

    step()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        g_ref, g_src = step()
    for rep_ in range(3):
        gout.copy_(torch.randn_like(gout))
        graph.replay()
        torch.cuda.synchronize()
        got = (vol.clone(), g_ref.clone(), g_src.clone())
        want = (vol.clone(),) + step()
        torch.cuda.synchronize()
        assert torch.equal(got[0], want[0]), rep_
        for a, b in zip(got[1:], want[1:]):     # grad_src is summed with atomics: not bit-reproducible
            assert float((a - b).abs().max()) <= 1e-5 * float(b.abs().max()), rep_


def test_buffer_kind_is_checked_before_launch(cuda):
    inp = make_inputs(B=1, V=2, D=32, H=8, W=16, C=64, seed=94).to(cuda)
    plan = magnet_b200.MatchingPlan(inp.ref_feat, inp.nghbr_feat, inp.nghbr_gmms, inp.nghbr_poses, inp.is_valid,
                                    inp.cam_intrins)
    h = inp.ref_feat.half()
    s16 = (ops.repack_split16(inp.ref_feat), ops.repack_split16(inp.nghbr_feat))
    h16 = (ops.repack_half16(h), ops.repack_half16(inp.nghbr_feat.half()))
    kw = dict(V=2, consistency=False, k=inp.k.tolist(), planes=True)
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    with pytest.raises(_lib.MagnetError):
        ops.cost_volume(h, s16[1], plan.rays, plan.cams, src_layout=_lib.SRC_HALF16, ref_split=s16[0], **kw)
    with pytest.raises(_lib.MagnetError):
        ops.cost_volume(inp.ref_feat, h16[1], plan.rays, plan.cams, src_layout=_lib.SRC_SPLIT16, ref_split=h16[0], **kw)
    with pytest.raises(_lib.MagnetError):
        ops.cost_volume(h, h16[1], plan.rays, plan.cams, src_layout=_lib.SRC_HALF16, ref_split=s16[0], **kw)
    assert _lib.launch_count() == n0


def test_no_hypothesis_origin_outside_its_window_box_half16(cuda):
    lib = _build.build(defines=("MAGNET_MMA_DEBUG",), tag="mmadbg")
    env = dict(os.environ, MAGNET_B200_LIB=str(lib))
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "half_box_probe.py")], env=env, cwd=ROOT,
                       capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    assert len(res) == 48
    outside = {case: c[0] for case, c in res.items() if c[0] != 0}
    assert not outside, outside
