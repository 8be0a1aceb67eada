"""Autograd of the consistency-weighted cost volume on the GPU: the drop-in est_costvolume_CW and MatchingPlan.cost
against the reference's frozen backward, autograd of the ATen port at full size, the linearity identities that prove the
backward applied the forward's consistency mask, a MagnetHead step with a trainable F-Net stand-in, and CUDA graphs."""
import numpy as np
import pytest
import torch

import magnet_b200
from magnet_b200 import _lib, ops
from magnet_b200.synthetic import CONFIGS, make_inputs
from oracle import torch_ref
from tests.util import FLIP_BUDGET, MARGIN_TOL, golden_inputs

pytestmark = pytest.mark.gpu

PATHS = {"mma": _lib.VARIANT_MMA, "direct": _lib.VARIANT_DIRECT}


def _leaves(g, dv):
    return (dv.clone().requires_grad_(True), g.ref_feat.clone().requires_grad_(True),
            g.nghbr_feat.clone().requires_grad_(True))


def _drop_in(inp, g, dv, ref, src, variant=_lib.VARIANT_AUTO):
    return magnet_b200.est_costvolume_CW(dv, ref, src, g.ref_gmms, g.nghbr_gmms, g.R, g.t, inp.is_valid,
                                         inp.cam_intrins, inp.thres, variant=variant)


def _grads(inp, g, dv0, gout, variant):
    dv, ref, src = _leaves(g, dv0)
    out = _drop_in(inp, g, dv, ref, src, variant)
    (out * gout).sum().backward()
    return out.detach(), dv.grad, ref.grad, src.grad


def _near_px(near):
    """(B,D,H,W) near-threshold flags -> (B,1,H,W): a pixel one of whose hypotheses is near the threshold."""
    return near.any(dim=1, keepdim=True)


def _check(got, want, rel, what, exclude=None):
    got, want = got.double(), want.double()
    scale = float(want.abs().max())
    bad = (got - want).abs() > rel * scale
    if exclude is not None:
        bad &= ~exclude
    assert not bad.any(), (what, int(bad.sum()), float((got - want).abs().max()), scale)


@pytest.mark.parametrize("path", sorted(PATHS))
def test_drop_in_gradients_match_reference_golden(cuda, path):
    z, inp = golden_inputs("cw_train")
    g = inp.to(cuda)
    gout = torch.from_numpy(z["gout"]).to(cuda)
    _, gd, gr, gs = _grads(inp, g, g.depth_volume(), gout, PATHS[path])
    margin = torch_ref.cw_threshold_margin(inp.depth_volume(), inp.nghbr_gmms, inp.R, inp.t, inp.is_valid,
                                           inp.cam_intrins, inp.thres).to(cuda)
    # the golden case has no element near the threshold: every gradient is compared without exclusions
    assert not (margin <= MARGIN_TOL).any()
    _check(gr, torch.from_numpy(z["g_ref"]).to(cuda), 2e-4, "ref")
    _check(gd, torch.from_numpy(z["g_depth"]).to(cuda), 1e-3, "depth")
    _check(gs, torch.from_numpy(z["g_src"]).to(cuda), 2e-4, "src")


def _full(cfg, seed, B=None):
    kw = dict(CONFIGS[cfg])
    if B is not None:
        kw["B"] = B
    return make_inputs(**kw, seed=seed, invalid=[(0, 3)])


@pytest.mark.parametrize("path", sorted(PATHS))
@pytest.mark.parametrize("cfg", ["cfg2", "cfg3"])
def test_mask_identity_per_pixel_full_shape(cuda, cfg, path):
    """The volume is linear in ref_feat (and in the source maps) for a fixed mask, so sum_c grad_ref*ref equals
    sum_j gout*out at every pixel and <grad_src, src> = <gout, out> globally.  A mask that differs from the forward's
    at a single hypothesis moves a pixel's sum by |gout_j * cost_j|, far above the tolerance."""
    inp = _full(cfg, seed=7)
    g = inp.to(cuda)
    gen = torch.Generator(device=cuda).manual_seed(3)
    gout = torch.randn(inp.B, inp.D, inp.ref_feat.shape[2], inp.ref_feat.shape[3], device=cuda, generator=gen)
    out, _, gr, gs = _grads(inp, g, g.depth_volume(), gout, PATHS[path])
    lhs = (gr.double() * g.ref_feat.double()).sum(dim=1)
    rhs = (gout.double() * out.double()).sum(dim=1)
    bound = gout.double().abs().sum(dim=1) * out.double().abs().amax(dim=1)
    bad = (lhs - rhs).abs() > 1e-4 * bound + 1e-30
    assert not bad.any(), (cfg, path, int(bad.sum()), float(((lhs - rhs).abs() / (bound + 1e-30)).max()))
    glhs = float((gs.double() * g.nghbr_feat.double()).sum())
    grhs = float(rhs.sum())
    assert abs(glhs - grhs) <= 1e-4 * float(bound.sum()), (glhs, grhs)


@pytest.mark.parametrize("cfg", ["cfg2", "cfg3"])
def test_full_shape_against_aten_autograd(cuda, cfg):
    inp = _full(cfg, seed=11, B=1)                               # the ATen arm's saved tensors at B = 1
    g = inp.to(cuda)
    gen = torch.Generator(device=cuda).manual_seed(5)
    H, W = inp.ref_feat.shape[2], inp.ref_feat.shape[3]
    gout = torch.randn(inp.B, inp.D, H, W, device=cuda, generator=gen)
    _, gd, gr, gs = _grads(inp, g, g.depth_volume(), gout, _lib.VARIANT_AUTO)
    dv, ref, src = _leaves(g, g.depth_volume())
    want = torch_ref.cost_volume_cw(dv, ref, src, g.ref_gmms, g.nghbr_gmms, g.R, g.t, inp.is_valid,
                                    {k: v.to(cuda) for k, v in inp.cam_intrins.items()}, inp.thres)
    (want * gout).sum().backward()
    margin = torch_ref.cw_threshold_margin(g.depth_volume(), g.nghbr_gmms, g.R, g.t, inp.is_valid,
                                           {k: v.to(cuda) for k, v in inp.cam_intrins.items()}, inp.thres)
    near = margin <= MARGIN_TOL
    # the bilinear derivative jumps across a cell edge: exclude depth-gradient elements within 1e-4 px of one
    edge = torch.zeros_like(near)
    intr = {k: v.to(cuda) for k, v in inp.cam_intrins.items()}
    for v in range(inp.V):
        if int(inp.is_valid[0, v]) != 1:
            continue
        K, rays = intr['intM'][0], intr['unit_ray_array_2D'][0]
        P = (K @ g.t[0, v]).view(1, 3, 1) + (K @ g.R[0, v] @ rays).unsqueeze(0) * g.depth_volume()[0].view(inp.D, 1, -1)
        P = P / (P[:, 2:3] + 1e-10)
        for c, n in ((0, W), (1, H)):
            pos = P[:, c] - 0.5
            frac = pos - torch.floor(pos)
            edge |= (torch.minimum(frac, 1 - frac) < 1e-4).view(1, inp.D, H, W)
    print(cfg, "near threshold:", int(near.sum()), "near a cell edge:", int(edge.sum()), "of", near.numel())
    # a mask flip between the two forwards (rounding of the sample position / of mu~, sigma~) moves every channel of
    # grad_ref at that pixel: elementwise, such pixels are counted against the flip budget of the volume comparisons
    bad = (gr - ref.grad).abs() > 2e-4 * ref.grad.abs().max()
    bad &= ~_near_px(near)
    bad_px = bad.any(dim=1)
    print(cfg, "grad_ref pixels beyond 2e-4 outside the margin:", int(bad_px.sum()), "min margin there:",
          float(margin.amin(dim=1)[bad_px].min()) if bad_px.any() else None)
    assert int(bad_px.sum()) <= max(1, FLIP_BUDGET * margin.numel()), int(bad_px.sum())
    assert float((gr - ref.grad).norm() / ref.grad.norm()) <= 1e-3
    _check(gd, dv.grad, 1e-3, "depth", near | edge | bad_px.unsqueeze(1))
    err = float((gs - src.grad).norm() / src.grad.norm())
    assert err <= 1e-3, err


FUZZ = [  # (seed, B, V, H, W, D, depths, invalid, ref scale, src scale, mode)
    (1, 1, 2, 13, 21, 32, "smooth", [], 1.0, 1.0, "volume"),
    (2, 2, 4, 19, 30, 80, "random", [(1, 2)], 1e-3, 1e3, "volume"),
    (3, 1, 6, 17, 35, 96, "smooth", [(0, 0), (0, 4)], 1e3, 1e-3, "gauss"),
    (4, 2, 3, 11, 26, 256, "random", [], 1.0, 1e2, "volume"),
    (5, 1, 5, 24, 19, 64, "behind", [(0, 1)], 1e-2, 1.0, "volume"),
    (6, 2, 4, 16, 24, 40, "smooth", [(1, 0)], 1.0, 1.0, "gauss"),
]


@pytest.mark.parametrize("case", FUZZ, ids=[f"seed{c[0]}" for c in FUZZ])
def test_tensor_core_backward_fuzz_against_cuda_core_kernel(cuda, case):
    """Feature gradients of the tensor-core kernel (on the split buffers) against the CUDA-core kernel, both applying the
    tensor-core forward's mask: the masks are the same computation on the same inputs, so no element may disagree."""
    seed, B, V, H, W, D, kind, invalid, sr, ss, mode = case
    inp = make_inputs(B=B, V=V, D=8, H=H, W=W, C=64, seed=seed, depth="smooth", invalid=invalid)
    g = inp.to(cuda)
    cams = ops.pack_cameras(inp.cam_intrins['intM'].to(cuda), g.R, g.t, inp.is_valid.to(cuda, torch.int32))
    rays = inp.cam_intrins['unit_ray_array_2D'].to(cuda).contiguous()
    ref, src = (g.ref_feat * sr).contiguous(), (g.nghbr_feat * ss).contiguous()
    gen = torch.Generator(device=cuda).manual_seed(seed)
    gout = torch.randn(B, D, H, W, device=cuda, generator=gen) * 10.0 ** (6 * torch.rand(B, D, H, W, device=cuda, generator=gen) - 3)
    k = np.linspace(-2.5, 2.5, D).astype(np.float32).tolist()
    dep = dict(ref_gmm=g.ref_gmms, k=k) if mode == "gauss" else {}
    if mode == "volume":
        mu = g.ref_gmms[:, :1]
        if kind == "random":
            dv = mu * (0.2 + 3 * torch.rand(B, D, H, W, device=cuda, generator=gen))
        elif kind == "behind":                                  # negative depths: behind both cameras
            dv = torch.linspace(-3.0, 6.0, D, device=cuda).view(1, D, 1, 1).expand(B, D, H, W).contiguous()
        else:
            dv = mu + g.ref_gmms[:, 1:] * torch.linspace(-2.5, 2.5, D, device=cuda).view(1, D, 1, 1)
        dep = dict(d_volume=dv.contiguous())
    rs, sp = ops.repack_split16(ref), ops.repack_split16(src, g.nghbr_gmms)
    common = dict(V=V, kappa=float(inp.thres), need_depth=False, fwd_layout=_lib.SRC_SPLIT16, fwd_variant=_lib.VARIANT_MMA)
    gr_tc, gs_tc, _ = ops.cost_volume_bwd(ref, src, g.nghbr_gmms, rays, cams, gout, ref_split=rs, src_split=sp,
                                          **common, **dep)
    gr_cc, gs_cc, _ = ops.cost_volume_bwd(ref, src, g.nghbr_gmms, rays, cams, gout, **common, **dep)
    torch.cuda.synchronize()
    assert torch.isfinite(gr_tc).all() and torch.isfinite(gs_tc).all()
    assert float(gr_cc.abs().max()) > 0
    _check(gr_tc, gr_cc, 2e-4, "ref")
    _check(gs_tc, gs_cc, 2e-4, "src")


def test_gauss_mode_chain_rule(cuda):
    """MatchingPlan.cost (sampler fused): grad_mu = sum_j grad_d_j, grad_sigma = sum_j k_j grad_d_j."""
    inp = make_inputs(B=2, V=3, D=8, H=20, W=28, C=64, seed=5, depth="smooth", invalid=[(1, 1)])
    g = inp.to(cuda)
    k = inp.k.tolist() * 5                                      # 40 hypotheses: the tensor-core forward
    for variant in (_lib.VARIANT_AUTO, _lib.VARIANT_DIRECT):
        gmm = g.ref_gmms.clone().requires_grad_(True)
        plan = magnet_b200.MatchingPlan(g.ref_feat, g.nghbr_feat, g.nghbr_gmms, g.nghbr_poses, inp.is_valid,
                                        inp.cam_intrins, thres=inp.thres)
        gen = torch.Generator(device=cuda).manual_seed(1)
        gout = torch.randn(2, len(k), 20, 28, device=cuda, generator=gen)
        (plan.cost(gmm, k, variant=variant) * gout).sum().backward()
        dv = ops.sample_depths(g.ref_gmms, k).requires_grad_(True)
        out = magnet_b200.est_costvolume_CW(dv, g.ref_feat, g.nghbr_feat, g.ref_gmms, g.nghbr_gmms, g.R, g.t,
                                            inp.is_valid, inp.cam_intrins, inp.thres,
                                            variant=_lib.VARIANT_MMA if variant == _lib.VARIANT_AUTO else variant)
        (out * gout).sum().backward()
        kk = torch.tensor(k, device=cuda).view(1, -1, 1, 1)
        want = torch.cat([dv.grad.sum(1, keepdim=True), (dv.grad * kk).sum(1, keepdim=True)], dim=1)
        _check(gmm.grad, want, 1e-4, f"gmm grad, variant {variant}")


def test_wrapper_rule(cuda):
    inp = make_inputs(B=1, V=2, D=8, H=12, W=16, C=16, seed=2, depth="smooth")
    g = inp.to(cuda)
    dv = g.depth_volume()
    out = _drop_in(inp, g, dv, g.ref_feat, g.nghbr_feat)
    assert out.grad_fn is None and not out.requires_grad
    with torch.no_grad():
        out2 = _drop_in(inp, g, dv.clone().requires_grad_(True), g.ref_feat.clone().requires_grad_(True), g.nghbr_feat)
    assert out2.grad_fn is None and torch.equal(out, out2)
    ref = g.ref_feat.clone().requires_grad_(True)
    gm = g.nghbr_gmms.clone().requires_grad_(True)
    out3 = magnet_b200.est_costvolume_CW(dv, ref, g.nghbr_feat, g.ref_gmms, gm, g.R, g.t, inp.is_valid,
                                         inp.cam_intrins, inp.thres)
    out3.sum().backward()
    assert ref.grad is not None and gm.grad is None
    R = g.R.clone().requires_grad_(True)
    with pytest.raises(_lib.MagnetError, match="R requires grad"):
        magnet_b200.est_costvolume_CW(dv, ref, g.nghbr_feat, g.ref_gmms, g.nghbr_gmms, R, g.t, inp.is_valid,
                                      inp.cam_intrins, inp.thres)
    with pytest.raises(_lib.MagnetError):
        _drop_in(inp, g, dv, ref, g.nghbr_feat, variant=_lib.VARIANT_TMA)


@pytest.fixture
def deterministic_cudnn():
    saved = torch.backends.cudnn.deterministic
    torch.backends.cudnn.deterministic = True
    yield
    torch.backends.cudnn.deterministic = saved


def test_head_step_trains_fnet_through_the_volume(cuda, deterministic_cudnn):
    torch.manual_seed(0)
    B, V, H, W = 1, 2, 16, 24
    inp = make_inputs(B=B, V=V, D=5, H=H, W=W, C=16, seed=21, depth="smooth")
    g = inp.to(cuda)
    imgs = torch.randn(B * (V + 1), 3, H, W, device=cuda)
    fnet = torch.nn.Conv2d(3, 16, 3, padding=1).to(cuda)
    head = magnet_b200.MagnetHead(n_samples=5, n_iter=2, thres=inp.thres, dnet_fdim=8, detach_cost=False).to(cuda)
    x_d3 = torch.randn(B, 8, H, W, device=cuda)
    feat = fnet(imgs)
    preds, _ = head.forward_quarter(feat[:B], feat[B:], g.ref_gmms, g.nghbr_gmms, x_d3, g.nghbr_poses,
                                    inp.is_valid, inp.cam_intrins)
    sum(p.square().mean() for p in preds).backward()
    got = [p.grad.clone() for p in fnet.parameters()]
    # the same data flow on the ATen port
    for p in list(fnet.parameters()) + list(head.parameters()):
        p.grad = None
    feat = fnet(imgs)
    intr = {k: v.to(cuda) for k, v in inp.cam_intrins.items()}
    cur, loss = g.ref_gmms, 0.0
    for _ in range(2):
        dv = torch_ref.sample_depth_candidates(cur.detach(), head.k_list)
        cv = torch_ref.cost_volume_cw(dv, feat[:B], feat[B:], g.ref_gmms, g.nghbr_gmms, g.R, g.t, inp.is_valid, intr,
                                      inp.thres)
        cur = torch_ref.gaussian_update(head.g_net.gnet(torch.cat([cv, x_d3], dim=1)), cur.detach())
        loss = loss + cur.square().mean()
    loss.backward()
    for a, b in zip(got, fnet.parameters()):
        assert float(b.grad.abs().max()) > 0
        _check(a, b.grad, 1e-3, "F-Net parameter gradient")
    # default detach_cost=True: exactly today's results and gradients, F-Net gets none
    head.detach_cost = True
    outs = []
    for f_req in (True, False):
        for p in head.parameters():
            p.grad = None
        feat = fnet(imgs) if f_req else fnet(imgs).detach()
        preds, _ = head.forward_quarter(feat[:B], feat[B:], g.ref_gmms, g.nghbr_gmms, x_d3, g.nghbr_poses,
                                        inp.is_valid, inp.cam_intrins)
        sum(p.square().mean() for p in preds).backward()
        outs.append(([p.detach() for p in preds], [p.grad for p in head.parameters()]))
    for a, b in zip(outs[0][0] + outs[0][1], outs[1][0] + outs[1][1]):
        assert (a is None and b is None) or torch.equal(a, b)
    assert all(p.grad is not None for p in head.g_net.parameters())


@pytest.mark.parametrize("path", sorted(PATHS))
def test_cuda_graph_forward_backward_replays(cuda, path):
    inp = make_inputs(B=2, V=3, D=32, H=16, W=24, C=64, seed=31, depth="smooth", invalid=[(0, 2)])
    g = inp.to(cuda)
    intr = {k: v.to(cuda) for k, v in inp.cam_intrins.items()}
    valid = inp.is_valid.to(cuda)
    st_dv = g.depth_volume().clone().requires_grad_(True)
    st_ref, st_src = g.ref_feat.clone().requires_grad_(True), g.nghbr_feat.clone().requires_grad_(True)
    st_gout = torch.randn(2, 32, 16, 24, device=cuda)

    def step():
        out = magnet_b200.est_costvolume_CW(st_dv, st_ref, st_src, g.ref_gmms, g.nghbr_gmms, g.R, g.t, valid, intr,
                                            inp.thres, variant=PATHS[path])
        return out, torch.autograd.grad((out * st_gout).sum(), (st_dv, st_ref, st_src))

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        st_out, st_grads = step()
    for seed in (1, 2):
        gen = torch.Generator(device=cuda).manual_seed(seed)
        with torch.no_grad():
            st_ref.copy_(g.ref_feat * (1 + 0.1 * torch.rand(g.ref_feat.shape, device=cuda, generator=gen)))
            st_gout.copy_(torch.randn(st_gout.shape, device=cuda, generator=gen))
        graph.replay()
        torch.cuda.synchronize()
        want_out, want = step()
        assert torch.equal(st_out, want_out.detach())
        for a, b, nm in zip(st_grads, want, ("depth", "ref", "src")):
            _check(a, b, 1e-5, f"graph replay {seed}: {nm}")
