"""F-Net training on the GPU: MagnetF, the fused soft-argmin L1 loss and the tensor-core backward of the plane-sweep
volume, against the reference's frozen training step, the CUDA-core backward kernel and autograd of the ATen port."""
import numpy as np
import pytest
import torch

import magnet_b200
from magnet_b200 import _lib, ops
from magnet_b200.homography import plane_sweep_f
from magnet_b200.synthetic import make_inputs
from oracle import torch_ref
from tests.fnet_ref import FNET_MAX_DEPTH, FNET_MIN_DEPTH, fnet_l1_loss, sid_centres
from tests.util import golden_inputs

pytestmark = pytest.mark.gpu


def _close(got, want, rel=2e-4, what=""):
    err, scale = float((got - want).abs().max()), float(want.abs().max())
    assert err <= rel * scale, (what, err, scale)


def _setup(inp, dev):
    g = inp.to(dev)
    cams = ops.pack_cameras(inp.cam_intrins['intM'].to(dev), g.R, g.t, inp.is_valid.to(dev, torch.int32))
    rays = inp.cam_intrins['unit_ray_array_2D'].to(dev).contiguous()
    return g, cams, rays


def test_magnetf_loss_and_gradients_match_reference_golden(cuda):
    z, inp = golden_inputs("fnet_train")
    g = inp.to(cuda)
    d_center = torch.from_numpy(z["planes"]).to(cuda).view(1, -1, 1, 1)
    ref, src = g.ref_feat.clone().requires_grad_(True), g.nghbr_feat.clone().requires_grad_(True)
    scores = plane_sweep_f(d_center, ref, src, g.R, g.t, inp.is_valid, inp.cam_intrins, softmax=False)
    gt = torch.from_numpy(z["gt_dmap"]).to(cuda)
    gt = torch.nn.functional.interpolate(torch.where(gt > FNET_MAX_DEPTH, torch.zeros_like(gt), gt), size=[12, 20],
                                         mode="nearest")
    loss = ops.fnet_l1_loss(scores, z["planes"].tolist(), gt, gt > FNET_MIN_DEPTH)
    loss.backward()
    assert abs(loss.item() - float(z["loss"])) <= 2e-4 * abs(float(z["loss"]))
    _close(ref.grad.cpu(), torch.from_numpy(z["g_ref"]), what="ref")
    _close(src.grad.cpu(), torch.from_numpy(z["g_src"]), what="src")


FUZZ = [  # (seed, B, V, H, W, D, planes, invalid, ref scale, src scale)
    (1, 1, 2, 13, 21, 32, "sid", [], 1.0, 1.0),
    (2, 2, 4, 19, 30, 80, "sid", [(1, 2)], 1e-3, 1e3),
    (3, 1, 6, 17, 35, 96, "linear", [(0, 0), (0, 4)], 1e3, 1e-3),
    (4, 2, 3, 11, 26, 256, "sid", [], 1.0, 1e2),
    (5, 1, 5, 24, 19, 80, "behind", [(0, 1)], 1e-2, 1.0),
]


def _planes(kind, D):
    if kind == "sid":
        return sid_centres(1e-3, 10.0, D).reshape(-1).tolist()
    if kind == "behind":                              # negative depths: behind both cameras
        return np.linspace(-3.0, 6.0, D).astype(np.float32).tolist()
    return np.linspace(0.3, 8.0, D).astype(np.float32).tolist()


@pytest.mark.parametrize("case", FUZZ, ids=[f"seed{c[0]}" for c in FUZZ])
def test_tensor_core_backward_fuzz_against_cuda_core_kernel(cuda, case):
    seed, B, V, H, W, D, kind, invalid, sr, ss = case
    inp = make_inputs(B=B, V=V, D=8, H=H, W=W, C=64, seed=seed, depth="smooth", invalid=invalid)
    g, cams, rays = _setup(inp, cuda)
    ref, src = (g.ref_feat * sr).contiguous(), (g.nghbr_feat * ss).contiguous()
    planes = _planes(kind, D)
    gen = torch.Generator(device=cuda).manual_seed(seed)
    gout = torch.randn(B, D, H, W, device=cuda, generator=gen) * 10.0 ** (6 * torch.rand(B, D, H, W, device=cuda, generator=gen) - 3)
    rs, sp = ops.repack_split16(ref), ops.repack_split16(src)
    gr_tc, gs_tc = ops.cost_volume_f_bwd(ref, src, rays, cams, planes, V, None, gout, softmax=False, ref_split=rs,
                                         src_split=sp)
    gr_cc, gs_cc = ops.cost_volume_f_bwd(ref, src, rays, cams, planes, V, None, gout, softmax=False)
    torch.cuda.synchronize()
    assert torch.isfinite(gr_tc).all() and torch.isfinite(gs_tc).all()
    _close(gr_tc, gr_cc, what="ref")
    _close(gs_tc, gs_cc, what="src")


@pytest.mark.parametrize("shape", [dict(B=2, V=4, H=120, W=160, max_depth=10.0, family="scannet"),
                                   dict(B=4, V=2, H=88, W=304, max_depth=80.0, family="kitti")],
                         ids=["scannet", "kitti"])
def test_full_fnet_shapes_against_autograd_of_reference_ops(cuda, shape):
    B, V, H, W = shape["B"], shape["V"], shape["H"], shape["W"]
    inp = make_inputs(B=B, V=V, D=8, H=H, W=W, C=64, seed=17, depth="smooth", family=shape["family"], invalid=[(0, 1)])
    g = inp.to(cuda)
    d_center = magnet_b200.sid_planes(1e-3, shape["max_depth"], 80, device=cuda)
    gout = torch.randn(B, 80, H, W, device=cuda)
    r1, s1 = g.ref_feat.clone().requires_grad_(True), g.nghbr_feat.clone().requires_grad_(True)
    (plane_sweep_f(d_center, r1, s1, g.R, g.t, inp.is_valid, inp.cam_intrins, softmax=False) * gout).sum().backward()
    r2, s2 = g.ref_feat.clone().requires_grad_(True), g.nghbr_feat.clone().requires_grad_(True)
    cam_d = {k: v.to(cuda) for k, v in inp.cam_intrins.items()}
    (torch_ref.cost_volume_f(d_center, r2, s2, g.R, g.t, inp.is_valid, cam_d, apply_softmax=False) * gout).sum().backward()
    _close(r1.grad, r2.grad, what="ref")
    _close(s1.grad, s2.grad, what="src")


def test_fused_loss_against_aten_expression(cuda):
    torch.manual_seed(3)
    B, D, H, W = 2, 80, 30, 41
    scores = (torch.randn(B, D, H, W, device=cuda) * 4).requires_grad_(True)
    d_center = magnet_b200.sid_planes(1e-3, 10.0, D, device=cuda)
    gt = torch.rand(B, 1, H, W, device=cuda) * 12
    gt[:, :, :5] = 0
    mask = gt > 1e-3
    loss = ops.fnet_l1_loss(scores, d_center.reshape(-1).tolist(), gt, mask)
    loss.backward()
    s2 = scores.detach().clone().requires_grad_(True)
    pred = torch.sum(torch.softmax(s2, dim=1) * d_center, dim=1, keepdim=True)
    want = torch.mean(torch.abs(pred[mask] - gt[mask]))
    want.backward()
    assert abs(loss.item() - want.item()) <= 1e-5 * want.item()
    _close(scores.grad, s2.grad, rel=1e-5, what="dscores")
    with pytest.raises(_lib.MagnetError):
        ops.fnet_l1_loss(scores, d_center.reshape(-1).tolist(), gt, torch.zeros_like(mask))


class _StandIn(torch.nn.Module):
    """A small seeded F-Net stand-in: two convolutions to 64 channels at quarter resolution."""

    def __init__(self):
        super().__init__()
        self.net = torch.nn.Sequential(torch.nn.Conv2d(3, 32, 3, stride=2, padding=1), torch.nn.ReLU(),
                                       torch.nn.Conv2d(32, 64, 3, stride=2, padding=1))

    def forward(self, x):
        return self.net(x)


def _fnet_batch(dev, B=2, V=2, h=16, w=24):
    inp = make_inputs(B=B, V=V, D=8, H=h, W=w, C=8, seed=23, depth="smooth", invalid=[(1, 1)])
    g = inp.to(dev)
    gen = torch.Generator(device=dev).manual_seed(4)
    ref_img = torch.rand(B, 3, 4 * h, 4 * w, device=dev, generator=gen)
    nghbr_imgs = torch.rand(V * B, 3, 4 * h, 4 * w, device=dev, generator=gen)
    gt = 0.5 + 6 * torch.rand(B, 1, 4 * h, 4 * w, device=dev, generator=gen)
    return inp, g, ref_img, nghbr_imgs, gt


def test_magnetf_training_step(cuda):
    inp, g, ref_img, nghbr_imgs, gt = _fnet_batch(cuda)
    d_center = magnet_b200.sid_planes(1e-3, 10.0, 80, device=cuda)
    torch.manual_seed(0)
    model = magnet_b200.MagnetF(_StandIn()).to(cuda)
    twin = magnet_b200.MagnetF(_StandIn()).to(cuda)
    twin.load_state_dict(model.state_dict())
    loss = model.loss(ref_img, nghbr_imgs, g.nghbr_poses, inp.is_valid, inp.cam_intrins, d_center, gt, 1e-3, 10.0)
    loss.backward()
    # the reference's data flow: MAGNET_F.forward with the ATen port of est_costvolume_F, then train_FNet.py's loss
    feat = twin.f_net(torch.cat((ref_img, nghbr_imgs), 0))
    cam_d = {k: v.to(cuda) for k, v in inp.cam_intrins.items()}
    vol = torch_ref.cost_volume_f(d_center, feat[:2], feat[2:], g.R, g.t, inp.is_valid, cam_d)
    want = fnet_l1_loss(vol, d_center, gt, 1e-3, 10.0)
    want.backward()
    assert abs(loss.item() - want.item()) <= 1e-4 * want.item()
    for (name, a), b in zip(model.named_parameters(), twin.parameters()):
        _close(a.grad, b.grad, what=name)
    prob = model(ref_img, nghbr_imgs, g.nghbr_poses, inp.is_valid, inp.cam_intrins, d_center)
    _close(prob.detach(), vol.detach(), rel=1e-4, what="probabilities")
    opt = torch.optim.AdamW(model.parameters(), lr=1e-3)
    losses = []
    for _ in range(5):
        opt.zero_grad()
        loss = model.loss(ref_img, nghbr_imgs, g.nghbr_poses, inp.is_valid, inp.cam_intrins, d_center, gt, 1e-3, 10.0)
        loss.backward()
        opt.step()
        losses.append(loss.item())
    assert losses[-1] < losses[0], losses


def test_loss_and_volume_backward_replay_in_a_cuda_graph(cuda):
    inp = make_inputs(B=2, V=3, D=8, H=20, W=30, C=64, seed=29, depth="smooth")
    g, cams, rays = _setup(inp, cuda)
    planes = sid_centres(1e-3, 10.0, 80).reshape(-1).tolist()
    rs, sp = ops.repack_split16(g.ref_feat), ops.repack_split16(g.nghbr_feat)
    gt = 0.5 + 6 * torch.rand(2, 1, 20, 30, device=cuda)
    mask = gt > 1.0
    count = int(mask.sum())

    def step():
        scores = ops.cost_volume(g.ref_feat, sp, rays, cams, V=3, src_layout=_lib.SRC_SPLIT16, consistency=False, k=planes,
                                 planes=True, ref_split=rs).requires_grad_(True)
        loss = ops.fnet_l1_loss(scores, planes, gt, mask, count=count)
        gsc, = torch.autograd.grad(loss, scores)
        gr, gs = ops.cost_volume_f_bwd(g.ref_feat, g.nghbr_feat, rays, cams, planes, 3, None, gsc, softmax=False,
                                       ref_split=rs, src_split=sp)
        return loss.detach(), gr, gs

    eager = step()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()                                        # warm-up on the side stream
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = step()
    for _ in range(2):
        graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(captured[0], eager[0])
    for a, b in zip(captured[1:], eager[1:]):
        _close(a, b, rel=1e-5)                         # grad_src: atomics, not bit-deterministic
