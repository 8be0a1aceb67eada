"""The fused mask head and upsampling of inference on the H100 (DESIGN §3.12): against a float64 evaluation of the mask
head and upsample_depth_via_mask, against the cuDNN module path, op order, determinism, CUDA-graph replay, a NaN in the
hoisted first layer, and MagnetHead / MAGNET with fused_upsample on and off."""
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import magnet_b200
from magnet_b200 import ops
from magnet_b200.synthetic import make_inputs
from tests import aux_ref as ar

pytestmark = pytest.mark.gpu


def _mask_head(dev, fdim=16, seed=0):
    torch.manual_seed(seed)
    return magnet_b200.MagnetHead(dnet_fdim=fdim).mask_head.to(dev).eval()


def _f64(mh, pre0, preds):
    """The mask head after its first convolution and the convex upsampling of each prediction, in float64."""
    d = lambda t: t.detach().double()
    h = F.relu(d(pre0))
    for i in (2, 4):
        h = F.relu(F.conv2d(h, d(mh[i].weight), d(mh[i].bias)))
    mask = F.conv2d(h, d(mh[6].weight), d(mh[6].bias))
    return [ar.convex_upsample(d(p), mask, 4)[0] for p in preds]


def _module(mh, pre0, preds):
    """The module path from pre0: cuDNN 1x1 convolutions at the current TF32 flags, then convex_upsample."""
    mask = mh[2:](F.relu(pre0))
    return [ops.convex_upsample(p, mask, 4) for p in preds]


def _fused(mh, pre0, preds):
    return ops.mask_upsample(pre0, ops.pack_mask_weights(mh), preds, 4)


def _err(got, want):
    """Per channel: max |got - want| over max |want|."""
    return [float((got[:, c].double() - want[:, c]).abs().max() / want[:, c].abs().max()) for c in range(2)]


def _inputs(B, H, W, P, scale, dev, seed):
    gen = torch.Generator(device=dev).manual_seed(seed)
    pre0 = scale * torch.randn(B, 128, H, W, device=dev, generator=gen)
    preds = []
    for _ in range(P):
        mu = scale * (1.0 + torch.rand(B, 1, H, W, device=dev, generator=gen))
        sg = scale * (0.1 + torch.rand(B, 1, H, W, device=dev, generator=gen))
        preds.append(torch.cat([mu, sg], 1))
    return pre0, preds


GRIDS = [(1, 1), (7, 13), (8, 16), (120, 160), (88, 304)]
BP = [(1, 1), (3, 3), (1, 8), (3, 9)]


@pytest.mark.parametrize("scale", [1e-3, 1.0, 1e3])
@pytest.mark.parametrize("bp", BP, ids=[f"B{b}P{p}" for b, p in BP])
@pytest.mark.parametrize("grid", GRIDS, ids=[f"{h}x{w}" for h, w in GRIDS])
def test_fused_matches_float64(cuda, grid, bp, scale):
    (H, W), (B, P) = grid, bp
    mh = _mask_head(cuda, seed=H + W)
    pre0, preds = _inputs(B, H, W, P, scale, cuda, seed=H * W + B + P)
    with torch.no_grad():
        got = _fused(mh, pre0, preds)
        mod = _module(mh, pre0, preds)
    want = _f64(mh, pre0, preds)
    assert len(got) == P
    for g, m, w in zip(got, mod, want):
        assert g.shape == (B, 2, 4 * H, 4 * W) and g.dtype == torch.float32
        eg, em = _err(g, w), _err(m, w)
        for c in range(2):
            assert eg[c] <= 1e-4, f"channel {c}: fused off by {eg[c]:.2e} of its max"
            # no further from float64 than cuDNN at the default flags; where cuDNN picks a full fp32 algorithm (small
            # grids) its error is below the SPLIT16 floor, so the comparison starts at 1e-5 of the channel's max
            assert eg[c] <= max(em[c], 1e-5), f"channel {c}: fused {eg[c]:.2e} vs module path {em[c]:.2e}"


def test_op_order_matches_convex_upsample_bit_for_bit(cuda):
    """W3 = 0 and b3 exact: the logits are b3 on both paths, so the fused upsampling must equal convex_upsample."""
    mh = _mask_head(cuda, seed=3)
    with torch.no_grad():
        mh[6].weight.zero_()
        mh[6].bias.copy_((torch.randn(144, device=cuda) * 4).round() / 8)
    B, H, W = 2, 19, 37
    pre0, preds = _inputs(B, H, W, 3, 1.0, cuda, seed=4)
    with torch.no_grad():
        got = _fused(mh, pre0, preds)
        mask = mh[2:](F.relu(pre0))
    assert torch.equal(mask, mh[6].bias.view(1, 144, 1, 1).expand_as(mask))
    for g, p in zip(got, preds):
        assert torch.equal(g, ops.convex_upsample(p, mask, 4))


def test_deterministic_and_graph_capturable(cuda):
    mh = _mask_head(cuda, seed=5)
    B, H, W = 2, 40, 56
    pre0, preds = _inputs(B, H, W, 3, 1.0, cuda, seed=6)
    with torch.no_grad():
        packed = ops.pack_mask_weights(mh)
        a = ops.mask_upsample(pre0, packed, preds)
        b = ops.mask_upsample(pre0, packed, preds)
        assert all(torch.equal(x, y) for x, y in zip(a, b))
        s_pre0, s_preds = pre0.clone(), [p.clone() for p in preds]
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):                                      # warm-up outside the capture
            ops.mask_upsample(s_pre0, packed, s_preds)
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            outs = ops.mask_upsample(s_pre0, packed, s_preds)
        pre1, preds1 = _inputs(B, H, W, 3, 2.0, cuda, seed=7)           # changed inputs
        s_pre0.copy_(pre1)
        for d, p in zip(s_preds, preds1):
            d.copy_(p)
        graph.replay()
        torch.cuda.synchronize()
        eager = ops.mask_upsample(pre1, packed, preds1)
    assert all(torch.equal(x, y) for x, y in zip(outs, eager))


def test_nan_in_pre0_poisons_only_its_block(cuda):
    mh = _mask_head(cuda, seed=8)
    B, H, W = 2, 20, 36
    pre0, preds = _inputs(B, H, W, 3, 1.0, cuda, seed=9)
    bad = pre0.clone()
    bad[1, 77, 5, 17] = float("nan")
    with torch.no_grad():
        clean = _fused(mh, pre0, preds)
        dirty = _fused(mh, bad, preds)
    block = torch.zeros(B, 2, 4 * H, 4 * W, dtype=torch.bool, device=cuda)
    block[1, :, 20:24, 68:72] = True
    for c, d in zip(clean, dirty):
        assert torch.isfinite(c).all()
        assert torch.equal(~torch.isfinite(d), block)
        assert torch.equal(d[~block], c[~block])


def _head_inputs(dev, B=2, H=24, W=40, fdim=64):
    inp = make_inputs(B=B, V=2, D=5, H=H, W=W, C=64, seed=11, depth="smooth").to(dev)
    x_d3 = torch.randn(B, fdim, H, W, generator=torch.Generator().manual_seed(12)).to(dev)
    return inp, x_d3


@pytest.fixture
def no_tf32():
    flag = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32 = flag


def _close(got, want):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert g.shape == w.shape
        for c in range(2):
            err = float((g[:, c].double() - w[:, c].double()).abs().max() / w[:, c].double().abs().max())
            assert err <= 1e-4, f"channel {c} off by {err:.2e}"


def test_magnet_head_fused_upsample(cuda, no_tf32):
    inp, x_d3 = _head_inputs(cuda)
    torch.manual_seed(13)
    head = magnet_b200.MagnetHead(n_samples=5, dnet_fdim=64).to(cuda).eval()
    args = (inp.ref_feat, inp.nghbr_feat, inp.ref_gmms, inp.nghbr_gmms, x_d3, inp.nghbr_poses, inp.is_valid,
            inp.cam_intrins)
    calls = []
    hook = head.mask_head.register_forward_hook(lambda *a: calls.append(1))
    with torch.no_grad():
        want = head(*args)
        assert len(calls) == 1
        head.fused_upsample = True
        got = head(*args)
        assert len(calls) == 1                                          # the full mask is never computed
        head.fused_upsample = False
        again = head(*args)
    hook.remove()
    _close(got, want)
    assert all(torch.equal(a, b) for a, b in zip(again, want))


class _DNet(nn.Module):
    def __init__(self, fdim):
        super().__init__()
        self.c = nn.Conv2d(3, 2 + fdim, 1)

    def forward(self, imgs):
        y = self.c(F.avg_pool2d(imgs, 4))
        return torch.cat([1.0 + y[:, :1].abs(), 0.1 + y[:, 1:2].abs()], 1), y[:, 2:]


def test_magnet_fused_upsample_test_mode(cuda, no_tf32):
    inp, _ = _head_inputs(cuda, B=2, H=16, W=24)
    torch.manual_seed(14)
    dnet, fnet = _DNet(32).to(cuda), nn.Conv2d(3, 64, 4, stride=4).to(cuda)
    ref_img, nghbr_imgs = torch.rand(2, 3, 64, 96, device=cuda), torch.rand(4, 3, 64, 96, device=cuda)
    outs = []
    for fused in (False, True):
        torch.manual_seed(15)
        model = magnet_b200.MAGNET(dnet, fnet, n_samples=5, dnet_fdim=32, fused_upsample=fused).to(cuda).eval()
        with torch.no_grad():
            outs.append(model(ref_img, nghbr_imgs, inp.nghbr_poses, inp.is_valid, inp.cam_intrins, mode="test"))
    assert outs[0][0].shape == (2, 2, 64, 96)
    _close(outs[1], outs[0])


def test_fallback_is_the_module_path(cuda):
    inp, x_d3 = _head_inputs(cuda, fdim=16)
    args = (inp.ref_feat, inp.nghbr_feat, inp.ref_gmms, inp.nghbr_gmms, x_d3, inp.nghbr_poses, inp.is_valid,
            inp.cam_intrins)
    torch.manual_seed(16)
    head = magnet_b200.MagnetHead(n_samples=5, dnet_fdim=16).to(cuda)
    want = head(*args)                                                  # grad mode on, trainable mask head
    head.fused_upsample = True
    got = head(*args)
    assert all(torch.equal(a, b) for a, b in zip(got, want))
    assert got[0].requires_grad
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        head.fused_upsample = False
        want = head(*args)
        head.fused_upsample = True
        got = head(*args)
    assert all(torch.equal(a, b) for a, b in zip(got, want))
