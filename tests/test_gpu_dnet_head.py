"""D-Net's fused heads on the H100 (DESIGN §3.15): DnetHead against the reference's own outputs (golden), every mu,
sigma and var element against float64 within 32 u times its bound, the epilogues bit for bit against torch, a NaN in a
hoisted first layer, run-to-run identity, the module path under grad and autocast, and MAGNET with a DnetHead d_net."""
import os

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import magnet_b200
from magnet_b200 import DnetHead, ops
from magnet_b200.synthetic import make_inputs
from tests import dnet_ref as dr

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "dnet_head.npz")
GATE = 32.0


def _head(dev, seed=0, dnet=True, in_dim=256):
    head = DnetHead(in_dim=in_dim, dnet=dnet)
    dr.seed_heads(head.depth_head, head.mask_head, seed)
    return head.to(dev).eval()


def _ws(head):
    d, m = head.depth_head, head.mask_head
    return (d[2].weight, d[2].bias, d[4].weight, d[4].bias), (m[2].weight, m[2].bias, m[4].weight, m[4].bias)


@pytest.fixture
def no_tf32():
    flag = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32 = flag


@pytest.mark.parametrize("name", list(dr.HEAD_CASES))
@pytest.mark.parametrize("fused", [True, False])
def test_golden_against_the_reference(cuda, no_tf32, name, fused):
    gold = np.load(GOLDEN)
    x = dr.head_input(name)
    for dnet in (True, False):
        head = _head("cpu", dr.HEAD_CASES[name]["seed"], dnet)
        assert str(gold[f"{name}_digest"]) == dr.digest(x.numpy(), dr.state_digest(head.depth_head, head.mask_head))
        head = head.to(cuda)
        xc = x.to(cuda)
        ctx = torch.no_grad() if fused else torch.enable_grad()
        with ctx:
            out = head(xc)
        if not dnet:
            out, feat = out
            assert feat is xc
        want = gold[f"{name}_dnet" if dnet else f"{name}_magnet"]
        assert out.shape == want.shape
        np.testing.assert_allclose(out.detach().cpu().numpy(), want, rtol=2e-4, atol=2e-5)


def _pre(B, H, W, scale, dev, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    return [scale * torch.randn(B, 128, H, W, device=dev, generator=g) for _ in range(2)]


SHAPES = [(1, 1, 1), (1, 1, 17), (2, 8, 16), (3, 13, 29), (1, 120, 160), (4, 120, 160), (1, 88, 304), (4, 88, 304),
          (20, 88, 304), (40, 120, 160)]


def _check_f64(head, pre_d, pre_m):
    dws, mws = _ws(head)
    packed = ops.pack_dnet_weights(head.depth_head, head.mask_head)
    raw = ops.dnet_depth(pre_d, packed, sigma=False)
    mono = ops.dnet_depth(pre_d, packed, sigma=True)
    up = ops.dnet_upsample(pre_m, packed, raw)
    ref = dr.depth_forward(pre_d, dws)
    r = {"mu": dr.ratio(raw[:, 0:1], ref["raw"][:, 0:1], ref["raw_bound"][:, 0:1]),
         "v": dr.ratio(raw[:, 1:2], ref["raw"][:, 1:2], ref["raw_bound"][:, 1:2]),
         "sigma": dr.ratio(mono[:, 1:2], ref["sigma"], ref["sigma_bound"])}
    assert torch.equal(mono[:, 0], raw[:, 0])
    want, bound = dr.upsample_forward(pre_m, mws, ref["raw"], ref["raw_bound"])
    r["up_mu"] = dr.ratio(up[:, 0:1], want[:, 0:1], bound[:, 0:1])
    r["var"] = dr.ratio(up[:, 1:2], want[:, 1:2], bound[:, 1:2])
    return r


@pytest.mark.parametrize("B, H, W", SHAPES)
def test_elementwise_against_float64(cuda, B, H, W):
    head = _head(cuda, seed=B * 1000 + H)
    with torch.no_grad():
        r = _check_f64(head, *_pre(B, H, W, 1.0, cuda, seed=H * W))
    assert max(r.values()) <= GATE, r


@pytest.mark.parametrize("scale", [1e-3, 1e3])
def test_elementwise_against_float64_at_input_scales(cuda, scale):
    head = _head(cuda, seed=7)
    with torch.no_grad():
        r = _check_f64(head, *_pre(2, 24, 40, scale, cuda, seed=9))
    assert max(r.values()) <= GATE, r


def test_variance_floor_below_minus_twenty(cuda):
    head = _head(cuda, seed=8)
    with torch.no_grad():
        head.depth_head[4].weight[1].zero_()
        head.depth_head[4].bias[1] = -40.0                 # raw v = -40 everywhere
        pre_d, pre_m = _pre(2, 16, 24, 1.0, cuda, seed=3)
        packed = ops.pack_dnet_weights(head.depth_head, head.mask_head)
        raw = ops.dnet_depth(pre_d, packed, sigma=False)
        assert (raw[:, 1] == -40.0).all()
        mono = ops.dnet_depth(pre_d, packed, sigma=True)
        up = ops.dnet_upsample(pre_m, packed, raw)
        r = _check_f64(head, pre_d, pre_m)
    assert max(r.values()) <= GATE, r
    # inside the image the convex weights sum to 1, so the upsampled v is -40 too; at the border the zero padding
    # drops taps and v rises
    assert (up[:, 1, 4:-4, 4:-4] == np.float32(1e-10)).all()
    assert (mono[:, 1] == np.sqrt(np.float32(1e-10))).all()


def test_epilogues_bit_for_bit(cuda):
    head = _head(cuda, seed=11)
    with torch.no_grad():
        pre_d, pre_m = _pre(3, 20, 36, 1.0, cuda, seed=12)
        packed = ops.pack_dnet_weights(head.depth_head, head.mask_head)
        raw = ops.dnet_depth(pre_d, packed, sigma=False)
        mono = ops.dnet_depth(pre_d, packed, sigma=True)
        assert torch.equal(mono[:, 1:2], torch.sqrt(F.elu(raw[:, 1:2]) + 1.0 + 1e-10))
        # logits exactly b3: pre_m <= 0 and b1 <= 0 make the hidden layer zero
        head.mask_head[2].bias.copy_(-head.mask_head[2].bias.abs())
        packed = ops.pack_dnet_weights(head.depth_head, head.mask_head)
        up = ops.dnet_upsample(-pre_m.abs(), packed, raw)
        b3 = head.mask_head[4].bias.view(1, 144, 1, 1).expand(3, 144, 20, 36).contiguous()
        want = ops.convex_upsample(raw, b3, 4)
        assert torch.equal(up[:, 0], want[:, 0])
        assert torch.equal(up[:, 1:2], F.elu(want[:, 1:2]) + 1.0 + 1e-10)


def test_nan_poisons_only_its_pixel_and_runs_are_identical(cuda):
    head = _head(cuda, seed=13)
    with torch.no_grad():
        pre_d, pre_m = _pre(2, 16, 24, 1.0, cuda, seed=14)
        packed = ops.pack_dnet_weights(head.depth_head, head.mask_head)
        raw = ops.dnet_depth(pre_d, packed, sigma=False)
        up = ops.dnet_upsample(pre_m, packed, raw)
        assert torch.equal(raw, ops.dnet_depth(pre_d, packed, sigma=False))
        assert torch.equal(up, ops.dnet_upsample(pre_m, packed, raw))
        assert torch.isfinite(raw).all() and torch.isfinite(up).all()
        bad = pre_d.clone()
        bad[1, 5, 7, 9] = float("nan")
        r2 = ops.dnet_depth(bad, packed, sigma=False)
        mask = torch.zeros_like(raw, dtype=torch.bool)
        mask[1, :, 7, 9] = True
        assert torch.isnan(r2[mask]).all() and torch.equal(r2[~mask], raw[~mask])
        bad = pre_m.clone()
        bad[0, 100, 3, 4] = float("nan")
        u2 = ops.dnet_upsample(bad, packed, raw)
        block = torch.zeros_like(up, dtype=torch.bool)
        block[0, :, 12:16, 16:20] = True
        assert torch.isnan(u2[block]).all() and torch.equal(u2[~block], up[~block])


def test_module_path_under_grad_and_autocast(cuda):
    for dnet in (True, False):
        head = _head(cuda, seed=15, dnet=dnet)
        x = torch.rand(2, 256, 12, 20, device=cuda)
        calls = []
        hook = head.depth_head.register_forward_hook(lambda *a: calls.append(1))
        out = head(x)                                            # parameters require grad: the module chain
        assert len(calls) == 1
        first = out if dnet else out[0]
        first.sum().backward()
        assert head.depth_head[2].weight.grad is not None
        depth = head.depth_head(x).detach()
        if dnet:
            up = ops.convex_upsample(depth, head.mask_head(x).detach(), 4)
            want = torch.cat([up[:, :1], F.elu(up[:, 1:]) + 1.0 + 1e-10], 1)
        else:
            want = torch.cat([depth[:, :1], torch.sqrt(F.elu(depth[:, 1:]) + 1.0 + 1e-10)], 1)
        assert torch.equal(first.detach(), want)
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
            from magnet_b200.matcher import fused_dnet_applies
            assert not fused_dnet_applies(head.depth_head, head.mask_head if dnet else None, x, 4)
            a = head(x)
            a = a if dnet else a[0]
            d = head.depth_head(x)
            if dnet:
                up = ops.convex_upsample(d.float(), head.mask_head(x).float(), 4)
                want = torch.cat([up[:, :1], F.elu(up[:, 1:]) + 1.0 + 1e-10], 1)
            else:
                want = torch.cat([d[:, :1], torch.sqrt(F.elu(d[:, 1:]) + 1.0 + 1e-10)], 1)
        assert torch.equal(a, want)
        hook.remove()


class _Trunk(nn.Module):
    """Stands for the EfficientNet encoder + DenseDepth decoder: images -> (N, 64, H/4, W/4) features."""

    def __init__(self):
        super().__init__()
        self.c = nn.Conv2d(3, 64, 4, stride=4)

    def forward(self, imgs):
        return F.relu(self.c(imgs))


class _ModuleHead(nn.Module):
    """DnetHead(dnet=False) forced onto the module chain: the reference's depth_head + activation_G_magnet."""

    def __init__(self, head):
        super().__init__()
        self.h = head

    def forward(self, x):
        d = self.h.depth_head(x)
        return torch.cat([d[:, :1], torch.sqrt(F.elu(d[:, 1:]) + 1.0 + 1e-10)], 1), x


def test_magnet_with_a_dnet_head(cuda):
    inp = make_inputs(B=2, V=2, D=5, H=16, W=24, C=64, seed=11, depth="smooth").to(cuda)
    torch.manual_seed(17)
    trunk, fnet = _Trunk().to(cuda), nn.Conv2d(3, 64, 4, stride=4).to(cuda)
    head = DnetHead(in_dim=64, dnet=False).to(cuda)
    with torch.no_grad():
        # W2 = 0: the raw output is b2 exactly on both paths (a rounding difference in the mono Gaussians would move
        # the hypotheses and the piecewise-constant consistency mask), so the two models must agree bit for bit
        head.depth_head[4].weight.zero_()
        head.depth_head[4].bias.copy_(torch.tensor([3.0, -0.5]))
    ref_img, nghbr_imgs = torch.rand(2, 3, 64, 96, device=cuda), torch.rand(4, 3, 64, 96, device=cuda)
    outs, calls = [], []
    hook = head.depth_head.register_forward_hook(lambda *a: calls.append(1))
    for d_net in (nn.Sequential(trunk, head), nn.Sequential(trunk, _ModuleHead(head))):
        torch.manual_seed(18)
        model = magnet_b200.MAGNET(d_net, fnet, n_samples=5, dnet_fdim=64).to(cuda).eval()
        with torch.no_grad():
            outs.append(model(ref_img, nghbr_imgs, inp.nghbr_poses, inp.is_valid, inp.cam_intrins, mode="test"))
    hook.remove()
    assert len(calls) == 1                                       # only the module arm ran the depth_head chain
    assert outs[0][0].shape == (2, 2, 64, 96)
    for g, w in zip(*outs):
        assert torch.equal(g, w)
