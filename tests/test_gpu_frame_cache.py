"""Sequence evaluation end to end (DESIGN §3.17): MAGNET.forward_frames against MAGNET.forward on the gathered batch,
and FrameCache against the per-sample loop of test_MaGNet (backbone passes, predictions, eviction, DepthMetrics).

The stand-in backbones run image by image inside the equality tests: cuDNN may pick another algorithm for another
batch size, and the frames then differ in their last bits before the matching starts."""
import pytest
import torch
import torch.nn as nn

import magnet_b200
from magnet_b200 import DnetHead, FrameCache, ops
from magnet_b200.synthetic import quarter_res_camera, scannet_sequence, trajectory

pytestmark = pytest.mark.gpu
H, W = 96, 128                                     # images; the matching runs at 24x32


class StandInD(nn.Module):
    """(N,3,H,W) -> ((N,2,H/4,W/4) [mu, sigma > 0], (N,256,H/4,W/4)); with ``head`` a DnetHead(dnet=False) after a
    trunk instead."""

    def __init__(self, head=False):
        super().__init__()
        self.trunk = nn.Conv2d(3, 256, 4, stride=4)
        self.a = nn.Conv2d(256, 2, 1)
        self.head = DnetHead(in_dim=256, dnet=False) if head else None
        if head:
            with torch.no_grad():
                self.head.depth_head[4].weight.mul_(0.01)
                self.head.depth_head[4].bias.copy_(torch.tensor([2.5, -1.0]))

    def forward(self, x):
        f = torch.relu(self.trunk(x))
        if self.head is not None:
            return self.head(f)
        g = self.a(f)
        return torch.cat([2.5 + 0.5 * torch.tanh(g[:, :1]), 0.2 + 0.05 * torch.sigmoid(g[:, 1:])], 1), f


class PerImage(nn.Module):
    """Runs the wrapped backbone on one image at a time and counts the images."""

    def __init__(self, net):
        super().__init__()
        self.net, self.images = net, 0

    def forward(self, x):
        self.images += x.shape[0]
        outs = [self.net(x[i:i + 1]) for i in range(x.shape[0])]
        if isinstance(outs[0], tuple):
            return tuple(torch.cat(o, 0) for o in zip(*outs))
        return torch.cat(outs, 0)


def _model(cuda, per_image=True, dnet_head=False, fused_upsample=False, seed=0):
    torch.manual_seed(seed)
    d, f = StandInD(dnet_head), nn.Conv2d(3, 64, 4, stride=4)
    if per_image:
        d, f = PerImage(d), PerImage(f)
    return magnet_b200.MAGNET(d, f, n_samples=5, test_iter=3, fused_upsample=fused_upsample).to(cuda).eval()


def _sequence(cuda, n_refs, seed=0):
    """A ScanNet-like sequence: frame images, the references and their neighbours (the loader's rule), extrinsics of
    a generated trajectory and the quarter-resolution intrinsics."""
    refs, nghbrs = scannet_sequence(n_refs)
    ids = sorted(set(refs) | set(f for row in nghbrs for f in row))
    g = torch.Generator().manual_seed(seed)
    imgs = {f: torch.rand(3, H, W, generator=g).to(cuda) for f in ids}
    ext = {f: torch.from_numpy(e).to(cuda) for f, e in trajectory(ids, seed).items()}
    K, rays = quarter_res_camera(H // 4, W // 4)
    return refs, nghbrs, imgs, ext, torch.from_numpy(K), torch.from_numpy(rays)


def _batch(seq, samples):
    """forward's arguments for the given samples of the sequence (neighbours view-major)."""
    refs, nghbrs, imgs, ext, K, rays = seq
    B, V = len(samples), len(nghbrs[0])
    ref_img = torch.stack([imgs[refs[s]] for s in samples])
    nghbr_imgs = torch.stack([imgs[nghbrs[s][v]] for v in range(V) for s in samples])
    poses, valid = ops.relative_poses(torch.stack([ext[refs[s]] for s in samples]),
                                      torch.stack([torch.stack([ext[nghbrs[s][v]] for s in samples]) for v in range(V)]))
    intr = {"intM": K[None].repeat(B, 1, 1), "unit_ray_array_2D": rays[None].repeat(B, 1, 1)}
    return ref_img, nghbr_imgs, poses, valid.cpu(), intr


@pytest.mark.parametrize("dnet_head,fused_upsample", [(False, False), (True, False), (False, True), (True, True)])
def test_forward_frames_equals_forward(cuda, dnet_head, fused_upsample):
    seq = _sequence(cuda, 10, seed=1)
    refs, nghbrs, imgs = seq[0], seq[1], seq[2]
    samples = list(range(1, 9))                    # B = 8 consecutive references
    model = _model(cuda, dnet_head=dnet_head, fused_upsample=fused_upsample)
    ref_img, nghbr_imgs, poses, valid, intr = _batch(seq, samples)
    ids = sorted(set(refs[s] for s in samples) | set(f for s in samples for f in nghbrs[s]))
    pos = {f: i for i, f in enumerate(ids)}
    frames = torch.stack([imgs[f] for f in ids])
    ref_index = torch.tensor([pos[refs[s]] for s in samples])
    src_index = torch.tensor([[pos[f] for f in nghbrs[s]] for s in samples], dtype=torch.int32)
    with torch.no_grad():
        want = model(ref_img, nghbr_imgs, poses, valid, intr, mode="test")
        n_forward = model.d_net.images
        got = model.forward_frames(frames, ref_index, src_index, poses, valid, intr, mode="test")
    assert model.d_net.images - n_forward == len(ids) < n_forward
    assert len(got) == len(want) == 3 and got[0].shape == (8, 2, H, W)
    for a, b in zip(got, want):
        assert torch.equal(a, b)


def test_forward_frames_batched_backbones_within_parity_tolerance(cuda):
    seq = _sequence(cuda, 10, seed=2)
    refs, nghbrs, imgs = seq[0], seq[1], seq[2]
    samples = list(range(8))
    model = _model(cuda, per_image=False)
    ref_img, nghbr_imgs, poses, valid, intr = _batch(seq, samples)
    ids = sorted(set(refs[s] for s in samples) | set(f for s in samples for f in nghbrs[s]))
    pos = {f: i for i, f in enumerate(ids)}
    with torch.no_grad():
        want = model(ref_img, nghbr_imgs, poses, valid, intr, mode="test")
        got = model.forward_frames(torch.stack([imgs[f] for f in ids]), torch.tensor([pos[refs[s]] for s in samples]),
                                   torch.tensor([[pos[f] for f in nghbrs[s]] for s in samples]), poses, valid, intr)
    for a, b in zip(got, want):
        d = (a - b).abs()
        assert float(d.median()) <= 1e-5 * float(b.abs().max())
        assert float((d > 1e-3 * float(b.abs().max())).float().mean()) < 2e-3


def _loop(seq, run, gt, metrics):
    refs, nghbrs = seq[0], seq[1]
    preds = []
    with torch.no_grad():
        for s in range(len(refs)):
            ref_img, nghbr_imgs, poses, valid, intr = _batch(seq, [s])
            out = run(s, ref_img, nghbr_imgs, poses, valid, intr)
            preds.append(out)
            metrics.update(out[-1], gt[s:s + 1])
    return preds


@pytest.mark.parametrize("capacity", [128, 3])
def test_frame_cache_matches_the_per_sample_loop(cuda, capacity):
    """60 references under the loader's rule: one backbone pass per distinct frame while the capacity holds them all
    (128 > the 66 distinct frames), recomputation of evicted frames with a capacity below one window (3); predictions
    and DepthMetrics equal the per-sample loop's."""
    seq = _sequence(cuda, 60, seed=3)
    refs, nghbrs = seq[0], seq[1]
    distinct = set(refs) | set(f for row in nghbrs for f in row)
    g = torch.Generator().manual_seed(4)
    gt = (0.5 + 4.0 * torch.rand(len(refs), 1, H, W, generator=g)).to(cuda)
    model = _model(cuda, seed=5)
    m_want = magnet_b200.DepthMetrics(min_depth=1e-3, max_depth=10.0)
    want = _loop(seq, lambda s, *a: model(*a, mode="test"), gt, m_want)
    assert model.d_net.images == 5 * len(refs)

    cache = FrameCache(model, capacity=capacity)
    model.d_net.images = model.f_net.images = 0
    m_got = magnet_b200.DepthMetrics(min_depth=1e-3, max_depth=10.0)
    got = _loop(seq, lambda s, *a: cache(*a, [refs[s]], [nghbrs[s]], mode="test"), gt, m_got)
    if capacity >= len(distinct):
        assert model.d_net.images == model.f_net.images == len(distinct) == cache.backbone_images
    else:
        assert len(distinct) < model.d_net.images < 5 * len(refs)
        assert len(cache) == capacity
    for a, b in zip(got, want):
        for x, y in zip(a, b):
            assert torch.equal(x, y)
    assert m_got.images() == m_want.images() == len(refs)
    assert m_got.value(all_predictions=True) == m_want.value(all_predictions=True)
    cache.clear()
    assert len(cache) == 0
