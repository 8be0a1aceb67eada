"""The inference path under torch.compile and CUDA-graph trees (DESIGN §3.18): ``torch.library.opcheck`` on every
registered op, no graph break in the evaluation entry points, and compiled outputs equal to eager, bit for bit, with
fullgraph=True and with mode="reduce-overhead" over replays with new inputs."""
import pytest
import torch
import torch.nn as nn

import magnet_b200
from magnet_b200 import _lib, library, ops
from magnet_b200.synthetic import make_inputs

pytestmark = pytest.mark.gpu
OPS = torch.ops.magnet_b200

SMALL = dict(B=1, V=4, D=5, H=30, W=40)
CFG2 = dict(B=8, V=4, D=64, H=120, W=160)


def _batch(dev, B, V, D, H, W, seed=1):
    """Matching inputs on the device, cameras and validity included (a CUDA graph has no host inputs)."""
    inp = make_inputs(B=B, V=V, D=D, H=H, W=W, C=64, seed=seed)
    g = inp.to(dev)
    cam = {k: v.to(dev) for k, v in inp.cam_intrins.items()}
    return g, cam, inp.is_valid.to(dev), inp.k.tolist()


def _positive(*shape, dev, lo=0.5, hi=5.0, seed=0):
    gen = torch.Generator(device=dev).manual_seed(seed)
    return lo + (hi - lo) * torch.rand(*shape, device=dev, generator=gen)


def _op_cases(dev, B, V, D, H, W):
    """(op name, arguments) covering every registered op: each cost-volume layout and variant ``route`` returns, both
    depth modes and the planes, consistency on and off, and every form of the depth metrics."""
    torch.manual_seed(0)
    g, cam, valid, k = _batch(dev, B, V, D, H, W)
    rays, intM = cam["unit_ray_array_2D"], cam["intM"]
    cams = ops.pack_cameras(intM, g.R, g.t, valid)
    ref, src, gmm, sgmm = g.ref_feat, g.nghbr_feat, g.ref_gmms, g.nghbr_gmms
    planes = torch.linspace(0.5, 6.0, D).tolist()
    split, half = ops.repack_split16(src, sgmm), ops.repack_half16(src.half(), sgmm)
    rsplit, rhalf = ops.repack_split16(ref), ops.repack_half16(ref.half())
    gnet = magnet_b200.GNET(ch_in=256 + D).to(dev)
    head = magnet_b200.MagnetHead(n_samples=D).to(dev)
    dnet = magnet_b200.DnetHead().to(dev)
    (_, d1, d2), m = ops.dnet_head_layers(dnet.depth_head, dnet.mask_head)
    dw = [t.detach() for t in (d1.weight, d1.bias, d2.weight, d2.bias, m[1].weight, m[1].bias, m[2].weight, m[2].bias)]
    c = gnet.gnet
    gw = [t.detach() for t in (c[0].weight[:, :D], c[2].weight, c[2].bias, c[4].weight, c[4].bias, c[6].weight, c[6].bias)]
    mc = head.mask_head
    mw = [t.detach() for t in (mc[2].weight, mc[2].bias, mc[4].weight, mc[4].bias, mc[6].weight, mc[6].bias)]
    hid = lambda: torch.randn(B, 128, H, W, device=dev)
    full, gt = _positive(B, 2, 4 * H, 4 * W, dev=dev, seed=1), _positive(B, 1, 4 * H, 4 * W, dev=dev, hi=9.0, seed=2)
    quarter, up = _positive(B, 2, H, W, dev=dev, seed=3), torch.randn(B, 144, H, W, device=dev)
    ext = torch.eye(4, device=dev) + 0.05 * torch.randn(V + 1, B, 4, 4, device=dev)
    ext[..., 3, :] = torch.tensor([0.0, 0.0, 0.0, 1.0], device=dev)
    raw = torch.tensor([[577.87, 577.87, 319.5, 239.5, 640, 480, 0, 0]] * B, device=dev, dtype=torch.float64)
    A = _lib
    cv = lambda layout, s, *rest: (ref, s, rays, cams, V, layout, *rest)
    return [
        ("pack_cameras", (intM, g.R, g.t, valid)),
        ("relative_poses", (ext[0].contiguous(), ext[1:].contiguous())),
        ("camera_rays", (raw, H, W)),
        ("sample_depths", (gmm, k)),
        ("repack_tiled32", (src,)),
        ("repack_pixc", (src, sgmm)),
        ("repack_split16", (src, sgmm)),
        ("repack_half16", (src.half(), sgmm)),
        ("cost_volume", cv(A.SRC_TILED32, ops.repack_tiled32(src), True, sgmm, 5.0, None, gmm, k, False, False,
                           A.VARIANT_AUTO, None)),
        ("cost_volume", cv(A.SRC_TILED32, ops.repack_tiled32(src), True, sgmm, 5.0, None, gmm, k, False, False,
                           A.VARIANT_CELLS, None)),
        ("cost_volume", cv(A.SRC_NCHW, src, True, sgmm, 5.0, ops.sample_depths(gmm, k), None, None, False, False,
                           A.VARIANT_DIRECT, None)),
        ("cost_volume", cv(A.SRC_PIXC, ops.repack_pixc(src, sgmm), True, None, 5.0, ops.sample_depths(gmm, k), None,
                           None, False, False, A.VARIANT_TMA, None)),
        ("cost_volume", cv(A.SRC_PIXC, ops.repack_pixc(src), False, None, 0.0, None, None, planes, True, True,
                           A.VARIANT_TMA, None)),
        ("cost_volume", cv(A.SRC_SPLIT16, split, True, None, 5.0, None, gmm, k, False, False, A.VARIANT_MMA, rsplit)),
        ("cost_volume", cv(A.SRC_SPLIT16, split, False, None, 0.0, None, None, planes, True, False, A.VARIANT_MMA,
                           rsplit)),
        ("cost_volume", (ref.half(), half, rays, cams, V, A.SRC_HALF16, True, None, 5.0, None, gmm, k, False, False,
                         A.VARIANT_MMA, rhalf)),
        ("gaussian_update", (torch.randn(B, 2, H, W, device=dev), gmm)),
        ("pack_gnet_weights", (gw, D)),
        ("gnet_update", (torch.randn(B, D, H, W, device=dev), hid(), ops._pack_gnet(gw, D), gmm)),
        ("convex_upsample", (quarter, up, 4)),
        ("pack_mask_weights", (mw,)),
        ("mask_upsample", (hid(), ops._pack_mask(mw), [quarter, quarter * 1.5, quarter + 0.25], 4)),
        ("pack_dnet_weights", (dw[:4], 0)),
        ("pack_dnet_weights", (dw, 4)),
        ("dnet_depth", (hid(), ops._pack_dnet(dw[:4], 0), True)),
        ("dnet_upsample", (hid(), ops._pack_dnet(dw, 4), torch.randn(B, 2, H, W, device=dev), 4)),
        ("plane_depth", (torch.randn(B, D, H, W, device=dev), planes, True)),
        ("plane_depth", (torch.softmax(torch.randn(B, D, H, W, device=dev), 1), planes, False)),
        ("depth_metrics", ([full, full * 1.1], gt, 1e-3, 10.0, None, None, None, False, False)),
        ("depth_metrics", ([quarter], gt, 1e-3, 10.0, None, up, 4, False, False)),
        ("depth_metrics", ([quarter[:, :1]], gt, 1e-3, 80.0, "garg", None, None, True, False)),
        ("depth_metrics", ([full], gt, 1e-3, 10.0, "eigen", None, None, False, True)),
        ("depth_metrics_update", (torch.zeros(2, 14, device=dev, dtype=torch.float64), [quarter, quarter * 0.9], gt,
                                  1e-3, 10.0, None, up, 4, False, False)),
    ]


# The weight packs leave the padding bytes of their layouts unwritten (the fused kernels never read them), so eager and
# traced outputs are not compared byte for byte there; the fused heads' outputs under torch.compile are (test_fullgraph_*).
_UNWRITTEN_PADDING = {"pack_gnet_weights", "pack_mask_weights", "pack_dnet_weights"}


@pytest.mark.parametrize("shape", [SMALL, CFG2], ids=["small", "cfg2"])
def test_opcheck_every_op(cuda, shape):
    cases = _op_cases(cuda, **shape)
    assert {name for name, _ in cases} == set(library.OPS)
    failed = []
    for name, args in cases:
        utils = ("test_schema", "test_autograd_registration", "test_faketensor") if name in _UNWRITTEN_PADDING \
            else ("test_schema", "test_autograd_registration", "test_faketensor", "test_aot_dispatch_dynamic")
        try:
            torch.library.opcheck(getattr(OPS, name).default, args, test_utils=utils)
        except Exception as e:                         # every op is checked; all failures are reported together
            failed.append(f"{name}: {str(e)[:300]}")
    assert not failed, failed


# --- the modules under torch.compile -------------------------------------------------------------------------------

def _head(dev, n_samples, fused_upsample, seed=0):
    torch.manual_seed(seed)
    return magnet_b200.MagnetHead(n_samples=n_samples, fused_upsample=fused_upsample).to(dev).eval()


def _head_args(dev, B, V, D, H, W, seed=1):
    g, cam, valid, _ = _batch(dev, B, V, D, H, W, seed=seed)
    x_d3 = torch.randn(B, 256, H, W, device=dev, generator=torch.Generator(device=dev).manual_seed(seed))
    return (g.ref_feat, g.nghbr_feat, g.ref_gmms, g.nghbr_gmms, x_d3, g.nghbr_poses, valid, cam)


def _fnet_args(dev, B, H, W, seed=2):
    g, cam, valid, _ = _batch(dev, B, 4, 8, H, W, seed=seed)
    planes = magnet_b200.sid_planes(1e-3, 10.0, 80).flatten().tolist()
    return (g.ref_feat, g.nghbr_feat, g.nghbr_poses, valid, cam, planes)


def _metrics_args(dev, B, H, W, P=3, seed=3):
    preds = [_positive(B, 2, H, W, dev=dev, seed=seed + i) for i in range(P)]
    return preds, _positive(B, 1, 4 * H, 4 * W, dev=dev, hi=12.0, seed=seed + P), torch.randn(B, 144, H, W, device=dev)


def _breaks(fn, *args):
    torch._dynamo.reset()
    e = torch._dynamo.explain(fn)(*args)
    return e.graph_break_count, [r.reason[:200] for r in e.break_reasons]


@pytest.mark.parametrize("n_samples", [5, 64])
@pytest.mark.parametrize("fused_upsample", [False, True])
def test_magnet_head_traces_without_graph_breaks(cuda, n_samples, fused_upsample):
    head = _head(cuda, n_samples, fused_upsample)
    with torch.no_grad():
        n, why = _breaks(head, *_head_args(cuda, B=1, V=4, D=n_samples, H=30, W=40))
    assert n == 0, why


@pytest.mark.parametrize("dnet", [True, False])
def test_dnet_head_traces_without_graph_breaks(cuda, dnet):
    head = magnet_b200.DnetHead(dnet=dnet).to(cuda).eval()
    with torch.no_grad():
        n, why = _breaks(head, torch.randn(1, 256, 30, 40, device=cuda))
    assert n == 0, why


def test_magnet_f_predict_and_metrics_trace_without_graph_breaks(cuda):
    model = magnet_b200.MagnetF(nn.Identity())
    n, why = _breaks(model.predict, *_fnet_args(cuda, 1, 30, 40))
    assert n == 0, why
    metrics = magnet_b200.DepthMetrics(1e-3, 10.0)
    preds, gt, up = _metrics_args(cuda, 1, 30, 40)
    metrics.update(preds, gt, up, 4)                   # the accumulator exists from here on
    n, why = _breaks(metrics.update, preds, gt, up, 4)
    assert n == 0, why


def test_magnet_forward_traces_without_graph_breaks(cuda):
    """MAGNET.forward(mode='test') with traceable stand-in backbones: nothing of the package breaks the graph."""
    torch.manual_seed(0)
    d_net = nn.Sequential(nn.Conv2d(3, 256, 3, padding=1), magnet_b200.DnetHead(dnet=False))
    model = magnet_b200.MAGNET(d_net, nn.Conv2d(3, 64, 3, padding=1), n_samples=5).to(cuda).eval()
    g, cam, valid, _ = _batch(cuda, 1, 4, 5, 30, 40)
    imgs = torch.randn(5, 3, 30, 40, device=cuda)
    with torch.no_grad():
        n, why = _breaks(lambda a, b: model(a, b, g.nghbr_poses, valid, cam, mode='test'), imgs[:1], imgs[1:])
    assert n == 0, why


def _equal(a, b):
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(_equal(x, y) for x, y in zip(a, b))
    return torch.equal(a, b)


HEAD_SHAPES = [dict(B=1, V=4, D=5, H=120, W=160), dict(B=1, V=4, D=5, H=88, W=304), CFG2]


@pytest.mark.parametrize("fused_upsample", [False, True])
@pytest.mark.parametrize("shape", HEAD_SHAPES, ids=["b1-120x160", "b1-88x304", "cfg2"])
def test_fullgraph_head_equals_eager(cuda, shape, fused_upsample):
    head = _head(cuda, shape["D"], fused_upsample)
    args = _head_args(cuda, **shape)
    with torch.no_grad():
        want = head(*args)
        got = torch.compile(head, fullgraph=True)(*args)
    assert _equal(got, want)


def test_fullgraph_dnet_fnet_metrics_equal_eager(cuda):
    x = torch.randn(1, 256, 120, 160, device=cuda)
    with torch.no_grad():
        for dnet in (True, False):
            head = magnet_b200.DnetHead(dnet=dnet).to(cuda).eval()
            assert _equal(torch.compile(head, fullgraph=True)(x), head(x)), dnet
    model = magnet_b200.MagnetF(nn.Identity())
    fargs = _fnet_args(cuda, 1, 120, 160)
    assert torch.equal(torch.compile(model.predict, fullgraph=True)(*fargs), model.predict(*fargs))
    quarter, gt, up = _metrics_args(cuda, 1, 120, 160)
    full = [_positive(1, 2, 480, 640, dev=cuda, seed=i) for i in range(2)]
    for preds, kw in ((quarter, dict(up_mask=up, k=4)), (full, {}), ([p[:, :1] for p in quarter], dict(nearest=True)),
                      (full, dict(variance=True))):
        e, c = magnet_b200.DepthMetrics(1e-3, 10.0), magnet_b200.DepthMetrics(1e-3, 10.0)
        e.update(preds, gt, **kw)
        c.update(preds, gt, **kw)                      # both accumulators exist: the compiled update is one graph
        step = torch.compile(c.update, fullgraph=True)
        assert torch.equal(step(preds, gt, **kw), e.update(preds, gt, **kw)), kw
        assert torch.equal(c._acc, e._acc), kw


def test_reduce_overhead_replays_equal_eager(cuda):
    """The head and the metrics update of one evaluation step under CUDA-graph trees: inputs copied into static
    buffers, several replays, each output and the final totals equal to the eager steps."""
    from torch._dynamo.utils import counters
    shape = dict(B=1, V=4, D=5, H=120, W=160)
    head = _head(cuda, 5, True)
    e_metrics, c_metrics = magnet_b200.DepthMetrics(1e-3, 10.0), magnet_b200.DepthMetrics(1e-3, 10.0)

    def step(metrics, ref_feat, nghbr_feat, ref_gmms, nghbr_gmms, x_d3, poses, valid, intM, rays, gt):
        preds = head(ref_feat, nghbr_feat, ref_gmms, nghbr_gmms, x_d3, poses, valid,
                     {"intM": intM, "unit_ray_array_2D": rays})
        return preds, metrics.update(preds, gt)

    def flat(seed):
        a = _head_args(cuda, **shape, seed=seed)
        return [*a[:7], a[7]["intM"], a[7]["unit_ray_array_2D"], _positive(1, 1, 480, 640, dev=cuda, seed=seed)]

    static = flat(10)
    compiled = torch.compile(step, mode="reduce-overhead")
    counters.clear()
    with torch.no_grad():
        for i in range(5):
            new = flat(20 + i)
            for s, n in zip(static, new):
                s.copy_(n)
            got = compiled(c_metrics, *static)
            want = step(e_metrics, *new)
            assert _equal(got, want), i
    assert torch.equal(c_metrics._acc, e_metrics._acc)
    assert c_metrics.value(all_predictions=True) == e_metrics.value(all_predictions=True)
    assert not counters["inductor"]["cudagraph_skips"], dict(counters["inductor"])
