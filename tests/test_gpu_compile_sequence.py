"""Sequence evaluation under torch.compile and CUDA-graph trees (DESIGN §3.17, §3.18): the device-side check of the
frame table against a numpy restatement and inside a CUDA graph, ``torch.library.opcheck`` of the indexed volume, no
graph break in the indexed head, compiled outputs equal to eager bit for bit (the head, the volume, a whole FrameCache
loop in CUDA graphs), and the NaN contract for out-of-range entries."""
import numpy as np
import pytest
import torch
import torch.nn as nn

import magnet_b200
from magnet_b200 import FrameCache, _lib, ops
from magnet_b200.synthetic import quarter_res_camera, scannet_sequence, trajectory

pytestmark = pytest.mark.gpu
OPS = torch.ops.magnet_b200


# --- the check kernel --------------------------------------------------------------------------------------------------

def _numpy_check(table: np.ndarray, n_src: int):
    ok = (table >= 0) & (table < n_src)
    return np.where(ok, table, 0).astype(np.int32), (~ok).any(axis=1).astype(np.int32)


def _check_equals_numpy(table: torch.Tensor, n_src: int, dev):
    want_t, want_b = _numpy_check(table.numpy(), n_src)
    got_t, got_b = ops.check_src_index_device(table.to(dev), n_src)
    assert got_t.dtype == got_b.dtype == torch.int32
    assert np.array_equal(got_t.cpu().numpy(), want_t)
    assert np.array_equal(got_b.cpu().numpy() != 0, want_b != 0)


@pytest.mark.parametrize("dtype", [torch.int32, torch.int64])
@pytest.mark.parametrize("B,V", [(1, 4), (8, 2), (5, 3), (3, 300)])
def test_check_kernel_equals_numpy(cuda, dtype, B, V):
    n_src = 7
    g = torch.Generator().manual_seed(B * 1000 + V)
    table = torch.randint(0, n_src, (B, V), generator=g, dtype=torch.int64)
    edges = [-1, n_src, n_src - 1, 0, -(2 ** 31)] + ([2 ** 31, 2 ** 32 + 3, -(2 ** 40)] if dtype == torch.int64 else
                                                        [2 ** 31 - 1])
    for i, e in enumerate(edges):                      # one edge value per row, the last rows left in range
        if i < B - 1:
            table[i, (3 * i) % V] = e
    # rows of views with is_valid == 0 are no different: the table alone decides (the host rule)
    _check_equals_numpy(table.to(dtype), n_src, cuda)
    _check_equals_numpy(torch.zeros(B, V, dtype=dtype), 1, cuda)
    _check_equals_numpy(torch.full((B, V), n_src, dtype=dtype), n_src, cuda)


def test_check_kernel_reads_a_strided_table_and_counts_one_launch(cuda):
    table = torch.tensor([[0, 9, 1, 2], [3, 1, 4, 1]], dtype=torch.int64, device=cuda).t()    # (4, 2), not contiguous
    n0 = _lib.launch_count()
    got_t, got_b = ops.check_src_index_device(table, 5)
    assert _lib.launch_count() - n0 == 1
    want_t, want_b = _numpy_check(table.cpu().numpy(), 5)
    assert np.array_equal(got_t.cpu().numpy(), want_t) and np.array_equal(got_b.cpu().numpy() != 0, want_b != 0)


def test_check_kernel_in_a_cuda_graph(cuda):
    """Captured once, replayed with new table contents written into the captured input between replays."""
    B, V, n_src = 4, 4, 6
    static = torch.zeros(B, V, dtype=torch.int64, device=cuda)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.check_src_index_device(static, n_src)     # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out_t, out_b = ops.check_src_index_device(static, n_src)
    g = torch.Generator().manual_seed(5)
    for i in range(6):
        table = torch.randint(-2, n_src + 2, (B, V), generator=g, dtype=torch.int64)
        if i % 2:
            table[i % B, 0] = 2 ** 31 + i
        static.copy_(table.to(cuda))
        graph.replay()
        want_t, want_b = _numpy_check(table.numpy(), n_src)
        assert np.array_equal(out_t.cpu().numpy(), want_t), i
        assert np.array_equal(out_b.cpu().numpy() != 0, want_b != 0), i


# --- opcheck ------------------------------------------------------------------------------------------------------------

def _frames(dev, S, B, H, W, seed=0):
    g = torch.Generator(device=dev).manual_seed(seed)
    frames = torch.randn(S, 64, H, W, device=dev, generator=g)
    mu = 1.5 + 2.0 * torch.rand(S, 1, H, W, device=dev, generator=g)
    ref = torch.randn(B, 64, H, W, device=dev, generator=g)
    rmu = 1.5 + 2.0 * torch.rand(B, 1, H, W, device=dev, generator=g)
    return frames, torch.cat([mu, 0.1 * mu], 1), ref, torch.cat([rmu, 0.1 * rmu], 1)


def _cameras(dev, B, V, H, W, family="scannet", seed=0):
    g = torch.Generator().manual_seed(seed)
    K, rays = quarter_res_camera(H, W, family)
    ang = 0.03 * (torch.rand(B, V, 3, generator=g) - 0.5)
    zero = torch.zeros_like(ang[..., 0])
    R = torch.linalg.matrix_exp(torch.stack([torch.stack([zero, -ang[..., 2], ang[..., 1]], -1),
                                             torch.stack([ang[..., 2], zero, -ang[..., 0]], -1),
                                             torch.stack([-ang[..., 1], ang[..., 0], zero], -1)], -2))
    t = 0.2 * (torch.rand(B, V, 3, generator=g) - 0.5)
    poses = torch.eye(4).repeat(B, V, 1, 1)
    poses[:, :, :3, :3], poses[:, :, :3, 3] = R, t
    intr = {"intM": torch.from_numpy(K)[None].repeat(B, 1, 1).to(dev),
            "unit_ray_array_2D": torch.from_numpy(rays)[None].repeat(B, 1, 1).contiguous().to(dev)}
    return poses.to(dev), intr


LAYOUTS = {   # name: (source layout, variant, feature dtype)
    "TILED32": (_lib.SRC_TILED32, _lib.VARIANT_AUTO, torch.float32),
    "PIXC": (_lib.SRC_PIXC, _lib.VARIANT_TMA, torch.float32),
    "NCHW": (_lib.SRC_NCHW, _lib.VARIANT_DIRECT, torch.float32),
    "SPLIT16": (_lib.SRC_SPLIT16, _lib.VARIANT_MMA, torch.float32),
    "HALF16_F16": (_lib.SRC_HALF16, _lib.VARIANT_MMA, torch.float16),
    "HALF16_BF16": (_lib.SRC_HALF16, _lib.VARIANT_MMA, torch.bfloat16),
}


def _operands(layout, dtype, frames, gmms, ref):
    """(ref operand, source operand, src_gmm, ref_split) of ``layout`` for per-frame maps."""
    if layout == _lib.SRC_TILED32:
        return ref, ops.repack_tiled32(frames), gmms, None
    if layout == _lib.SRC_PIXC:
        return ref, ops.repack_pixc(frames, gmms), None, None
    if layout == _lib.SRC_NCHW:
        return ref, frames, gmms, None
    if layout == _lib.SRC_SPLIT16:
        return ref, ops.repack_split16(frames, gmms), None, ops.repack_split16(ref)
    return ref.to(dtype), ops.repack_half16(frames.to(dtype), gmms), None, ops.repack_half16(ref.to(dtype))


def _indexed_args(layout_name, mode, consistency, frames, gmms, ref, ref_gmm, rays, cams, V, table, D=5, n_src=None):
    layout, variant, dtype = LAYOUTS[layout_name]
    r, src, sgmm, rsplit = _operands(layout, dtype, frames, gmms, ref)
    k = torch.linspace(-1.0, 1.0, D).tolist()
    planes = torch.linspace(1.0, 4.0, D).tolist()
    d_volume = ops.sample_depths(ref_gmm, k) if mode == "VOLUME" else None
    return (r, src, rays, cams, V, layout, consistency, sgmm, 5.0, d_volume,
            ref_gmm if mode == "GAUSS" else None, planes if mode == "PLANES" else (k if mode == "GAUSS" else None),
            mode == "PLANES", False, variant, rsplit, table, n_src)


@pytest.mark.parametrize("layout_name", list(LAYOUTS))
def test_opcheck_indexed_volume(cuda, layout_name):
    B, V, S, H, W = 2, 4, 6, 30, 40
    frames, gmms, ref, ref_gmm = _frames(cuda, S, B, H, W)
    poses, intr = _cameras(cuda, B, V, H, W)
    valid = torch.ones(B, V, dtype=torch.int32, device=cuda)
    valid[1, 2] = 0
    cams = ops.pack_cameras(intr["intM"], poses[:, :, :3, :3], poses[:, :, :3, 3], valid)
    tables = [torch.tensor([[0, 1, 2, 3], [5, 3, 1, 4]], dtype=torch.int32, device=cuda),
              torch.tensor([[2, 2, 0, 5], [1, 1, 1, 1]], dtype=torch.int64, device=cuda)]
    failed = []
    for mode in ("GAUSS", "VOLUME", "PLANES"):
        for consistency in (True, False):
            for i, table in enumerate(tables):
                args = _indexed_args(layout_name, mode, consistency, frames, gmms, ref, ref_gmm, intr["unit_ray_array_2D"],
                                     cams, V, table, n_src=S if i else None)
                try:
                    torch.library.opcheck(OPS.cost_volume_indexed.default, args)
                except Exception as e:                 # every case is checked; all failures are reported together
                    failed.append(f"{mode} cw={consistency} table {i}: {str(e)[:300]}")
    assert not failed, failed
    torch.library.opcheck(OPS.check_src_index.default, (tables[1], S))


# --- the head under torch.compile ------------------------------------------------------------------------------------

class StandInD(nn.Module):
    """(N,3,H,W) -> ((N,2,H/4,W/4) [mu, sigma > 0], (N,256,H/4,W/4)): plain convolutions, not D-Net."""

    def __init__(self):
        super().__init__()
        self.trunk = nn.Conv2d(3, 256, 4, stride=4)
        self.a = nn.Conv2d(256, 2, 1)

    def forward(self, x):
        f = torch.relu(self.trunk(x))
        g = self.a(f)
        return torch.cat([2.5 + 0.5 * torch.tanh(g[:, :1]), 0.2 + 0.05 * torch.sigmoid(g[:, 1:])], 1), f


def _model(dev, n_samples, fused_upsample=True, seed=0):
    torch.manual_seed(seed)
    return magnet_b200.MAGNET(StandInD(), nn.Conv2d(3, 64, 4, stride=4), n_samples=n_samples, test_iter=3,
                              fused_upsample=fused_upsample).to(dev).eval()


def _source_args(dev, B, V, H, W, family="scannet", seed=0, table=None):
    """forward_sources's arguments for B consecutive references of a ScanNet-like sequence: per-frame maps of the
    distinct neighbour frames, every one of them named by the (B, V) int32 table."""
    refs, nghbrs = scannet_sequence(B, window_radius=20 if V == 4 else 10, n_views=V)
    ids = sorted(set(f for row in nghbrs for f in row))
    pos = {f: i for i, f in enumerate(ids)}
    if table is None:
        table = torch.tensor([[pos[f] for f in row] for row in nghbrs], dtype=torch.int32)
    frames, gmms, ref, ref_gmm = _frames(dev, len(ids), B, H, W, seed)
    x_d3 = torch.randn(B, 256, H, W, device=dev, generator=torch.Generator(device=dev).manual_seed(seed + 1))
    poses, intr = _cameras(dev, B, V, H, W, family, seed)
    valid = torch.ones(B, V, dtype=torch.int32, device=dev)
    return [ref, ref_gmm, x_d3, frames, gmms, table, poses, valid, intr]


def _breaks(fn, *args):
    torch._dynamo.reset()
    e = torch._dynamo.explain(fn)(*args)
    return e.graph_break_count, [r.reason[:200] for r in e.break_reasons]


@pytest.mark.parametrize("n_samples", [5, 64])
@pytest.mark.parametrize("dtype", [torch.int32, torch.int64])
@pytest.mark.parametrize("on_device", [False, True], ids=["cpu-table", "device-table"])
def test_indexed_head_traces_without_graph_breaks(cuda, n_samples, dtype, on_device):
    model = _model(cuda, n_samples)
    args = _source_args(cuda, 2, 4, 30, 40)
    table = args[5].to(dtype)
    args[5] = table.to(cuda) if on_device else table
    with torch.no_grad():
        n, why = _breaks(model.forward_sources, *args)
        assert n == 0, why
        ref, ref_gmm, x_d3, frames, gmms, tbl, poses, valid, intr = args
        n, why = _breaks(lambda *a: model.head(*a, src_index=tbl), ref, frames, ref_gmm, gmms, x_d3, poses, valid, intr)
        assert n == 0, why
        torch._dynamo.reset()                          # the whole head as one graph (ATen, no code generation)
        got = torch.compile(model.forward_sources, fullgraph=True, backend="aot_eager")(*args)
        want = model.forward_sources(*args)
    assert all(torch.equal(a, b) for a, b in zip(got, want))


def test_a_host_table_is_copied_not_read(cuda):
    """The traced head reads no host value of a CPU table: the graph copies it to the device and holds nothing that
    brings a value back to the host."""
    model = _model(cuda, 5)
    args = _source_args(cuda, 2, 4, 30, 40)
    graphs = []

    def backend(gm, example_inputs):
        graphs.append(gm)
        return gm.forward

    torch._dynamo.reset()
    with torch.no_grad():
        torch.compile(model.forward_sources, backend=backend, fullgraph=True)(*args)
    assert len(graphs) == 1
    code = graphs[0].code
    for host_read in (".item()", ".tolist()", ".cpu()", "aminmax", "unique"):
        assert host_read not in code, host_read
    assert "magnet_b200.cost_volume_indexed" in code and "magnet_b200.cost_volume." not in code


HEAD_SHAPES = [(4, 120, 160, "scannet"), (2, 88, 304, "kitti")]   # (V, h, w, family), B = 8


@pytest.mark.parametrize("n_samples", [5, 64])
@pytest.mark.parametrize("V,H,W,family", HEAD_SHAPES, ids=["cfg2-120x160", "cfg3-88x304"])
def test_compiled_forward_sources_equals_eager(cuda, n_samples, V, H, W, family):
    model = _model(cuda, n_samples)
    args = _source_args(cuda, 8, V, H, W, family, seed=3)
    torch._dynamo.reset()
    with torch.no_grad():
        want = model.forward_sources(*args)
        got = torch.compile(model.forward_sources, fullgraph=True)(*args)
    assert len(got) == len(want) == 3
    assert all(torch.equal(a, b) for a, b in zip(got, want))


@pytest.mark.parametrize("layout_name", ["TILED32", "SPLIT16", "HALF16_BF16"])
def test_compiled_indexed_volume_equals_eager_with_unused_frames(cuda, layout_name):
    B, V, S, H, W = 2, 4, 9, 120, 160
    frames, gmms, ref, ref_gmm = _frames(cuda, S, B, H, W, seed=4)
    poses, intr = _cameras(cuda, B, V, H, W)
    valid = torch.ones(B, V, dtype=torch.int32, device=cuda)
    cams = ops.pack_cameras(intr["intM"], poses[:, :, :3, :3], poses[:, :, :3, 3], valid)
    layout, variant, dtype = LAYOUTS[layout_name]
    r, src, sgmm, rsplit = _operands(layout, dtype, frames, gmms, ref)
    k = torch.linspace(-1.0, 1.0, 64).tolist()
    rays = intr["unit_ray_array_2D"]

    def volume(table):
        return ops.cost_volume(r, src, rays, cams, V=V, src_layout=layout, consistency=True, src_gmm=sgmm, kappa=5.0,
                               ref_gmm=ref_gmm, k=k, variant=variant, ref_split=rsplit, src_index=table)

    torch._dynamo.reset()
    compiled = torch.compile(volume, fullgraph=True)
    with torch.no_grad():
        for table in (torch.tensor([[1, 3, 5, 7], [3, 5, 7, 3]]),              # frames 0, 2, 4, 6, 8 unused
                      torch.tensor([[8, 0, 4, 2], [6, 1, 0, 8]], dtype=torch.int32, device=cuda)):
            assert torch.equal(compiled(table), volume(table.to(cuda)))   # eager takes a device table


# --- the evaluation loop in CUDA graphs ------------------------------------------------------------------------------

def _loop_samples(dev, n_refs, h=120, w=160):
    refs, nghbrs = scannet_sequence(n_refs)
    ids = sorted(set(refs) | set(f for row in nghbrs for f in row))
    g = torch.Generator(device=dev).manual_seed(6)
    imgs = {f: torch.rand(3, 4 * h, 4 * w, device=dev, generator=g) for f in ids}
    ext = {f: torch.from_numpy(e).to(dev) for f, e in trajectory(ids, 0).items()}
    K, rays = quarter_res_camera(h, w)
    intr = {"intM": torch.from_numpy(K)[None].to(dev), "unit_ray_array_2D": torch.from_numpy(rays)[None].to(dev)}
    out = []
    for r, row in zip(refs, nghbrs):
        poses, valid = ops.relative_poses(ext[r][None], torch.stack([ext[f] for f in row])[:, None])
        out.append((r, row, imgs[r][None], torch.stack([imgs[f] for f in row]), poses, valid, intr))
    return out, len(ids)


def test_frame_cache_with_a_compiled_head_in_cuda_graphs(cuda):
    """About 20 consecutive samples through a FrameCache whose head is forward_sources compiled with
    mode="reduce-overhead": every output equals the eager cache's, the backbones run as often, nothing skips the
    CUDA graphs."""
    from torch._dynamo.utils import counters
    model = _model(cuda, 5)
    samples, n_frames = _loop_samples(cuda, 20)
    eager = FrameCache(model, capacity=32)
    torch._dynamo.reset()
    compiled = FrameCache(model, capacity=32, head=torch.compile(model.forward_sources, mode="reduce-overhead"))
    counters.clear()
    with torch.no_grad():
        for i, (r, row, ri, ni, p, v, intr) in enumerate(samples):
            want = eager(ri, ni, p, v, intr, [r], [row], mode="test")
            got = [x.clone() for x in compiled(ri, ni, p, v, intr, [r], [row], mode="test")]
            assert len(got) == len(want) == 3
            assert all(torch.equal(a, b) for a, b in zip(got, want)), i
    assert compiled.backbone_images == eager.backbone_images == n_frames
    assert not counters["inductor"]["cudagraph_skips"], dict(counters["inductor"])


# --- out-of-range entries under compile --------------------------------------------------------------------------------

def test_out_of_range_entry_gives_nan_for_its_sample_only(cuda):
    B, V, H, W = 4, 4, 30, 40
    model = _model(cuda, 5)
    args = _source_args(cuda, B, V, H, W, seed=7)
    S = args[3].shape[0]
    good = args[5].clone()
    bad = good.clone()
    bad[2, 1] = S                                      # sample 2 names a frame that does not exist
    with torch.no_grad():
        with pytest.raises(_lib.MagnetError, match=r"src_index entries must lie in \[0, %d\)" % S):
            model.forward_sources(*args[:5], bad, *args[6:])
        sanitised = bad.clone()
        sanitised[2, 1] = 0                            # what the device check hands the kernels; frame 0 stays named
        want = model.forward_sources(*args[:5], sanitised, *args[6:])
        torch._dynamo.reset()
        got = torch.compile(model.forward_sources, fullgraph=True)(*args[:5], bad.to(cuda), *args[6:])
    others = [0, 1, 3]
    for a, b in zip(got, want):
        assert torch.isnan(a[2]).all()
        assert torch.equal(a[others], b[others])

    # the volume alone: NaN for exactly the flagged samples, the others equal to eager on the same buffer
    frames, gmms, ref, ref_gmm = _frames(cuda, S, B, H, W, seed=8)
    poses, intr = _cameras(cuda, B, V, H, W)
    cams = ops.pack_cameras(intr["intM"], poses[:, :, :3, :3], poses[:, :, :3, 3],
                            torch.ones(B, V, dtype=torch.int32, device=cuda))
    src, rsplit = ops.repack_split16(frames, gmms), ops.repack_split16(ref)
    k = torch.linspace(-1.0, 1.0, 64).tolist()

    def volume(table):
        return ops.cost_volume(ref, src, intr["unit_ray_array_2D"], cams, V=V, src_layout=_lib.SRC_SPLIT16,
                               consistency=True, kappa=5.0, ref_gmm=ref_gmm, k=k, variant=_lib.VARIANT_AUTO,
                               ref_split=rsplit, src_index=table)

    wide = good.to(torch.int64)
    wide[0, 3], wide[3, 0] = -1, 2 ** 31
    torch._dynamo.reset()
    with torch.no_grad():
        with pytest.raises(_lib.MagnetError, match="must lie in"):
            volume(wide.to(cuda))
        got = torch.compile(volume, fullgraph=True)(wide.to(cuda))
        fixed = wide.clone()
        fixed[0, 3] = fixed[3, 0] = 0
        want = volume(fixed.to(cuda))
    assert torch.isnan(got[[0, 3]]).all() and not torch.isnan(got[[1, 2]]).any()
    assert torch.equal(got[[1, 2]], want[[1, 2]])


def test_forward_frames_flags_a_bad_reference_index(cuda):
    """ref_index under trace: a sample whose reference is not a frame gets NaN predictions, the other sample the eager
    result.  The stand-in backbones are traced too, so this runs without code generation (aot_eager): the same ATen
    calls as eager, bit for bit."""
    model = _model(cuda, 5)
    B, V, h, w = 2, 4, 30, 40
    imgs = torch.rand(6, 3, 4 * h, 4 * w, device=cuda)
    table = torch.tensor([[1, 2, 3, 4], [2, 3, 4, 5]], dtype=torch.int32)
    poses, intr = _cameras(cuda, B, V, h, w)
    valid = torch.ones(B, V, dtype=torch.int32, device=cuda)
    ok, bad = torch.tensor([0, 1]), torch.tensor([0, 6])
    with torch.no_grad():
        with pytest.raises(_lib.MagnetError, match="ref_index entries must lie in"):
            model.forward_frames(imgs, bad, table, poses, valid, intr)
        want = model.forward_frames(imgs, ok, table, poses, valid, intr)
        torch._dynamo.reset()
        step = torch.compile(model.forward_frames, fullgraph=True, backend="aot_eager")
        got_ok = step(imgs, ok.to(cuda), table, poses, valid, intr)
        got_bad = step(imgs, bad.to(cuda), table, poses, valid, intr)
    assert all(torch.equal(a, b) for a, b in zip(got_ok, want))
    for a, b in zip(got_bad, want):
        assert torch.isnan(a[1]).all() and torch.equal(a[0], b[0])
