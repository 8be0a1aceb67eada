"""Cost volumes that read their source views through a frame table (magnet_cost_volume_indexed_f32, DESIGN §3.17):
for every kernel, depth mode and source layout the indexed volume is bit for bit the volume of the view-major gather
``frames[src_index.T.flatten()]``, and MatchingPlan with a table is bit for bit the plan over the gathered maps."""
import pytest
import torch

import magnet_b200
from magnet_b200 import _lib, ops
from magnet_b200.homography import repack_source
from magnet_b200.synthetic import quarter_res_camera, scannet_sequence

pytestmark = pytest.mark.gpu

F32, F16, BF16 = torch.float32, torch.float16, torch.bfloat16
KERNELS = {   # name: (source layout, variant, feature dtype)
    "DIRECT": (_lib.SRC_NCHW, _lib.VARIANT_DIRECT, F32),
    "CELLS": (_lib.SRC_TILED32, _lib.VARIANT_CELLS, F32),
    "CELLS_NOREUSE": (_lib.SRC_TILED32, _lib.VARIANT_CELLS_NOREUSE, F32),
    "TMA": (_lib.SRC_PIXC, _lib.VARIANT_TMA, F32),
    "MMA": (_lib.SRC_SPLIT16, _lib.VARIANT_MMA, F32),
    "MMA_F16": (_lib.SRC_HALF16, _lib.VARIANT_MMA, F16),
    "MMA_BF16": (_lib.SRC_HALF16, _lib.VARIANT_MMA, BF16),
}
MODES = ("GAUSS", "VOLUME", "PLANES", "PLANES_SOFTMAX")


def _sequence_table(B, V):
    """B consecutive references of a ScanNet-like sequence and their neighbours (window 20 for V = 4, 10 for V = 2)
    renumbered over the distinct frames: (S, table (B, V) int64)."""
    refs, nghbrs = scannet_sequence(B, window_radius=20 if V == 4 else 10, n_views=V)
    ids = sorted(set(f for row in nghbrs for f in row))
    pos = {f: i for i, f in enumerate(ids)}
    return len(ids), torch.tensor([[pos[f] for f in row] for row in nghbrs])


def _tables():
    """name -> (B, V, S, table, invalid views, family, H, W)"""
    out = {}
    S, t = _sequence_table(1, 2)
    out["b1v2"] = (1, 2, S, t, (), "scannet", 24, 40)
    S, t = _sequence_table(8, 4)
    out["b8v4_cfg2"] = (8, 4, S, t, (), "scannet", 30, 40)
    S, t = _sequence_table(8, 2)
    out["b8v2_cfg3"] = (8, 2, S, t, (), "kitti", 22, 76)
    S, t = _sequence_table(4, 4)
    out["b4v4_ragged"] = (4, 4, S, t, ((0, 1), (2, 0), (2, 3), (3, 2)), "scannet", 30, 40)
    out["b4v4_one_frame"] = (4, 4, 1, torch.zeros(4, 4, dtype=torch.int64), (), "scannet", 30, 40)
    # frames the table never names (references that are never sources): the indexed operand holds only the used ones
    out["b2v4_unused"] = (2, 4, 9, torch.tensor([[1, 3, 5, 7], [3, 5, 7, 3]]), ((1, 3),), "scannet", 24, 40)
    return out


TABLES = _tables()


def _inputs(name, D, dtype, seed=0, cuda="cuda"):
    B, V, S, table, invalid, family, H, W = TABLES[name]
    g = torch.Generator().manual_seed(seed)
    frames = torch.randn(S, 64, H, W, generator=g)
    mu = 1.5 + 2.0 * torch.rand(S, 1, H, W, generator=g)
    gmms = torch.cat([mu, 0.1 * mu], 1)
    ref = torch.randn(B, 64, H, W, generator=g)
    rmu = 1.5 + 2.0 * torch.rand(B, 1, H, W, generator=g)
    ref_gmm = torch.cat([rmu, 0.1 * rmu], 1)
    K, rays = quarter_res_camera(H, W, family)
    ang = 0.03 * (torch.rand(B, V, 3, generator=g) - 0.5)
    R = torch.linalg.matrix_exp(torch.stack([
        torch.stack([torch.zeros_like(ang[..., 0]), -ang[..., 2], ang[..., 1]], -1),
        torch.stack([ang[..., 2], torch.zeros_like(ang[..., 0]), -ang[..., 0]], -1),
        torch.stack([-ang[..., 1], ang[..., 0], torch.zeros_like(ang[..., 0])], -1)], -2))
    t = 0.2 * (torch.rand(B, V, 3, generator=g) - 0.5)
    valid = torch.ones(B, V, dtype=torch.int32)
    for b, v in invalid:
        valid[b, v] = 0
    intM = torch.from_numpy(K)[None].repeat(B, 1, 1)
    cams = ops.pack_cameras(intM.to(cuda), R.to(cuda), t.to(cuda), valid.to(cuda))
    rays = torch.from_numpy(rays)[None].repeat(B, 1, 1).contiguous().to(cuda)
    return dict(B=B, V=V, frames=frames.to(cuda, dtype), gmms=gmms.to(cuda), ref=ref.to(cuda, dtype),
                ref_gmm=ref_gmm.to(cuda), table=table, rays=rays, cams=cams, valid=valid, R=R, t=t, intM=intM,
                rays_cpu=rays.cpu())


def _depth_kwargs(mode, D, ref_gmm):
    k = [float(x) for x in torch.linspace(-3.0, 3.0, D)]
    if mode == "GAUSS":
        return dict(ref_gmm=ref_gmm, k=k)
    if mode == "VOLUME":
        return dict(d_volume=ops.sample_depths(ref_gmm, k))
    planes = [float(x) for x in torch.linspace(0.8, 5.0, D)]
    return dict(k=planes, planes=True, softmax=mode == "PLANES_SOFTMAX")


def _pair(inp, kernel, mode, cw, D):
    """(gathered volume, indexed volume) of one case."""
    layout, variant, _ = KERNELS[kernel]
    B, V, table = inp["B"], inp["V"], inp["table"]
    frames, gmms, ref = inp["frames"], inp["gmms"], inp["ref"]
    gather = table.t().reshape(-1).to(frames.device)               # view-major: image v*B + b is table[b, v]
    used = torch.unique(table)
    remap = torch.full((int(table.max()) + 1,), -1, dtype=torch.int64)
    remap[used] = torch.arange(used.numel())
    idx = remap[table].to(torch.int32).to(frames.device)
    used = used.to(frames.device)
    vols = []
    for src_feat, src_gmm, kw in ((frames[gather], gmms[gather], {}),
                                  (frames[used], gmms[used], dict(src_index=idx, n_src=int(used.numel())))):
        src, ref_split = repack_source(layout, src_feat, src_gmm, ref if layout in ops.PACKED_LAYOUTS else None)
        ref_op = ref if layout == _lib.SRC_HALF16 else ref.float()
        vols.append(ops.cost_volume(ref_op, src, inp["rays"], inp["cams"], V=V, src_layout=layout, consistency=cw,
                                    src_gmm=src_gmm.contiguous(), kappa=5.0, variant=variant, ref_split=ref_split,
                                    **_depth_kwargs(mode, D, inp["ref_gmm"]), **kw))
    return vols


def _applies(kernel, mode, cw):
    if kernel == "CELLS_NOREUSE" and mode != "GAUSS":
        return False
    return not (cw and mode == "PLANES_SOFTMAX")


@pytest.mark.parametrize("table", list(TABLES))
@pytest.mark.parametrize("kernel", list(KERNELS))
def test_indexed_volume_equals_gathered(cuda, table, kernel):
    inp = _inputs(table, 8, KERNELS[kernel][2])
    n = 0
    for mode in MODES:
        for cw in (True, False):
            if not _applies(kernel, mode, cw):
                continue
            gathered, indexed = _pair(inp, kernel, mode, cw, D=8)
            assert torch.isfinite(gathered).all()
            assert torch.equal(gathered, indexed), (kernel, mode, cw)
            n += 1
    assert n >= 1


@pytest.mark.parametrize("kernel", ["MMA", "MMA_F16", "CELLS", "TMA"])
def test_indexed_volume_full_cfg2(cuda, kernel):
    """cfg2's full shape (B = 8, V = 4, D = 64, 120x160) on a sequence table, GAUSS with consistency."""
    TABLES["cfg2_full"] = (8, 4, *_sequence_table(8, 4), (), "scannet", 120, 160)
    try:
        inp = _inputs("cfg2_full", 64, KERNELS[kernel][2], seed=3)
        gathered, indexed = _pair(inp, kernel, "GAUSS", True, D=64)
    finally:
        del TABLES["cfg2_full"]
    assert torch.equal(gathered, indexed)


@pytest.mark.parametrize("table", ["b8v4_cfg2", "b4v4_ragged", "b2v4_unused"])
@pytest.mark.parametrize("D,dtype", [(5, F32), (64, F32), (64, F16)])
def test_plan_with_a_table_equals_the_gathered_plan(cuda, table, D, dtype):
    """MatchingPlan over per-frame maps and a table (CPU or device) against the plan over the gathered maps, for the
    layout route() picks (TILED32 for D = 5, SPLIT16 / HALF16 for D = 64); frames no view names are gathered out."""
    inp = _inputs(table, D, dtype, seed=5)
    B, V, tab = inp["B"], inp["V"], inp["table"]
    poses = torch.zeros(B, V, 4, 4)
    poses[:, :, :3, :3], poses[:, :, :3, 3], poses[:, :, 3, 3] = inp["R"], inp["t"], 1.0
    intr = {"intM": inp["intM"], "unit_ray_array_2D": inp["rays_cpu"]}
    gather = tab.t().reshape(-1).to(cuda)
    k = [float(x) for x in torch.linspace(-3.0, 3.0, D)]
    g = magnet_b200.MatchingPlan(inp["ref"], inp["frames"][gather], inp["gmms"][gather], poses.to(cuda), inp["valid"],
                                 intr, thres=5)
    want = g.cost(inp["ref_gmm"], k)
    for t in (tab, tab.to(torch.int32).to(cuda)):
        p = magnet_b200.MatchingPlan(inp["ref"], inp["frames"], inp["gmms"], poses.to(cuda), inp["valid"], intr,
                                     thres=5, src_index=t)
        assert p.V == V and p._nghbr_feat.shape[0] == torch.unique(tab).numel()
        assert torch.equal(p.cost(inp["ref_gmm"], k), want)


def test_device_table_out_of_range_is_refused_before_launch(cuda):
    inp = _inputs("b4v4_ragged", 8, F32)
    src, _ = repack_source(_lib.SRC_TILED32, inp["frames"])
    launches = _lib.lib().magnet_launch_count()
    for bad in (inp["table"].clone().fill_(inp["frames"].shape[0]), inp["table"] - 1):
        with pytest.raises(_lib.MagnetError, match="must lie in"):
            ops.cost_volume(inp["ref"], src, inp["rays"], inp["cams"], V=4, src_layout=_lib.SRC_TILED32,
                            consistency=False, ref_gmm=inp["ref_gmm"], k=[0.0] * 8,
                            src_index=bad.to(torch.int32).to(cuda))
    assert _lib.lib().magnet_launch_count() == launches
