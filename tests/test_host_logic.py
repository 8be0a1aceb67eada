"""CPU-side tests: C-ABI exports and argument validation (no compute calls), sampler offsets, prep cache,
shard arithmetic."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from magnet_b200 import _lib
from magnet_b200._lib import CostArgs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_loads_and_exports_every_declared_symbol():
    L = _lib.lib()
    header = open(os.path.join(ROOT, "include", "magnet_b200.h")).read()
    declared = set(re.findall(r"\b(magnet_[a-z0-9_]+)\s*\(", header))
    declared -= {"magnet_status", "magnet_camera", "magnet_cost_args", "magnet_cost_f_bwd_args"}
    assert declared == set(_lib.EXPORTS), declared ^ set(_lib.EXPORTS)
    for name in declared:
        assert hasattr(L, name), name
    assert L.magnet_abi_version() == _lib.MAGNET_ABI_VERSION
    assert L.magnet_strerror(0) == b"ok"
    assert C.sizeof(CostArgs) == 12 * 4 + 9 * 8


def test_struct_mirrors_match_the_header():
    """Every ctypes mirror names its header struct's fields in the header's order, each an int32, a float or a
    pointer as the header declares it: a field out of order would pass its size check and corrupt memory silently."""
    mirrors = {"magnet_cost_args": _lib.CostArgs, "magnet_cost_f_bwd_args": _lib.CostFBwdArgs,
               "magnet_cost_bwd_args": _lib.CostBwdArgs, "magnet_cost_geom_bwd_args": _lib.CostGeomBwdArgs,
               "magnet_gnet_args": _lib.GnetArgs, "magnet_gnet_train_args": _lib.GnetTrainArgs,
               "magnet_mask_upsample_args": _lib.MaskUpsampleArgs, "magnet_mask_train_args": _lib.MaskTrainArgs,
               "magnet_depth_metrics_args": _lib.DepthMetricsArgs,
               "magnet_depth_metrics_nearest_args": _lib.DepthMetricsNearestArgs}
    header = open(os.path.join(ROOT, "include", "magnet_b200.h")).read()
    header = re.sub(r"/\*.*?\*/", "", header, flags=re.S)
    structs = dict(re.findall(r"typedef struct (magnet_\w+_args) \{(.*?)\}", header, flags=re.S))
    assert set(structs) == set(mirrors), set(structs) ^ set(mirrors)

    def kind(ctype):
        if ctype is C.c_int32:
            return "int32"
        if ctype is C.c_float:
            return "float"
        assert ctype is C.c_void_p or issubclass(ctype, C._Pointer), ctype
        return "pointer"

    for name, body in structs.items():
        declared = []
        for decl in filter(None, (d.strip() for d in body.split(";"))):
            m = re.fullmatch(r"(.*?[\s*])(\w+(?:\s*,\s*\w+)*)", decl, flags=re.S)
            assert m, (name, decl)
            ctype = m.group(1)
            k = "pointer" if "*" in ctype else {"int32_t": "int32", "float": "float"}[ctype.split()[-1]]
            declared += [(f.strip(), k) for f in m.group(2).split(",")]
        mirrored = [(f, kind(t)) for f, t in mirrors[name]._fields_]
        assert mirrored == declared, name


def test_cost_args_validation_without_gpu():
    L = _lib.lib()
    assert L.magnet_cost_volume_f32(None, None) == _lib.ERR_NULL
    a = CostArgs()
    assert L.magnet_cost_volume_f32(C.byref(a), None) == _lib.ERR_SHAPE
    a.B, a.V, a.D, a.C, a.H, a.W = 1, 2, 4, 16, 8, 8
    assert L.magnet_cost_volume_f32(C.byref(a), None) == _lib.ERR_NULL          # pointers missing
    buf = (C.c_float * 64)()
    p = C.cast(buf, C.c_void_p)
    a.ref_feat = a.src_feat = a.rays = a.cams = a.out = p
    a.depth_mode = _lib.DEPTH_VOLUME
    assert L.magnet_cost_volume_f32(C.byref(a), None) == _lib.ERR_NULL          # d_volume missing
    a.depth_mode = 7
    assert L.magnet_cost_volume_f32(C.byref(a), None) == _lib.ERR_UNSUPPORTED
    a.depth_mode = _lib.DEPTH_PLANES
    a.k_host = p
    a.D = _lib.MAGNET_MAX_PLANES + 1
    assert L.magnet_cost_volume_f32(C.byref(a), None) == _lib.ERR_UNSUPPORTED
    a.D = 4
    a.consistency = 1                                                           # needs src_gmm
    assert L.magnet_cost_volume_f32(C.byref(a), None) == _lib.ERR_NULL
    a.consistency = 0
    a.src_layout = _lib.SRC_TILED32
    a.C = 18
    assert L.magnet_cost_volume_f32(C.byref(a), None) == _lib.ERR_UNSUPPORTED   # C % 4
    a.C = 16
    a.src_feat = C.c_void_p(C.addressof(buf) + 4)
    assert L.magnet_cost_volume_f32(C.byref(a), None) == _lib.ERR_ALIGN
    a.src_feat = p
    a.variant = _lib.VARIANT_CELLS
    a.C = 20
    assert L.magnet_cost_volume_f32(C.byref(a), None) == _lib.ERR_UNSUPPORTED   # cells kernel: C in {16,32,64}
    assert L.magnet_repack_tiled32_f32(p, p, 1, 6, 2, 2, None) == _lib.ERR_UNSUPPORTED
    assert L.magnet_gaussian_update_fwd_f32(None, p, 1, 4, p, None) == _lib.ERR_NULL
    with pytest.raises(_lib.MagnetError):
        _lib.check(_lib.ERR_SHAPE, "x")


def test_launch_info_matches_design():
    from magnet_b200 import ops
    grid, block, smem = ops.cost_launch_info(8, 4, 64, 64, 120, 160, variant=_lib.VARIANT_TMA)   # TMA-staged kernel
    assert (grid, block) == (8 * 10 * 30, 256)                          # 16 x 4 pixel tiles x 4 lanes, one chunk of 64
    assert smem == (228 * 1024 - 2 * 1024) // 2                         # two CTAs per SM
    assert ops.cost_launch_info(8, 4, 256, 64, 120, 160, variant=_lib.VARIANT_TMA)[0] == 8 * 10 * 30 * 4
    grid, block, smem = ops.cost_launch_info(8, 4, 64, 64, 120, 160)     # AUTO (TILED32) -> global-gather kernel
    assert (grid, block) == (8 * 10 * 15 * 2, 128)                      # 16 x 8 pixel tiles x 2 chunks of 32 planes
    assert smem == 5 * 3 * 128 * 16 + 5 * 128 * 8 + 32 * 128 * 4 + 32 * 4    # 5 records + headers + chunk + k
    grid, block, smem = ops.cost_launch_info(8, 4, 64, 64, 120, 160, variant=_lib.VARIANT_DIRECT)
    assert (grid, block, smem) == (150 * 64 * 8, 128, 0)


def test_split16_entry_points_without_gpu():
    """MAGNET_SRC_SPLIT16 (tensor-core kernel): buffer size formula, argument validation, launch geometry — no compute calls."""
    from magnet_b200 import ops
    L = _lib.lib()
    # header + fp16 hi/lo planes (N,2,H,W,64) + paired (mu, sigma) table (N,H,W+1,4)
    assert L.magnet_split16_bytes(2, 3, 5) == 256 + 2 * 3 * 5 * 256 + 2 * 3 * 6 * 16
    assert L.magnet_split16_bytes(0, 3, 5) == 0
    buf = (C.c_float * 64)()
    p = C.cast(buf, C.c_void_p)
    assert L.magnet_repack_split16_f32(None, None, p, 1, 64, 2, 2, None) == _lib.ERR_NULL
    assert L.magnet_repack_split16_f32(p, None, p, 1, 32, 2, 2, None) == _lib.ERR_UNSUPPORTED      # C == 64 only
    assert L.magnet_repack_split16_f32(p, None, C.c_void_p(C.addressof(buf) + 4), 1, 64, 2, 2, None) == _lib.ERR_ALIGN
    a = CostArgs()
    a.B, a.V, a.D, a.C, a.H, a.W = 1, 2, 64, 32, 8, 8
    a.ref_feat = a.src_feat = a.rays = a.cams = a.out = a.k_host = p
    a.depth_mode, a.src_layout = _lib.DEPTH_PLANES, _lib.SRC_SPLIT16
    assert L.magnet_cost_volume_f32(C.byref(a), None) == _lib.ERR_UNSUPPORTED                     # C == 64 only
    a.C, a.variant = 64, _lib.VARIANT_CELLS
    assert L.magnet_cost_volume_f32(C.byref(a), None) == _lib.ERR_UNSUPPORTED                     # SPLIT16 is read by the MMA kernel only
    a.variant, a.src_layout = _lib.VARIANT_MMA, _lib.SRC_TILED32
    assert L.magnet_cost_volume_f32(C.byref(a), None) == _lib.ERR_UNSUPPORTED                     # and the MMA kernel reads nothing else
    grid, block, smem = ops.cost_launch_info(8, 4, 64, 64, 120, 160, variant=_lib.VARIANT_MMA)
    assert block == 256 and grid <= 8 * 15 * 20 and grid % 2 == 0      # persistent: two CTAs per SM (or one per work item)
    assert 2 * (smem + 1024) <= 227 * 1024                              # two CTAs per SM fit
    with pytest.raises(_lib.MagnetError):
        ops.repack_split16(torch.zeros(1, 64, 2, 2))                    # CPU tensor


def test_ops_refuse_cpu_tensors():
    from magnet_b200 import ops
    x = torch.zeros(1, 2, 4, 4)
    with pytest.raises(_lib.MagnetError):
        ops.gaussian_update(x, x)
    with pytest.raises(_lib.MagnetError):
        ops.repack_tiled32(torch.zeros(1, 4, 2, 2))


def test_k_offsets():
    from magnet_b200.sampling import depth_sampling, k_offsets_f32
    k64 = depth_sampling(3, 64)
    assert len(k64) == 64 and abs(k64[0] + 2.560835) < 1e-5 and abs(k64[-1] - 2.560835) < 1e-5
    assert np.allclose(k64, -np.asarray(k64)[::-1], atol=1e-12)
    gaps = np.diff(k64)
    assert 0.03 < gaps.min() < 0.05 and 0.5 < gaps.max() < 0.6       # SURVEY §8 a1
    assert k_offsets_f32(3, 5).dtype == np.float32


def test_prep_cache_identity_and_version():
    from magnet_b200.homography import _PrepCache
    c = _PrepCache(capacity=2)
    a = torch.zeros(3)
    assert c.get("x", (a,)) is None
    c.put("x", (a,), "va")
    assert c.get("x", (a,)) == "va"
    a.add_(1)                                  # in-place modification bumps _version -> miss
    assert c.get("x", (a,)) is None
    b = torch.zeros(3)
    c.put("x", (b,), "vb")
    del b                                      # dead tensor can never hit, even if id() is reused
    d = torch.zeros(3)
    assert c.get("x", (d,)) is None


def test_shard_range_partitions_exactly():
    from magnet_b200.dist import shard_range
    for total in (1, 7, 8, 32, 33):
        for world in (1, 2, 3, 8):
            spans = [shard_range(total, r, world) for r in range(world)]
            assert spans[0][0] == 0 and spans[-1][1] == total
            assert all(spans[i][1] == spans[i + 1][0] for i in range(world - 1))
            sizes = [hi - lo for lo, hi in spans]
            assert max(sizes) - min(sizes) <= 1


def test_synthetic_conventions():
    from magnet_b200.synthetic import make_inputs, quarter_res_camera
    K, rays = quarter_res_camera(120, 160)
    assert np.allclose(K[0, 0], 144.4) and rays.shape == (3, 19200)
    # ray of pixel (y=0, x=0) is the back-projected pixel CENTRE (dataloader_scannet.py:119-120,141-144)
    assert np.allclose(rays[:, 0], [(0.5 - 80.0) / 144.4, (0.5 - 60.0) / 145.0, 1.0], atol=1e-6)
    inp = make_inputs(B=2, V=3, D=5, H=8, W=8, C=4, seed=0, invalid=[(1, 0)])
    assert inp.nghbr_feat.shape[0] == 6 and inp.is_valid.dtype == torch.int32 and not inp.is_valid.is_cuda
    assert int(inp.is_valid[1, 0]) == 0 and inp.R.shape == (2, 3, 3, 3) and not inp.R.is_contiguous()
    assert inp.depth_volume().shape == (2, 5, 8, 8)


def test_product_never_imports_the_oracle():
    """oracle/ is test infrastructure: nothing under magnet_b200/ (or the C sources) may import, call or link it."""
    pkg = os.path.join(ROOT, "magnet_b200")
    offenders = []
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                text = open(os.path.join(dirpath, f), errors="ignore").read()
                if re.search(r"^\s*(from|import)\s+oracle\b", text, re.M) or "oracle/" in text or "torch_ref" in text:
                    offenders.append(os.path.join(dirpath, f))
    assert not offenders, offenders
    # and the only top-level users are the allowed ones
    allowed = {"bench.py", "__graft_entry__.py"}
    for f in os.listdir(ROOT):
        if f.endswith(".py") and f not in allowed:
            assert not re.search(r"^\s*(from|import)\s+oracle\b", open(os.path.join(ROOT, f)).read(), re.M), f


def test_drop_in_repack_cache_hits_on_the_callers_tensor(monkeypatch):
    """ADVICE r1 (medium): the repack must be keyed on the tensor object the caller passes — a `.detach()` temporary dies
    before the next call and made every est_costvolume_CW call repack (157 MB at config 2).  Counted with mocked ops."""
    from magnet_b200 import homography as hg, ops
    calls = {"pixc": 0, "tiled": 0, "split": 0}

    def fake_pixc(x, gmm=None, out=None):
        calls["pixc"] += 1
        return torch.zeros(1)

    def fake_tiled(x, out=None):
        calls["tiled"] += 1
        return torch.zeros(1)

    def fake_split(x, gmm=None, out=None):
        calls["split"] += 1
        return torch.zeros(1, dtype=torch.uint8)

    monkeypatch.setattr(ops, "repack_pixc", fake_pixc)
    monkeypatch.setattr(ops, "repack_tiled32", fake_tiled)
    monkeypatch.setattr(ops, "repack_split16", fake_split)
    hg.clear_cache()

    def packed(feat, gmm, variant, ref, D=5):
        layout, _ = hg.route(feat.shape[1], 2, D, variant, _lib.DEPTH_VOLUME, ref.dtype, feat.dtype)
        return (layout,) + hg._packed_source(layout, feat, gmm, ref)

    feat, gmm, ref = torch.zeros(4, 16, 3, 5), torch.zeros(4, 2, 3, 5), torch.zeros(2, 16, 3, 5)
    for _ in range(3):                                       # the N_iter calls of one forward
        assert packed(feat, gmm, _lib.VARIANT_AUTO, ref)[0] == _lib.SRC_PIXC
    assert calls["pixc"] == 1
    feat.add_(1.0)                                           # next forward writes new features in place
    packed(feat, gmm, _lib.VARIANT_AUTO, ref)
    assert calls["pixc"] == 2
    for _ in range(2):                                       # cross-check variants read TILED32, cached separately
        assert packed(feat, gmm, _lib.VARIANT_CELLS, ref)[0] == _lib.SRC_TILED32
    assert calls["tiled"] == 1
    # C == 64: the tensor-core kernel's fp16 hi/lo planes, source views and reference features split once per forward
    feat64, ref64 = torch.zeros(4, 64, 3, 5), torch.zeros(2, 64, 3, 5)
    for _ in range(3):
        layout, _, ref_split = packed(feat64, gmm, _lib.VARIANT_AUTO, ref64, 64)
        assert layout == _lib.SRC_SPLIT16 and ref_split is not None
    assert calls["split"] == 2
    assert packed(feat64, gmm, _lib.VARIANT_AUTO, ref64, 5)[0] == _lib.SRC_PIXC   # N_s = 5: CUDA-core kernel
    ref64.add_(1.0)
    packed(feat64, gmm, _lib.VARIANT_AUTO, ref64, 64)
    assert calls["split"] == 3                               # only the reference features changed
    hg.prep_cache(False)
    packed(feat, gmm, _lib.VARIANT_AUTO, ref)
    packed(feat, gmm, _lib.VARIANT_AUTO, ref)
    assert calls["pixc"] == 5                                # disabled: every call repacks
    hg.prep_cache(True)
    layout = packed(torch.zeros(4, 20, 3, 5), None, _lib.VARIANT_AUTO, torch.zeros(2, 20, 3, 5))[0]
    assert layout == _lib.SRC_TILED32                        # C = 20: not a PIXC channel count
    hg.clear_cache()


def test_camera_table_cache_tracks_both_pose_views(monkeypatch):
    """ADVICE r1 (low): t must be part of the key with its own base tensor and version, like R."""
    from magnet_b200 import homography as hg, ops
    n = {"c": 0}

    def fake_pack(intM, R, t, valid):
        n["c"] += 1
        return torch.zeros(1)

    monkeypatch.setattr(ops, "pack_cameras", fake_pack)
    hg.clear_cache()
    poses = torch.eye(4).repeat(2, 3, 1, 1)
    cam = {"intM": torch.eye(3).repeat(2, 1, 1), "unit_ray_array_2D": torch.zeros(2, 3, 12)}
    valid = torch.ones(2, 3, dtype=torch.int32)
    dev = torch.device("cpu")
    for _ in range(3):
        hg._camera_table(cam, poses[:, :, :3, :3], poses[:, :, :3, 3], valid, dev)
    assert n["c"] == 1
    t_sep = poses[:, :, :3, 3].clone()                       # t allocated separately from R
    hg._camera_table(cam, poses[:, :, :3, :3], t_sep, valid, dev)
    assert n["c"] == 2
    t_sep.add_(0.5)                                          # modified in place: must miss
    hg._camera_table(cam, poses[:, :, :3, :3], t_sep, valid, dev)
    assert n["c"] == 3
    hg.clear_cache()
