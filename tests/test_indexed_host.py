"""Host checks of the indexed cost volume (no GPU): the C entry points' argument checks, and the frame-table checks of
ops and MatchingPlan, which all refuse before any launch."""
import ctypes as C

import pytest
import torch

import magnet_b200
from magnet_b200 import _lib, ops
from magnet_b200._lib import CostArgs


def _args(**over):
    a = CostArgs()
    a.B, a.V, a.D, a.C, a.H, a.W = 2, 4, 8, 64, 16, 24
    a.depth_mode, a.src_layout, a.consistency, a.variant, a.kappa = _lib.DEPTH_VOLUME, _lib.SRC_NCHW, 1, 0, 5.0
    buf = (C.c_float * 64)()
    p = C.cast(buf, C.c_void_p).value
    a.ref_feat = a.src_feat = a.src_gmm = a.rays = a.cams = a.d_volume = a.out = p
    for k, v in over.items():
        setattr(a, k, v)
    a._keep = buf
    return a, p


def test_indexed_entry_points_validate_without_gpu():
    L = _lib.lib()
    assert {"magnet_cost_volume_indexed_f32", "magnet_cost_indexed_launch_info"} <= set(_lib.EXPORTS)
    assert L.magnet_abi_version() == 4
    a, p = _args()
    launches = L.magnet_launch_count()
    g, b, s = C.c_int(), C.c_int(), C.c_int()
    for fn in (lambda *x: L.magnet_cost_volume_indexed_f32(*x, None),
               lambda *x: L.magnet_cost_indexed_launch_info(*x, C.byref(g), C.byref(b), C.byref(s))):
        assert fn(None, p, 4) == _lib.ERR_NULL
        assert fn(C.byref(a), None, 4) == _lib.ERR_NULL                 # no table
        assert fn(C.byref(a), p, 0) == _lib.ERR_SHAPE                   # n_src >= 1
        assert fn(C.byref(a), p, -3) == _lib.ERR_SHAPE
        assert fn(C.byref(a), p + 2, 4) == _lib.ERR_ALIGN               # int32 table
        bad, _ = _args(D=0)
        assert fn(C.byref(bad), p, 4) == _lib.ERR_SHAPE                 # the forward's own checks come first
        bad, _ = _args(src_layout=_lib.SRC_SPLIT16, variant=_lib.VARIANT_CELLS)
        assert fn(C.byref(bad), p, 4) == _lib.ERR_UNSUPPORTED
    assert L.magnet_cost_indexed_launch_info(C.byref(a), p, 4, C.byref(g), C.byref(b), C.byref(s)) == _lib.OK
    want = (C.c_int(), C.c_int(), C.c_int())
    assert L.magnet_cost_launch_info(C.byref(a), *map(C.byref, want)) == _lib.OK
    assert (g.value, b.value, s.value) == tuple(w.value for w in want)   # the same kernels and grid
    assert L.magnet_launch_count() == launches


@pytest.mark.parametrize("table,n_src,match", [
    (torch.zeros(2, 3, dtype=torch.int32), 5, "shape"),
    (torch.zeros(4, 2, dtype=torch.int32), 5, "shape"),
    (torch.zeros(8, dtype=torch.int32), 5, "shape"),
    (torch.zeros(2, 4, dtype=torch.float32), 5, "int32 or int64"),
    (torch.zeros(2, 4, dtype=torch.int16), 5, "int32 or int64"),
    (torch.tensor([[0, 1, 2, 5], [0, 1, 2, 3]], dtype=torch.int32), 5, "must lie in"),
    (torch.tensor([[0, 1, 2, 3], [0, -1, 2, 3]], dtype=torch.int64), 5, "must lie in"),
    (torch.zeros(2, 4, dtype=torch.int32), 0, "at least one source image"),
])
def test_check_src_index_refuses(table, n_src, match):
    with pytest.raises(_lib.MagnetError, match=match):
        ops.check_src_index(table, 2, 4, n_src)


def test_check_src_index_accepts_and_converts():
    t = ops.check_src_index(torch.tensor([[4, 0], [1, 4]], dtype=torch.int64).t(), 2, 2, 5)
    assert t.dtype == torch.int32 and t.is_contiguous() and t.tolist() == [[4, 1], [0, 4]]
    with pytest.raises(TypeError):
        ops.check_src_index([[0, 1]], 1, 2, 2)


def test_source_images_counts_the_operand():
    assert ops.source_images(_lib.SRC_NCHW, torch.empty(7, 64, 4, 6), 64, 4, 6) == 7
    assert ops.source_images(_lib.SRC_PIXC, torch.empty(3, 4, 6, 68), 64, 4, 6) == 3
    assert ops.source_images(_lib.SRC_TILED32, torch.empty(2, 4, 1, 16, 32, 4), 64, 4, 6) == 2
    with pytest.raises(_lib.MagnetError, match="n_src"):
        ops.source_images(_lib.SRC_NCHW, torch.empty(7, 32, 4, 6), 64, 4, 6)
    with pytest.raises(_lib.MagnetError, match="n_src"):
        ops.source_images(_lib.SRC_NCHW, torch.empty(0, 64, 4, 6), 64, 4, 6)


def _plan_inputs(B=2, V=4, S=6, H=8, W=12):
    ref = torch.zeros(B, 64, H, W)
    feat, gmms = torch.zeros(S, 64, H, W), torch.ones(S, 2, H, W)
    poses = torch.eye(4).repeat(B, V, 1, 1)
    intr = {"intM": torch.eye(3).repeat(B, 1, 1), "unit_ray_array_2D": torch.ones(B, 3, H * W)}
    table = torch.tensor([[0, 1, 2, 3], [2, 3, 4, 5]], dtype=torch.int32)
    return dict(ref=ref, feat=feat, gmms=gmms, poses=poses, intr=intr, table=table, valid=torch.ones(B, V, dtype=torch.int32))


def _plan(x, **over):
    x = dict(x, **over)
    return magnet_b200.MatchingPlan(x["ref"], x["feat"], x["gmms"], x["poses"], x["valid"], x["intr"],
                                    src_index=x["table"])


@pytest.mark.parametrize("what", ["ref", "feat", "gmms", "poses", "intM", "rays"])
def test_plan_refuses_a_table_with_gradients(what):
    x = _plan_inputs()
    if what in ("intM", "rays"):
        key = "intM" if what == "intM" else "unit_ray_array_2D"
        x["intr"] = dict(x["intr"], **{key: x["intr"][key].clone().requires_grad_(True)})
    else:
        x[what] = x[what].clone().requires_grad_(True)
    with pytest.raises(_lib.MagnetError, match="requires grad"):
        _plan(x)
    with torch.no_grad():                                      # no gradient can be asked for: the checks go on
        with pytest.raises(Exception) as e:
            _plan(x)
        assert "requires grad" not in str(e.value)


@pytest.mark.parametrize("over,match", [
    (dict(table=torch.tensor([[0, 1, 2, 6], [2, 3, 4, 5]], dtype=torch.int32)), "must lie in"),
    (dict(table=torch.tensor([[0, 1, 2, -1], [2, 3, 4, 5]], dtype=torch.int32)), "must lie in"),
    (dict(table=torch.zeros(3, 4, dtype=torch.int32)), "shape"),
    (dict(table=torch.zeros(2, 3, dtype=torch.int32)), "like src_index"),
    (dict(table=torch.zeros(2, 4, dtype=torch.float64)), "int32 or int64"),
    (dict(gmms=torch.ones(5, 2, 8, 12)), "nghbr_gmms"),            # S of the Gaussians != S of the features
    (dict(feat=torch.zeros(6, 32, 8, 12)), "per-frame maps"),
    (dict(poses=torch.eye(4).repeat(2, 3, 1, 1)), "nghbr_poses"),
])
def test_plan_refuses_bad_tables(over, match):
    L = _lib.lib()
    n = L.magnet_launch_count()
    with pytest.raises(_lib.MagnetError, match=match):
        _plan(_plan_inputs(), **over)
    assert L.magnet_launch_count() == n
