"""F-Net evaluation without a GPU: the seeded inputs and the float64 restatement (tests/fnet_metrics_ref.py) against
the reference's own train_FNet validate() output (tests/golden/fnet_metrics.npz), ATen's nearest index rule, and the
argument checks of magnet_plane_depth_f32 / magnet_depth_metrics_nearest_f32 and their Python wrappers."""
import ctypes as C
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from magnet_b200 import _lib, ops
from magnet_b200.metrics import DepthMetrics
from tests.depth_metrics_ref import KEYS, inputs_digest
from tests.fnet_metrics_ref import CASES, NLL, assert_rows_match, case_inputs, metric_rows_nearest, \
    nearest_index, nearest_upsample, soft_argmin64, soft_argmin_bound, threshold_allowance

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "fnet_metrics.npz")


def golden():
    return np.load(GOLDEN, allow_pickle=False)


def restated_rows(name, pred_q):
    """Rows of the nearest form for a (n,1,h,w) prediction, and the a1-a3 allowance around the float64 soft-argmin."""
    kw, inp = CASES[name], case_inputs(name)
    p64 = soft_argmin64(inp["scores"], inp["planes"], scores=True)
    bound = soft_argmin_bound(inp["planes"])
    rows = metric_rows_nearest(pred_q, inp["gt"], kw["min_depth"], kw["max_depth"], kw["crop"])
    return rows, threshold_allowance(p64, inp["gt"], kw["min_depth"], kw["max_depth"], kw["crop"], bound)


def test_golden_carries_every_case_and_digest():
    z = golden()
    assert tuple(z["keys"]) == KEYS
    for name in CASES:
        assert str(z[f"{name}_digest"]) == inputs_digest(case_inputs(name)), f"{name}: seeded inputs drifted"


@pytest.mark.parametrize("name", list(CASES))
def test_restatement_matches_reference_validate(name):
    """The float64 soft-argmin, rounded to float32, through the nearest-form rows reproduces the reference's rows."""
    z = golden()
    inp = case_inputs(name)
    pred = soft_argmin64(inp["scores"], inp["planes"], scores=True).astype(np.float32)
    rows, allowance = restated_rows(name, pred)
    assert_rows_match(rows, z[f"{name}_n"], z[f"{name}_rows"], allowance)
    with np.errstate(all="ignore"):
        np.testing.assert_allclose(rows[:, 1:].mean(axis=0), z[f"{name}_avg"], rtol=1e-4, atol=1e-6, equal_nan=True)


def test_golden_covers_the_edge_cases():
    z = golden()
    assert z["empty_n"][1] == 0 and np.isnan(z["empty_rows"][1, :NLL]).all() and z["empty_rows"][1, NLL] == 0.0
    assert np.isnan(z["empty_avg"][:NLL]).all() and z["empty_avg"][NLL] == 0.0
    for name in CASES:
        assert (z[f"{name}_rows"][:, NLL] == 0.0).all()
        inp = case_inputs(name)
        pred = soft_argmin64(inp["scores"], inp["planes"], scores=True)
        assert np.isnan(pred).sum() >= 3 * CASES[name]["n"]           # -inf row, +inf plane, NaN plane per image
        assert (pred == inp["planes"][len(inp["planes"]) // 2]).any()  # the dominant plane
    ratio = CASES["ratio"]
    assert ratio["H"] % ratio["h"] and ratio["W"] % ratio["w"]          # a non-integer upsampling ratio


@pytest.mark.parametrize("h,H", [(12, 48), (15, 50), (22, 88), (20, 70), (7, 7), (9, 18), (5, 13), (120, 480),
                                 (88, 352), (304, 1216), (1, 5), (37, 64), (76, 304)])
def test_nearest_index_is_atens_interpolate(h, H):
    x = torch.arange(h, dtype=torch.float32).view(1, 1, h, 1)
    want = F.interpolate(x, size=[H, 1], mode="nearest").reshape(-1).numpy().astype(np.int64)
    np.testing.assert_array_equal(nearest_index(H, h), want)
    pred = np.random.default_rng(h * 1000 + H).random((1, 1, h, h + 1)).astype(np.float32)
    got = nearest_upsample(pred, H, H + 3)
    np.testing.assert_array_equal(got, F.interpolate(torch.from_numpy(pred), size=[H, H + 3], mode="nearest").numpy())


def _args(**kw):
    a = _lib.DepthMetricsNearestArgs(P=1, B=2, H=8, W=12, h=2, w=3, row0=0, row1=8, col0=0, col1=12, min_depth=1e-3,
                                     max_depth=10.0)
    for key, v in kw.items():
        setattr(a, key, v)
    return a


def test_nearest_metrics_abi_validation_without_gpu():
    L = _lib.lib()
    n0 = _lib.launch_count()
    buf = (C.c_double * 64)()
    p = C.cast(buf, C.c_void_p).value
    ptrs = (C.c_void_p * 9)(*([p] * 9))
    full = dict(pred=C.cast(ptrs, C.POINTER(C.c_void_p)), gt=p, workspace=p, out=p)

    def ws(**kw):
        return L.magnet_depth_metrics_nearest_workspace(C.byref(_args(**kw)))

    def run(**kw):
        return L.magnet_depth_metrics_nearest_f32(C.byref(_args(**{**full, **kw})), None)

    assert L.magnet_depth_metrics_nearest_workspace(None) == _lib.ERR_NULL
    assert L.magnet_depth_metrics_nearest_f32(None, None) == _lib.ERR_NULL
    # sizing as the other forms: 13 doubles per CTA row (128 columns x 4 GT rows) per (prediction, image)
    assert ws() == 1 * 2 * 1 * 2 * 13
    assert ws(P=3, H=9, W=300, h=3, w=75, row1=9, col1=300) == 3 * 2 * 3 * 3 * 13
    assert ws(h=8, w=12) == ws()                                             # h == H, w == W is allowed
    assert ws(row0=4, row1=4) == 2 * 1 * 13
    for bad in (dict(P=0), dict(B=0), dict(H=0), dict(W=-1), dict(h=0), dict(w=-3), dict(h=9), dict(w=13),
                dict(P=2, B=40000), dict(row0=-1), dict(row1=9), dict(row0=5, row1=4), dict(col0=-2), dict(col1=13),
                dict(col0=7, col1=6)):
        assert ws(**bad) == _lib.ERR_SHAPE, bad
        assert run(**bad) == _lib.ERR_SHAPE, bad
    assert ws(P=_lib.MAGNET_METRICS_MAX_PRED + 1) == _lib.ERR_UNSUPPORTED
    assert run(P=_lib.MAGNET_METRICS_MAX_PRED + 1) == _lib.ERR_UNSUPPORTED
    for missing in ("pred", "gt", "workspace", "out"):
        assert run(**{missing: None}) == _lib.ERR_NULL, missing
    holes = (C.c_void_p * 2)(p, None)
    assert run(P=2, pred=C.cast(holes, C.POINTER(C.c_void_p))) == _lib.ERR_NULL
    assert _lib.launch_count() == n0                                         # nothing was launched


def test_plane_depth_abi_validation_without_gpu():
    L = _lib.lib()
    n0 = _lib.launch_count()
    buf = (C.c_float * 64)()
    p = C.cast(buf, C.c_void_p).value
    planes = (C.c_float * 300)(*range(300))
    pl = C.cast(planes, C.c_void_p)

    def run(vol=p, pln=pl, B=2, D=8, H=4, W=6, scores=1, out=p):
        return L.magnet_plane_depth_f32(vol, pln, B, D, H, W, scores, out, None)

    for missing in (dict(vol=None), dict(pln=None), dict(out=None)):
        assert run(**missing) == _lib.ERR_NULL, missing
    for bad in (dict(B=0), dict(D=0), dict(D=-1), dict(H=0), dict(W=-2), dict(B=70000), dict(H=1 << 14, W=1 << 13)):
        assert run(**bad) == _lib.ERR_SHAPE, bad
        assert run(scores=0, **bad) == _lib.ERR_SHAPE, bad
    assert run(D=_lib.MAGNET_MAX_PLANES + 1) == _lib.ERR_UNSUPPORTED
    assert run(D=_lib.MAGNET_MAX_PLANES + 1, scores=0) == _lib.ERR_UNSUPPORTED
    assert _lib.launch_count() == n0


def test_python_api_refuses_bad_input_without_gpu():
    gt = torch.ones(1, 1, 8, 8)
    with pytest.raises(_lib.MagnetError):
        ops.depth_metrics(torch.ones(1, 1, 2, 2), gt, min_depth=1e-3, max_depth=10.0, nearest=True)     # CPU tensors
    with pytest.raises(_lib.MagnetError):
        ops.depth_metrics(torch.ones(1, 1, 2, 2), gt, min_depth=1e-3, max_depth=10.0, nearest=True,
                          up_mask=torch.ones(1, 144, 2, 2), k=4)
    with pytest.raises(_lib.MagnetError):
        ops.depth_metrics(torch.ones(1, 1, 2, 2), gt, min_depth=1e-3, max_depth=10.0, nearest=True, k=4)
    with pytest.raises(_lib.MagnetError):
        DepthMetrics(1e-3, 10.0).update(torch.ones(1, 1, 2, 2), gt, up_mask=torch.ones(1, 144, 2, 2), k=4,
                                        nearest=True)
    with pytest.raises(_lib.MagnetError):
        ops.plane_depth(torch.ones(1, 4, 2, 2), [1.0, 2.0, 3.0, 4.0], scores=True)                     # CPU tensor
