"""Depth evaluation without a GPU: the numpy restatement (tests/depth_metrics_ref.py) against the reference's own
validate() output (tests/golden/depth_metrics.npz), the crop box, the C ABI's argument checks and the cross-rank sum of
DepthMetrics."""
import ctypes as C
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from magnet_b200 import _lib, ops
from magnet_b200.metrics import DepthMetrics
from tests.depth_metrics_ref import CASES, KEYS, LOG_KEYS, case_inputs, convex_upsample, eval_mask, inputs_digest, \
    metric_rows

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "depth_metrics.npz")


def _golden():
    return np.load(GOLDEN, allow_pickle=False)


def full_res_pred(name):
    inp = case_inputs(name)
    if "k" in CASES[name]:
        return convex_upsample(inp["depth"], inp["logits"], CASES[name]["k"]), inp
    return inp["pred"], inp


def assert_rows_match_golden(rows, z, name, rtol=2e-5):
    """rows (n,13) as ops.depth_metrics returns them, against the reference's per-image dicts: counts and a1/a2/a3
    exact, the rest within rtol (the reference's float32 means dominate the difference); NaN where it has NaN."""
    want, n = z[f"{name}_rows"], z[f"{name}_n"]
    np.testing.assert_array_equal(rows[:, 0], n)
    np.testing.assert_array_equal(rows[:, 1:4], want[:, :3])
    np.testing.assert_allclose(rows[:, 4:], want[:, 3:], rtol=rtol, atol=0, equal_nan=True)


def test_golden_carries_every_case_and_digest():
    z = _golden()
    assert tuple(z["keys"]) == KEYS
    for name in CASES:
        assert str(z[f"{name}_digest"]) == inputs_digest(case_inputs(name)), f"{name}: seeded inputs drifted"


@pytest.mark.parametrize("name", list(CASES))
def test_restatement_matches_reference_validate(name):
    z = _golden()
    pred, inp = full_res_pred(name)
    kw = CASES[name]
    rows = metric_rows(pred, inp["gt"], kw["min_depth"], kw["max_depth"], kw["crop"])
    assert_rows_match_golden(rows, z, name)
    # the running average over images (the reference averages in float32, DepthMetrics in float64)
    np.testing.assert_allclose(rows[:, 1:].mean(axis=0), z[f"{name}_avg"], rtol=2e-5, atol=0, equal_nan=True)


def test_golden_covers_the_edge_cases():
    z = _golden()
    assert z["scannet_empty_n"][1] == 0 and np.isnan(z["scannet_empty_avg"]).all()
    assert np.isnan(z["kitti_garg_rows"][2, KEYS.index("nll")]) and np.isfinite(z["kitti_garg_rows"][:2]).all()
    for name in CASES:
        if name != "scannet_empty" and name != "kitti_garg":
            assert np.isfinite(z[f"{name}_avg"]).all(), name


def test_thresholds_compare_in_float32():
    """GT exactly at float32(1e-3) is invalid only if min_depth is compared in float32: the golden's counts say it is."""
    z = _golden()
    inp = case_inputs("scannet")
    gt = inp["gt"][:, 0]
    at_min = (gt == np.float32(1e-3)).sum(axis=(1, 2))
    assert (at_min > 0).all()
    n64 = ((gt.astype(np.float64) > 1e-3) & (gt.astype(np.float64) < 10.0)).sum(axis=(1, 2))
    n32 = ((gt > np.float32(1e-3)) & (gt < np.float32(10.0))).sum(axis=(1, 2))
    np.testing.assert_array_equal(n32, z["scannet_n"])
    assert (n64 != n32).all()


def test_ratio_exactly_1_25_is_not_counted():
    gt = np.full((1, 1, 2, 2), 5.0, dtype=np.float32)
    pred = np.stack([np.array([[4.0, 5.0], [4.0, 4.0]]), np.ones((2, 2))])[None].astype(np.float32)
    rows = metric_rows(pred, gt, 1e-3, 10.0)
    assert rows[0, 0] == 4 and rows[0, 1] == 0.25 and rows[0, 2] == 1.0


@pytest.mark.parametrize("crop", [None, "garg", "eigen"])
def test_crop_box_is_the_reference_eval_mask(crop):
    for H in (1, 2, 7, 37, 88, 352, 375, 480):
        for W in (1, 3, 28, 304, 640, 1216, 1242):
            r0, r1, c0, c1 = ops.crop_box(crop, H, W)
            m = np.zeros((H, W), dtype=bool)
            m[r0:r1, c0:c1] = True
            np.testing.assert_array_equal(m, eval_mask(H, W, crop), err_msg=f"{crop} {H}x{W}")
            assert 0 <= r0 <= r1 <= H and 0 <= c0 <= c1 <= W
    with pytest.raises(_lib.MagnetError):
        ops.crop_box("kitti", 352, 1216)


def _args(**kw):
    a = _lib.DepthMetricsArgs(P=1, B=2, H=8, W=12, k=0, row0=0, row1=8, col0=0, col1=12, min_depth=1e-3,
                              max_depth=10.0)
    for key, v in kw.items():
        setattr(a, key, v)
    return a


def test_depth_metrics_abi_validation_without_gpu():
    L = _lib.lib()
    buf = (C.c_double * 64)()
    p = C.cast(buf, C.c_void_p).value
    ptrs = (C.c_void_p * 9)(*([p] * 9))
    full = dict(pred=C.cast(ptrs, C.POINTER(C.c_void_p)), gt=p, workspace=p, out=p)

    def ws(**kw):
        return L.magnet_depth_metrics_workspace(C.byref(_args(**kw)))

    def run(**kw):
        return L.magnet_depth_metrics_f32(C.byref(_args(**{**full, **kw})), None)

    assert L.magnet_depth_metrics_workspace(None) == _lib.ERR_NULL
    assert L.magnet_depth_metrics_f32(None, None) == _lib.ERR_NULL
    # sizing: 13 doubles per CTA row per (prediction, image); 128 columns x 4 rows per CTA
    assert ws() == 1 * 2 * 1 * 2 * 13
    assert ws(P=3, H=9, W=300, row1=9, col1=300) == 3 * 2 * 3 * 3 * 13
    assert ws(row0=4, row1=4) == 2 * 1 * 13                                  # empty box: one idle CTA per image
    # shapes
    for bad in (dict(P=0), dict(B=0), dict(H=0), dict(W=-1), dict(k=-1), dict(k=3), dict(P=2, B=40000)):
        assert ws(**bad) == _lib.ERR_SHAPE, bad
        assert run(**bad) == _lib.ERR_SHAPE, bad
    assert ws(P=_lib.MAGNET_METRICS_MAX_PRED + 1) == _lib.ERR_UNSUPPORTED
    assert run(P=_lib.MAGNET_METRICS_MAX_PRED + 1) == _lib.ERR_UNSUPPORTED
    # crop box outside the image or inverted
    for bad in (dict(row0=-1), dict(row1=9), dict(row0=5, row1=4), dict(col0=-2), dict(col1=13), dict(col0=7, col1=6)):
        assert ws(**bad) == _lib.ERR_SHAPE, bad
        assert run(**bad) == _lib.ERR_SHAPE, bad
    # NULL pointers
    for missing in ("pred", "gt", "workspace", "out"):
        assert run(**{missing: None}) == _lib.ERR_NULL, missing
    assert run(k=4) == _lib.ERR_NULL                                        # the fused form needs up_mask
    holes = (C.c_void_p * 2)(p, None)
    assert run(P=2, pred=C.cast(holes, C.POINTER(C.c_void_p))) == _lib.ERR_NULL


def test_python_api_refuses_bad_input_without_gpu():
    gt = torch.ones(1, 1, 8, 8)
    with pytest.raises(_lib.MagnetError):
        ops.depth_metrics(torch.ones(1, 2, 8, 8), gt, min_depth=1e-3, max_depth=10.0)     # CPU tensors
    with pytest.raises(_lib.MagnetError):
        ops.depth_metrics([], gt, min_depth=1e-3, max_depth=10.0)
    with pytest.raises(_lib.MagnetError):
        ops.depth_metrics([gt] * 9, gt, min_depth=1e-3, max_depth=10.0)
    with pytest.raises(_lib.MagnetError):
        DepthMetrics(1e-3, 80.0, crop="kitti")
    with pytest.raises(_lib.MagnetError):
        DepthMetrics(1e-3, 80.0).value()


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    from magnet_b200 import dist as md
    md.init_process_group("gloo")
    m = DepthMetrics(1e-3, 10.0)
    # rank r has seen r + 1 images whose rows are all (r + 1): the pooled average is sum((r+1)^2) / sum(r+1)
    m._acc = torch.tensor([[float(rank + 1)] + [float((rank + 1) ** 2)] * 13], dtype=torch.float64)
    m.all_reduce()
    q.put((rank, m.images(), m.value()))
    dist.destroy_process_group()


@pytest.mark.timeout(120)
def test_all_reduce_pools_the_ranks_images():
    world, port = 2, _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted((q.get(timeout=100) for _ in range(world)), key=lambda r: r[0])
    for p in procs:
        p.join(timeout=30)
        assert p.exitcode == 0
    for _, images, value in res:
        assert images == 3
        assert list(value) == list(KEYS)
        assert all(v == pytest.approx(5.0 / 3.0, rel=1e-15) for v in value.values())


def test_log_keys_are_metric_keys():
    assert set(LOG_KEYS) <= set(KEYS) and tuple(ops.METRIC_KEYS) == KEYS
