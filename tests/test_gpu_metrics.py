"""Depth evaluation on the H100 (ops.depth_metrics, DepthMetrics): against the reference's validate() output
(tests/golden/depth_metrics.npz) in both input forms, against the numpy restatement over fuzz shapes, fused upsampling
bit-identical to convex_upsample + the full-resolution form, run-to-run bit-identity and CUDA-graph capture."""
import numpy as np
import pytest
import torch

import magnet_b200
from magnet_b200 import _lib, ops
from tests.depth_metrics_ref import CASES, KEYS, LOG_KEYS, case_inputs, metric_rows
from tests.test_metrics_cpu import _golden, assert_rows_match_golden

pytestmark = pytest.mark.gpu

FULL = [n for n in CASES if "k" not in CASES[n]]
FUSED = [n for n in CASES if "k" in CASES[n]]


def _t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _score(name, dev):
    kw, inp = CASES[name], case_inputs(name)
    gt = _t(inp["gt"], dev)
    m = magnet_b200.DepthMetrics(kw["min_depth"], kw["max_depth"], crop=kw["crop"])
    if "k" in kw:
        rows = m.update(_t(inp["depth"], dev), gt, up_mask=_t(inp["logits"], dev), k=kw["k"])
    else:
        rows = m.update(_t(inp["pred"], dev), gt)
    return rows, m


@pytest.mark.parametrize("name", FULL + FUSED)
def test_matches_reference_validate(cuda, name):
    """Every image of the batch at once; counts and a1/a2/a3 exact, the rest within 2e-5 of the reference's float32
    means; the running average within 2e-5 of RunningAverageDict's."""
    z = _golden()
    rows, m = _score(name, cuda)
    assert rows.shape == (1, CASES[name]["n"], 13) and rows.dtype == torch.float64
    assert_rows_match_golden(rows[0].cpu().numpy(), z, name)
    got = np.array([m.value()[key] for key in KEYS])
    np.testing.assert_allclose(got, z[f"{name}_avg"], rtol=2e-5, atol=0, equal_nan=True)
    assert m.images() == CASES[name]["n"]


def _fuzz_inputs(B, H, W, P, k, seed, dev):
    rng = np.random.default_rng(seed)
    gt = rng.uniform(0.3, 12.0, (B, 1, H, W)).astype(np.float32)
    gt[rng.random(gt.shape) < 0.15] = 0
    gt[rng.random(gt.shape) < 0.02] = 15.0                                    # above max_depth
    if k:
        h, w = H // k, W // k
        depth = np.empty((P, B, 2, h, w), dtype=np.float32)
        depth[:, :, 0] = rng.uniform(0.5, 12.0, (P, B, h, w))
        depth[:, :, 1] = rng.normal(0.0, 0.5, (P, B, h, w))
        mask = (2.0 * rng.standard_normal((B, 9 * k * k, h, w))).astype(np.float32)
        return _t(gt, dev), [_t(d, dev) for d in depth], _t(mask, dev)
    pred = np.empty((P, B, 2, H, W), dtype=np.float32)
    pred[:, :, 0] = gt[None, :, 0] * np.exp(rng.normal(0.2, 0.3, (P, B, H, W)))
    pred[:, :, 0][pred[:, :, 0] == 0] = 3.0
    pred[:, :, 1] = rng.normal(0.0, 0.4, (P, B, H, W))
    flat = pred.reshape(P, B, 2, -1)
    for val, ch in ((np.nan, 0), (np.inf, 0), (-np.inf, 0), (1e-5, 0), (50.0, 0), (1e-4, 1), (0.0, 1)):
        sel = rng.random(flat.shape[-1]) < 0.01
        flat[:, :, ch, sel] = val
    return _t(gt, dev), [_t(p, dev) for p in pred], None


FUZZ = [  # B, H, W, P, k, crop
    (1, 37, 130, 1, None, None),
    (3, 21, 257, 2, None, "garg"),
    (4, 44, 100, 3, None, "eigen"),
    (1, 5, 9, 1, None, "garg"),
    (2, 36, 260, 3, 2, None),
    (4, 48, 132, 2, 4, "garg"),
    (3, 88, 300, 3, 4, "eigen"),
    (1, 8, 12, 1, 4, None),
]


def assert_rows_match_restatement(got, want):
    """Counts exact; sums of float32 terms to 1e-9 relative, those built on logf / log10f to 1e-6."""
    np.testing.assert_array_equal(got[..., :4], want[..., :4])
    for i, key in enumerate(KEYS[3:], start=4):
        rtol = 1e-6 if key in LOG_KEYS else 1e-9
        np.testing.assert_allclose(got[..., i], want[..., i], rtol=rtol, atol=0, equal_nan=True, err_msg=key)


@pytest.mark.parametrize("B,H,W,P,k,crop", FUZZ)
def test_matches_restatement_over_fuzz_shapes(cuda, B, H, W, P, k, crop):
    gt, preds, mask = _fuzz_inputs(B, H, W, P, k, seed=B * 1000 + H * 10 + W + P, dev=cuda)
    got = ops.depth_metrics(preds, gt, min_depth=1e-3, max_depth=10.0, crop=crop, up_mask=mask, k=k)
    assert got.shape == (P, B, 13)
    full = [ops.convex_upsample(p, mask, k) for p in preds] if k else preds
    want = np.stack([metric_rows(f.cpu().numpy(), gt.cpu().numpy(), 1e-3, 10.0, crop) for f in full])
    assert (want[..., 0] > 0).all() or (H, W) == (5, 9)
    assert_rows_match_restatement(got.cpu().numpy(), want)


@pytest.mark.parametrize("k,crop", [(2, None), (4, "garg"), (4, "eigen")])
def test_fused_form_is_convex_upsample_then_full_form_bit_for_bit(cuda, k, crop):
    gt, preds, mask = _fuzz_inputs(3, 48, 136, 3, k, seed=5 + k, dev=cuda)
    fused = ops.depth_metrics(preds, gt, min_depth=1e-3, max_depth=10.0, crop=crop, up_mask=mask, k=k)
    full = ops.depth_metrics([ops.convex_upsample(p, mask, k) for p in preds], gt, min_depth=1e-3, max_depth=10.0,
                             crop=crop)
    assert torch.isfinite(fused).all()
    assert torch.equal(fused, full)


def test_several_predictions_equal_one_call_each_and_runs_are_bit_identical(cuda):
    gt, preds, _ = _fuzz_inputs(4, 64, 200, 3, None, seed=17, dev=cuda)
    n0 = _lib.launch_count()
    a = ops.depth_metrics(preds, gt, min_depth=1e-3, max_depth=10.0, crop="garg")
    assert _lib.launch_count() - n0 == 2                                      # partial rows + final reduction
    b = ops.depth_metrics(preds, gt, min_depth=1e-3, max_depth=10.0, crop="garg")
    assert torch.equal(a, b)
    for i, p in enumerate(preds):
        assert torch.equal(ops.depth_metrics(p, gt, min_depth=1e-3, max_depth=10.0, crop="garg")[0], a[i])


def test_depth_metrics_captures_in_a_cuda_graph(cuda):
    B, H, W, k = 2, 48, 64, 4
    gt, preds, mask = _fuzz_inputs(B, H, W, 2, k, seed=23, dev=cuda)
    m = magnet_b200.DepthMetrics(1e-3, 10.0, crop="eigen")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        m.update(preds, gt, up_mask=mask, k=k)                               # warm-up creates the accumulator
    torch.cuda.current_stream().wait_stream(s)
    m.reset()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        m.update(preds, gt, up_mask=mask, k=k)
    rows = []
    for seed in (31, 32, 33):
        gt2, preds2, mask2 = _fuzz_inputs(B, H, W, 2, k, seed=seed, dev=cuda)
        gt.copy_(gt2)
        mask.copy_(mask2)
        for p, p2 in zip(preds, preds2):
            p.copy_(p2)
        g.replay()
        rows.append(ops.depth_metrics(preds2, gt2, min_depth=1e-3, max_depth=10.0, crop="eigen", up_mask=mask2, k=k))
    torch.cuda.synchronize()
    rows = torch.cat(rows, dim=1).cpu().numpy()                               # (P, 3B, 13)
    assert m.images() == 3 * B
    for p, value in enumerate(m.value(all_predictions=True)):
        want = rows[p, :, 1:].mean(axis=0)
        np.testing.assert_allclose([value[key] for key in KEYS], want, rtol=1e-13, atol=0)
    assert m.value() == m.value(all_predictions=True)[-1]


def test_errors_leave_no_sticky_cuda_error(cuda):
    gt = torch.rand(1, 1, 16, 24, device=cuda)
    pred = torch.rand(1, 2, 16, 24, device=cuda)
    with pytest.raises(_lib.MagnetError):
        ops.depth_metrics([pred] * 9, gt, min_depth=1e-3, max_depth=10.0)
    with pytest.raises(_lib.MagnetError):
        ops.depth_metrics(pred[:, :, :8], gt, min_depth=1e-3, max_depth=10.0)
    with pytest.raises(_lib.MagnetError):
        ops.depth_metrics(pred, gt, min_depth=1e-3, max_depth=10.0, up_mask=torch.rand(1, 144, 4, 6, device=cuda))
    with pytest.raises(_lib.MagnetError):
        ops.depth_metrics(pred.double(), gt, min_depth=1e-3, max_depth=10.0)
    m = magnet_b200.DepthMetrics(1e-3, 10.0)
    m.update(pred, gt)
    with pytest.raises(_lib.MagnetError):
        m.update([pred, pred], gt)
    out = ops.depth_metrics(pred + 1.0, gt * 5.0 + 1.0, min_depth=1e-3, max_depth=10.0)
    torch.cuda.synchronize()
    assert out[0, 0, 0].item() == 16 * 24
