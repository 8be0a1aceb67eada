"""The variance form of the depth metrics on the H100 (DESIGN §3.15) against the reference's test_DNet.validate
(tests/golden/dnet_metrics.npz): counts and a1..a3 equal, the other metrics within the 2e-5 of DESIGN §3.6; and a
DepthMetrics instance keeps to one form."""
import os

import numpy as np
import pytest
import torch

import magnet_b200
from magnet_b200 import _lib, ops
from tests.depth_metrics_ref import inputs_digest
from tests.dnet_ref import METRIC_CASES, metric_inputs, metric_rows_var

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "dnet_metrics.npz")


@pytest.mark.parametrize("name", list(METRIC_CASES))
def test_variance_form_matches_validate(cuda, name):
    gold = np.load(GOLDEN)
    inp = metric_inputs(name)
    assert str(gold[f"{name}_digest"]) == inputs_digest(inp)
    kw = METRIC_CASES[name]
    pred, gt = torch.from_numpy(inp["pred"]).to(cuda), torch.from_numpy(inp["gt"]).to(cuda)
    rows = ops.depth_metrics(pred, gt, min_depth=kw["min_depth"], max_depth=kw["max_depth"], crop=kw["crop"],
                             variance=True)[0].cpu().numpy()
    want = gold[f"{name}_rows"]
    np.testing.assert_array_equal(rows[:, 0], gold[f"{name}_n"])
    np.testing.assert_array_equal(rows[:, 1:4], want[:, :3])
    np.testing.assert_allclose(rows[:, 4:], want[:, 3:], rtol=2e-5, atol=0, equal_nan=True)
    restated = metric_rows_var(inp["pred"], inp["gt"], kw["min_depth"], kw["max_depth"], kw["crop"])
    np.testing.assert_allclose(rows, restated, rtol=2e-5, atol=0, equal_nan=True)

    m = magnet_b200.DepthMetrics(kw["min_depth"], kw["max_depth"], crop=kw["crop"])
    for i in range(kw["n"]):
        m.update(pred[i:i + 1], gt[i:i + 1], variance=True)
    value = m.value()
    np.testing.assert_allclose([value[k] for k in gold["keys"]], gold[f"{name}_avg"], rtol=2e-5, atol=0, equal_nan=True)


def test_sigma_form_is_unchanged_and_instances_refuse_mixing(cuda):
    inp = metric_inputs("nyu")
    pred, gt = torch.from_numpy(inp["pred"]).to(cuda), torch.from_numpy(inp["gt"]).to(cuda)
    sq = pred.clone()
    sq[:, 1] = pred[:, 1] * pred[:, 1]
    a = ops.depth_metrics(sq, gt, min_depth=1e-3, max_depth=10.0, variance=True)
    b = ops.depth_metrics(pred, gt, min_depth=1e-3, max_depth=10.0)
    assert torch.equal(a.nan_to_num(), b.nan_to_num())                 # var = sigma * sigma: the same sums
    m = magnet_b200.DepthMetrics(1e-3, 10.0)
    m.update(pred, gt, variance=True)
    with pytest.raises(_lib.MagnetError):
        m.update(pred, gt)
    with pytest.raises(_lib.MagnetError):
        m.update(pred[:, :1], gt, nearest=True)
    g = magnet_b200.DepthMetrics(1e-3, 10.0)
    g.update(pred, gt)
    with pytest.raises(_lib.MagnetError):
        g.update(pred, gt, variance=True)
