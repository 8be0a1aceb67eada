"""F-Net evaluation on the H100 (ops.plane_depth, ops.depth_metrics(nearest=True), MagnetF.predict): the soft-argmin
against float64 and bit for bit against the training loss's prediction, the reference's train_FNet validate() output
(tests/golden/fnet_metrics.npz), the nearest form against the numpy restatement over fuzz shapes, the end-to-end flow
against the reference's data flow on the device, run-to-run bit-identity and CUDA-graph capture."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import magnet_b200
from magnet_b200 import _lib, ops
from magnet_b200.homography import plane_sweep_f
from magnet_b200.synthetic import make_inputs
from tests.depth_metrics_ref import KEYS
from tests.fnet_metrics_ref import CASES, NLL, assert_rows_match, case_inputs, metric_rows_nearest, soft_argmin64, \
    soft_argmin_bound, threshold_allowance
from tests.fnet_ref import sid_centres
from tests.test_fnet_metrics_cpu import golden
from tests.test_gpu_metrics import assert_rows_match_restatement

pytestmark = pytest.mark.gpu


def _t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _scores(B, D, h, w, seed):
    """Seeded scores with planted rows: all -inf, one +inf, one NaN, one dominant plane."""
    rng = np.random.default_rng(seed)
    s = rng.normal(0.0, 4.0, (B, D, h, w)).astype(np.float32)
    s[0, :, 0, 0] = -np.inf
    s[0, D // 2, 0, 1] = np.inf
    s[B - 1, D - 1, 1, 2] = np.nan
    s[B - 1, D // 3, 2, 3] = np.float32(1e4)
    return s


@pytest.mark.parametrize("scores", [True, False], ids=["scores", "probabilities"])
@pytest.mark.parametrize("D", [1, 5, 80, 256])
def test_soft_argmin_within_bound_of_float64(cuda, D, scores):
    s = _scores(2, D, 37, 53, seed=D)
    planes = sid_centres(1e-3, 80.0, D).numpy().reshape(-1)
    prob = torch.softmax(torch.from_numpy(s), dim=1)
    vol = s if scores else prob.numpy()
    got = ops.plane_depth(_t(vol, cuda), planes.tolist(), scores=scores)
    assert got.shape == (2, 1, 37, 53) and got.dtype == torch.float32
    got = got.cpu().numpy()
    want = soft_argmin64(vol, planes, scores)
    torch_nan = torch.isnan(torch.sum(prob * torch.from_numpy(planes).view(1, -1, 1, 1), 1, keepdim=True)).numpy()
    np.testing.assert_array_equal(np.isnan(got), np.isnan(want))
    np.testing.assert_array_equal(np.isnan(got), torch_nan)
    assert np.isnan(got[0, 0, 0, 0]) and np.isnan(got[1, 0, 1, 2]) and (D == 1 or np.isnan(got[0, 0, 0, 1]))
    fin = ~np.isnan(want)
    err = np.abs(got[fin] - want[fin]).max()
    assert err <= soft_argmin_bound(planes), (err, soft_argmin_bound(planes))
    if scores:
        assert got[1, 0, 2, 3] == planes[D // 3]                            # the dominant plane, exactly


def test_scores_form_is_the_training_loss_prediction_bit_for_bit(cuda):
    """fnet_l1's forward with a one-pixel mask, gt = 0 and count 1 returns exactly that pixel's |prediction|."""
    B, D, h, w = 2, 80, 30, 41
    s = _t(_scores(B, D, h, w, seed=7), cuda)
    d_center = magnet_b200.sid_planes(1e-3, 10.0, D, device=cuda)
    got = ops.plane_depth(s, d_center, scores=True)
    gt = torch.zeros(B, 1, h, w, device=cuda)
    rng = np.random.default_rng(3)
    pixels = [(1, 2, 3)] + [(int(rng.integers(B)), int(rng.integers(h)), int(rng.integers(w))) for _ in range(7)]
    for b, y, x in pixels:
        if torch.isnan(got[b, 0, y, x]):                                     # a planted row
            continue
        mask = torch.zeros(B, 1, h, w, device=cuda, dtype=torch.uint8)
        mask[b, 0, y, x] = 1
        loss = ops.fnet_l1_loss(s, d_center.reshape(-1).tolist(), gt, mask, count=1)
        assert loss.item() == abs(got[b, 0, y, x].item()), (b, y, x)


@pytest.mark.parametrize("name", list(CASES))
def test_matches_reference_validate(cuda, name):
    """The ops call on the scores against train_FNet's validate() on the probabilities: n exact, a1-a3 within the
    pixels the soft-argmin bound can move across a threshold, the rest within 1e-4, nll exactly 0.0."""
    z, kw, inp = golden(), CASES[name], case_inputs(name)
    pred = ops.plane_depth(_t(inp["scores"], cuda), inp["planes"].tolist(), scores=True)
    m = magnet_b200.DepthMetrics(kw["min_depth"], kw["max_depth"], crop=kw["crop"])
    rows = m.update(pred, _t(inp["gt"], cuda), nearest=True)
    assert rows.shape == (1, kw["n"], 13) and rows.dtype == torch.float64
    p64 = soft_argmin64(inp["scores"], inp["planes"], scores=True)
    allowance = threshold_allowance(p64, inp["gt"], kw["min_depth"], kw["max_depth"], kw["crop"],
                                    soft_argmin_bound(inp["planes"]))
    assert_rows_match(rows[0].cpu().numpy(), z[f"{name}_n"], z[f"{name}_rows"], allowance)
    value = m.value()
    assert value["nll"] == 0.0 and list(value) == list(KEYS)
    got = np.array([value[key] for key in KEYS])
    np.testing.assert_allclose(got[3:], z[f"{name}_avg"][3:], rtol=1e-4, atol=0, equal_nan=True)
    # the average of a1-a3 moves by at most the mean over images of each image's allowance / n
    tol = (allowance / np.maximum(z[f"{name}_n"], 1)[:, None]).sum(axis=0) / kw["n"] + 1e-12
    np.testing.assert_array_equal(np.isnan(got[:3]), np.isnan(z[f"{name}_avg"][:3]))
    assert (np.nan_to_num(np.abs(got[:3] - z[f"{name}_avg"][:3])) <= tol).all(), (got[:3], z[f"{name}_avg"][:3], tol)
    assert m.images() == kw["n"]


FUZZ = [  # B, h, w, H, W, P, crop
    (1, 12, 16, 48, 64, 1, None),
    (2, 15, 20, 50, 70, 2, None),
    (3, 37, 130, 37, 130, 1, "garg"),            # h == H, w == W
    (2, 22, 76, 88, 304, 3, "eigen"),
    (1, 7, 9, 30, 31, 1, None),
    (2, 30, 64, 61, 64, 2, "garg"),              # w == W, odd ratio in y
    (1, 1, 1, 5, 9, 1, None),
    (2, 44, 100, 88, 200, 1, None),              # exactly doubled: ATen's shortcut
]


@pytest.mark.parametrize("B,h,w,H,W,P,crop", FUZZ)
def test_nearest_form_matches_restatement_over_fuzz_shapes(cuda, B, h, w, H, W, P, crop):
    rng = np.random.default_rng(B * 1000 + h * 10 + W + P)
    planes = np.linspace(0.3, 11.0, 16).astype(np.float32).tolist()
    preds = []
    for p in range(P):
        pred = ops.plane_depth(_t(rng.normal(0.0, 3.0, (B, 16, h, w)).astype(np.float32), cuda), planes, scores=True)
        flat = pred.view(-1)
        for val in (np.nan, np.inf, -np.inf, 1e-5, 50.0):
            flat[_t(rng.random(flat.numel()) < 0.01, cuda)] = float(val)
        preds.append(pred)
    gt = rng.uniform(0.3, 12.0, (B, 1, H, W)).astype(np.float32)
    gt[rng.random(gt.shape) < 0.15] = 0
    gt[rng.random(gt.shape) < 0.02] = 15.0                                    # above max_depth
    got = ops.depth_metrics(preds, _t(gt, cuda), min_depth=1e-3, max_depth=10.0, crop=crop, nearest=True)
    assert got.shape == (P, B, 13)
    want = np.stack([metric_rows_nearest(p.cpu().numpy(), gt, 1e-3, 10.0, crop) for p in preds])
    got = got.cpu().numpy()
    assert (want[..., 0] > 0).all()
    assert (got[..., 1 + NLL] == 0.0).all()
    assert_rows_match_restatement(got, want)


def _gt(B, H, W, hi, seed, dev):
    rng = np.random.default_rng(seed)
    gt = rng.uniform(0.5, 0.9 * hi, (B, 1, H, W)).astype(np.float32)
    gt[rng.random(gt.shape) < 0.2] = 0
    gt[rng.random(gt.shape) < 0.02] = np.float32(1.5 * hi)
    return _t(gt, dev)


@pytest.mark.parametrize("shape", [dict(B=2, V=4, h=120, w=160, hi=10.0, family="scannet", crop=None),
                                   dict(B=2, V=2, h=88, w=304, hi=80.0, family="kitti", crop="garg")],
                         ids=["scannet", "kitti"])
def test_predict_and_metrics_against_reference_data_flow(cuda, shape):
    """MagnetF(Identity).predict + DepthMetrics(nearest) against est_costvolume_F -> torch.sum(prob * d_center) ->
    F.interpolate(nearest) -> the metric block, at full ScanNet / KITTI sizes with 80 SID planes."""
    B, V, h, w, hi, crop = shape["B"], shape["V"], shape["h"], shape["w"], shape["hi"], shape["crop"]
    inp = make_inputs(B=B, V=V, D=8, H=h, W=w, C=64, seed=43, depth="smooth", family=shape["family"],
                      invalid=[(1, V - 1)])
    g = inp.to(cuda)
    d_center = magnet_b200.sid_planes(1e-3, hi, 80, device=cuda)
    gt = _gt(B, 4 * h, 4 * w, hi, seed=44, dev=cuda)
    model = magnet_b200.MagnetF(torch.nn.Identity()).to(cuda)
    pred = model.predict(g.ref_feat, g.nghbr_feat, g.nghbr_poses, inp.is_valid, inp.cam_intrins, d_center)
    assert pred.shape == (B, 1, h, w) and not pred.requires_grad
    m = magnet_b200.DepthMetrics(1e-3, hi, crop=crop)
    rows = m.update(pred, gt, nearest=True)[0].cpu().numpy()
    # the reference's data flow on the device
    prob = magnet_b200.est_costvolume_F(d_center, g.ref_feat, g.nghbr_feat, g.R, g.t, inp.is_valid, inp.cam_intrins)
    ref_pred = torch.sum(prob * d_center, dim=1, keepdim=True)
    up = F.interpolate(ref_pred, size=[4 * h, 4 * w], mode="nearest")
    want = metric_rows_nearest(up.cpu().numpy(), gt.cpu().numpy(), 1e-3, hi, crop)
    # both predictions lie within the soft-argmin bound of the float64 soft-argmin of the scores
    scores = plane_sweep_f(d_center, g.ref_feat, g.nghbr_feat, g.R, g.t, inp.is_valid, inp.cam_intrins, softmax=False)
    planes = d_center.reshape(-1).cpu().numpy()
    p64 = soft_argmin64(scores.cpu().numpy(), planes, scores=True)
    bound = soft_argmin_bound(planes)
    assert np.isfinite(p64).all()
    assert np.abs(pred.cpu().numpy() - p64).max() <= bound
    assert np.abs(ref_pred.cpu().numpy() - p64).max() <= 2 * bound
    allowance = threshold_allowance(p64, gt.cpu().numpy(), 1e-3, hi, crop, 2 * bound)
    assert_rows_match(rows, want[:, 0], want[:, 1:], allowance)
    assert (rows[:, 0] > 1000).all()


def test_runs_are_bit_identical_and_capture_in_a_cuda_graph(cuda):
    B, D, h, w, H, W = 2, 80, 22, 76, 88, 304
    planes = sid_centres(1e-3, 80.0, D).numpy().reshape(-1).tolist()
    s = _t(_scores(B, D, h, w, seed=61), cuda)
    gt = _gt(B, H, W, 80.0, seed=62, dev=cuda)
    a, b = ops.plane_depth(s, planes, scores=True), ops.plane_depth(s, planes, scores=True)
    assert torch.equal(a.nan_to_num(), b.nan_to_num()) and torch.equal(a.isnan(), b.isnan())
    r1 = ops.depth_metrics(a, gt, min_depth=1e-3, max_depth=80.0, crop="garg", nearest=True)
    r2 = ops.depth_metrics(b, gt, min_depth=1e-3, max_depth=80.0, crop="garg", nearest=True)
    assert torch.equal(r1, r2)
    m = magnet_b200.DepthMetrics(1e-3, 80.0, crop="garg")
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        m.update(ops.plane_depth(s, planes, scores=True), gt, nearest=True)   # warm-up creates the accumulator
    torch.cuda.current_stream().wait_stream(st)
    m.reset()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = m.update(ops.plane_depth(s, planes, scores=True), gt, nearest=True)
    eager = []
    for seed in (63, 64, 65):
        s2, gt2 = _t(_scores(B, D, h, w, seed=seed), cuda), _gt(B, H, W, 80.0, seed=seed + 10, dev=cuda)
        s.copy_(s2)
        gt.copy_(gt2)
        graph.replay()
        want = ops.depth_metrics(ops.plane_depth(s2, planes, scores=True), gt2, min_depth=1e-3, max_depth=80.0,
                                 crop="garg", nearest=True)
        assert torch.equal(captured.nan_to_num(), want.nan_to_num())
        eager.append(want)
    torch.cuda.synchronize()
    rows = torch.cat(eager, dim=1).cpu().numpy()
    assert m.images() == 3 * B
    value = m.value()
    assert value["nll"] == 0.0
    np.testing.assert_allclose([value[key] for key in KEYS], rows[0, :, 1:].mean(axis=0), rtol=1e-13, atol=0)
    with pytest.raises(_lib.MagnetError):                                    # the other form is refused
        m.update(torch.ones(B, 2, H, W, device=cuda), gt)


def test_half_volume_is_upcast_and_gaussian_instance_refuses_nearest(cuda):
    s = _t(_scores(1, 8, 9, 11, seed=5), cuda)
    planes = np.linspace(0.5, 4.0, 8).tolist()
    assert torch.equal(ops.plane_depth(s.half(), planes, scores=True).nan_to_num(),
                       ops.plane_depth(s.half().float(), planes, scores=True).nan_to_num())
    m = magnet_b200.DepthMetrics(1e-3, 10.0)
    gt = torch.rand(1, 1, 36, 44, device=cuda) * 5
    m.update(torch.rand(1, 2, 36, 44, device=cuda) + 1, gt)
    with pytest.raises(_lib.MagnetError):
        m.update(ops.plane_depth(s, planes, scores=True), gt, nearest=True)
    with pytest.raises(_lib.MagnetError):
        ops.plane_depth(s, planes[:7], scores=True)
    with pytest.raises(_lib.MagnetError):
        ops.depth_metrics(torch.rand(1, 1, 37, 11, device=cuda), gt, min_depth=1e-3, max_depth=10.0, nearest=True)
