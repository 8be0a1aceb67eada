"""tests/dnet_loss_ref.py without a GPU: the float64 restatement of the fused D-Net loss (loss, raw and mask gradients)
against float64 autograd of the reference's formula — upsample_depth_via_mask, activation_G and DnetLoss with its
boolean indexing — and the properties of its bounds and ambiguity report."""
import pytest
import torch
import torch.nn.functional as F

from tests import dnet_loss_ref as dr


def _upsample(raw, mask, k):
    """upsample_depth_via_mask (D_dense_depth.py:86-100), restated in torch: softmax over the 9 taps, weighted sum of
    the zero-padded 3x3 neighbourhood, pixel shuffle."""
    B, C, H, W = raw.shape
    m = torch.softmax(mask.view(B, 1, 9, k, k, H, W), 2)
    nb = F.unfold(raw, 3, padding=1).view(B, C, 9, 1, 1, H, W)
    up = (m * nb).sum(2).permute(0, 1, 4, 2, 5, 3)
    return up.reshape(B, C, k * H, k * W)


def _autograd(raw, mask, gt, gtm, k):
    raw = raw.double().requires_grad_()
    mask = mask.double().requires_grad_()
    up = _upsample(raw, mask, k)
    mu, v = torch.split(up, 1, 1)
    var = F.elu(v) + 1.0 + 1e-10                                    # activation_G (DNET.py:56-60)
    g, mu, var = gt.double()[gtm], mu[gtm], var[gtm]                # DnetLoss (utils/losses.py:13-22)
    var = torch.where(var < 1e-10, torch.full_like(var, 1e-10), var)
    loss = (torch.square(mu - g) / (2 * var) + 0.5 * torch.log(var)).mean()
    loss.backward()
    return float(loss.detach()), raw.grad, mask.grad


@pytest.mark.parametrize("B,H,W,k,mask", [(1, 1, 1, 1, "dense"), (2, 5, 7, 2, "dense"), (1, 3, 9, 4, "sparse"),
                                          (2, 4, 3, 8, "dense"), (3, 6, 5, 4, "dense")])
def test_restatement_matches_float64_autograd(B, H, W, k, mask):
    raw, lg, gt, gtm, _ = dr.loss_inputs(B, H, W, k, mask=mask, high=2, seed=B * 10 + k)
    r = dr.dnet_nll(raw, lg, gt, gtm, k)
    loss, g_raw, g_mask = _autograd(raw, lg, gt, gtm, k)
    assert abs(r["loss"] - loss) <= 1e-12 * abs(loss)
    torch.testing.assert_close(r["grad_raw"], g_raw, rtol=1e-10, atol=1e-12 * float(g_raw.abs().max()))
    torch.testing.assert_close(r["grad_mask"], g_mask, rtol=1e-10, atol=1e-12 * float(g_mask.abs().max()))
    for key in ("loss_bound",):
        assert r[key] > 0
    for key in ("grad_raw_bound", "grad_mask_bound"):
        assert (r[key] > 0).all() and torch.isfinite(r[key]).all()


def test_upstream_gradient_scales_the_gradients():
    raw, lg, gt, gtm, _ = dr.loss_inputs(2, 4, 5, 4, seed=3)
    r1, r3 = dr.dnet_nll(raw, lg, gt, gtm, 4), dr.dnet_nll(raw, lg, gt, gtm, 4, grad=-3.0)
    torch.testing.assert_close(r3["grad_raw"], -3.0 * r1["grad_raw"], rtol=1e-14, atol=0)
    torch.testing.assert_close(r3["grad_raw_bound"], 3.0 * r1["grad_raw_bound"], rtol=1e-14, atol=0)


def test_deep_blocks_are_collapsed_and_unclamped():
    """v_up <= -20: the restatement takes var = fp32(1e-10) exactly (expm1f(v) == -1 in fp32), which is not below the
    clamp, so the gradient into v is not cut (g_v = g_var e^v != 0); the band just above -17.5 is reported ambiguous."""
    raw, lg, gt, gtm, deep = dr.loss_inputs(2, 8, 9, 4, deep=3, seed=5)
    r = dr.dnet_nll(raw, lg, gt, gtm, 4)
    assert deep.any() and r["collapsed"][deep].all()
    assert (r["var"][r["collapsed"]] == dr.VAR_MIN).all()
    assert torch.tensor(1e-10, dtype=torch.float32) == torch.tensor(dr.VAR_MIN, dtype=torch.float32)
    assert not (torch.tensor(dr.VAR_MIN, dtype=torch.float32) < 1e-10)        # torch's fp32 comparison: no clamp
    assert (r["grad_raw"][:, 1] != 0).any()
    mid = (r["var"] > dr.VAR_MIN) & (r["var"] < 1e-5)
    assert r["ambiguous"][mid].all()


def test_float64_elu_is_never_clamped():
    """In float64 as well, elu(v) + 1 + 1e-10 >= 1e-10 for every finite v: the clamp of DnetLoss is dead."""
    v = torch.tensor([-1e30, -800.0, -103.0, -20.0, -17.0, -1e-30, 0.0, 1e-30, 5.0, 1e30], dtype=torch.float64)
    assert (F.elu(v) + 1.0 + 1e-10 >= 1e-10).all()
    v32 = v.float()
    assert (F.elu(v32) + 1.0 + 1e-10 >= torch.tensor(1e-10, dtype=torch.float32)).all()
