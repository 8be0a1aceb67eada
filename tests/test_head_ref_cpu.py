"""The float64 restatements of tests/head_ref.py, on the CPU: their values against float64 autograd of the modules (GNET
and MagnetHead().mask_head, plain ATen ops) at 1e-12 of each bound, and their bounds against a numpy emulation of the
kernels' SPLIT16 arithmetic (fp16 split with subnormals and the shift clamp, exact products, an fp32 rounding after
each MMA) on per-pixel magnitude ladders: the emulation must lie within c u bound, and emulated mutants of the kernels
outside it, so the gate of tests/test_gpu_head_f64.py is sharp before it runs on a device."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from magnet_b200.matcher import GNET, MagnetHead
from oracle import torch_ref
from tests import head_ref as hr

REL = 1e-12
C_TOL = 32.0


def _close(got, want, bound, what):
    got, want, bound = (torch.as_tensor(x, dtype=torch.float64) for x in (got, want, bound))
    assert got.shape == want.shape, (what, got.shape, want.shape)
    assert torch.isfinite(got).all(), what
    err = (got - want).abs()
    assert (err <= REL * bound).all(), (what, float((err / bound.clamp_min(1e-300)).max()))


# ---------------------------------------------------------------------------------------------------------------------
# values against float64 autograd

def _gnet_case(B, D, H, W, seed):
    torch.manual_seed(seed)
    g = GNET(ch_in=D + 16).double()
    gen = torch.Generator().manual_seed(seed)
    cost = torch.randn(B, D, H, W, generator=gen, dtype=torch.float64)
    x_d3 = torch.randn(B, 16, H, W, generator=gen, dtype=torch.float64)
    prev = torch.cat([1 + torch.rand(B, 1, H, W, generator=gen, dtype=torch.float64),
                      0.1 + torch.rand(B, 1, H, W, generator=gen, dtype=torch.float64)], 1)
    gout = torch.randn(B, 2, H, W, generator=gen, dtype=torch.float64)
    return g, cost, x_d3, prev, gout


@pytest.mark.parametrize("shape", [(1, 1, 1, 1), (2, 5, 7, 9), (3, 17, 4, 6)], ids=lambda s: "x".join(map(str, s)))
def test_gnet_restatement_is_autograd(shape):
    B, D, H, W = shape
    g, cost, x_d3, prev, gout = _gnet_case(B, D, H, W, seed=D + H)
    s = g.gnet
    prev = prev.clone().requires_grad_(True)
    z = [s[0](torch.cat([cost, x_d3], 1))]
    h = [F.relu(z[0])]
    for i in (2, 4):
        z.append(s[i](h[-1]))
        h.append(F.relu(z[-1]))
    raw = s[6](h[-1])
    for t in z + [raw]:
        t.retain_grad()
    out = torch.cat([prev[:, :1] + raw[:, :1] * prev[:, 1:], (F.elu(raw[:, 1:]) + 1 + 1e-10) * prev[:, 1:]], 1)
    out.backward(gout)
    inv = g.invariant_part(x_d3, D).detach()
    ws = (s[0].weight[:, :D], s[2].weight, s[2].bias, s[4].weight, s[4].bias, s[6].weight, s[6].bias)
    r = hr.gnet_forward(cost, inv, ws, prev)
    for name, want in (("h0", h[0]), ("h1", h[1]), ("h2", h[2]), ("raw", raw), ("out", out)):
        _close(r[name], want.detach(), r[name + "_bound"], name)
    d_raw, b_raw, gp, bp = hr.update_bwd(raw, prev, gout)
    _close(d_raw, raw.grad, b_raw, "d_raw")
    _close(gp, prev.grad, bp, "grad_prev")
    v, b = hr.w3t(s[6].weight, raw.grad, h[2])
    _close(v, z[2].grad, b, "d_h2")
    v, b = hr.grad_layer(s[4].weight, z[2].grad, h[1])
    _close(v, z[1].grad, b, "d_h1")
    v, b = hr.grad_layer(s[2].weight, z[1].grad, h[0])
    _close(v, z[0].grad, b, "d_h0")
    for a, x, li, nm in ((z[1].grad, h[0], 2, "1"), (z[2].grad, h[1], 4, "2"), (raw.grad, h[2], 6, "3")):
        dw, bw, db, bb = hr.wgrad(a, x)
        _close(dw, s[li].weight.grad.view(dw.shape), bw, "dW" + nm)
        _close(db, s[li].bias.grad, bb, "db" + nm)
    dw, bw = hr.wgrad0(z[0].grad, cost)
    _close(dw, s[0].weight.grad[:, :D], bw, "dW0")


@pytest.mark.parametrize("P", [1, 3])
def test_mask_restatement_is_autograd(P):
    torch.manual_seed(P)
    mh = MagnetHead(dnet_fdim=8).mask_head.double()
    gen = torch.Generator().manual_seed(P)
    B, H, W = 2, 5, 7
    pre0 = torch.randn(B, 128, H, W, generator=gen, dtype=torch.float64)
    preds = [torch.cat([1 + torch.rand(B, 1, H, W, generator=gen, dtype=torch.float64),
                        0.1 + torch.rand(B, 1, H, W, generator=gen, dtype=torch.float64)], 1) for _ in range(P)]
    with torch.no_grad():
        mask = mh[2:](F.relu(pre0))
        want = [torch_ref.convex_upsample(p, mask, 4) for p in preds]
    ws = (mh[2].weight, mh[2].bias, mh[4].weight, mh[4].bias, mh[6].weight, mh[6].bias)
    lg, blg, outs = hr.mask_forward(pre0, ws, preds)
    _close(lg, mask, blg, "logits")
    for (o, b), w in zip(outs, want):
        _close(o, w, b, "out")


# ---------------------------------------------------------------------------------------------------------------------
# bounds against the emulated kernels

def _worst(got, want, bound):
    """Largest |got - want| / (u bound): inf where a non-finite value or an error meets a zero bound."""
    got = np.asarray(got, np.float64)
    want, bound = (np.asarray(torch.as_tensor(x).numpy(), np.float64) for x in (want, bound))
    err = np.abs(got - want)
    err = np.where(np.isfinite(got), err, np.inf)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(err == 0, 0.0, err / (hr.U * bound))
    return float(r.max())


KB8 = [slice(16 * k, 16 * k + 16) for k in range(8)]


def _hidden_case(M, seed, signed=False):
    """M pixels (rows of 16) of 128 activations on the ladder 2^0 ... 2^-45, and a 128 x 128 layer."""
    rng = np.random.default_rng(seed)
    a = rng.standard_normal((M, 128))
    a = (a if signed else np.maximum(a, 0)) * hr.ladder(M)[:, None]
    w = rng.uniform(-1, 1, (128, 128)) / np.sqrt(128)
    return a.astype(np.float32), w.astype(np.float32)


def _as_map(x):
    """(M, C) -> (1, C, 1, M)."""
    return torch.from_numpy(np.ascontiguousarray(np.asarray(x, np.float64).T))[None, :, None, :]


def _hidden_forward(a, w, **mut):
    y = hr.split16_gemm(a, w, KB8, **mut)
    return np.maximum(y, 0).T[None, :, None, :]


@pytest.mark.parametrize("seed", [0, 1])
def test_hidden_layer_emulation_within_its_bound_on_the_ladder(seed):
    a, w = _hidden_case(64, seed)
    want, bound = hr.layer(torch.from_numpy(w.astype(np.float64)), None, _as_map(a), torch.zeros(1, 128, 1, 64))
    assert _worst(_hidden_forward(a, w), want, bound) <= C_TOL
    # one scale per 16-pixel row: the small pixels of each row lose every bit
    assert _worst(_hidden_forward(a, w, row_shift="row16"), want, bound) > 1e3 * C_TOL


def test_grad_layer_emulation_within_its_bound_on_the_ladder():
    d, w = _hidden_case(64, 2, signed=True)
    h = torch.ones(1, 128, 1, 64)
    want, bound = hr.grad_layer(torch.from_numpy(w.astype(np.float64)), _as_map(d), h)
    got = hr.split16_gemm(d, w.T, KB8).T[None, :, None, :]
    assert _worst(got, want, bound) <= C_TOL
    # row g's scale for row g + 8: where g + 8 is the larger, fp16 overflows; where it is the smaller, lo underflows
    with np.errstate(over="ignore", invalid="ignore"):
        bad = hr.split16_gemm(d, w.T, KB8, row_shift="g").T[None, :, None, :]
    assert _worst(bad, want, bound) > 1e3 * C_TOL


def test_dropped_lo_hi_product_leaves_the_bound():
    """Activations whose fp16 residual has one sign (0.4 ulp above an fp16 value at the pixel's scale) and positive
    weights: without lo_a hi_w the error is coherent, about 2^-12 of sum |a||w|."""
    rng = np.random.default_rng(5)
    M = 32
    hi = rng.uniform(2.0 ** 14, 2.0 ** 15, (M, 128)).astype(np.float16).astype(np.float64)
    a = (hi * (1 + 0.4 * 2.0 ** -10) * hr.ladder(M)[:, None] * 2.0 ** -14).astype(np.float32)
    w = (rng.uniform(0, 2, (128, 128)) / np.sqrt(128)).astype(np.float32)
    want, bound = hr.layer(torch.from_numpy(w.astype(np.float64)), None, _as_map(a), torch.zeros(1, 128, 1, M))
    assert _worst(_hidden_forward(a, w), want, bound) <= C_TOL
    assert _worst(_hidden_forward(a, w, drop_lohi=True), want, bound) > C_TOL


@pytest.mark.parametrize("bias", [False, True])
def test_mask_layer_emulation_within_its_bound(bias):
    """The 144-column layer on the ladder.  With a bias the small pixels' logits are the bias to within its rounding,
    so the row-scale mutant is only visible with zero biases (as the device test's ladder has them)."""
    rng = np.random.default_rng(7)
    a, _ = _hidden_case(48, 7)
    w = (rng.uniform(-1, 1, (144, 128)) / np.sqrt(128)).astype(np.float32)
    b = rng.uniform(-0.1, 0.1, 144).astype(np.float32) * np.float32(bias)
    want, bound = hr.layer(torch.from_numpy(w.astype(np.float64)), torch.from_numpy(b.astype(np.float64)), _as_map(a),
                           torch.zeros(1, 128, 1, 48), relu=False)
    got = (hr.split16_gemm(a, w, KB8) + b).astype(np.float32).T[None, :, None, :]
    assert _worst(got, want, bound) <= C_TOL
    if not bias:
        bad = (hr.split16_gemm(a, w, KB8, row_shift="row16") + b).T[None, :, None, :]
        assert _worst(bad, want, bound) > 1e3 * C_TOL


@pytest.mark.parametrize("D", [1, 17, 33])
def test_conv3x3_emulation_within_its_bound_in_a_mixed_scale_batch(D):
    """The 3x3 conv of the cost volume with one scale per call: image 0 x 1e3, image 1 x 1e-3, K in the kernel's order
    (16-channel chunk, tap, channel); the small image's error is the floor sum |W0| / s_c of the bound."""
    rng = np.random.default_rng(D)
    B, H, W = 2, 5, 7
    cost = rng.standard_normal((B, D, H, W)) * np.array([1e3, 1e-3]).reshape(B, 1, 1, 1)
    cost = cost.astype(np.float32)
    w0 = (rng.uniform(-1, 1, (128, D, 3, 3)) / np.sqrt(9 * D)).astype(np.float32)
    nc = -(-D // 16)
    unf = F.unfold(torch.from_numpy(cost).double(), 3, padding=1).view(B, D, 9, H * W).numpy()
    A = np.zeros((B, H * W, nc, 9, 16), np.float32)
    Wm = np.zeros((128, nc, 9, 16), np.float32)
    for c in range(D):
        A[:, :, c // 16, :, c % 16] = unf[:, c].transpose(0, 2, 1)
        Wm[:, c // 16, :, c % 16] = w0[:, c].reshape(128, 9)
    A = A.reshape(B * H * W, 144 * nc)
    y = hr.split16_gemm(A, Wm.reshape(128, -1), [slice(16 * k, 16 * k + 16) for k in range(9 * nc)], row_shift="all")
    got = np.maximum(y, 0).reshape(B, H * W, 128).transpose(0, 2, 1).reshape(B, 128, H, W)
    z = lambda *s: torch.zeros(*s, dtype=torch.float64)
    ws = (torch.from_numpy(w0), z(128, 128, 1, 1), z(128), z(128, 128, 1, 1), z(128), z(2, 128, 1, 1), z(2))
    r = hr.gnet_forward(torch.from_numpy(cost), z(B, 128, H, W), ws, torch.ones(B, 2, H, W))
    assert _worst(got, r["h0"], r["h0_bound"]) <= C_TOL


def test_wgrad_emulation_within_its_bound():
    """3xTF32 with the per-slab flush against §3.10's bound, on a laddered gradient and ragged chunk (2500 pixels)."""
    rng = np.random.default_rng(9)
    P = 2500
    a = (rng.standard_normal((P, 24)) * hr.ladder(P)[:, None]).astype(np.float32)
    b = np.maximum(rng.standard_normal((P, 16)), 0).astype(np.float32)
    want = a.astype(np.float64).T @ b.astype(np.float64)
    n = -(-P // 1024)
    bound = (24 + 32 + n) * (np.abs(a).astype(np.float64).T @ np.abs(b).astype(np.float64))
    assert _worst(hr.wgrad3(a, b), want, bound) <= C_TOL
