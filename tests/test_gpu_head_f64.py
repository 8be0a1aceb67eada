"""The fused heads on the tensor cores, element by element, against the float64 restatements of tests/head_ref.py: the
G-Net head's forward (h0, h1, h2, raw, the updated Gaussian), every stage of its backward chain (d_raw, grad_prev,
d_h2, d_h1, grad_invariant) and every weight and bias gradient, and the mask head with the learned upsampling.

The G-Net head is driven through the C ABI (pack, training forward, backward on a workspace this file owns), so the
saved maps and the workspace's d_h2, d_h1, d_raw are readable: each backward stage is checked from the kernel's own
fp32 input to that stage, with the ReLU masks of the kernel's saved activations (exact, so no pixel is left out).

Tolerance: |got - ref| <= c u bound, u = 2^-24, c = C_TOL = 32 for every output; the worst err / (u bound) is printed
per output.  Cases: D at the edges of the 16-channel chunks, grids at the edges of the 8 x 16 tiles and of the
1024-pixel weight-gradient chunks, cfg2 / cfg3 / N_s = 5, per-pixel magnitude ladders 2^0 ... 2^-45 across every
16-pixel row (zero hidden biases, so every layer sees them), a batch whose images differ by 1e6 in cost magnitude
(one cost scale per call) and uniform input scales 1e-3 ... 1e3."""
import ctypes as C

import numpy as np
import pytest
import torch

import magnet_b200
from magnet_b200 import _lib, ops
from magnet_b200._lib import check, lib
from magnet_b200.matcher import GNET
from tests import head_ref as hr

pytestmark = pytest.mark.gpu

C_TOL = 32.0


def _close(got, want, bound, what):
    got = got.detach().to(torch.float64)
    want = torch.as_tensor(want, dtype=torch.float64, device=got.device).reshape(got.shape)
    bound = torch.as_tensor(bound, dtype=torch.float64, device=got.device).reshape(got.shape)
    assert torch.isfinite(got).all(), f"{what}: non-finite output"
    tol = C_TOL * hr.U * bound
    err = (got - want).abs()
    bad = err > tol
    ratio = float(torch.where(tol > 0, err / torch.where(tol > 0, tol, torch.ones_like(tol)),
                              torch.where(err > 0, torch.full_like(err, float("inf")), torch.zeros_like(err))).max())
    print(f"{what}: max |err| / (u bound) = {ratio * C_TOL:.3g}")
    if bad.any():
        i = np.unravel_index(int(torch.argmax(torch.where(bad, err / tol.clamp_min(1e-300), torch.zeros_like(err)))),
                             bad.shape)
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements beyond c u bound; worst at {i}: got "
                             f"{float(got[i])!r}, want {float(want[i])!r}, tol {float(tol[i])!r}")


def _tile_ladder(H, W, dev):
    """(H, W) scales: hr.ladder along each row of 16 pixels (an 8 x 16 tile's warp row), reversed between
    horizontally and vertically neighbouring tiles."""
    rows = [hr.ladder(W, parity=y // 8) for y in range(H)]
    return torch.tensor(np.stack(rows), dtype=torch.float32, device=dev)


def _flat_ladder(H, W, dev):
    """(H, W) scales: hr.ladder over the flattened pixels, i.e. the backward chain's 16-pixel groups."""
    return torch.tensor(hr.ladder(H * W).reshape(H, W), dtype=torch.float32, device=dev)


def _ids(c):
    return "_".join(f"{k}{v}" for k, v in c.items())


# ---------------------------------------------------------------------------------------------------------------------
# G-Net head, forward and backward

def _gnet_inputs(B, D, H, W, dev, seed, scale=None, ladder=False, mixed=False):
    torch.manual_seed(seed)
    g = GNET(ch_in=D + 16).to(dev)
    gen = torch.Generator(device=dev).manual_seed(seed)
    cost = torch.randn(B, D, H, W, device=dev, generator=gen)
    inv = 0.3 * torch.randn(B, 128, H, W, device=dev, generator=gen)
    prev = torch.cat([1 + torch.rand(B, 1, H, W, device=dev, generator=gen),
                      0.1 + 0.5 * torch.rand(B, 1, H, W, device=dev, generator=gen)], 1)
    gout = torch.randn(B, 2, H, W, device=dev, generator=gen)
    if scale is not None:
        cost *= scale
        inv *= scale / 0.3
    if ladder:
        cost.zero_()
        with torch.no_grad():
            g.gnet[2].bias.zero_()
            g.gnet[4].bias.zero_()
        inv *= _tile_ladder(H, W, dev)
        gout *= _flat_ladder(H, W, dev)
    if mixed:
        cost[0] *= 1e3
        cost[1] *= 1e-3
    return g, cost, inv, prev, gout


def _gnet_run(g, cost, inv, prev, gout):
    """Pack, training forward and backward through the C ABI -> dict of every output and intermediate (fp32)."""
    B, D, H, W = cost.shape
    L = lib()
    dev = cost.device
    s = g.gnet
    ws = [t.detach().contiguous() for t in (s[0].weight[:, :D], s[2].weight, s[2].bias, s[4].weight, s[4].bias,
                                             s[6].weight, s[6].bias)]
    new = lambda *shape: torch.empty(*shape, device=dev, dtype=torch.float32)
    packed = torch.empty(int(L.magnet_gnet_train_weights_bytes(D)), device=dev, dtype=torch.uint8)
    saved = new(int(L.magnet_gnet_saved_bytes(B, H, W)) // 4)
    work = new(int(L.magnet_gnet_bwd_workspace_bytes(B, D, H, W)) // 4)
    scratch = torch.empty(_lib.MAGNET_GNET_SCRATCH_BYTES // 4, device=dev, dtype=torch.int32)
    r = dict(out=new(B, 2, H, W), grad_inv=new(B, 128, H, W), dW0=new(128, D, 3, 3), dW1=new(128, 128), db1=new(128),
             dW2=new(128, 128), db2=new(128), dW3=new(2, 128), db3=new(2), grad_prev=new(B, 2, H, W))
    a = _lib.GnetTrainArgs(B=B, D=D, H=H, W=W, cost=cost.data_ptr(), invariant=inv.data_ptr(),
                           packed_weights=packed.data_ptr(), prev_gmm=prev.data_ptr(), scratch=scratch.data_ptr(),
                           out=r["out"].data_ptr(), saved=saved.data_ptr(), grad_out=gout.data_ptr(),
                           workspace=work.data_ptr(), grad_invariant=r["grad_inv"].data_ptr(),
                           grad_w0_cost=r["dW0"].data_ptr(), grad_w1=r["dW1"].data_ptr(), grad_b1=r["db1"].data_ptr(),
                           grad_w2=r["dW2"].data_ptr(), grad_b2=r["db2"].data_ptr(), grad_w3=r["dW3"].data_ptr(),
                           grad_b3=r["db3"].data_ptr(), grad_prev=r["grad_prev"].data_ptr())
    st = torch.cuda.current_stream(dev).cuda_stream
    with torch.cuda.device(dev):
        check(L.magnet_gnet_pack_train_weights_f32(*(t.data_ptr() for t in ws), D, packed.data_ptr(), st),
              "magnet_gnet_pack_train_weights_f32")
        check(L.magnet_gnet_train_fwd_f32(C.byref(a), st), "magnet_gnet_train_fwd_f32")
        check(L.magnet_gnet_bwd_f32(C.byref(a), st), "magnet_gnet_bwd_f32")
    torch.cuda.synchronize(dev)
    plane, pix = B * 128 * H * W, B * H * W
    for i, n in enumerate(("h0", "h1", "h2")):
        r[n] = saved[i * plane:(i + 1) * plane].view(B, 128, H, W)
    r["raw"] = saved[3 * plane:3 * plane + 2 * pix].view(B, 2, H, W)
    r["d_h2"] = work[:plane].view(B, 128, H, W)                     # launch_gnet_bwd: dh, dh + plane, dh + 2 plane
    r["d_h1"] = work[plane:2 * plane].view(B, 128, H, W)
    r["d_raw"] = work[2 * plane:2 * plane + 2 * pix].view(B, 2, H, W)
    return ws, r


def _check_gnet(g, cost, inv, prev, gout):
    ws, k = _gnet_run(g, cost, inv, prev, gout)
    f = hr.gnet_forward(cost, inv, ws, prev)
    for n in ("h0", "h1", "h2", "raw", "out"):
        _close(k[n], f[n], f[n + "_bound"], n)
    w0, w1, b1, w2, b2, w3, b3 = ws
    d_raw, b_raw, gp, bp = hr.update_bwd(k["raw"], prev, gout)
    _close(k["d_raw"], d_raw, b_raw, "d_raw")
    _close(k["grad_prev"], gp, bp, "grad_prev")
    _close(k["d_h2"], *hr.w3t(w3, k["d_raw"], k["h2"]), "d_h2")
    _close(k["d_h1"], *hr.grad_layer(w2, k["d_h2"], k["h1"]), "d_h1")
    _close(k["grad_inv"], *hr.grad_layer(w1, k["d_h1"], k["h0"]), "grad_inv")
    for nm, a, x in (("1", k["d_h1"], k["h0"]), ("2", k["d_h2"], k["h1"]), ("3", k["d_raw"], k["h2"])):
        dw, bw, db, bb = hr.wgrad(a, x)
        _close(k["dW" + nm], dw, bw, "dW" + nm)
        _close(k["db" + nm], db, bb, "db" + nm)
    _close(k["dW0"], *hr.wgrad0(k["grad_inv"], cost), "dW0")


GNET_CASES = (
    # D at the edges of the 16-channel chunks (and of the 64-column dW0 tiles: 9 D = 45, 63, 72, 153)
    [dict(B=2, D=d, H=9, W=17) for d in (1, 5, 7, 8, 15, 16, 17, 31, 33, 64, 255, 256)]
    # grids at the 8 x 16 tile edges, B = 3; B H W = 1023, 1024, 1025 around one weight-gradient chunk
    + [dict(B=3, D=17, H=h, W=w) for h, w in ((1, 1), (7, 15), (8, 16), (9, 17), (17, 33))]
    + [dict(B=3, D=8, H=11, W=31), dict(B=2, D=8, H=16, W=32), dict(B=1, D=8, H=25, W=41)]
    # production shapes: cfg2, cfg3, N_s = 5 at cfg2
    + [dict(B=8, D=64, H=120, W=160), dict(B=4, D=64, H=88, W=304), dict(B=8, D=5, H=120, W=160)]
    # magnitude ladders, a mixed-scale batch, uniform scales
    + [dict(B=2, D=16, H=16, W=64, ladder=True), dict(B=3, D=7, H=9, W=40, ladder=True),
       dict(B=3, D=16, H=12, W=20, mixed=True)]
    + [dict(B=2, D=64, H=24, W=40, scale=s) for s in (1e-3, 1.0, 1e3)])


@pytest.mark.parametrize("case", GNET_CASES, ids=_ids)
def test_gnet_head_forward_and_backward(cuda, case):
    case = dict(case)
    B, D, H, W = (case.pop(n) for n in "BDHW")
    _check_gnet(*_gnet_inputs(B, D, H, W, cuda, seed=B * 1000 + D * 7 + H * W, **case))


# ---------------------------------------------------------------------------------------------------------------------
# mask head and upsampling

def _mask_inputs(B, H, W, P, dev, seed, scale=1.0, ladder=False):
    torch.manual_seed(seed)
    mh = magnet_b200.MagnetHead(dnet_fdim=16).mask_head.to(dev).eval()
    gen = torch.Generator(device=dev).manual_seed(seed)
    pre0 = scale * torch.randn(B, 128, H, W, device=dev, generator=gen)
    preds = [torch.cat([1 + torch.rand(B, 1, H, W, device=dev, generator=gen),
                        0.1 + torch.rand(B, 1, H, W, device=dev, generator=gen)], 1) * scale for _ in range(P)]
    if ladder:
        with torch.no_grad():
            for i in (2, 4, 6):
                mh[i].bias.zero_()
        pre0 *= _tile_ladder(H, W, dev)
    return mh, pre0, preds


MASK_CASES = (
    [dict(B=3, H=h, W=w, P=p) for (h, w), p in (((1, 1), 9), ((7, 13), 3), ((8, 16), 8), ((9, 17), 1), ((17, 33), 9))]
    + [dict(B=8, H=120, W=160, P=3), dict(B=4, H=88, W=304, P=3)]
    + [dict(B=2, H=16, W=64, P=3, ladder=True), dict(B=3, H=9, W=40, P=1, ladder=True)]
    + [dict(B=2, H=24, W=40, P=3, scale=s) for s in (1e-3, 1.0, 1e3)])


@pytest.mark.parametrize("case", MASK_CASES, ids=_ids)
def test_mask_head_and_upsampling(cuda, case):
    case = dict(case)
    B, H, W, P = (case.pop(n) for n in "BHWP")
    mh, pre0, preds = _mask_inputs(B, H, W, P, cuda, seed=B + H * W + P, **case)
    with torch.no_grad():
        got = ops.mask_upsample(pre0, ops.pack_mask_weights(mh), preds)
    ws = (mh[2].weight, mh[2].bias, mh[4].weight, mh[4].bias, mh[6].weight, mh[6].bias)
    _, _, want = hr.mask_forward(pre0, ws, preds)
    assert len(got) == P
    for i, (g, (w, b)) in enumerate(zip(got, want)):
        _close(g, w, b, f"mask out[{i}]")
