"""The fused mask-head training loss on the H100, element by element, against the bounded float64 restatement of
tests/mask_train_ref.py (DESIGN §3.13): the saved h1, h2, the loss, the logits' gradient, every prediction gradient,
each backward stage (d_h2, d_h1, grad_pre0) from the kernel's own fp32 input to that stage, and every weight and bias
gradient.  Driven through the C ABI with a saved buffer and a workspace this file owns, so the intermediates are
readable.  Tolerance: |got - ref| <= c u bound, c = 32 for every output; the worst err / (u bound) is printed per
output.  Cases: grids at the tile edges and cfg2 / cfg3, P 1 / 3 / 8, input scales 1e-3 ... 1e3, dense, sparse and
empty gt masks, clamped sigma and an upstream gradient of 0.37.  Sub-pixels where |mu - gt| or sigma^2 - 1e-10 lies
within the bound of a decision (aux_ref.upsample_nll's `ambiguous`) are left unsupervised."""
import ctypes as C

import pytest
import torch

import magnet_b200
from magnet_b200 import _lib
from magnet_b200._lib import check, lib
from tests import head_ref as hr
from tests import mask_train_ref as mr
from tests.test_gpu_head_f64 import _close

pytestmark = pytest.mark.gpu


def _inputs(B, P, H, W, dev, seed, scale=1.0, gt_mask="half", clamp=False):
    torch.manual_seed(seed)
    mh = magnet_b200.MagnetHead(dnet_fdim=16).mask_head.to(dev)
    gen = torch.Generator(device=dev).manual_seed(seed)
    pre0 = scale * torch.randn(B, 128, H, W, device=dev, generator=gen)
    preds = [torch.cat([1 + torch.rand(B, 1, H, W, device=dev, generator=gen),
                        0.1 + 0.5 * torch.rand(B, 1, H, W, device=dev, generator=gen)], 1) for _ in range(P)]
    if clamp:
        preds[-1][:, 1] = 1e-6                                        # sigma^2 < 1e-10: var clamps, no sigma gradient
    gt = 1 + torch.rand(B, 1, 4 * H, 4 * W, device=dev, generator=gen)
    r = torch.rand(B, 1, 4 * H, 4 * W, device=dev, generator=gen)
    gtm = r < 0.5
    if gt_mask == "mixed":                                            # image 0 dense, 1 sparse, 2 empty
        gtm[0] = True
        gtm[1] = r[1] < 0.02
        gtm[2:] = False
    return mh, pre0, preds, gt, gtm


def _run(mh, pre0, preds, gt, gtm, gamma, g):
    """Pack, training forward and backward through the C ABI -> weights, dict of every output and intermediate."""
    L = lib()
    dev = pre0.device
    B, _, H, W = pre0.shape
    P = len(preds)
    ws = [t.detach().contiguous() for t in (mh[2].weight, mh[2].bias, mh[4].weight, mh[4].bias, mh[6].weight,
                                             mh[6].bias)]
    new = lambda *shape: torch.empty(*shape, device=dev, dtype=torch.float32)
    count = int(gtm.sum())
    packed = torch.empty(int(L.magnet_mask_train_weights_bytes(4)), device=dev, dtype=torch.uint8)
    partial = new(int(L.magnet_mask_train_partials(B, H, W)) * P)
    saved = new(int(L.magnet_mask_saved_bytes(P, B, H, W)) // 4)
    work = new(int(L.magnet_mask_bwd_workspace_bytes(B, H, W)) // 4)
    gs = torch.full((1,), g, device=dev, dtype=torch.float32)
    gtm8 = gtm.to(torch.uint8).contiguous()
    r = dict(grad_pre0=new(B, 128, H, W), dW1=new(128, 128, 1, 1), db1=new(128), dW2=new(128, 128, 1, 1),
             db2=new(128), dW3=new(144, 128, 1, 1), db3=new(144))
    r["grad_pred"] = [new(B, 2, H, W) for _ in preds]
    gammas = [gamma ** (P - i - 1) for i in range(P)]
    scale = (C.c_float * P)(*[gm / count for gm in gammas])
    pp = (C.c_void_p * P)(*[x.data_ptr() for x in preds])
    gp = (C.c_void_p * P)(*[x.data_ptr() for x in r["grad_pred"]])
    a = _lib.MaskTrainArgs(P=P, B=B, H=H, W=W, k=4, pre0=pre0.data_ptr(), packed_weights=packed.data_ptr(),
                           pred=C.cast(pp, C.POINTER(C.c_void_p)), gt=gt.data_ptr(), gt_mask=gtm8.data_ptr(),
                           pred_scale=C.cast(scale, C.POINTER(C.c_float)), save_maps=1, pred_grad=1,
                           partial=partial.data_ptr(), saved=saved.data_ptr(), grad_scale=gs.data_ptr(),
                           workspace=work.data_ptr(), grad_pre0=r["grad_pre0"].data_ptr(), grad_w1=r["dW1"].data_ptr(),
                           grad_b1=r["db1"].data_ptr(), grad_w2=r["dW2"].data_ptr(), grad_b2=r["db2"].data_ptr(),
                           grad_w3=r["dW3"].data_ptr(), grad_b3=r["db3"].data_ptr(),
                           grad_pred=C.cast(gp, C.POINTER(C.c_void_p)))
    st = torch.cuda.current_stream(dev).cuda_stream
    with torch.cuda.device(dev):
        check(L.magnet_mask_pack_train_weights_f32(*(t.data_ptr() for t in ws), packed.data_ptr(), st),
              "magnet_mask_pack_train_weights_f32")
        check(L.magnet_mask_train_fwd_f32(C.byref(a), st), "magnet_mask_train_fwd_f32")
        check(L.magnet_mask_bwd_f32(C.byref(a), st), "magnet_mask_bwd_f32")
    torch.cuda.synchronize(dev)
    pix = B * H * W
    plane = 128 * pix
    r["pred_unit"] = [saved[2 * i * pix:2 * (i + 1) * pix].view(B, 2, H, W) for i in range(P)]
    maps = saved[2 * P * pix:]                                        # h0, h1, h2, d_logits rows 0..127 and 128..143
    for i, n in enumerate(("h0", "h1", "h2")):
        r[n] = maps[i * plane:(i + 1) * plane].view(B, 128, H, W)
    r["d_logits"] = torch.cat([maps[3 * plane:4 * plane].view(B, 128, H, W),
                               maps[4 * plane:4 * plane + 16 * pix].view(B, 16, H, W)], 1)
    r["d_h2"] = work[:plane].view(B, 128, H, W)
    r["d_h1"] = work[plane:2 * plane].view(B, 128, H, W)
    terms = partial.view(-1, P).sum(0, dtype=torch.float64).to(torch.float32) / float(count)   # as ops.MaskLossTrain
    loss = 0.0
    for i in range(P):
        loss = loss + gammas[i] * terms[i]
    r["loss"] = loss
    return ws, r


def _check(mh, pre0, preds, gt, gtm, gamma=0.8, g=1.0):
    ws = [mh[i].weight if j == 0 else mh[i].bias for i in (2, 4, 6) for j in (0, 1)]
    f = mr.train_forward(pre0, ws, preds, gt, gtm, gamma)
    if f["ambiguous"].any():                                          # decisions within their own bound: unsupervised
        gtm = gtm & ~f["ambiguous"]
        f = mr.train_forward(pre0, ws, preds, gt, gtm, gamma)
    ws, k = _run(mh, pre0, preds, gt, gtm, gamma, g)
    w1, b1, w2, b2, w3, b3 = ws
    _close(k["h1"], f["h1"], f["h1_bound"], "h1")
    _close(k["h2"], f["h2"], f["h2_bound"], "h2")
    _close(k["loss"], f["loss"], f["loss_bound"], "loss")
    _close(k["d_logits"], f["grad_mask"], f["grad_mask_bound"], "d_logits")
    for i, (gp, bp) in enumerate(zip(f["grad_preds"], f["grad_preds_bound"])):
        _close(k["pred_unit"][i], gp, bp, f"grad_pred{i} (unit)")
        _close(k["grad_pred"][i], *mr.scaled(gp, bp, g), f"grad_pred{i}")
    _close(k["d_h2"], *mr.logit_grad_layer(w3, k["d_logits"], k["h2"]), "d_h2")
    _close(k["d_h1"], *hr.grad_layer(w2, k["d_h2"], k["h1"]), "d_h1")
    _close(k["grad_pre0"], *mr.scaled(*hr.grad_layer(w1, k["d_h1"], k["h0"]), g), "grad_pre0")
    for nm, a, x in (("1", k["d_h1"], k["h0"]), ("2", k["d_h2"], k["h1"]), ("3", k["d_logits"], k["h2"])):
        dw, bw, db, bb = mr.wgrad(a, x)
        _close(k["dW" + nm].view(dw.shape), *mr.scaled(dw, bw, g), "dW" + nm)
        _close(k["db" + nm], *mr.scaled(db, bb, g), "db" + nm)


CASES = ([dict(B=2, H=h, W=w, P=p) for h, w in ((1, 1), (1, 17), (8, 16), (13, 29)) for p in (1, 3, 8)]
         + [dict(B=8, H=120, W=160, P=3), dict(B=4, H=88, W=304, P=3)]
         + [dict(B=2, H=13, W=29, P=3, scale=s) for s in (1e-3, 1e3)]
         + [dict(B=3, H=13, W=29, P=3, gt_mask="mixed"), dict(B=2, H=8, W=16, P=3, clamp=True),
            dict(B=2, H=13, W=29, P=3, g=0.37), dict(B=2, H=13, W=29, P=8, scale=1e3, g=0.37)])


@pytest.mark.parametrize("case", CASES, ids=lambda c: "_".join(f"{k}{v}" for k, v in c.items()))
def test_training_loss_element_by_element(cuda, case):
    case = dict(case)
    g = case.pop("g", 1.0)
    B, H, W, P = (case.pop(n) for n in ("B", "H", "W", "P"))
    mh, pre0, preds, gt, gtm = _inputs(B, P, H, W, cuda, seed=B * 1000 + H * W + P, **case)
    _check(mh, pre0, preds, gt, gtm, g=g)
