"""The fixed-order (``_det``) backwards without a GPU (DESIGN §3.20): the entry points are exported and declared, refuse
bad arguments before any launch, size their workspaces by the stated formulas, and the Python wrappers pick them exactly
when torch.use_deterministic_algorithms is on, leaving the flag-off entry points as they were."""
import ctypes as C
import warnings

import pytest
import torch

from magnet_b200 import _lib, ops

DET = ("magnet_convex_upsample_bwd_det_f32", "magnet_upsample_nll_bwd_det_f32", "magnet_upsample_nll_bwd_dev_det_f32",
       "magnet_dnet_nll_bwd_det_f32", "magnet_dnet_nll_bwd_dev_det_f32", "magnet_mask_train_fwd_det_f32",
       "magnet_mask_train_fwd_dev_det_f32", "magnet_upsample_nll_bwd_det_workspace_bytes",
       "magnet_mask_train_det_workspace_bytes")


@pytest.fixture
def flag():
    """Set torch's deterministic flag for one test and restore both of its settings afterwards."""
    saved = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()

    def set_flag(on: bool, warn_only: bool = False):
        torch.use_deterministic_algorithms(on, warn_only=warn_only)
    yield set_flag
    torch.use_deterministic_algorithms(saved[0], warn_only=saved[1])


def test_entry_points_are_exported_with_the_flag_off_signatures_plus_a_workspace():
    L = _lib.lib()
    for name in DET:
        assert name in _lib.EXPORTS and hasattr(L, name), name
    S = _lib.SIGNATURES
    assert S["magnet_convex_upsample_bwd_det_f32"] == S["magnet_convex_upsample_bwd_f32"]
    assert S["magnet_mask_train_fwd_det_f32"] == S["magnet_mask_train_fwd_f32"]
    assert S["magnet_mask_train_fwd_dev_det_f32"] == S["magnet_mask_train_fwd_dev_f32"]
    for form in ("upsample", "dnet"):
        for dev in ("", "_dev"):
            res, args = S[f"magnet_{form}_nll_bwd{dev}_f32"]
            assert S[f"magnet_{form}_nll_bwd{dev}_det_f32"] == (res, args[:9] + [C.c_void_p] + args[9:])


def _buf():
    buf = (C.c_float * 64)()
    return buf, C.cast(buf, C.c_void_p).value


def test_upsampling_entry_points_validate_before_any_launch():
    L = _lib.lib()
    keep, a = _buf()
    launches = L.magnet_launch_count()
    shapes = (dict(B=0), dict(H=0), dict(W=-1), dict(k=0), dict(B=65536), dict(H=20000, k=4))

    def convex(ptrs, B=2, CH=2, H=3, W=4, k=4):
        return L.magnet_convex_upsample_bwd_det_f32(*ptrs[:3], B, CH, H, W, k, *ptrs[3:], None)
    full = [a] * 5
    for i in range(5):
        assert convex(full[:i] + [None] + full[i + 1:]) == _lib.ERR_NULL, i
    for shape in shapes:
        assert convex(full, **shape) == _lib.ERR_SHAPE, shape
    assert convex(full, CH=3) == _lib.ERR_UNSUPPORTED

    for name in ("magnet_upsample_nll_bwd_det_f32", "magnet_upsample_nll_bwd_dev_det_f32", "magnet_dnet_nll_bwd_det_f32",
                 "magnet_dnet_nll_bwd_dev_det_f32"):
        fn = getattr(L, name)
        on_device = "_dev_" in name

        def call(ptrs, B=2, H=3, W=4, k=4):
            scale = ptrs[4] if on_device else 0.5
            return fn(ptrs[0], ptrs[1], ptrs[2], ptrs[3], scale, B, H, W, k, ptrs[5], ptrs[6], ptrs[7], None)
        full = [a] * 8
        for i in range(8):
            if i == 4 and not on_device:
                continue
            assert call(full[:i] + [None] + full[i + 1:]) == _lib.ERR_NULL, (name, i)
        for shape in shapes:
            assert call(full, **shape) == _lib.ERR_SHAPE, (name, shape)
        assert call(full[:5] + [a + 2] + full[6:]) == _lib.ERR_ALIGN, name      # the workspace holds floats
    assert L.magnet_launch_count() == launches


def _mask_args(addr, pred_arr, P=2, B=2, H=8, W=16, workspace=True):
    a = _lib.MaskTrainArgs(P=P, B=B, H=H, W=W, k=4, pre0=addr, packed_weights=addr,
                           pred=C.cast(pred_arr, C.POINTER(C.c_void_p)), gt=addr, gt_mask=addr,
                           pred_scale=C.cast((C.c_float * 8)(), C.POINTER(C.c_float)), save_maps=0, pred_grad=1,
                           partial=addr, saved=addr, workspace=addr if workspace else None)
    return a


def test_mask_train_entry_points_validate_before_any_launch():
    L = _lib.lib()
    buf = (C.c_float * 64)()
    addr = (C.cast(buf, C.c_void_p).value + 15) // 16 * 16
    preds = (C.c_void_p * 8)(*([addr] * 8))
    launches = L.magnet_launch_count()
    for name in ("magnet_mask_train_fwd_det_f32", "magnet_mask_train_fwd_dev_det_f32"):
        def call(a):
            fn = getattr(L, name)
            return fn(C.byref(a), addr, None) if "_dev_" in name else fn(C.byref(a), None)
        assert call(_mask_args(addr, preds, workspace=False)) == _lib.ERR_NULL
        a = _mask_args(addr, preds)
        a.workspace = addr + 4
        assert call(a) == _lib.ERR_ALIGN
        assert call(_mask_args(addr, preds, P=8, B=8192)) == _lib.ERR_SHAPE          # P*B > 65535 grid rows
        assert call(_mask_args(addr, preds, P=9)) == _lib.ERR_UNSUPPORTED
        a = _mask_args(addr, preds)
        a.k = 2
        assert call(a) == _lib.ERR_UNSUPPORTED
        a = _mask_args(addr, preds)
        a.gt = None
        assert call(a) == _lib.ERR_NULL
    assert L.magnet_launch_count() == launches


def test_workspace_sizes():
    L = _lib.lib()
    for B, H, W, k in ((1, 1, 1, 1), (2, 30, 40, 4), (8, 120, 160, 4), (4, 88, 304, 4), (3, 7, 5, 8)):
        assert L.magnet_upsample_nll_bwd_det_workspace_bytes(B, H, W, k) == 4 * B * 2 * (k * H) * (k * W)
    for bad in ((0, 3, 4, 4), (2, 3, 4, 0), (65536, 1, 1, 1)):
        assert L.magnet_upsample_nll_bwd_det_workspace_bytes(*bad) == 0
    for P, B, H, W in ((1, 1, 1, 1), (3, 8, 120, 160), (8, 4, 88, 304)):
        # the 144 softmax weights per quarter-resolution pixel, then (d mu, d sigma) per full-resolution pixel and prediction
        assert L.magnet_mask_train_det_workspace_bytes(P, B, H, W) == 4 * (144 + 2 * 16 * P) * B * H * W
    for bad in ((0, 2, 3, 4), (9, 2, 3, 4), (2, 0, 3, 4), (8, 8192, 1, 1)):
        assert L.magnet_mask_train_det_workspace_bytes(*bad) == 0


def test_alert_follows_torch_flag(flag):
    flag(False)
    ops._alert_not_deterministic("x")                  # nothing with the flag off
    flag(True)
    with pytest.raises(RuntimeError, match="deterministic"):
        ops._alert_not_deterministic("magnet_cost_volume_bwd_f32 (grad_src)")
    flag(True, warn_only=True)
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        ops._alert_not_deterministic("magnet_cost_volume_f_bwd_f32 (grad_src)")
    assert len(w) == 1 and "magnet_cost_volume_f_bwd_f32" in str(w[0].message)


@pytest.fixture
def recorded(monkeypatch):
    """The wrappers on CPU tensors: the device checks pass them through and each launch is recorded by name instead of
    run, so that the choice of entry point is observable without a GPU."""
    names = []
    monkeypatch.setattr(ops, "_need_cuda", lambda name, x: x)
    monkeypatch.setattr(ops, "_need_cuda_u8_mask", lambda name, m, shape, text: m.contiguous())
    monkeypatch.setattr(ops, "_launch", lambda dev, name, *args: names.append(name))
    return names


def _wrapper_calls():
    B, H, W, k = 2, 3, 4, 4
    depth, up = torch.rand(B, 2, H, W), torch.rand(B, 9 * k * k, H, W)
    gt, gtm = torch.rand(B, 1, k * H, k * W), torch.ones(B, 1, k * H, k * W, dtype=torch.uint8)
    ops.convex_upsample_bwd(torch.rand(B, 2, k * H, k * W), depth, up, k)
    for dnet in (False, True):
        ops.upsample_nll_bwd(depth, up, gt, gtm, k, 0.25, dnet)
        ops.upsample_nll_bwd(depth, up, gt, gtm, k, torch.tensor([0.25]), dnet)
    pre0 = torch.rand(B, 128, H, W)
    ws = [torch.rand(s) for _, s in ops.mask_weight_shapes()]
    for pred_grad in (False, True):
        for scales in ([0.5, 0.25], torch.tensor([0.5, 0.25])):
            ops.mask_train_fwd(pre0, ws, [depth, depth], gt, gtm, False, pred_grad, scales)


def test_wrappers_pick_det_entry_points_exactly_under_the_flag(flag, recorded):
    flag(False)
    _wrapper_calls()
    off = list(recorded)
    recorded.clear()
    flag(True)
    _wrapper_calls()
    on = list(recorded)
    pack = "magnet_mask_pack_train_weights_f32"
    assert off == ["magnet_convex_upsample_bwd_f32",
                   "magnet_upsample_nll_bwd_f32", "magnet_upsample_nll_bwd_dev_f32",
                   "magnet_dnet_nll_bwd_f32", "magnet_dnet_nll_bwd_dev_f32",
                   pack, "magnet_mask_train_fwd_f32", pack, "magnet_mask_train_fwd_dev_f32",
                   pack, "magnet_mask_train_fwd_f32", pack, "magnet_mask_train_fwd_dev_f32"]
    # without pred_grad the mask-loss forward has no scatter: the flag-off entry points run either way
    assert on == ["magnet_convex_upsample_bwd_det_f32",
                  "magnet_upsample_nll_bwd_det_f32", "magnet_upsample_nll_bwd_dev_det_f32",
                  "magnet_dnet_nll_bwd_det_f32", "magnet_dnet_nll_bwd_dev_det_f32",
                  pack, "magnet_mask_train_fwd_f32", pack, "magnet_mask_train_fwd_dev_f32",
                  pack, "magnet_mask_train_fwd_det_f32", pack, "magnet_mask_train_fwd_dev_det_f32"]
