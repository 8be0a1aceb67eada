"""CPU tests of the D-Net heads (DESIGN §3.15): structure detection, the fused-path rule, the pack size and argument
validation of the C ABI, and the numpy restatement of the variance form of the depth metrics against the reference's
test_DNet.validate golden."""
import ctypes as C
import os

import numpy as np
import pytest
import torch
import torch.nn as nn

from magnet_b200 import DnetHead, _lib, ops
from magnet_b200.matcher import fused_dnet_applies
from tests.depth_metrics_ref import KEYS, inputs_digest
from tests.dnet_ref import METRIC_CASES, metric_inputs, metric_rows_var

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "dnet_metrics.npz")


def _chain(cin, cout, bias=True, k0=3, extra=False):
    layers = [nn.Conv2d(cin, 128, k0, padding=k0 // 2, bias=bias), nn.ReLU(inplace=True),
              nn.Conv2d(128, 128, 1, bias=bias), nn.ReLU(inplace=True)]
    if extra:
        layers += [nn.Conv2d(128, 128, 1), nn.ReLU(inplace=True)]
    return nn.Sequential(*layers, nn.Conv2d(128, cout, 1, bias=bias))


def test_structure_detection_accepts_the_reference_heads():
    head = DnetHead()
    d, m = ops.dnet_head_layers(head.depth_head, head.mask_head)
    assert d[0] is head.depth_head[0] and m[2] is head.mask_head[4]
    assert ops.dnet_head_layers(head.depth_head) == (d, None)
    assert ops.dnet_head_layers(_chain(64, 2), _chain(64, 144)) is not None


@pytest.mark.parametrize("depth, mask", [
    (_chain(256, 2, bias=False), None),                    # no bias
    (_chain(256, 2), _chain(256, 144, bias=False)),
    (_chain(256, 2), _chain(256, 9 * 8 * 8)),              # k = 8
    (_chain(256, 2), _chain(256, 9 * 2 * 2)),              # k = 2
    (_chain(256, 2, extra=True), None),                    # an extra layer (MaGNet's mask-head depth)
    (_chain(256, 2), _chain(256, 144, extra=True)),
    (_chain(256, 1), None),                                # output_dim 1
    (_chain(256, 2, k0=1), None),                          # 1x1 first layer
    (nn.Sequential(*list(_chain(256, 2))[:4]), None),      # a layer short
])
def test_structure_detection_rejects_variants(depth, mask):
    assert ops.dnet_head_layers(depth, mask) is None
    with pytest.raises(_lib.MagnetError):
        ops.pack_dnet_weights(depth, mask)


def test_mask_head_missing_when_dnet_true_is_not_the_fused_structure():
    head = DnetHead()
    x = torch.zeros(1, 256, 4, 4)
    with torch.no_grad():
        assert fused_dnet_applies(head.depth_head, head.mask_head, x, 4)
        assert not fused_dnet_applies(head.depth_head, nn.Identity(), x, 4)
        assert not fused_dnet_applies(head.depth_head, head.mask_head, x, 8)
        assert fused_dnet_applies(head.depth_head, None, x, 8)       # dnet=False: no mask head, k does not matter


def test_rule_under_grad_autocast_and_dtype():
    head = DnetHead()
    x = torch.zeros(1, 256, 4, 4)
    assert not fused_dnet_applies(head.depth_head, head.mask_head, x, 4)          # parameters require grad
    with torch.no_grad():
        assert fused_dnet_applies(head.depth_head, head.mask_head, x, 4)
        assert not fused_dnet_applies(head.depth_head, head.mask_head, x.double(), 4)
        assert not fused_dnet_applies(head.depth_head.half(), None, x, 4)
    head = DnetHead().requires_grad_(False)
    assert fused_dnet_applies(head.depth_head, head.mask_head, x, 4)
    assert not fused_dnet_applies(head.depth_head, head.mask_head, x.requires_grad_(), 4)
    # CUDA autocast (which needs a device to be enabled) is covered in tests/test_gpu_dnet_head.py


def test_reference_checkpoint_names_load_strictly():
    head = DnetHead(dnet=False)
    sd = {f"d_net.decoder.{k}": v for k, v in DnetHead().state_dict().items()}
    head.load_state_dict({k[len("d_net.decoder."):]: v for k, v in sd.items()}, strict=True)
    assert sorted(head.state_dict()) == sorted(f"{h}.{i}.{p}" for h in ("depth_head", "mask_head") for i in (0, 2, 4)
                                                for p in ("weight", "bias"))


def test_pack_size_formula_and_abi_validation():
    L = _lib.lib()
    depth = 4096 + 128 * 128 * 4                           # header + vectors, W1 as hi/lo fp16 fragments
    mask = 4096 + 128 * 128 * 4 + 144 * 128 * 4            # header + vectors, W1 and W3
    assert ops.dnet_weights_bytes(0) == depth and ops.dnet_weights_bytes(4) == depth + mask
    for k in (-1, 1, 2, 8):
        assert ops.dnet_weights_bytes(k) == 0
    p = C.c_void_p(256)
    assert L.magnet_dnet_pack_weights_f32(p, p, p, p, None, None, None, None, 8, p, None) == _lib.ERR_UNSUPPORTED
    assert L.magnet_dnet_pack_weights_f32(None, p, p, p, None, None, None, None, 0, p, None) == _lib.ERR_NULL
    assert L.magnet_dnet_pack_weights_f32(p, p, p, p, None, p, p, p, 4, p, None) == _lib.ERR_NULL
    assert L.magnet_dnet_pack_weights_f32(p, p, p, p, None, None, None, None, 0, C.c_void_p(258), None) == _lib.ERR_ALIGN
    assert L.magnet_dnet_depth_f32(p, p, 0, 4, 4, 1, p, None) == _lib.ERR_SHAPE
    assert L.magnet_dnet_depth_f32(p, p, 1 << 16, 1 << 8, 1 << 8, 1, p, None) == _lib.ERR_SHAPE
    assert L.magnet_dnet_depth_f32(None, p, 1, 4, 4, 1, p, None) == _lib.ERR_NULL
    assert L.magnet_dnet_depth_f32(p, p, 1, 4, 4, 1, C.c_void_p(260), None) == _lib.ERR_ALIGN
    assert L.magnet_dnet_upsample_f32(p, p, p, 1, 4, 4, 8, p, None) == _lib.ERR_UNSUPPORTED
    assert L.magnet_dnet_upsample_f32(p, p, None, 1, 4, 4, 4, p, None) == _lib.ERR_NULL
    assert L.magnet_dnet_upsample_f32(p, p, p, 1, -4, 4, 4, p, None) == _lib.ERR_SHAPE
    a = _lib.DepthMetricsArgs(P=1, B=1, H=8, W=8, k=4, row0=0, row1=8, col0=0, col1=8, min_depth=1e-3, max_depth=10.0)
    assert L.magnet_depth_metrics_var_f32(C.byref(a), None) == _lib.ERR_UNSUPPORTED
    a.k = 0
    assert L.magnet_depth_metrics_var_f32(C.byref(a), None) == _lib.ERR_NULL
    assert L.magnet_depth_metrics_var_f32(None, None) == _lib.ERR_NULL


def test_python_wrappers_refuse_bad_arguments_before_any_launch():
    cpu = torch.zeros(1, 128, 4, 4)
    with pytest.raises(_lib.MagnetError):
        ops.dnet_upsample(cpu, torch.zeros(8, dtype=torch.uint8), cpu, k=8)
    with pytest.raises(_lib.MagnetError):
        ops.dnet_depth(cpu, torch.zeros(8, dtype=torch.uint8), sigma=True)           # no CPU path
    g = torch.zeros(1, 1, 8, 8)
    for kw in (dict(nearest=True), dict(up_mask=torch.zeros(1, 144, 2, 2), k=4)):
        with pytest.raises(_lib.MagnetError):
            ops.depth_metrics(torch.zeros(1, 2, 8, 8), g, min_depth=1e-3, max_depth=10.0, variance=True, **kw)


@pytest.mark.parametrize("name", list(METRIC_CASES))
def test_variance_restatement_matches_the_validate_golden(name):
    gold = np.load(GOLDEN)
    inp = metric_inputs(name)
    assert str(gold[f"{name}_digest"]) == inputs_digest(inp)
    kw = METRIC_CASES[name]
    rows = metric_rows_var(inp["pred"], inp["gt"], kw["min_depth"], kw["max_depth"], kw["crop"])
    np.testing.assert_array_equal(rows[:, 0], gold[f"{name}_n"])
    np.testing.assert_allclose(rows[:, 1:], gold[f"{name}_rows"], rtol=2e-5, atol=0, equal_nan=True)
    assert list(gold["keys"]) == list(KEYS)
