"""The torch.library registration of the training entry points, without a GPU: every training op is registered, each
forward op has an autograd registration tying it to its backward op, no op writes into an argument, and each fake
implementation gives the shapes, dtypes and byte sizes the eager functions return, at several shape sets and for 1 to 8
predictions.  Fake CUDA tensors need no driver; the byte counts come from the library's host size functions.  The
fake-against-real comparison (``torch.library.opcheck``) runs on the GPU (tests/test_gpu_compile_train.py)."""
import pytest
import torch
from torch._subclasses.fake_tensor import FakeTensorMode

from magnet_b200 import MagnetHead, _lib, library, ops

OPS = torch.ops.magnet_b200

# forward op -> the backward op its autograd registration calls
AUTOGRAD = {"gaussian_update": "gaussian_update_bwd", "convex_upsample": "convex_upsample_bwd",
            "gnet_train_fwd": "gnet_bwd", "mask_train_fwd": "mask_bwd", "upsample_nll_fwd": "upsample_nll_bwd",
            "fnet_l1_fwd": "fnet_l1_bwd", "cost_volume_f": "cost_volume_f_bwd"}


def test_every_training_op_is_registered():
    assert not set(library.TRAIN_OPS) & set(library.OPS)
    for name in library.TRAIN_OPS:
        assert hasattr(OPS, name), name
        assert OPS.__getattr__(name).default._schema.name == f"magnet_b200::{name}"
    assert set(AUTOGRAD.values()) | (set(AUTOGRAD) - set(library.OPS)) == set(library.TRAIN_OPS)


def test_forward_ops_have_autograd_registrations():
    for fwd, bwd in AUTOGRAD.items():
        op = getattr(library, fwd)
        assert op._backward_fn is not None and op._setup_context_fn is not None, fwd
        assert getattr(library, bwd)._backward_fn is None, bwd       # the backward ops are not differentiated again


def test_no_training_op_mutates():
    for name in library.TRAIN_OPS:
        schema = OPS.__getattr__(name).default._schema
        written = [a.name for a in schema.arguments if a.alias_info is not None and a.alias_info.is_write]
        assert written == [], (name, str(schema))
        assert all(r.alias_info is None for r in schema.returns), str(schema)


def test_flags_and_counts_are_op_arguments():
    schema = str(OPS.mask_train_fwd.default._schema)
    for arg in ("Tensor count", "Tensor[] preds", "float gamma", "bool save_maps", "bool pred_grad"):
        assert arg in schema, (arg, schema)
    assert "bool[] need" in str(OPS.gnet_bwd.default._schema)
    assert "Tensor count" in str(OPS.upsample_nll_fwd.default._schema)
    assert "float[] planes" in str(OPS.fnet_l1_fwd.default._schema)
    assert "Tensor? ref_split" in str(OPS.cost_volume_f.default._schema)


def _cuda(*shape, dtype=torch.float32):
    return torch.empty(shape, device="cuda", dtype=dtype)


def _mask_w():
    return [_cuda(*s) for _, s in ops.mask_weight_shapes()]


def _gnet_w(D):
    return [_cuda(*s) for _, s in ops.gnet_weight_shapes(D)]


# (op, argument builder, expected (shape, dtype) of each output)
def _cases(B, V, H, W, D, P):
    f32, u8 = torch.float32, torch.uint8
    L = _lib.lib()
    hid = _lib.MAGNET_HIDDEN_CHANNELS
    planes = [0.5 + 0.1 * i for i in range(D)]
    count = lambda: _cuda(dtype=torch.int64)
    full = (B, 1, 4 * H, 4 * W)
    split = ops.packed_bytes(_lib.SRC_SPLIT16, V * B, H, W)
    rsplit = ops.packed_bytes(_lib.SRC_SPLIT16, B, H, W)
    gsaved = int(L.magnet_gnet_saved_bytes(B, H, W)) // 4
    gnet_grads = lambda need: [((B, hid, H, W), f32)] + [(s if n else (0,), f32) for (_, s), n in
                                                         zip(ops.gnet_weight_shapes(D), need[:7])] \
        + [((B, 2, H, W) if need[7] else (0,), f32)]
    mask_grads = lambda need, pg: [((B, hid, H, W) if need[0] else (0,), f32)] \
        + [(s if n else (0,), f32) for (_, s), n in zip(ops.mask_weight_shapes(), need[1:])] \
        + [((B, 2, H, W) if pg else (0,), f32)] * P
    all8, some = [True] * 8, [False, True, False, True, True, False, True, False]
    return [
        ("gaussian_update_bwd", lambda: (_cuda(B, 2, H, W), _cuda(B, 2, H, W), _cuda(B, 2, H, W)), [((B, 2, H, W), f32)]),
        ("convex_upsample_bwd", lambda: (_cuda(B, 2, 4 * H, 4 * W), _cuda(B, 2, H, W), _cuda(B, 144, H, W), 4),
         [((B, 2, H, W), f32), ((B, 144, H, W), f32)]),
        ("gnet_train_fwd", lambda: (_cuda(B, D, H, W), _cuda(B, hid, H, W), *_gnet_w(D), _cuda(B, 2, H, W)),
         [((B, 2, H, W), f32), ((int(L.magnet_gnet_train_weights_bytes(D)),), u8), ((gsaved,), f32)]),
        ("gnet_bwd", lambda: (_cuda(B, 2, H, W), _cuda(B, D, H, W), _cuda(B, 2, H, W),
                              _cuda(int(L.magnet_gnet_train_weights_bytes(D)), dtype=u8), _cuda(gsaved), all8),
         gnet_grads(all8)),
        ("gnet_bwd", lambda: (_cuda(B, 2, H, W), _cuda(B, D, H, W), _cuda(B, 2, H, W),
                              _cuda(int(L.magnet_gnet_train_weights_bytes(D)), dtype=u8), _cuda(gsaved), some),
         gnet_grads(some)),
        ("mask_train_fwd", lambda: (_cuda(B, hid, H, W), *_mask_w(), _cuda(*full), _cuda(*full, dtype=u8), count(),
                                    [_cuda(B, 2, H, W) for _ in range(P)], 0.8, True, True),
         [((), f32), ((int(L.magnet_mask_train_weights_bytes(4)),), u8),
          ((int(L.magnet_mask_saved_bytes(P, B, H, W)) // 4,), f32)]),
        ("mask_train_fwd", lambda: (_cuda(B, hid, H, W), *_mask_w(), _cuda(*full), _cuda(*full, dtype=u8), count(),
                                    [_cuda(B, 2, H, W) for _ in range(P)], 0.8, False, True),
         [((), f32), ((int(L.magnet_mask_train_weights_bytes(4)),), u8), ((2 * P * B * H * W,), f32)]),
        ("mask_bwd", lambda: (_cuda(), _cuda(int(L.magnet_mask_train_weights_bytes(4)), dtype=u8),
                              _cuda(int(L.magnet_mask_saved_bytes(P, B, H, W)) // 4), P, B, H, W, all8[:7], True),
         mask_grads(all8[:7], True)),
        ("mask_bwd", lambda: (_cuda(), _cuda(int(L.magnet_mask_train_weights_bytes(4)), dtype=u8),
                              _cuda(2 * P * B * H * W), P, B, H, W, [False] * 7, True), mask_grads([False] * 7, True)),
        ("mask_bwd", lambda: (_cuda(), _cuda(int(L.magnet_mask_train_weights_bytes(4)), dtype=u8),
                              _cuda(int(L.magnet_mask_saved_bytes(P, B, H, W)) // 4), P, B, H, W, some[:7], False),
         mask_grads(some[:7], False)),
        ("upsample_nll_fwd", lambda: (_cuda(B, 2, H, W), _cuda(B, 144, H, W), _cuda(*full), _cuda(*full, dtype=u8), 4,
                                      count(), 0.64), [((), f32)]),
        ("upsample_nll_bwd", lambda: (_cuda(), _cuda(B, 2, H, W), _cuda(B, 144, H, W), _cuda(*full),
                                      _cuda(*full, dtype=u8), 4, count(), 0.64),
         [((B, 2, H, W), f32), ((B, 144, H, W), f32)]),
        ("fnet_l1_fwd", lambda: (_cuda(B, D, H, W), planes, _cuda(B, 1, H, W), _cuda(B, 1, H, W, dtype=u8), count()),
         [((), f32)]),
        ("fnet_l1_bwd", lambda: (_cuda(), _cuda(B, D, H, W), planes, _cuda(B, 1, H, W), _cuda(B, 1, H, W, dtype=u8),
                                 count()), [((B, D, H, W), f32)]),
        ("cost_volume_f", lambda: (_cuda(B, 64, H, W), _cuda(V * B, 64, H, W), _cuda(split, dtype=u8),
                                   _cuda(rsplit, dtype=u8), _cuda(B, 3, H * W), _cuda(B * V, 16), V, _lib.SRC_SPLIT16,
                                   _lib.VARIANT_AUTO, planes, False, True), [((B, D, H, W), f32)]),
        ("cost_volume_f", lambda: (_cuda(B, 32, H, W), _cuda(V * B, 32, H, W), _cuda(V * B, H, W, 36), None,
                                   _cuda(B, 3, H * W), _cuda(B * V, 16), V, _lib.SRC_PIXC, _lib.VARIANT_AUTO, planes,
                                   True, True), [((B, D, H, W), f32)]),
        ("cost_volume_f_bwd", lambda: (_cuda(B, D, H, W), _cuda(B, 64, H, W, dtype=torch.float16),
                                       _cuda(V * B, 64, H, W, dtype=torch.float16), _cuda(B, 3, H * W),
                                       _cuda(B * V, 16), V, planes, None, False,
                                       _cuda(ops.packed_bytes(_lib.SRC_HALF16, B, H, W), dtype=u8),
                                       _cuda(ops.packed_bytes(_lib.SRC_HALF16, V * B, H, W), dtype=u8),
                                       _lib.SRC_HALF16),
         [((B, 64, H, W), torch.float16), ((V * B, 64, H, W), torch.float16)]),
        ("cost_volume_f_bwd", lambda: (_cuda(B, D, H, W), _cuda(B, 32, H, W), _cuda(V * B, 32, H, W),
                                       _cuda(B, 3, H * W), _cuda(B * V, 16), V, planes, _cuda(B, D, H, W), True, None,
                                       None, _lib.SRC_NCHW), [((B, 32, H, W), f32), ((V * B, 32, H, W), f32)]),
    ]


# (B, V, H, W, D, P): the training drivers' shapes (ScanNet 120x160 and KITTI 88x304 at batch 4, F-Net's 80 planes),
# a small one and the largest hypothesis count
_SHAPES = [(4, 4, 120, 160, 5, 3), (4, 2, 88, 304, 5, 3), (2, 4, 120, 160, 80, 1), (1, 2, 30, 40, 64, 8),
           (3, 3, 24, 40, 256, 2), (1, 4, 30, 40, 16, 5)]


@pytest.mark.parametrize("B,V,H,W,D,P", _SHAPES)
def test_fake_outputs_match_the_eager_contract(B, V, H, W, D, P):
    seen = set()
    with FakeTensorMode():
        for name, args, want in _cases(B, V, H, W, D, P):
            seen.add(name)
            out = getattr(OPS, name)(*args())
            outs = list(out) if isinstance(out, (list, tuple)) else [out]
            assert [(tuple(o.shape), o.dtype) for o in outs] == [(tuple(s), d) for s, d in want], name
            assert all(o.device.type == "cuda" for o in outs), name
    assert seen == set(library.TRAIN_OPS) - {"gaussian_update", "convex_upsample"}


@pytest.mark.parametrize("P", range(1, _lib.MAGNET_MASK_MAX_PRED + 1))
def test_mask_loss_fakes_for_every_prediction_count(P):
    B, H, W = 2, 30, 40
    with FakeTensorMode():
        preds = [_cuda(B, 2, H, W) for _ in range(P)]
        loss, packed, saved = OPS.mask_train_fwd(_cuda(B, 128, H, W), *_mask_w(), _cuda(B, 1, 4 * H, 4 * W),
                                                 _cuda(B, 1, 4 * H, 4 * W, dtype=torch.uint8),
                                                 _cuda(dtype=torch.int64), preds, 0.8, True, True)
        assert saved.numel() * 4 == _lib.lib().magnet_mask_saved_bytes(P, B, H, W)
        grads = OPS.mask_bwd(loss, packed, saved, P, B, H, W, [True] * 7, True)
        assert [tuple(g.shape) for g in grads[7:]] == [(B, 2, H, W)] * P


def test_eager_losses_count_on_the_host_and_traced_ones_on_the_device(monkeypatch):
    """Outside tracing the losses read the count on the host and refuse an empty mask before any launch; the traced
    forms keep it on the device (the op path), so an explicit host count is refused there for the F-Net loss."""
    assert not ops._traced()
    with pytest.raises(_lib.MagnetError, match="no pixel"):
        ops.fnet_l1_loss(torch.empty(1, 2, 3, 4), [1.0, 2.0], torch.empty(1, 1, 3, 4), torch.zeros(1, 1, 3, 4))
    with pytest.raises(_lib.MagnetError, match="no pixel"):
        ops.magnet_loss([torch.empty(1, 2, 3, 4)], torch.empty(1, 144, 3, 4), torch.empty(1, 1, 12, 16),
                        torch.zeros(1, 1, 12, 16, dtype=torch.bool), 4)
    with pytest.raises(_lib.MagnetError, match="no pixel"):
        ops.mask_head_loss(torch.empty(1, 128, 3, 4), MagnetHead().mask_head, [torch.empty(1, 2, 3, 4)],
                           torch.empty(1, 1, 12, 16), torch.zeros(1, 1, 12, 16, dtype=torch.bool))
    monkeypatch.setattr(torch.compiler, "is_compiling", lambda: True)
    with pytest.raises(_lib.MagnetError, match="count=None"):
        ops.fnet_l1_loss(torch.empty(1, 2, 3, 4), [1.0, 2.0], torch.empty(1, 1, 3, 4), torch.ones(1, 1, 3, 4), count=5)


def test_device_scales_round_like_the_host():
    """The device scale is the host's float(g / float(count)): a float64 quotient rounded once to fp32; 0 for count 0."""
    gammas = [0.8 ** (7 - i) for i in range(8)]
    for count in (1, 3, 7, 12345, 4 * 480 * 640):
        got = ops.device_scales(torch.tensor(gammas, dtype=torch.float64), torch.tensor(count))
        want = torch.tensor([g / float(count) for g in gammas], dtype=torch.float32)
        assert torch.equal(got, want), count
    zero = ops.device_scales(torch.tensor(gammas, dtype=torch.float64), torch.tensor(0))
    assert torch.equal(zero, torch.zeros(8)) and not zero.isinf().any()
