"""The torch.library registration of the inference entry points, without a GPU: every op is registered with the schema
its eager function implies, only ``depth_metrics_update`` writes into an argument, and each fake implementation gives
the shapes and dtypes the eager function returns.  Fake CUDA tensors need no driver; the byte counts of the packed
buffers come from the library's host functions.  The fake-against-real comparison (``torch.library.opcheck``) runs on
the GPU (tests/test_gpu_compile.py)."""
import pytest
import torch
from torch._subclasses.fake_tensor import FakeTensorMode

from magnet_b200 import _lib, library, ops

OPS = torch.ops.magnet_b200


def test_every_op_is_registered():
    for name in library.OPS:
        assert hasattr(OPS, name), name
        assert OPS.__getattr__(name).default._schema.name == f"magnet_b200::{name}"


def test_only_the_metrics_update_mutates():
    for name in library.OPS:
        schema = OPS.__getattr__(name).default._schema
        written = [a.name for a in schema.arguments if a.alias_info is not None and a.alias_info.is_write]
        assert written == (["acc"] if name == "depth_metrics_update" else []), (name, str(schema))
        assert all(r.alias_info is None for r in schema.returns), str(schema)


def test_scalar_arguments_are_op_arguments():
    schema = str(OPS.cost_volume.default._schema)
    for arg in ("SymInt V", "SymInt src_layout", "bool consistency", "float kappa", "float[]? k", "bool planes",
                "bool softmax", "SymInt variant"):
        assert arg in schema, (arg, schema)
    assert "float[] k" in str(OPS.sample_depths.default._schema)
    assert "str? crop" in str(OPS.depth_metrics.default._schema)


def _cuda(*shape, dtype=torch.float32):
    return torch.empty(shape, device="cuda", dtype=dtype)


# (op, argument builder, expected (shape, dtype) of each output); the shapes of the host tests' cases
def _cases(B, V, C, H, W, D):
    k = [0.1 * i for i in range(D)]
    split = ops.packed_bytes(_lib.SRC_SPLIT16, V * B, H, W)
    half = ops.packed_bytes(_lib.SRC_HALF16, V * B, H, W)
    f32, u8 = torch.float32, torch.uint8
    gnet_w = lambda: [_cuda(128, D, 3, 3), _cuda(128, 128, 1, 1), _cuda(128), _cuda(128, 128, 1, 1), _cuda(128),
                      _cuda(2, 128, 1, 1), _cuda(2)]
    mask_w = lambda: [_cuda(128, 128, 1, 1), _cuda(128), _cuda(128, 128, 1, 1), _cuda(128), _cuda(144, 128, 1, 1),
                      _cuda(144)]
    dnet_w = lambda n: [_cuda(128, 128, 1, 1), _cuda(128), _cuda(2, 128, 1, 1), _cuda(2), _cuda(128, 128, 1, 1),
                        _cuda(128), _cuda(144, 128, 1, 1), _cuda(144)][:n]
    cv_common = lambda layout, src: (_cuda(B, C, H, W), src, _cuda(B, 3, H * W), _cuda(B * V, 16), V, layout)
    return [
        ("pack_cameras", lambda: (_cuda(B, 3, 3), _cuda(B, V, 3, 3), _cuda(B, V, 3), _cuda(B, V, dtype=torch.int32)),
         [((B * V, 16), f32)]),
        ("relative_poses", lambda: (_cuda(B, 4, 4), _cuda(V, B, 4, 4)), [((B, V, 4, 4), f32), ((B, V), torch.int32)]),
        ("camera_rays", lambda: (_cuda(B, 8, dtype=torch.float64), H, W), [((B, 3, 3), f32), ((B, 3, H * W), f32)]),
        ("sample_depths", lambda: (_cuda(B, 2, H, W), k), [((B, D, H, W), f32)]),
        ("repack_tiled32", lambda: (_cuda(V * B, C, H, W),), [((V * B, H, (W + 31) // 32, C // 4, 32, 4), f32)]),
        ("repack_pixc", lambda: (_cuda(V * B, C, H, W), _cuda(V * B, 2, H, W)), [((V * B, H, W, C + 4), f32)]),
        ("repack_split16", lambda: (_cuda(V * B, 64, H, W), None), [((split,), u8)]),
        ("repack_half16", lambda: (_cuda(V * B, 64, H, W, dtype=torch.float16), _cuda(V * B, 2, H, W)), [((half,), u8)]),
        ("cost_volume", lambda: (*cv_common(_lib.SRC_TILED32, _cuda(V * B, H, (W + 31) // 32, C // 4, 32, 4)), True,
                                 _cuda(V * B, 2, H, W), 5.0, None, _cuda(B, 2, H, W), k, False, False,
                                 _lib.VARIANT_AUTO, None), [((B, D, H, W), f32)]),
        ("cost_volume", lambda: (*cv_common(_lib.SRC_NCHW, _cuda(V * B, C, H, W)), True, _cuda(V * B, 2, H, W), 5.0,
                                 _cuda(B, D + 3, H, W), None, None, False, False, _lib.VARIANT_AUTO, None),
         [((B, D + 3, H, W), f32)]),
        ("cost_volume", lambda: (*cv_common(_lib.SRC_SPLIT16, _cuda(split, dtype=u8)), False, None, 0.0, None, None, k,
                                 True, True, _lib.VARIANT_AUTO, _cuda(ops.packed_bytes(_lib.SRC_SPLIT16, B, H, W), dtype=u8)),
         [((B, D, H, W), f32)]),
        ("gaussian_update", lambda: (_cuda(B, 2, H, W), _cuda(B, 2, H, W)), [((B, 2, H, W), f32)]),
        ("pack_gnet_weights", lambda: (gnet_w(), D), [((ops.gnet_weights_bytes(D),), u8)]),
        ("gnet_update", lambda: (_cuda(B, D, H, W), _cuda(B, 128, H, W), _cuda(ops.gnet_weights_bytes(D), dtype=u8),
                                 _cuda(B, 2, H, W)), [((B, 2, H, W), f32)]),
        ("convex_upsample", lambda: (_cuda(B, 2, H, W), _cuda(B, 144, H, W), 4), [((B, 2, 4 * H, 4 * W), f32)]),
        ("pack_mask_weights", lambda: (mask_w(),), [((ops.mask_weights_bytes(4),), u8)]),
        ("mask_upsample", lambda: (_cuda(B, 128, H, W), _cuda(ops.mask_weights_bytes(4), dtype=u8),
                                   [_cuda(B, 2, H, W) for _ in range(3)], 4), [((B, 2, 4 * H, 4 * W), f32)] * 3),
        ("pack_dnet_weights", lambda: (dnet_w(4), 0), [((ops.dnet_weights_bytes(0),), u8)]),
        ("pack_dnet_weights", lambda: (dnet_w(8), 4), [((ops.dnet_weights_bytes(4),), u8)]),
        ("dnet_depth", lambda: (_cuda(B, 128, H, W), _cuda(ops.dnet_weights_bytes(0), dtype=u8), True),
         [((B, 2, H, W), f32)]),
        ("dnet_upsample", lambda: (_cuda(B, 128, H, W), _cuda(ops.dnet_weights_bytes(4), dtype=u8), _cuda(B, 2, H, W), 4),
         [((B, 2, 4 * H, 4 * W), f32)]),
        ("plane_depth", lambda: (_cuda(B, D, H, W), k, True), [((B, 1, H, W), f32)]),
        ("depth_metrics", lambda: ([_cuda(B, 2, 4 * H, 4 * W)] * 2, _cuda(B, 1, 4 * H, 4 * W), 1e-3, 10.0, None, None,
                                   None, False, False), [((2, B, _lib.MAGNET_METRICS_COLS), torch.float64)]),
        ("depth_metrics", lambda: ([_cuda(B, 1, H, W)], _cuda(B, 1, 4 * H, 4 * W), 1e-3, 80.0, "garg", None, None,
                                   True, False), [((1, B, _lib.MAGNET_METRICS_COLS), torch.float64)]),
        ("depth_metrics_update", lambda: (_cuda(3, 14, dtype=torch.float64), [_cuda(B, 2, H, W)] * 3,
                                          _cuda(B, 1, 4 * H, 4 * W), 1e-3, 10.0, None, _cuda(B, 144, H, W), 4, False,
                                          False), [((3, B, _lib.MAGNET_METRICS_COLS), torch.float64)]),
    ]


_SHAPES = [(1, 4, 64, 30, 40, 5), (2, 3, 64, 24, 40, 64), (8, 4, 64, 120, 160, 64), (1, 2, 32, 22, 76, 16)]


@pytest.mark.parametrize("B,V,C,H,W,D", _SHAPES)
def test_fake_outputs_match_the_eager_contract(B, V, C, H, W, D):
    seen = set()
    with FakeTensorMode():
        for name, args, want in _cases(B, V, C, H, W, D):
            seen.add(name)
            out = getattr(OPS, name)(*args())
            outs = list(out) if isinstance(out, (list, tuple)) else [out]
            assert [(tuple(o.shape), o.dtype) for o in outs] == [(tuple(s), d) for s, d in want], name
            assert all(o.device.type == "cuda" for o in outs), name
    assert seen == set(library.OPS)


def test_eager_calls_do_not_go_through_the_dispatcher(monkeypatch):
    """Outside tracing the wrappers call the C entry points directly; the ops are only reached while torch.compile
    traces (DESIGN §3.18)."""
    assert not ops._traced()
    monkeypatch.setattr(torch.compiler, "is_compiling", lambda: True)
    assert ops._traced()
    with pytest.raises(_lib.MagnetError, match="sequence of Python floats"):
        ops.k_array(torch.tensor([0.5, 1.0]))
    assert ops.k_array((0.5, 1)) == [0.5, 1.0]
    with pytest.raises(_lib.MagnetError, match="out="):
        ops._no_out_traced(torch.empty(1))
