"""The traced frame-table path of sequence evaluation without a GPU (DESIGN §3.18): the registration of
``cost_volume_indexed`` and ``check_src_index``, their fakes for every source layout and depth mode, the argument checks
of ``magnet_check_src_index``, and eager indexed calls that never reach the dispatcher."""
import ctypes as C

import pytest
import torch
from torch._subclasses.fake_tensor import FakeTensorMode

from magnet_b200 import _lib, library, ops

OPS = torch.ops.magnet_b200


def test_sequence_ops_are_registered_apart_from_the_inference_ops():
    assert set(library.SEQUENCE_OPS) == {"check_src_index", "cost_volume_indexed"}
    assert not set(library.SEQUENCE_OPS) & (set(library.OPS) | set(library.TRAIN_OPS))
    for name in library.SEQUENCE_OPS:
        assert OPS.__getattr__(name).default._schema.name == f"magnet_b200::{name}"


def test_sequence_ops_do_not_mutate_or_alias():
    for name in library.SEQUENCE_OPS:
        schema = OPS.__getattr__(name).default._schema
        assert all(a.alias_info is None for a in schema.arguments), str(schema)
        assert all(r.alias_info is None for r in schema.returns), str(schema)


def test_indexed_volume_takes_the_cost_volume_arguments_then_the_table():
    indexed, plain = OPS.cost_volume_indexed.default._schema, OPS.cost_volume.default._schema
    names = [a.name for a in indexed.arguments]
    assert names == [a.name for a in plain.arguments] + ["src_index", "n_src"]
    text = str(indexed)
    for arg in ("SymInt V", "SymInt src_layout", "bool consistency", "float kappa", "float[]? k", "bool planes",
                "bool softmax", "SymInt variant", "Tensor src_index", "SymInt? n_src"):
        assert arg in text, (arg, text)
    assert "SymInt n_src" in str(OPS.check_src_index.default._schema)


def _cuda(*shape, dtype=torch.float32):
    return torch.empty(shape, device="cuda", dtype=dtype)


def _indexed_cases(B, V, S, C, H, W, D):
    """(name, arguments of cost_volume_indexed, D of the volume): every source layout, the three depth modes."""
    k = [0.1 * i for i in range(D)]
    split = ops.packed_bytes(_lib.SRC_SPLIT16, S, H, W)
    half = ops.packed_bytes(_lib.SRC_HALF16, S, H, W)
    rsplit = ops.packed_bytes(_lib.SRC_SPLIT16, B, H, W)
    rhalf = ops.packed_bytes(_lib.SRC_HALF16, B, H, W)
    u8, A = torch.uint8, _lib
    common = lambda layout, src, ref=None: ((ref if ref is not None else _cuda(B, C, H, W)), src, _cuda(B, 3, H * W),
                                           _cuda(B * V, 16), V, layout)
    table = lambda dtype=torch.int32: _cuda(B, V, dtype=dtype)
    return [
        ("tiled32-gauss", (*common(A.SRC_TILED32, _cuda(S, H, (W + 31) // 32, C // 4, 32, 4)), True, _cuda(S, 2, H, W),
                           5.0, None, _cuda(B, 2, H, W), k, False, False, A.VARIANT_AUTO, None, table(), S), D),
        ("nchw-volume", (*common(A.SRC_NCHW, _cuda(S, C, H, W)), True, _cuda(S, 2, H, W), 5.0, _cuda(B, D + 3, H, W),
                         None, None, False, False, A.VARIANT_DIRECT, None, table(torch.int64), None), D + 3),
        ("pixc-volume", (*common(A.SRC_PIXC, _cuda(S, H, W, C + 4)), True, None, 5.0, _cuda(B, D, H, W), None, None,
                         False, False, A.VARIANT_TMA, None, table(), S), D),
        ("split16-gauss", (*common(A.SRC_SPLIT16, _cuda(split, dtype=u8)), True, None, 5.0, None, _cuda(B, 2, H, W), k,
                           False, False, A.VARIANT_AUTO, _cuda(rsplit, dtype=u8), table(torch.int64), S), D),
        ("split16-planes", (*common(A.SRC_SPLIT16, _cuda(split, dtype=u8)), False, None, 0.0, None, None, k, True,
                            True, A.VARIANT_AUTO, _cuda(rsplit, dtype=u8), table(), None), D),
        ("half16-gauss", (*common(A.SRC_HALF16, _cuda(half, dtype=u8), _cuda(B, C, H, W, dtype=torch.bfloat16)), True,
                          None, 5.0, None, _cuda(B, 2, H, W), k, False, False, A.VARIANT_MMA, _cuda(rhalf, dtype=u8),
                          table(), S), D),
    ]


_SHAPES = [(1, 4, 4, 64, 30, 40, 5), (1, 2, 2, 64, 22, 76, 64), (8, 4, 11, 64, 120, 160, 64), (2, 3, 5, 64, 24, 40, 16)]


@pytest.mark.parametrize("B,V,S,C,H,W,D", _SHAPES)
def test_indexed_fake_gives_the_volume_shape(B, V, S, C, H, W, D):
    with FakeTensorMode():
        for name, args, d in _indexed_cases(B, V, S, C, H, W, D):
            out = OPS.cost_volume_indexed(*args)
            assert (tuple(out.shape), out.dtype, out.device.type) == ((B, d, H, W), torch.float32, "cuda"), name
        table, bad = OPS.check_src_index(_cuda(B, V, dtype=torch.int64), S)
        assert [(tuple(t.shape), t.dtype) for t in (table, bad)] == [((B, V), torch.int32), ((B,), torch.int32)]


def test_indexed_fake_refuses_a_count_the_buffer_does_not_hold():
    B, V, S, C, H, W, D = 1, 4, 4, 64, 30, 40, 5
    with FakeTensorMode():
        for name, args, _ in _indexed_cases(B, V, S, C, H, W, D):
            with pytest.raises(_lib.MagnetError, match="does not match src_feat"):
                OPS.cost_volume_indexed(*args[:-1], S + 1)
        split = _cuda(ops.packed_bytes(_lib.SRC_SPLIT16, S, H, W) + 16, dtype=torch.uint8)   # not a whole buffer
        _, args, _ = _indexed_cases(B, V, S, C, H, W, D)[3]
        with pytest.raises(_lib.MagnetError, match="repack_split16 buffer"):
            OPS.cost_volume_indexed(*args[:1], split, *args[2:])


def test_check_entry_point_validates_without_gpu():
    L = _lib.lib()
    assert "magnet_check_src_index" in _lib.EXPORTS
    buf = (C.c_int64 * 16)()
    p = C.cast(buf, C.c_void_p).value
    I32, I64 = _lib.INDEX_I32, _lib.INDEX_I64
    launches = L.magnet_launch_count()
    fn = lambda src, dtype, B, V, n, out, bad: L.magnet_check_src_index(src, dtype, B, V, n, out, bad, None)
    assert fn(None, I32, 2, 4, 5, p, p) == _lib.ERR_NULL
    assert fn(p, I32, 2, 4, 5, None, p) == _lib.ERR_NULL
    assert fn(p, I32, 2, 4, 5, p, None) == _lib.ERR_NULL
    for B, V, n in ((0, 4, 5), (2, 0, 5), (-1, 4, 5), (2, 4, 0), (2, 4, -2), (1 << 16, 1 << 15, 5)):
        assert fn(p, I64, B, V, n, p, p) == _lib.ERR_SHAPE, (B, V, n)
    for dtype in (2, -1, 7):
        assert fn(p, dtype, 2, 4, 5, p, p) == _lib.ERR_UNSUPPORTED, dtype
    assert fn(p + 4, I64, 2, 4, 5, p, p) == _lib.ERR_ALIGN             # an int64 table is 8-byte aligned
    assert fn(p + 2, I32, 2, 4, 5, p, p) == _lib.ERR_ALIGN
    assert fn(p + 4, I32, 2, 4, 5, p + 2, p) == _lib.ERR_ALIGN
    assert fn(p + 4, I32, 2, 4, 5, p, p + 1) == _lib.ERR_ALIGN
    assert L.magnet_launch_count() == launches                           # nothing was launched


@pytest.mark.parametrize("table,match", [
    (torch.zeros(2, 4, dtype=torch.float32), "int32 or int64"),
    (torch.zeros(2, 4, dtype=torch.int16), "int32 or int64"),
    (torch.zeros(8, dtype=torch.int32), "shape"),
])
def test_device_check_refuses_before_any_launch(monkeypatch, table, match):
    monkeypatch.setattr(ops, "_need_cuda", lambda name, x: x)             # a CPU tensor stands in for a device one
    launches = _lib.launch_count()
    with pytest.raises(_lib.MagnetError, match=match):
        ops.check_src_index_device(table, 5)
    with pytest.raises(_lib.MagnetError, match="at least one source image"):
        ops.check_src_index_device(torch.zeros(2, 4, dtype=torch.int32), 0)
    assert _lib.launch_count() == launches


def test_eager_indexed_calls_do_not_go_through_the_dispatcher(monkeypatch):
    """Outside tracing an indexed ops.cost_volume checks its table on the host and calls the C entry point directly;
    the op, and the device check inside it, are only reached while torch.compile traces."""
    assert not ops._traced()
    called = []
    monkeypatch.setattr(ops, "_op", lambda name: called.append(name) or (lambda *args: None))
    table = torch.tensor([[0, 1, 2, 9]], dtype=torch.int32)
    with pytest.raises(_lib.MagnetError, match="must lie in"):                # the host range check, before any launch
        ops.check_src_index(table, 1, 4, 5)
    with pytest.raises(_lib.MagnetError, match="CUDA tensor"):               # the eager path's checks, not an op
        ops.cost_volume(torch.zeros(1, 64, 8, 8), torch.zeros(5, 64, 8, 8), torch.zeros(1, 3, 64),
                        torch.zeros(4, 16), V=4, src_layout=_lib.SRC_NCHW, consistency=False, k=[1.0], planes=True,
                        src_index=table)
    assert called == []
    monkeypatch.setattr(torch.compiler, "is_compiling", lambda: True)
    assert ops._traced()
    ops.check_src_index_device(table, 5)
    assert called == ["check_src_index"]
