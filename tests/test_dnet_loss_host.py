"""The fused D-Net loss without a GPU: the three C entry points refuse null pointers, bad shapes and k <= 0 before any
launch, the ops are registered with autograd and fakes of the eager shapes, and the Python layer refuses what it must
before touching the device."""
import ctypes as C

import pytest
import torch
from torch._subclasses.fake_tensor import FakeTensorMode

from magnet_b200 import DnetHead, _lib, library, ops

OPS = torch.ops.magnet_b200
NAMES = ("magnet_dnet_nll_fwd_f32", "magnet_dnet_nll_bwd_f32", "magnet_dnet_nll_bwd_dev_f32")


def test_entry_points_are_exported_and_declared():
    L = _lib.lib()
    assert L.magnet_abi_version() == _lib.MAGNET_ABI_VERSION == 4
    for name in NAMES:
        assert name in _lib.EXPORTS and hasattr(L, name)
    assert _lib.SIGNATURES["magnet_dnet_nll_fwd_f32"] == _lib.SIGNATURES["magnet_upsample_nll_fwd_f32"]
    assert _lib.SIGNATURES["magnet_dnet_nll_bwd_f32"] == _lib.SIGNATURES["magnet_upsample_nll_bwd_f32"]
    assert _lib.SIGNATURES["magnet_dnet_nll_bwd_dev_f32"] == _lib.SIGNATURES["magnet_upsample_nll_bwd_dev_f32"]


def _call(L, name, ptrs, B=2, H=3, W=4, k=4):
    """One call with the pointers of ``ptrs`` (a dict name -> address or None) in the trio's argument order."""
    p = lambda n: ptrs.get(n)
    head = [p("raw"), p("up_mask"), p("gt"), p("gt_mask")]
    if name.endswith("fwd_f32"):
        return getattr(L, name)(*head, B, H, W, k, p("partial"), None)
    scale = p("scale") if name.endswith("dev_f32") else 0.5
    return getattr(L, name)(*head, scale, B, H, W, k, p("grad_raw"), p("grad_mask"), None)


def test_entry_points_validate_before_any_launch():
    L = _lib.lib()
    buf = (C.c_float * 64)()
    addr = C.cast(buf, C.c_void_p).value
    args = {"fwd": ("raw", "up_mask", "gt", "gt_mask", "partial"),
            "bwd": ("raw", "up_mask", "gt", "gt_mask", "grad_raw", "grad_mask"),
            "dev": ("raw", "up_mask", "gt", "gt_mask", "scale", "grad_raw", "grad_mask")}
    launches = L.magnet_launch_count()
    for name, kind in zip(NAMES, ("fwd", "bwd", "dev")):
        full = {n: addr for n in args[kind]}
        for n in args[kind]:
            assert _call(L, name, {**full, n: None}) == _lib.ERR_NULL, (name, n)
        for shape in (dict(B=0), dict(H=0), dict(W=-1), dict(k=0), dict(k=-4), dict(B=65536), dict(H=20000, k=4)):
            assert _call(L, name, full, **shape) == _lib.ERR_SHAPE, (name, shape)
    assert L.magnet_launch_count() == launches
    assert L.magnet_upsample_nll_partials(2, 3, 4, 0) == _lib.ERR_SHAPE


def test_ops_are_registered_with_autograd_and_do_not_mutate():
    assert set(library.DNET_TRAIN_OPS) == {"dnet_nll_fwd", "dnet_nll_bwd"}
    assert not set(library.DNET_TRAIN_OPS) & (set(library.OPS) | set(library.TRAIN_OPS) | set(library.SEQUENCE_OPS))
    for name in library.DNET_TRAIN_OPS:
        schema = getattr(OPS, name).default._schema
        assert schema.name == f"magnet_b200::{name}"
        assert all(a.alias_info is None for a in schema.arguments), str(schema)
        assert all(r.alias_info is None for r in schema.returns), str(schema)
    assert "Tensor count" in str(OPS.dnet_nll_fwd.default._schema)
    assert library.dnet_nll_fwd._backward_fn is not None and library.dnet_nll_fwd._setup_context_fn is not None
    assert library.dnet_nll_bwd._backward_fn is None


@pytest.mark.parametrize("B,h,w,k", [(16, 104, 136, 4), (16, 88, 176, 4), (1, 1, 1, 1), (3, 5, 7, 2), (2, 9, 3, 8)])
def test_fakes_give_the_eager_shapes(B, h, w, k):
    cuda = lambda *s, dtype=torch.float32: torch.empty(s, device="cuda", dtype=dtype)
    with FakeTensorMode():
        full = (B, 1, k * h, k * w)
        args = (cuda(B, 2, h, w), cuda(B, 9 * k * k, h, w), cuda(*full), cuda(*full, dtype=torch.uint8), k)
        loss = OPS.dnet_nll_fwd(*args, cuda(dtype=torch.int64))
        assert loss.shape == () and loss.dtype == torch.float32 and loss.device.type == "cuda"
        g_raw, g_mask = OPS.dnet_nll_bwd(cuda(), *args, cuda(dtype=torch.int64))
        assert (tuple(g_raw.shape), tuple(g_mask.shape)) == ((B, 2, h, w), (B, 9 * k * k, h, w))
        assert g_raw.dtype == g_mask.dtype == torch.float32


def test_python_layer_refuses_before_the_device():
    raw, mask = torch.empty(1, 2, 3, 4), torch.empty(1, 144, 3, 4)
    gt, none = torch.empty(1, 1, 12, 16), torch.zeros(1, 1, 12, 16, dtype=torch.bool)
    with pytest.raises(_lib.MagnetError, match="no pixel"):
        ops.dnet_loss(raw, mask, gt, none, 4)
    with pytest.raises(_lib.MagnetError, match="k must be >= 1"):
        ops.dnet_loss(raw, mask, gt, none, 0)
    with pytest.raises(_lib.MagnetError, match="dnet=True"):
        DnetHead(in_dim=8, dnet=False).loss(torch.empty(1, 8, 3, 4), gt, none)
    with pytest.raises(_lib.MagnetError, match="no pixel"):
        DnetHead(in_dim=8).loss(torch.rand(1, 8, 3, 4), gt, none)


def test_dnet_head_forward_is_unchanged_by_the_loss():
    """``loss`` is an addition: the module's parameters and its forward contract are those of the inference head."""
    h = DnetHead(in_dim=8)
    names = [n for n, _ in h.named_parameters()]
    assert names == [f"{hd}.{i}.{p}" for hd in ("depth_head", "mask_head") for i in (0, 2, 4) for p in ("weight", "bias")]
