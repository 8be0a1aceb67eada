"""Which source layout and kernel variant each matching entry point hands to the cost kernel, and which backward runs
after it — on the CPU, with the launching ops replaced by recorders.  One row per branch of ``homography.route`` and
per entry point (the drop-in CW volume, the F volume, MagnetF's plane sweep, the fused sampler of MatchingPlan)."""
import pytest
import torch

from magnet_b200 import _lib, homography as hg, matcher, ops

SPLIT16, HALF16, PIXC, TILED32, NCHW = (_lib.SRC_SPLIT16, _lib.SRC_HALF16, _lib.SRC_PIXC, _lib.SRC_TILED32,
                                        _lib.SRC_NCHW)
AUTO, DIRECT, CELLS, TMA, MMA = (_lib.VARIANT_AUTO, _lib.VARIANT_DIRECT, _lib.VARIANT_CELLS, _lib.VARIANT_TMA,
                                 _lib.VARIANT_MMA)
ERR = "MagnetError"


@pytest.fixture
def recorded(monkeypatch):
    rec = []

    def cost_volume(ref_feat, src_feat, rays, cams, *, V, src_layout, d_volume=None, k=None, variant=AUTO, **kw):
        rec.append(("fwd", src_layout, variant))
        D = d_volume.shape[1] if d_volume is not None else len(k)
        return torch.zeros(ref_feat.shape[0], D, *ref_feat.shape[2:])

    def cost_volume_bwd(*a, fwd_layout, fwd_variant, ref_split=None, **kw):
        rec.append(("cw_bwd", fwd_layout, fwd_variant, ref_split is not None))
        return None, None, None

    def cost_volume_f_bwd(ref, src, *a, ref_split=None, split_layout=SPLIT16, **kw):
        rec.append(("f_bwd", split_layout if ref_split is not None else NCHW))
        return torch.zeros(ref.shape), torch.zeros(src.shape)

    monkeypatch.setattr(ops, "cost_volume", cost_volume)
    monkeypatch.setattr(ops, "cost_volume_bwd", cost_volume_bwd)
    monkeypatch.setattr(ops, "cost_volume_f_bwd", cost_volume_f_bwd)
    for name in ("repack_pixc", "repack_split16", "repack_half16"):
        monkeypatch.setattr(ops, name, lambda x, gmm=None, out=None: torch.zeros(1, dtype=torch.uint8))
    monkeypatch.setattr(ops, "repack_tiled32", lambda x, out=None: torch.zeros(1))
    monkeypatch.setattr(ops, "pack_cameras", lambda *a: torch.zeros(1))
    hg.clear_cache()
    yield rec
    hg.clear_cache()


def run_entry(rec, entry, C, V, D, variant, dtype, grad):
    """The records of one call (and of its backward when ``grad``), or ERR when the call raises MagnetError."""
    B, H, W = 1, 3, 5
    ref_dtype = torch.float32 if dtype == "mixed" else dtype
    src_dtype = torch.float16 if dtype == "mixed" else dtype
    ref = torch.randn(B, C, H, W).to(ref_dtype).requires_grad_(grad)
    src = torch.randn(V * B, C, H, W).to(src_dtype).requires_grad_(grad)
    gmm = torch.rand(V * B, 2, H, W)
    poses = torch.eye(4).repeat(B, V, 1, 1)
    R, t = poses[:, :, :3, :3], poses[:, :, :3, 3]
    valid = torch.ones(B, V, dtype=torch.int32)
    cam = {"intM": torch.eye(3).repeat(B, 1, 1), "unit_ray_array_2D": torch.zeros(B, 3, H * W)}
    k = [float(i) for i in range(D)]
    planes = torch.tensor(k).view(1, D, 1, 1)
    rec.clear()
    try:
        if entry == "CW":
            out = hg.est_costvolume_CW(torch.rand(B, D, H, W), ref, src, None, gmm, R, t, valid, cam, 5, variant=variant)
        elif entry == "F":
            out = hg.est_costvolume_F(planes, ref, src, R, t, valid, cam, variant=variant)
        elif entry == "PSF":
            assert variant == AUTO
            out = hg.plane_sweep_f(planes, ref, src, R, t, valid, cam, softmax=False)
        else:
            plan = matcher.MatchingPlan(ref, src, gmm, poses, valid, cam, thres=5)
            out = plan.cost(torch.rand(B, 2, H, W), k, variant=variant)
        if grad:
            out.sum().backward()
    except _lib.MagnetError:
        return ERR
    return list(rec)


F32, F16, BF16 = torch.float32, torch.float16, torch.bfloat16

ROWS = [
    # entry, C, V, D, variant, maps, grad -> records
    # tensor cores: C == 64, V <= 16, MMA or AUTO with >= MMA_MIN_PLANES hypotheses; HALF16 for one half dtype
    ("CW", 64, 2, 64, AUTO, F32, False, [("fwd", SPLIT16, AUTO)]),
    ("CW", 64, 2, 5, MMA, BF16, False, [("fwd", HALF16, MMA)]),
    ("CW", 64, 2, 64, AUTO, "mixed", False, [("fwd", SPLIT16, AUTO)]),
    ("F", 64, 2, 64, AUTO, F16, False, [("fwd", HALF16, AUTO)]),
    ("PSF", 64, 2, 32, AUTO, F32, False, [("fwd", SPLIT16, AUTO)]),
    ("plan", 64, 2, 64, AUTO, F16, False, [("fwd", HALF16, AUTO)]),
    ("plan", 64, 16, 32, MMA, F32, False, [("fwd", SPLIT16, MMA)]),
    # MMA anywhere else is refused
    ("CW", 32, 2, 64, MMA, F32, False, ERR),
    ("F", 64, 17, 64, MMA, F32, False, ERR),
    ("plan", 16, 2, 64, MMA, F32, False, ERR),
    # AUTO below the tensor cores: PIXC in the drop-in and plane-sweep paths, the gather kernel in the fused sampler
    ("CW", 64, 2, 5, AUTO, F16, False, [("fwd", PIXC, AUTO)]),
    ("F", 16, 2, 5, AUTO, F32, False, [("fwd", PIXC, AUTO)]),
    ("PSF", 32, 2, 5, AUTO, F32, False, [("fwd", PIXC, AUTO)]),
    ("plan", 64, 2, 5, AUTO, F32, False, [("fwd", TILED32, AUTO)]),
    ("plan", 32, 2, 64, AUTO, F32, False, [("fwd", TILED32, AUTO)]),
    # TMA reads PIXC, and is refused where PIXC does not fit
    ("CW", 32, 2, 64, TMA, F32, False, [("fwd", PIXC, TMA)]),
    ("plan", 64, 2, 64, TMA, F16, False, [("fwd", PIXC, TMA)]),
    ("F", 20, 2, 5, TMA, F32, False, ERR),
    ("plan", 64, 17, 5, TMA, F32, False, ERR),
    # everything else: TILED32, or NCHW when C is not a multiple of 4
    ("CW", 64, 2, 64, CELLS, F32, False, [("fwd", TILED32, CELLS)]),
    ("CW", 64, 17, 64, AUTO, F32, False, [("fwd", TILED32, AUTO)]),
    ("F", 20, 2, 5, AUTO, F32, False, [("fwd", TILED32, AUTO)]),
    ("plan", 64, 2, 64, DIRECT, F32, False, [("fwd", TILED32, DIRECT)]),
    ("CW", 10, 2, 5, AUTO, F32, False, [("fwd", NCHW, AUTO)]),
    ("PSF", 10, 2, 5, AUTO, F32, False, [("fwd", NCHW, AUTO)]),
    ("plan", 10, 2, 5, CELLS, F32, False, [("fwd", NCHW, CELLS)]),
    # differentiable CW: the tensor-core forward (backward on its split buffers), else NCHW with DIRECT
    ("CW", 64, 2, 64, AUTO, F32, True, [("fwd", SPLIT16, AUTO), ("cw_bwd", SPLIT16, AUTO, True)]),
    ("plan", 64, 2, 64, MMA, F16, True, [("fwd", HALF16, MMA), ("cw_bwd", HALF16, MMA, True)]),
    ("CW", 64, 2, 5, AUTO, F16, True, [("fwd", NCHW, DIRECT), ("cw_bwd", NCHW, DIRECT, False)]),
    ("plan", 10, 2, 64, DIRECT, F32, True, [("fwd", NCHW, DIRECT), ("cw_bwd", NCHW, DIRECT, False)]),
    ("CW", 64, 2, 64, CELLS, F32, True, ERR),
    ("plan", 32, 2, 64, TMA, F32, True, ERR),
    ("CW", 32, 2, 64, MMA, F32, True, ERR),
    ("plan", 72, 2, 64, AUTO, F32, True, ERR),
    # the F volume: est_costvolume_F keeps the CUDA-core backward; MagnetF's plane sweep reads the forward's buffers
    ("F", 64, 2, 64, AUTO, F32, True, [("fwd", SPLIT16, AUTO), ("f_bwd", NCHW)]),
    ("F", 64, 2, 64, MMA, F16, True, [("fwd", HALF16, MMA), ("f_bwd", NCHW)]),
    ("PSF", 64, 2, 64, AUTO, F32, True, [("fwd", SPLIT16, AUTO), ("f_bwd", SPLIT16)]),
    ("PSF", 64, 2, 64, AUTO, BF16, True, [("fwd", HALF16, AUTO), ("f_bwd", HALF16)]),
    ("PSF", 32, 2, 5, AUTO, F32, True, [("fwd", PIXC, AUTO), ("f_bwd", NCHW)]),
]


@pytest.mark.parametrize("entry,C,V,D,variant,dtype,grad,want", ROWS)
def test_entry_points_route_as_the_rule_says(recorded, entry, C, V, D, variant, dtype, grad, want):
    assert run_entry(recorded, entry, C, V, D, variant, dtype, grad) == want
