"""The SPLIT16 / HALF16 producer (ops.repack_split16, ops.repack_half16) byte for byte, header included, against a
restatement of its rule in torch: the largest finite |x| (0 without one), the power-of-two scale of the SPLIT16 rule
(absmax * s in [2^14, 2^15), shift clamped to [-100, 100], scale 1 for an all-zero or non-finite map), fp16 planes
hi = fp16(x * s) and lo = fp16(x * s - hi) (HALF16: hi alone), and the paired (mu, sigma) table.  The producer's
reduction keeps its running maximum in a slot that its last block re-arms, so calls into one buffer, many calls in a
row and CUDA-graph replays on changed inputs are covered as well."""
import pytest
import torch
import torch.nn.functional as F

from magnet_b200 import _lib, ops
from magnet_b200.synthetic import make_config

pytestmark = pytest.mark.gpu

FORMS = ["split16", "fp16", "bf16"]
DT = {"split16": torch.float32, "fp16": torch.float16, "bf16": torch.bfloat16}


def _repack(form, x, gmm=None, out=None):
    fn = ops.repack_split16 if form == "split16" else ops.repack_half16
    return fn(x, gmm, out=out)


def _expected(form, x, gmm=None):
    """The buffer the producer's rule gives, computed with torch on the same device (the same IEEE fp32 multiply and
    round-to-nearest fp16 conversions as the kernels)."""
    N, C, H, W = x.shape
    xf = x.float()
    a = xf.abs()
    a = torch.where(torch.isfinite(a), a, torch.zeros_like(a))
    bits = int(a.max().view(torch.int32)) if a.numel() else 0
    e = (bits >> 23) & 0xFF
    sh = 0 if e in (0, 255) else max(-100, min(100, 14 - (e - 127)))
    s = 2.0 ** sh
    header = torch.zeros(256, dtype=torch.uint8, device=x.device)
    header[:8] = torch.tensor([s, 1.0 / s], dtype=torch.float32, device=x.device).view(torch.uint8)
    header[8:12] = torch.tensor([bits], dtype=torch.int32, device=x.device).view(torch.uint8)
    v = (xf * s).permute(0, 2, 3, 1)                                   # (N, H, W, 64)
    hi = v.half()
    planes = [hi] if form != "split16" else [hi, (v - hi.float()).half()]
    planes = torch.stack(planes, 1).contiguous()                       # (N, PLANES, H, W, 64)
    ms = torch.zeros(N, H, W, 2, device=x.device) if gmm is None else gmm.permute(0, 2, 3, 1)
    ms = F.pad(ms, (0, 0, 1, 1))                                       # zeros outside the row
    table = torch.cat([ms[:, :, :-1], ms[:, :, 1:]], -1).contiguous()  # entry j = (mu, sigma)[j - 1], (mu, sigma)[j]
    return torch.cat([header, planes.view(torch.uint8).reshape(-1), table.view(torch.uint8).reshape(-1)])


def _check(form, buf, x, gmm=None, what=""):
    want = _expected(form, x, gmm)
    assert buf.numel() == want.numel(), (what, buf.numel(), want.numel())
    if torch.equal(buf, want):
        return
    N, _, H, W = x.shape
    plane_end = 256 + N * H * W * 128 * (2 if form == "split16" else 1)
    for name, lo, hi in (("header", 0, 256), ("planes", 256, plane_end), ("table", plane_end, want.numel())):
        bad = (buf[lo:hi] != want[lo:hi]).nonzero()
        assert bad.numel() == 0, f"{what}: {name} differs at {bad.numel()} bytes, first at offset {int(bad[0]) + lo}"


def _map(form, N, H, W, dev, scale=1.0, seed=0):
    g = torch.Generator(device=dev).manual_seed(seed)
    return (torch.randn(N, 64, H, W, device=dev, generator=g) * scale).to(DT[form])


def _gmm(N, H, W, dev):
    return torch.rand(N, 2, H, W, device=dev) + 0.1


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("cfg", ["cfg2", "cfg3"])
def test_bench_shapes(cuda, cfg, form):
    g = make_config(cfg, seed=0).to(cuda)
    for what, feat, gmm in (("source", g.nghbr_feat, g.nghbr_gmms), ("reference", g.ref_feat, None)):
        x = feat.to(DT[form])
        _check(form, _repack(form, x, gmm), x, gmm, f"{cfg} {what}")


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("N,H,W", [(1, 1, 1), (1, 5, 5), (3, 7, 13), (2, 3, 4), (1, 120, 161), (2, 9, 300)])
@pytest.mark.parametrize("with_gmm", [True, False], ids=["gmm", "nogmm"])
def test_ragged_and_small_shapes(cuda, form, N, H, W, with_gmm):
    x = _map(form, N, H, W, cuda, scale=3.0)
    gmm = _gmm(N, H, W, cuda) if with_gmm else None
    _check(form, _repack(form, x, gmm), x, gmm, f"{N}x{H}x{W}")


@pytest.mark.parametrize("form", FORMS)
def test_non_finite_zero_and_extreme_maps(cuda, form):
    N, H, W = 2, 12, 20
    big = torch.finfo(DT[form]).max
    base = _map(form, N, H, W, cuda)
    cases = {"zeros": torch.zeros_like(base), "inf_nan": base.clone(), "all_non_finite": torch.full_like(base, float("nan")),
             "largest": base.clone(), "tiny": (base.float() * 1e-6).to(DT[form])}
    cases["inf_nan"][0, 3, 2, 5] = float("inf")
    cases["inf_nan"][1, 60, 11, 19] = -float("inf")
    cases["inf_nan"][1, 0, 0, 0] = float("nan")
    cases["all_non_finite"][0, 0, 0, :2] = torch.tensor([float("inf"), -float("inf")])
    cases["largest"][1, 7, 3, 3] = -big
    if form == "split16":
        cases["huge"] = base * 1e37                                    # shift clamped at -100
        cases["very_small"] = base * 1e-33                             # shift clamped at +100
        cases["subnormal"] = base * 1e-42                              # absmax subnormal: scale 1
    for name, x in cases.items():
        gmm = _gmm(N, H, W, cuda)
        _check(form, _repack(form, x, gmm), x, gmm, name)


@pytest.mark.parametrize("form", FORMS)
def test_views(cuda, form):
    """A non-contiguous view is packed from its contiguous copy; a contiguous view that is not 16-byte aligned is refused
    (the kernels read the map in 16-byte vectors)."""
    N, H, W = 2, 8, 12
    wide = _map(form, N, H, W, cuda).repeat(1, 2, 1, 1)
    x = wide[:, 1:65]
    assert not x.is_contiguous()
    _check(form, _repack(form, x), x.contiguous(), None, "channel slice")
    flat = torch.zeros(N * 64 * H * W + 1, device=cuda, dtype=DT[form])
    off = flat[1:].view(N, 64, H, W)
    assert off.is_contiguous() and off.data_ptr() % 16 != 0
    with pytest.raises(_lib.MagnetError):
        _repack(form, off)


@pytest.mark.parametrize("form", FORMS)
def test_back_to_back_calls_into_one_buffer(cuda, form):
    N, H, W = 3, 10, 16
    maps = [_map(form, N, H, W, cuda, scale=1e3, seed=1), _map(form, N, H, W, cuda, scale=1e-2, seed=2),
            torch.zeros(N, 64, H, W, device=cuda, dtype=DT[form]), _map(form, N, H, W, cuda, seed=3)]
    gmms = [_gmm(N, H, W, cuda), None, _gmm(N, H, W, cuda), None]
    buf = _repack(form, maps[0], gmms[0])
    for i, (x, gmm) in enumerate(zip(maps, gmms)):
        before = _lib.launch_count()
        _repack(form, x, gmm, out=buf)
        assert _lib.launch_count() - before == 2
        _check(form, buf, x, gmm, f"call {i}")


def test_many_calls_in_a_row(cuda):
    """More calls than there are reduction slots, every one on a new maximum."""
    N, H, W = 1, 4, 8
    base = _map("split16", N, H, W, cuda)
    buf = ops.repack_split16(base)
    for i in range(1100):
        ops.repack_split16(base * (1.0 + i), out=buf)
        if i % 97 == 0 or i == 1099:
            _check("split16", buf, base * (1.0 + i), None, f"call {i}")


@pytest.mark.parametrize("form", FORMS)
def test_graph_replay_with_changed_inputs(cuda, form):
    N, H, W = 4, 16, 24
    x = _map(form, N, H, W, cuda, seed=4)
    gmm = _gmm(N, H, W, cuda)
    buf = _repack(form, x, gmm)
    eager = _repack(form, x, gmm)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream(device=cuda)
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side), torch.cuda.graph(graph, stream=side):
        _repack(form, x, gmm, out=buf)
    torch.cuda.current_stream().wait_stream(side)
    fills = [_map(form, N, H, W, cuda, scale=50.0, seed=5), _map(form, N, H, W, cuda, scale=1e-3, seed=6),
             torch.zeros(N, 64, H, W, device=cuda, dtype=DT[form]), _map(form, N, H, W, cuda, seed=7)]
    fills[3][2, 5, 1, 1] = float("nan")
    for i, f in enumerate(fills):
        x.copy_(f)
        gmm.copy_(_gmm(N, H, W, cuda))
        graph.replay()
        _repack(form, f * 2, gmm, out=eager)                           # an eager call between replays
        torch.cuda.synchronize()
        _check(form, buf, x, gmm, f"replay {i}")
        _check(form, eager, f * 2, gmm, f"eager {i}")
