"""The kernels off the single-stream path: other streams, host threads, a second device and work-slot reuse.

Each result is compared with the same call run serially on the default stream of cuda:0, and that serial run is held
once, at a small case, to the float64 reference of tests/cw_grad_ref.py under the bound and clean-flip rule of
test_gpu_grad_f64.  Outputs with one owner and a fixed summation order (every forward volume, the CUDA-core depth
gradient, the heads, the metrics) must be bit-identical to the serial run.  The tensor-core feature gradients are
accumulated with atomics, whose rounding order varies between eager runs too: they are held to the float64 bound.

Where a test has to order kernels across streams it holds a stream with ``torch.cuda._sleep``, so the order it checks
does not depend on timing."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import magnet_b200
from magnet_b200 import _lib, homography, ops
from magnet_b200.synthetic import make_inputs
from tests.cw_grad_ref import Reference
from tests.test_gpu_grad_f64 import C_TOL, U, _case, _close, _close_fwd, _mma_fwd_floor, _tc_floors

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOLD = 100_000_000          # GPU cycles a held stream sleeps (tens of ms): far longer than the host needs to enqueue


def _bits(x):
    return x.detach().reshape(-1).view(torch.int32) if x.dtype == torch.float32 else x.detach().reshape(-1)


def _equal(got, want, what):
    assert got.shape == want.shape and got.dtype == want.dtype, (what, got.shape, want.shape)
    diff = _bits(got) != _bits(want)
    assert not bool(diff.any()), f"{what}: {int(diff.sum())} of {diff.numel()} elements differ from the serial run"


# ---------------------------------------------------------------------------------------------------------------------
# tensor-core work of one float64 case (tests/test_gpu_grad_f64.py): repacks, forward, CW and F backwards

class TcWork:
    """The tensor-core kernels on the inputs of a tensor-core CW case of test_gpu_grad_f64, called through ``ops`` so
    that each call is exactly one launch per kernel family, with the float64 references of its CW and F gradients."""

    def __init__(self, name, cuda, f_reference=True):
        cs = _case(name, cuda)
        self.cs, self.dev = cs, cuda
        self.ref = torch.from_numpy(cs.ref).to(cuda)
        self.src = torch.from_numpy(cs.src).to(cuda)
        self.gmm = cs.g.nghbr_gmms.contiguous()
        self.dvol = torch.from_numpy(cs.depth_vol).to(cuda)
        self.gout = torch.from_numpy(cs.gout).to(cuda)
        self.kappa = float(cs.inp.thres)
        self.planes = magnet_b200.sid_planes(1e-3, 10.0, cs.D).reshape(-1).tolist()
        self.f_want = None
        if f_reference:                         # the F volume's planes at the same D: cs.gout serves as its gradient
            depth = np.broadcast_to(np.float32(self.planes).reshape(1, -1, 1, 1), (cs.B, cs.D, cs.H, cs.W))
            rf = Reference(depth, cs.ref, cs.src, None, cs.cams.cpu().numpy(),
                           cs.inp.cam_intrins['unit_ray_array_2D'].numpy(), 0.0, pos="mma", consistency=False,
                           device=cuda)
            gsc = cs.gout.astype(np.float64) / cs.V
            self.f_want = rf.backward(gsc, np.abs(gsc))
            self.f_floors = _tc_floors(np.abs(gsc), cs.ref, cs.src, cs.V)

    def repack(self):
        return ops.repack_split16(self.ref), ops.repack_split16(self.src, self.gmm), ops.repack_split16(self.src)

    def forward(self, rs, sp, out=None):
        cs = self.cs
        return ops.cost_volume(self.ref, sp, cs.rays, cs.cams, V=cs.V, src_layout=_lib.SRC_SPLIT16, consistency=True,
                               kappa=self.kappa, d_volume=self.dvol, variant=_lib.VARIANT_MMA, ref_split=rs, out=out)

    def cw_backward(self, rs, sp, gout=None, need_depth=True):
        cs = self.cs
        return ops.cost_volume_bwd(self.ref, self.src, self.gmm, cs.rays, cs.cams, self.gout if gout is None else gout,
                                   V=cs.V, kappa=self.kappa, d_volume=self.dvol, fwd_layout=_lib.SRC_SPLIT16,
                                   fwd_variant=_lib.VARIANT_MMA, need_depth=need_depth, ref_split=rs, src_split=sp)

    def f_backward(self, rs, spf):
        cs = self.cs
        return ops.cost_volume_f_bwd(self.ref, self.src, cs.rays, cs.cams, self.planes, cs.V, None, self.gout,
                                     softmax=False, ref_split=rs, src_split=spf)

    def run(self):
        """Everything on the current stream: (volume, CW grad_ref, grad_src, grad_d, F grad_ref, grad_src)."""
        rs, sp, spf = self.repack()
        vol = self.forward(rs, sp)
        gr, gs, gd = self.cw_backward(rs, sp)
        fr, fs = self.f_backward(rs, spf)
        return vol, gr, gs, gd, fr, fs

    def check(self, res, serial, what):
        """Forward and depth gradient bit for bit against the serial run, feature gradients against float64."""
        vol, gr, gs, gd, fr, fs = res
        _equal(vol, serial[0], f"{what} volume")
        _equal(gd, serial[3], f"{what} CW grad_d")
        self.cs.check_grads(None, gr, gs, f"{what} CW", tc_features=True)
        if self.f_want is not None:
            w, (f_ref, f_src) = self.f_want, self.f_floors
            _close(fr, w["ref"], w["ref_b"], f"{what} F ref", f_ref)
            _close(fs, w["src"], w["src_b"], f"{what} F src", f_src)


_WORK = {}


def _work(name, cuda):
    if name not in _WORK:
        _WORK[name] = TcWork(name, cuda)
    return _WORK[name]


def test_serial_reference_against_float64(cuda):
    """The serial runs the other tests compare with, held once to float64: the tensor-core volume through the drop-in
    entry point and through ops, and every gradient of both backwards."""
    w = _work("tc_d32", cuda)
    cs = w.cs
    torch.cuda.synchronize()
    _close_fwd(cs.forward_variant("mma"), cs.rf, "drop-in tensor-core forward", floor=_mma_fwd_floor(cs))
    res = w.run()
    torch.cuda.synchronize()
    _close_fwd(res[0], cs.rf, "ops tensor-core forward", floor=_mma_fwd_floor(cs))
    cs.check_grads(res[3], res[1], res[2], "serial CW backward", tc_features=True)
    w.check(res, res, "serial")


# ---------------------------------------------------------------------------------------------------------------------
# 1. the preparation cache across streams

def _call(kind, cuda):
    """A no-grad drop-in call whose preparations are cached, the camera table and the intrinsics included.  Nothing in
    it waits for the device: the intrinsics are float64 and the validity int64 device tensors (their casts are device
    kernels, where host tensors would be blocking copies), and the plane depths are a host list."""
    C, D, dtype, fn = {
        "cw_split16": (64, 32, torch.float32, "cw"),
        "cw_pixc": (32, 8, torch.float32, "cw"),
        "cw_tiled32": (48, 8, torch.float32, "cw"),
        "cw_half16": (64, 32, torch.float16, "cw"),
        "cw_bf16_upcast": (32, 8, torch.bfloat16, "cw"),
        "f_split16": (64, 40, torch.float32, "f"),
        "plane_sweep_pixc": (32, 12, torch.float32, "ps"),
    }[kind]
    inp = make_inputs(B=2, V=3, D=D, H=24, W=40, C=C, seed=C + D, depth="smooth", invalid=[(1, 2)])
    g = inp.to(cuda)
    ref, src = g.ref_feat.to(dtype), g.nghbr_feat.to(dtype)
    dvol = g.depth_volume()
    planes = magnet_b200.sid_planes(0.2, 10.0, D).reshape(-1).tolist()
    intr = {k: v.to(cuda, torch.float64) for k, v in inp.cam_intrins.items()}
    valid = inp.is_valid.to(cuda, torch.int64)
    want_layout = {"cw_split16": _lib.SRC_SPLIT16, "cw_pixc": _lib.SRC_PIXC, "cw_tiled32": _lib.SRC_TILED32,
                   "cw_half16": _lib.SRC_HALF16, "cw_bf16_upcast": _lib.SRC_PIXC, "f_split16": _lib.SRC_SPLIT16,
                   "plane_sweep_pixc": _lib.SRC_PIXC}[kind]
    mode = _lib.DEPTH_VOLUME if fn == "cw" else _lib.DEPTH_PLANES
    assert homography.route(C, 3, D, _lib.VARIANT_AUTO, mode, dtype, dtype)[0] == want_layout

    def call():
        with torch.no_grad():
            if fn == "cw":
                return magnet_b200.est_costvolume_CW(dvol, ref, src, g.ref_gmms, g.nghbr_gmms, g.R, g.t, valid, intr,
                                                     inp.thres)
            if fn == "f":
                return magnet_b200.est_costvolume_F(planes, ref, src, g.R, g.t, valid, intr)
            return homography.plane_sweep_f(planes, ref, src, g.R, g.t, valid, intr, softmax=False)
    return call


CACHED_KINDS = ["cw_split16", "cw_pixc", "cw_tiled32", "cw_half16", "cw_bf16_upcast", "f_split16", "plane_sweep_pixc"]


def _cached_tensors():
    out = []
    for _, value in list(homography._cache._items.values()):
        for v in (value if isinstance(value, tuple) else (value,)):
            if isinstance(v, torch.Tensor) and v.is_cuda:
                out.append(v)
    return out


def _poison(nbytes):
    """Blocks of these sizes on the current stream, filled with 0xff (NaN as floats) and freed: the next allocations of
    the same sizes on this stream get them back, so a read of a buffer whose producer has not run yet sees NaN."""
    blocks = [torch.full((n,), 255, dtype=torch.uint8, device="cuda") for n in nbytes]
    del blocks


@pytest.mark.parametrize("kind", CACHED_KINDS)
def test_cross_stream_cache_hit(cuda, kind):
    """The same call on s1 (held behind a sleep) and then on s2: s2 must not read the preparations s1 has queued but
    not yet made.  Every call equals the serial one.  s1 must still be asleep after both calls are enqueued, or the
    test would not check what it claims.

    The blocks s1 allocates from are filled with 0xff first, so a read of an unwritten preparation sees NaN cameras,
    features and scales.  Every kernel these calls reach bounds a sample position before it forms an address (the
    DIRECT kernel's +-10 clamp with its NaN test, fminf(fmaxf(x, -2), W) in the TMA, global-gather, tensor-core and
    window-box code, which maps NaN to -2), and reads the SPLIT16 / HALF16 scales only as factors, so such a read
    gives a wrong volume, never an access outside the buffers."""
    call = _call(kind, cuda)
    homography.clear_cache()
    want = call()
    torch.cuda.synchronize()
    sizes = [t.numel() * t.element_size() for t in _cached_tensors()]
    assert len(sizes) >= 3, sizes                       # the source maps, the camera table and the intrinsics at least
    homography.clear_cache()
    main, s1, s2 = torch.cuda.current_stream(), torch.cuda.Stream(), torch.cuda.Stream()
    s1.wait_stream(main)
    s2.wait_stream(main)
    with torch.cuda.stream(s1):
        _poison(sizes)
        torch.cuda._sleep(HOLD)
        out1 = call()
    assert not s1.query(), "the s1 call waited for the device: s1 is no longer held"
    with torch.cuda.stream(s2):
        out2 = call()
    assert not s1.query(), "s1 finished before the s2 call was enqueued"
    torch.cuda.synchronize()
    _equal(out2, want, f"{kind} on s2")
    _equal(out1, want, f"{kind} on s1")
    homography.clear_cache()


@pytest.mark.parametrize("kind", ["cw_split16", "cw_half16", "f_split16"])
def test_dropped_entry_outlives_pending_work(cuda, kind):
    """Preparations made on s1, then a call on s2 held behind a sleep, then the cache dropped and same-sized tensors
    allocated and filled on s1 while s2 still waits: the s2 result must not change."""
    call = _call(kind, cuda)
    homography.clear_cache()
    want = call()
    torch.cuda.synchronize()
    main, s1, s2 = torch.cuda.current_stream(), torch.cuda.Stream(), torch.cuda.Stream()
    s1.wait_stream(main)
    s2.wait_stream(main)
    homography.clear_cache()
    with torch.cuda.stream(s1):
        call()                                          # entries made on s1
    torch.cuda.synchronize()
    sizes = [t.numel() * t.element_size() for t in _cached_tensors()]
    with torch.cuda.stream(s2):
        s2.wait_stream(main)
        torch.cuda._sleep(HOLD)
        out2 = call()
    assert not s2.query(), "the s2 call waited for the device: s2 is no longer held"
    homography.clear_cache()
    with torch.cuda.stream(s1):
        fill = [torch.full((n,), 255, dtype=torch.uint8, device="cuda") for n in sizes]
    assert not s2.query(), "s2 finished before the s1 fills were enqueued"
    torch.cuda.synchronize()
    del fill
    _equal(out2, want, f"{kind} on s2")


# ---------------------------------------------------------------------------------------------------------------------
# 2. concurrent persistent launches

CONCURRENT = ["stress_v2_d32", "cfg3_volume", "tc_d33_v6", "tc_d65_scales"]


def test_concurrent_persistent_launches(cuda):
    """Four streams, each with its own inputs: repacks, tensor-core forward, CW and F tensor-core backwards, all issued
    before one synchronise.  Every output matches its serial run."""
    works = [_work(n, cuda) for n in CONCURRENT]
    serial = []
    for w in works:
        serial.append(w.run())
        torch.cuda.synchronize()
    main = torch.cuda.current_stream()
    streams = [torch.cuda.Stream() for _ in works]
    results = []
    for s, w in zip(streams, works):
        s.wait_stream(main)
        with torch.cuda.stream(s):
            results.append(w.run())
    torch.cuda.synchronize()
    for n, w, res, ser in zip(CONCURRENT, works, results, serial):
        w.check(res, ser, f"{n} concurrent")


# ---------------------------------------------------------------------------------------------------------------------
# 3. work-slot wrap-around

EAGER_LAUNCHES = 1100       # > 2 x 512: every eager slot is taken at least twice
GRAPHS = 513                # > 512: two graphs share a captured slot whatever tickets earlier tests took


def _scales(n):
    """Per-launch powers of two for the upstream gradient: a launch that skipped work items and kept another launch's
    values would be off by a factor of 2 or more, while g / scale is exactly the unscaled run's result."""
    return [2.0 ** (i % 7 - 3) for i in range(n)]


class _GradCheck:
    """On-device count of the feature-gradient elements beyond the float64 bound, per launch (one read at the end)."""

    def __init__(self, w, n):
        cs = w.cs
        dev = w.dev
        f_ref, f_src = cs.floors
        self.want = [torch.from_numpy(cs.want[k]).to(dev) for k in ("ref", "src")]
        self.tol = [torch.from_numpy(C_TOL * U * cs.want[k + "_b"] + f).to(dev)
                    for k, f in (("ref", f_ref), ("src", f_src))]
        self.bad = torch.zeros(n, dtype=torch.int64, device=dev)

    def add(self, i, scale, gr, gs):
        for g, want, tol in zip((gr, gs), self.want, self.tol):
            err = (g.double() / scale - want).abs()
            self.bad[i] += ((err > tol) | ~torch.isfinite(g)).sum()   # NaN compares false: count it explicitly

    def assert_clean(self, what):
        bad = self.bad.cpu()
        idx = torch.nonzero(bad).reshape(-1).tolist()
        assert not idx, f"{what}: feature gradients beyond the float64 bound at launches {idx[:20]} ({bad[idx[:20]]})"


def test_eager_work_slot_wraparound(cuda):
    """1100 eager launches each of the tensor-core forward and the tensor-core backward on one small case: every volume
    equals the first bit for bit, every gradient is within the float64 bound."""
    w = _work("tc_d32", cuda)
    rs, sp, _ = w.repack()
    cs = w.cs
    outs = torch.full((EAGER_LAUNCHES, cs.B, cs.D, cs.H, cs.W), float("nan"), device=cuda)
    check = _GradCheck(w, EAGER_LAUNCHES)
    for i, s in enumerate(_scales(EAGER_LAUNCHES)):
        w.forward(rs, sp, out=outs[i])
        gr, gs, _ = w.cw_backward(rs, sp, gout=w.gout * s, need_depth=False)
        check.add(i, s, gr, gs)
    torch.cuda.synchronize()
    _close_fwd(outs[0], cs.rf, "first launch", floor=_mma_fwd_floor(cs))
    diff = (outs.view(EAGER_LAUNCHES, -1).view(torch.int32) != outs[0].reshape(1, -1).view(torch.int32)).any(1)
    idx = torch.nonzero(diff).reshape(-1).tolist()
    assert not idx, f"volumes differ from the first launch at launches {idx[:20]}"
    check.assert_clean("eager")


def test_captured_work_slot_wraparound(cuda):
    """513 captured graphs of the forward and the backward, replayed in sequence with an eager launch of each after
    every replay: each replay equals the eager volume and its gradients are within the float64 bound."""
    w = _work("tc_d32", cuda)
    rs, sp, _ = w.repack()
    cs = w.cs
    eager = w.forward(rs, sp)
    scales = _scales(GRAPHS)
    gouts = [w.gout * s for s in scales]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):                       # warm-up off the default stream before capture
        w.forward(rs, sp)
        w.cw_backward(rs, sp, need_depth=False)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    pool = torch.cuda.graph_pool_handle()
    graphs, outs = [], []
    with torch.cuda.stream(side):                       # capture_begin / end: torch.cuda.graph would collect garbage
        for j in range(GRAPHS):                         # at every one of the 513 captures
            graph = torch.cuda.CUDAGraph()
            graph.capture_begin(pool=pool)
            out = torch.full_like(eager, float("nan"))
            w.forward(rs, sp, out=out)
            gr, gs, _ = w.cw_backward(rs, sp, gout=gouts[j], need_depth=False)
            graph.capture_end()
            graphs.append(graph)
            outs.append((out, gr, gs))
    torch.cuda.current_stream().wait_stream(side)
    captured, eager_check = _GradCheck(w, GRAPHS), _GradCheck(w, GRAPHS)
    bad_vol = torch.zeros(GRAPHS, dtype=torch.bool, device=cuda)
    for j, graph in enumerate(graphs):
        graph.replay()
        out, gr, gs = outs[j]
        bad_vol[j] = (out.view(torch.int32) != eager.view(torch.int32)).any()
        captured.add(j, scales[j], gr, gs)
        out.fill_(float("nan"))                         # a later replay of this graph must write it again
        e_out = w.forward(rs, sp)
        bad_vol[j] |= (e_out.view(torch.int32) != eager.view(torch.int32)).any()
        e_gr, e_gs, _ = w.cw_backward(rs, sp, gout=gouts[j], need_depth=False)
        eager_check.add(j, scales[j], e_gr, e_gs)
    graphs[0].replay()                                  # once more after every other graph has used the slots
    torch.cuda.synchronize()
    _equal(outs[0][0], eager, "graph 0 replayed last")
    idx = torch.nonzero(bad_vol.cpu()).reshape(-1).tolist()
    assert not idx, f"volumes differ from eager at graphs {idx[:20]}"
    captured.assert_clean("captured")
    eager_check.assert_clean("eager between replays")
    _close_fwd(eager, cs.rf, "eager forward", floor=_mma_fwd_floor(cs))


# ---------------------------------------------------------------------------------------------------------------------
# 4. first use from several host threads

THREAD_SCRIPT = r'''
import sys, threading
import torch
import magnet_b200
from magnet_b200 import ops
from magnet_b200.synthetic import make_inputs

dev = torch.device("cuda:0")
torch.cuda.init()


def inputs(seed):
    torch.manual_seed(seed)
    inp = make_inputs(B=2, V=3, D=32, H=24, W=40, C=64, seed=seed, depth="smooth", invalid=[(1, 1)])
    head = magnet_b200.GNET(ch_in=32 + 8).to(dev)
    x = dict(inp=inp, g=inp.to(dev), head=head, xd3=torch.randn(2, 8, 24, 40, device=dev),
             mask=torch.randn(2, 144, 24, 40, device=dev), gt=1.0 + 9.0 * torch.rand(2, 1, 96, 160, device=dev))
    x["gtm"] = x["gt"] > 2.0
    return x


def steps(x):
    inp, g = x["inp"], x["g"]
    out = []
    pred = g.ref_gmms
    preds = []
    packed = None
    for it in range(3):
        dvol = ops.sample_depths(pred, inp.k.tolist()).requires_grad_(True)
        ref = g.ref_feat.clone().requires_grad_(True)
        cv = magnet_b200.est_costvolume_CW(dvol, ref, g.nghbr_feat, g.ref_gmms, g.nghbr_gmms, g.R, g.t, inp.is_valid,
                                           inp.cam_intrins, inp.thres)
        (cv * cv.detach().sign()).sum().backward()
        with torch.no_grad():
            inv = x["head"].invariant_part(x["xd3"], 32)
            if packed is None:
                packed = ops.pack_gnet_weights(x["head"], 32)
            raw = ops.gnet_update(cv.detach(), inv, packed, torch.cat([torch.zeros_like(pred[:, :1]),
                                                                        torch.ones_like(pred[:, :1])], 1))
            pred = ops.gaussian_update(raw, pred)
        preds.append(pred)
        out += [cv.detach(), dvol.grad, ref.grad, raw, pred]
    with torch.no_grad():
        loss = ops.magnet_loss(preds, x["mask"], x["gt"], x["gtm"], 4)
        m = magnet_b200.DepthMetrics(1e-3, 10.0)
        rows = m.update(preds, x["gt"], up_mask=x["mask"], k=4)
    return out + [loss.reshape(1), rows]


# each matching step yields (volume, grad_d, grad_ref, G-Net output, Gaussians): the tensor-core grad_ref (shared-memory
# atomics) varies in its last bits between runs; everything else has one owner and a fixed order
ATOMIC = {2 + 5 * i for i in range(3)}


def same(a, b):
    return (a.shape == b.shape and a.dtype == b.dtype and torch.equal(a.isnan(), b.isnan())
            and torch.equal(a.nan_to_num(), b.nan_to_num()))

data = [inputs(100 + i) for i in range(4)]
results, errors = [None] * 4, []
barrier = threading.Barrier(4, timeout=120)


def worker(i):
    try:
        s = torch.cuda.Stream(device=dev)
        s.wait_stream(torch.cuda.default_stream(dev))
        barrier.wait()
        with torch.cuda.stream(s):
            r = steps(data[i])
        s.synchronize()
        results[i] = r
    except BaseException as e:                       # reported by the main thread
        errors.append(f"thread {i}: {type(e).__name__}: {e}")
        barrier.abort()                              # the others leave the barrier instead of waiting for it


threads = [threading.Thread(target=worker, args=(i,)) for i in range(4)]
for t in threads:
    t.start()
for t in threads:
    t.join()
if errors:
    print("\n".join(errors))
    sys.exit(1)
torch.cuda.synchronize()
bad = []
for i in range(4):
    magnet_b200.clear_cache()
    want = steps(data[i])
    torch.cuda.synchronize()
    for j, (a, b) in enumerate(zip(results[i], want)):
        if j in ATOMIC:
            scale = float(b.abs().max())
            ok = float((a - b).abs().max()) <= 2.0 ** -17 * scale
        else:
            ok = same(a, b)
        if not ok:
            bad.append((i, j))
if bad:
    print("mismatches (thread, output):", bad)
    sys.exit(1)
print("threads ok")
'''


def test_first_use_in_host_threads(cuda):
    """A fresh interpreter, so that every kernel's first use (shared-memory opt-in, tensor-map encoder, the library
    binding) happens inside four threads that each run matching steps on their own stream: cost volume forward and
    backward, fused G-Net update, Gaussian update, magnet_loss and DepthMetrics.update.  Every result must equal a
    serial run afterwards (the tensor-core grad_ref to 2^-17 of its maximum: its atomics reorder)."""
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    r = subprocess.run([sys.executable, "-s", "-c", THREAD_SCRIPT], cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=300)
    print(r.stdout[-4000:], r.stderr[-4000:])
    assert r.returncode == 0, (r.returncode, r.stdout[-2000:], r.stderr[-2000:])
    assert "threads ok" in r.stdout


# ---------------------------------------------------------------------------------------------------------------------
# 5. a second device

def _device_calls(dev):
    """One representative call of each entry-point family with every operand on ``dev``; returns the outputs."""
    torch.manual_seed(0)
    inp = make_inputs(B=2, V=3, D=32, H=16, W=24, C=64, seed=11, depth="smooth", invalid=[(1, 2)])
    g = inp.to(dev)
    intr = {k: v.to(dev) for k, v in inp.cam_intrins.items()}
    out = []
    with torch.no_grad():
        dvol = g.depth_volume()
        for v in (_lib.VARIANT_DIRECT, _lib.VARIANT_CELLS, _lib.VARIANT_TMA, _lib.VARIANT_MMA):
            out.append(magnet_b200.est_costvolume_CW(dvol, g.ref_feat, g.nghbr_feat, g.ref_gmms, g.nghbr_gmms, g.R,
                                                     g.t, inp.is_valid, inp.cam_intrins, inp.thres, variant=v))
        plan = magnet_b200.MatchingPlan(g.ref_feat, g.nghbr_feat, g.nghbr_gmms, g.nghbr_poses, inp.is_valid,
                                        inp.cam_intrins, thres=inp.thres)
        out.append(plan.cost(g.ref_gmms, inp.k.tolist()))
        planes = magnet_b200.sid_planes(0.2, 10.0, 32, device=dev).reshape(1, -1, 1, 1)
        scores = homography.plane_sweep_f(planes, g.ref_feat, g.nghbr_feat, g.R, g.t, inp.is_valid, intr,
                                          softmax=False)
        out += [scores, ops.plane_depth(scores, planes.reshape(-1).tolist(), scores=True)]
    # both backwards (CUDA-core: one owner per element for grad_ref / grad_d) and the camera gradients
    dv = g.depth_volume().requires_grad_(True)
    rf = g.ref_feat.clone().requires_grad_(True)
    R, t = g.R.clone().requires_grad_(True), g.t.clone().requires_grad_(True)
    with homography.geometry_grad():
        cw = magnet_b200.est_costvolume_CW(dv, rf, g.nghbr_feat, g.ref_gmms, g.nghbr_gmms, R, t, inp.is_valid, intr,
                                           inp.thres, variant=_lib.VARIANT_DIRECT)
        cw.square().sum().backward()
    rf2 = g.ref_feat.clone().requires_grad_(True)
    magnet_b200.est_costvolume_F(planes, rf2, g.nghbr_feat, g.R, g.t, inp.is_valid, intr).square().sum().backward()
    out += [cw.detach(), dv.grad, rf.grad, R.grad, t.grad, rf2.grad]
    # fused heads and their packs, the update and the upsampling, the metrics
    with torch.no_grad():
        gh = magnet_b200.GNET(ch_in=32 + 8).to(dev)
        cv = torch.randn(2, 32, 16, 24, device=dev)
        inv = gh.invariant_part(torch.randn(2, 8, 16, 24, device=dev), 32)
        prev = torch.cat([torch.zeros(2, 1, 16, 24, device=dev), torch.ones(2, 1, 16, 24, device=dev)], 1)
        raw = ops.gnet_update(cv, inv, ops.pack_gnet_weights(gh, 32), prev)
        pred = ops.gaussian_update(raw, g.ref_gmms)
        mh = magnet_b200.MagnetHead(dnet_fdim=16).mask_head.to(dev).eval()
        ups = ops.mask_upsample(torch.randn(2, 128, 16, 24, device=dev), ops.pack_mask_weights(mh), [pred], 4)
        mask = torch.randn(2, 144, 16, 24, device=dev)
        up = ops.convex_upsample(pred, mask, 4)
        dh = magnet_b200.DnetHead(in_dim=256, dnet=True).to(dev).eval()
        packed = ops.pack_dnet_weights(dh.depth_head, dh.mask_head)
        pre_d, pre_m = torch.randn(2, 128, 16, 24, device=dev), torch.randn(2, 128, 16, 24, device=dev)
        draw = ops.dnet_depth(pre_d, packed, sigma=False)
        gt = 1.0 + 9.0 * torch.rand(2, 1, 64, 96, device=dev)
        out += [raw, pred, *ups, up, draw, ops.dnet_depth(pre_d, packed, sigma=True), ops.dnet_upsample(pre_m, packed, draw),
                ops.depth_metrics(up, gt, min_depth=1e-3, max_depth=10.0)]
    torch.cuda.synchronize(dev)
    return out


def test_second_device(cuda, monkeypatch):
    if torch.cuda.device_count() < 2:
        pytest.skip("one CUDA device: the operands-on-cuda:1 runs need a second one")
    homography.clear_cache()
    want = [x.cpu() for x in _device_calls(torch.device("cuda:0"))]
    d1 = torch.device("cuda:1")
    for current in (0, 1):
        homography.clear_cache()
        with torch.cuda.device(current):
            got = _device_calls(d1)
        assert all(x.device == d1 for x in got)
        for i, (a, b) in enumerate(zip(got, want)):
            _equal(a.cpu(), b, f"output {i} on cuda:1 with cuda:{current} current")
    # the grid of the persistent kernels is sized by the SM count of the device asked about: the library is asked
    # with that device current, whichever device the caller has current
    L = _lib.lib()
    real, seen = L.magnet_cost_launch_info, []

    def spy(*args):
        seen.append(torch.cuda.current_device())
        return real(*args)
    monkeypatch.setattr(L, "magnet_cost_launch_info", spy)
    info = {}
    for current in (0, 1):
        with torch.cuda.device(current):
            info[current] = ops.cost_launch_info(2, 3, 64, 64, 120, 160, variant=_lib.VARIANT_MMA, device=d1)
            assert torch.cuda.current_device() == current
    sms = torch.cuda.get_device_properties(d1).multi_processor_count
    assert seen == [1, 1], seen
    assert info[0] == info[1] and info[0][0] == min(2 * 15 * 20, 2 * sms), info
