"""Every forward cost-volume kernel instance against the float64 reference of tests/cw_grad_ref.py: DIRECT (NCHW and
TILED32 gathers), CELLS (and its no-reuse variant in GAUSS mode), TMA and MMA, in each depth mode (VOLUME, GAUSS,
PLANES), with and without the consistency weighting, and with the softmax over the hypotheses where consistency is off.
The cases of tests/forward_f64_cases.py put the shapes on both sides of the kernels' tile and chunk edges and of the
16-camera limit of the staged kernels; every (variant, layout) pair the library refuses must raise MagnetError.

Tolerances are those of tests/test_gpu_grad_f64.py: |got - ref| <= c u bound (+ the tensor-core floor), and with the
consistency weighting an element beyond it must be a clean flip of one view within 1e-3 of its threshold.  Kernels
that place their samples with project() (every one but DIRECT) carry the position-error term of DESIGN §3.1."""
import numpy as np
import pytest
import torch

import magnet_b200
from magnet_b200 import _lib, ops
from magnet_b200 import homography as hg
from magnet_b200.synthetic import CONFIGS, make_inputs
from tests import forward_f64_cases as fc
from tests import test_gpu_grad_f64 as gf
from tests.cw_grad_ref import U, Reference, gauss_depths

pytestmark = pytest.mark.gpu

VARIANTS = {"direct": _lib.VARIANT_DIRECT, "cells": _lib.VARIANT_CELLS, "cells_noreuse": _lib.VARIANT_CELLS_NOREUSE,
            "tma": _lib.VARIANT_TMA, "mma": _lib.VARIANT_MMA, "auto": _lib.VARIANT_AUTO}
LAYOUTS = {"nchw": _lib.SRC_NCHW, "tiled32": _lib.SRC_TILED32, "pixc": _lib.SRC_PIXC, "split16": _lib.SRC_SPLIT16}
DEPTH_MODES = {"volume": _lib.DEPTH_VOLUME, "gauss": _lib.DEPTH_GAUSS, "planes": _lib.DEPTH_PLANES}


def _ordered(vals, order, rng):
    vals = list(vals)
    if order == "descending":
        return sorted(vals, reverse=True)
    if order == "shuffled":
        while True:
            perm = [vals[i] for i in rng.permutation(len(vals))]
            if any(b < a for a, b in zip(perm, perm[1:])):
                return perm
    return vals


class FwdCase:
    """The inputs of one case of forward_f64_cases.CASES on the device, its depths per mode, and one float64
    reference per (mode, consistency), built on first use."""

    def __init__(self, name, cuda):
        self.__dict__.update(fc.spec(name, CONFIGS))
        self.name, self.dev = name, cuda
        B, V, D, H, W, C = self.B, self.V, self.D, self.H, self.W, self.C
        seed = sum(map(ord, name))
        rng = np.random.default_rng(seed)
        inp = make_inputs(B=B, V=V, D=D, H=H, W=W, C=C, seed=seed, depth=self.depth, invalid=self.invalid,
                          family=self.family)
        gf._wide_baseline(inp)
        # a source camera behind the reference one at the nearest planes (t_z < 0): view 1 of batch element 0
        if V >= 2:
            inp.nghbr_poses[0, 1, 2, 3] = -0.05
        else:
            inp.nghbr_poses[0, 0, :3, 3] = torch.tensor([0.3, 0.05, -0.02])
        ref = inp.ref_feat.numpy() * np.float32(self.sr)
        src = inp.nghbr_feat.numpy() * np.float32(self.ss)
        if self.tiny:                          # some pixels at 2^-20 of the tensor's max: the split16 floor
            ref = np.where(rng.random((B, 1, H, W)) < 0.15, ref * np.float32(2.0 ** -20), ref).astype(np.float32)
            src = np.where(rng.random((V * B, 1, H, W)) < 0.15, src * np.float32(2.0 ** -20), src).astype(np.float32)
        self.inp, self.ref, self.src = inp, ref, src
        self.g = g = inp.to(cuda)
        self.ref_t, self.src_t = torch.from_numpy(ref).to(cuda), torch.from_numpy(src).to(cuda)
        intr = {k: v.to(cuda) for k, v in inp.cam_intrins.items()}
        self.cams = ops.pack_cameras(intr['intM'], g.R, g.t, inp.is_valid.to(cuda, torch.int32))
        self.rays = intr['unit_ray_array_2D'].contiguous()
        self.kappa = float(inp.thres)
        gmm = inp.ref_gmms.numpy()
        # VOLUME: batch element 0 behind the source cameras at hypothesis 0 and beyond the +-10 clamp at hypothesis 1
        mu, sg = gmm[:, :1], gmm[:, 1:]
        dv = mu * (0.2 + 3 * rng.random((B, D, H, W))) if self.depth == "random" else \
            mu + sg * np.linspace(-2.5, 2.5, D).reshape(1, D, 1, 1)
        dv = dv.astype(np.float32)
        dv[0, 0] = -dv[0, 0]
        if D > 1:
            dv[0, 1] *= np.float32(0.002)
        # GAUSS: k = -40 reaches behind the camera, k = -9.98 the clamp
        k = [-40.0, -9.98] + np.linspace(-2.5, 2.5, D - 2).astype(np.float32).tolist() if D > 2 else [-40.0] * D
        far = 10.0 if self.family == "scannet" else 80.0
        # the first D of at least 64 SID planes, so that even a few planes reach the clamp and the camera behind
        planes = magnet_b200.sid_planes(1e-3, far, max(D, 64)).reshape(-1)[:D].tolist()
        self.k = {"gauss": _ordered(k, self.order, rng), "planes": _ordered(planes, self.order, rng)}
        pl = np.asarray(self.k["planes"], np.float32).reshape(1, D, 1, 1)
        self.depth_np = {"volume": dv, "gauss": gauss_depths(gmm, self.k["gauss"], "direct"),
                         "planes": np.broadcast_to(pl, (B, D, H, W))}
        self.dv_t = torch.from_numpy(dv).to(cuda)
        self.dead = [b for b in range(B) if all((b, v) in self.invalid for v in range(V))]
        self._refs, self._src = {}, {}

    def reference(self, mode, cw, pos="direct"):
        key = (mode, cw, pos)
        if key not in self._refs:
            self._refs[key] = Reference(self.depth_np[mode], self.ref, self.src, self.inp.nghbr_gmms.numpy(),
                                        self.cams.cpu().numpy(), self.inp.cam_intrins['unit_ray_array_2D'].numpy(),
                                        self.kappa, pos=pos, consistency=cw, device=self.dev)
        return self._refs[key]

    def source(self, layout):
        """(source operand, reference split or None) of ``layout``, made once."""
        if layout not in self._src:
            self._src[layout] = hg.repack_source(LAYOUTS[layout], self.src_t, self.g.nghbr_gmms, self.ref_t)
        return self._src[layout]

    def blank(self, layout):
        """Zero operands of ``layout``'s shape, for calls that must be refused before anything is read (the repacks
        themselves refuse some widths)."""
        n, B, C, H, W = self.V * self.B, self.B, self.C, self.H, self.W
        z = lambda *s: torch.zeros(s, device=self.dev)
        if layout == "split16":
            nb = lambda N: torch.zeros(ops.packed_bytes(_lib.SRC_SPLIT16, N, H, W), device=self.dev, dtype=torch.uint8)
            return nb(n), nb(B)
        return {"nchw": z(n, C, H, W), "tiled32": z(n, H, (W + 31) // 32, C // 4, 32, 4),
                "pixc": z(n, H, W, C + 4)}[layout], None

    def depth_kw(self, mode):
        if mode == "volume":
            return dict(d_volume=self.dv_t)
        if mode == "gauss":
            return dict(ref_gmm=self.g.ref_gmms, k=self.k["gauss"])
        return dict(k=self.k["planes"], planes=True)

    def forward(self, variant, layout, mode, cw, softmax=False, blank=False):
        src, rs = self.blank(layout) if blank else self.source(layout)
        out = ops.cost_volume(self.ref_t, src, self.rays, self.cams, V=self.V, src_layout=LAYOUTS[layout],
                              consistency=cw, src_gmm=self.g.nghbr_gmms, kappa=self.kappa, softmax=softmax,
                              variant=VARIANTS[variant], ref_split=rs, **self.depth_kw(mode))
        torch.cuda.synchronize()
        return out

    def reach(self, mode):
        keys = ["tap_outside"]
        if self.D > 1:
            keys += ["clamped", "behind"]
        elif mode != "planes":
            keys += ["behind"]
        return keys


_CASES = {}


def _case(name, cuda):
    if name not in _CASES:
        _CASES[name] = FwdCase(name, cuda)
    return _CASES[name]


def _check_scores(got, rf, what, pos_err, floor):
    """The volume element by element; prints the worst |err| / (u bound + floor) and the clean flips."""
    got = gf._np(got)
    assert np.isfinite(got).all(), f"{what}: non-finite output"
    want, bound = rf.forward(pos_err)[:2]
    tol = gf.C_TOL * U * bound + floor
    bad, rejected = gf._fwd_bad(got, rf, pos_err, floor)
    err = np.abs(got - want)
    ratio = float(np.max(np.where(tol > 0, err / np.where(tol > 0, tol, 1.0), 0.0))) * gf.C_TOL
    print(f"{what}: max |err| / (u bound + floor) = {ratio:.3g} (beyond c = {gf.C_TOL:g} only for flips), "
          f"{int(bad.sum())} clean flips of {bad.size}")
    if rejected.any():
        i = np.unravel_index(np.argmax(np.where(rejected, err / np.maximum(tol, 1e-300), 0)), got.shape)
        raise AssertionError(f"{what}: {int(rejected.sum())} of {got.size} elements beyond c u bound and not a clean "
                             f"flip; worst at {i}: got {got[i]!r}, want {want[i]!r}, tol {tol[i]!r}")


def _check_probs(got, rf, what, pos_err, floor):
    """Softmax probabilities against the float64 softmax of the reference scores, with the bound
    p (tol_s + sum_j p tol_s) + c u p that test_f_volume_against_float64 uses."""
    score, score_b = rf.forward(pos_err)[:2]
    tol_s = gf.C_TOL * U * score_b + floor
    e = np.exp(score - score.max(1, keepdims=True))
    prob = e / e.sum(1, keepdims=True)
    dprob = prob * (tol_s + (prob * tol_s).sum(1, keepdims=True)) + gf.C_TOL * U * prob
    got = gf._np(got)
    assert np.isfinite(got).all(), f"{what}: non-finite output"
    bad = np.abs(got - prob) > dprob
    print(f"{what}: max |err| / bound = {float(np.max(np.abs(got - prob) / np.maximum(dprob, 1e-300))):.3g}")
    assert not bad.any(), (what, int(bad.sum()))


def _run_matrix(cs, mode, cw):
    rf = cs.reference(mode, cw)
    reached = {k: bool(rf.reached[k].any()) for k in cs.reach(mode)}
    assert all(reached.values()), (cs.name, mode, reached)
    ran = []
    runs = [(v, l) for v, l in fc.CANDIDATES]
    if cs.auto:                        # AUTO on the layout route() picks for these sizes
        layout = {LAYOUTS[k]: k for k in LAYOUTS}[hg.route(cs.C, cs.V, cs.D, _lib.VARIANT_AUTO, DEPTH_MODES[mode],
                                                          torch.float32, torch.float32)[0]]
        runs.append(("auto", layout))
    for variant, layout in runs:
        what = f"{cs.name} {mode} cw={int(cw)} {variant}/{layout}"
        if variant != "auto" and not fc.accepts(variant, layout, cs.C, cs.V, mode):
            with pytest.raises(_lib.MagnetError):
                cs.forward(variant, layout, mode, cw, blank=True)
            continue
        ran.append(variant)
        pos_err = variant != "direct"
        floor = gf._mma_fwd_floor(cs) if variant == "mma" else 0.0
        got = cs.forward(variant, layout, mode, cw)
        _check_scores(got, rf, what, pos_err, floor)
        for b in cs.dead:
            assert bool((got[b] == 0).all()), (what, "batch element without a valid view", b)
        if not cw:
            prob = cs.forward(variant, layout, mode, cw, softmax=True)
            _check_probs(prob, rf, f"{what} softmax", pos_err, floor)
            for b in cs.dead:
                assert bool((prob[b] == np.float32(1.0) / np.float32(cs.D)).all()), (what, "softmax not uniform", b)
    assert "direct" in ran, ran


@pytest.mark.parametrize("name", list(fc.CASES))
def test_forward_matrix_against_float64(cuda, name):
    """Every kernel that takes the case, in every depth mode and consistency setting of the case, against one float64
    reference per (mode, consistency); every other (variant, layout) pair raises MagnetError."""
    cs = _case(name, cuda)
    for mode, cw in cs.runs:
        _run_matrix(cs, mode, cw)


def test_consistency_with_softmax_is_refused(cuda):
    cs = _case("c16_d33_v3", cuda)
    with pytest.raises(_lib.MagnetError):
        cs.forward("direct", "nchw", "planes", True, softmax=True)


def test_sixteen_views_tensor_core_backwards(cuda):
    """All 16 staged cameras, and in batch element 1 only the 16th: the CW backward (feature gradients on the tensor
    cores from the split buffers, depth gradient with the tensor-core mask) and the F backward on the tensor cores,
    against the float64 reference on project() positions.  The upstream gradient is zeroed where a mask margin, a cell
    edge or the projection bound makes the reference ambiguous (as in test_gpu_grad_f64.py)."""
    cs = _case("v16", cuda)
    V, rng = cs.V, np.random.default_rng(16)
    sp, rs = cs.source("split16")
    for mode, cw in (("volume", True), ("planes", False)):
        rf = cs.reference(mode, cw, pos="mma")
        amb = rf.ambiguous()
        print(f"v16 {mode}: zeroed {amb.mean():.4f} of gout")
        assert amb.mean() <= 0.06, amb.mean()
        gout = np.where(amb, np.float32(0), gf._spanning_gout(rng, amb.shape)).astype(np.float32)
        gs = gout.astype(np.float64) / V
        want = rf.backward(gs)
        f_ref, f_src = gf._tc_floors(gs, cs.ref, cs.src, V)
        gt = torch.from_numpy(gout).to(cuda)
        if mode == "volume":
            r, s, d = ops.cost_volume_bwd(cs.ref_t, cs.src_t, cs.g.nghbr_gmms, cs.rays, cs.cams, gt, V=V,
                                          kappa=cs.kappa, d_volume=cs.dv_t, fwd_layout=_lib.SRC_SPLIT16,
                                          fwd_variant=_lib.VARIANT_MMA, ref_split=rs, src_split=sp)
            torch.cuda.synchronize()
            gf._close(d, want["d"], want["d_b"], "v16 CW depth (tensor-core mask)")
        else:
            r, s = ops.cost_volume_f_bwd(cs.ref_t, cs.src_t, cs.rays, cs.cams, cs.k["planes"], V, None, gt,
                                         softmax=False, ref_split=rs, src_split=sp)
            torch.cuda.synchronize()
        gf._close(r, want["ref"], want["ref_b"], f"v16 {mode} tensor-core ref", f_ref)
        gf._close(s, want["src"], want["src_b"], f"v16 {mode} tensor-core src", f_src)
        live = gf._np(s).reshape(V, cs.B, -1)[15, 1]
        assert np.abs(live).max() > 0, "view 15 of batch element 1 received no gradient"


def test_seventeen_views_refused_on_the_tensor_core_backwards(cuda):
    """V = 17: the split-buffer backwards refuse the call (tensor_core_gate); the forwards are refused in the matrix
    and AUTO is routed to a kernel checked there."""
    cs = _case("v17", cuda)
    sp, rs = ops.repack_split16(cs.src_t, cs.g.nghbr_gmms), ops.repack_split16(cs.ref_t)
    gt = torch.zeros(cs.B, cs.D, cs.H, cs.W, device=cuda)
    with pytest.raises(_lib.MagnetError):
        ops.cost_volume_bwd(cs.ref_t, cs.src_t, cs.g.nghbr_gmms, cs.rays, cs.cams, gt, V=cs.V, kappa=cs.kappa,
                            d_volume=cs.dv_t, fwd_layout=_lib.SRC_SPLIT16, fwd_variant=_lib.VARIANT_MMA,
                            ref_split=rs, src_split=sp)
    with pytest.raises(_lib.MagnetError):
        ops.cost_volume_f_bwd(cs.ref_t, cs.src_t, cs.rays, cs.cams, cs.k["planes"], cs.V, None, gt, softmax=False,
                              ref_split=rs, src_split=sp)


# ---------------------------------------------------------------------------------------------------------------------
# The check has teeth: outputs that pass, changed in Python, must be rejected where the change exceeds the tolerance
# and nowhere else.

def _rejects_exactly(got, mutated, region, delta, rf, pos_err, floor, what, vmargin=None):
    want, bound = rf.forward(pos_err)[:2]
    tol = gf.C_TOL * U * bound + floor
    assert not gf._fwd_bad(got, rf, pos_err, floor)[1].any(), what
    musts = region & (np.abs(delta) > tol)
    if vmargin is not None:
        musts &= vmargin > 1e-3
    rejected = gf._fwd_bad(mutated, rf, pos_err, floor)[1]
    print(f"{what}: {int(rejected.sum())} rejected, {int(musts.sum())} of the {int(region.sum())} changed elements "
          f"must be")
    assert musts.any() and rejected[musts].all() and not (rejected & ~region).any(), what
    return musts


def test_gate_rejects_mutations(cuda):
    # (a) view 15's term removed from one 8x8 tile of the V = 16 TMA output (consistency on: where view 15 is outside
    # the mask this adds a spurious term instead)
    cs = _case("v16", cuda)
    rf = cs.reference("volume", True)
    _, _, terms, vmargin = rf.forward(True)
    got = gf._np(cs.forward("tma", "pixc", "volume", True))
    tile = np.zeros(got.shape, bool)
    tile[0, :, 0:8, 8:16] = True
    delta = np.where(tile, -terms[15], 0.0)
    _rejects_exactly(got, got + delta, tile, delta, rf, True, 0.0, "v16 TMA without view 15 on one tile",
                     vmargin=vmargin[15])
    # (b) hypotheses 63 and 64 swapped in the D = 65 CELLS output: 64 is the last, partial 32-hypothesis chunk
    cs = _case("c16_d65_v4", cuda)
    rf = cs.reference("volume", False)
    got = gf._np(cs.forward("cells", "tiled32", "volume", False))
    mutated = got.copy()
    mutated[0, [63, 64]] = got[0, [64, 63]]
    region = np.zeros(got.shape, bool)
    region[0, [63, 64]] = True
    _rejects_exactly(got, mutated, region, mutated - got, rf, True, 0.0, "c16_d65 CELLS hypotheses 63 / 64 swapped")
    # (c) the ragged last column of a CW-off MMA output (W = 21: one column in the last 8-pixel tile) scaled.  The
    # position-error term of project() grows with |ix| (DESIGN §3.1): at x = 20 a relative error of 2^-12 stays inside
    # the bound everywhere, 2^-5 exceeds it on most of the column
    cs = _case("c64_d31", cuda)
    rf = cs.reference("volume", False)
    floor = gf._mma_fwd_floor(cs)
    got = gf._np(cs.forward("mma", "split16", "volume", False))
    col = np.zeros(got.shape, bool)
    col[:, :, :, -1] = True
    mutated = np.where(col, got * (1 + 2.0 ** -5), got)
    musts = _rejects_exactly(got, mutated, col, mutated - got, rf, True, floor, "c64_d31 MMA last column x (1 + 2^-5)")
    live = col & (rf.forward(True)[1] > 0)
    print(f"scaled column: beyond the tolerance on {musts[live].mean():.3f} of its elements")
    assert musts[live].mean() > 0.5
