"""Both cost volumes and every gradient their backward kernels write, element by element, against the float64
reference of tests/cw_grad_ref.py (gathers and scatters in torch float64 on the test's GPU), from toy sizes up to the
production shapes of synthetic.CONFIGS, BASELINE.json's stress points and the F-Net training shapes.

Tolerance: |got - ref| <= c u bound (+ floor on tensor-core outputs), u = 2^-24, c = C_TOL = 32, where bound is the
same sum as the output with the absolute value of every factor (plus, on positions from project(), the position-error
term of DESIGN §3.1).  Every output is a sum of products of at most three rounded factors (score gradient, bilinear
weight, feature; 1-3 u each) accumulated in fp32 chains: the channel dot products (<= 16 terms per lane, a 2-step quad
butterfly; <= 64 in the tensor-core accumulator), the tap coefficients G_t over the hypotheses of one cell, and grad_ref /
grad_d / (mu, sigma) over the cells and hypotheses of all views (n <= 4 D V terms).  The worst case of an n-term chain is
n u sum|terms|, but the terms here carry independent random signs, so the partial sums grow like sqrt(k) and the
rounding errors add in quadrature: the error is about u sum|terms| whatever n, and c = 32 leaves a wide margin (the
observed ratio is printed per output).  Tensor-core outputs add the documented floor of DESIGN §4, 2^-39 x the work
item's g bound (max over the 8x8 tile of sum_j |g|) x max|feature|, times c.

Ambiguity is removed by construction, never budgeted: every case zeroes the upstream gradient at each (b, j, p) whose
float64 mask margin is <= 1e-3, whose position is within 1e-3 px of a cell edge, or whose projection amplification A
exceeds the tensor-core kernel's fallback limit.  A zero g removes the hypothesis from all three gradients, whichever
side the kernel chose, so every gradient element is compared.  The forward cannot be zeroed: an element beyond the
tolerance must be a clean flip (the reference with exactly one near-threshold view's term added or removed)."""
import numpy as np
import pytest
import torch

import magnet_b200
from magnet_b200 import _lib, ops
from magnet_b200.homography import plane_sweep_f
from magnet_b200.synthetic import CONFIGS, make_inputs
from tests.cw_grad_ref import U, Reference, gauss_chain, gauss_depths, softmax_score_grad

pytestmark = pytest.mark.gpu

C_TOL = 32.0
FLOOR = 2.0 ** -39
FWD_VARIANTS = {"direct": _lib.VARIANT_DIRECT, "cells": _lib.VARIANT_CELLS, "tma": _lib.VARIANT_TMA,
                "mma": _lib.VARIANT_MMA}


def _np(x):
    return x.detach().double().cpu().numpy()


def _beyond(got, want, bound, floor=0.0):
    """Mask of the elements beyond c u bound + floor."""
    return np.abs(got - want) > C_TOL * U * bound + floor


def _close(got, want, bound, what, floor=0.0):
    got = _np(got) if isinstance(got, torch.Tensor) else np.asarray(got, np.float64)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    assert np.isfinite(got).all(), f"{what}: non-finite output"
    tol = C_TOL * U * bound + floor
    err = np.abs(got - want)
    bad = _beyond(got, want, bound, floor)
    ratio = float(np.max(np.where(tol > 0, err / np.where(tol > 0, tol, 1.0), 0.0))) * C_TOL
    print(f"{what}: max |err| / (u bound + floor) = {ratio:.3g}")
    if bad.any():
        i = np.unravel_index(np.argmax(np.where(bad, err / np.maximum(tol, 1e-300), 0)), bad.shape)
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.size} elements beyond c u bound; worst at {i}: got "
                             f"{got[i]!r}, want {want[i]!r}, tol {tol[i]!r}")


def _fwd_bad(got, rf, pos_err=None, floor=0.0):
    """(beyond, rejected): the volume's elements beyond the tolerance, and those of them that are not a clean flip of
    one view whose float64 margin is <= 1e-3."""
    want, bound, terms, vmargin = rf.forward(pos_err)
    tol = C_TOL * U * bound + floor
    bad = _beyond(got, want, bound, floor)
    clean = np.zeros_like(bad)
    for v in range(terms.shape[0]):
        for sign in (1.0, -1.0):
            clean |= (vmargin[v] <= 1e-3) & (np.abs(got - want - sign * terms[v]) <= tol)
    return bad, bad & ~clean


def _close_fwd(got, rf, what, pos_err=None, floor=0.0):
    """The volume, element by element; an element beyond the tolerance must be a clean flip of one view whose float64
    margin is <= 1e-3."""
    got = _np(got)
    assert np.isfinite(got).all(), f"{what}: non-finite output"
    bad, rejected = _fwd_bad(got, rf, pos_err, floor)
    print(f"{what}: {int(bad.sum())} clean flips of {bad.size}")
    if rejected.any():
        want, bound = rf.forward(pos_err)[:2]
        tol = C_TOL * U * bound + floor
        raise AssertionError((what, int(rejected.sum()), float(np.max(np.abs(got - want)[rejected] / tol[rejected]))))


def _tile_gbound(gs):
    """(B,D,H,W) score gradient -> (B,H,W): max over the pixel's 8x8 tile of sum_j |g| (the tensor-core item scale)."""
    s = np.abs(gs).sum(1)
    B, H, W = s.shape
    Hp, Wp = -(-H // 8) * 8, -(-W // 8) * 8
    pad = np.zeros((B, Hp, Wp))
    pad[:, :H, :W] = s
    t = pad.reshape(B, Hp // 8, 8, Wp // 8, 8).max(axis=(2, 4))
    return np.repeat(np.repeat(t, 8, 1), 8, 2)[:, :H, :W], t.reshape(B, -1).sum(1)


def _tc_floors(gs, ref, src, V):
    """Floors of the tensor-core feature gradients: grad_ref per pixel from its tile's g bound and max|src|, grad_src
    per (view, batch element) from the sum of the element's tile bounds and max|ref|."""
    tile, total = _tile_gbound(gs)
    B = gs.shape[0]
    f_ref = C_TOL * FLOOR * tile[:, None] * np.abs(src).max()
    f_src = C_TOL * FLOOR * np.abs(ref).max() * np.tile(total, V).reshape(V * B, 1, 1, 1)
    return f_ref, f_src


# ---------------------------------------------------------------------------------------------------------------------
# CW cases.  path: "direct" (est_costvolume_CW, variant DIRECT), "auto" (AUTO with D < 32 or C != 64: DIRECT forward,
# CUDA-core backward), "tc" (AUTO, C = 64, D >= 32: tensor-core forward and feature gradients, CUDA-core depth gradient
# with the tensor-core mask; plus ops.cost_volume_bwd without split buffers), "nocw" (ops.cost_volume_bwd with
# consistency off).  mode "gauss" runs MatchingPlan.cost with the Gaussian requiring grad.
CASES = {
    # DIRECT path, every CPL instantiation and both sides of each boundary; widths that are not multiples of 4
    "c1": dict(C=1, B=2, V=2, H=9, W=13, D=5, path="direct"),
    "c2_h1": dict(C=2, B=1, V=3, H=1, W=37, D=8, path="direct", depth="random"),
    # W = 1: every sample sits near the cell edge x = 0 (the ray through the single pixel column), so more is zeroed
    "c3_w1": dict(C=3, B=2, V=2, H=29, W=1, D=6, path="auto", max_zeroed=0.1),
    "c4_v1": dict(C=4, B=3, V=1, H=7, W=10, D=31, path="auto", invalid=[(2, 0)]),
    "c5_zero_g": dict(C=5, B=2, V=4, H=12, W=17, D=5, path="direct", depth="random", gout="zero"),
    "c7_v6": dict(C=7, B=1, V=6, H=10, W=14, D=33, path="direct"),
    "c8_scales": dict(C=8, B=2, V=3, H=11, W=15, D=8, path="auto", sr=1e-3, ss=1e3),
    "c9": dict(C=9, B=2, V=2, H=8, W=11, D=65, path="direct", depth="random"),
    "c15_d1": dict(C=15, B=1, V=5, H=13, W=9, D=1, path="direct"),
    "c16_scales": dict(C=16, B=2, V=2, H=12, W=20, D=16, path="auto", sr=1e3, ss=1e-3),
    "c17_dead_b": dict(C=17, B=2, V=3, H=9, W=35, D=5, path="direct", depth="random",
                       invalid=[(1, 0), (1, 1), (1, 2)]),
    "c24": dict(C=24, B=1, V=4, H=15, W=15, D=12, path="auto"),
    "c31_tiny": dict(C=31, B=2, V=2, H=6, W=33, D=7, path="direct", tiny=True),
    "c32_d256": dict(C=32, B=1, V=3, H=5, W=9, D=256, path="direct", depth="random"),
    "c33": dict(C=33, B=2, V=2, H=10, W=13, D=20, path="auto"),
    "c40_d64": dict(C=40, B=1, V=2, H=9, W=12, D=64, path="direct"),
    "c48_wide": dict(C=48, B=2, V=3, H=13, W=21, D=6, path="auto", trans=0.6),
    "c63": dict(C=63, B=1, V=2, H=11, W=15, D=9, path="direct", depth="random"),
    "c64_d5": dict(C=64, B=2, V=2, H=12, W=16, D=5, path="auto"),
    # tensor-core path (C = 64, D >= 32)
    "tc_d32": dict(C=64, B=2, V=3, H=16, W=24, D=32, path="tc"),
    "tc_d65_scales": dict(C=64, B=1, V=4, H=13, W=21, D=65, path="tc", depth="random", sr=1e-3, ss=1e3),
    "tc_d64_tiny_dead_b": dict(C=64, B=2, V=2, H=12, W=20, D=64, path="tc", tiny=True, invalid=[(1, 0), (1, 1)]),
    "tc_d33_v6": dict(C=64, B=2, V=6, H=9, W=35, D=33, path="tc", sr=1e3, ss=1e-3),
    "tc_d256": dict(C=64, B=1, V=2, H=10, W=14, D=256, path="tc", depth="random"),
    # Gaussian depths (MatchingPlan.cost)
    "gauss_c64_tc": dict(C=64, B=2, V=3, H=12, W=16, D=40, path="tc", mode="gauss"),
    "gauss_c13": dict(C=13, B=2, V=2, H=10, W=14, D=6, path="direct", mode="gauss"),
    "gauss_c64_d5": dict(C=64, B=3, V=2, H=9, W=15, D=5, path="auto", mode="gauss", invalid=[(1, 0), (1, 1)]),
    # consistency off
    "nocw_c8": dict(C=8, B=2, V=3, H=10, W=14, D=9, path="nocw"),
    "nocw_c64_mma_mask": dict(C=64, B=1, V=3, H=12, W=16, D=32, path="nocw", mask="mma"),
    # production shapes (synthetic.CONFIGS): each persistent CTA of the tensor-core kernels takes at least `per_cta` work
    # items, the geometry reduction runs its block loop, the windows span every width of DESIGN §3.1
    "cfg2_gauss": dict(cfg="cfg2", path="tc", mode="gauss", invalid=[(2, 1), (1, 0), (1, 1), (1, 2), (1, 3)],
                       per_cta=4, max_zeroed=0.02),
    "cfg3_volume": dict(cfg="cfg3", path="tc", per_cta=4, max_zeroed=0.02),
    # BASELINE.json's stress points: V = 8, and D = 256 (4 hypothesis chunks per tile); B = 2 gives 600 tiles, two or
    # more per CTA
    "stress_v8_d256": dict(cfg="cfg2", B=2, V=8, D=256, path="tc", depth="random", per_cta=2, max_zeroed=0.05),
    "stress_v2_d32": dict(cfg="cfg2", B=2, V=2, D=32, path="tc", per_cta=2, max_zeroed=0.015),
    # one partial 32-hypothesis chunk, ragged tiles on both axes, feature scales far apart, pixels at the split16 floor
    "ragged_many_items": dict(C=64, B=6, V=5, H=117, W=157, D=96, path="tc", depth="random", sr=1e-3, ss=1e3,
                              tiny=True, per_cta=4, max_zeroed=0.035),
    # the shipped N_s = 5 point: DIRECT forward, CUDA-core backward
    "cfg2_ship_d5": dict(cfg="ship", B=8, path="auto", max_zeroed=0.025),
}


def _spanning_gout(rng, shape):
    """Upstream gradient spanning 1e6 element to element, times a ramp over the 8-pixel tile columns (rows when the
    image is one tile wide) from 1 down to 1e-6: the tensor-core work items then have g bounds far apart, so an error
    on the small items is not hidden by a floor taken from the large ones."""
    B, D, H, W = shape
    g = rng.standard_normal(shape) * 10.0 ** (6 * rng.random(shape) - 3)
    tx = (np.arange(W) // 8) / max(1, (W - 1) // 8)
    ty = (np.arange(H) // 8) / max(1, (H - 1) // 8)
    ramp = 10.0 ** (-6 * (tx[None, :] if W > 8 else ty[:, None] * np.ones((1, W))))
    return (g * ramp).astype(np.float32)


def _wide_baseline(inp):
    """View 0 of batch element 0 moves sideways (t_z small against t_x): a hypothesis at a few mm projects beyond the
    +-10 clamp while z stays far from 0 (A < 1)."""
    inp.nghbr_poses[0, 0, :3, 3] = torch.tensor([0.3, 0.05, 0.01])


def _check_persistent(B, V, D, H, W, per_cta, dev):
    """The persistent tensor-core kernels hand each CTA at least ``per_cta`` work items: the forward's (batch element,
    8x8 tile, 64-hypothesis chunk) items against the grid it launches, the backward's (batch element, tile) items
    against its two CTAs per SM.  So the state carried from one item to the next is compared too."""
    tiles = B * -(-H // 8) * -(-W // 8)
    grid = ops.cost_launch_info(B, V, D, 64, H, W, variant=_lib.VARIANT_MMA)[0]
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    print(f"work items per CTA: forward {tiles * -(-D // 64) / grid:.1f}, backward {tiles / (2 * sms):.1f}")
    assert tiles * -(-D // 64) >= per_cta * grid and tiles >= per_cta * 2 * sms, (tiles, D, grid, sms)


class Case:
    def __init__(self, name, cuda):
        spec = dict(depth="smooth", invalid=[], sr=1.0, ss=1.0, tiny=False, gout="span", mode="volume", trans=None,
                    mask=None, max_zeroed=0.06, family="scannet", per_cta=None)
        spec.update(CONFIGS.get(CASES[name].get("cfg"), {}))
        spec.update(CASES[name])
        self.__dict__.update(spec)
        self.name = name
        C, B, V, H, W, D = self.C, self.B, self.V, self.H, self.W, self.D
        seed = sum(map(ord, name))
        depth_kind = "smooth" if self.mode == "gauss" else self.depth
        inp = make_inputs(B=B, V=V, D=D, H=H, W=W, C=C, seed=seed, depth=depth_kind, invalid=self.invalid,
                          trans=self.trans, family=self.family)
        _wide_baseline(inp)
        rng = np.random.default_rng(seed)
        ref = inp.ref_feat.numpy() * np.float32(self.sr)
        src = inp.nghbr_feat.numpy() * np.float32(self.ss)
        if self.tiny:                          # some pixels at 2^-20 of the tensor's max: the split16 floor
            ref = np.where(rng.random((B, 1, H, W)) < 0.15, ref * np.float32(2.0 ** -20), ref).astype(np.float32)
            src = np.where(rng.random((V * B, 1, H, W)) < 0.15, src * np.float32(2.0 ** -20), src).astype(np.float32)
        self.inp, self.ref, self.src = inp, ref, src
        gmm = inp.ref_gmms.numpy()
        if self.mode == "gauss":
            # sorted k: batch element 0 reaches behind the camera (k = -40) and the clamp (k = -9.98: d ~ 0.002 mu)
            self.k = [-40.0, -9.98] + np.linspace(-2.5, 2.5, D - 2).astype(np.float32).tolist() if D > 2 else [-40.0] * D
            self.depth_vol = gauss_depths(gmm, self.k, "direct")
        else:
            mu, sg = gmm[:, :1], gmm[:, 1:]
            if self.depth == "random":
                dv = mu * (0.2 + 3 * rng.random((B, D, H, W)))
            else:
                dv = mu + sg * np.linspace(-2.5, 2.5, D).reshape(1, D, 1, 1)
            dv = dv.astype(np.float32)
            dv[0, 0] = -dv[0, 0]                   # batch element 0: behind the source cameras ...
            if D > 1:
                dv[0, 1] *= np.float32(0.002)      # ... and so close that the sample leaves the +-10 clamp
            self.depth_vol = dv
        self.dev = cuda
        g = inp.to(cuda)
        self.g = g
        self.intr = {k: v.to(cuda) for k, v in inp.cam_intrins.items()}
        self.cams = ops.pack_cameras(self.intr['intM'], g.R, g.t, inp.is_valid.to(cuda, torch.int32))
        self.rays = self.intr['unit_ray_array_2D'].contiguous()
        tc = self.path == "tc" or self.mask == "mma"
        self.pos = "mma" if tc else "direct"
        self.rf = Reference(self.depth_vol, ref, src, inp.nghbr_gmms.numpy(), self.cams.cpu().numpy(),
                            inp.cam_intrins['unit_ray_array_2D'].numpy(), float(inp.thres), pos=self.pos,
                            consistency=self.path != "nocw", device=cuda)
        amb = self.rf.ambiguous()
        self.amb = amb
        if self.gout == "zero":
            gout = np.zeros(amb.shape, np.float32)
        else:
            gout = _spanning_gout(rng, amb.shape)
        self.gout = np.where(amb, np.float32(0), gout).astype(np.float32)
        self.gs = self.gout.astype(np.float64) / V
        self.want = self.rf.backward(self.gs)
        if self.mode == "gauss":
            self.want["gmm"], self.want["gmm_b"] = gauss_chain(self.want["d"], self.want["d_b"], self.k)
        self.floors = _tc_floors(self.gs, ref, src, V) if self.path == "tc" else (0.0, 0.0)

    def check_geometry(self):
        keep = ~self.amb
        print(f"{self.name}: zeroed {self.amb.mean():.4f} of gout")
        assert self.amb.mean() <= self.max_zeroed, self.amb.mean()
        reach = ["tap_outside", "behind"] + (["clamped"] if self.D > 1 else [])
        for k in reach:
            assert (self.rf.reached[k].reshape(keep.shape) & keep).any(), (self.name, k)
        if self.per_cta:
            _check_persistent(self.B, self.V, self.D, self.H, self.W, self.per_cta, self.dev)

    def leaves(self, need=("d", "ref", "src"), ref=None):
        d = torch.from_numpy(self.depth_vol if self.mode == "volume" else self.inp.ref_gmms.numpy()).to(self.dev)
        ref = self.ref if ref is None else ref
        return (d.clone().requires_grad_("d" in need), torch.from_numpy(ref).to(self.dev).requires_grad_("ref" in need),
                torch.from_numpy(self.src).to(self.dev).requires_grad_("src" in need))

    def run(self, need=("d", "ref", "src"), variant=None, ref=None):
        """Forward + backward through the public entry point, optionally on other reference features; returns (out,
        grad_d, grad_ref, grad_src)."""
        d, ref, src = self.leaves(need, ref)
        g, inp = self.g, self.inp
        if variant is None:
            variant = _lib.VARIANT_DIRECT if self.path == "direct" else _lib.VARIANT_AUTO
        if self.mode == "gauss":
            plan = magnet_b200.MatchingPlan(ref, src, g.nghbr_gmms, g.nghbr_poses, inp.is_valid, inp.cam_intrins,
                                            thres=inp.thres)
            out = plan.cost(d, self.k, variant=variant)
        else:
            out = magnet_b200.est_costvolume_CW(d, ref, src, g.ref_gmms, g.nghbr_gmms, g.R, g.t, inp.is_valid,
                                                inp.cam_intrins, inp.thres, variant=variant)
        (out * torch.from_numpy(self.gout).to(self.dev)).sum().backward()
        torch.cuda.synchronize()
        return out.detach(), d.grad, ref.grad, src.grad

    def forward_variant(self, name, src=None):
        """No-grad forward on one kernel variant (optionally on other source features), or None when the variant does
        not take this call."""
        g, inp = self.g, self.inp
        src = self.src if src is None else src
        ref, src = torch.from_numpy(self.ref).to(self.dev), torch.from_numpy(src).to(self.dev)
        try:
            with torch.no_grad():
                if self.mode == "gauss":
                    plan = magnet_b200.MatchingPlan(ref, src, g.nghbr_gmms, g.nghbr_poses, inp.is_valid,
                                                    inp.cam_intrins, thres=inp.thres)
                    out = plan.cost(g.ref_gmms, self.k, variant=FWD_VARIANTS[name])
                else:
                    out = magnet_b200.est_costvolume_CW(torch.from_numpy(self.depth_vol).to(self.dev), ref, src,
                                                        g.ref_gmms, g.nghbr_gmms, g.R, g.t, inp.is_valid,
                                                        inp.cam_intrins, inp.thres, variant=FWD_VARIANTS[name])
        except _lib.MagnetError:
            return None
        torch.cuda.synchronize()
        return out

    def check_grads(self, gd, gr, gs, what, tc_features):
        w = self.want
        f_ref, f_src = self.floors if tc_features else (0.0, 0.0)
        if gd is not None:
            if self.mode == "gauss":
                _close(gd, w["gmm"], w["gmm_b"], f"{what} (mu, sigma)")
            else:
                _close(gd, w["d"], w["d_b"], f"{what} depth")
        if gr is not None:
            _close(gr, w["ref"], w["ref_b"], f"{what} ref", f_ref)
        if gs is not None:
            _close(gs, w["src"], w["src_b"], f"{what} src", f_src)


_CASES = {}


def _case(name, cuda):
    """The reference of a case is computed once per session (the CPU side dominates)."""
    if name not in _CASES:
        _CASES[name] = Case(name, cuda)
    return _CASES[name]


@pytest.mark.parametrize("name", sorted(n for n in CASES if CASES[n]["path"] != "nocw"))
def test_cw_gradients_against_float64(cuda, name):
    cs = _case(name, cuda)
    cs.check_geometry()
    out, gd, gr, gs = cs.run()
    tc = cs.path == "tc"
    cs.check_grads(gd, gr, gs, name, tc_features=tc)
    _close_fwd(out, cs.rf, f"{name} forward (differentiable)", floor=_mma_fwd_floor(cs) if tc else 0.0)
    if tc:
        # the CUDA-core kernel computes every gradient with the tensor-core forward's mask (the cross-check path)
        kw = dict(V=cs.V, kappa=float(cs.inp.thres), fwd_layout=_lib.SRC_SPLIT16, fwd_variant=_lib.VARIANT_MMA)
        dep = (dict(ref_gmm=cs.g.ref_gmms, k=cs.k) if cs.mode == "gauss"
               else dict(d_volume=torch.from_numpy(cs.depth_vol).to(cuda)))
        r, s, d = ops.cost_volume_bwd(torch.from_numpy(cs.ref).to(cuda), torch.from_numpy(cs.src).to(cuda),
                                      cs.g.nghbr_gmms, cs.rays, cs.cams, torch.from_numpy(cs.gout).to(cuda), **kw, **dep)
        torch.cuda.synchronize()
        cs.check_grads(d, r, s, f"{name} CUDA-core, tensor-core mask", tc_features=False)


def _mma_fwd_floor(cs):
    """Forward on the fp16 hi/lo split: elements below 2^-18 of their tensor's max keep an absolute error of 2^-39 of
    it (DESIGN §3.1), summed over C channels and 4 taps."""
    return C_TOL * FLOOR * 4 * cs.C * float(np.abs(cs.ref).max()) * float(np.abs(cs.src).max())


@pytest.mark.parametrize("name", sorted(n for n in CASES if CASES[n]["path"] != "nocw"))
def test_cw_forward_variants_against_float64(cuda, name):
    """Every forward variant that takes the call, element by element (clean flips only)."""
    cs = _case(name, cuda)
    ran = []
    for v in FWD_VARIANTS:
        out = cs.forward_variant(v)
        if out is None:
            continue
        ran.append(v)
        pos_err = v != "direct" or cs.pos == "mma"
        _close_fwd(out, cs.rf, f"{name} forward {v}", pos_err=pos_err, floor=_mma_fwd_floor(cs) if v == "mma" else 0.0)
    assert "direct" in ran, ran


@pytest.mark.parametrize("name", sorted(n for n in CASES if CASES[n]["path"] == "nocw"))
def test_cw_without_consistency(cuda, name):
    cs = _case(name, cuda)
    cs.check_geometry()
    mma = cs.mask == "mma"
    ref, src = torch.from_numpy(cs.ref).to(cuda), torch.from_numpy(cs.src).to(cuda)
    dv = torch.from_numpy(cs.depth_vol).to(cuda)
    if mma:
        rs, sp = ops.repack_split16(ref), ops.repack_split16(src)
        out = ops.cost_volume(ref, sp, cs.rays, cs.cams, V=cs.V, src_layout=_lib.SRC_SPLIT16, consistency=False,
                              d_volume=dv, variant=_lib.VARIANT_MMA, ref_split=rs)
        fwd = dict(fwd_layout=_lib.SRC_SPLIT16, fwd_variant=_lib.VARIANT_MMA)
    else:
        out = ops.cost_volume(ref, src, cs.rays, cs.cams, V=cs.V, src_layout=_lib.SRC_NCHW, consistency=False,
                              d_volume=dv, variant=_lib.VARIANT_DIRECT)
        fwd = dict(fwd_layout=_lib.SRC_NCHW, fwd_variant=_lib.VARIANT_DIRECT)
    r, s, d = ops.cost_volume_bwd(ref, src, None, cs.rays, cs.cams, torch.from_numpy(cs.gout).to(cuda), V=cs.V,
                                  kappa=float(cs.inp.thres), consistency=False, d_volume=dv, **fwd)
    torch.cuda.synchronize()
    _close_fwd(out, cs.rf, f"{name} forward", floor=_mma_fwd_floor(cs) if mma else 0.0)
    cs.check_grads(d, r, s, name, tc_features=False)
    if mma:                                   # tensor-core feature gradients on the split buffers
        r2, s2, _ = ops.cost_volume_bwd(ref, src, None, cs.rays, cs.cams, torch.from_numpy(cs.gout).to(cuda), V=cs.V,
                                        kappa=float(cs.inp.thres), consistency=False, d_volume=dv, need_depth=False,
                                        ref_split=rs, src_split=sp, **fwd)
        torch.cuda.synchronize()
        f_ref, f_src = _tc_floors(cs.gs, cs.ref, cs.src, cs.V)
        _close(r2, cs.want["ref"], cs.want["ref_b"], f"{name} tensor-core ref", f_ref)
        _close(s2, cs.want["src"], cs.want["src_b"], f"{name} tensor-core src", f_src)


SUBSETS = [("d",), ("ref",), ("src",), ("d", "ref"), ("d", "src"), ("ref", "src")]


@pytest.mark.parametrize("name", ["c3_w1", "c8_scales", "c16_scales", "c24", "c64_d5", "tc_d32", "gauss_c13",
                                  "cfg2_gauss"])
def test_gradient_subsets(cuda, name):
    """Asking for fewer gradients changes none of the others.  The CUDA-core kernel's grad_ref and grad_d have one owner
    each and a fixed summation order: bit-identical to the run with all three.  grad_src (global atomics) and the
    tensor-core grad_ref (its coefficient matrix is summed with shared-memory atomics, so the rounding order varies from
    run to run) are held to the float64 bound instead."""
    cs = _case(name, cuda)
    tc = cs.path == "tc"
    _, gd_all, gr_all, _ = cs.run()
    for need in SUBSETS:
        _, gd, gr, gs = cs.run(need)
        for nm, got, full in (("d", gd, gd_all), ("ref", gr, gr_all)):
            if nm not in need:
                assert got is None
            elif nm == "ref" and tc:
                cs.check_grads(None, got, None, f"{name} subset {need}", tc_features=True)
            else:
                assert torch.equal(got, full), (name, need, nm)
        if "src" in need:
            cs.check_grads(None, None, gs, f"{name} subset {need}", tc_features=tc)
        else:
            assert gs is None


def _window_cells(rf):
    """Cells of the tensor-core window of every (batch element, 8x8 tile, 64-hypothesis chunk, valid view): the box of
    the float64 reference's cell origins plus the right / lower taps, cut into 8-cell segments (cost_mma.cu)."""
    x0, x1, y0, y1 = rf.origins                                   # (B, V, chunks, HW)
    B, V, nk = x0.shape[:3]
    H, W = rf.H, rf.W
    Hp, Wp = -(-H // 8) * 8, -(-W // 8) * 8

    def tile(a, red, fill):
        pad = np.full((B, V, nk, Hp, Wp), fill)
        pad[..., :H, :W] = a.reshape(B, V, nk, H, W)
        return red(pad.reshape(B, V, nk, Hp // 8, 8, Wp // 8, 8), axis=(4, 6))
    lx, hx, ly, hy = tile(x0, np.min, np.inf), tile(x1, np.max, -np.inf), tile(y0, np.min, np.inf), tile(y1, np.max, -np.inf)
    live = np.isfinite(lx)                                        # the valid views
    return (((hx - lx + 2 + 7) // 8) * (hy - ly + 2) * 8)[live]


def test_tensor_core_cases_reach_every_window_width(cuda):
    """Across the tensor-core CW cases the windows take all four shapes of DESIGN §3.1: warpgroup 1 idle (<= 128
    cells), n64 (129-192), n128 (193-256) and sub-windows (> 256)."""
    cells = np.concatenate([_window_cells(_case(n, cuda).rf) for n in sorted(CASES) if CASES[n]["path"] == "tc"])
    widths = {"<= 128": cells <= 128, "129-192": (cells > 128) & (cells <= 192),
              "193-256": (cells > 192) & (cells <= 256), "> 256": cells > 256}
    print({k: int(m.sum()) for k, m in widths.items()})
    assert all(m.any() for m in widths.values())


def test_gate_rejects_subtle_errors_at_production_scale(cuda):
    """At cfg2 the bounds sum over many more terms than at the small cases; they must still reject a forward on source
    maps rounded to fp16 (relative error 2^-11), a grad_src on a reference map rounded to bf16 (2^-8), and one view's
    term cost_v / V subtracted over the last work item handed out (the last 8x8 tile of the last batch element): where
    the view is in the mask that removes its term, elsewhere it adds a spurious one.  The gate must flag that tile and
    nothing else.

    The rounded inputs go through the kernels whose positions the reference reproduces exactly (the DIRECT forward,
    the CUDA-core backward with its mask): on project() positions the bound carries the position error
    (A + 8) u |ix + 0.5| |d cost / d ix|, at |ix| ~ 100 px some 2^-9 of the value, which a 2^-11 feature error hides in."""
    cs = _case("cfg2_gauss", cuda)
    V = cs.V
    rf = Reference(cs.depth_vol, cs.ref, cs.src, cs.inp.nghbr_gmms.numpy(), cs.cams.cpu().numpy(),
                   cs.inp.cam_intrins['unit_ray_array_2D'].numpy(), float(cs.inp.thres), pos="direct", device=cuda)
    amb = rf.ambiguous()
    assert not _fwd_bad(_np(cs.forward_variant("direct")), rf, pos_err=False)[1].any()
    src16 = cs.src.astype(np.float16).astype(np.float32)
    _, rejected = _fwd_bad(_np(cs.forward_variant("direct", src=src16)), rf, pos_err=False)
    live = ~amb & (rf.forward(False)[1] > 0)
    print(f"fp16 source maps: forward rejected at {rejected[live].mean():.3f} of the unambiguous elements")
    assert rejected[live].mean() > 0.5
    gout = np.where(amb, np.float32(0), cs.gout).astype(np.float32)
    want = rf.backward(gout.astype(np.float64) / V)
    ref16 = torch.from_numpy(cs.ref).bfloat16().float().numpy()
    for ref, rounded in ((cs.ref, False), (ref16, True)):
        _, gsrc, _ = ops.cost_volume_bwd(torch.from_numpy(ref).to(cuda), torch.from_numpy(cs.src).to(cuda),
                                         cs.g.nghbr_gmms, cs.rays, cs.cams, torch.from_numpy(gout).to(cuda), V=V,
                                         kappa=float(cs.inp.thres), fwd_layout=_lib.SRC_NCHW,
                                         fwd_variant=_lib.VARIANT_DIRECT, need_ref=False, need_depth=False,
                                         ref_gmm=cs.g.ref_gmms, k=cs.k)
        bad = _beyond(_np(gsrc), want["src"], want["src_b"])
        live = want["src_b"] > 0
        print(f"reference map rounded={rounded}: grad_src rejected at {bad[live].mean():.3f} of its elements")
        assert bad[live].mean() > 0.5 if rounded else not bad.any()
    # one view's term subtracted over one tile, on the tensor-core forward and its own reference
    floor = _mma_fwd_floor(cs)
    want, bound, terms, vmargin = cs.rf.forward()
    got = _np(cs.forward_variant("mma"))
    assert not _fwd_bad(got, cs.rf, floor=floor)[1].any()
    tile = np.zeros(got.shape, bool)
    tile[-1, :, -8:, -8:] = True
    tol = C_TOL * U * bound + floor
    # the view whose samples of the corner tile fall inside the image most often; an element must be rejected when
    # the subtracted term exceeds the tolerance and the view is not within 1e-3 of a mask flip
    musts = {v: tile & (np.abs(terms[v]) > tol) & (vmargin[v] > 1e-3) for v in range(cs.V) if (cs.B - 1, v) in cs.rf.valid}
    v = max(musts, key=lambda v: musts[v].sum())
    got[tile] -= terms[v][tile]
    _, rejected = _fwd_bad(got, cs.rf, floor=floor)
    print(f"view {v}'s term subtracted: {int(rejected.sum())} rejected, {int(musts[v].sum())} of the tile's "
          f"{int(tile.sum())} elements must be")
    assert musts[v].any() and rejected[musts[v]].all() and not (rejected & ~tile).any()


# ---------------------------------------------------------------------------------------------------------------------
# F volume

F_CASES = {
    "f8": dict(C=8, B=2, V=3, H=11, W=17, D=12),
    "f16": dict(C=16, B=1, V=4, H=13, W=9, D=7),
    "f32": dict(C=32, B=2, V=2, H=10, W=14, D=20),
    "f64": dict(C=64, B=1, V=3, H=12, W=16, D=9),
    "f64_tc_sid": dict(C=64, B=2, V=3, H=12, W=20, D=48, tc=True),
    # the F-Net training shapes (test_gpu_fnet.py): 80 SID planes from 1e-3 to the family's maximum depth
    "fnet_scannet": dict(C=64, B=2, V=4, H=120, W=160, D=80, tc=True, per_cta=2),
    "fnet_kitti": dict(C=64, B=4, V=2, H=88, W=304, D=80, tc=True, family="kitti", far=80.0, per_cta=4),
}


class FCase:
    def __init__(self, name, cuda):
        spec = dict(tc=False, family="scannet", far=10.0, per_cta=None)
        spec.update(F_CASES[name])
        self.__dict__.update(spec)
        self.name = name
        seed = sum(map(ord, name))
        inp = make_inputs(B=self.B, V=self.V, D=self.D, H=self.H, W=self.W, C=self.C, seed=seed, depth="smooth",
                          invalid=[(0, 1)], family=self.family)
        _wide_baseline(inp)
        self.inp, self.dev = inp, cuda
        if self.per_cta:
            _check_persistent(self.B, self.V, self.D, self.H, self.W, self.per_cta, cuda)
        if self.tc:                            # SID planes from 1e-3: a tile spreads along an epipolar line
            self.planes = magnet_b200.sid_planes(1e-3, self.far, self.D, device=cuda).reshape(1, -1, 1, 1)
        else:                                  # the first plane is close enough to reach the clamp
            self.planes = torch.tensor([0.002] + np.linspace(0.3, 8.0, self.D - 1).tolist(),
                                       device=cuda).reshape(1, -1, 1, 1)
        g = inp.to(cuda)
        self.g = g
        intr = {k: v.to(cuda) for k, v in inp.cam_intrins.items()}
        cams = ops.pack_cameras(intr['intM'], g.R, g.t, inp.is_valid.to(cuda, torch.int32))
        pl = np.float32(self.planes.reshape(-1).cpu().numpy())
        depth = np.broadcast_to(pl.reshape(1, -1, 1, 1), (self.B, self.D, self.H, self.W))
        self.rf = Reference(depth, inp.ref_feat.numpy(), inp.nghbr_feat.numpy(), None, cams.cpu().numpy(),
                            inp.cam_intrins['unit_ray_array_2D'].numpy(), 0.0, pos="mma", consistency=False, device=cuda)
        rng = np.random.default_rng(seed)
        self.gout = _spanning_gout(rng, (self.B, self.D, self.H, self.W))

    def run(self, softmax):
        g, inp = self.g, self.inp
        ref, src = g.ref_feat.clone().requires_grad_(True), g.nghbr_feat.clone().requires_grad_(True)
        if softmax and not self.tc:
            out = magnet_b200.est_costvolume_F(self.planes, ref, src, g.R, g.t, inp.is_valid, inp.cam_intrins)
        else:
            out = plane_sweep_f(self.planes, ref, src, g.R, g.t, inp.is_valid, inp.cam_intrins,
                                            softmax=softmax)
        (out * torch.from_numpy(self.gout).to(self.dev)).sum().backward()
        torch.cuda.synchronize()
        return out.detach(), ref.grad, src.grad


_FCASES = {}


@pytest.mark.parametrize("softmax", [True, False])
@pytest.mark.parametrize("name", sorted(F_CASES))
def test_f_volume_against_float64(cuda, name, softmax):
    """Scores / probabilities and both feature gradients of the F volume.  The backward's score gradient is restated
    from the kernel's own probabilities (the forward is checked separately), so the backward is held to its own
    bound."""
    if name not in _FCASES:
        _FCASES[name] = FCase(name, cuda)
    fc = _FCASES[name]
    assert fc.rf.reached["clamped"].any()
    out, gr, gs = fc.run(softmax)
    score, score_b, _, _ = fc.rf.forward()
    V = fc.V
    tol_s = C_TOL * U * score_b + (_mma_fwd_floor_f(fc) if fc.C == 64 and fc.D >= 32 else 0.0)
    if softmax:
        e = np.exp(score - score.max(1, keepdims=True))
        prob = e / e.sum(1, keepdims=True)
        dprob = prob * (tol_s + (prob * tol_s).sum(1, keepdims=True)) + C_TOL * U * prob
        got = _np(out)
        assert np.isfinite(got).all()
        bad = np.abs(got - prob) > dprob
        assert not bad.any(), (name, "prob", int(bad.sum()))
        gsc, gsc_b = softmax_score_grad(got, fc.gout, V)
    else:
        _close(out, score, (tol_s / (C_TOL * U)), f"{name} scores")
        gsc, gsc_b = fc.gout.astype(np.float64) / V, np.abs(fc.gout.astype(np.float64)) / V
    want = fc.rf.backward(gsc, gsc_b)
    tc = fc.tc                                   # plane_sweep_f: tensor-core backward after a tensor-core forward
    f_ref, f_src = _tc_floors(gsc_b, fc.inp.ref_feat.numpy(), fc.inp.nghbr_feat.numpy(), V) if tc else (0.0, 0.0)
    _close(gr, want["ref"], want["ref_b"], f"{name} softmax={softmax} ref", f_ref)
    _close(gs, want["src"], want["src_b"], f"{name} softmax={softmax} src", f_src)


def _mma_fwd_floor_f(fc):
    return C_TOL * FLOOR * 4 * fc.C * float(fc.inp.ref_feat.abs().max()) * float(fc.inp.nghbr_feat.abs().max())


@pytest.mark.parametrize("C_", [12, 20])
def test_f_backward_rejects_unsupported_width(cuda, C_):
    """The CUDA-core F backward takes C in {8, 16, 32, 64}: another width raises MagnetError and leaves no sticky CUDA
    error behind (the next valid call succeeds)."""
    inp = make_inputs(B=1, V=2, D=6, H=8, W=12, C=C_, seed=C_, depth="smooth")
    g = inp.to(cuda)
    planes = torch.linspace(0.5, 5.0, 6, device=cuda).reshape(1, -1, 1, 1)
    ref = g.ref_feat.clone().requires_grad_(True)
    out = magnet_b200.est_costvolume_F(planes, ref, g.nghbr_feat, g.R, g.t, inp.is_valid, inp.cam_intrins)
    with pytest.raises(_lib.MagnetError):
        out.sum().backward()
    inp8 = make_inputs(B=1, V=2, D=6, H=8, W=12, C=8, seed=1, depth="smooth")
    g8 = inp8.to(cuda)
    ref8 = g8.ref_feat.clone().requires_grad_(True)
    magnet_b200.est_costvolume_F(planes, ref8, g8.nghbr_feat, g8.R, g8.t, inp8.is_valid, inp8.cam_intrins).sum().backward()
    torch.cuda.synchronize()
    assert ref8.grad is not None and torch.isfinite(ref8.grad).all() and float(ref8.grad.abs().max()) > 0
