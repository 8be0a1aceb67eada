"""Shared helpers for the parity tests (oracle = checker; nothing here is product code)."""
import ast
import hashlib
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

# Parity gate (BASELINE.md §4, SURVEY §7 hard part 2): fp32, 1e-4 relative to the volume's max norm
# on every element whose consistency mask agrees; elements that differ more must sit on the hard
# '<' threshold (relative distance of |z-mu~| to kappa*sigma~ below MARGIN_TOL in the oracle) and
# their fraction is bounded.
REL_TOL = 1e-4
# Calibration (cw_cfg1, random depth): the reference's own fp32 result vs an fp64 evaluation of the same
# formulas flips 7 / 327 680 elements (2.1e-5), with relative threshold margins up to 1.5e-5.
MARGIN_TOL = 1e-4
FLIP_BUDGET = 5e-5


def input_digest(inp) -> str:
    """sha256 of the seeded inputs a golden case was generated from (tests/golden/make_golden.py)."""
    h = hashlib.sha256()
    for tsr in (inp.ref_feat, inp.nghbr_feat, inp.ref_gmms, inp.nghbr_gmms, inp.nghbr_poses, inp.is_valid,
                inp.cam_intrins['intM'], inp.cam_intrins['unit_ray_array_2D'], inp.k):
        h.update(np.ascontiguousarray(tsr.numpy()).tobytes())
    return h.hexdigest()


def load_golden(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"), allow_pickle=False)
    kw = ast.literal_eval(str(z["kwargs"])) if "kwargs" in z.files else None
    return z, kw


def golden_inputs(name):
    """Rebuild the seeded inputs of a golden case and verify them against the stored digest."""
    from magnet_b200.synthetic import make_inputs
    z, kw = load_golden(name)
    inp = make_inputs(**kw)
    assert input_digest(inp) == str(z["digest"]), "synthetic generator drifted from the golden fixture"
    return z, inp


def oracle_cw(inp, d_volume, dtype=np.float32, return_margin=False):
    from oracle import magnet_oracle as mo
    return mo.cost_volume_cw(np.asarray(d_volume), inp.ref_feat.numpy(), inp.nghbr_feat.numpy(),
                             inp.nghbr_gmms.numpy(), inp.R.numpy(), inp.t.numpy(), inp.is_valid.numpy(),
                             inp.cam_intrins['intM'].numpy(), inp.cam_intrins['unit_ray_array_2D'].numpy(),
                             inp.thres, dtype=dtype, return_margin=return_margin)


def compare_volume(got, want, margin=None, rel=REL_TOL, flip_budget=FLIP_BUDGET, what=""):
    """Norm-wise comparison with consistency-mask flip accounting.  Returns a small report dict."""
    got = np.asarray(got, dtype=np.float64)
    want = np.asarray(want, dtype=np.float64)
    assert got.shape == want.shape, (got.shape, want.shape)
    assert np.isfinite(got).all(), f"{what}: non-finite output"
    scale = max(np.abs(want).max(), 1e-30)
    diff = np.abs(got - want)
    bad = diff > rel * scale
    n_bad = int(bad.sum())
    rep = dict(scale=float(scale), max_rel=float(diff.max() / scale), n_bad=n_bad, n=int(got.size),
               max_rel_agree=float(np.where(bad, 0.0, diff).max() / scale))
    if n_bad:
        assert margin is not None, f"{what}: {n_bad} elements beyond {rel:g} rel and no flip margin given: {rep}"
        near = np.asarray(margin)[bad] <= MARGIN_TOL
        rep["n_flip"] = int(near.sum())
        assert near.all(), (f"{what}: {int((~near).sum())} elements differ by more than {rel:g}*max and are NOT "
                            f"near the consistency threshold: {rep}")
        assert n_bad <= max(1, flip_budget * got.size), f"{what}: flip budget exceeded: {rep}"
    return rep
