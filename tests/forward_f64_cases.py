"""The case table of tests/test_gpu_forward_f64.py and the rule that says which forward kernel takes which call.  Plain
Python, importable without a GPU or the built library, so that tests/test_forward_f64_cpu.py can check that the table
reaches every instance of the four forward kernels.

Each case is chosen for an edge of the kernels' tiling (cost_tma.cu: 16x4-pixel tiles, 64-hypothesis chunks;
cost_cells.cu: 16x8-pixel tiles, 32-hypothesis chunks, NCELL = 5 cell records per round; cost_mma.cu: 8x8 tiles,
64-hypothesis chunks, MMAXV = TMAXV = 16 staged cameras).  Every case is run in each of its depth modes and consistency
settings against one float64 reference, on every (variant, layout) that ``accepts`` the call; every other pair must be
refused."""

MODES = ("volume", "gauss", "planes")
# (variant, source layout) pairs a caller of ops.cost_volume can name; the GPU test maps them to the _lib constants
CANDIDATES = (("direct", "nchw"), ("direct", "tiled32"), ("cells", "tiled32"), ("cells_noreuse", "tiled32"),
              ("tma", "pixc"), ("mma", "split16"))
STAGED_VIEWS = 16                      # MMAXV (cost_mma.cu), TMAXV (cost_tma.cu), f_bwd_mma_supports

CASES = {
    # C = 16 / 32: ragged tiles, one past a CELLS chunk (D = 33) and a TMA / MMA chunk (D = 65), V = 3 (1/V divides) and
    # V = 4 (inv_v_exact multiplies), random depths at C = 32 (pixels visit more cells than NCELL)
    "c16_d33_v3": dict(C=16, B=3, V=3, H=13, W=21, D=33),
    "c16_d65_v4": dict(C=16, B=3, V=4, H=11, W=19, D=65),
    "c32_d33_v4_random": dict(C=32, B=3, V=4, H=13, W=21, D=33, depth="random"),
    "c32_d65_v3": dict(C=32, B=3, V=3, H=10, W=27, D=65),
    # C = 64: the tensor cores below AUTO's 32 hypotheses, MAGNET_MAX_PLANES (four MMA chunks), a single hypothesis and
    # view, one past an MMA chunk with feature scales far apart and pixels at the SPLIT16 floor
    "c64_d31": dict(C=64, B=3, V=3, H=13, W=21, D=31),
    "c64_d256": dict(C=64, B=3, V=3, H=9, W=13, D=256),
    "c64_d1_v1": dict(C=64, B=2, V=1, H=11, W=17, D=1),
    "c64_scales_tiny": dict(C=64, B=3, V=3, H=12, W=20, D=65, sr=1e-3, ss=1e3, tiny=True),
    # widths no specialised kernel takes: TILED32 (DIRECT) only, then NCHW only
    "c24": dict(C=24, B=3, V=3, H=10, W=14, D=12),
    "c13": dict(C=13, B=3, V=3, H=9, W=15, D=9),
    # the staged-camera limit: batch element 0 reads all 16 slots, element 1 only slot 15, element 2 none; then V = 17,
    # which the staged kernels refuse and AUTO routes elsewhere
    "v16": dict(C=64, B=3, V=16, H=12, W=20, D=64, invalid=[(1, v) for v in range(15)] + [(2, v) for v in range(16)],
                tc_bwd=True),
    "v17": dict(C=64, B=3, V=17, H=10, W=12, D=64, auto=True),
    # unsorted hypotheses: the tensor-core exact fallback (C = 64) and the CELLS exact cell walk (C = 32)
    "c64_k_descending": dict(C=64, B=3, V=3, H=12, W=20, D=64, modes=("gauss", "planes"), order="descending"),
    "c64_k_shuffled": dict(C=64, B=3, V=3, H=12, W=20, D=64, modes=("gauss", "planes"), order="shuffled"),
    "c32_k_descending": dict(C=32, B=3, V=3, H=13, W=21, D=40, modes=("gauss", "planes"), order="descending"),
    "c32_k_shuffled": dict(C=32, B=3, V=3, H=13, W=21, D=40, modes=("gauss", "planes"), order="shuffled"),
    # one production row: many work items per persistent CTA.  The CW volume in VOLUME and GAUSS mode is checked at
    # cfg2 by test_gpu_grad_f64.py already, so only PLANES runs with consistency here
    "cfg2": dict(cfg="cfg2", invalid=[(2, 1)] + [(7, v) for v in range(4)],
                 runs=[(m, False) for m in MODES] + [("planes", True)]),
}

def spec(name, configs=None):
    """The case with its defaults filled in; ``configs`` (synthetic.CONFIGS) resolves a ``cfg`` entry."""
    s = dict(depth="smooth", sr=1.0, ss=1.0, tiny=False, order="sorted", modes=MODES, tc_bwd=False, auto=False,
             family="scannet")
    if "cfg" in CASES[name]:
        if configs is None:
            raise ValueError(f"case {name} needs synthetic.CONFIGS")
        s.update({k: configs[CASES[name]["cfg"]][k] for k in ("B", "V", "D", "H", "W", "C", "family")})
    s.update(CASES[name])
    if "invalid" not in s:
        s["invalid"] = default_invalid(s["B"], s["V"])
    if "runs" not in s:
        s["runs"] = [(m, cw) for m in s["modes"] for cw in (True, False)]
    return s


def default_invalid(B, V):
    """One invalid (b, v) pair in a live batch element, and the last batch element with every view invalid."""
    dead = [(B - 1, v) for v in range(V)]
    if V >= 2 and B >= 3:              # batch element 0 keeps every view: its views 0 and 1 are the odd cameras
        return [(1, 0)] + dead
    if V >= 3:
        return [(0, V - 1)] + dead
    return dead


def accepts(variant, layout, C, V, mode):
    """Whether magnet_cost_volume_f32 runs ``variant`` on ``layout`` (api.cu validate_cost): CELLS and TMA for
    C in {16, 32, 64}, TMA and MMA for V <= 16, MMA for C = 64, NOREUSE in GAUSS mode only, TILED32 for C % 4 == 0."""
    if layout == "tiled32" and C % 4:
        return False
    if variant == "direct":
        return True
    if variant in ("cells", "cells_noreuse"):
        return C in (16, 32, 64) and (variant == "cells" or mode == "gauss")
    if variant == "tma":
        return C in (16, 32, 64) and V <= STAGED_VIEWS
    if variant == "mma":
        return C == 64 and V <= STAGED_VIEWS
    raise ValueError(variant)


def planned(configs=None):
    """Every forward the GPU test runs: (case, variant, layout, C, mode, consistency, softmax).  Softmax runs with
    consistency off only (api.cu refuses the other combination)."""
    out = []
    for name in CASES:
        s = spec(name, configs)
        for mode, cw in s["runs"]:
            for variant, layout in CANDIDATES:
                if accepts(variant, layout, s["C"], s["V"], mode):
                    for sm in ((False,) if cw else (False, True)):
                        out.append((name, variant, layout, s["C"], mode, cw, sm))
    return out


def instance(variant, layout, C, mode, cw):
    """The template instance a run reaches (non-indexed, fp32): cost_mma_kernel<MODE, CW, SPLIT16>,
    cost_tma_kernel<C, MODE, CW>, cost_cells_kernel<C, MODE, CW, REUSE>, cost_direct_kernel<CW> with the depth mode and
    the gather layout chosen at run time."""
    if variant == "mma":
        return ("mma", mode, cw)
    if variant == "direct":
        return ("direct", layout, mode, cw)
    return (variant, C, mode, cw)
