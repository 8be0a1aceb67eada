"""The case table of tests/test_gpu_forward_f64.py reaches every non-indexed fp32 instance of the four forward cost
kernels, and puts its shapes on both sides of their tile, chunk and staged-camera limits.  The instance list is read
from the kernels' dispatch calls, so a new channel width there fails this test until the table covers it."""
import os
import re

from magnet_b200.synthetic import CONFIGS
from tests import forward_f64_cases as fc

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "magnet_b200", "csrc")


def _source(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def _widths(name):
    """The channel widths a launcher dispatches over: its ``Choice<int, ...>{C}``."""
    m = re.findall(r"Choice<int,\s*([\d,\s]+)>\{C\}", _source(name))
    assert len(m) == 1, (name, m)
    return tuple(int(c) for c in m[0].split(","))


def _constant(name, ident):
    m = re.search(rf"\b{ident}\s*=\s*(\d+)", _source(name)) or re.search(rf"#define\s+MAGNET_{ident}\s+(\d+)",
                                                                         _source(name))
    assert m, (name, ident)
    return int(m.group(1))


def test_every_forward_instance_is_planned():
    modes, flags = fc.MODES, (False, True)
    want = {("mma", m, cw) for m in modes for cw in flags}
    want |= {("tma", c, m, cw) for c in _widths("cost_tma.cu") for m in modes for cw in flags}
    want |= {("cells", c, m, cw) for c in _widths("cost_cells.cu") for m in modes for cw in flags}
    want |= {("cells_noreuse", c, "gauss", cw) for c in _widths("cost_cells.cu") for cw in flags}
    want |= {("direct", lay, m, cw) for lay in ("nchw", "tiled32") for m in modes for cw in flags}
    runs = fc.planned(CONFIGS)
    got = {fc.instance(v, lay, c, m, cw) for _, v, lay, c, m, cw, _ in runs}
    assert not want - got, sorted(want - got, key=str)
    # with consistency off every instance also runs under the softmax, and no run asks for both
    soft = {fc.instance(v, lay, c, m, cw) for _, v, lay, c, m, cw, sm in runs if sm}
    assert {w for w in want if not w[-1]} <= soft
    assert not any(cw and sm for *_, cw, sm in runs)
    print(f"{len(runs)} forward runs cover {len(want)} instances")


def test_acceptance_rule_matches_the_kernels():
    """``accepts`` against the launchers: CELLS and TMA for the widths they dispatch over, MMA at 64, and the
    staged kernels up to their camera slots."""
    assert _constant("cost_mma.cu", "MMAXV") == _constant("cost_tma.cu", "TMAXV") == fc.STAGED_VIEWS
    for c in (1, 8, 13, 16, 24, 32, 48, 64, 96):
        for v in (1, 16, 17):
            for m in fc.MODES:
                assert fc.accepts("cells", "tiled32", c, v, m) == (c in _widths("cost_cells.cu") and c % 4 == 0)
                assert fc.accepts("tma", "pixc", c, v, m) == (c in _widths("cost_tma.cu") and v <= 16)
                assert fc.accepts("mma", "split16", c, v, m) == (c == 64 and v <= 16)
                assert fc.accepts("cells_noreuse", "tiled32", c, v, m) == (fc.accepts("cells", "tiled32", c, v, m)
                                                                            and m == "gauss")
                assert fc.accepts("direct", "nchw", c, v, m) and fc.accepts("direct", "tiled32", c, v, m) == (c % 4 == 0)


def test_cases_straddle_the_kernel_edges():
    tiles = {"tma": (_constant("cost_tma.cu", "TTW"), _constant("cost_tma.cu", "TTH")),
             "cells": (_constant("cost_cells.cu", "TILE_W"), 128 // _constant("cost_cells.cu", "TILE_W")),
             "mma": (_constant("cost_mma.cu", "MTW"), _constant("cost_mma.cu", "MTH"))}
    chunks = {"tma": 4 * _constant("cost_tma.cu", "TJL"), "cells": _constant("cost_cells.cu", "JCHUNK"),
              "mma": _constant("cost_mma.cu", "MCH")}
    specs = [fc.spec(n, CONFIGS) for n in fc.CASES]
    for k, (tw, th) in tiles.items():
        runs_k = [s for s in specs if fc.accepts(k, {"tma": "pixc", "cells": "tiled32", "mma": "split16"}[k], s["C"],
                                                 s["V"], "volume")]
        assert any(s["W"] % tw and s["H"] % th for s in runs_k), k
        assert any(s["D"] % chunks[k] == 1 and s["D"] > chunks[k] for s in runs_k), k
        assert any(s["D"] < chunks[k] for s in runs_k), k
        assert any(s["V"] == fc.STAGED_VIEWS for s in runs_k) or k == "cells", k
    assert {s["V"] for s in specs} >= {1, 3, 4, fc.STAGED_VIEWS, fc.STAGED_VIEWS + 1}
    assert max(s["D"] for s in specs) == 256
    assert {s["order"] for s in specs} >= {"sorted", "descending", "shuffled"}
    for s in specs:                    # an invalid view, and a batch element with none valid
        assert s["invalid"] and any(all((b, v) in s["invalid"] for v in range(s["V"])) for b in range(s["B"])), s
