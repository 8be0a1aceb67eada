"""The tensor-core kernel's window boxes come from the projections of each pixel's smallest and largest depth (widened by
a rounding margin) instead of from every hypothesis.  A debug build counts the hypotheses whose cell origin fell outside
their box: none may, over the fuzz shapes, the full cfg2 / cfg3 shapes in both depth modes, and SID planes behind a
source camera, which must take the exact per-hypothesis pass."""
import json
import os
import subprocess
import sys

import pytest

from magnet_b200 import build as _build

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_no_hypothesis_origin_outside_its_window_box(cuda):
    lib = _build.build(defines=("MAGNET_MMA_DEBUG",), tag="mmadbg")
    env = dict(os.environ, MAGNET_B200_LIB=str(lib))
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "mma_box_probe.py")], env=env, cwd=ROOT,
                       capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    outside = {case: c[0] for case, c in res.items() if c[0] != 0}
    assert not outside, outside
    assert res["sid_planes"][1] > 0, res["sid_planes"]     # z <= 0 at the nearest planes: exact pass
    assert res["cfg2/gauss"][1] == 0 and res["cfg3/gauss"][1] == 0, (res["cfg2/gauss"], res["cfg3/gauss"])
    print({case: c for case, c in res.items() if not case.startswith("fuzz")})
