"""The drop-in F volume against the reference's own est_costvolume_F output (tests/golden/live_reference.npz)."""
import pytest
import torch

import magnet_b200
from magnet_b200.synthetic import make_inputs
from tests.util import input_digest, load_golden

pytestmark = pytest.mark.gpu


def test_reference_f_volume_through_install(cuda):
    """MAGNET_F.forward's call (MAGNET.py:197-200), forward values against the reference's est_costvolume_F output on
    the same inputs (tests/golden/live_reference.npz)."""
    z, _ = load_golden("live_reference")
    inp = make_inputs(B=2, V=2, D=8, H=20, W=28, C=16, seed=98, depth="smooth")
    assert input_digest(inp) == str(z["digest_98"]), "synthetic generator drifted from the golden fixture"
    g = inp.to(cuda)
    d_center = torch.linspace(0.8, 6.0, 12, device=cuda).view(1, -1, 1, 1)
    want = torch.from_numpy(z["install_f"]).to(cuda)
    with torch.no_grad():
        got = magnet_b200.est_costvolume_F(d_center, g.ref_feat, g.nghbr_feat, g.R, g.t, inp.is_valid, inp.cam_intrins)
    assert float((got - want).abs().max()) <= 1e-4 * float(want.abs().max())
