"""Standard-normal depth-candidate offsets k_j (SURVEY §8 row a1).

Follows the reference's ``MAGNET.depth_sampling`` (models/MAGNET.py:120-128): the
central probability mass ``P = erf(beta / sqrt(2))`` of N(0,1) is cut into ``N_s``
equal-probability bins; ``k_j`` is the midpoint of the two bin edges (in z-score
units) that bound bin ``j``.  Host-side, fp64, evaluated once.

The normal quantile is evaluated with ``scipy.special.ndtri`` when scipy is
importable (the reference uses ``scipy.stats.norm.ppf``, which is ndtri) and with
a self-contained fp64 Newton refinement of ``erfinv`` otherwise, so the package
has no hard scipy dependency.
"""
from __future__ import annotations

import math
from typing import List

import numpy as np


def _ndtri(p: np.ndarray) -> np.ndarray:
    try:
        from scipy.special import ndtri  # same function scipy.stats.norm.ppf calls

        return ndtri(p)
    except Exception:  # pragma: no cover - scipy is present in this image
        out = np.empty_like(p)
        for i, pi in enumerate(p):
            # bisection + Newton on Phi(x) = p, fp64
            lo, hi = -40.0, 40.0
            for _ in range(200):
                mid = 0.5 * (lo + hi)
                if 0.5 * math.erfc(-mid / math.sqrt(2.0)) < pi:
                    lo = mid
                else:
                    hi = mid
            out[i] = 0.5 * (lo + hi)
        return out


def depth_sampling(sampling_range: float, n_samples: int) -> List[float]:
    """k_list exactly as models/MAGNET.py:120-128 builds it (list of fp64 scalars)."""
    p_total = math.erf(sampling_range / math.sqrt(2.0))
    idx = np.arange(0, n_samples + 1)
    p_list = (1.0 - p_total) / 2.0 + (idx / n_samples) * p_total
    edges = _ndtri(p_list)
    k = (edges[1:] + edges[:-1]) / 2.0
    return [float(v) for v in k]


def k_offsets_f32(sampling_range: float, n_samples: int) -> np.ndarray:
    """The offsets as the sampler consumes them: rounded to fp32 (MAGNET.py:155 multiplies
    an fp32 tensor by a Python/numpy scalar, which torch casts to the tensor dtype)."""
    return np.asarray(depth_sampling(sampling_range, n_samples), dtype=np.float64).astype(np.float32)
