"""magnet_b200 — H100-native multi-view matching hot path of MaGNet (baegwangbin/MaGNet).

Only the hot path of SURVEY §8: depth-candidate sampler, plane-sweep warp + bilinear feature
sampling + depth-consistency weighting + view fusion (one fused sm_90a kernel), Gaussian update,
and their reference-facing wrappers.  The CUDA library is mandatory; there is no CPU fallback.
"""
from . import _lib
from .sampling import depth_sampling, k_offsets_f32
from .homography import est_costvolume_CW, est_costvolume_F, clear_cache, prep_cache
from .matcher import GNET, MAGNET, MagnetHead, MatchingPlan, matching_loop, install

__all__ = [
    "depth_sampling", "k_offsets_f32", "est_costvolume_CW", "est_costvolume_F", "clear_cache", "prep_cache",
    "GNET", "MAGNET", "MagnetHead", "MatchingPlan", "matching_loop", "install",
]
