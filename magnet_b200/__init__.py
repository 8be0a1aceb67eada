"""magnet_b200 — H100-native multi-view matching hot path of MaGNet (baegwangbin/MaGNet).

Only the hot path of SURVEY §8: depth-candidate sampler, plane-sweep warp + bilinear feature
sampling + depth-consistency weighting + view fusion (one fused sm_90a kernel), Gaussian update,
their reference-facing wrappers, and the depth evaluation of validate() (``DepthMetrics``).
The CUDA library is mandatory; there is no CPU fallback.
"""
from . import _lib
from .sampling import depth_sampling, k_offsets_f32
from .homography import est_costvolume_CW, est_costvolume_F, clear_cache, geometry_grad, prep_cache
from .matcher import GNET, MAGNET, DnetHead, MagnetF, MagnetHead, MatchingPlan, matching_loop, install, sid_planes
from .metrics import DepthMetrics
from .ops import depth_metrics, plane_depth

__all__ = [
    "depth_sampling", "k_offsets_f32", "est_costvolume_CW", "est_costvolume_F", "clear_cache", "prep_cache",
    "geometry_grad",
    "GNET", "MAGNET", "DnetHead", "MagnetF", "MagnetHead", "MatchingPlan", "matching_loop", "install", "sid_planes",
    "DepthMetrics", "depth_metrics", "plane_depth",
]
