"""Seeded synthetic inputs for the multi-view matching path (SURVEY §8 rows a8 / d).

The generator reproduces the *conventions* of the reference's callers, not their
code: quarter-resolution intrinsics and per-pixel rays through pixel centres
(data/dataloader_scannet.py:113-153), relative poses that map reference-camera to
source-camera coordinates (utils/utils.py:92), source tensors stacked view-major
(index = v*B + b, test_MaGNet.py:45-46), Gaussians as [mu, sigma(stdev)]
(models/DNET.py:62-67), ``is_valid`` int32 on the CPU and ``cam_intrins`` a dict of
CPU tensors (test_MaGNet.py:36-50).

Everything is generated with numpy (fp64 -> fp32) from an explicit seed so that the
same arrays can be rebuilt on any machine without shipping fixtures.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, Optional

import numpy as np
import torch

from .sampling import k_offsets_f32

# quarter-resolution intrinsics quoted in SURVEY §8(d)
SCANNET_Q = dict(fx=144.4, fy=145.0, cx=80.0, cy=60.0, W=160, H=120)
KITTI_Q = dict(fx=180.4, fy=180.4, cx=149.1, cy=37.5, W=304, H=88)


@dataclass
class MatchingInputs:
    """One batch of inputs in the layout ``MAGNET.forward`` hands to the matching loop."""

    ref_feat: torch.Tensor      # (B, C, H, W)
    nghbr_feat: torch.Tensor    # (V*B, C, H, W)  view-major
    ref_gmms: torch.Tensor      # (B, 2, H, W)    [mu, sigma]
    nghbr_gmms: torch.Tensor    # (V*B, 2, H, W)
    nghbr_poses: torch.Tensor   # (B, V, 4, 4)    ref-cam -> source-cam
    is_valid: torch.Tensor      # (B, V) int32, CPU
    cam_intrins: Dict[str, torch.Tensor]  # 'intM' (B,3,3), 'unit_ray_array_2D' (B,3,H*W); CPU
    k: torch.Tensor             # (D,) fp32 sampler offsets
    thres: int = 5
    meta: dict = field(default_factory=dict)

    @property
    def B(self) -> int:
        return self.ref_feat.shape[0]

    @property
    def V(self) -> int:
        return self.nghbr_feat.shape[0] // self.ref_feat.shape[0]

    @property
    def D(self) -> int:
        return self.k.shape[0]

    @property
    def R(self) -> torch.Tensor:
        return self.nghbr_poses[:, :, :3, :3]   # non-contiguous view, as MAGNET.py:147

    @property
    def t(self) -> torch.Tensor:
        return self.nghbr_poses[:, :, :3, 3]    # non-contiguous view, as MAGNET.py:148

    def depth_volume(self, gmms: Optional[torch.Tensor] = None) -> torch.Tensor:
        """The sampler of MAGNET.py:154-156 in plain torch: d_j = mu + sigma * k_j."""
        g = self.ref_gmms if gmms is None else gmms
        mu, sigma = g[:, 0:1], g[:, 1:2]
        return torch.cat([mu + sigma * float(kj) for kj in self.k.tolist()], dim=1)

    def to(self, device) -> "MatchingInputs":
        """Move what the reference moves: features, Gaussians, poses.  ``is_valid`` and
        ``cam_intrins`` stay on the CPU like in test_MaGNet.py:41-50."""
        return MatchingInputs(
            ref_feat=self.ref_feat.to(device), nghbr_feat=self.nghbr_feat.to(device),
            ref_gmms=self.ref_gmms.to(device), nghbr_gmms=self.nghbr_gmms.to(device),
            nghbr_poses=self.nghbr_poses.to(device), is_valid=self.is_valid,
            cam_intrins=self.cam_intrins, k=self.k.to(device), thres=self.thres, meta=dict(self.meta))


def _rot_y(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]], dtype=np.float64)


def _rot_x(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[1, 0, 0], [0, c, -s], [0, s, c]], dtype=np.float64)


def quarter_res_camera(H: int, W: int, family: str = "scannet"):
    """intM (3,3) and rays (3, H*W) in the reference's quarter-resolution convention.

    Rays are ``K_raw^-1 (x+0.5, y+0.5, 1)`` at quarter-res pixel centres, which in
    quarter-res units is ``((x+0.5-cx)/fx, (y+0.5-cy)/fy, 1)``; flat index n = y*W + x
    (data/dataloader_scannet.py:119-120,141-146).  For grids other than the family's
    native one the intrinsics are scaled with the grid."""
    base = SCANNET_Q if family == "scannet" else KITTI_Q
    sx, sy = W / base["W"], H / base["H"]
    fx, fy, cx, cy = base["fx"] * sx, base["fy"] * sy, base["cx"] * sx, base["cy"] * sy
    K = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], dtype=np.float64)
    xs = (np.arange(W, dtype=np.float64) + 0.5 - cx) / fx
    ys = (np.arange(H, dtype=np.float64) + 0.5 - cy) / fy
    rays = np.ones((3, H, W), dtype=np.float64)
    rays[0] = xs[None, :]
    rays[1] = ys[:, None]
    return K.astype(np.float32), rays.reshape(3, H * W).astype(np.float32)


def make_inputs(B: int, V: int, D: int, H: int, W: int, C: int = 64, *, seed: int = 0,
                family: str = "scannet", depth: str = "smooth", sigma_rel: float = 0.10,
                sampling_range: float = 3.0, thres: int = 5, invalid=(),
                rot_deg: Optional[float] = None, trans: Optional[float] = None) -> MatchingInputs:
    """Build one seeded batch.

    depth="smooth": the perf distribution of SURVEY §8(d) (smooth mu, sigma = sigma_rel*mu,
    source Gaussians = the same field +2 % noise) so that 50-80 % of samples pass the
    consistency test and the gather pattern is coherent.
    depth="random": i.i.d. mu in [0.5, 6), sigma in [0.05, 0.6) — the incoherent numerics stress.
    ``invalid`` is an iterable of (b, v) pairs whose is_valid flag is cleared.
    """
    rng = np.random.default_rng(seed)
    HW = H * W
    ref_feat = rng.standard_normal((B, C, H, W)).astype(np.float32)
    nghbr_feat = rng.standard_normal((V * B, C, H, W)).astype(np.float32)

    yy, xx = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
    if depth == "smooth":
        if family == "scannet":
            field_mu = 2.5 + 1.2 * np.sin(2 * np.pi * xx / W) * np.cos(2 * np.pi * yy / H)
        else:
            field_mu = 8.0 + 40.0 * (1.0 - yy / H) ** 2
        mu = field_mu[None] * (1.0 + 0.01 * rng.standard_normal((B, H, W)))
        sigma = sigma_rel * mu
        nmu = field_mu[None] * (1.0 + 0.02 * rng.standard_normal((V * B, H, W)))
        nsigma = sigma_rel * nmu
    elif depth == "random":
        mu = rng.uniform(0.5, 6.0, (B, H, W))
        sigma = rng.uniform(0.05, 0.6, (B, H, W))
        nmu = rng.uniform(0.5, 6.0, (V * B, H, W))
        nsigma = rng.uniform(0.05, 0.6, (V * B, H, W))
    else:
        raise ValueError(depth)
    ref_gmms = np.stack([mu, sigma], axis=1).astype(np.float32)
    nghbr_gmms = np.stack([nmu, nsigma], axis=1).astype(np.float32)

    K, rays = quarter_res_camera(H, W, family)
    intM = np.repeat(K[None], B, axis=0)
    ray2d = np.repeat(rays[None], B, axis=0)

    poses = np.zeros((B, V, 4, 4), dtype=np.float64)
    for b in range(B):
        for v in range(V):
            if family == "scannet":
                a = np.deg2rad(3.0 if rot_deg is None else rot_deg)
                tr = 0.15 if trans is None else trans
                Rm = _rot_y(rng.uniform(-a, a)) @ _rot_x(rng.uniform(-a, a))
                tv = rng.uniform(-tr, tr, 3)
            else:
                a = np.deg2rad(1.5 if rot_deg is None else rot_deg)
                Rm = _rot_y(rng.uniform(-a, a))
                tz = rng.choice([-2.0, -1.0, 1.0, 2.0]) * (1.0 if trans is None else trans)
                tv = np.array([rng.uniform(-0.05, 0.05), rng.uniform(-0.02, 0.02), tz])
            poses[b, v, :3, :3] = Rm
            poses[b, v, :3, 3] = tv
            poses[b, v, 3, 3] = 1.0
    is_valid = np.ones((B, V), dtype=np.int32)
    for (b, v) in invalid:
        is_valid[b, v] = 0

    return MatchingInputs(
        ref_feat=torch.from_numpy(ref_feat), nghbr_feat=torch.from_numpy(nghbr_feat),
        ref_gmms=torch.from_numpy(ref_gmms), nghbr_gmms=torch.from_numpy(nghbr_gmms),
        nghbr_poses=torch.from_numpy(poses.astype(np.float32)),
        is_valid=torch.from_numpy(is_valid),
        cam_intrins={"intM": torch.from_numpy(intM), "unit_ray_array_2D": torch.from_numpy(ray2d)},
        k=torch.from_numpy(k_offsets_f32(sampling_range, D)), thres=thres,
        meta=dict(B=B, V=V, D=D, H=H, W=W, C=C, seed=seed, family=family, depth=depth,
                  sigma_rel=sigma_rel))


# the named configurations of BASELINE.json (grids at quarter resolution, SURVEY §0 / §8 d)
CONFIGS = {
    "cfg1": dict(B=1, V=2, D=16, H=128, W=160, C=64, family="scannet", depth="random"),
    "cfg2": dict(B=8, V=4, D=64, H=120, W=160, C=64, family="scannet", depth="smooth"),
    "cfg3": dict(B=4, V=4, D=64, H=88, W=304, C=64, family="kitti", depth="smooth"),
    "ship": dict(B=1, V=4, D=5, H=120, W=160, C=64, family="scannet", depth="smooth"),
}


def make_config(name: str, seed: int = 0, **over) -> MatchingInputs:
    kw = dict(CONFIGS[name])
    kw.update(over)
    return make_inputs(seed=seed, **kw)


# ---------------------------------------------------------------------------------------------------------------------
# Sequences (sequence evaluation, ``MAGNET.forward_frames`` / ``FrameCache``)

def window_neighbours(img_idx: int, last: int, window_radius: int = 20, n_views: int = 4):
    """The neighbour frames of reference frame ``img_idx`` in a sequence whose frames are 0..last, by the rule of the
    reference's ScanNet loader (data/dataloader_scannet.py:157-164): offsets k * interval for k in [-n/2, n/2] \\ {0},
    interval = window_radius // (n/2); an offset i that leaves the sequence is replaced by -i - sign(i) * (interval // 2).
    Returns the V = n_views frame ids in the loader's order."""
    interval = window_radius // (n_views // 2)
    out = []
    for k in range(-(n_views // 2), n_views // 2 + 1):
        i = k * interval
        if i == 0:
            continue
        out.append(img_idx + i if 0 <= img_idx + i <= last else img_idx - i - int(np.sign(i)) * int(interval * 0.5))
    return out


def scannet_sequence(n_refs: int, stride: int = 10, window_radius: int = 20, n_views: int = 4):
    """A test sequence as ScanNet's split lists it: references every ``stride`` frames (frames 0, stride, ...,
    (n_refs-1)*stride exist, and every frame in between), each with its ``window_neighbours``.  Returns (ref_ids,
    nghbr_ids): n_refs frame ids and n_refs lists of V ids."""
    last = (n_refs - 1) * stride
    refs = [r * stride for r in range(n_refs)]
    return refs, [window_neighbours(r, last, window_radius, n_views) for r in refs]


def trajectory(frames, seed: int = 0, step: float = 0.004, turn_deg: float = 0.12) -> dict:
    """Camera-to-world extrinsics (4,4) float32 of a smooth hand-held path, one per frame id in ``frames``: per frame
    a forward-leaning translation of about ``step`` and a rotation of about ``turn_deg`` degrees, with a seeded
    wobble.  Relative poses come from ``ops.relative_poses`` as in the reference's data_preprocess."""
    frames = sorted(set(int(f) for f in frames))
    rng = np.random.default_rng(seed)
    lo, hi = frames[0], frames[-1]
    n = hi - lo + 1
    wob = rng.standard_normal((n, 4)).cumsum(axis=0) * 0.05
    out = {}
    for f in frames:
        i = f - lo
        yaw = np.deg2rad(turn_deg * i + 2.0 * np.sin(wob[i, 0]))
        pitch = np.deg2rad(1.5 * np.sin(wob[i, 1]))
        E = np.eye(4)
        E[:3, :3] = _rot_y(yaw) @ _rot_x(pitch)
        E[:3, 3] = [step * i * 0.3 + 0.02 * np.sin(wob[i, 2]), 0.01 * np.sin(wob[i, 3]), step * i]
        out[f] = E.astype(np.float32)
    return out
