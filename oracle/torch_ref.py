"""Torch (ATen) port of the reference's matching path — TEST / BASELINE INFRASTRUCTURE ONLY.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py`` (``cpu_baseline`` leg and
``--impl reference``) may import this file; ``magnet_b200`` never does.

Why a second oracle next to ``magnet_oracle.py``: the reference is pure PyTorch, so its
"CPU implementation" *is* a sequence of stock ATen kernels (matmul, repeat, grid_sample,
mul, sum ...).  The reference is not part of this repository, so the two baselines that
BASELINE.md asks for — reference-CPU on the host cores and reference-CUDA (``grid_sample``)
on the GPU — are produced by this port, which issues the same ATen operator sequence with
the same temporaries (including the D-fold ``repeat`` materialisations that dominate the
reference's cost, homography.py:92-93,105-110).  ``tests/test_oracle_golden.py`` checks that
this port is BIT-IDENTICAL on CPU to outputs of the reference functions frozen under
tests/golden/ by tests/golden/make_golden.py.

Restated from: models/submodules/homography.py:10-161 (cost volumes),
models/MAGNET.py:15-27 (convex upsampling), :58-70 (Gaussian update), :154-156 (sampler).
"""
from __future__ import annotations

import torch
import torch.nn.functional as F


def sample_depth_candidates(gmm: torch.Tensor, k_list) -> torch.Tensor:
    """MAGNET.py:154-156 — per-pixel candidates mu + sigma*k_j, concatenated over j."""
    mu, sigma = torch.split(gmm.detach(), 1, dim=1)
    return torch.cat([mu + sigma * k for k in k_list], dim=1)


def _sweep_grid(term_t, term_r, depth_rows, H, W):
    """Projected, normalised and clamped sampling grid (homography.py:56-67 / :130-148).
    term_t (3,1), term_r (3,HW), depth_rows broadcastable to (D,1,HW) -> (D,H,W,2), P (D,3,HW)."""
    D = depth_rows.shape[0]
    grid = torch.zeros(D, H, W, 2, device=term_r.device)
    stacked = term_r.unsqueeze(0).repeat(D, 1, 1)
    P = term_t.unsqueeze(0) + stacked * depth_rows
    P = P / (P[:, 2, :].unsqueeze(1) + 1e-10)
    grid[:, :, :, 0] = P[:, 0, :].reshape(D, H, W)
    grid[:, :, :, 1] = P[:, 1, :].reshape(D, H, W)
    half_h, half_w = H / 2., W / 2.
    grid[:, :, :, 0] = (grid[:, :, :, 0] - half_w) / half_w
    grid[:, :, :, 1] = (grid[:, :, :, 1] - half_h) / half_h
    grid[grid > 10.0] = 10.0
    grid[grid < -10.0] = -10.0
    return grid


def _warp(x, grid):
    return F.grid_sample(x, grid, mode='bilinear', padding_mode='zeros', align_corners=False)


def cost_volume_cw(d_volume, ref_feat, nghbr_feat, ref_gmms, nghbr_gmms, R, t, is_valid, cam_intrins, thres):
    """Consistency-weighted cost volume; same signature and operator sequence as
    homography.est_costvolume_CW (homography.py:79-161).  ``ref_gmms`` is unused there too."""
    B, D, H, W = d_volume.shape
    V = int(nghbr_feat.shape[0] / B)
    n_mu, n_sigma = torch.split(nghbr_gmms, 1, dim=1)
    dev = ref_feat.device
    volume = torch.zeros(B, D, H, W, device=dev)
    for b in range(B):
        K = cam_intrins['intM'][b, :, :].to(dev)
        rays = cam_intrins['unit_ray_array_2D'][b, :, :].to(dev)
        ref_rep = ref_feat[b, ...].unsqueeze(0).repeat(D, 1, 1, 1)
        fused = torch.zeros(D, H, W, device=dev)
        for v in range(V):
            if is_valid[b, v].item() != 1:
                continue
            eye = torch.eye(3, device=dev)
            cam_t = eye.matmul(t[b, v, :]).reshape(3, 1)
            cam_r = eye.matmul(R[b, v, :, :]).matmul(rays)
            pix_t = K.matmul(t[b, v, :]).reshape(3, 1)
            pix_r = K.matmul(R[b, v, :, :]).matmul(rays)
            src = v * B + b
            feat_rep = nghbr_feat[src, ...].unsqueeze(0).repeat(D, 1, 1, 1)
            mu_rep = n_mu[src, ...].unsqueeze(0).repeat(D, 1, 1, 1)
            sg_rep = n_sigma[src, ...].unsqueeze(0).repeat(D, 1, 1, 1)
            d_rows = d_volume[b, ...].reshape(D, 1, -1)
            grid = _sweep_grid(pix_t, pix_r, d_rows, H, W)
            z_cam = (cam_t.unsqueeze(0) + cam_r.unsqueeze(0).repeat(D, 1, 1) * d_rows)[:, 2, :].reshape(D, H, W)
            feat_w = _warp(feat_rep, grid)
            mu_w = _warp(mu_rep, grid)
            sg_w = _warp(sg_rep, grid)
            score = torch.sum(ref_rep * feat_w, axis=1)
            gap = torch.abs(z_cam - mu_w[:, 0, :, :])
            keep = (gap < (sg_w[:, 0, :, :] * thres)).double()
            fused = fused + score * keep
        volume[b, :, :, :] = fused
    return volume / float(V)


def cw_threshold_margin(d_volume, nghbr_gmms, R, t, is_valid, cam_intrins, thres):
    """How close every output element is to a consistency-mask flip, on any device and at full size: min over the
    valid views of | |z - mu~| - kappa*sigma~ | / max(|z|, kappa*sigma~, 1e-30) (the quantity magnet_oracle's
    ``return_margin`` reports), with z, mu~, sigma~ produced by the same operators as cost_volume_cw above
    (homography.py:130-158).  Used by the full-size parity tests: an element that differs from the reference by more
    than the tolerance must have a margin below tests/util.MARGIN_TOL."""
    B, D, H, W = d_volume.shape
    V = int(nghbr_gmms.shape[0] / B)
    n_mu, n_sigma = torch.split(nghbr_gmms, 1, dim=1)
    dev = d_volume.device
    margin = torch.full((B, D, H, W), float("inf"), device=dev, dtype=torch.float64)
    for b in range(B):
        K = cam_intrins['intM'][b, :, :].to(dev)
        rays = cam_intrins['unit_ray_array_2D'][b, :, :].to(dev)
        for v in range(V):
            if is_valid[b, v].item() != 1:
                continue
            eye = torch.eye(3, device=dev)
            cam_t = eye.matmul(t[b, v, :]).reshape(3, 1)
            cam_r = eye.matmul(R[b, v, :, :]).matmul(rays)
            pix_t = K.matmul(t[b, v, :]).reshape(3, 1)
            pix_r = K.matmul(R[b, v, :, :]).matmul(rays)
            src = v * B + b
            d_rows = d_volume[b, ...].reshape(D, 1, -1)
            grid = _sweep_grid(pix_t, pix_r, d_rows, H, W)
            z_cam = (cam_t.unsqueeze(0) + cam_r.unsqueeze(0).repeat(D, 1, 1) * d_rows)[:, 2, :].reshape(D, H, W)
            mu_w = _warp(n_mu[src, ...].unsqueeze(0).repeat(D, 1, 1, 1), grid)[:, 0]
            sg_w = _warp(n_sigma[src, ...].unsqueeze(0).repeat(D, 1, 1, 1), grid)[:, 0]
            gap, thr = torch.abs(z_cam - mu_w).double(), (sg_w * thres).double()
            scale = torch.maximum(torch.maximum(z_cam.abs().double(), thr.abs()), torch.full_like(thr, 1e-30))
            mg = (gap - thr).abs() / scale
            mg = torch.where(torch.isfinite(mg), mg, torch.zeros_like(mg))
            margin[b] = torch.minimum(margin[b], mg)
    return margin


def cost_volume_f(d_center, ref_feat, nghbr_feat, R, t, is_valid, cam_intrins, apply_softmax=True):
    """Fronto-parallel plane-sweep volume for F-Net training; same operator sequence as
    homography.est_costvolume_F (homography.py:10-75).  Differentiable in both feature maps."""
    B, _, H, W = ref_feat.shape
    D = d_center.shape[1]
    V = int(nghbr_feat.shape[0] / B)
    dev = ref_feat.device
    volume = torch.zeros(B, D, H, W, device=dev)
    for b in range(B):
        K = cam_intrins['intM'][b, :, :].to(dev)
        rays = cam_intrins['unit_ray_array_2D'][b, :, :].to(dev)
        ref_rep = ref_feat[b, ...].unsqueeze(0).repeat(D, 1, 1, 1)
        fused = torch.zeros(D, H, W, device=dev)
        for v in range(V):
            if is_valid[b, v].item() != 1:
                continue
            pix_t = K.matmul(t[b, v, :]).reshape(3, 1)
            pix_r = K.matmul(R[b, v, :, :]).matmul(rays)
            feat_rep = nghbr_feat[v * B + b, ...].unsqueeze(0).repeat(D, 1, 1, 1)
            grid = _sweep_grid(pix_t, pix_r, d_center.reshape(D, 1, 1), H, W)
            fused = fused + torch.sum(ref_rep * _warp(feat_rep, grid), axis=1)
        volume[b, :, :, :] = fused
    volume = volume / float(V)
    return F.softmax(volume, dim=1) if apply_softmax else volume


def gaussian_update(d_output, ref_gmm):
    """MAGNET.py:60,65-69 — mu' = mu0 + mu1*sigma0 ; sigma' = (elu(sigma1) + 1 + 1e-10)*sigma0."""
    mu0, s0 = torch.split(ref_gmm, 1, dim=1)
    mu1, s1 = torch.split(d_output, 1, dim=1)
    return torch.cat([mu0 + (mu1 * s0), (F.elu(s1) + 1.0 + 1e-10) * s0], dim=1)


def convex_upsample(depth, up_mask, k):
    """MAGNET.py:15-27 — learned convex k-times upsampling."""
    N, C, H, W = depth.shape
    m = torch.softmax(up_mask.view(N, 1, 9, k, k, H, W), dim=2)
    nb = F.unfold(depth, [3, 3], padding=1).view(N, C, 9, 1, 1, H, W)
    up = torch.sum(m * nb, dim=2).permute(0, 1, 4, 2, 5, 3)
    return up.reshape(N, C, k * H, k * W)


def matching_iterations(inp, g_net, x_d3, n_iter, k_list, thres):
    """The loop of MAGNET.py:150-169 on pre-computed backbone outputs: sampler -> CW cost
    volume -> cat with x_d3 -> G-Net conv head -> Gaussian update.  ``g_net`` maps the
    (B, D+256, H, W) tensor to the raw (B,2,H,W) update.  Returns the list of Gaussians."""
    preds = [inp.ref_gmms]
    for _ in range(n_iter):
        dvol = sample_depth_candidates(preds[-1], k_list)
        cv = cost_volume_cw(dvol, inp.ref_feat, inp.nghbr_feat, inp.ref_gmms, inp.nghbr_gmms,
                            inp.R, inp.t, inp.is_valid, inp.cam_intrins, thres)
        raw = g_net(torch.cat([cv.detach(), x_d3], dim=1))
        preds.append(gaussian_update(raw, preds[-1].detach()))
    return preds
