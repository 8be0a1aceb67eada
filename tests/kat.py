"""Analytic known-answer cases for the CW / F cost volumes (SURVEY Appendix B.1).  Each builder returns
(inputs, d_volume, expected, rel_tol); the same cases are run against the oracle on CPU and against the
CUDA kernels on the GPU."""
import numpy as np
import torch

from magnet_b200.synthetic import make_inputs


def _identity_poses(inp):
    inp.nghbr_poses.zero_()
    for i in range(4):
        inp.nghbr_poses[:, :, i, i] = 1.0


def _per_pixel_dot(inp, shift=0):
    B, V = inp.B, inp.V
    ref = inp.ref_feat.numpy().astype(np.float64)
    src = inp.nghbr_feat.numpy().astype(np.float64)
    out = np.zeros((V, B) + ref.shape[2:])
    for v in range(V):
        s = src[v * B:(v + 1) * B]
        if shift:
            s = np.concatenate([s[..., shift:], np.zeros_like(s[..., :shift])], axis=-1)
        out[v] = (ref * s).sum(axis=1)
    return out  # (V,B,H,W)


def base(seed=5, B=2, V=2, D=4, H=12, W=16, C=16):
    return make_inputs(B=B, V=V, D=D, H=H, W=W, C=C, seed=seed, depth="smooth")


def identity_open_mask(**kw):
    inp = base(**kw)
    _identity_poses(inp)
    inp.nghbr_gmms[:, 1] = 1e6
    dots = _per_pixel_dot(inp)
    exp = np.repeat(dots.mean(axis=0)[:, None], inp.D, axis=1)
    return inp, inp.depth_volume(), exp, 1e-4


def all_invalid(**kw):
    inp = base(**kw)
    inp.is_valid.zero_()
    return inp, inp.depth_volume(), np.zeros((inp.B, inp.D) + tuple(inp.ref_feat.shape[2:])), 0.0


def one_invalid_view(**kw):
    inp = base(**kw)
    _identity_poses(inp)
    inp.nghbr_gmms[:, 1] = 1e6
    inp.is_valid[:, 1] = 0
    dots = _per_pixel_dot(inp)
    exp = np.repeat((dots[0] / inp.V)[:, None], inp.D, axis=1)     # still divided by ALL views (homography.py:120)
    return inp, inp.depth_volume(), exp, 1e-4


def closed_mask(**kw):
    inp = base(**kw)
    inp.nghbr_gmms[:, 1] = 1e-9
    return inp, inp.depth_volume(), np.zeros((inp.B, inp.D) + tuple(inp.ref_feat.shape[2:])), 0.0


def one_pixel_shift(**kw):
    inp = base(**kw)
    _identity_poses(inp)
    inp.nghbr_gmms[:, 1] = 1e6
    d = 2.0
    inp.ref_gmms[:, 0] = d
    inp.ref_gmms[:, 1] = 0.0
    fx = float(inp.cam_intrins['intM'][0, 0, 0])
    inp.nghbr_poses[:, :, 0, 3] = d / fx
    dots = _per_pixel_dot(inp, shift=1)
    exp = np.repeat(dots.mean(axis=0)[:, None], inp.D, axis=1)
    return inp, inp.depth_volume(), exp, 1e-4


CW_CASES = dict(identity_open_mask=identity_open_mask, all_invalid=all_invalid, one_invalid_view=one_invalid_view,
                closed_mask=closed_mask, one_pixel_shift=one_pixel_shift)


def f_identity(**kw):
    inp = base(**kw)
    _identity_poses(inp)
    planes = np.linspace(0.7, 6.0, 9).astype(np.float32)
    exp = np.full((inp.B, 9) + tuple(inp.ref_feat.shape[2:]), 1.0 / 9)
    return inp, planes, exp, 1e-6
