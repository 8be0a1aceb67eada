"""Test-time pose refinement through the plane-sweep volume: recover a perturbed translation by gradient steps on the
matching score, with the camera gradients of ``magnet_b200.geometry_grad()``.

The scene is the known answer of SURVEY B.1: with R = I and t = (t_x, 0, 0), a reference pixel at depth d appears in the
source view f_x t_x / d pixels to the right, so a source image that is the reference shifted by exactly +1 px is matched
perfectly by t_x = d / f_x at constant depth d.  The features are smooth (a few low-frequency sinusoids per channel), so
the score has a wide basin around that t_x.  The example starts from t_x with a 0.6 px error and runs Adam on t_x alone
(step 0.1 px, decaying by 0.9),
maximising the mean plane-sweep score (``plane_sweep_f``, ``softmax=False``) at the true depth over the pixels at least
3 px from the border, whose samples stay inside the source image.

The same trajectory is first rehearsed on the CPU in float64 with autograd of the ATen port of the reference's
operators (``oracle/torch_ref.py``); on a GPU the kernels' trajectory is printed next to it.

usage: python examples/refine_pose.py [--steps N]
"""
from __future__ import annotations

import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

B, V, C, H, W = 1, 1, 8, 24, 32
FX, DEPTH, SHIFT0 = 40.0, 2.0, 1.6          # start: 1.6 px instead of 1 px


def scene(dtype=torch.float64):
    """(ref_feat, src_feat, intM, rays, is_valid, d_center, base poses) on the CPU."""
    g = torch.Generator().manual_seed(0)
    freq = torch.rand(C, 3, 2, generator=g, dtype=torch.float64) * 0.5 + 0.1
    phase = torch.rand(C, 3, generator=g, dtype=torch.float64) * 6.283
    yy, xx = torch.meshgrid(torch.arange(H, dtype=torch.float64), torch.arange(W, dtype=torch.float64), indexing="ij")

    def feat(shift):
        x = xx - shift
        return sum(torch.sin(freq[:, k, 0, None, None] * x + freq[:, k, 1, None, None] * yy + phase[:, k, None, None])
                   for k in range(3)).unsqueeze(0)

    ref, src = feat(0.0), feat(1.0)                 # src(x) = ref(x - 1): the +1 px shift
    K = torch.tensor([[FX, 0.0, W / 2.0], [0.0, FX, H / 2.0], [0.0, 0.0, 1.0]], dtype=torch.float64)
    pix = torch.stack([xx.reshape(-1) + 0.5, yy.reshape(-1) + 0.5, torch.ones(H * W, dtype=torch.float64)])
    rays = (torch.linalg.inv(K) @ pix).unsqueeze(0)  # pixel centres: the identity pose samples at ix = x
    poses = torch.eye(4, dtype=torch.float64).expand(B, V, 4, 4).clone()
    d_center = torch.full((1, 1, 1, 1), DEPTH, dtype=torch.float64)
    is_valid = torch.ones(B, V, dtype=torch.int64)
    return (ref.to(dtype), src.to(dtype), K.unsqueeze(0).to(dtype), rays.to(dtype), is_valid, d_center.to(dtype),
            poses.to(dtype))


def refine(impl: str, steps: int = 40, lr_px: float = 0.1, device=None):
    """Adam on t_x; returns the error of the shift f_x t_x / d in pixels before each step and after the last.
    impl "port": float64 autograd of the ATen port on the CPU; "magnet": plane_sweep_f on ``device`` under
    geometry_grad()."""
    dtype = torch.float64 if impl == "port" else torch.float32
    ref, src, K, rays, is_valid, d_center, base = scene(dtype)
    tx = torch.tensor(SHIFT0 * DEPTH / FX, dtype=dtype, requires_grad=True)
    unit = torch.zeros(B, V, 4, 4, dtype=dtype)
    unit[:, :, 0, 3] = 1.0
    if impl == "magnet":
        ref, src, base, unit, d_center = (x.to(device) for x in (ref, src, base, unit, d_center))
    opt = torch.optim.Adam([tx], lr=lr_px * DEPTH / FX)
    sched = torch.optim.lr_scheduler.ExponentialLR(opt, gamma=0.9)   # at most lr / (1 - 0.9) = 1 px of travel
    errs = []
    for _ in range(steps + 1):
        errs.append(float(tx.detach()) * FX / DEPTH - 1.0)
        if len(errs) == steps + 1:
            break
        poses = base + tx.to(base.device) * unit
        intr = {'intM': K, 'unit_ray_array_2D': rays}
        if impl == "port":
            from oracle import torch_ref
            default = torch.get_default_dtype()
            torch.set_default_dtype(torch.float64)
            try:
                score = torch_ref.cost_volume_f(d_center, ref, src, poses[:, :, :3, :3], poses[:, :, :3, 3], is_valid,
                                                intr, apply_softmax=False)
            finally:
                torch.set_default_dtype(default)
        else:
            import magnet_b200
            from magnet_b200.homography import plane_sweep_f
            with magnet_b200.geometry_grad():
                score = plane_sweep_f(d_center, ref, src, poses[:, :, :3, :3], poses[:, :, :3, 3], is_valid, intr,
                                      softmax=False)
        opt.zero_grad()
        (-score[..., 3:-3, 3:-3].mean()).backward()      # interior: no sample near the zero padding
        opt.step()
        sched.step()
    return errs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=40)
    args = ap.parse_args()
    cpu = refine("port", args.steps)
    gpu = refine("magnet", args.steps, device=torch.device("cuda")) if torch.cuda.is_available() else None
    print("step  shift error (px): float64 port on the CPU" + ("   | magnet_b200 on the GPU" if gpu else ""))
    for i, e in enumerate(cpu):
        print(f"{i:4d}  {e:+.5f}" + (f"   | {gpu[i]:+.5f}" if gpu else ""))


if __name__ == "__main__":
    main()
