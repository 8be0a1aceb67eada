"""Generate tests/golden/*.npz by running the UNMODIFIED reference (a checkout of baegwangbin/MaGNet):
    MAGNET_REFERENCE=<path of the checkout> python tests/golden/make_golden.py

Inputs are not stored: they are rebuilt from the seed by magnet_b200.synthetic (numpy Generator
streams are version-stable); each file carries a sha256 of the inputs so a drifting generator is
detected instead of silently comparing against the wrong reference output.

Reference entry points exercised:
  models/submodules/homography.py  est_costvolume_CW (:79), est_costvolume_F (:10)
  models/MAGNET.py                 GNET.forward update equations (:58-70), upsample_depth_via_mask (:15-27),
                                   MAGNET.depth_sampling (:120-128), the sampler expression (:154-156)
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ.get("MAGNET_REFERENCE", "")
sys.path.insert(0, ROOT)

from tests.util import input_digest  # noqa: E402

CASES = {
    # name: (make_inputs kwargs)
    "cw_small_random": dict(B=2, V=3, D=8, H=24, W=32, C=16, seed=1, depth="random", invalid=[(1, 2)]),
    "cw_small_smooth": dict(B=2, V=3, D=8, H=24, W=32, C=16, seed=2, depth="smooth"),
    "cw_c64_d64": dict(B=1, V=2, D=64, H=16, W=64, C=64, seed=3, depth="smooth"),
    "cw_kitti": dict(B=1, V=2, D=12, H=22, W=76, C=32, seed=4, depth="smooth", family="kitti"),
    "cw_cfg1": dict(B=1, V=2, D=16, H=128, W=160, C=64, seed=0, depth="random"),
}
F_PLANES = 12


def f_planes(n=F_PLANES, d_min=0.5, d_max=8.0):
    """SID plane centres as train_FNet.py:56-66 builds them (n planes instead of 80)."""
    idx = np.arange(n + 1)
    gamma = 1 - d_min
    bounds = np.exp(np.log(d_max + gamma) * idx / n) - gamma
    return ((bounds[:-1] + bounds[1:]) / 2).astype(np.float32)


def _import_reference():
    if not os.path.isdir(os.path.join(REF, "models")):
        raise SystemExit("set MAGNET_REFERENCE to a checkout of the reference (baegwangbin/MaGNet)")
    sys.path.insert(0, REF)
    # utils/utils.py:5-7 imports matplotlib, which is absent; the hot path never touches it.
    for name in ("matplotlib", "matplotlib.pyplot"):
        m = types.ModuleType(name)
        m.use = lambda *a, **k: None
        sys.modules.setdefault(name, m)


def live_reference_cases(refh):
    """Outputs of the reference's est_costvolume_CW / est_costvolume_F (CPU) on the inputs of the bit-identity test of
    oracle/torch_ref.py and of the drop-in F-volume test (tests/test_oracle_golden.py, tests/test_gpu_reference_module.py)."""
    from magnet_b200.synthetic import make_inputs
    threads = torch.get_num_threads()
    torch.set_num_threads(1)          # the softmax of the F volume reduces in a thread-count dependent order
    out = {}
    for seed, depth in ((11, "random"), (12, "smooth")):
        inp = make_inputs(B=2, V=2, D=6, H=20, W=28, C=8, seed=seed, depth=depth, invalid=[(0, 1)])
        dv = inp.depth_volume()
        out[f"cw_{seed}"] = refh.est_costvolume_CW(dv, inp.ref_feat, inp.nghbr_feat, inp.ref_gmms, inp.nghbr_gmms, inp.R,
                                                   inp.t, inp.is_valid, inp.cam_intrins, 5).numpy()
        dc = torch.linspace(0.5, 7, 9).view(1, 9, 1, 1)
        out[f"f_{seed}"] = refh.est_costvolume_F(dc, inp.ref_feat, inp.nghbr_feat, inp.R, inp.t, inp.is_valid,
                                                 inp.cam_intrins).numpy()
        out[f"digest_{seed}"] = np.array(input_digest(inp))
    inp = make_inputs(B=2, V=2, D=8, H=20, W=28, C=16, seed=98, depth="smooth")
    d_center = torch.linspace(0.8, 6.0, 12).view(1, -1, 1, 1)
    out["install_f"] = refh.est_costvolume_F(d_center, inp.ref_feat, inp.nghbr_feat, inp.R, inp.t, inp.is_valid,
                                             inp.cam_intrins).numpy()
    out["digest_98"] = np.array(input_digest(inp))
    np.savez_compressed(os.path.join(HERE, "live_reference.npz"), **out)
    torch.set_num_threads(threads)
    print("live reference cases written:", sorted(out))


def main():
    _import_reference()
    import models.submodules.homography as refh
    from models.MAGNET import GNET, MAGNET, upsample_depth_via_mask
    from magnet_b200.synthetic import make_inputs

    torch.set_num_threads(4)
    for name, kw in CASES.items():
        inp = make_inputs(**kw)
        # the sampler exactly as MAGNET.py:154-156 writes it (k_list = python/numpy floats)
        mu, sigma = torch.split(inp.ref_gmms, 1, dim=1)
        holder = types.SimpleNamespace(sampling_range=3, n_samples=kw["D"])
        k_list = MAGNET.depth_sampling(holder)
        dvol = torch.cat([mu + sigma * k for k in k_list], dim=1)
        out = refh.est_costvolume_CW(dvol, inp.ref_feat, inp.nghbr_feat, inp.ref_gmms, inp.nghbr_gmms,
                                     inp.R, inp.t, inp.is_valid, inp.cam_intrins, inp.thres)
        save = dict(cost_cw=out.numpy(), k_list=np.asarray(k_list, dtype=np.float64),
                    digest=np.array(input_digest(inp)), kwargs=np.array(repr(kw)))
        if name != "cw_cfg1":
            save["d_volume"] = dvol.numpy()
            dc = torch.from_numpy(f_planes()).view(1, F_PLANES, 1, 1)
            save["planes"] = dc.numpy().reshape(-1)
            save["cost_f"] = refh.est_costvolume_F(dc, inp.ref_feat, inp.nghbr_feat, inp.R, inp.t,
                                                    inp.is_valid, inp.cam_intrins).numpy()
        np.savez_compressed(os.path.join(HERE, name + ".npz"), **save)
        print(name, out.shape, "nonzero", float((out != 0).float().mean()))

    # Gaussian update: the reference's GNET.forward with the conv stack replaced by identity,
    # forward value and autograd gradient w.r.t. the (would-be) conv output.
    g = torch.Generator().manual_seed(7)
    d_output = (torch.randn(2, 2, 9, 11, generator=g) * 1.5).requires_grad_(True)
    ref_gmm = torch.stack([torch.rand(2, 9, 11, generator=g) * 4 + 0.5, torch.rand(2, 9, 11, generator=g) + 0.05], 1)
    gn = GNET(ch_in=2)
    gn.gnet = torch.nn.Identity()
    new = gn(d_output, ref_gmm)
    gout = torch.randn(new.shape, generator=g)
    (new * gout).sum().backward()
    # learned convex upsampling
    depth = torch.rand(2, 2, 6, 7, generator=g) * 3
    mask = torch.randn(2, 9 * 16, 6, 7, generator=g)
    up = upsample_depth_via_mask(depth, mask, 4)
    ks = {f"k_{b}_{n}": np.asarray(MAGNET.depth_sampling(types.SimpleNamespace(sampling_range=b, n_samples=n)))
          for (b, n) in ((3, 5), (3, 16), (3, 64), (2, 7))}
    np.savez_compressed(os.path.join(HERE, "update_upsample.npz"),
                        d_output=d_output.detach().numpy(), ref_gmm=ref_gmm.numpy(), new_gmm=new.detach().numpy(),
                        grad_out=gout.numpy(), grad_d_output=d_output.grad.numpy(),
                        depth=depth.numpy(), mask=mask.numpy(), up=up.numpy(), **ks)
    print("update / upsample / k_list written")
    camera_prep_and_loss(g)
    live_reference_cases(refh)


def _camera_prep_case():
    """(V+1) x B extrinsics with a NaN source pose and a NaN reference pose (same generator as the tests use)."""
    rng = np.random.default_rng(9)
    B, V = 3, 4
    ext = np.tile(np.eye(4, dtype=np.float32), (V + 1, B, 1, 1))
    for f in range(V + 1):
        for b in range(B):
            a = rng.uniform(-0.2, 0.2, 3)
            Rz = np.array([[np.cos(a[0]), -np.sin(a[0]), 0], [np.sin(a[0]), np.cos(a[0]), 0], [0, 0, 1]])
            Ry = np.array([[np.cos(a[1]), 0, np.sin(a[1])], [0, 1, 0], [-np.sin(a[1]), 0, np.cos(a[1])]])
            ext[f, b, :3, :3] = (Rz @ Ry).astype(np.float32)
            ext[f, b, :3, 3] = rng.uniform(-1, 1, 3).astype(np.float32)
    ext_ref, ext_nghbr = ext[V // 2].copy(), np.delete(ext, V // 2, axis=0).copy()
    ext_nghbr[0, 1, 0, 0] = np.nan          # NaN source extrinsic: that view is invalid
    ext_ref[2, 1, 1] = np.nan               # NaN reference extrinsic: all views of that element invalid
    return ext_ref, ext_nghbr


SCANNET_RAW = [1169.621094, 1167.105103, 646.295044, 489.927032, 1296.0, 968.0]      # fx fy cx cy raw_W raw_H
KITTI_RAW = [721.5377, 721.5377, 609.5593, 172.854, 1242.0, 375.0]                    # K_cam2 of a 1242 x 375 drive


def camera_prep_and_loss(g):
    """SURVEY §8 f-4 / f-2 pins: the reference's own data_preprocess (utils/utils.py:72-98), get_cam_intrinsics of the
    ScanNet and KITTI loaders (data/dataloader_scannet.py:113-153, data/dataloader_kitti.py:94-127) and MagnetLoss
    (utils/losses.py:34-50, with autograd gradients through upsample_depth_via_mask)."""
    import tempfile
    import utils.utils as ref_utils
    import utils.losses as ref_losses
    from models.MAGNET import upsample_depth_via_mask
    # numpy 2 cannot take a torch tensor in np.linalg.inv(tensor) the way the 2021 code does (utils.py:92): hand the
    # same values over as an ndarray.  Nothing else of data_preprocess is touched.
    real_inv = np.linalg.inv

    class _NP:
        def __getattr__(self, name):
            return getattr(np, name)

    class _LA:
        def __getattr__(self, name):
            return getattr(np.linalg, name)

        @staticmethod
        def inv(a):
            return real_inv(np.asarray(a))

    shim = _NP()
    shim.linalg = _LA()
    ref_utils.np = shim
    ext_ref, ext_nghbr = _camera_prep_case()
    V, B = ext_nghbr.shape[:2]
    frames = [{"extM": torch.from_numpy(ext_nghbr[v])} for v in range(V)]
    data_array = frames[:V // 2] + [{"extM": torch.from_numpy(ext_ref)}] + frames[V // 2:]
    _, _, poses, valid = ref_utils.data_preprocess(data_array, B)
    ref_utils.np = np

    # ScanNet loader: unbound methods on a stub self, intrinsics from a temp 'intrinsic_color.txt'
    for name in ("pykitti",):
        if name not in sys.modules:
            sys.modules[name] = types.ModuleType(name)
    import data.dataloader_scannet as ds
    import data.dataloader_kitti as dk
    H, W = 120, 160
    stub = types.SimpleNamespace(dpv_H=H, dpv_W=W, raw_WH_dict={"scene0000_00": (int(SCANNET_RAW[4]), int(SCANNET_RAW[5]))})
    cls = ds.ScannetLoadPreprocess
    stub.ray_array = cls.get_ray_array(stub)
    with tempfile.TemporaryDirectory() as td:
        os.makedirs(os.path.join(td, "intrinsic"))
        K4 = np.eye(4)
        K4[0, 0], K4[1, 1], K4[0, 2], K4[1, 2] = SCANNET_RAW[:4]
        with open(os.path.join(td, "intrinsic", "intrinsic_color.txt"), "w") as f:
            for row in K4:
                f.write(" ".join(repr(float(x)) for x in row) + "\n")
        cam_s = cls.get_cam_intrinsics(stub, td, "scene0000_00")
    # KITTI loader: crop to 1216 x 352 (left margin (raw_W-1216)/2, top margin raw_H-352)
    clsk = dk.KittiLoadPreprocess
    Hk, Wk = 88, 304
    stubk = types.SimpleNamespace(dpv_H=Hk, dpv_W=Wk, img_H=352, img_W=1216)
    stubk.ray_array = clsk.get_ray_array(stubk)
    Kk = np.eye(3)
    Kk[0, 0], Kk[1, 1], Kk[0, 2], Kk[1, 2] = KITTI_RAW[:4]
    p_data = types.SimpleNamespace(get_cam2=lambda i: types.SimpleNamespace(size=(int(KITTI_RAW[4]), int(KITTI_RAW[5]))),
                                   calib=types.SimpleNamespace(K_cam2=Kk))
    cam_k = clsk.get_cam_intrinsics(stubk, p_data)

    # MagnetLoss on two upsampled predictions, gradients w.r.t. the quarter-resolution predictions and the mask logits
    preds = [(torch.cat([torch.rand(2, 1, 6, 7, generator=g) * 3 + 0.5, torch.rand(2, 1, 6, 7, generator=g) * 0.4 + 0.05], 1)
              ).requires_grad_(True) for _ in range(2)]
    with torch.no_grad():
        preds[1][0, 1, 2, 3] = 1e-7                       # var below the 1e-10 clamp (losses.py:45)
    mask = torch.randn(2, 9 * 16, 6, 7, generator=g).requires_grad_(True)
    gt = torch.rand(2, 1, 24, 28, generator=g) * 3 + 0.4
    gt_mask = torch.rand(2, 1, 24, 28, generator=g) > 0.3
    loss_fn = ref_losses.MagnetLoss(types.SimpleNamespace(loss_fn="gaussian", loss_gamma=0.8))
    ups = [upsample_depth_via_mask(p, mask, 4) for p in preds]
    loss = loss_fn(ups, gt, gt_mask)
    loss.backward()
    np.savez_compressed(os.path.join(HERE, "camera_prep_loss.npz"),
                        ext_ref=ext_ref, ext_nghbr=ext_nghbr, poses=poses.numpy(), valid=valid.numpy(),
                        scannet_raw=np.asarray(SCANNET_RAW), scannet_intM=cam_s["intM"].numpy(),
                        scannet_rays=cam_s["unit_ray_array_2D"].numpy(),
                        kitti_raw=np.asarray(KITTI_RAW), kitti_intM=cam_k["intM"].numpy(),
                        kitti_rays=cam_k["unit_ray_array_2D"].numpy(),
                        pred0=preds[0].detach().numpy(), pred1=preds[1].detach().numpy(), up_mask=mask.detach().numpy(),
                        gt=gt.numpy(), gt_mask=gt_mask.numpy(), loss=np.float32(loss.item()),
                        g_pred0=preds[0].grad.numpy(), g_pred1=preds[1].grad.numpy(), g_mask=mask.grad.numpy())
    print("camera prep + loss written: valid", valid.tolist(), "loss", float(loss))


if __name__ == "__main__":
    main()
