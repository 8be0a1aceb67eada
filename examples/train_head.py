#!/usr/bin/env python
"""BASELINE.json configs[3]: MaGNet head training step at ScanNet shape, batch sharded over the GPUs of one box.

    python examples/train_head.py --steps 20                       # 1 GPU, batch 4
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 \
        examples/train_head.py --global-batch 32 --steps 20        # 8 GPUs x batch 4

What is trained is what the reference trains (train_MaGNet.py:48 after MAGNET.__init__ froze the backbones):
G-Net + mask head (0.75 M fp32 parameters at N_s=64), loss = gamma-weighted Gaussian NLL over the N_iter
upsampled predictions (utils/losses.py:34-50), AdamW, gradient clipping at 1.0, one flat-bucket NCCL gradient
all-reduce per step (magnet_b200.dist.FlatGradAllReduce) instead of DistributedDataParallel.  The frozen
D-Net / F-Net are replaced by fixed random tensors of their output shapes (they need torch.hub + checkpoints in
the reference and are out of scope): features (B,64,h,w) / (V*B,64,h,w), Gaussians, x_d3 (B,256,h,w).
The matching loop runs on the H100 kernels (sampler fused, update kernel with backward).

--compile default / reduce-overhead compiles the function that returns the loss (torch.compile, or CUDA-graph trees);
its backward is compiled with it and runs at loss.backward().  The all-reduce, clipping and AdamW step stay eager."""
import argparse, json, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import magnet_b200
from magnet_b200 import dist as md
from magnet_b200.synthetic import make_inputs


def gaussian_nll(pred_list, gt, mask, gamma=0.8):
    """utils/losses.py:34-50 (MagnetLoss, 'gaussian')."""
    loss = 0.0
    n = len(pred_list)
    gt = gt[mask]
    for i, pred in enumerate(pred_list):
        mu, sigma = pred[:, 0:1][mask], pred[:, 1:2][mask]
        var = torch.square(sigma).clamp_min(1e-10)
        loss = loss + gamma ** (n - i - 1) * torch.mean(torch.square(mu - gt) / (2 * var) + 0.5 * torch.log(var))
    return loss


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--global-batch", type=int, default=None)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--hypotheses", type=int, default=64)
    ap.add_argument("--views", type=int, default=4)
    ap.add_argument("--unfused-loss", action="store_true",
                    help="materialise the N_iter upsampled (B,2,4H,4W) predictions and evaluate the NLL in torch (the "
                         "reference's data flow) instead of the fused upsample+NLL kernels (SURVEY §8 f-2)")
    ap.add_argument("--fused-head", action="store_true",
                    help="train the G-Net head through the fused tensor-core forward and backward (DESIGN §3.10) "
                         "instead of the cuDNN module chain")
    ap.add_argument("--fused-mask", action="store_true",
                    help="run the mask head after its first convolution, the upsampling and the loss as one fused "
                         "tensor-core op with its backward (MagnetHead.train_loss with fused_upsample, DESIGN §3.13) "
                         "instead of the cuDNN mask head and the fused upsample+NLL kernels")
    ap.add_argument("--compile", choices=("none", "default", "reduce-overhead"), default="none",
                    help="compile the loss function (the training kernels are custom ops with registered backwards)")
    args = ap.parse_args()
    if args.fused_mask and args.unfused_loss:
        raise SystemExit("--fused-mask and --unfused-loss exclude each other")
    rank, local_rank, world = md.env_world()
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    md.init_process_group("nccl", device_id=dev)
    gb = args.global_batch or 4 * world
    lo, hi = md.shard_range(gb, rank, world)
    B, H, W, D, V = hi - lo, 120, 160, args.hypotheses, args.views

    inp = make_inputs(B=B, V=V, D=D, H=H, W=W, C=64, seed=100 + rank, depth="smooth").to(dev)
    g = torch.Generator().manual_seed(7 + rank)
    x_d3 = torch.randn(B, 256, H, W, generator=g).to(dev)
    gt = (inp.ref_gmms[:, 0:1] * 1.03)                                    # quarter-res "ground truth" ...
    gt = torch.nn.functional.interpolate(gt, scale_factor=4, mode="nearest")   # ... at full resolution
    mask = gt > 1e-3

    torch.manual_seed(0)                                                   # same init on every rank
    head = magnet_b200.MagnetHead(n_samples=D, sampling_range=3, n_iter=3, thres=5, fused_train=args.fused_head,
                                   fused_upsample=args.fused_mask).to(dev)
    reducer = md.FlatGradAllReduce(head.parameters())
    reducer.broadcast_parameters(0)
    opt = torch.optim.AdamW(head.parameters(), lr=3.57e-4, weight_decay=1e-2)

    def loss_fn(ref_feat, nghbr_feat, ref_gmms, nghbr_gmms, x_d3, poses, is_valid, intM, rays, gt, mask):
        cam = {"intM": intM, "unit_ray_array_2D": rays}
        if args.unfused_loss:
            return gaussian_nll(head(ref_feat, nghbr_feat, ref_gmms, nghbr_gmms, x_d3, poses, is_valid, cam), gt, mask)
        if args.fused_mask:
            return head.train_loss(ref_feat, nghbr_feat, ref_gmms, nghbr_gmms, x_d3, poses, is_valid, cam, gt, mask)
        preds_q, up_mask = head.forward_quarter(ref_feat, nghbr_feat, ref_gmms, nghbr_gmms, x_d3, poses, is_valid, cam)
        return head.loss(preds_q, up_mask, gt, mask)         # f-2: no (B,2,4H,4W) tensors, fwd or bwd

    if args.compile != "none" and args.unfused_loss:
        raise SystemExit("--compile needs a loss without boolean indexing (drop --unfused-loss)")
    step_loss = loss_fn if args.compile == "none" else torch.compile(loss_fn, mode=None if args.compile == "default"
                                                                     else args.compile)
    # the eager step takes is_valid and cam_intrins on the host, as the reference's loaders give them; a compiled one
    # takes them on the device (CUDA-graph trees do not capture a graph with host inputs)
    host = (inp.is_valid, inp.cam_intrins["intM"], inp.cam_intrins["unit_ray_array_2D"])
    step_args = (inp.ref_feat, inp.nghbr_feat, inp.ref_gmms, inp.nghbr_gmms, x_d3, inp.nghbr_poses,
                 *(host if args.compile == "none" else (t.to(dev) for t in host)), gt, mask)

    WARM = 5                                                               # cuDNN autotuning, NCCL lazy init, allocator growth
    losses, t0, marks = [], None, []
    for step in range(args.steps + WARM):
        if step == WARM:
            torch.cuda.synchronize(); md.barrier(); t0 = time.perf_counter()
        if step >= WARM:
            ev = torch.cuda.Event(enable_timing=True); ev.record(); marks.append(ev)
        opt.zero_grad(set_to_none=True)
        loss = step_loss(*step_args)
        loss.backward()
        reducer()                                                          # one 3 MB all-reduce
        torch.nn.utils.clip_grad_norm_(head.parameters(), 1.0)
        opt.step()
        losses.append(md.sum_over_ranks(float(loss.detach()), device=dev) / world)
    ev = torch.cuda.Event(enable_timing=True); ev.record(); marks.append(ev)
    torch.cuda.synchronize(); md.barrier()
    dt = time.perf_counter() - t0
    per_step = sorted(marks[i].elapsed_time(marks[i + 1]) for i in range(len(marks) - 1))   # device time between step starts
    if rank == 0:
        print(json.dumps({"config": "train head, ScanNet shape", "n_gpus": world, "global_batch": gb, "steps": args.steps,
                          "head_path": "fused G-Net kernels" if args.fused_head else "cuDNN module chain",
                          "loss_path": "unfused (torch NLL on upsampled predictions)" if args.unfused_loss else
                                       "fused mask head + upsample + NLL kernel" if args.fused_mask else "fused upsample+NLL kernels",
                          "compile": args.compile, "ms_per_step": 1e3 * dt / args.steps, "frames_per_s": gb * args.steps / dt,
                          "rank0_step_ms_median": per_step[len(per_step) // 2], "rank0_step_ms_max": per_step[-1],
                          "loss_first": losses[0], "loss_last": losses[-1], "trainable_params": reducer.bucket.numel()}))
    md.shutdown()


if __name__ == "__main__":
    main()
