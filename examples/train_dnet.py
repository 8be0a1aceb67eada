"""D-Net training in the shape of train_DNet.py, with the loss on the package's fused kernels (DESIGN §3.19):
a STAND-IN trunk (plain convolutions to 256 channels at quarter resolution; EfficientNet-B5 needs torch.hub and is not
used) + ``DnetHead`` + ``DnetHead.loss`` (DnetLoss through ``ops.dnet_loss``), AdamW with gradient clipping, and
test_DNet's validation through ``DepthMetrics.update(variance=True)``.  Synthetic seeded images and depth maps stand in
for the data loaders.

``--compile default | reduce-overhead`` compiles the loss function (trunk + heads + loss) with torch.compile; the
optimizer step stays eager.  Under CUDA graphs the inputs are copied into static buffers each step.

usage: python examples/train_dnet.py [--steps N] [--batch B] [--size H W] [--compile {none,default,reduce-overhead}]"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402
import torch.nn as nn  # noqa: E402

from magnet_b200 import DepthMetrics, DnetHead  # noqa: E402


class StandInTrunk(nn.Module):
    """STAND-IN for D-Net's encoder-decoder (not EfficientNet-B5): image (B,3,H,W) -> x_feat (B,256,H/4,W/4)."""

    def __init__(self):
        super().__init__()
        self.net = nn.Sequential(nn.Conv2d(3, 64, 4, stride=4), nn.ReLU(inplace=True),
                                 nn.Conv2d(64, 256, 3, padding=1), nn.ReLU(inplace=True),
                                 nn.Conv2d(256, 256, 3, padding=1), nn.ReLU(inplace=True))

    def forward(self, img):
        return self.net(img)


class Dnet(nn.Module):
    def __init__(self):
        super().__init__()
        self.trunk, self.head = StandInTrunk(), DnetHead(in_dim=256)

    def forward(self, img):
        return self.head(self.trunk(img))

    def loss(self, img, gt_dmap, gt_dmap_mask):
        return self.head.loss(self.trunk(img), gt_dmap, gt_dmap_mask)


def batch(B, H, W, device, seed, max_depth=10.0, min_depth=1e-3):
    """A smooth synthetic scene: depth from a few sinusoids, the image a function of it; gt > max_depth zeroed and the
    mask gt > min_depth as train_DNet.py forms them."""
    g = torch.Generator(device=device).manual_seed(seed)
    yy, xx = torch.meshgrid(torch.linspace(0, 1, H, device=device), torch.linspace(0, 1, W, device=device),
                            indexing="ij")
    f = torch.rand(B, 4, 1, 1, device=device, generator=g)
    depth = 1.0 + 4.0 * (1 + torch.sin(6 * f[:, 0:1] * xx + 4 * f[:, 1:2] * yy)) * (0.5 + f[:, 2:3])
    img = torch.cat([depth / 10, torch.sin(depth), torch.cos(3 * depth)], 1)
    gt = depth.clone()
    gt[torch.rand(gt.shape, device=device, generator=g) < 0.1] = 0.0          # holes
    gt[gt > max_depth] = 0.0
    return img, gt, gt > min_depth


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--size", type=int, nargs=2, default=(416, 544))
    ap.add_argument("--lr", type=float, default=3.57e-4)
    ap.add_argument("--grad-clip", type=float, default=0.1)
    ap.add_argument("--compile", choices=("none", "default", "reduce-overhead"), default="none")
    ap.add_argument("--validate-every", type=int, default=10)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    torch.backends.cudnn.benchmark = True
    model = Dnet().to(dev).train()
    opt = torch.optim.AdamW(model.parameters(), lr=args.lr, weight_decay=1e-2)
    H, W = args.size
    loss_fn = model.loss if args.compile == "none" else torch.compile(model.loss, mode=args.compile)
    static = [t.clone() for t in batch(args.batch, H, W, dev, 0)]
    metrics = DepthMetrics(min_depth=1e-3, max_depth=10.0)
    t0 = time.perf_counter()
    for step in range(args.steps):
        new = batch(args.batch, H, W, dev, 1 + step)
        for s, n in zip(static, new):
            s.copy_(n)
        opt.zero_grad(set_to_none=True)
        loss = loss_fn(*static)
        loss.backward()
        nn.utils.clip_grad_norm_(model.parameters(), args.grad_clip)
        opt.step()
        if (step + 1) % args.validate_every == 0 or step + 1 == args.steps:
            model.eval()
            metrics.reset()
            with torch.no_grad():
                for i in range(2):                          # test_DNet's validate(): one image per batch
                    img, gt, _ = batch(1, H, W, dev, 10_000 + i)
                    metrics.update(model(img), gt, variance=True)
            model.train()
            print(json.dumps({"step": step + 1, "loss": float(loss), "val": metrics.value(),
                              "s_per_step": (time.perf_counter() - t0) / (step + 1)}), flush=True)


if __name__ == "__main__":
    main()
