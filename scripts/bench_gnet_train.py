#!/usr/bin/env python
"""Forward + backward of one G-Net head iteration: the module path (cuDNN, cudnn.benchmark, PyTorch's default TF32
flags, plus the update kernel) against the fused training kernels (DESIGN §3.10), alternated in one process; then the
whole MagnetHead training step of examples/train_head.py with and without the fused head.

    python scripts/bench_gnet_train.py --config cfg2          # B 8, 120x160
    python scripts/bench_gnet_train.py --config cfg3          # B 4, 88x304

CUDA events, median of --repeats after warm-up.  Asserts gradient agreement (fused vs module against float64) at the
timed size.  One JSON line per measurement, with the card name and its power limit."""
import argparse, json, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F
import magnet_b200
from magnet_b200 import ops
from magnet_b200.matcher import GNET
from magnet_b200.synthetic import make_inputs

CONFIGS = {"cfg2": (8, 120, 160), "cfg3": (4, 88, 304)}


def card():
    name = torch.cuda.get_device_name()
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                            text=True, timeout=10).stdout.strip().splitlines()[torch.cuda.current_device()]
    except Exception:
        pl = "unknown"
    return {"gpu": name, "power_limit": pl}


def timed(fn, warm, reps):
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); b.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def iteration(args, D, info):
    B, H, W = CONFIGS[args.config]
    dev = torch.device("cuda")
    torch.manual_seed(0)
    g = GNET(ch_in=D + 256).to(dev).train()
    gen = torch.Generator(device=dev).manual_seed(1)
    cost = torch.randn(B, D, H, W, device=dev, generator=gen)
    x_d3 = torch.randn(B, 256, H, W, device=dev, generator=gen)
    with torch.no_grad():
        inv = g.invariant_part(x_d3, D)
    prev = torch.cat([1 + torch.rand(B, 1, H, W, device=dev, generator=gen),
                      0.1 + 0.5 * torch.rand(B, 1, H, W, device=dev, generator=gen)], 1)
    grad_out = torch.randn(B, 2, H, W, device=dev, generator=gen)
    # zero upstream gradient at pixels within 1e-5 of a ReLU kink (tests/test_gpu_gnet_train.unambiguous), where the
    # gradient itself is discontinuous and no fp32 evaluation can be compared to float64 element by element
    with torch.no_grad():
        z = F.conv2d(cost.double(), g.gnet[0].weight[:, :D].double(), None, padding=1) + inv.double()
        ok = torch.ones_like(z[:, :1], dtype=torch.bool)
        for layer in (2, 4, None):
            ok &= (z.abs() > 1e-5 * z.abs().max()).all(1, keepdim=True)
            if layer is None:
                break
            z = F.conv2d(F.relu(z), g.gnet[layer].weight.double(), g.gnet[layer].bias.double())
        grad_out *= ok.float()
        del z
    inv_leaf = inv.clone().requires_grad_(True)

    def module():
        g.zero_grad(set_to_none=True); inv_leaf.grad = None
        ops.gaussian_update(g.raw_from_parts(cost, inv_leaf), prev).backward(grad_out)

    def fused():
        g.zero_grad(set_to_none=True); inv_leaf.grad = None
        ops.gnet_head_train(cost, inv_leaf, g, prev).backward(grad_out)

    def grads():
        s = g.gnet
        return [inv_leaf.grad, s[0].weight.grad[:, :D]] + [p.grad for p in (s[2].weight, s[2].bias, s[4].weight,
                                                                             s[4].bias, s[6].weight, s[6].bias)]
    # gradient agreement at the timed size: fused error vs float64 within 1e-4 of the largest entry and no larger
    # than the module path's
    ws = [p.detach().double().requires_grad_(True) for p in (g.gnet[0].weight, g.gnet[2].weight, g.gnet[2].bias,
                                                              g.gnet[4].weight, g.gnet[4].bias, g.gnet[6].weight,
                                                              g.gnet[6].bias)]
    i64 = inv.double().requires_grad_(True)
    h = F.relu(F.conv2d(cost.double(), ws[0][:, :D], None, padding=1) + i64)
    h = F.relu(F.conv2d(h, ws[1], ws[2]))
    h = F.relu(F.conv2d(h, ws[3], ws[4]))
    raw = F.conv2d(h, ws[5], ws[6])
    out = torch.cat([prev[:, :1].double() + raw[:, :1] * prev[:, 1:].double(),
                     (F.elu(raw[:, 1:]) + 1 + 1e-10) * prev[:, 1:].double()], 1)
    gr = torch.autograd.grad(out, [i64] + ws, grad_out.double())
    want = [gr[0], gr[1][:, :D]] + list(gr[2:])
    del h, raw, out, gr
    fused(); gf = [t.clone() for t in grads()]
    module(); gm = [t.clone() for t in grads()]
    check = {}
    for n, a, b, w in zip(("inv", "W0c", "W1", "b1", "W2", "b2", "W3", "b3"), gf, gm, want):
        ef, em = float((a.double() - w).abs().max()), float((b.double() - w).abs().max())
        check[n] = {"fused_err": ef, "module_err": em, "max": float(w.abs().max())}
        assert ef <= 1e-4 * float(w.abs().max()) and (n.startswith("b") or ef <= em), (n, check[n])
    del want, gf, gm
    torch.cuda.empty_cache()
    t_mod, t_fus = [], []
    for _ in range(2):                                   # alternate the two paths
        t_mod.append(timed(module, args.warmup, args.repeats))
        t_fus.append(timed(fused, args.warmup, args.repeats))
    for path, t in (("module (cuDNN, default TF32 flags)", min(t_mod)), ("fused", min(t_fus))):
        print(json.dumps({"measurement": "G-Net head fwd+bwd, one iteration", "config": args.config, "B": B, "H": H,
                          "W": W, "D": D, "path": path, "ms_median": round(t, 4), "repeats": args.repeats,
                          "grad_check": check if path == "fused" else "passed", **info}), flush=True)


def train_step(args, D, info):
    here = os.path.dirname(os.path.abspath(__file__))
    ex = os.path.join(os.path.dirname(here), "examples", "train_head.py")
    env = dict(os.environ, WORLD_SIZE="1", RANK="0", LOCAL_RANK="0", MASTER_ADDR="127.0.0.1",
               MASTER_PORT=str(29500 + D))
    for flag in ([], ["--fused-head"]):
        r = subprocess.run([sys.executable, ex, "--steps", str(args.repeats), "--hypotheses", str(D), *flag],
                           capture_output=True, text=True, env=env)
        if r.returncode != 0:
            raise RuntimeError(r.stdout + r.stderr)
        res = json.loads(r.stdout.strip().splitlines()[-1])
        print(json.dumps({"measurement": "MagnetHead training step (examples/train_head.py, batch 4, 120x160)",
                          "D": D, "path": res["head_path"], "ms_median": round(res["rank0_step_ms_median"], 3),
                          "steps": args.repeats, "loss_first": res["loss_first"], "loss_last": res["loss_last"],
                          **info}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", choices=sorted(CONFIGS), default="cfg2")
    ap.add_argument("--repeats", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--skip-train-step", action="store_true")
    args = ap.parse_args()
    torch.backends.cudnn.benchmark = True
    info = card()
    for D in (64, 5):
        iteration(args, D, info)
    if not args.skip_train_step:
        for D in (64, 5):
            train_step(args, D, info)


if __name__ == "__main__":
    main()
