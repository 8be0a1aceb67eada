"""The fused G-Net head of inference on the H100 (DESIGN §3.8): against a float64 evaluation of the same head and update,
against the cuDNN module path, the dispatch rule of matching_loop, determinism, CUDA-graph replay and non-finite
cost values."""
import pytest
import torch
import torch.nn.functional as F

import magnet_b200
from magnet_b200 import ops
from magnet_b200.matcher import GNET, fused_gnet_applies, matching_loop
from magnet_b200.synthetic import make_inputs

pytestmark = pytest.mark.gpu


def _head(D, dev, seed=0):
    torch.manual_seed(seed)
    return GNET(ch_in=D + 16).to(dev).eval()


def _f64(g, cost, inv, prev):
    """The head and the update in float64 on the same cost volume and invariant."""
    D = cost.shape[1]
    s = g.gnet
    h = F.relu(F.conv2d(cost.double(), s[0].weight[:, :D].double(), None, padding=1) + inv.double())
    h = F.relu(F.conv2d(h, s[2].weight.double(), s[2].bias.double()))
    h = F.relu(F.conv2d(h, s[4].weight.double(), s[4].bias.double()))
    raw = F.conv2d(h, s[6].weight.double(), s[6].bias.double())
    mu0, s0 = prev[:, :1].double(), prev[:, 1:].double()
    return torch.cat([mu0 + raw[:, :1] * s0, (F.elu(raw[:, 1:]) + 1 + 1e-10) * s0], 1)


def _unit_prev(B, H, W, dev):
    return torch.cat([torch.zeros(B, 1, H, W, device=dev), torch.ones(B, 1, H, W, device=dev)], 1)


def _channel_err(got, want):
    """Per channel: max |got - want| over max |want|."""
    return [float((got[:, c].double() - want[:, c]).abs().max() / want[:, c].abs().max()) for c in range(2)]


def _fused(g, cost, inv, prev):
    with torch.no_grad():
        return ops.gnet_update(cost, inv, ops.pack_gnet_weights(g, cost.shape[1]), prev)


GRIDS = [(1, 1), (7, 9), (24, 40), (120, 160), (88, 304)]


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("D", [1, 5, 8, 16, 33, 64, 256])
@pytest.mark.parametrize("grid", GRIDS, ids=[f"{h}x{w}" for h, w in GRIDS])
def test_fused_head_matches_float64(cuda, D, grid, B):
    H, W = grid
    g = _head(D, cuda, seed=D)
    gen = torch.Generator(device=cuda).manual_seed(H * W + D)
    cost = torch.randn(B, D, H, W, device=cuda, generator=gen)
    inv = 0.3 * torch.randn(B, 128, H, W, device=cuda, generator=gen)
    prev = _unit_prev(B, H, W, cuda)
    got = _fused(g, cost, inv, prev)
    with torch.no_grad():
        want = _f64(g, cost, inv, prev)
    for c, e in enumerate(_channel_err(got, want)):
        assert e <= 1e-5, f"channel {c}: {e:.2e}"


@pytest.mark.parametrize("cost_scale", [1e-3, 1.0, 1e3])
@pytest.mark.parametrize("inv_scale", [1e-3, 1.0, 1e3])
def test_fused_head_across_input_scales(cuda, cost_scale, inv_scale):
    B, D, H, W = 3, 64, 24, 40
    g = _head(D, cuda, seed=1)
    gen = torch.Generator(device=cuda).manual_seed(11)
    cost = cost_scale * torch.randn(B, D, H, W, device=cuda, generator=gen)
    inv = inv_scale * torch.randn(B, 128, H, W, device=cuda, generator=gen)
    prev = torch.cat([torch.rand(B, 1, H, W, device=cuda, generator=gen) * 5,
                      0.1 + torch.rand(B, 1, H, W, device=cuda, generator=gen)], 1)
    got = _fused(g, cost, inv, prev)
    with torch.no_grad():
        want = _f64(g, cost, inv, prev)
        raw_want = _f64(g, cost, inv, _unit_prev(B, H, W, cuda))
    raw_got = _fused(g, cost, inv, _unit_prev(B, H, W, cuda))
    for c, e in enumerate(_channel_err(raw_got, raw_want)):
        assert e <= 1e-5, f"raw channel {c}: {e:.2e}"
    for c, e in enumerate(_channel_err(got, want)):
        assert e <= 1e-5, f"updated channel {c}: {e:.2e}"


# cfg2, cfg3 at D 64 and the shipped N_s = 5 at the cfg2 grid
SHAPES = [(8, 64, 120, 160), (4, 64, 88, 304), (8, 5, 120, 160)]


@pytest.mark.parametrize("shape", SHAPES, ids=["cfg2", "cfg3", "ns5"])
def test_fused_head_matches_module_path(cuda, shape):
    B, D, H, W = shape
    g = _head(D, cuda, seed=2)
    gen = torch.Generator(device=cuda).manual_seed(5)
    cost = torch.randn(B, D, H, W, device=cuda, generator=gen)
    x_d3 = torch.randn(B, 16, H, W, device=cuda, generator=gen)
    prev = torch.cat([2 + torch.rand(B, 1, H, W, device=cuda, generator=gen),
                      0.1 + 0.2 * torch.rand(B, 1, H, W, device=cuda, generator=gen)], 1)
    tf32 = torch.backends.cudnn.allow_tf32
    try:
        with torch.no_grad():
            torch.backends.cudnn.allow_tf32 = False
            inv = g.invariant_part(x_d3, D)
            module = ops.gaussian_update(g.raw_from_parts(cost, inv), prev)
            fused = _fused(g, cost, inv, prev)
            for c in range(2):
                ref = module[:, c].abs().max()
                assert float((fused[:, c] - module[:, c]).abs().max()) <= 1e-4 * float(ref)
            want = _f64(g, cost, inv, prev)
            torch.backends.cudnn.allow_tf32 = True             # PyTorch's default: the module path in TF32
            module_tf32 = ops.gaussian_update(g.raw_from_parts(cost, inv), prev)
        e_fused, e_module = _channel_err(fused, want), _channel_err(module_tf32, want)
        for c in range(2):
            assert e_fused[c] <= e_module[c], (c, e_fused[c], e_module[c])
    finally:
        torch.backends.cudnn.allow_tf32 = tf32


def _plan_inputs(dev, D=16):
    inp = make_inputs(B=2, V=2, D=D, H=24, W=40, C=64, seed=21, depth="smooth")
    g = inp.to(dev)
    plan = magnet_b200.MatchingPlan(g.ref_feat, g.nghbr_feat, g.nghbr_gmms, g.nghbr_poses, inp.is_valid,
                                    inp.cam_intrins, thres=inp.thres)
    x_d3 = torch.randn(2, 16, 24, 40, device=dev, generator=torch.Generator(device=dev).manual_seed(4))
    return inp, g, plan, x_d3


def test_matching_loop_runs_the_fused_head_without_grad(cuda):
    inp, g, plan, x_d3 = _plan_inputs(cuda)
    head = _head(16, cuda, seed=3)
    k = inp.k.tolist()
    with torch.no_grad():
        preds = matching_loop(plan, g.ref_gmms, x_d3, head, 3, k)
        inv = head.invariant_part(x_d3, 16)
        packed = ops.pack_gnet_weights(head, 16)
        cur, want = g.ref_gmms, []
        for _ in range(3):
            cur = ops.gnet_update(plan.cost(cur, k), inv, packed, cur)
            want.append(cur)
    for a, b in zip(preds[1:], want):
        assert torch.equal(a, b)


def _module_chain(plan, ref, x_d3, head, k, n, detach=True):
    inv = head.invariant_part(x_d3, len(k))
    cur, out = ref, []
    for _ in range(n):
        cur = cur.detach().float()
        if detach:
            with torch.no_grad():
                cv = plan.cost(cur, k)
        else:
            cv = plan.cost(cur, k)
        cur = ops.gaussian_update(head.raw_from_parts(cv, inv).float(), cur)
        out.append(cur)
    return out


def test_matching_loop_keeps_the_module_path_when_a_gradient_is_needed(cuda):
    inp, g, plan, x_d3 = _plan_inputs(cuda)
    head = _head(16, cuda, seed=3).train()
    k = inp.k.tolist()
    preds = matching_loop(plan, g.ref_gmms, x_d3, head, 2, k)          # grad mode on, trainable parameters
    want = _module_chain(plan, g.ref_gmms, x_d3, head, k, 2)
    for a, b in zip(preds[1:], want):
        assert torch.equal(a.detach(), b.detach()) and a.requires_grad

    # detach_cost=False with feature maps that require grad, frozen head
    for prm in head.parameters():
        prm.requires_grad_(False)
    rf, sf = g.ref_feat.clone().requires_grad_(True), g.nghbr_feat.clone().requires_grad_(True)
    plan2 = magnet_b200.MatchingPlan(rf, sf, g.nghbr_gmms, g.nghbr_poses, inp.is_valid, inp.cam_intrins, thres=inp.thres)
    preds = matching_loop(plan2, g.ref_gmms, x_d3, head, 2, k, detach_cost=False)
    want = _module_chain(plan2, g.ref_gmms, x_d3, head, k, 2, detach=False)
    for a, b in zip(preds[1:], want):
        assert torch.equal(a.detach(), b.detach()) and a.requires_grad

    # autocast: the module path, whatever the grad mode
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        preds = matching_loop(plan, g.ref_gmms, x_d3, head, 2, k)
        want = _module_chain(plan, g.ref_gmms, x_d3, head, k, 2)
    for a, b in zip(preds[1:], want):
        assert torch.equal(a, b)


def test_dispatch_rule_on_device_tensors(cuda):
    head = _head(8, cuda)
    cv, inv = torch.zeros(1, 8, 4, 4, device=cuda), torch.zeros(1, 128, 4, 4, device=cuda)
    with torch.no_grad():
        assert fused_gnet_applies(head, cv, inv)
    assert not fused_gnet_applies(head, cv, inv)                        # grad mode on, trainable parameters


def test_fused_head_is_deterministic_and_graph_capturable(cuda):
    inp, g, plan, x_d3 = _plan_inputs(cuda, D=64)
    head = _head(64, cuda, seed=6)
    k = inp.k.tolist()
    with torch.no_grad():
        inv = head.invariant_part(x_d3, 64)
        packed = ops.pack_gnet_weights(head, 64)
        eager = [ops.gnet_update(plan.cost(g.ref_gmms, k), inv, packed, g.ref_gmms) for _ in range(2)]
        assert torch.equal(eager[0], eager[1])
        static_in = g.ref_gmms.clone()
        static_out = torch.empty_like(eager[0])
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):                                      # warm-up outside the capture
            ops.gnet_update(plan.cost(static_in, k), inv, packed, static_in, out=static_out)
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            ops.gnet_update(plan.cost(static_in, k), inv, packed, static_in, out=static_out)
        static_out.zero_()
        graph.replay()
        torch.cuda.synchronize()
    assert torch.equal(static_out, eager[0])


def test_non_finite_cost_poisons_only_its_windows(cuda):
    B, D, H, W = 2, 16, 20, 36
    head = _head(D, cuda, seed=8)
    gen = torch.Generator(device=cuda).manual_seed(9)
    cost = torch.randn(B, D, H, W, device=cuda, generator=gen)
    cost[0, 0, 0, 0] = 10.0                       # the largest finite |cost| in both runs: the same scale
    inv = torch.randn(B, 128, H, W, device=cuda, generator=gen)
    prev = _unit_prev(B, H, W, cuda)
    clean = _fused(head, cost, inv, prev)
    bad = cost.clone()
    bad[0, 3, 5, 17] = float("nan")
    bad[1, 15, 0, 35] = float("inf")
    dirty = _fused(head, bad, inv, prev)
    hit = torch.zeros(B, H, W, dtype=torch.bool, device=cuda)
    hit[0, 4:7, 16:19] = True
    hit[1, 0:2, 34:36] = True
    finite = torch.isfinite(dirty).all(1)
    assert not finite[hit].any()
    assert torch.equal(dirty.permute(0, 2, 3, 1)[~hit], clean.permute(0, 2, 3, 1)[~hit])
