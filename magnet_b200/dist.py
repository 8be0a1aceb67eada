"""Multi-GPU plumbing for the matching path (SURVEY §8 e): one process per GPU, batch elements sharded
across ranks with NO data-path collective; for head training one flat-bucket gradient all-reduce
(replaces DistributedDataParallel's bucketed all-reduce, train_MaGNet.py:209-210 — the trainable set is
~0.75 M fp32 parameters = 3 MB, latency-bound, so a single bucket is the right shape).
"""
from __future__ import annotations

import os
from typing import Iterable, List, Tuple

import torch
import torch.distributed as dist


def env_world() -> Tuple[int, int, int]:
    """(rank, local_rank, world_size) from the torchrun environment; (0, 0, 1) when absent."""
    return (int(os.environ.get("RANK", 0)), int(os.environ.get("LOCAL_RANK", 0)),
            int(os.environ.get("WORLD_SIZE", 1)))


def init_process_group(backend: str | None = None, device_id=None) -> Tuple[int, int, int]:
    rank, local_rank, world = env_world()
    if world > 1 and not dist.is_initialized():
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29511")
        kw = {"device_id": device_id} if (device_id is not None and backend == "nccl") else {}
        dist.init_process_group(backend=backend, rank=rank, world_size=world, **kw)
    return rank, local_rank, world


def shutdown() -> None:
    if dist.is_available() and dist.is_initialized():
        dist.destroy_process_group()


def shard_range(total: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous [lo, hi) slice of ``total`` independent batch elements owned by ``rank``;
    sizes differ by at most one and cover the range exactly."""
    base, rem = divmod(total, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def max_over_ranks(value: float, device=None) -> float:
    """Max over ranks of a device-measured time (multi-GPU numbers are max over ranks, never wall clock)."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return float(value)
    t = torch.tensor([float(value)], dtype=torch.float64, device=device or ("cuda" if dist.get_backend() == "nccl" else "cpu"))
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def sum_over_ranks(value: float, device=None) -> float:
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return float(value)
    t = torch.tensor([float(value)], dtype=torch.float64, device=device or ("cuda" if dist.get_backend() == "nccl" else "cpu"))
    dist.all_reduce(t, op=dist.ReduceOp.SUM)
    return float(t.item())


def gather_over_ranks(values, device=None):
    """Every rank's list of floats, as a list (one entry per rank) of lists — for per-rank diagnostics next to a
    max-over-ranks number (which rank was the slow one, at which clock)."""
    vals = [float(v) for v in values]
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return [vals]
    t = torch.tensor(vals, dtype=torch.float64, device=device or ("cuda" if dist.get_backend() == "nccl" else "cpu"))
    out = [torch.empty_like(t) for _ in range(dist.get_world_size())]
    dist.all_gather(out, t)
    return [[float(x) for x in o.tolist()] for o in out]


def barrier() -> None:
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        dist.barrier()


class FlatGradAllReduce:
    """Average the gradients of ``params`` across ranks with ONE all-reduce over a flat fp32 bucket."""

    def __init__(self, params: Iterable[torch.nn.Parameter]):
        self.params: List[torch.nn.Parameter] = [p for p in params if p.requires_grad]
        n = sum(p.numel() for p in self.params)
        dev = self.params[0].device if self.params else "cpu"
        self.bucket = torch.zeros(n, dtype=torch.float32, device=dev)

    @torch.no_grad()
    def broadcast_parameters(self, src: int = 0) -> None:
        if not (dist.is_initialized() and dist.get_world_size() > 1):
            return
        flat = torch.cat([p.detach().reshape(-1) for p in self.params]) if self.params else self.bucket
        dist.broadcast(flat, src=src)
        off = 0
        for p in self.params:
            p.copy_(flat[off:off + p.numel()].view_as(p))
            off += p.numel()

    @torch.no_grad()
    def __call__(self) -> None:
        if not (dist.is_initialized() and dist.get_world_size() > 1):
            return
        off = 0
        for p in self.params:
            g = p.grad if p.grad is not None else torch.zeros_like(p)
            self.bucket[off:off + p.numel()].copy_(g.reshape(-1))
            off += p.numel()
        dist.all_reduce(self.bucket, op=dist.ReduceOp.SUM)
        self.bucket.div_(dist.get_world_size())
        off = 0
        for p in self.params:
            if p.grad is None:
                p.grad = torch.empty_like(p)
            p.grad.copy_(self.bucket[off:off + p.numel()].view_as(p))
            off += p.numel()


def sum_tensor_over_ranks_(t: torch.Tensor) -> torch.Tensor:
    """In-place sum of ``t`` over ranks (a no-op in a single process).  NCCL reduces device tensors where they are;
    other backends reduce a host copy, which is written back."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return t
    if dist.get_backend() == "nccl" or not t.is_cuda:
        dist.all_reduce(t, op=dist.ReduceOp.SUM)
    else:
        h = t.cpu()
        dist.all_reduce(h, op=dist.ReduceOp.SUM)
        t.copy_(h)
    return t
