"""Batch data-parallelism of the hot path over the GPUs of one box (SURVEY.md 8e).

Samples are independent everywhere (GroupNorm per sample, LayerNorm per position, attention
per sample), so inference shards the batch with NO collective; training adds one gradient
all-reduce (NCCL over NVLink) -- either torch DDP around `DiffusionModel`, or the explicit
flat-bucket `allreduce_gradients` below.  One process per GPU (torchrun)."""
from typing import Iterable, List, Optional

import torch
import torch.distributed as dist
from torch import Tensor


def shard_bounds(n: int, rank: int, world: int):
    """Contiguous, balanced split of n items: first (n % world) ranks get one extra."""
    base, extra = divmod(n, world)
    start = rank * base + min(rank, extra)
    return start, start + base + (1 if rank < extra else 0)


def shard_batch(t: Tensor, rank: Optional[int] = None, world: Optional[int] = None) -> Tensor:
    rank = dist.get_rank() if rank is None else rank
    world = dist.get_world_size() if world is None else world
    lo, hi = shard_bounds(t.shape[0], rank, world)
    return t[lo:hi]


def gather_batch(local: Tensor, total: int) -> Tensor:
    """Inverse of shard_batch (ragged shards allowed): every rank gets the full batch."""
    world, rank = dist.get_world_size(), dist.get_rank()
    sizes = [shard_bounds(total, r, world)[1] - shard_bounds(total, r, world)[0] for r in range(world)]
    pad = max(sizes)
    buf = local.new_zeros((pad,) + tuple(local.shape[1:]))
    buf[: local.shape[0]] = local
    out = [torch.empty_like(buf) for _ in range(world)]
    dist.all_gather(out, buf)
    return torch.cat([o[:s] for o, s in zip(out, sizes)], dim=0)


@torch.no_grad()
def sample_sharded(model, noise: Tensor, num_steps: int, gather: bool = True, **kwargs) -> Tensor:
    """Each rank runs VSampler on its slice of the batch; no communication inside the loop."""
    rank, world = dist.get_rank(), dist.get_world_size()
    lo, hi = shard_bounds(noise.shape[0], rank, world)
    kw = {k: (v[lo:hi] if torch.is_tensor(v) and v.shape[:1] == noise.shape[:1] else v)
          for k, v in kwargs.items()}
    local = model.sample(noise[lo:hi], num_steps=num_steps, **kw)
    return gather_batch(local, noise.shape[0]) if gather else local


@torch.no_grad()
def allreduce_gradients(params: Iterable[torch.nn.Parameter], bucket_mb: float = 256.0) -> None:
    """Mean of `.grad` over ranks in flat buckets (each shard's loss is a mean over its own
    samples, so averaging equal-sized shards gives the global-batch gradient)."""
    world = dist.get_world_size()
    bucket: List[Tensor] = []
    nbytes = 0

    def flush():
        nonlocal bucket, nbytes
        if not bucket:
            return
        flat = torch.cat([g.reshape(-1) for g in bucket])
        dist.all_reduce(flat)
        flat.div_(world)
        off = 0
        for g in bucket:
            g.copy_(flat[off:off + g.numel()].view_as(g))
            off += g.numel()
        bucket, nbytes = [], 0

    for p in params:
        if p.grad is None:
            continue
        bucket.append(p.grad)
        nbytes += p.grad.numel() * p.grad.element_size()
        if nbytes >= bucket_mb * 2 ** 20:
            flush()
    flush()


# ----------------------------------------------------------------- overlapped gradient all-reduce
def merge_intervals(intervals):
    """Union of half-open [a, b) ranges as a sorted list of maximal ranges."""
    out: List[List[int]] = []
    for a, b in sorted((int(a), int(b)) for a, b in intervals if b > a):
        if out and a <= out[-1][1]:
            out[-1][1] = max(out[-1][1], b)
        else:
            out.append([a, b])
    return [(a, b) for a, b in out]


def bucket_schedule(marks, bucket_elems: int):
    """marks: gradient-arena ranges in the order the backward program completes them.  Returns
    {index of the mark after which to communicate: [maximal contiguous ranges]} such that every
    flush carries >= bucket_elems elements (the last one takes the remainder)."""
    sched, pending, size = {}, [], 0
    for i, (a, b) in enumerate(marks):
        pending.append((a, b))
        size += b - a
        if size >= bucket_elems or i == len(marks) - 1:
            merged = merge_intervals(pending)
            if merged:
                sched[i] = merged
            pending, size = [], 0
    return sched


class _Done:
    def wait(self):
        return True


def average_async(t: Tensor, group=None):
    """In-place mean over ranks; returns a handle with .wait().  NCCL: ReduceOp.AVG, asynchronous
    on NCCL's stream.  Other backends (gloo in the CPU tests): sum, then scale, synchronously."""
    if dist.get_backend(group) == "nccl":
        return dist.all_reduce(t, op=dist.ReduceOp.AVG, group=group, async_op=True)
    dist.all_reduce(t, group=group)
    t.div_(dist.get_world_size(group))
    return _Done()


class GradSync:
    """Attached to a B200UNet (`net._grad_sync`) by OverlappedDataParallel: training.py calls it
    from inside the backward program."""

    def __init__(self, process_group=None, bucket_mb: float = 64.0):
        self.group = process_group
        self.bucket_elems = int(bucket_mb * 2 ** 20 / 4)
        self.world = dist.get_world_size(process_group)

    def flush_schedule(self, plan):
        if not plan.mark_log:
            return None
        if getattr(plan, "_flush", None) is None:
            plan._flush = bucket_schedule(plan.mark_log, self.bucket_elems)
        return plan._flush

    def all_reduce_async(self, t: Tensor):
        return average_async(t, self.group)

    @torch.no_grad()
    def conditioning_gradients(self, plan) -> None:
        """dW_cond / db_cond averaged over ranks WITHOUT all-reducing the [47 K x 1024] matrix:
        gather the rank-B factors (dss [B, n], cond [B, 1024]) and redo the small product."""
        from . import ops
        if plan.n_tot == 0:              # use_modulation=False: no conditioning projection
            return
        B, Fm = plan.cond.shape
        n = plan.dss_all.shape[1]
        dss_g = torch.empty(self.world * B, n, device=plan.dss_all.device)
        cond_g = torch.empty(self.world * B, Fm, device=plan.dss_all.device)
        dist.all_gather_into_tensor(dss_g, plan.dss_all.contiguous(), group=self.group)
        dist.all_gather_into_tensor(cond_g, plan.cond_bf.view(B, Fm).float(), group=self.group)
        # d cond is a local quantity (already computed by the backward program): not wanted here
        ops.cond_bwd(dss_g, cond_g, plan.P["cond_w"], plan.dw_all, plan.dbias_all, None, plan.n_tot)
        plan.dw_all.div_(self.world)
        plan.dbias_all.div_(self.world)


class OverlappedDataParallel(torch.nn.Module):
    """Data parallelism for the training step of the CUDA path (SURVEY.md 8e): replicas + ONE
    gradient average per step over NCCL, overlapped with the hand-written backward program.

        ddp = OverlappedDataParallel(model)            # broadcasts rank 0's weights
        loss = ddp(x); loss.backward(); ddp.finish_gradient_sync(); opt.step()

    The U-Net's gradients are averaged inside `loss.backward()` (bucketed, each bucket's all-reduce
    issued as soon as the backward program has finished it); `finish_gradient_sync()` averages the
    handful of parameters whose gradients come from PyTorch autograd (time-embedding MLP, the
    vocoder's `to_flat`, the guidance mask embedding).  Every backward synchronises (no `no_sync`
    gradient accumulation)."""

    def __init__(self, module: torch.nn.Module, process_group=None, bucket_mb: float = 64.0):
        super().__init__()
        from .unet import B200UNet
        self.module = module
        self.group = process_group
        nets = [m for m in module.modules() if isinstance(m, B200UNet)]
        assert len(nets) == 1, "OverlappedDataParallel wraps a model with exactly one B200UNet"
        self.net = nets[0]
        self.net._grad_sync = GradSync(process_group, bucket_mb)
        with torch.no_grad():
            for p in module.parameters():
                dist.broadcast(p, src=0, group=process_group)
        from .training import _net_params
        inside = {id(p) for p in _net_params(self.net)}
        self.outside = [p for p in module.parameters() if id(p) not in inside]

    def forward(self, *args, **kwargs):
        return self.module(*args, **kwargs)

    @torch.no_grad()
    def finish_gradient_sync(self) -> None:
        grads = [p.grad for p in self.outside if p.grad is not None]
        if not grads:
            return
        flat = torch.cat([g.reshape(-1) for g in grads])
        average_async(flat, self.group).wait()
        off = 0
        for g in grads:
            g.copy_(flat[off:off + g.numel()].view_as(g))
            off += g.numel()
