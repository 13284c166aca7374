# -*- coding: utf-8 -*-
"""Data parallelism for the H100 build: one process per GPU (torch.distributed, NCCL over NVLink; gloo in the CPU tests)
instead of the reference's single-process `nn.DataParallel` (lfd/execution/executor.py:39).

Inference shards the batch across ranks with no collective.  Training reduces gradients with ONE all-reduce over a single
flat bucket (the model has 1.2-1.9 M parameters, 5-7.5 MB fp32: latency bound on NVSwitch) and normalises the loss by the
GLOBAL number of positives like the reference does after its DataParallel gather (lfd/model/lfd.py:323,340,383).
"""
import torch
import torch.distributed as dist

__all__ = ['world', 'shard_range', 'shard_batch', 'allreduce_gradients', 'allreduce_scalar', 'broadcast_module_state']


def world():
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


def shard_range(total, rank, world_size):
    """Contiguous [begin, end) of `total` items owned by `rank`; sizes differ by at most one, earlier ranks get the extras."""
    base, extra = divmod(total, world_size)
    begin = rank * base + min(rank, extra)
    return begin, begin + base + (1 if rank < extra else 0)


def shard_batch(batch, rank=None, world_size=None):
    """Slice every element of a (image_batch, annotation_batch, meta_batch) tuple along the batch dimension."""
    r, w = world()
    rank = r if rank is None else rank
    world_size = w if world_size is None else world_size
    n = len(batch[1]) if len(batch) > 1 else len(batch[0])
    b, e = shard_range(n, rank, world_size)
    return tuple(x[b:e] for x in batch)


def allreduce_scalar(value, op='sum'):
    r, w = world()
    if w == 1:
        return value
    t = torch.as_tensor([float(value)], dtype=torch.float64)
    if dist.get_backend() == 'nccl':
        t = t.cuda()
    dist.all_reduce(t, op=dist.ReduceOp.SUM if op == 'sum' else dist.ReduceOp.MAX)
    return float(t.item())


def allreduce_gradients(parameters, average=True):
    """One all-reduce over a single flat bucket holding every gradient; returns the bucket size in elements.
    Parameters without a gradient contribute zeros so that every rank reduces the same layout."""
    r, w = world()
    params = [p for p in parameters if p.requires_grad]
    if w == 1 or not params:
        return sum(p.numel() for p in params)
    flat = torch.cat([(p.grad if p.grad is not None else torch.zeros_like(p)).reshape(-1).float() for p in params])
    dist.all_reduce(flat, op=dist.ReduceOp.SUM)
    if average:
        flat /= w
    off = 0
    for p in params:
        n = p.numel()
        g = flat[off:off + n].view_as(p).to(p.dtype)
        if p.grad is None:
            p.grad = g.clone()
        else:
            p.grad.copy_(g)
        off += n
    return off


def broadcast_module_state(module, src=0):
    """Every parameter and buffer of `module` takes rank `src`'s value (one flat bucket per dtype).  No-op for one process."""
    r, w = world()
    if w == 1:
        return 0
    tensors = [p.data for p in module.parameters()] + [b.data for b in module.buffers()]
    seen, uniq = set(), []
    for t in tensors:                       # shared tensors (share_head_flag aliases) travel once
        if t.data_ptr() not in seen and t.numel():
            seen.add(t.data_ptr())
            uniq.append(t)
    n = 0
    for dt in sorted(set(t.dtype for t in uniq), key=str):
        group = [t for t in uniq if t.dtype == dt]
        flat = torch.cat([t.reshape(-1) for t in group])
        dist.broadcast(flat, src)
        off = 0
        for t in group:
            t.copy_(flat[off:off + t.numel()].view_as(t))
            off += t.numel()
        n += off
    return n
