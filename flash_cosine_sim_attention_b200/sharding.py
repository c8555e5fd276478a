"""Multi-GPU use of the operator: one process per GPU, batch x heads sharding.

The reference has no distributed code at all.  Every (batch, head) pair is an
independent attention problem (reference grid dims: flash_cosine_sim_attention_cuda.cu:1091-1092,
1366-1367), so the path shards with NO collective on the data path: each rank runs the fused
kernels on its slice.  Collectives (torch.distributed; NCCL over NVLink on GPUs, gloo in the CPU
tests) appear only at the edges, and only when asked for:

  * gather=True         one all-gather of `o` when the caller wants the whole-batch output
  * heads split while   the keys/values are shared by all heads (3-D k, v): their gradients are
    kv is single-headed  summed over ranks with one all-reduce in the backward

Partitioning: batch first (config 5: 8 batch elements -> one per GPU); if the batch does not
divide over the ranks, heads are split instead.
"""
import torch
import torch.distributed as dist
from torch.autograd import Function

from .flash_cosine_sim_attention import flash_cosine_sim_attention


def shard_range(total, rank, world):
    """Contiguous, balanced [lo, hi) slice of range(total) for `rank` of `world`."""
    base, rem = divmod(total, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def plan(batch, heads, world, kv_heads=None):
    """('batch' | 'heads', size of the sharded dim).  Batch is preferred (keeps single-head
    keys/values local); heads are used when the batch does not divide evenly but heads do.
    With grouped-query keys/values (1 < kv_heads < heads) heads are split only when the kv heads
    divide over the ranks too, so that every query head's group stays on one rank."""
    if batch % world == 0 or heads % world != 0:
        return "batch", batch
    if kv_heads not in (None, 1, heads) and kv_heads % world != 0:
        return "batch", batch
    return "heads", heads


class _AllGather(Function):
    """All-gather along `dim` (equal-sized or ragged shards); backward returns this rank's slice."""

    @staticmethod
    def forward(ctx, x, dim, sizes, rank, group):
        ctx.dim, ctx.sizes, ctx.rank = dim, sizes, rank
        parts = []
        for s in sizes:
            shape = list(x.shape)
            shape[dim] = s
            parts.append(torch.empty(shape, dtype=x.dtype, device=x.device))
        dist.all_gather(parts, x.contiguous(), group=group)
        return torch.cat(parts, dim=dim)

    @staticmethod
    def backward(ctx, g):
        lo = sum(ctx.sizes[:ctx.rank])
        return g.narrow(ctx.dim, lo, ctx.sizes[ctx.rank]).contiguous(), None, None, None, None


class _SharedAcrossRanks(Function):
    """Identity in the forward; sums the gradient over ranks in the backward.  Wraps keys/values
    that every rank reads in full while query heads are split."""

    @staticmethod
    def forward(ctx, x, group):
        ctx.group = group
        return x.view_as(x)

    @staticmethod
    def backward(ctx, g):
        g = g.contiguous()
        dist.all_reduce(g, op=dist.ReduceOp.SUM, group=ctx.group)
        return g, None


def local_shard(t, rank, world, dim=0):
    """This rank's contiguous slice of `t` along `dim` (the batch dimension by default): what a
    data-parallel rank holds when the global batch is split over the ranks."""
    lo, hi = shard_range(t.shape[dim], rank, world)
    return t.narrow(dim, lo, hi - lo)


def sharded_flash_cosine_sim_attention(q, k, v, mask=None, *, gather=False, group=None, attn_fn=None,
                                       presharded=False, **kwargs):
    """Run this rank's (batch x heads) shard of the attention; q, k, v, mask are the FULL tensors
    (identical on every rank).  Returns the local output shard, or the full output if gather=True.

    presharded=True: q, k, v, mask are ALREADY this rank's batch shard (the usual data-parallel
    situation: every rank owns its batch elements, equal counts per rank) - nothing is sliced, gradients
    have the shard's size, and the only possible collective is the optional all-gather of `o`.

    attn_fn defaults to the fused CUDA operator; the CPU tests pass plain_cosine_sim_attention."""
    attn_fn = attn_fn or flash_cosine_sim_attention
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    if presharded:
        o = attn_fn(q, k, v, mask=mask, **kwargs)
        if gather and world > 1:
            o = _AllGather.apply(o, 0, [q.shape[0]] * world, rank, group)
        return o
    if q.ndim == 3 or world == 1:
        dim, total = 0, q.shape[0]                      # merged batch-heads: plain batch split
        kind = "batch"
    else:
        kind, total = plan(q.shape[0], q.shape[1], world, kv_heads=k.shape[1] if k.ndim == 4 else None)
        dim = 0 if kind == "batch" else 1
    lo, hi = shard_range(total, rank, world)
    sizes = [shard_range(total, r, world)[1] - shard_range(total, r, world)[0] for r in range(world)]

    ql = q.narrow(dim, lo, hi - lo)
    if kind == "batch":
        kl, vl = k.narrow(0, lo, hi - lo), v.narrow(0, lo, hi - lo)
        ml = mask.narrow(0, lo, hi - lo) if mask is not None else None
    else:
        ml = mask
        if k.ndim == 3:                                  # one kv head read by all ranks
            kl = _SharedAcrossRanks.apply(k, group) if world > 1 else k
            vl = _SharedAcrossRanks.apply(v, group) if world > 1 else v
        elif k.shape[1] == q.shape[1]:
            kl, vl = k.narrow(1, lo, hi - lo), v.narrow(1, lo, hi - lo)
        else:                                            # grouped-query: this rank's whole groups
            klo, khi = shard_range(k.shape[1], rank, world)
            kl, vl = k.narrow(1, klo, khi - klo), v.narrow(1, klo, khi - klo)
    if hi - lo == 0:
        o = q.new_zeros(ql.shape)
    else:
        o = attn_fn(ql, kl, vl, mask=ml, **kwargs)
    if gather and world > 1:
        o = _AllGather.apply(o, dim, sizes, rank, group)
    return o
