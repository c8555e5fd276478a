"""Context (sequence) parallel cosine-sim attention: one long sequence split over the ranks.

Sequence parallelism: the reference has nothing of the kind (README.md:501 only
promises long N).  What makes it easy HERE is the fixed-shift formulation (cu:1216, 1236): a partial result over a
block of keys is the pair
        num_s = sum_{j in block s} p_ij v_j ,   den_s = sum_{j in block s} p_ij        with p_ij = exp(scale q.k - shift)
and partial results simply ADD - no running max, no rescaling when blocks are merged (ring attention for softmax
needs both).  The fused forward already returns o_s = num_s / den_s and inv_l_s = 1 / den_s per call, so

        o = sum_s o_s den_s / sum_s den_s

Layout: rank r owns the r-th contiguous block of the sequence - queries AND keys/values (equal blocks).  Forward:
one all-gather of (k_hat, v), then one fused forward per visible block on the local queries (causal: blocks before
the rank's own are fully visible, its own is the causal diagonal block, later ones are skipped), merged in fp32.
Backward: one fused backward per visible block with the GLOBAL o and 1/den (that is all the closed form needs:
P = p * inv_l, delta = rowsum(dO o), cu:1513-1570), dq summed locally, the per-block dk, dv returned to their owners
with one reduce-scatter.  Collectives are torch.distributed (NCCL over NVLink on GPUs, gloo in the CPU tests): two
per layer and direction-pair, both bandwidth-trivial next to the O(N^2) compute they enable to spread.

The attention itself is pluggable (`primitives`): the fused CUDA kernels by default, a float64 torch restatement
in the CPU tests (tests/test_sharding.py).
"""
import torch
import torch.distributed as dist
from torch.autograd import Function

__all__ = ["context_parallel_cosine_sim_attention", "TorchPrimitives", "FusedPrimitives"]


class FusedPrimitives:
    """(o, inv_l) = forward(q_hat, k_hat, v, causal) and (dq, dk, dv) = backward(...) on the sm_90a kernels, with the
    unrounded fp32 `o` of the partial results (out_f32) so that the merge adds no rounding of its own."""

    def __init__(self, scale, shift):
        self.scale, self.shift = float(scale), float(shift)

    def forward(self, q, k, v, causal):
        from .flash_cosine_sim_attention import _ext
        o, inv_l = _ext().forward_ex(q, k, v, None, None, False, None, self.scale, self.shift, causal, 0, True, True)[:2]
        # the extension returns inv_l as (B, H, N), H = 1 for merged (B*H, N, D) inputs; the merge broadcasts it
        # against o, so it takes q's row shape (the backward reads only its pointer)
        return o, inv_l.view(q.shape[:-1])

    def backward(self, do, o, inv_l, q, k, v, causal):
        # o: the merged output in fp32; dq, dk, dv come back in fp32 (out_f32) so that the sums over blocks and
        # over ranks (reduce-scatter) are fp32 sums, rounded once at the very end
        from .flash_cosine_sim_attention import _ext
        return _ext().backward_ex(do, o, inv_l, q, k, v, None, None, None, None, False, None, False, None,
                                  self.scale, self.shift, causal, 0, True)[:3]


class TorchPrimitives:
    """The same two primitives as plain torch ops in the tensors' own dtype (float64 in the CPU tests): forward of
    cu:1216-1246, closed-form backward of cu:1487-1626.  Test infrastructure for the merge / collective logic."""

    def __init__(self, scale, shift):
        self.scale, self.shift = float(scale), float(shift)

    def _p(self, q, k, causal):
        s = torch.matmul(q, k.transpose(-1, -2)) * self.scale - self.shift
        p = torch.exp(s)
        if causal:
            i, j = p.shape[-2:]
            p = p.masked_fill(torch.ones(i, j, dtype=torch.bool, device=p.device).triu(j - i + 1), 0.0)
        return p

    def forward(self, q, k, v, causal):
        p = self._p(q, k, causal)
        l = p.sum(-1)
        inv_l = 1.0 / l.clamp_min(1e-300)
        return torch.matmul(p, v) * inv_l[..., None], inv_l

    def backward(self, do, o, inv_l, q, k, v, causal):
        P = self._p(q, k, causal) * inv_l[..., None]
        delta = (do * o).sum(-1, keepdim=True)
        dv = torch.matmul(P.transpose(-1, -2), do)
        dS = P * (torch.matmul(do, v.transpose(-1, -2)) - delta)
        return self.scale * torch.matmul(dS, k), self.scale * torch.matmul(dS.transpose(-1, -2), q), dv


def _wide(t):
    """16-bit partial results are accumulated in fp32; fp32 / fp64 stay as they are."""
    return t.float() if t.dtype in (torch.float16, torch.bfloat16) else t


def _reduce_scatter_blocks(blocks, rank, group):
    """Sum block s over the ranks and hand it to rank s.  NCCL: one reduce-scatter; gloo (CPU tests) has none:
    all-reduce of the stack, keep the own block."""
    if dist.get_backend(group) == "gloo":
        stack = torch.stack(blocks)
        dist.all_reduce(stack, op=dist.ReduceOp.SUM, group=group)
        return stack[rank].clone()
    out = torch.empty_like(blocks[rank])
    dist.reduce_scatter(out, blocks, op=dist.ReduceOp.SUM, group=group)
    return out


class _ContextParallel(Function):
    @staticmethod
    def forward(ctx, q, k, v, causal, prims, group):
        world = dist.get_world_size(group)
        rank = dist.get_rank(group)
        k, v = k.contiguous(), v.contiguous()
        ks = [torch.empty_like(k) for _ in range(world)]
        vs = [torch.empty_like(v) for _ in range(world)]
        dist.all_gather(ks, k, group=group)                 # every rank needs every key block: ONE collective each
        dist.all_gather(vs, v, group=group)
        num = den = None
        for s in range(world):
            if causal and s > rank:
                continue                                    # a later block: nothing visible to these queries
            o_s, inv_l_s = prims.forward(q, ks[s], vs[s], causal and s == rank)
            den_s = 1.0 / inv_l_s
            num_s = _wide(o_s).to(den_s.dtype) * den_s[..., None]
            num = num_s if num is None else num + num_s
            den = den_s if den is None else den + den_s
        inv_l = 1.0 / den
        o_wide = num * inv_l[..., None]                      # fp32 (fp64 in the CPU tests): what the backward reads
        ctx.save_for_backward(o_wide, inv_l, q, *ks, *vs)
        ctx.meta = (causal, prims, group, world, rank, k.dtype)
        return o_wide.to(q.dtype)

    @staticmethod
    def backward(ctx, do):
        causal, prims, group, world, rank, kv_dtype = ctx.meta
        saved = ctx.saved_tensors
        o, inv_l, q = saved[:3]
        ks, vs = saved[3:3 + world], saved[3 + world:]
        do = do.contiguous()
        inv_l_k = inv_l
        wide = o.dtype
        dq = None
        dks, dvs = [], []
        for s in range(world):
            if causal and s > rank:
                dks.append(torch.zeros(ks[s].shape, dtype=wide, device=do.device))
                dvs.append(torch.zeros(vs[s].shape, dtype=wide, device=do.device))
                continue
            dq_s, dk_s, dv_s = prims.backward(do, o, inv_l_k, q, ks[s], vs[s], causal and s == rank)
            dq = _wide(dq_s) if dq is None else dq + _wide(dq_s)
            dks.append(dk_s.to(wide).contiguous())
            dvs.append(dv_s.to(wide).contiguous())
        # the gradients of block s belong to rank s: sum over the ranks that saw the block, deliver to the owner
        dk = _reduce_scatter_blocks(dks, rank, group)
        dv = _reduce_scatter_blocks(dvs, rank, group)
        return dq.to(q.dtype), dk.to(kv_dtype), dv.to(kv_dtype), None, None, None


def context_parallel_cosine_sim_attention(q, k, v, *, scale=8, groups=1, causal=False, l2norm_qk=True, group=None,
                                          primitives=None, window=None):
    """q, k, v: THIS RANK'S contiguous block of the sequence, (batch, heads, n_local, dim) or merged
    (batch*heads, n_local, dim), equal n_local on every rank (block r = positions [r n_local, (r+1) n_local)).
    Returns this rank's block of the output; gradients flow to the local q, k, v.  Key-padding masks / attn_bias are
    not supported on this path.

    With the fused kernels (primitives=None) the inputs must be float16 or bfloat16 CUDA tensors with head dim 64 or
    128; anything else is rejected here, before any collective.  float16 warns where exp(scale*q.k - shift) can exceed
    its range (as `flash_cosine_sim_attention` does).  Sliding-window attention (`window`) is not supported on this
    path and is rejected before any collective."""
    from .flash_cosine_sim_attention import (_KERNEL_DTYPES, _KERNEL_HEAD_DIMS, _choose_shift, _warn_fp16_overflow,
                                             l2norm_tensors)
    if window is not None:
        raise NotImplementedError("context_parallel_cosine_sim_attention: window (sliding-window attention) is not "
                                  "supported with context parallelism")
    assert dist.is_initialized(), "context parallelism needs an initialised process group"
    assert q.shape[-2] == k.shape[-2] == v.shape[-2], "every rank holds the same number of queries and keys"
    assert k.shape[:-2] == q.shape[:-2] and v.shape[:-2] == q.shape[:-2], (
        "context parallelism needs keys/values with as many heads as the queries (grouped-query or single-head "
        "keys/values are not supported on this path: expand them with repeat_interleave first)")
    if primitives is None:
        if q.dtype not in _KERNEL_DTYPES or k.dtype != q.dtype or v.dtype != q.dtype:
            raise TypeError(f"context_parallel_cosine_sim_attention: dtype {q.dtype} (k {k.dtype}, v {v.dtype}) is not "
                            "supported: q, k, v must all be float16 or all bfloat16 (no float32 on this path)")
        if q.shape[-1] not in _KERNEL_HEAD_DIMS:
            raise NotImplementedError(f"context_parallel_cosine_sim_attention: head dim {q.shape[-1]} is not "
                                      "supported: 64 or 128 only")
        if not (q.is_cuda and k.is_cuda and v.is_cuda):
            raise RuntimeError("context_parallel_cosine_sim_attention: CUDA tensors required (the fused kernels)")
        _warn_fp16_overflow(q.dtype, scale, groups, l2norm_qk)
    if l2norm_qk:
        q, k = l2norm_tensors(q, k, groups=groups)        # per row: local, differentiable (fused kernels on CUDA)
    if primitives is None:
        shift = _choose_shift(q.dtype, scale, groups if l2norm_qk else 1, l2norm_qk)
        primitives = FusedPrimitives(scale, shift)
    return _ContextParallel.apply(q, k, v, bool(causal), primitives, group)
