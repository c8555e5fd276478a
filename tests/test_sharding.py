"""CPU, world_size 2 over gloo: the batch x heads sharding logic (host side of the multi-GPU
path).  The attention itself is the naive formulation here - no GPU in this container."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from flash_cosine_sim_attention_b200 import plain_cosine_sim_attention
from flash_cosine_sim_attention_b200.sharding import plan, shard_range, sharded_flash_cosine_sim_attention


def test_shard_range_partitions_exactly():
    for total in (1, 7, 8, 16, 33):
        for world in (1, 2, 3, 8):
            spans = [shard_range(total, r, world) for r in range(world)]
            assert spans[0][0] == 0 and spans[-1][1] == total
            assert all(a[1] == b[0] for a, b in zip(spans, spans[1:]))
            sizes = [hi - lo for lo, hi in spans]
            assert max(sizes) - min(sizes) <= 1


def test_plan_prefers_batch():
    assert plan(8, 16, 8) == ("batch", 8)        # config 5: one batch element per GPU
    assert plan(4, 8, 8) == ("heads", 8)
    assert plan(4, 8, 2) == ("batch", 4)
    assert plan(3, 5, 2) == ("batch", 3)         # nothing divides: ragged batch split
    assert plan(3, 2, 2) == ("heads", 2)         # the batch does not divide, the heads do


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, case, out):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        g = torch.Generator().manual_seed(0)                     # same full tensors on every rank
        qs, kvs, kw, use_mask = case
        q = torch.randn(qs, generator=g, dtype=torch.float64).requires_grad_()
        k = torch.randn(kvs, generator=g, dtype=torch.float64).requires_grad_()
        v = torch.randn(kvs, generator=g, dtype=torch.float64).requires_grad_()
        do = torch.randn(qs, generator=g, dtype=torch.float64)
        mask = None
        if use_mask:
            mask = torch.rand((qs[0], kvs[-2]), generator=g) > 0.3
            mask[:, 0] = True
        o = sharded_flash_cosine_sim_attention(q, k, v, mask=mask, gather=True,
                                               attn_fn=plain_cosine_sim_attention, **kw)
        (o * do).sum().backward()
        # every rank holds the full output; input grads hold this rank's contribution
        grads = [t.grad.clone() for t in (q, k, v)]
        for gr in grads:
            dist.all_reduce(gr)                                  # sum of per-rank contributions
        q2, k2, v2 = (t.detach().clone().requires_grad_() for t in (q, k, v))
        ref = plain_cosine_sim_attention(q2, k2, v2, mask=mask, **kw)
        (ref * do).sum().backward()
        ok = torch.allclose(o, ref, atol=1e-12)
        # each rank back-propagates only through its own shard, so the per-rank grads sum to the
        # true gradient - except shared keys/values, already all-reduced inside the op (x world)
        for got, want in zip(grads, (q2.grad, k2.grad, v2.grad)):
            ratio = round((got.abs().sum() / want.abs().sum()).item())
            ok = ok and ratio in (1, world) and torch.allclose(got / ratio, want, atol=1e-10)
        out[rank] = bool(ok)
    finally:
        dist.destroy_process_group()


CASES = [
    ((4, 2, 9, 64), (4, 2, 11, 64), dict(causal=True), False),          # batch split
    ((1, 4, 9, 64), (1, 4, 9, 64), dict(groups=2), False),              # heads split, per-head kv
    ((1, 4, 9, 64), (1, 12, 64), dict(), True),                         # heads split, shared kv (all-reduce of dk, dv)
    ((3, 2, 5, 64), (3, 2, 5, 64), dict(scale=2.0), False),             # heads split at B = 3 (plan(3, 2, 2))
    ((6, 7, 64), (6, 7, 64), dict(causal=True), False),                 # merged batch-heads
]


@pytest.mark.parametrize("case", CASES, ids=["batch", "heads", "heads_shared_kv", "heads_batch3", "merged"])
def test_sharded_equals_unsharded_world2(case):
    world = 2
    port = _free_port()
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_worker, args=(world, port, case, out), nprocs=world, join=True)
    assert all(out[r] for r in range(world)), dict(out)


# ---- context (sequence) parallelism: one long sequence split over the ranks -----------------------------------
def _cp_worker(rank, world, port, causal, out):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from flash_cosine_sim_attention_b200.context_parallel import (TorchPrimitives,
                                                                      context_parallel_cosine_sim_attention)
        g = torch.Generator().manual_seed(3)
        B, H, N, D = 2, 3, 24, 16                                   # N split in `world` blocks of 12
        q, k, v, do = (torch.randn(B, H, N, D, generator=g, dtype=torch.float64) for _ in range(4))
        n = N // world
        sl = slice(rank * n, (rank + 1) * n)
        ql, kl, vl = (t[:, :, sl].clone().requires_grad_() for t in (q, k, v))
        prims = TorchPrimitives(scale=8.0, shift=8.0)
        o = context_parallel_cosine_sim_attention(ql, kl, vl, causal=causal, primitives=prims)
        (o * do[:, :, sl]).sum().backward()
        q2, k2, v2 = (t.clone().requires_grad_() for t in (q, k, v))
        ref = plain_cosine_sim_attention(q2, k2, v2, causal=causal)
        (ref * do).sum().backward()
        ok = torch.allclose(o, ref[:, :, sl], atol=1e-12)
        for got, want in ((ql.grad, q2.grad), (kl.grad, k2.grad), (vl.grad, v2.grad)):
            ok = ok and torch.allclose(got, want[:, :, sl], atol=1e-10)
        out[rank] = bool(ok)
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("causal", [False, True])
def test_context_parallel_equals_unsharded_world2(causal):
    """Sequence split over 2 ranks: all-gather of k, v; per-block partial results merged additively (no running
    max); dk, dv returned to their owners by a reduce-scatter.  Outputs and all three gradients of every rank's
    block equal the unsharded naive attention."""
    world = 2
    with mp.Manager() as m:
        out = m.dict()
        mp.spawn(_cp_worker, args=(world, _free_port(), causal, out), nprocs=world, join=True)
        assert all(out[r] for r in range(world)), dict(out)
