"""Two (or more) GPUs, one process each, NCCL: the sharded operator with the fused CUDA kernels.
Run on a multi-GPU box:
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 \
        --master-port 29533 tests/gpu_sharding_nccl.py
Checks, on every rank, against the unsharded fused operator computed locally:
  * batch split + gather=True: the all-gathered output and the gradients of the local shard
  * heads split with single-head keys/values: dk, dv summed over ranks by the all-reduce in the backward
  * context parallelism (the sequence split over the ranks): all-gather of k, v, one fused forward / backward per key
    block, additive merge, reduce-scatter of dk, dv - against the unsharded fused operator on the whole sequence
(The CPU/gloo version of the same logic with the plain operator is tests/test_sharding.py.)"""
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from flash_cosine_sim_attention_b200 import flash_cosine_sim_attention  # noqa: E402
from flash_cosine_sim_attention_b200.sharding import shard_range, sharded_flash_cosine_sim_attention  # noqa: E402


def relerr(a, b):
    a, b = a.detach().float(), b.detach().float()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-6))


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    dev = torch.device("cuda", local)
    dt = torch.bfloat16
    g = torch.Generator().manual_seed(1234)                    # identical tensors on every rank
    worst = 0.0

    # ---- 1. batch split, gathered output -------------------------------------------------------
    B, H, N, D = 2 * world, 4, 384, 64
    q, k, v, do = (torch.randn(B, H, N, D, generator=g).to(dt).to(dev) for _ in range(4))
    qf, kf, vf = (t.clone().requires_grad_() for t in (q, k, v))
    of = flash_cosine_sim_attention(qf, kf, vf, causal=True)
    of.backward(do)
    qs, ks, vs = (t.clone().requires_grad_() for t in (q, k, v))
    o = sharded_flash_cosine_sim_attention(qs, ks, vs, causal=True, gather=True)
    assert o.shape == of.shape
    o.backward(do)
    lo, hi = shard_range(B, rank, world)
    e = [relerr(o, of)] + [relerr(a.grad[lo:hi], b.grad[lo:hi]) for a, b in ((qs, qf), (ks, kf), (vs, vf))]
    # rows of the other ranks get no gradient on this rank
    assert float(qs.grad[:lo].abs().sum() + qs.grad[hi:].abs().sum()) == 0.0
    worst = max(worst, *e)
    # same kernels on the same data: o, dk and dv are bitwise equal; dq is summed by fp32 atomics in no fixed
    # order (DESIGN 4.2), so it is held to the gradient tolerance
    assert torch.equal(o, of), f"batch split: o differs ({e[0]:.3g})"
    assert torch.equal(ks.grad[lo:hi], kf.grad[lo:hi]) and torch.equal(vs.grad[lo:hi], vf.grad[lo:hi]), (
        f"batch split: dk / dv differ ({e[2]:.3g}, {e[3]:.3g})")
    assert e[1] <= 2e-2, f"batch split: dq {e[1]:.3g}"    # TOL_GRAD of bf16 (tests/test_gpu_parity.py)

    # ---- 2. heads split, single-head keys/values: dk, dv all-reduced ---------------------------------
    B, H, N, D = 1, 2 * world, 256, 64
    q = torch.randn(B, H, N, D, generator=g).to(dt).to(dev)
    k, v = (torch.randn(B, N, D, generator=g).to(dt).to(dev) for _ in range(2))
    do = torch.randn(B, H, N, D, generator=g).to(dt).to(dev)
    m = (torch.rand(B, N, generator=g) > 0.3).to(dev)
    m[:, 0] = True
    qf, kf, vf = (t.clone().requires_grad_() for t in (q, k, v))
    of = flash_cosine_sim_attention(qf, kf, vf, mask=m)
    of.backward(do)
    qs, ks, vs = (t.clone().requires_grad_() for t in (q, k, v))
    o = sharded_flash_cosine_sim_attention(qs, ks, vs, mask=m, gather=True)
    o.backward(do)
    lo, hi = shard_range(H, rank, world)
    e = [relerr(o, of), relerr(qs.grad[:, lo:hi], qf.grad[:, lo:hi]), relerr(ks.grad, kf.grad), relerr(vs.grad, vf.grad)]
    worst = max(worst, *e)
    # dk, dv: sum over ranks of per-rank 16-bit partial results vs one fp32 accumulation over all heads
    assert e[0] < 1e-6 and e[1] < 1e-6 and e[2] < 2e-2 and e[3] < 2e-2, f"heads split: {e}"

    # ---- 3. context (sequence) parallelism: one sequence split over the ranks, fused kernels per key block ---------
    from flash_cosine_sim_attention_b200.context_parallel import context_parallel_cosine_sim_attention
    cp_worst = 0.0
    for causal in (True, False):
        B, H, n, D = 2, 4, 384, 64
        N = n * world
        q, k, v, do = (torch.randn(B, H, N, D, generator=g).to(dt).to(dev) for _ in range(4))
        qf, kf, vf = (t.clone().requires_grad_() for t in (q, k, v))
        of = flash_cosine_sim_attention(qf, kf, vf, causal=causal)
        of.backward(do)
        sl = slice(rank * n, (rank + 1) * n)
        ql, kl, vl = (t[:, :, sl].clone().requires_grad_() for t in (q, k, v))
        o = context_parallel_cosine_sim_attention(ql, kl, vl, causal=causal)
        o.backward(do[:, :, sl].contiguous())
        e = [relerr(o, of[:, :, sl]), relerr(ql.grad, qf.grad[:, :, sl]), relerr(kl.grad, kf.grad[:, :, sl]),
             relerr(vl.grad, vf.grad[:, :, sl])]
        cp_worst = max(cp_worst, *e)
        # two roundings apart: per-block 16-bit P / dS vs the single-pass kernel; same operands, fp32 merges
        assert max(e) < 2e-2, f"context parallel (causal={causal}): {e}"
    worst = max(worst, cp_worst)

    t = torch.tensor([worst], device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    if rank == 0:
        print(f"gpu_sharding_nccl ok: world {world}, worst relative error {float(t):.3e}")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
