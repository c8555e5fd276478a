"""CPU: grouped-query attention (kv_heads dividing heads) in everything that runs without a GPU - the plain PyTorch
formulation (against the repeated-keys computation and the float64 oracle), shape canonicalisation, the C ABI's
problem check and workspace size, and the batch x heads sharding over gloo."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from flash_cosine_sim_attention_b200 import _abi, plain_cosine_sim_attention
from flash_cosine_sim_attention_b200.flash_cosine_sim_attention import _Shapes
from flash_cosine_sim_attention_b200.sharding import plan, sharded_flash_cosine_sim_attention
from gqa_reference import gqa_attention

# (heads, kv_heads, keyword arguments, key-padding mask, attn_bias: None | "heads" | "batch")
CASES = [
    (4, 2, dict(causal=True), False, None),
    (6, 3, dict(groups=2), True, None),
    (8, 2, dict(scale=4), False, "heads"),
    (6, 2, dict(causal=True), False, "batch"),
    (4, 1, dict(), True, None),                  # 4-D keys/values with one head
]
IDS = ["h4_kv2_causal", "h6_kv3_mask_groups2", "h8_kv2_bias_heads", "h6_kv2_bias_batch", "h4_kv1_4d"]


def _inputs(B, H, Hk, Nq, Nk, D, mask, bias, seed=0):
    g = np.random.default_rng(seed)
    q = g.standard_normal((B, H, Nq, D))
    k = g.standard_normal((B, Hk, Nk, D))
    v = g.standard_normal((B, Hk, Nk, D))
    do = g.standard_normal((B, H, Nq, D))
    m = None
    if mask:
        m = g.random((B, Nk)) > 0.3
        m[:, 0] = True
    b = None
    if bias is not None:
        b = g.standard_normal((B if bias == "batch" else H, Nq, Nk))
    return q, k, v, do, m, b


@pytest.mark.parametrize("H,Hk,kw,mask,bias", CASES, ids=IDS)
def test_plain_gqa_equals_expanded_and_oracle(H, Hk, kw, mask, bias):
    B, Nq, Nk, D = 2, 9, 13 if not kw.get("causal") else 9, 16
    q, k, v, do, m, b = _inputs(B, H, Hk, Nq, Nk, D, mask, bias, seed=1)
    G = H // Hk
    t = lambda x: torch.tensor(x, dtype=torch.float64, requires_grad=True)
    mt = None if m is None else torch.tensor(m)
    extra = dict(mask=mt, attn_bias_batch_dim=bias == "batch", **kw)
    q1, k1, v1 = t(q), t(k), t(v)
    b1 = None if b is None else t(b)
    o1 = plain_cosine_sim_attention(q1, k1, v1, attn_bias=b1, **extra)
    (o1 * torch.tensor(do)).sum().backward()
    q2, k2, v2 = t(q), t(k), t(v)
    b2 = None if b is None else t(b)
    o2 = plain_cosine_sim_attention(q2, k2.repeat_interleave(G, dim=1), v2.repeat_interleave(G, dim=1),
                                    attn_bias=b2, **extra)
    (o2 * torch.tensor(do)).sum().backward()
    assert o1.shape == (B, H, Nq, D)
    torch.testing.assert_close(o1, o2, rtol=0, atol=1e-12)
    for x1, x2 in ((q1, q2), (k1, k2), (v1, v2)) + (((b1, b2),) if b is not None else ()):
        assert x1.grad.shape == x1.shape
        torch.testing.assert_close(x1.grad, x2.grad, rtol=0, atol=1e-12)
    # and the float64 oracle, through the group reference (the plain path gives rows with no visible key the mean
    # of v; none here)
    ref = gqa_attention(q, k, v, mask=m, attn_bias=b, attn_bias_batch_dim=bias == "batch", d_out=do, **kw)
    np.testing.assert_allclose(o1.detach().numpy(), ref[0], rtol=0, atol=1e-12)
    np.testing.assert_allclose(k1.grad.numpy(), ref[2], rtol=0, atol=1e-12)


def test_plain_rejects_bad_kv_heads():
    q = torch.randn(1, 6, 5, 16)
    with pytest.raises(ValueError, match="kv_heads"):
        plain_cosine_sim_attention(q, torch.randn(1, 4, 5, 16), torch.randn(1, 4, 5, 16))
    with pytest.raises(ValueError, match="kv_heads"):
        plain_cosine_sim_attention(q, torch.randn(1, 3, 5, 16), torch.randn(1, 2, 5, 16))


def test_shapes_gqa():
    q = torch.empty(2, 8, 10, 64)
    s = _Shapes(q, torch.empty(2, 2, 12, 64), torch.empty(2, 2, 12, 64))
    assert (s.B, s.H, s.kv_heads, s.Nq, s.Nk, s.D, s.merged, s.kkind) == (2, 8, 2, 10, 12, 64, False, "bhnd")
    s = _Shapes(q, torch.empty(2, 8, 12, 64), torch.empty(2, 8, 12, 64))
    assert s.kv_heads == 8
    with pytest.raises(ValueError, match="kv_heads"):
        _Shapes(q, torch.empty(2, 3, 12, 64), torch.empty(2, 3, 12, 64))
    with pytest.raises(ValueError, match="kv_heads"):
        _Shapes(q, torch.empty(2, 2, 12, 64), torch.empty(2, 4, 12, 64))


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(_abi.LIB_PATH):
        from flash_cosine_sim_attention_b200.build import build_library
        build_library()
    return _abi.load()


def _problem(B, H, Hk, Nq, Nk, D):
    p = _abi.FcsaProblem()
    p.dtype, p.batch, p.heads, p.kv_heads, p.seq_q, p.seq_k, p.head_dim = _abi.FCSA_BF16, B, H, Hk, Nq, Nk, D
    p.scale, p.shift = 8.0, 8.0
    return p


def test_abi_version(lib):
    assert lib.fcsa_version() == 300


def test_check_problem_kv_heads(lib):
    t = _abi.FcsaTensor(None, 0, 0, 0)
    fwd = lambda p: lib.fcsa_forward(_abi.ref(p), _abi.ref(t), _abi.ref(t), _abi.ref(t), _abi.ref(t), None, None)
    # (6, 3) passes the problem check and fails on the null tensors; (6, 4) and 0 kv heads fail on kv_heads
    assert fwd(_problem(1, 6, 3, 16, 16, 64)) == _abi.FCSA_ERR_INVALID
    assert b"null" in lib.fcsa_last_error()
    for hk in (4, 0, -2):
        assert fwd(_problem(1, 6, hk, 16, 16, 64)) == _abi.FCSA_ERR_INVALID
        assert b"kv_heads" in lib.fcsa_last_error()
        assert lib.fcsa_backward_workspace_bytes(_abi.ref(_problem(1, 6, hk, 16, 16, 64))) == 0


def test_workspace_size_gqa(lib):
    B, H, Hk, N, D = 2, 8, 2, 1000, 64
    nqt = (N + 63) // 64
    stats = B * H * nqt * 2 * 64 * 4
    p = _problem(B, H, Hk, N, N, D)
    assert lib.fcsa_backward_workspace_bytes(_abi.ref(p)) == stats + 2 * B * Hk * N * D * 4
    assert lib.fcsa_backward_zeroed_bytes(_abi.ref(p)) == B * H * nqt * 64 * D * 4
    p = _problem(B, H, 1, N, N, D)                       # MQA: the same formula with kv_heads = 1
    assert lib.fcsa_backward_workspace_bytes(_abi.ref(p)) == stats + 2 * B * N * D * 4


def test_plan_with_kv_heads():
    assert plan(4, 8, 8) == ("heads", 8)                  # the existing rules hold with kv_heads unset
    assert plan(4, 8, 8, kv_heads=8) == ("heads", 8)
    assert plan(4, 8, 8, kv_heads=1) == ("heads", 8)
    assert plan(1, 8, 2, kv_heads=2) == ("heads", 8)      # kv heads divide over the ranks: whole groups per rank
    assert plan(1, 8, 2, kv_heads=4) == ("heads", 8)
    assert plan(3, 8, 2, kv_heads=1) == ("heads", 8)
    assert plan(3, 8, 4, kv_heads=2) == ("batch", 3)      # a group would straddle two ranks
    assert plan(4, 8, 2, kv_heads=2) == ("batch", 4)


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, qs, kvs, kw, out):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        g = torch.Generator().manual_seed(0)                     # same full tensors on every rank
        q = torch.randn(qs, generator=g, dtype=torch.float64).requires_grad_()
        k = torch.randn(kvs, generator=g, dtype=torch.float64).requires_grad_()
        v = torch.randn(kvs, generator=g, dtype=torch.float64).requires_grad_()
        do = torch.randn(qs, generator=g, dtype=torch.float64)
        o = sharded_flash_cosine_sim_attention(q, k, v, gather=True, attn_fn=plain_cosine_sim_attention, **kw)
        (o * do).sum().backward()
        grads = [t.grad.clone() for t in (q, k, v)]
        for gr in grads:
            dist.all_reduce(gr)                                  # sum of per-rank contributions
        q2, k2, v2 = (t.detach().clone().requires_grad_() for t in (q, k, v))
        ref = plain_cosine_sim_attention(q2, k2, v2, **kw)
        (ref * do).sum().backward()
        ok = torch.allclose(o, ref, atol=1e-12)
        for got, want in zip(grads, (q2.grad, k2.grad, v2.grad)):
            ok = ok and torch.allclose(got, want, atol=1e-10)
        out[rank] = bool(ok)
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("qs,kvs,kw", [
    ((1, 4, 9, 64), (1, 2, 9, 64), dict(causal=True)),          # heads split: one kv head (and its group) per rank
    ((2, 6, 7, 64), (2, 3, 11, 64), dict(groups=2)),            # batch split
], ids=["heads_gqa", "batch_gqa"])
def test_sharded_gqa_equals_unsharded_world2(qs, kvs, kw):
    world = 2
    port = _free_port()
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_worker, args=(world, port, qs, kvs, kw, out), nprocs=world, join=True)
    assert all(out[r] for r in range(world)), dict(out)
