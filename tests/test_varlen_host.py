"""CPU: packed variable-length attention without a device - the Python API's rejections, the C ABI's argument checks
and workspace sizes through ctypes, the tile-padded layout of the backward's stats and dq accumulator,
and the transformer's packed path with the plain attention in float64."""
import itertools
import os
import random

import pytest
import torch

from flash_cosine_sim_attention_b200 import _abi, flash_cosine_sim_attention_varlen
from flash_cosine_sim_attention_b200.transformer import CosineSimCausalTransformer
from tile_ranges import tiles


def args(total=10, H=2, Hk=2, D=64, dtype=torch.bfloat16):
    q = torch.randn(total, H, D).to(dtype)
    k = torch.randn(total, Hk, D).to(dtype)
    cu = torch.tensor([0, 4, total], dtype=torch.int32)
    return q, k, k.clone(), cu


# ---- the Python API's rejections (all before any device is touched) ----------------------------------------------
@pytest.mark.parametrize("case,exc,match", [
    ("float32", TypeError, "float32"),
    ("head_dim", NotImplementedError, "head_dim"),
    ("mask", NotImplementedError, "mask"),
    ("attn_bias", NotImplementedError, "attn_bias"),
    ("cpu", RuntimeError, "CUDA"),
    ("cu_int64", TypeError, "int32"),
    ("cu_2d", TypeError, "shape"),
    ("cu_strided", ValueError, "contiguous"),
    ("cu_expanded", ValueError, "contiguous"),
    ("cu_lengths_differ", ValueError, "same length"),
    ("kv_heads", ValueError, "divide"),
    ("four_dims", ValueError, "total_q"),
    ("max_not_int", TypeError, "max_seqlen"),
    ("groups", ValueError, "groups"),
])
def test_rejections(case, exc, match):
    q, k, v, cu = args(Hk=1 if case != "kv_heads" else 3, H=2 if case != "kv_heads" else 4)
    cq = ck = cu
    kw = {}
    mq = mk = 6
    if case == "float32":
        q, k, v = q.float(), k.float(), v.float()
    elif case == "head_dim":
        q, k, v = q[..., :32], k[..., :32], v[..., :32]
    elif case == "mask":
        kw["mask"] = torch.ones(2, 10, dtype=torch.bool)
    elif case == "attn_bias":
        kw["attn_bias"] = torch.zeros(2, 10, 10)
    elif case == "cu_int64":
        cq = cu.long()
    elif case == "cu_2d":
        cq = cu[None]
    elif case == "cu_strided":
        cq = torch.tensor([0, 9, 4, 9, 10, 9], dtype=torch.int32)[::2]
    elif case == "cu_expanded":
        cq = torch.zeros(1, dtype=torch.int32).expand(3)
    elif case == "cu_lengths_differ":
        ck = torch.tensor([0, 10], dtype=torch.int32)
    elif case == "four_dims":
        q = q[None]
    elif case == "max_not_int":
        mq = torch.tensor(6)
    elif case == "groups":
        kw["groups"] = 3
    with pytest.raises(exc, match=match):
        flash_cosine_sim_attention_varlen(q, k, v, cq, ck, mq, mk, **kw)


# ---- the C ABI through ctypes ---------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(_abi.LIB_PATH):
        from flash_cosine_sim_attention_b200.build import build_library
        build_library()
    return _abi.load()


def problem(B=3, H=8, Hk=2, max_q=300, max_k=300, D=64, dtype=_abi.FCSA_BF16):
    p = _abi.FcsaProblem()
    p.dtype, p.batch, p.heads, p.kv_heads, p.seq_q, p.seq_k, p.head_dim = dtype, B, H, Hk, max_q, max_k, D
    p.causal, p.scale, p.shift = 1, 8.0, 8.0
    return p


def varlen(total_q=500, total_k=700):
    return _abi.FcsaVarlen(16, 32, total_q, total_k)     # device pointers are never dereferenced by the checks


def expected_bytes(B, H, Hk, total_q, total_k, D):
    """(scratch, zeroed) bytes: per head total_q / 64 + B + 1 tiles of 64 rows of {c3, -delta} and of the fp32 dq
    accumulator; fp32 dk / dv accumulators over the packed keys when kv_heads < heads.  256-byte aligned pieces."""
    up = lambda x: (x + 255) // 256 * 256
    ntile = total_q // 64 + B + 1
    stats = H * ntile * 2 * 64 * 4
    dkv = 2 * Hk * total_k * D * 4 if Hk < H else 0
    return up(stats) + up(dkv), up(H * ntile * 64 * D * 4)


@pytest.mark.parametrize("B,H,Hk,tq,tk,D", [(3, 8, 2, 500, 700, 64), (1, 4, 4, 64, 64, 128), (17, 6, 3, 12345, 999, 128),
                                           (5, 8, 1, 63, 1, 64)])
def test_workspace_sizes(lib, B, H, Hk, tq, tk, D):
    p, vl = problem(B=B, H=H, Hk=Hk, D=D), varlen(tq, tk)
    s, z = expected_bytes(B, H, Hk, tq, tk, D)
    assert lib.fcsa_backward_fused_varlen_workspace_bytes(_abi.ref(p), _abi.ref(vl)) == s
    assert lib.fcsa_backward_fused_varlen_zeroed_bytes(_abi.ref(p), _abi.ref(vl)) == z
    # the maxima do not enter the sizes
    p2 = problem(B=B, H=H, Hk=Hk, D=D, max_q=7, max_k=9000)
    assert lib.fcsa_backward_fused_varlen_workspace_bytes(_abi.ref(p2), _abi.ref(vl)) == s


def test_abi_argument_checks(lib):
    p, vl = problem(), varlen()
    ws = lib.fcsa_backward_fused_varlen_workspace_bytes
    assert ws(_abi.ref(p), None) == 0
    assert ws(_abi.ref(p), _abi.ref(_abi.FcsaVarlen(None, 32, 10, 10))) == 0
    assert ws(_abi.ref(p), _abi.ref(_abi.FcsaVarlen(18, 32, 10, 10))) == 0            # misaligned int32 array
    assert ws(_abi.ref(p), _abi.ref(varlen(0, 10))) == 0
    masked = problem()
    masked.causal, masked.key_mask = 0, 64
    assert ws(_abi.ref(masked), _abi.ref(vl)) == 0
    f32 = problem()
    f32.out_f32 = 1
    assert ws(_abi.ref(f32), _abi.ref(vl)) == 0
    t = _abi.FcsaTensor(256, 0, 64, 512)
    n = _abi.FcsaL2Norm(1, t, t, 64, 64)
    fwd = lambda pp, vv: lib.fcsa_forward_fused_varlen(_abi.ref(pp), vv, _abi.ref(t), _abi.ref(t), _abi.ref(t),
                                                       _abi.ref(n), _abi.ref(t), 64, None)
    assert fwd(p, None) == _abi.FCSA_ERR_INVALID
    assert fwd(masked, _abi.ref(vl)) == _abi.FCSA_ERR_UNSUPPORTED
    assert fwd(problem(D=32), _abi.ref(vl)) == _abi.FCSA_ERR_UNSUPPORTED
    assert fwd(problem(dtype=7), _abi.ref(vl)) == _abi.FCSA_ERR_UNSUPPORTED
    assert fwd(problem(Hk=3), _abi.ref(vl)) == _abi.FCSA_ERR_INVALID
    assert b"kv_heads" in lib.fcsa_last_error()
    bwd = lambda wsb, zb: lib.fcsa_backward_fused_varlen(_abi.ref(p), _abi.ref(vl), _abi.ref(n), _abi.ref(t), _abi.ref(t),
                                                         _abi.ref(t), 64, _abi.ref(t), _abi.ref(t), _abi.ref(t), 256, wsb,
                                                         512, zb, None)
    s, z = expected_bytes(3, 8, 2, 500, 700, 64)
    assert bwd(s - 1, z) == _abi.FCSA_ERR_WORKSPACE
    assert bwd(s, z - 1) == _abi.FCSA_ERR_WORKSPACE
    assert b"zeroed" in lib.fcsa_last_error()


# ---- the tile-padded layout ----------------------------------------------------------------------------------------
def assert_disjoint_and_inside(lengths):
    ranges, ntile = tiles(lengths)
    for (lo, hi), (lo2, _) in zip(ranges, ranges[1:]):
        assert hi <= lo2, lengths                          # base(b + 1) - base(b) >= ceil(len_b / 64)
    assert all(hi <= ntile for _, hi in ranges), lengths


def test_tile_layout_exhaustive_small():
    for a, b in itertools.product(range(0, 200), repeat=2):
        assert_disjoint_and_inside([a, b])
    for ls in itertools.product(range(0, 140, 3), repeat=3):
        assert_disjoint_and_inside(list(ls))


def test_tile_layout_random_large():
    rng = random.Random(0)
    for _ in range(2000):
        B = rng.randint(1, 64)
        assert_disjoint_and_inside([rng.choice([0, 1, 63, 64, 65, rng.randint(0, 70000)]) for _ in range(B)])


# ---- the transformer's packed path (plain attention, float64) ------------------------------------------------------
@pytest.mark.parametrize("kv_heads", [None, 2])
def test_transformer_packed_equals_documents(kv_heads):
    torch.manual_seed(0)
    model = CosineSimCausalTransformer(num_tokens=50, dim=64, max_seq_len=64, depth=2, heads=4, dim_head=16,
                                       kv_heads=kv_heads).double().eval()
    docs = [5, 0, 17, 1, 30]
    x = torch.randint(0, 50, (1, sum(docs)))
    cu = torch.tensor([0] + list(itertools.accumulate(docs)), dtype=torch.int32)
    with torch.no_grad():
        packed = model(x, cu_seqlens=cu, max_seqlen=max(docs))
        s = 0
        for n in docs:
            if n:
                # each document alone, positions from 0: the packed logits restart there too
                assert torch.allclose(packed[:, s:s + n], model(x[:, s:s + n]), rtol=0, atol=1e-12)
            s += n
        # a document moved elsewhere in the pack gives the same logits (positions restart per document)
        cu2 = torch.tensor([0, 17, 22], dtype=torch.int32)
        x2 = torch.cat([x[:, 5:22], x[:, :5]], dim=1)
        assert torch.allclose(model(x2, cu_seqlens=cu2)[:, 17:22], packed[:, :5], rtol=0, atol=1e-12)


def test_transformer_packed_rejections():
    model = CosineSimCausalTransformer(num_tokens=50, dim=64, max_seq_len=64, depth=1, heads=4, dim_head=16)
    x = torch.randint(0, 50, (1, 10))
    cu = torch.tensor([0, 4, 10], dtype=torch.int32)
    with pytest.raises(NotImplementedError):
        model(x, return_loss=True, cu_seqlens=cu)
    with pytest.raises(NotImplementedError):
        model(x, cache=model.new_cache(), cu_seqlens=cu)
    with pytest.raises(ValueError):
        model(torch.randint(0, 50, (2, 10)), cu_seqlens=cu)
    with pytest.raises(ValueError):
        model(x, cu_seqlens=cu, max_seqlen=65)
    with pytest.raises(NotImplementedError):
        model.layers[0][0](torch.randn(1, 10, 64), cache=object(), cu_seqlens=cu)


def test_transformer_packed_rows_after_the_last_document():
    """cu_seqlens ending before the total (a packing buffer that is not full): the documents are unaffected and the
    attention of the spare rows is zero, as the kernel gives it"""
    torch.manual_seed(1)
    model = CosineSimCausalTransformer(num_tokens=50, dim=64, max_seq_len=64, depth=1, heads=4, dim_head=16).double().eval()
    x = torch.randint(0, 50, (1, 30))
    cu = torch.tensor([0, 12, 25], dtype=torch.int32)
    attn = model.layers[0][0]
    with torch.no_grad():
        full = model(x, cu_seqlens=cu, max_seqlen=13)
        assert torch.allclose(full[:, :12], model(x[:, :12]), rtol=0, atol=1e-12)
        assert torch.allclose(full[:, 12:25], model(x[:, 12:25]), rtol=0, atol=1e-12)
        h = torch.randn(1, 30, 64, dtype=torch.float64)
        assert (attn(h, cu_seqlens=cu, max_seqlen=13)[:, 25:] == 0).all()
