"""GPU tests of packed variable-length attention (flash_cosine_sim_attention_varlen).

Every sequence of a packed batch is checked against the float64 reference of tests/elementwise_bounds.py on that
sequence alone, with the relative tolerances of test_gpu_parity.py and the element-wise bound at C = 2; against the
dense op called on each sequence (o bitwise, and dk / dv bitwise where the backward keeps each group in one CTA);
for isolation from the other sequences, slack in max_seqlen, the zeroed dq workspace after non-finite inputs, strided
views, CUDA graph replay with new lengths, and the transformer's packed path."""
import functools

import pytest
import torch

from elementwise_bounds import FMT, attention_bounds, check_bound, kernel_shift
from test_gpu_gqa import sm_count
from tile_ranges import group_split
from test_gpu_parity import TOL_GRAD, TOL_OUT, fcsa, record, rel_err  # noqa: F401
from window_bounds import window_attention_bounds

pytestmark = pytest.mark.gpu

# lengths around the 64-row query tiles and the 128-row key tiles, plus longer ones, in one batch
LONG = [0, 1, 63, 64, 65, 127, 128, 129, 700, 1500]
SHORT = [0, 1, 65, 129, 300]           # few key tiles: grouped backward grids below the SM count (split)


def cu_of(lengths):
    return torch.tensor([0] + list(torch.tensor(lengths).cumsum(0).tolist()), dtype=torch.int32)


def make_packed(lq, lk, H, Hk, D, dtype, seed, amp=1.0):
    g = torch.Generator().manual_seed(seed)
    q = (torch.randn(sum(lq), H, D, generator=g) * amp).to(dtype)
    k = (torch.randn(sum(lk), Hk, D, generator=g) * amp).to(dtype)
    v = torch.randn(sum(lk), Hk, D, generator=g).to(dtype)
    do = torch.randn(sum(lq), H, D, generator=g).to(dtype)
    return q, k, v, do


def run_varlen(fcsa, q, k, v, do, cu_q, cu_k, max_q, max_k, **kw):
    """Forward and backward through the public API; returns (o, dq, dk, dv, kernels launched by the backward)."""
    qd, kd, vd = (t.cuda().requires_grad_() for t in (q, k, v))
    o = fcsa.flash_cosine_sim_attention_varlen(qd, kd, vd, cu_q.cuda(), cu_k.cuda(), max_q, max_k, **kw)
    assert o.shape == q.shape and o.dtype == q.dtype
    torch.cuda.synchronize()
    before = fcsa.debug()
    o.backward(do.cuda())
    torch.cuda.synchronize()
    return o.detach(), qd.grad, kd.grad, vd.grad, fcsa.debug() - before


def per_seq(t, s, n):
    """rows [s, s + n) of a packed (total, heads, D) tensor as the (1, heads, n, D) tensor of the dense op"""
    return t[s:s + n].transpose(0, 1).unsqueeze(0)


def seq_check(dtype, got, q, k, v, do, lq, lk, only=None, window=None, **kw):
    """Each sequence (or only sequence `only`) against the float64 reference on it alone (with a sliding window: the
    windowed reference of tests/window_bounds.py)."""
    fmt = FMT[dtype]
    l2 = kw.get("l2norm_qk", True)
    shift = kernel_shift(fmt, kw.get("scale", 8), kw.get("groups", 1), l2)
    o, dq, dk, dv = got
    sq = sk = 0
    for i, (a, b) in enumerate(zip(lq, lk)):
        if only is None or i == only:
            if a == 0 or b == 0:
                # no query or no key: o, dq are zero (rows see no key), dk, dv are zero (no query sees the keys)
                for t in (o[sq:sq + a], dq[sq:sq + a], dk[sk:sk + b], dv[sk:sk + b]):
                    assert (t == 0).all(), (i, a, b)
            else:
                bounds = attention_bounds if window is None else functools.partial(window_attention_bounds,
                                                                                   window=window)
                ref, bound = bounds(per_seq(q, sq, a), per_seq(k, sk, b), per_seq(v, sk, b), per_seq(do, sq, a),
                                    round_qk=fmt if l2 else None, fmt=fmt, shift=shift, device="cuda", **kw)
                for name, t, s0, n in (("o", o, sq, a), ("dq", dq, sq, a), ("dk", dk, sk, b), ("dv", dv, sk, b)):
                    got_t = per_seq(t, s0, n)
                    e = rel_err(got_t, ref[name].cpu().numpy())
                    tol = TOL_OUT[dtype] if name == "o" else TOL_GRAD[dtype]
                    record(dtype, f"varlen {name}", e, tol)
                    assert e <= tol, (i, a, b, name, e)
                    record(dtype, f"varlen {name}/bound", check_bound(name, got_t, ref, bound, fmt), 1.0)
        sq += a
        sk += b


def expected_launches(B, H, Hk, max_k, l2norm_qk=True):
    """Kernels of the varlen backward: preprocess, main, dq finish, the pass over the rows outside every sequence;
    + dk / dv finish (and the dk l2norm pass) when the groups are split over CTAs"""
    split = group_split(B, H, Hk, max_k, sm_count())
    return 4 if split == 1 else 6 + (1 if l2norm_qk else 0)


# ---- 1. parity grid ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("lengths", ["long", "short"])
@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("heads,kv_heads", [(8, 8), (8, 2), (8, 1), (6, 3)])
@pytest.mark.parametrize("dim_head", [64, 128])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_varlen_grid(fcsa, lengths, causal, heads, kv_heads, dim_head, dtype):
    ls = LONG if lengths == "long" else SHORT
    q, k, v, do = make_packed(ls, ls, heads, kv_heads, dim_head, dtype, seed=heads + kv_heads + dim_head)
    cu = cu_of(ls)
    *got, launched = run_varlen(fcsa, q, k, v, do, cu, cu, max(ls), max(ls), causal=causal)
    split = group_split(len(ls), heads, kv_heads, max(ls), sm_count())
    if heads != kv_heads and kv_heads > 1:
        # both sides of the split rule: the long batch fills the device with whole groups, the short one does not
        assert (split == 1) == (lengths == "long"), (lengths, split)
    assert launched == expected_launches(len(ls), heads, kv_heads, max(ls)), launched
    seq_check(dtype, got, q, k, v, do, ls, ls, causal=causal)


@pytest.mark.parametrize("opts", [dict(groups=8, scale=1), dict(l2norm_qk=False, scale=1),
                                  dict(groups=8, scale=1, l2norm_qk=False)])
@pytest.mark.parametrize("heads,kv_heads", [(8, 8), (8, 2)])
@pytest.mark.parametrize("dim_head", [64, 128])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_varlen_options(fcsa, opts, heads, kv_heads, dim_head, dtype):
    ls = [65, 0, 300, 129, 1]
    # without the l2norm, q.k is unbounded: small inputs as in test_gpu_parity.py's test_no_l2norm
    amp = 1.0 if opts.get("l2norm_qk", True) else 0.2
    q, k, v, do = make_packed(ls, ls, heads, kv_heads, dim_head, dtype, seed=7, amp=amp)
    cu = cu_of(ls)
    *got, launched = run_varlen(fcsa, q, k, v, do, cu, cu, max(ls), max(ls), causal=True, **opts)
    assert launched == expected_launches(len(ls), heads, kv_heads, max(ls), opts.get("l2norm_qk", True)), launched
    seq_check(dtype, got, q, k, v, do, ls, ls, causal=True, **opts)


@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("heads,kv_heads", [(8, 8), (8, 2)])
@pytest.mark.parametrize("dim_head", [64, 128])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_varlen_cross(fcsa, causal, heads, kv_heads, dim_head, dtype):
    # len_q != len_k, including len_q > len_k (causal: the first len_q - len_k rows see no key) and empty sides
    lq = [100, 64, 300, 0, 129, 5, 1000]
    lk = [40, 200, 300, 10, 1, 0, 1300]
    q, k, v, do = make_packed(lq, lk, heads, kv_heads, dim_head, dtype, seed=11)
    *got, _ = run_varlen(fcsa, q, k, v, do, cu_of(lq), cu_of(lk), max(lq), max(lk), causal=causal)
    seq_check(dtype, got, q, k, v, do, lq, lk, causal=causal)


# ---- 2. agreement with the dense op on each sequence --------------------------------------------------------------
@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("heads,kv_heads", [(8, 8), (8, 2), (8, 1), (6, 3)])
@pytest.mark.parametrize("dim_head", [64, 128])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_varlen_matches_dense(fcsa, causal, heads, kv_heads, dim_head, dtype):
    ls = [1, 63, 64, 65, 129, 700]
    q, k, v, do = make_packed(ls, ls, heads, kv_heads, dim_head, dtype, seed=3)
    cu = cu_of(ls)
    o, dq, dk, dv, _ = run_varlen(fcsa, q, k, v, do, cu, cu, max(ls), max(ls), causal=causal)
    s = 0
    for n in ls:
        qd, kd, vd = (per_seq(t, s, n).cuda().requires_grad_() for t in (q, k, v))
        od = fcsa.flash_cosine_sim_attention(qd, kd, vd, causal=causal)
        od.backward(per_seq(do, s, n).cuda())
        assert torch.equal(per_seq(o, s, n), od.detach()), ("o", n)
        if heads == kv_heads:
            assert torch.equal(per_seq(dk, s, n), kd.grad), ("dk", n)
            assert torch.equal(per_seq(dv, s, n), vd.grad), ("dv", n)
        s += n
    seq_check(dtype, (o, dq, dk, dv), q, k, v, do, ls, ls, causal=causal)


# ---- 3. isolation -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("heads,kv_heads", [(8, 8), (8, 2), (8, 1)])
@pytest.mark.parametrize("dim_head", [64, 128])
def test_varlen_isolation(fcsa, heads, kv_heads, dim_head):
    dtype = torch.bfloat16
    ls = [129, 65, 300, 63, 1]
    cu = cu_of(ls)
    q, k, v, do = make_packed(ls, ls, heads, kv_heads, dim_head, dtype, seed=5)
    first = run_varlen(fcsa, q, k, v, do, cu, cu, max(ls), max(ls), causal=True)
    test, s0 = 1, ls[0]                       # the sequence between two others
    rows = torch.zeros(sum(ls), dtype=torch.bool)
    rows[s0:s0 + ls[test]] = True
    q2, k2, v2, do2 = make_packed(ls, ls, heads, kv_heads, dim_head, dtype, seed=6)
    keep = lambda a, b: torch.where(rows[:, None, None], a, b)
    q2, k2, v2, do2 = keep(q, q2), keep(k, k2), keep(v, v2), keep(do, do2)
    second = run_varlen(fcsa, q2, k2, v2, do2, cu, cu, max(ls), max(ls), causal=True)
    sl = slice(s0, s0 + ls[test])
    assert torch.equal(first[0][sl], second[0][sl]), "o"
    one_cta = group_split(len(ls), heads, kv_heads, max(ls), sm_count()) == 1
    if one_cta:
        assert torch.equal(first[2][sl], second[2][sl]), "dk"
        assert torch.equal(first[3][sl], second[3][sl]), "dv"
    seq_check(dtype, second[:4], q2, k2, v2, do2, ls, ls, only=test, causal=True)


# ---- 4. slack in max_seqlen ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("heads,kv_heads", [(8, 8), (8, 2)])
@pytest.mark.parametrize("dim_head", [64, 128])
def test_varlen_slack(fcsa, heads, kv_heads, dim_head):
    dtype = torch.float16
    ls = [129, 0, 700, 65]
    cu = cu_of(ls)
    q, k, v, do = make_packed(ls, ls, heads, kv_heads, dim_head, dtype, seed=9)
    tight = run_varlen(fcsa, q, k, v, do, cu, cu, max(ls), max(ls), causal=True)
    loose = run_varlen(fcsa, q, k, v, do, cu, cu, max(ls) + 300, max(ls) + 300, causal=True)
    assert torch.equal(tight[0], loose[0]), "o"
    if heads == kv_heads:
        assert torch.equal(tight[2], loose[2]) and torch.equal(tight[3], loose[3]), "dk / dv"
    seq_check(dtype, loose[:4], q, k, v, do, ls, ls, causal=True)


# ---- 5. the zeroed dq workspace survives non-finite inputs ---------------------------------------------------------
def test_varlen_nan_keys_leave_workspace_zero(fcsa):
    dtype, H, D = torch.bfloat16, 4, 64
    ls = [100, 300]                            # sequence 0 ends inside a query tile: padding rows in its tail tile
    cu = cu_of(ls)
    q, k, v, do = make_packed(ls, ls, H, H, D, dtype, seed=13)
    k[10] = float("nan")                       # a key of sequence 0: dS K of its padding rows is NaN
    run_varlen(fcsa, q, k, v, do, cu, cu, max(ls), max(ls), causal=True)
    # a smaller dense backward on the same stream reuses the same zeroed buffer
    g = torch.Generator().manual_seed(14)
    qd, kd, vd, dod = (torch.randn(1, H, 200, D, generator=g).to(dtype) for _ in range(4))
    qc, kc, vc = (t.cuda().requires_grad_() for t in (qd, kd, vd))
    o = fcsa.flash_cosine_sim_attention(qc, kc, vc, causal=True)
    o.backward(dod.cuda())
    assert torch.isfinite(qc.grad).all()
    fmt = FMT[dtype]
    ref, bound = attention_bounds(qd, kd, vd, dod, causal=True, round_qk=fmt, fmt=fmt,
                                  shift=kernel_shift(fmt, 8, 1, True), device="cuda")
    check_bound("dq", qc.grad, ref, bound, fmt)


# ---- 6. strided views of a packed projection ----------------------------------------------------------------------
@pytest.mark.parametrize("dim_head", [64, 128])
def test_varlen_strided_views(fcsa, dim_head):
    from flash_cosine_sim_attention_b200.flash_cosine_sim_attention import _tma_ready
    dtype, H = torch.bfloat16, 4
    ls = [65, 300, 1, 129]
    cu = cu_of(ls).cuda()
    T, HD = sum(ls), H * dim_head
    g = torch.Generator().manual_seed(17)
    qkv = torch.randn(T, 3 * HD, generator=g).to(dtype).cuda().requires_grad_()
    do = torch.randn(T, H, dim_head, generator=g).to(dtype).cuda()
    q, k, v = (qkv[:, i * HD:(i + 1) * HD].view(T, H, dim_head) for i in range(3))
    assert all(_tma_ready(t) is t for t in (q, k, v))     # read as they are, no copy
    o = fcsa.flash_cosine_sim_attention_varlen(q, k, v, cu, cu, max(ls), max(ls), causal=True)
    o.backward(do)
    dq, dk, dv = (qkv.grad[:, i * HD:(i + 1) * HD].reshape(T, H, dim_head) for i in range(3))
    qc, kc, vc = (t.detach().contiguous().cpu() for t in (q, k, v))
    c = run_varlen(fcsa, qc, kc, vc, do.cpu(), cu.cpu(), cu.cpu(), max(ls), max(ls), causal=True)
    assert torch.equal(o.detach(), c[0]) and torch.equal(dk, c[2]) and torch.equal(dv, c[3])
    seq_check(dtype, (o.detach(), dq, dk, dv), qc, kc, vc, do.cpu(), ls, ls, causal=True)


# ---- rows outside every sequence ----------------------------------------------------------------------------------
@pytest.mark.parametrize("heads,kv_heads", [(8, 8), (8, 2), (8, 1)])
@pytest.mark.parametrize("dim_head", [64, 128])
def test_varlen_rows_outside_sequences(fcsa, heads, kv_heads, dim_head):
    """cu[-1] below the total (a packing buffer that is not full): o = 0 and zero gradients in the unused rows, even
    when the allocator hands out memory that held NaN"""
    dtype = torch.bfloat16
    ls, spare_q, spare_k = [129, 65, 300], 77, 130
    q, k, v, do = make_packed(ls + [spare_q], ls + [spare_k], heads, kv_heads, dim_head, dtype, seed=23)
    cu = cu_of(ls)
    T = sum(ls)
    for _ in range(3):     # leave NaN in freed blocks of the sizes the outputs take
        torch.full((q.numel() + k.numel(),), float("nan"), dtype=dtype, device="cuda")
    o, dq, dk, dv, launched = run_varlen(fcsa, q, k, v, do, cu, cu, max(ls), max(ls), causal=True)
    assert launched == expected_launches(len(ls), heads, kv_heads, max(ls)), launched
    for name, t in (("o", o), ("dq", dq), ("dk", dk), ("dv", dv)):
        assert (t[T:] == 0).all(), name
    seq_check(dtype, (o, dq, dk, dv), q, k, v, do, ls, ls, causal=True)


def test_varlen_empty_totals_have_zero_gradients(fcsa):
    q = torch.randn(5, 2, 64, device="cuda", dtype=torch.float16, requires_grad=True)
    k = torch.zeros(0, 2, 64, device="cuda", dtype=torch.float16, requires_grad=True)
    v = torch.zeros(0, 2, 64, device="cuda", dtype=torch.float16, requires_grad=True)
    cq = torch.tensor([0, 5], dtype=torch.int32, device="cuda")
    ck = torch.tensor([0, 0], dtype=torch.int32, device="cuda")
    o = fcsa.flash_cosine_sim_attention_varlen(q, k, v, cq, ck, 5, 0, causal=True)
    assert (o == 0).all()
    o.backward(torch.ones_like(o))
    assert (q.grad == 0).all() and k.grad.shape == k.shape and v.grad.shape == v.shape


# ---- 7. CUDA graph replay with new lengths ------------------------------------------------------------------------
def test_varlen_cuda_graph(fcsa):
    dtype, H, D = torch.bfloat16, 8, 64
    ls, ls2 = [300, 65, 129, 6], [129, 300, 6, 65]      # same total and maximum
    q, k, v, do = (t.cuda() for t in make_packed(ls, ls, H, H, D, dtype, seed=19))
    cu = cu_of(ls).cuda()
    qs, ks, vs = (t.clone().requires_grad_() for t in (q, k, v))
    out = {}

    def step():
        for t in (qs, ks, vs):
            t.grad = None
        o = fcsa.flash_cosine_sim_attention_varlen(qs, ks, vs, cu, cu, max(ls), max(ls), causal=True)
        o.backward(do)
        out["o"] = o.detach()

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        step()
    for lengths in (ls2, ls):
        cu.copy_(cu_of(lengths).cuda())                   # new contents on the device, same buffer
        graph.replay()
        torch.cuda.synchronize()
        eager = run_varlen(fcsa, q.cpu(), k.cpu(), v.cpu(), do.cpu(), cu_of(lengths), cu_of(lengths), max(ls), max(ls),
                           causal=True)
        assert torch.equal(out["o"], eager[0]), lengths
        assert torch.equal(ks.grad, eager[2]) and torch.equal(vs.grad, eager[3]), lengths
        assert rel_err(qs.grad, eager[1].double().cpu().numpy()) <= TOL_GRAD[dtype]
        seq_check(dtype, (out["o"], qs.grad, ks.grad, vs.grad), q.cpu(), k.cpu(), v.cpu(), do.cpu(), lengths, lengths,
                  causal=True)


# ---- rejections that need a CUDA tensor ---------------------------------------------------------------------------
def test_varlen_rejects_on_device(fcsa):
    q = torch.randn(10, 2, 64, device="cuda", dtype=torch.bfloat16)
    cu = torch.tensor([0, 4, 10], dtype=torch.int32, device="cuda")
    op = fcsa.flash_cosine_sim_attention_varlen
    with pytest.raises(ValueError, match="contiguous"):
        op(q, q, q, torch.tensor([0, 0, 4, 0, 10, 0], dtype=torch.int32, device="cuda")[::2], cu, 6, 6)
    with pytest.raises(ValueError, match="contiguous"):
        op(q, q, q, torch.zeros(1, dtype=torch.int32, device="cuda").expand(3), cu, 6, 6)
    with pytest.raises(TypeError, match="int32"):
        op(q, q, q, cu.long(), cu, 6, 6)
    with pytest.raises(TypeError, match="float32"):
        op(q.float(), q.float(), q.float(), cu, cu, 6, 6)
    with pytest.raises(NotImplementedError, match="head_dim"):
        op(q[..., :32], q[..., :32], q[..., :32], cu, cu, 6, 6)
    with pytest.raises(NotImplementedError, match="attn_bias"):
        op(q, q, q, cu, cu, 6, 6, attn_bias=torch.zeros(2, 10, 10, device="cuda"))
    with pytest.raises(NotImplementedError, match="mask"):
        op(q, q, q, cu, cu, 6, 6, mask=torch.ones(2, 10, dtype=torch.bool, device="cuda"))


# ---- 8. the transformer's packed path ------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_transformer_packed_matches_documents(fcsa, dtype):
    from flash_cosine_sim_attention_b200.transformer import CosineSimCausalTransformer
    torch.manual_seed(0)
    model = CosineSimCausalTransformer(num_tokens=64, dim=128, max_seq_len=512, depth=2, heads=4, dim_head=64,
                                       kv_heads=2, use_cuda_kernel=True).cuda().to(dtype).eval()
    docs = [70, 1, 300, 129]
    x = torch.randint(0, 64, (1, sum(docs)), device="cuda")
    cu = cu_of(docs).cuda()
    with torch.no_grad():
        packed = model(x, cu_seqlens=cu, max_seqlen=max(docs)).float()
        s, per_doc = 0, []
        for n in docs:
            per_doc.append(model(x[:, s:s + n]).float())
            s += n
    per_doc = torch.cat(per_doc, dim=1)
    err = ((packed - per_doc).abs().max() / per_doc.abs().max()).item()
    record(dtype, "varlen transformer logits", err, TOL_OUT[dtype])
    assert err <= TOL_OUT[dtype], err
