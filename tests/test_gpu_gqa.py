"""GPU parity of grouped-query attention (k, v with kv_heads heads dividing the query heads; query head h reads
key/value head h // (heads // kv_heads)) against the float64 oracle, with the tolerances of test_gpu_parity.py.
The reference of a grouped problem is the oracle on k, v repeated to the query heads, with dk, dv summed over each
group (tests/gqa_reference.py).

The backward kernel either keeps a kv head's whole group of query heads in one CTA (the "loop" path: dk, dv written
by the epilogue, bitwise reproducible) or, when B * kv_heads * key tiles CTAs would leave SMs idle, splits each
group over several CTAs (the "split" path: fp32 dk / dv accumulators and finish passes).  Every test that targets
one of the two computes the choice from the device's SM count and checks it by the number of kernels the backward
launched: 3 on the loop path (preprocess, main, dq finish), at least 5 on the split path (+ dk / dv finish)."""
import math

import pytest
import torch

from gqa_reference import gqa_attention
from test_gpu_parity import ROUND, TOL_GRAD, TOL_OUT, fcsa, make_inputs, record, rel_err  # noqa: F401

pytestmark = pytest.mark.gpu


def sm_count():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def group_split(B, H, Hk, Nk, sms, bias=False):
    """Slices per group the backward chooses (mirror of bwd_group_split in csrc/bwd_kernel.cuh)."""
    G = H // Hk
    if G == 1:
        return 1
    if bias or Hk == 1:
        return G
    unsplit = math.ceil(Nk / 128) * B * Hk
    if unsplit >= sms:
        return 1
    return next((s for s in range(2, G) if G % s == 0 and unsplit * s >= sms), G)


def loop_batch(Hk, Nk):
    """Smallest batch whose backward grid fills the device without splitting the groups."""
    return math.ceil(sm_count() / (math.ceil(Nk / 128) * Hk))


def gqa_check(fcsa, qs, kvs, dtype, seed=0, mask_p=None, path=None, **kw):
    """check() of test_gpu_parity.py for GQA shapes (any dtype and head dim it takes), plus the backward path:
    path = "loop" | "split" | None."""
    B, H, Nq, D = qs
    Hk, Nk = kvs[1], kvs[2]
    if path is not None:
        s = group_split(B, H, Hk, Nk, sm_count())
        assert (s == 1) == (path == "loop"), (path, s)
    q, k, v, do, mask = make_inputs(qs, kvs, dtype, seed, mask_p)
    qd, kd, vd = (t.cuda().requires_grad_() for t in (q, k, v))
    o = fcsa.flash_cosine_sim_attention(qd, kd, vd, mask=None if mask is None else mask.cuda(), **kw)
    assert o.shape == q.shape and o.dtype == dtype
    torch.cuda.synchronize()
    before = fcsa.debug()
    o.backward(do.cuda())
    torch.cuda.synchronize()
    launched = fcsa.debug() - before
    if path == "loop":
        assert launched == 3, launched
    elif path == "split":
        assert launched >= 5, launched
    ref = gqa_attention(q.float().numpy(), k.float().numpy(), v.float().numpy(),
                        mask=None if mask is None else mask.numpy(), d_out=do.float().numpy(),
                        empty_rows="zero", round_qk=ROUND[dtype], **kw)
    e = rel_err(o, ref[0])
    record(dtype, "o", e, TOL_OUT[dtype])
    assert e <= TOL_OUT[dtype], "o"
    for name, t, r in (("dq", qd, ref[1]), ("dk", kd, ref[2]), ("dv", vd, ref[3])):
        assert t.grad.shape == t.shape and t.grad.dtype == dtype
        e = rel_err(t.grad, r)
        record(dtype, name, e, TOL_GRAD[dtype])
        assert e <= TOL_GRAD[dtype], name
    return qd, kd, vd


# ---- the reference grid with grouped keys/values, on both sides of the split selection ---------------------------
@pytest.mark.parametrize("path", ["split", "loop"])
@pytest.mark.parametrize("causal,mask", [(True, False), (False, True), (False, False)])
@pytest.mark.parametrize("seq_len", [63, 200])
@pytest.mark.parametrize("heads,kv_heads", [(4, 2), (8, 2), (6, 3)])
@pytest.mark.parametrize("dim_head", [64, 128])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_gqa_grid(fcsa, path, causal, mask, seq_len, heads, kv_heads, dim_head, dtype):
    B = 2 if path == "split" else loop_batch(kv_heads, seq_len)
    gqa_check(fcsa, (B, heads, seq_len, dim_head), (B, kv_heads, seq_len, dim_head), dtype,
              seed=seq_len + dim_head + heads, mask_p=0.5 if mask else None, causal=causal, path=path)


@pytest.mark.parametrize("path", ["split", "loop"])
@pytest.mark.parametrize("qn,kn", [(200, 456), (456, 200), (129, 300)])
@pytest.mark.parametrize("dim_head", [64, 128])
def test_gqa_causal_cross(fcsa, path, qn, kn, dim_head):
    B = 1 if path == "split" else loop_batch(2, kn)
    gqa_check(fcsa, (B, 8, qn, dim_head), (B, 2, kn, dim_head), torch.bfloat16, seed=qn + kn, causal=True, path=path)


def test_split_path_with_several_heads_per_cta(fcsa):
    """An intermediate split (1 < slices < group): each CTA loops over two query heads and adds its dk / dv into
    the fp32 accumulators."""
    H, Hk, N = 24, 4, 256
    B = math.ceil(sm_count() / 24)
    s = group_split(B, H, Hk, N, sm_count())
    assert 1 < s < H // Hk, s
    gqa_check(fcsa, (B, H, N, 64), (B, Hk, N, 64), torch.bfloat16, seed=3, causal=True, path="split")


def test_split_path_small_batch(fcsa):
    gqa_check(fcsa, (1, 8, 256, 64), (1, 2, 256, 64), torch.bfloat16, seed=4, causal=True, path="split")


def test_loop_path_large_against_expand_and_reproducible(fcsa):
    """(8, 16 heads, 4 kv heads, 2048, 64): 512 CTAs of four query heads each.  Against the expand workaround
    (repeat_interleave -> the MHA kernels, autograd sums dk / dv): o is bitwise equal (the same tiles meet the
    same forward kernel), the gradients agree to 16-bit rounding.  dk and dv are bitwise equal across calls."""
    B, H, Hk, N, D = 8, 16, 4, 2048, 64
    assert group_split(B, H, Hk, N, sm_count()) == 1
    q, k, v, do, _ = make_inputs((B, H, N, D), (B, Hk, N, D), torch.bfloat16, seed=5)
    q, k, v, do = (t.cuda() for t in (q, k, v, do))

    def run(expand):
        qd, kd, vd = (t.clone().requires_grad_() for t in (q, k, v))
        G = H // Hk
        kk, vv = (kd.repeat_interleave(G, 1), vd.repeat_interleave(G, 1)) if expand else (kd, vd)
        before = fcsa.debug()
        o = fcsa.flash_cosine_sim_attention(qd, kk, vv, causal=True)
        o.backward(do)
        torch.cuda.synchronize()
        return o, qd.grad, kd.grad, vd.grad, fcsa.debug() - before

    o1, dq1, dk1, dv1, n1 = run(False)
    o2, dq2, dk2, dv2, _ = run(False)
    oe, dqe, dke, dve, _ = run(True)
    assert n1 == 2 + 3                           # l2norm pair + forward; preprocess + main + dq finish
    assert torch.equal(dk1, dk2) and torch.equal(dv1, dv2)
    assert torch.equal(o1, o2) and torch.equal(o1, oe)
    for got, want in ((dq1, dqe), (dk1, dke), (dv1, dve)):
        ref = want.double().cpu().numpy()
        e = rel_err(got, ref)
        record(torch.bfloat16, "gqa-vs-expand", e, TOL_GRAD[torch.bfloat16])
        assert e <= TOL_GRAD[torch.bfloat16]


@pytest.mark.parametrize("path", ["split", "loop"])
@pytest.mark.parametrize("groups", [2, 8])
def test_gqa_l2norm_groups(fcsa, path, groups):
    """Grouped l2norm: the l2norm backward of dk folded into the epilogue (loop) or its own pass (split)."""
    B = 1 if path == "split" else loop_batch(2, 200)
    gqa_check(fcsa, (B, 8, 200, 64), (B, 2, 200, 64), torch.bfloat16, seed=groups, groups=groups,
              causal=True, path=path)


@pytest.mark.parametrize("batch_dim", [False, True])
@pytest.mark.parametrize("dim_head", [64, 128])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_gqa_attn_bias(fcsa, batch_dim, dim_head, dtype):
    B, H, Hk, Nq, Nk = 2, 6, 3, 150, 203
    q, k, v, do, m = make_inputs((B, H, Nq, dim_head), (B, Hk, Nk, dim_head), dtype, seed=dim_head + batch_dim,
                                 mask_p=0.4)
    g = torch.Generator().manual_seed(98)
    bias = torch.randn((B if batch_dim else H, Nq, Nk), generator=g).to(dtype)
    qd, kd, vd, bd = (t.cuda().requires_grad_() for t in (q, k, v, bias))
    o = fcsa.flash_cosine_sim_attention(qd, kd, vd, mask=m.cuda(), attn_bias=bd, attn_bias_batch_dim=batch_dim)
    o.backward(do.cuda())
    ref = gqa_attention(q.float().numpy(), k.float().numpy(), v.float().numpy(), mask=m.numpy(),
                        attn_bias=bias.float().numpy(), attn_bias_batch_dim=batch_dim, d_out=do.float().numpy(),
                        empty_rows="zero", round_qk=ROUND[dtype])
    e = rel_err(o, ref[0])
    record(dtype, "o", e, TOL_OUT[dtype])
    assert e <= TOL_OUT[dtype], "o"
    for name, t, r in (("dq", qd, ref[1]), ("dk", kd, ref[2]), ("dv", vd, ref[3]), ("d_bias", bd, ref[4])):
        assert t.grad is not None and t.grad.shape == t.shape and t.grad.dtype == dtype, name
        e = rel_err(t.grad, r)
        record(dtype, name, e, TOL_GRAD[dtype])
        assert e <= TOL_GRAD[dtype], name


@pytest.mark.parametrize("causal", [False, True])
def test_gqa_float32(fcsa, causal):
    gqa_check(fcsa, (2, 8, 200, 64), (2, 2, 200, 64), torch.float32, seed=31, causal=causal)


@pytest.mark.parametrize("dim_head", [32, 96])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_gqa_padded_head_dims(fcsa, dim_head, dtype):
    gqa_check(fcsa, (2, 6, 127, dim_head), (2, 3, 127, dim_head), dtype, seed=dim_head, causal=True)


def test_gqa_strided_views_as_in_transformer(fcsa):
    """'b n (h d) -> b h n d' views of q (8 heads) and k, v (2 heads), as transformer.py makes them."""
    g = torch.Generator().manual_seed(12)
    dt = torch.bfloat16
    B, N, H, Hk, D = 2, 300, 8, 2, 64
    base = [torch.randn(B, N, h * D, generator=g).to(dt) for h in (H, Hk, Hk)]
    views = [t.view(B, N, -1, D).transpose(1, 2) for t in base]
    qd, kd, vd = (t.cuda().view(B, N, -1, D).transpose(1, 2).requires_grad_() for t in base)
    assert not kd.is_contiguous()
    do = torch.randn(B, H, N, D, generator=g).to(dt)
    o = fcsa.flash_cosine_sim_attention(qd, kd, vd, causal=True)
    o.backward(do.cuda())
    ref = gqa_attention(*(t.float().numpy() for t in views), causal=True, d_out=do.float().numpy(),
                        round_qk="bf16")
    assert rel_err(o, ref[0]) <= TOL_OUT[dt]
    for t, r in zip((qd, kd, vd), ref[1:]):
        assert rel_err(t.grad, r) <= TOL_GRAD[dt]


def test_gqa_rejections(fcsa):
    q = torch.randn(1, 6, 64, 64, device="cuda", dtype=torch.bfloat16)
    k4, k3 = (torch.randn(1, h, 64, 64, device="cuda", dtype=torch.bfloat16) for h in (4, 3))
    v2 = torch.randn(1, 2, 64, 64, device="cuda", dtype=torch.bfloat16)
    with pytest.raises(ValueError, match="kv_heads"):
        fcsa.flash_cosine_sim_attention(q, k4, k4)                 # 4 does not divide 6
    with pytest.raises(ValueError, match="kv_heads"):
        fcsa.flash_cosine_sim_attention(q, k3, v2)                 # v heads != k heads
    # the compiled host layer checks the same on its own
    from flash_cosine_sim_attention_b200.flash_cosine_sim_attention import _ext
    with pytest.raises(RuntimeError, match="kv_heads"):
        _ext().forward_ex(q, k4, k4, None, None, False, None, 8.0, 8.0, False, 1, True, False)
    with pytest.raises(RuntimeError, match="kv_heads"):
        _ext().forward_ex(q, k3, v2, None, None, False, None, 8.0, 8.0, False, 1, True, False)


def test_c_abi_gqa_forward_backward(fcsa):
    """fcsa_forward / fcsa_backward straight through ctypes with kv_heads = 2 (q, k already normalised)."""
    from flash_cosine_sim_attention_b200 import _abi
    lib = _abi.load()
    B, H, Hk, N, D = 2, 4, 2, 200, 64
    dt = torch.bfloat16
    g = torch.Generator().manual_seed(41)
    nrm = lambda t: torch.nn.functional.normalize(t, dim=-1).to(dt)
    q, k = nrm(torch.randn(B, H, N, D, generator=g)), nrm(torch.randn(B, Hk, N, D, generator=g))
    v = torch.randn(B, Hk, N, D, generator=g).to(dt)
    do = torch.randn(B, H, N, D, generator=g).to(dt)
    qd, kd, vd, dod = (t.cuda() for t in (q, k, v, do))
    o, dq = torch.empty_like(qd), torch.empty_like(qd)
    dk, dv = torch.empty_like(kd), torch.empty_like(vd)
    inv_l = torch.empty(B, H, N, device="cuda", dtype=torch.float32)
    p = _abi.FcsaProblem()
    p.dtype, p.batch, p.heads, p.kv_heads, p.seq_q, p.seq_k, p.head_dim = _abi.FCSA_BF16, B, H, Hk, N, N, D
    p.scale, p.shift = 8.0, 8.0
    tv = lambda t: _abi.FcsaTensor(t.data_ptr(), t.stride(0), t.stride(1), t.stride(2))
    stream = torch.cuda.current_stream().cuda_stream
    _abi.check(lib.fcsa_forward(_abi.ref(p), _abi.ref(tv(qd)), _abi.ref(tv(kd)), _abi.ref(tv(vd)), _abi.ref(tv(o)),
                                inv_l.data_ptr(), stream))
    ns, nz = lib.fcsa_backward_workspace_bytes(_abi.ref(p)), lib.fcsa_backward_zeroed_bytes(_abi.ref(p))
    assert ns > 0 and nz > 0
    ws = torch.empty(ns, device="cuda", dtype=torch.uint8)
    zs = torch.zeros(nz, device="cuda", dtype=torch.uint8)
    _abi.check(lib.fcsa_backward(_abi.ref(p), _abi.ref(tv(qd)), _abi.ref(tv(kd)), _abi.ref(tv(vd)), _abi.ref(tv(o)),
                                 _abi.ref(tv(dod)), inv_l.data_ptr(), _abi.ref(tv(dq)), _abi.ref(tv(dk)),
                                 _abi.ref(tv(dv)), ws.data_ptr(), ns, zs.data_ptr(), nz, stream))
    torch.cuda.synchronize()
    assert int(zs.count_nonzero()) == 0           # the zeroed workspace is left zero
    ref = gqa_attention(q.float().numpy(), k.float().numpy(), v.float().numpy(), l2norm_qk=False, scale=8,
                        d_out=do.float().numpy())
    assert rel_err(o, ref[0]) <= TOL_OUT[dt]
    for t, r in zip((dq, dk, dv), ref[1:]):
        assert rel_err(t, r) <= TOL_GRAD[dt]


def test_transformer_attention_kv_heads(fcsa):
    """Attention(kv_heads=2, use_cuda_kernel=True) in bf16 against the plain path in float32 with the same (rounded)
    weights and input: forward and every gradient."""
    from flash_cosine_sim_attention_b200.transformer import Attention
    torch.manual_seed(0)
    kw = dict(dim=256, dim_head=64, heads=8, kv_heads=2)
    fast = Attention(use_cuda_kernel=True, **kw).cuda().to(torch.bfloat16)
    slow = Attention(use_cuda_kernel=False, **kw).cuda()
    assert fast.to_k.weight.shape == (2 * 64, 256) and fast.to_q.weight.shape == (8 * 64, 256)
    slow.load_state_dict({n: t.float() for n, t in fast.state_dict().items()})
    x = torch.randn(2, 300, 256, device="cuda").to(torch.bfloat16)
    xf = x.float().requires_grad_()
    xb = x.clone().requires_grad_()
    of, os_ = fast(xb), slow(xf)
    do = torch.randn_like(os_)
    of.backward(do.to(torch.bfloat16))
    os_.backward(do)
    err = lambda a, b: ((a.float() - b).abs().max() / b.abs().max()).item()
    assert err(of, os_) <= 3e-2
    assert err(xb.grad, xf.grad) <= 5e-2
    for (n, pf), (_, ps) in zip(fast.named_parameters(), slow.named_parameters()):
        assert err(pf.grad, ps.grad) <= 5e-2, n
