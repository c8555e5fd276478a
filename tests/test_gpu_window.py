"""GPU: sliding-window attention (the `window` keyword) against the float64 reference with the band
(tests/window_bounds.py), at the element-wise bound with C = 2 and the relative tolerances of test_gpu_parity.py.

Covering grid: windows {1, 63, 64, 65, 127, 128, 129, 200, 1000, >= Nq + Nk}, causal and not, Nq = Nk, Nq < Nk and
Nq > Nk, both dtypes and both head dims, MHA, GQA on both sides of the backward's split rule (the HEAD_LOOP path with
2 and 3 query heads per CTA, checked by the launch count), MQA and merged 3-D layouts, a key-padding mask, the float32
path, head dims 32 and 96, l2norm_qk=False and two (groups, scale) points.  Also: a window of Nq + Nk is bitwise the
unwindowed op, each packed sequence's o, dq, dk, dv match the windowed reference and the dense op (o bitwise, dk, dv
bitwise where the groups stay in one CTA), decode matches the dense forward on the valid prefix, the
dq workspace stays zero, and the transformer's windowed CUDA path matches its plain path."""
import numpy as np
import pytest
import torch

from elementwise_bounds import FMT, check_bound, kernel_shift
from window_bounds import window_attention_bounds
from test_gpu_gqa import loop_batch, sm_count
from tile_ranges import group_split
from test_gpu_parity import TOL_GRAD, TOL_OUT, fcsa, float32_ds_scale, float32_operands, make_inputs, record  # noqa: F401
from test_gpu_varlen import seq_check

pytestmark = pytest.mark.gpu

WINDOWS = (1, 63, 64, 65, 127, 128, 129, 200, 1000, "full")


def rel(got, ref):
    got = got.detach().double().to(ref.device)
    assert torch.isfinite(got).all(), "NaN/Inf in CUDA result"
    return float((got - ref).abs().max() / ref.abs().max().clamp_min(1e-30))


def wcheck(fcsa, qs, kvs, dtype, window, seed=0, mask_p=None, path=None, grads=True, **kw):
    """Run the op with `window` (forward and backward) and judge o, dq, dk, dv against the float64 reference."""
    q, k, v, do, mask = make_inputs(qs, kvs, dtype, seed, mask_p)
    if path is not None:
        s = group_split(qs[0], qs[1], kvs[1], kvs[-2], sm_count())
        assert (s == 1) == (path == "loop"), (path, s)
    qd, kd, vd = (t.cuda().requires_grad_(grads) for t in (q, k, v))
    o = fcsa.flash_cosine_sim_attention(qd, kd, vd, mask=None if mask is None else mask.cuda(), window=window, **kw)
    got = {"o": o}
    if grads:
        torch.cuda.synchronize()
        before = fcsa.debug()
        o.backward(do.cuda())
        torch.cuda.synchronize()
        launched = fcsa.debug() - before
        if path == "loop":
            assert launched == 3, launched
        elif path == "split":
            assert launched >= 5, launched
        got.update(dq=qd.grad, dk=kd.grad, dv=vd.grad)
    l2 = kw.get("l2norm_qk", True)
    ds_scale = 1.0
    if dtype == torch.float32:
        ds_scale = float32_ds_scale(v, do if grads else None)
        fmt, q, k, v, do, _ = float32_operands(q, k, v, do, None, kw.get("scale", 8), kw.get("groups", 1), l2)
    else:
        fmt = FMT[dtype]
    shift = kernel_shift(fmt, kw.get("scale", 8), kw.get("groups", 1), l2)
    ref, bound = window_attention_bounds(q, k, v, do if grads else None, mask=mask, round_qk=fmt if l2 else None,
                                         fmt=fmt, shift=shift, device="cuda", window=window,
                                         ds_scale=ds_scale, **kw)
    for name, t in got.items():
        assert t.shape == ref[name].shape
        record(dtype, f"window:{name}/bound", check_bound(name, t, ref, bound, fmt), 1.0)
        tol = TOL_OUT[dtype] if name == "o" else TOL_GRAD[dtype]
        if ref[name].abs().max() > 1e-6:
            e = rel(t, ref[name])
            record(dtype, f"window:{name}", e, tol)
            assert e <= tol, name
    return got


def W(window, nq, nk):
    return nq + nk if window == "full" else window


# ---- the covering grid -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("window", WINDOWS)
@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("nq,nk", [(300, 300), (300, 700), (700, 300)])
def test_window_grid_bf16_d64(fcsa, window, causal, nq, nk):
    wcheck(fcsa, (1, 2, nq, 64), (1, 2, nk, 64), torch.bfloat16, W(window, nq, nk), seed=nq + nk, causal=causal)


@pytest.mark.parametrize("window", (1, 64, 129, 1000))
@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("dtype,dim", [(torch.float16, 64), (torch.float16, 128), (torch.bfloat16, 128)])
def test_window_dtypes_and_head_dims(fcsa, window, causal, dtype, dim):
    wcheck(fcsa, (2, 2, 333, dim), (2, 2, 333, dim), dtype, window, seed=window + dim, causal=causal)


@pytest.mark.parametrize("path,heads,kv_heads", [("loop", 4, 2), ("loop", 6, 2), ("split", 8, 2)])
@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("dim", [64, 128])
def test_window_gqa_both_sides_of_the_split(fcsa, path, heads, kv_heads, causal, dim):
    """loop: one CTA per group, HEAD_LOOP with 2 and 3 query heads per CTA (the row0 restart at the window's first tile)"""
    N = 400
    B = loop_batch(kv_heads, N) if path == "loop" else 1
    wcheck(fcsa, (B, heads, N, dim), (B, kv_heads, N, dim), torch.bfloat16, 129, seed=heads + dim, path=path,
           causal=causal)


@pytest.mark.parametrize("causal", [True, False])
def test_window_mqa_and_merged(fcsa, causal):
    wcheck(fcsa, (2, 4, 300, 64), (2, 300, 64), torch.bfloat16, 65, seed=1, causal=causal)
    wcheck(fcsa, (6, 260, 64), (6, 260, 64), torch.bfloat16, 100, seed=2, causal=causal)


def test_window_with_key_mask(fcsa):
    wcheck(fcsa, (2, 3, 250, 64), (2, 3, 380, 64), torch.bfloat16, 90, seed=3, mask_p=0.4)
    wcheck(fcsa, (2, 3, 250, 128), (2, 3, 380, 128), torch.float16, 129, seed=4, mask_p=0.4)


@pytest.mark.parametrize("dim", [32, 64, 96])
@pytest.mark.parametrize("causal", [True, False])
def test_window_float32_and_padded_head_dims(fcsa, dim, causal):
    wcheck(fcsa, (1, 2, 270, dim), (1, 2, 270, dim), torch.float32, 70, seed=dim, causal=causal)
    if dim != 64:
        wcheck(fcsa, (1, 2, 270, dim), (1, 2, 270, dim), torch.bfloat16, 70, seed=dim + 1, causal=causal)


def test_window_without_l2norm_and_at_two_logit_range_points(fcsa):
    wcheck(fcsa, (1, 2, 300, 64), (1, 2, 300, 64), torch.bfloat16, 64, seed=5, causal=True, l2norm_qk=False, scale=1)
    wcheck(fcsa, (1, 4, 300, 64), (1, 4, 300, 64), torch.bfloat16, 130, seed=6, groups=4, scale=8, causal=True)
    wcheck(fcsa, (1, 4, 300, 64), (1, 4, 300, 64), torch.float16, 130, seed=7, groups=2, scale=5)


# ---- equivalences ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("dim", [64, 128])
def test_window_of_nq_plus_nk_is_the_unwindowed_op(fcsa, causal, dim):
    """o, dk and dv bitwise equal to the call without a window (dq is summed by fp32 atomics in no fixed order)."""
    q, k, v, do, _ = make_inputs((2, 3, 300, dim), (2, 3, 456, dim), torch.bfloat16, 8)
    outs = []
    for window in (None, 755, 756, 10 ** 9):          # 755 = Nq + Nk - 1: the windowed kernels, hiding nothing
        qd, kd, vd = (t.cuda().requires_grad_() for t in (q, k, v))
        o = fcsa.flash_cosine_sim_attention(qd, kd, vd, causal=causal, window=window)
        o.backward(do.cuda())
        outs.append((o, kd.grad, vd.grad))
    for other in outs[1:]:
        for a, b in zip(outs[0], other):
            assert torch.equal(a, b)


def window_varlen_case(fcsa, dtype, heads, kv_heads, causal, dim):
    """Packed sequences with rows outside every sequence at both ends: each sequence's o, dq, dk, dv against the
    float64 windowed reference on it alone, o bitwise the dense op's, and dk, dv bitwise the dense op's where both
    calls keep each kv group in one CTA."""
    g = torch.Generator().manual_seed(9)
    lq, lk = [130, 0, 257, 64, 1], ([130, 40, 300, 64, 1] if not causal else [130, 0, 257, 64, 1])
    cq = torch.tensor(np.cumsum([3] + lq), dtype=torch.int32)
    ck = torch.tensor(np.cumsum([0] + lk), dtype=torch.int32)
    Tq, Tk = int(cq[-1]) + 5, int(ck[-1])
    q = torch.randn(Tq, heads, dim, generator=g).to(dtype).cuda().requires_grad_()
    k = torch.randn(Tk, kv_heads, dim, generator=g).to(dtype).cuda().requires_grad_()
    v = torch.randn(Tk, kv_heads, dim, generator=g).to(dtype).cuda().requires_grad_()
    do = torch.randn(Tq, heads, dim, generator=g).to(dtype).cuda()
    window = 70
    o = fcsa.flash_cosine_sim_attention_varlen(q, k, v, cq.cuda(), ck.cuda(), max(lq), max(lk), causal=causal,
                                               window=window)
    o.backward(do)
    assert (o[:3] == 0).all() and (o[-5:] == 0).all() and (q.grad[:3] == 0).all() and (q.grad[-5:] == 0).all()
    inside = slice(3, Tq - 5)
    seq_check(dtype, (o.detach()[inside], q.grad[inside], k.grad, v.grad), q.detach()[inside], k.detach(), v.detach(),
              do[inside], lq, lk, window=window, causal=causal)
    packed_one_cta = group_split(len(lq), heads, kv_heads, max(lk), sm_count()) == 1
    for b in range(len(lq)):
        if lq[b] == 0 or lk[b] == 0:
            continue
        qs, ks = slice(int(cq[b]), int(cq[b + 1])), slice(int(ck[b]), int(ck[b + 1]))
        dense = lambda t, s: t.detach()[s].transpose(0, 1).unsqueeze(0)
        qd, kd, vd = (dense(t, s).requires_grad_() for t, s in ((q, qs), (k, ks), (v, ks)))
        od = fcsa.flash_cosine_sim_attention(qd, kd, vd, causal=causal, window=window)
        od.backward(dense(do, qs))
        assert torch.equal(o[qs].detach(), od.detach()[0].transpose(0, 1))
        if packed_one_cta and group_split(1, heads, kv_heads, lk[b], sm_count()) == 1:
            assert torch.equal(k.grad[ks], kd.grad[0].transpose(0, 1)), ("dk", b)
            assert torch.equal(v.grad[ks], vd.grad[0].transpose(0, 1)), ("dv", b)


@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("dim", [64, 128])
def test_window_varlen_per_sequence_is_the_dense_op(fcsa, causal, dim):
    window_varlen_case(fcsa, torch.bfloat16, 4, 2, causal, dim)


@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("dim", [64, 128])
@pytest.mark.parametrize("dtype,heads,kv_heads", [(torch.float16, 4, 2), (torch.float16, 4, 4), (torch.bfloat16, 4, 4)],
                         ids=["f16-4:2", "f16-4:4", "bf16-4:4"])
def test_window_varlen_dtypes_and_heads(fcsa, dtype, heads, kv_heads, causal, dim):
    window_varlen_case(fcsa, dtype, heads, kv_heads, causal, dim)


@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("G,nq", [(1, 1), (4, 1), (8, 3)])
def test_window_decode_matches_the_dense_forward(fcsa, causal, G, nq):
    """Lengths around the window's edges and the split edges; few items (several splits) and many (one split)."""
    dim, cap, window = 128, 2048, 200
    for B, Hk in ((1, 2), (32, 8)):
        g = torch.Generator().manual_seed(G * 10 + nq + B)
        for L in (0, 1, window - 1, window, window + 1, 255, 256, 1500):
            q = torch.randn(B, G * Hk, nq, dim, generator=g).to(torch.bfloat16).cuda()
            kc = torch.randn(B, Hk, cap, dim, generator=g).to(torch.bfloat16).cuda()
            vc = torch.randn(B, Hk, cap, dim, generator=g).to(torch.bfloat16).cuda()
            k = torch.randn(B, Hk, nq, dim, generator=g).to(torch.bfloat16).cuda()
            v = torch.randn(B, Hk, nq, dim, generator=g).to(torch.bfloat16).cuda()
            kc[:, :, :L] = fcsa.l2norm_tensors(kc[:, :, :L])[0] if L > 0 else kc[:, :, :L]
            seq = torch.full((B,), L, dtype=torch.int32, device="cuda")
            with torch.no_grad():
                o = fcsa.flash_cosine_sim_attention_with_kv_cache(q, kc, vc, seq, k, v, causal=causal, window=window)
            T = L + nq
            kk, vv = kc[:, :, :T], vc[:, :, :T]
            ref, bound = window_attention_bounds(q, kk, vv, causal=causal, round_qk="bf16", l2norm_qk=True,
                                                 fmt="bf16", shift=kernel_shift("bf16", 8), device="cuda", window=window)
            # the cache holds normalised keys: the dense op re-normalises them (an exact no-op up to rounding)
            record(torch.bfloat16, "window:decode_o/bound", check_bound("o", o, ref, bound, "bf16"), 1.0)
            assert rel(o, ref["o"]) <= TOL_OUT[torch.bfloat16]


def test_window_leaves_the_dq_workspace_zero(fcsa):
    """Non-causal Nq >> Nk: most query rows see no key (dq = 0 there); the zeroed workspace stays zero, so a later
    unwindowed call on the same buffers is exact."""
    q, k, v, do, _ = make_inputs((2, 2, 900, 64), (2, 2, 100, 64), torch.bfloat16, 11)
    qd, kd, vd = (t.cuda().requires_grad_() for t in (q, k, v))
    o = fcsa.flash_cosine_sim_attention(qd, kd, vd, window=50)
    o.backward(do.cuda())
    off = 100 - 900
    rows = torch.arange(900)
    blind = (rows + off - 99 >= 50) | (rows + off <= -50)
    assert (o.detach().cpu()[:, :, blind] == 0).all() and (qd.grad.cpu()[:, :, blind] == 0).all()
    wcheck(fcsa, (2, 2, 900, 64), (2, 2, 100, 64), torch.bfloat16, 50, seed=11)
    # the persistent accumulator is zero again: the next call on it matches the reference
    wcheck(fcsa, (2, 2, 900, 64), (2, 2, 900, 64), torch.bfloat16, 1800, seed=12, causal=True)


# ---- the transformer ---------------------------------------------------------------------------------------------
def test_transformer_window_cuda_against_plain_and_cached():
    from flash_cosine_sim_attention_b200.transformer import CosineSimCausalTransformer
    torch.manual_seed(0)
    kw = dict(num_tokens=100, dim=128, max_seq_len=512, depth=2, heads=4, dim_head=64, kv_heads=2, window=96)
    plain = CosineSimCausalTransformer(**kw).cuda().eval()
    cuda = CosineSimCausalTransformer(use_cuda_kernel=True, **kw).cuda().eval()
    cuda.load_state_dict(plain.state_dict())
    x = torch.randint(0, 100, (2, 300), device="cuda")
    with torch.no_grad():
        a = plain(x)
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        b = cuda(x).float()
        assert (a - b).abs().max() / a.abs().max() < 5e-2
        cache = cuda.new_cache()
        steps = [cuda(x[:, :200], cache=cache)] + [cuda(x[:, t:t + 1], cache=cache) for t in range(200, 300)]
        c = torch.cat(steps, 1).float()
    assert (c - b).abs().max() / b.abs().max() < 3e-2
