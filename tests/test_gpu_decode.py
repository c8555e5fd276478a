"""GPU tests of flash_cosine_sim_attention_with_kv_cache: new queries against a key/value cache whose valid length
differs per batch element, with the new keys / values appended in the same call.

o is checked per batch element against the float64 reference (tests/elementwise_bounds.py, GQA as in
tests/gqa_reference.py) on the exact 16-bit operands the kernel reads: q^ = l2norm_tensors(q) (the append pass is
the same row kernel) and the key / value rows read back from the cache.  Tolerances: the relative one of
test_gpu_parity.py and the element-wise bound at C = 2.  Cache rows the call must not touch hold a NaN sentinel,
so a stray write, or a NaN value row leaking into P V, shows up.

The split count (key ranges per work item) is chosen on the host from the SM count; tests that target one side of
the rule compute it with the library's own rule (tile_ranges.decode_split) and check it through the number of
launches: append pass + decode kernel, + the combine kernel when it splits."""
import functools
import math

import pytest
import torch

from elementwise_bounds import FMT, attention_bounds, check_bound, kernel_shift
from tile_ranges import decode_split, decode_window_keys
from test_gpu_parity import TOL_OUT, fcsa, record, rel_err  # noqa: F401
from window_bounds import window_attention_bounds

pytestmark = pytest.mark.gpu

SENTINEL = -1          # int16 0xFFFF: a NaN in both float16 and bfloat16


def sm_count():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def n_split_of(B, H, Hk, Nq, cap, window=None, causal=True):
    """The split count of a decode call; with a window below Nq + cap, the keys the split rule sees are bounded by it."""
    G = H // Hk
    if window is not None and window < Nq + cap:
        cap = int(decode_window_keys(cap, window, causal)[0])
    return decode_split(B * Hk * math.ceil(G * Nq / 64), cap, sm_count())


def make_cache(B, Hk, cap, D, dtype, lens, g, l2norm_qk, groups, amp):
    """Caches with valid rows [0, L_b) in the stored form (normalised keys when l2norm_qk) and the sentinel after."""
    from flash_cosine_sim_attention_b200 import l2norm_tensors
    kc = (torch.randn(B, Hk, cap, D, generator=g) * amp).to(dtype).cuda()
    if l2norm_qk:
        kc = l2norm_tensors(kc, groups=groups)[0]
    vc = torch.randn(B, Hk, cap, D, generator=g).to(dtype).cuda()
    for b, L in enumerate(lens):
        kc[b, :, L:].view(torch.int16).fill_(SENTINEL)
        vc[b, :, L:].view(torch.int16).fill_(SENTINEL)
    return kc.contiguous(), vc.contiguous()


def check_case(fcsa, dtype, D, H, Hk, Nq, lens, cap, n_new, causal=True, groups=1, l2norm_qk=True, scale=8,
               seed=0, launches=None, window=None):
    """One call; checks the append bitwise, the untouched rows, and o per batch element (against the windowed
    reference of tests/window_bounds.py when `window` is set).  Returns o."""
    from flash_cosine_sim_attention_b200 import l2norm_tensors
    B = len(lens)
    g = torch.Generator().manual_seed(seed)
    amp = 1.0 if l2norm_qk else 0.15
    if not l2norm_qk or groups > 1:
        scale = 1           # exp(scale * q.k) within fp16's range (q.k reaches `groups`), as train.py runs it
    q = (torch.randn(B, H, Nq, D, generator=g) * amp).to(dtype).cuda()
    kc, vc = make_cache(B, Hk, cap, D, dtype, lens, g, l2norm_qk, groups, amp)
    k = v = None
    if n_new:
        k = (torch.randn(B, Hk, n_new, D, generator=g) * amp).to(dtype).cuda()
        v = torch.randn(B, Hk, n_new, D, generator=g).to(dtype).cuda()
    seqlens = torch.tensor(lens, dtype=torch.int32, device="cuda")
    kc0, vc0 = kc.clone(), vc.clone()
    torch.cuda.synchronize()
    before = fcsa.debug()
    with torch.no_grad():
        o = fcsa.flash_cosine_sim_attention_with_kv_cache(q, kc, vc, seqlens, k, v, scale=scale, groups=groups,
                                                          causal=causal, l2norm_qk=l2norm_qk, window=window)
    torch.cuda.synchronize()
    if launches is not None:
        assert fcsa.debug() - before == launches
    assert o.shape == q.shape and o.dtype == dtype
    assert torch.equal(seqlens.cpu(), torch.tensor(lens, dtype=torch.int32))      # not advanced by the op
    # ---- the append: rows [L, L + n_new) below the capacity, bitwise; everything else untouched ----
    kn = (l2norm_tensors(k, groups=groups)[0] if l2norm_qk else k) if n_new else None
    exp_k, exp_v = kc0.clone(), vc0.clone()
    for b, L in enumerate(lens):
        n = max(0, min(n_new, cap - L))
        if n:
            exp_k[b, :, L:L + n] = kn[b, :, :n]
            exp_v[b, :, L:L + n] = v[b, :, :n]
    assert torch.equal(kc.view(torch.int16), exp_k.view(torch.int16)), "k_cache"
    assert torch.equal(vc.view(torch.int16), exp_v.view(torch.int16)), "v_cache"
    # ---- o per batch element ----
    qh = l2norm_tensors(q, groups=groups)[0] if l2norm_qk else q
    fmt = FMT[dtype]
    shift = kernel_shift(fmt, scale, groups, l2norm_qk)
    for b, L in enumerate(lens):
        T = min(L + n_new, cap)
        if T == 0:
            assert int(o[b].count_nonzero()) == 0
            continue
        bounds = attention_bounds if window is None else functools.partial(window_attention_bounds, window=window)
        ref, bound = bounds(qh[b:b + 1], kc[b:b + 1, :, :T], vc[b:b + 1, :, :T], scale=scale, causal=causal,
                            l2norm_qk=False, fmt=fmt, shift=shift, device="cuda")
        r = ref["o"].cpu().numpy()
        e = rel_err(o[b:b + 1], r) if abs(r).max() > 0 else float(o[b].abs().max())
        record(dtype, "decode o", e, TOL_OUT[dtype])
        assert e <= TOL_OUT[dtype], f"batch element {b} (L = {L}, T = {T})"
        w = check_bound("o", o[b:b + 1], ref, bound, fmt)
        record(dtype, "decode o/bound", w, 1.0)
    return o


# ---- the covering grid: every value of every axis with both dtypes and both head dims ---------------------------
_BASE = dict(H=8, Hk=2, Nq=5, causal=True, groups=1, l2norm_qk=True, append=True, window=None)
_VARIANTS = [dict()]
_VARIANTS += [dict(H=h, Hk=hk) for h, hk in ((8, 8), (8, 1), (6, 3))]
_VARIANTS += [dict(Nq=n) for n in (1, 2, 33, 130)]
_VARIANTS += [dict(H=h, Hk=hk, Nq=64 // (h // hk) + d) for h, hk in ((8, 8), (8, 2), (8, 1), (6, 3)) for d in (-1, 1)]
_VARIANTS += [dict(causal=False), dict(groups=8), dict(l2norm_qk=False), dict(append=False),
              dict(causal=False, append=False, Nq=1)]
# sliding windows (640 = the capacity: the windowed kernel with a band that hides nothing), lengths around their edges
_VARIANTS += [dict(window=w) for w in (1, 65, 200, 640)]
_VARIANTS += [dict(window=65, causal=False), dict(window=200, Nq=33), dict(window=65, H=8, Hk=8),
              dict(window=200, append=False), dict(window=200, causal=False, groups=8)]


def _case_id(v):
    return "-".join(f"{k}{int(x) if isinstance(x, bool) else x}" for k, x in v.items()) or "base"


@pytest.mark.parametrize("variant", _VARIANTS, ids=_case_id)
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_decode_grid(fcsa, variant, D, dtype):
    c = {**_BASE, **variant}
    Nq = c["Nq"]
    n_new = Nq if c["append"] else 0
    cap = 640
    W = c["window"]
    lens = [0, 131, 383, cap - n_new]
    if W is not None:
        # T_b = L_b + n_new at W - 1, W, W + 1 and 2 W: the band's first key at 0 and past it
        lens += [min(max(t - n_new, 0), cap - n_new) for t in (W - 1, W, W + 1, 2 * W)]
    check_case(fcsa, dtype, D, c["H"], c["Hk"], Nq, lens, cap, n_new, causal=c["causal"], groups=c["groups"],
               l2norm_qk=c["l2norm_qk"], seed=_VARIANTS.index(variant) + D, window=W)


# ---- lengths in one call ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_lengths_around_tiles_and_split_boundaries(fcsa, D, dtype):
    """One new token per element (n_new = 1), G = 8: one row block per (batch, kv head), so the call splits the keys.
    T_b = 1 (empty prefix), 127, 128, 129, at and around the end of the first split's key range, and = capacity."""
    H, Hk = 8, 1
    B = 10
    s = n_split_of(B, H, Hk, 1, 4096)
    assert s > 1
    cap = 4096
    nt = cap // 128
    edge = 128 * (nt // s)                      # the first split's key range for T_b = capacity
    T = [1, 127, 128, 129, edge - 1, edge, edge + 1, 2 * edge, cap - 1, cap]
    check_case(fcsa, dtype, D, H, Hk, 1, [t - 1 for t in T], cap, 1, seed=D, launches=3)


def test_lengths_empty_and_zero_rows(fcsa):
    """L_b = 0 without append (no key at all: o = 0), and causal Nq > T_b (the first Nq - T_b queries see no key)."""
    check_case(fcsa, torch.bfloat16, 64, 4, 2, 40, [0, 3, 20, 200], 256, 0, seed=1)
    check_case(fcsa, torch.bfloat16, 64, 4, 2, 40, [0, 3, 20, 200], 256, 5, seed=2)


# ---- both sides of the split rule -------------------------------------------------------------------------------
@pytest.mark.parametrize("side", ["split", "one"])
@pytest.mark.parametrize("D", [64, 128])
def test_split_rule_sides(fcsa, side, D):
    H, Hk, Nq = 8, 8, 1
    B = 2 if side == "split" else math.ceil(sm_count() / Hk)
    s = n_split_of(B, H, Hk, Nq, 1024)
    assert (s == 1) == (side == "one"), s
    lens = [(977 * b) % 1023 for b in range(B)]
    check_case(fcsa, torch.bfloat16, D, H, Hk, Nq, lens, 1024, 1, seed=B + D, launches=2 if s == 1 else 3)


@pytest.mark.parametrize("side", ["split", "one"])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_window_split_rule_sides(fcsa, side, D, dtype):
    """The windowed decode kernel with and without the combine kernel; the split rule bounds the keys by the window."""
    H, Hk, Nq, cap, window = 8, 8, 1, 1024, 200
    B = 2 if side == "split" else math.ceil(sm_count() / Hk)
    s = n_split_of(B, H, Hk, Nq, cap, window)
    assert (s == 1) == (side == "one"), s
    lens = [(window - 2 + 37 * b) % (cap - 1) for b in range(B)]
    check_case(fcsa, dtype, D, H, Hk, Nq, lens, cap, 1, seed=B + D, launches=2 if s == 1 else 3, window=window)


@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_direct_epilogue_grouped_several_row_blocks(fcsa, D, dtype):
    """n_split = 1 (o written by the decode kernel, no combine) with G = 4 and Nq = 33: 132 rows in three row blocks,
    the last one mostly padding rows, so the row mapping i = r / G and the padding-row skip of that epilogue are
    checked against the reference."""
    H, Hk, Nq = 8, 2, 33
    B = math.ceil(sm_count() / (Hk * 3))
    assert n_split_of(B, H, Hk, Nq, 512) == 1
    lens = [(131 * b) % (512 - Nq) for b in range(B)]
    check_case(fcsa, dtype, D, H, Hk, Nq, lens, 512, Nq, seed=D + 11, launches=2)


def test_split_capped_by_capacity_tiles(fcsa):
    """A short cache: the split count is the number of key tiles of the capacity."""
    assert n_split_of(1, 8, 2, 1, 256) == 2
    check_case(fcsa, torch.float16, 64, 8, 2, 1, [200], 256, 1, seed=3, launches=3)


# ---- the append guard ----------------------------------------------------------------------------------------------
def test_append_past_capacity_writes_nothing_outside(fcsa):
    """L_b + n_new > capacity: the rows that do not fit are dropped.  The caches are narrowed views of larger
    buffers whose margins (rows past the capacity, and the next batch element's rows) hold the sentinel: a write past
    the capacity lands inside the allocation, where this test reads it back."""
    dt, B, Hk, cap, pad, D, n_new = torch.bfloat16, 3, 2, 200, 56, 64, 24
    g = torch.Generator().manual_seed(7)
    kbuf = torch.randn(B, Hk, cap + pad, D, generator=g).to(dt).cuda()
    vbuf = torch.randn(B, Hk, cap + pad, D, generator=g).to(dt).cuda()
    kbuf[:, :, cap:].view(torch.int16).fill_(SENTINEL)
    vbuf[:, :, cap:].view(torch.int16).fill_(SENTINEL)
    kc, vc = kbuf[:, :, :cap], vbuf[:, :, :cap]
    lens = [cap - 10, cap, cap + 5]
    seqlens = torch.tensor(lens, dtype=torch.int32, device="cuda")
    q = torch.randn(B, 4, n_new, D, generator=g).to(dt).cuda()
    k, v = (torch.randn(B, Hk, n_new, D, generator=g).to(dt).cuda() for _ in range(2))
    k0, v0 = kbuf.clone(), vbuf.clone()
    from flash_cosine_sim_attention_b200 import l2norm_tensors
    with torch.no_grad():
        o = fcsa.flash_cosine_sim_attention_with_kv_cache(q, kc, vc, seqlens, k, v)
    torch.cuda.synchronize()
    assert torch.isfinite(o).all()
    assert torch.equal(kbuf[:, :, cap:].view(torch.int16), k0[:, :, cap:].view(torch.int16))
    assert torch.equal(vbuf[:, :, cap:].view(torch.int16), v0[:, :, cap:].view(torch.int16))
    kn = l2norm_tensors(k)[0]
    assert torch.equal(kbuf[0, :, cap - 10:cap], kn[0, :, :10]) and torch.equal(vbuf[0, :, cap - 10:cap], v[0, :, :10])
    assert torch.equal(kbuf[1:, :, :cap], k0[1:, :, :cap]) and torch.equal(vbuf[1:, :, :cap], v0[1:, :, :cap])


# ---- agreement with the training operator, reproducibility -----------------------------------------------------
@pytest.mark.parametrize("Nq", [1, 70])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_agrees_with_flash_cosine_sim_attention(fcsa, Nq, dtype):
    """Uniform lengths: o against flash_cosine_sim_attention on the valid prefix (the same normalised keys), within
    the element-wise bound of the float64 reference."""
    B, H, Hk, D, L, cap = 2, 8, 2, 64, 300, 512
    g = torch.Generator().manual_seed(Nq)
    q = torch.randn(B, H, Nq, D, generator=g).to(dtype).cuda()
    k, v = (torch.randn(B, Hk, L + Nq, D, generator=g).to(dtype).cuda() for _ in range(2))
    kc = torch.zeros(B, Hk, cap, D, dtype=dtype, device="cuda")
    vc = torch.zeros_like(kc)
    seqlens = torch.zeros(B, dtype=torch.int32, device="cuda")
    with torch.no_grad():
        # prefill the cache with the first L keys through the op itself (queries: the first token of each row)
        fcsa.flash_cosine_sim_attention_with_kv_cache(q[:, :, :1], kc, vc, seqlens, k[:, :, :L], v[:, :, :L])
        seqlens += L
        o = fcsa.flash_cosine_sim_attention_with_kv_cache(q, kc, vc, seqlens, k[:, :, L:], v[:, :, L:])
        want = fcsa.flash_cosine_sim_attention(q, k, v, causal=True)
    fmt = FMT[dtype]
    from flash_cosine_sim_attention_b200 import l2norm_tensors
    ref, bound = attention_bounds(l2norm_tensors(q)[0], kc[:, :, :L + Nq], vc[:, :, :L + Nq], causal=True,
                                  l2norm_qk=False, fmt=fmt, shift=kernel_shift(fmt, 8), device="cuda")
    assert torch.equal(kc[:, :, :L + Nq], l2norm_tensors(k)[0])
    check_bound("o", o, ref, bound, fmt)
    check_bound("o", want, ref, bound, fmt)
    e = rel_err(o, want.double().cpu().numpy())
    record(dtype, "decode-vs-forward", e, TOL_OUT[dtype])
    assert e <= TOL_OUT[dtype]


@pytest.mark.parametrize("side", ["split", "one"])
def test_bitwise_reproducible(fcsa, side):
    B = 1 if side == "split" else 40
    H, Hk, D, cap = 8, 4, 128, 2048
    g = torch.Generator().manual_seed(9)
    kc, vc = (torch.randn(B, Hk, cap, D, generator=g).to(torch.bfloat16).cuda() for _ in range(2))
    q = torch.randn(B, H, 3, D, generator=g).to(torch.bfloat16).cuda()
    seqlens = torch.randint(1000, 2000, (B,), generator=g).to(torch.int32).cuda()
    assert (n_split_of(B, H, Hk, 3, cap) > 1) == (side == "split")
    with torch.no_grad():
        a = fcsa.flash_cosine_sim_attention_with_kv_cache(q, kc, vc, seqlens)
        b = fcsa.flash_cosine_sim_attention_with_kv_cache(q, kc, vc, seqlens)
    assert torch.equal(a.view(torch.int16), b.view(torch.int16))


# ---- CUDA graph --------------------------------------------------------------------------------------------------
def test_cuda_graph_decode_step(fcsa):
    """One step (append + decode) captured once and replayed 3 times, cache_seqlens advanced on the device between
    replays; each replay equals the eager call on a copy of the caches, bitwise."""
    dt, B, H, Hk, D, cap = torch.float16, 3, 8, 2, 64, 1024
    g = torch.Generator().manual_seed(21)
    kc, vc = (torch.randn(B, Hk, cap, D, generator=g).to(dt).cuda() for _ in range(2))
    sq = torch.zeros(B, H, 1, D, dtype=dt, device="cuda")
    sk, sv = (torch.zeros(B, Hk, 1, D, dtype=dt, device="cuda") for _ in range(2))
    seqlens = torch.tensor([5, 300, 700], dtype=torch.int32, device="cuda")

    def step(kc_, vc_, sl):
        return fcsa.flash_cosine_sim_attention_with_kv_cache(sq, kc_, vc_, sl, sk, sv)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.no_grad(), torch.cuda.stream(side):
        step(kc.clone(), vc.clone(), seqlens.clone())       # warm-up: the workspace of this stream exists
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.no_grad(), torch.cuda.graph(graph, stream=side):
        out = step(kc, vc, seqlens)
    for _ in range(3):
        with torch.no_grad():
            sq.copy_(torch.randn(sq.shape, generator=g).to(dt))
            sk.copy_(torch.randn(sk.shape, generator=g).to(dt))
            sv.copy_(torch.randn(sv.shape, generator=g).to(dt))
            kce, vce, sle = kc.clone(), vc.clone(), seqlens.clone()
            want = step(kce, vce, sle)
            graph.replay()
            torch.cuda.synchronize()
            assert torch.equal(out.view(torch.int16), want.view(torch.int16))
            assert torch.equal(kc.view(torch.int16), kce.view(torch.int16))
            assert torch.equal(vc.view(torch.int16), vce.view(torch.int16))
            seqlens += 1


# ---- rejections ---------------------------------------------------------------------------------------------------
def test_rejections(fcsa):
    f = fcsa.flash_cosine_sim_attention_with_kv_cache
    dt = torch.bfloat16
    q = torch.randn(2, 8, 1, 64, device="cuda", dtype=dt)
    kc = torch.zeros(2, 2, 128, 64, device="cuda", dtype=dt)
    vc = torch.zeros_like(kc)
    sl = torch.zeros(2, dtype=torch.int32, device="cuda")
    with torch.no_grad():
        with pytest.raises(NotImplementedError, match="attn_bias"):
            f(q, kc, vc, sl, attn_bias=torch.zeros(8, 1, 128, device="cuda", dtype=dt))
        with pytest.raises(NotImplementedError, match="mask"):
            f(q, kc, vc, sl, mask=torch.ones(2, 128, dtype=torch.bool, device="cuda"))
        with pytest.raises(TypeError, match="float32"):
            f(q.float(), kc.float(), vc.float(), sl)
        with pytest.raises(NotImplementedError, match="head_dim 96"):
            f(q.new_zeros(2, 8, 1, 96), kc.new_zeros(2, 2, 128, 96), kc.new_zeros(2, 2, 128, 96), sl)
        with pytest.raises(ValueError, match="kv_heads"):
            f(q[:, :6], kc.new_zeros(2, 4, 128, 64), kc.new_zeros(2, 4, 128, 64), sl)
        with pytest.raises(TypeError, match="int32"):
            f(q, kc, vc, sl.long())
        with pytest.raises(RuntimeError, match="CUDA"):
            f(q, kc, vc, sl.cpu())
        # uniform lengths written as an expanded view: the kernels index cache_seqlens as a dense array
        with pytest.raises(ValueError, match="contiguous"):
            f(q, kc, vc, torch.tensor([5], dtype=torch.int32, device="cuda").expand(2))
        with pytest.raises(ValueError, match="contiguous"):
            f(q, kc, vc, torch.zeros(2, 2, dtype=torch.int32, device="cuda")[:, 0])
        from flash_cosine_sim_attention_b200.flash_cosine_sim_attention import _ext
        with pytest.raises(RuntimeError, match="contiguous"):
            _ext().decode(q, kc, vc, torch.tensor([5], dtype=torch.int32, device="cuda").expand(2), None, None, 8.0,
                          8.0, True, 1)
        with pytest.raises(ValueError, match="merged"):
            f(q[:, 0], kc[:, 0], vc[:, 0], sl)
    with pytest.raises(RuntimeError, match="no autograd"):
        f(q.clone().requires_grad_(), kc, vc, sl)


# ---- the transformer ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw", [dict(attn_scale=1, attn_l2norm_groups=8), dict(attn_scale=0.125, l2norm_qk=False)],
                         ids=["groups8", "no_l2norm"])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_transformer_incremental_logits_match_full_forward(dtype, kw):
    """kw: the model's attention settings; l2norm_qk=False is a keyword the model hands the operator, on the cached
    path as on the uncached one."""
    from flash_cosine_sim_attention_b200.transformer import CosineSimCausalTransformer
    torch.manual_seed(0)
    m = CosineSimCausalTransformer(num_tokens=256, dim=128, max_seq_len=64, depth=2, heads=4, dim_head=64,
                                   kv_heads=2, pre_norm=True, use_cuda_kernel=True, **kw).cuda().eval()
    x = torch.randint(0, 256, (2, 40), device="cuda")
    with torch.no_grad(), torch.autocast("cuda", dtype=dtype):
        full = m(x).float()
        cache = m.new_cache()
        steps = [m(x[:, :16], cache=cache)]
        for i in range(16, 40):
            steps.append(m(x[:, i:i + 1], cache=cache))
        inc = torch.cat(steps, 1).float()
    assert inc.shape == full.shape
    assert torch.isfinite(inc).all()
    assert (inc - full).abs().max() <= 5e-2 * full.abs().max() + 1e-6
    with torch.no_grad(), torch.autocast("cuda", dtype=dtype):
        out = m.generate(x, 30, kv_cache=True)             # 40 + 30 tokens: past max_seq_len = 64
    assert out.shape == (2, 30)


def test_transformer_float32_cache_needs_16_bit():
    from flash_cosine_sim_attention_b200.transformer import CosineSimCausalTransformer
    m = CosineSimCausalTransformer(num_tokens=256, dim=128, max_seq_len=64, depth=1, heads=2, dim_head=64,
                                   use_cuda_kernel=True).cuda().eval()
    with torch.no_grad(), pytest.raises(RuntimeError, match="16-bit or under autocast"):
        m(torch.randint(0, 256, (1, 5), device="cuda"), cache=m.new_cache())
