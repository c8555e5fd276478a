"""GPU tests of flash_cosine_sim_attention_with_kv_cache with packed new tokens (cu_seqlens_q, max_seqlen_q): a
different number of new tokens per batch element in one call.

o of every sequence is checked against the float64 reference (tests/elementwise_bounds.py, the windowed one of
tests/window_bounds.py) on the exact 16-bit operands the kernel reads, with the relative tolerance of
test_gpu_parity.py and the element-wise bound, as test_gpu_decode.py does for the dense call.  Cache rows the call
must not touch hold a NaN sentinel.  Packs put n_b on both sides of the 64 / G row-block edges (0, 1, 7, 64 / G +- 1
and 130 in one call), L_b around the 128-key tile edges, and leave packed rows before cu[0] and after cu[B] that
belong to no sequence.  Launches: append pass + decode kernel (+ combine when the keys are split) + the pass that
zeroes the rows outside every sequence."""
import functools
import math

import pytest
import torch

from elementwise_bounds import FMT, attention_bounds, check_bound, kernel_shift
from test_gpu_decode import SENTINEL, make_cache, sm_count
from test_gpu_parity import TOL_OUT, fcsa, record, rel_err  # noqa: F401
from tile_ranges import decode_split, decode_window_keys
from window_bounds import window_attention_bounds

pytestmark = pytest.mark.gpu


def packed_split(B, H, Hk, max_q, cap, window=None, causal=True):
    """The split count of a packed call: decode_split on the grid of the maxima."""
    if window is not None and window < max_q + cap:
        cap = int(decode_window_keys(cap, window, causal)[0])
    return decode_split(B * Hk * math.ceil(H // Hk * max_q / 64), cap, sm_count())


def make_pack(ns, lead, trail):
    cu = [lead]
    for n in ns:
        cu.append(cu[-1] + n)
    return cu, cu[-1] + trail


def run_packed(fcsa, dtype, D, H, Hk, ns, lens, cap, append=True, causal=True, groups=1, l2norm_qk=True,
               window=None, lead=3, trail=2, seed=0, launches=None, max_q=None, check=True):
    """One packed call with sequence b bringing ns[b] new tokens onto L_b = lens[b] cached rows.  Checks the append
    bitwise, the untouched cache rows, o = 0 outside every sequence and, with `check`, o of every sequence against the
    reference.  Returns (o, inputs)."""
    from flash_cosine_sim_attention_b200 import l2norm_tensors
    B = len(ns)
    g = torch.Generator().manual_seed(seed)
    amp = 1.0 if l2norm_qk else 0.15
    scale = 1 if (not l2norm_qk or groups > 1) else 8
    cu, total = make_pack(ns, lead, trail)
    q = (torch.randn(total, H, D, generator=g) * amp).to(dtype).cuda()
    kc, vc = make_cache(B, Hk, cap, D, dtype, lens, g, l2norm_qk, groups, amp)
    k = v = None
    if append:
        k = (torch.randn(total, Hk, D, generator=g) * amp).to(dtype).cuda()
        v = torch.randn(total, Hk, D, generator=g).to(dtype).cuda()
    seqlens = torch.tensor(lens, dtype=torch.int32, device="cuda")
    cu_t = torch.tensor(cu, dtype=torch.int32, device="cuda")
    kc0, vc0 = kc.clone(), vc.clone()
    torch.cuda.synchronize()
    before = fcsa.debug()
    with torch.no_grad():
        o = fcsa.flash_cosine_sim_attention_with_kv_cache(q, kc, vc, seqlens, k, v, scale=scale, groups=groups,
                                                          causal=causal, l2norm_qk=l2norm_qk, window=window,
                                                          cu_seqlens_q=cu_t, max_seqlen_q=max_q or max(ns))
    torch.cuda.synchronize()
    if launches is not None:
        assert fcsa.debug() - before == launches
    assert o.shape == q.shape and o.dtype == dtype
    assert seqlens.tolist() == list(lens) and cu_t.tolist() == cu      # neither is advanced
    # ---- the append: sequence b's rows at [L_b, L_b + n_b) below the capacity, bitwise; nothing else written ----
    exp_k, exp_v = kc0.clone(), vc0.clone()
    if append:
        kn = l2norm_tensors(k, groups=groups)[0] if l2norm_qk else k
        for b, L in enumerate(lens):
            n = max(0, min(ns[b], cap - L))
            exp_k[b, :, L:L + n] = kn[cu[b]:cu[b] + n].transpose(0, 1)
            exp_v[b, :, L:L + n] = v[cu[b]:cu[b] + n].transpose(0, 1)
    assert torch.equal(kc.view(torch.int16), exp_k.view(torch.int16)), "k_cache"
    assert torch.equal(vc.view(torch.int16), exp_v.view(torch.int16)), "v_cache"
    # ---- o: zero outside every sequence, the reference inside ----
    assert int(o[:cu[0]].count_nonzero()) == 0 and int(o[cu[-1]:].count_nonzero()) == 0
    if check:
        qh = l2norm_tensors(q, groups=groups)[0] if l2norm_qk else q
        fmt = FMT[dtype]
        shift = kernel_shift(fmt, scale, groups, l2norm_qk)
        bounds = attention_bounds if window is None else functools.partial(window_attention_bounds, window=window)
        for b, L in enumerate(lens):
            n = ns[b]
            if n == 0:
                continue
            T = min(L + (n if append else 0), cap)
            ob = o[cu[b]:cu[b + 1]].transpose(0, 1).unsqueeze(0)
            if T == 0:
                assert int(ob.count_nonzero()) == 0
                continue
            ref, bound = bounds(qh[cu[b]:cu[b + 1]].transpose(0, 1).unsqueeze(0), kc[b:b + 1, :, :T],
                                vc[b:b + 1, :, :T], scale=scale, causal=causal, l2norm_qk=False, fmt=fmt, shift=shift,
                                device="cuda")
            r = ref["o"].cpu().numpy()
            e = rel_err(ob, r) if abs(r).max() > 0 else float(ob.abs().max())
            record(dtype, "decode varlen o", e, TOL_OUT[dtype])
            assert e <= TOL_OUT[dtype], f"sequence {b} (n_b = {n}, L = {L}, T = {T})"
            w = check_bound("o", ob, ref, bound, fmt)
            record(dtype, "decode varlen o/bound", w, 1.0)
    return o, dict(q=q, k=k, v=v, kc=kc, vc=vc, kc0=kc0, vc0=vc0, seqlens=seqlens, cu=cu_t, scale=scale)


# ---- per-sequence parity over the covering grid -------------------------------------------------------------------
_BASE = dict(H=8, Hk=2, causal=True, groups=1, l2norm_qk=True, append=True, window=None)
_VARIANTS = [dict(), dict(H=8, Hk=8), dict(H=8, Hk=1), dict(causal=False), dict(groups=8), dict(l2norm_qk=False),
             dict(append=False), dict(window=65), dict(window=200, causal=False), dict(window=65, append=False)]


def _case_id(v):
    return "-".join(f"{k}{int(x) if isinstance(x, bool) else x}" for k, x in v.items()) or "base"


@pytest.mark.parametrize("variant", _VARIANTS, ids=_case_id)
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_packed_grid(fcsa, variant, D, dtype):
    c = {**_BASE, **variant}
    G = c["H"] // c["Hk"]
    e = 64 // G                              # queries per row block
    ns = [0, 1, 7, e - 1, e + 1, 130, 2 * e + 1]
    lens = [127, 128, 129, 255, 0, 300, 383]
    run_packed(fcsa, dtype, D, c["H"], c["Hk"], ns, lens, 640, append=c["append"], causal=c["causal"],
               groups=c["groups"], l2norm_qk=c["l2norm_qk"], window=c["window"], seed=_VARIANTS.index(variant) + D)


# ---- both sides of the split rule, and the launches ---------------------------------------------------------------
@pytest.mark.parametrize("side", ["split", "one"])
@pytest.mark.parametrize("D", [64, 128])
def test_split_rule_sides(fcsa, side, D):
    H, Hk, cap = 8, 8, 1024
    B = 3 if side == "split" else math.ceil(sm_count() / Hk)
    ns = [(1, 5, 3)[b % 3] for b in range(B)]
    s = packed_split(B, H, Hk, max(ns), cap)
    assert (s == 1) == (side == "one"), s
    lens = [(977 * b) % (cap - 8) for b in range(B)]
    run_packed(fcsa, torch.bfloat16, D, H, Hk, ns, lens, cap, seed=B + D, launches=3 if s == 1 else 4)
    # no append and no l2norm: no append pass
    run_packed(fcsa, torch.bfloat16, D, H, Hk, ns, lens, cap, append=False, l2norm_qk=False, seed=B + D + 1,
               launches=2 if s == 1 else 3)


# ---- equal lengths: bitwise the dense op -----------------------------------------------------------------------------
@pytest.mark.parametrize("side", ["split", "one"])
@pytest.mark.parametrize("window", [None, 100])
def test_equal_lengths_equal_dense_bitwise(fcsa, side, window):
    """cu = (0, n, 2n, ...): the same grid, splits and per-row arithmetic as the dense call, so o and both caches match
    it bit for bit."""
    dt, H, Hk, D, cap, n = torch.float16, 8, 2, 128, 1024, 5
    B = 2 if side == "split" else math.ceil(sm_count() / Hk)
    assert (packed_split(B, H, Hk, n, cap, window) == 1) == (side == "one")
    lens = [(311 * b + 90) % (cap - n) for b in range(B)]
    o, t = run_packed(fcsa, dt, D, H, Hk, [n] * B, lens, cap, lead=0, trail=0, window=window, seed=B, check=False)
    kc, vc = t["kc0"].clone(), t["vc0"].clone()
    dense = lambda x: x.view(B, n, *x.shape[1:]).transpose(1, 2).contiguous()
    with torch.no_grad():
        od = fcsa.flash_cosine_sim_attention_with_kv_cache(dense(t["q"]), kc, vc, t["seqlens"], dense(t["k"]),
                                                           dense(t["v"]), scale=t["scale"], window=window)
    torch.cuda.synchronize()
    assert torch.equal(o.view(B, n, H, D).transpose(1, 2).view(torch.int16), od.view(torch.int16))
    assert torch.equal(kc.view(torch.int16), t["kc"].view(torch.int16))
    assert torch.equal(vc.view(torch.int16), t["vc"].view(torch.int16))


# ---- isolation ---------------------------------------------------------------------------------------------------------
def test_other_sequences_do_not_change_a_sequence(fcsa):
    """New contents for every other sequence's q, k, v (all lengths kept): sequence b's rows of o stay bitwise the
    same."""
    dt, H, Hk, D, cap = torch.bfloat16, 8, 2, 64, 640
    ns, lens = [9, 1, 17, 40], [100, 129, 0, 255]
    b = 1
    cu, total = make_pack(ns, 3, 2)
    rows = slice(cu[b], cu[b + 1])
    o1, t = run_packed(fcsa, dt, D, H, Hk, ns, lens, cap, seed=4, check=False)
    g = torch.Generator().manual_seed(99)
    q, k, v = (x.clone() for x in (t["q"], t["k"], t["v"]))
    for x in (q, k, v):
        keep = x[rows].clone()
        x.copy_(torch.randn(x.shape, generator=g).to(dt))
        x[rows] = keep
    kc, vc = t["kc0"].clone(), t["vc0"].clone()
    with torch.no_grad():
        o2 = fcsa.flash_cosine_sim_attention_with_kv_cache(q, kc, vc, t["seqlens"], k, v, cu_seqlens_q=t["cu"],
                                                           max_seqlen_q=max(ns))
    torch.cuda.synchronize()
    assert torch.equal(o1[rows].view(torch.int16), o2[rows].view(torch.int16))
    assert torch.equal(kc[b].view(torch.int16), t["kc"][b].view(torch.int16))


# ---- edge inputs -----------------------------------------------------------------------------------------------------
def test_empty_sequences_and_rows_outside_every_sequence(fcsa):
    """Empty sequences (first, middle and last) write nothing; rows before cu[0] and after cu[B] give 0."""
    run_packed(fcsa, torch.bfloat16, 64, 4, 2, [0, 6, 0, 0, 33, 0], [5, 200, 0, 77, 128, 300], 512, lead=7, trail=9,
               seed=5)
    run_packed(fcsa, torch.float16, 128, 4, 2, [0, 0, 0], [5, 200, 0], 512, lead=4, trail=3, max_q=3, seed=6)


def test_append_past_capacity_writes_nothing_outside(fcsa):
    """L_b + n_b > capacity: T_b is clamped, the rows that do not fit are dropped.  The caches are narrowed views of
    larger buffers whose rows past the capacity hold the sentinel."""
    dt, Hk, cap, pad, D = torch.bfloat16, 2, 200, 56, 64
    ns, lens = [24, 3, 30], [cap - 10, cap, cap + 5]
    B = len(ns)
    g = torch.Generator().manual_seed(7)
    kbuf = torch.randn(B, Hk, cap + pad, D, generator=g).to(dt).cuda()
    vbuf = torch.randn(B, Hk, cap + pad, D, generator=g).to(dt).cuda()
    kbuf[:, :, cap:].view(torch.int16).fill_(SENTINEL)
    vbuf[:, :, cap:].view(torch.int16).fill_(SENTINEL)
    kc, vc = kbuf[:, :, :cap], vbuf[:, :, :cap]
    cu, total = make_pack(ns, 2, 2)
    q = torch.randn(total, 4, D, generator=g).to(dt).cuda()
    k, v = (torch.randn(total, Hk, D, generator=g).to(dt).cuda() for _ in range(2))
    k0, v0 = kbuf.clone(), vbuf.clone()
    from flash_cosine_sim_attention_b200 import l2norm_tensors
    with torch.no_grad():
        o = fcsa.flash_cosine_sim_attention_with_kv_cache(
            q, kc, vc, torch.tensor(lens, dtype=torch.int32, device="cuda"), k, v,
            cu_seqlens_q=torch.tensor(cu, dtype=torch.int32, device="cuda"), max_seqlen_q=max(ns))
    torch.cuda.synchronize()
    assert torch.isfinite(o).all()
    assert torch.equal(kbuf[:, :, cap:].view(torch.int16), k0[:, :, cap:].view(torch.int16))
    assert torch.equal(vbuf[:, :, cap:].view(torch.int16), v0[:, :, cap:].view(torch.int16))
    kn = l2norm_tensors(k)[0]
    assert torch.equal(kbuf[0, :, cap - 10:cap], kn[cu[0]:cu[0] + 10].transpose(0, 1))
    assert torch.equal(vbuf[0, :, cap - 10:cap], v[cu[0]:cu[0] + 10].transpose(0, 1))
    assert torch.equal(kbuf[1:, :, :cap], k0[1:, :, :cap]) and torch.equal(vbuf[1:, :, :cap], v0[1:, :, :cap])
    # T_b = capacity: sequence 0's queries see the whole cache, the last one every key
    from elementwise_bounds import FMT as _FMT
    qh = l2norm_tensors(q)[0]
    ref, bound = attention_bounds(qh[cu[0]:cu[1]].transpose(0, 1).unsqueeze(0), kbuf[:1, :, :cap], vbuf[:1, :, :cap],
                                  causal=True, l2norm_qk=False, fmt=_FMT[dt], shift=kernel_shift(_FMT[dt], 8),
                                  device="cuda")
    check_bound("o", o[cu[0]:cu[1]].transpose(0, 1).unsqueeze(0), ref, bound, _FMT[dt])


def test_no_rows(fcsa):
    dt = torch.bfloat16
    kc = torch.zeros(2, 2, 128, 64, dtype=dt, device="cuda")
    before = fcsa.debug()
    with torch.no_grad():
        o = fcsa.flash_cosine_sim_attention_with_kv_cache(
            torch.zeros(0, 8, 64, dtype=dt, device="cuda"), kc, kc.clone(), torch.zeros(2, dtype=torch.int32,
                                                                                        device="cuda"),
            torch.zeros(0, 2, 64, dtype=dt, device="cuda"), torch.zeros(0, 2, 64, dtype=dt, device="cuda"),
            cu_seqlens_q=torch.zeros(3, dtype=torch.int32, device="cuda"), max_seqlen_q=0)
    assert o.shape == (0, 8, 64) and fcsa.debug() == before


# ---- CUDA graph --------------------------------------------------------------------------------------------------------
def test_cuda_graph_packed_step(fcsa):
    """One packed step captured once; replayed after new contents of cu_seqlens_q (same max_seqlen_q) and cache_seqlens
    advanced on the device.  Each replay equals the eager call on a copy of the caches, bitwise."""
    dt, B, H, Hk, D, cap, total, max_q = torch.float16, 3, 8, 2, 64, 1024, 12, 8
    g = torch.Generator().manual_seed(21)
    kc, vc = (torch.randn(B, Hk, cap, D, generator=g).to(dt).cuda() for _ in range(2))
    sq = torch.zeros(total, H, D, dtype=dt, device="cuda")
    sk, sv = (torch.zeros(total, Hk, D, dtype=dt, device="cuda") for _ in range(2))
    seqlens = torch.tensor([5, 300, 700], dtype=torch.int32, device="cuda")
    cu = torch.tensor([0, 1, 9, 10], dtype=torch.int32, device="cuda")

    def step(kc_, vc_, sl, cu_):
        return fcsa.flash_cosine_sim_attention_with_kv_cache(sq, kc_, vc_, sl, sk, sv, cu_seqlens_q=cu_,
                                                             max_seqlen_q=max_q)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.no_grad(), torch.cuda.stream(side):
        step(kc.clone(), vc.clone(), seqlens.clone(), cu.clone())     # warm-up: the workspace of this stream exists
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.no_grad(), torch.cuda.graph(graph, stream=side):
        out = step(kc, vc, seqlens, cu)
    for new_cu in ([2, 10, 11, 12], [0, 8, 8, 9], [1, 2, 3, 11]):
        with torch.no_grad():
            cu.copy_(torch.tensor(new_cu, dtype=torch.int32))
            for x in (sq, sk, sv):
                x.copy_(torch.randn(x.shape, generator=g).to(dt))
            kce, vce, sle = kc.clone(), vc.clone(), seqlens.clone()
            want = step(kce, vce, sle, cu.clone())
            graph.replay()
            torch.cuda.synchronize()
            assert torch.equal(out.view(torch.int16), want.view(torch.int16))
            assert torch.equal(kc.view(torch.int16), kce.view(torch.int16))
            assert torch.equal(vc.view(torch.int16), vce.view(torch.int16))
            seqlens += cu[1:] - cu[:-1]


# ---- agreement with the training operator -------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_prefill_agrees_with_varlen_training_op(fcsa, dtype):
    """A prefill onto empty caches with causal=True: per sequence, flash_cosine_sim_attention_varlen on the same packed
    q, k, v within the relative tolerance."""
    H, Hk, D, cap = 8, 2, 128, 512
    ns = [1, 70, 0, 129, 13]
    cu, total = make_pack(ns, 0, 0)
    g = torch.Generator().manual_seed(3)
    q = torch.randn(total, H, D, generator=g).to(dtype).cuda()
    k, v = (torch.randn(total, Hk, D, generator=g).to(dtype).cuda() for _ in range(2))
    kc = torch.zeros(len(ns), Hk, cap, D, dtype=dtype, device="cuda")
    vc = torch.zeros_like(kc)
    cu_t = torch.tensor(cu, dtype=torch.int32, device="cuda")
    with torch.no_grad():
        o = fcsa.flash_cosine_sim_attention_with_kv_cache(q, kc, vc, torch.zeros(len(ns), dtype=torch.int32,
                                                                                 device="cuda"), k, v,
                                                          cu_seqlens_q=cu_t, max_seqlen_q=max(ns))
        want = fcsa.flash_cosine_sim_attention_varlen(q, k, v, cu_t, cu_t, max(ns), max(ns), causal=True)
    for b, n in enumerate(ns):
        if n:
            e = rel_err(o[cu[b]:cu[b + 1]], want[cu[b]:cu[b + 1]].double().cpu().numpy())
            record(dtype, "decode varlen vs varlen", e, TOL_OUT[dtype])
            assert e <= TOL_OUT[dtype], f"sequence {b}"
