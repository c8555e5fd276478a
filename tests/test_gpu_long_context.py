"""GPU: every kernel against the float64 reference at long context, 32k to 256k keys, on outputs whose memory starts
as NaN.

The other GPU tests stop at 4096 rows (16384 for one bf16 case), the decode tests at a 4096-row cache.  Three things
only show up past that: decode splits that hold many key tiles (and a tile count that does not divide over the
splits), rounding that grows with the number of keys (fp16 P ~ 1/N and dS fall into the subnormal range at about 16k
visible keys; the fp32 row sums and dQ reduce-adds run 8-32 times longer), and stores that a kernel skips.  The host
allocates o, inv_l, dq, dk, dv and the backward scratch with `empty`, and long tensors come from fresh `cudaMalloc`
segments that usually read as zero: a kernel that skips the store of rows that see no key, or of keys no query sees,
would pass every "exactly 0 there" check on such memory.  So before every forward and every backward `poison` fills
all free memory of the caching allocator with 0xFF bytes (NaN in fp16, bf16 and fp32) and asserts that fresh `empty`
tensors of the shapes the op is about to allocate read back as NaN.

Every check compares with the float64 reference of tests/elementwise_bounds.py (tests/window_bounds.py with a
window) computed on the GPU, on one or two (batch, head) slices per shape: the element-wise bound at C = 2 on o, dq, dk
and dv and the relative tolerances of test_gpu_parity.py.  Worst values are recorded under 'long ...' keys; the worst
per case of the dense causal D = 64 lengths, and the share of the fp16 bound that comes from its eta terms, are printed
by the last test with the file's runtime and peak device memory."""
import math
import time

import pytest
import torch

import logit_range
from elementwise_bounds import C, FMT, attention_bounds, check_bound, kernel_shift, ratio
from test_gpu_gqa import sm_count
from tile_ranges import decode_split, group_split
from test_gpu_parity import TOL_GRAD, TOL_OUT, fcsa, float32_ds_scale, float32_operands, record  # noqa: F401
from window_bounds import window_attention_bounds

pytestmark = pytest.mark.gpu

CHUNK = 256          # query rows per chunk of the float64 reference: 256 x 131072 float64 temporaries of 256 MB
SENTINEL = -1        # int16 0xFFFF: NaN in fp16 and bf16
DTYPES = [torch.bfloat16, torch.float16]
TREND = {}           # (dtype, N) -> {quantity: (worst err / (C u M), relative error)}, dense causal D = 64
ETA_SHARE = {}       # N -> {quantity: median over elements of the eta share of the fp16 bound}
_RUN = {}


@pytest.fixture(scope="module", autouse=True)
def _file_cost():
    """Runtime and peak device memory of the file; releases the workspaces and the cache at its end."""
    if torch.cuda.is_available():
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
    _RUN["t0"] = time.perf_counter()
    yield
    if torch.cuda.is_available():
        from flash_cosine_sim_attention_b200 import release_workspaces
        release_workspaces()
        torch.cuda.synchronize()
        torch.cuda.empty_cache()


# ---- memory that starts as NaN -----------------------------------------------------------------------------------
def _fill_free_blocks():
    """Fill every free block of the caching allocator on this device with 0xFF: allocate each one back (ascending sizes,
    so best fit hands out exactly that block; small-pool blocks in pieces of at most 1 MB, the small-pool limit), fill,
    free."""
    dev = torch.cuda.current_device()
    sizes = []
    for seg in torch.cuda.memory_snapshot():
        if seg["device"] != dev:
            continue
        for blk in seg["blocks"]:
            if blk["state"] != "inactive":
                continue
            s = blk["size"]
            if seg["segment_type"] == "small":
                while s > 0:
                    sizes.append(min(s, 1 << 20))
                    s -= sizes[-1]
            else:
                sizes.append(s)
    held = []
    for s in sorted(sizes):
        t = torch.empty(s, dtype=torch.uint8, device="cuda")
        t.fill_(0xFF)
        held.append(t)
    torch.cuda.synchronize()
    del held


def poison(specs):
    """Make the next allocations of `specs` ((shape, dtype) of what the op allocates, in its order; a third element
    True marks an fp32 row statistic) start as NaN.  Releases the backward workspaces, makes the allocator hold room
    for every spec, fills all of its free memory with 0xFF and asserts that the poison took: `empty` tensors of every
    spec but the statistics read back all NaN (0xFF for bytes)."""
    from flash_cosine_sim_attention_b200 import release_workspaces
    specs = [(sp[0], sp[1], len(sp) > 2 and sp[2]) for sp in specs]
    release_workspaces()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    room = [torch.empty(s, dtype=d, device="cuda") for s, d, _ in specs]
    del room
    _fill_free_blocks()
    for _ in range(3):
        # the allocator hands the same blocks to the same sequence of requests: where a probe is not poisoned yet,
        # poison the probes themselves and look again.  Probes are read on the host: a device temporary would take a
        # free block and write into it.
        probe = [torch.empty(s, dtype=d, device="cuda") for s, d, _ in specs]
        host = [t.cpu() for t in probe]
        # (fp32 row statistics, inv_l and the reciprocal norms, are poisoned where the allocator allows; every other
        # buffer must be)
        missed = [(s, d) for (s, d, stat), t in zip(specs, host) if not stat
                  and not bool((t == 0xFF).all() if d == torch.uint8 else torch.isnan(t).all())]
        del host
        if not missed:
            break
        for t in probe:
            t.view(-1).view(torch.uint8).fill_(0xFF)
        torch.cuda.synchronize()
        del probe
    assert not missed, f"the NaN poison did not reach fresh tensors of (shape, dtype) {missed}"


def dense_scratch_bytes(dtype, B, H, Hk, Nq, Nk, D):
    """Bytes of the backward's scratch workspace (the ABI's fcsa_backward_workspace_bytes)."""
    from flash_cosine_sim_attention_b200 import _abi
    p = _abi.FcsaProblem()
    p.dtype = _abi.FCSA_BF16 if dtype == torch.bfloat16 else _abi.FCSA_F16
    p.batch, p.heads, p.kv_heads, p.seq_q, p.seq_k, p.head_dim = B, H, Hk, Nq, Nk, 64 if D <= 64 else 128
    p.scale, p.shift = 8.0, 8.0
    n = _abi.load().fcsa_backward_workspace_bytes(_abi.ref(p))
    assert n > 0
    return n


def varlen_scratch_bytes(dtype, cu, H, Hk, max_len, Tq, Tk, D):
    """Bytes of the varlen backward's scratch workspace (fcsa_backward_fused_varlen_workspace_bytes; a host query that
    only checks the cumulative-length pointers, never reads them)."""
    from flash_cosine_sim_attention_b200 import _abi
    p = _abi.FcsaProblem()
    p.dtype = _abi.FCSA_BF16 if dtype == torch.bfloat16 else _abi.FCSA_F16
    p.batch, p.heads, p.kv_heads, p.seq_q, p.seq_k, p.head_dim = cu.numel() - 1, H, Hk, max_len, max_len, D
    p.scale, p.shift = 8.0, 8.0
    vl = _abi.FcsaVarlen()
    vl.cu_seqlens_q = vl.cu_seqlens_k = cu.data_ptr()
    vl.total_q, vl.total_k = Tq, Tk
    n = _abi.load().fcsa_backward_fused_varlen_workspace_bytes(_abi.ref(p), _abi.ref(vl))
    assert n > 0
    return n


def forward_specs(q, k, dtype, groups=1):
    """What a dense forward allocates: o, inv_l, q^, k^ and their reciprocal norms."""
    B, H, Nq = q.shape[0], q.shape[1], q.shape[-2]
    kv = k.shape[1] if k.ndim == 4 else 1
    return [(q.shape, dtype), ((B, H, Nq), torch.float32, True), (q.shape, dtype), (k.shape, dtype),
            ((B, H, Nq, groups), torch.float32, True), ((B, kv, k.shape[-2], groups), torch.float32, True)]


def backward_specs(q, k, v, dtype):
    """What a dense backward allocates: dq, dk, dv and the scratch workspace."""
    B, H, Nq, D = q.shape[0], q.shape[1], q.shape[-2], q.shape[-1]
    kv = k.shape[1] if k.ndim == 4 else 1
    k16 = torch.float16 if dtype == torch.float32 else dtype
    return [(q.shape, dtype), (k.shape, dtype), (v.shape, dtype),
            ((dense_scratch_bytes(k16, B, H, kv, Nq, k.shape[-2], D),), torch.uint8)]


def finite(name, t):
    assert bool(torch.isfinite(t).all()), f"{name}: NaN/Inf (an element never written keeps the NaN poison)"


def run_dense(fcsa, q, k, v, do, dtype, mask=None, launches=None, **kw):
    """Forward and backward on poisoned memory; returns {o, dq, dk, dv (, d_bias)}.  launches: kernels the backward
    must launch (the grouped-query path)."""
    bias = kw.get("attn_bias")
    qd, kd, vd = (t.clone().requires_grad_() for t in (q, k, v))
    if bias is not None:
        kw = dict(kw, attn_bias=bias.clone().requires_grad_())
    poison(forward_specs(q, k, dtype, kw.get("groups", 1)))
    o = fcsa.flash_cosine_sim_attention(qd, kd, vd, mask=mask, **kw)
    poison(backward_specs(q, k, v, dtype))
    torch.cuda.synchronize()
    before = fcsa.debug()
    o.backward(do)
    torch.cuda.synchronize()
    if launches == "loop":
        assert fcsa.debug() - before == 3
    elif launches == "split":
        assert fcsa.debug() - before >= 5
    got = {"o": o.detach(), "dq": qd.grad, "dk": kd.grad, "dv": vd.grad}
    if bias is not None:
        got["d_bias"] = kw["attn_bias"].grad
    for name, t in got.items():
        finite(name, t)
    return got


def judge(dtype, got, q, k, v, do, bounds=attention_bounds, rel_only=("o", "dq", "dk", "dv", "d_bias"), trend=None,
          **kw):
    """Bound and relative tolerance of every output in `got` (already sliced like q, k, v, do) against the float64
    reference on the GPU.  float32 inputs are judged on the operands the 16-bit kernels see."""
    l2 = kw.get("l2norm_qk", True)
    bias = kw.get("attn_bias")
    if dtype == torch.float32:
        kw["ds_scale"] = float32_ds_scale(v, do)
        fmt, q, k, v, do, b = float32_operands(q, k, v, do, bias, kw.get("scale", 8), kw.get("groups", 1), l2)
        if bias is not None:
            kw["attn_bias"] = b
    else:
        fmt = FMT[dtype]
    shift = kernel_shift(fmt, kw.get("scale", 8), kw.get("groups", 1), l2, bias)
    ref, bound = bounds(q, k, v, do, round_qk=fmt if l2 else None, fmt=fmt, shift=shift, device="cuda", chunk=CHUNK,
                        **kw)
    worst = {}
    for name, t in got.items():
        r = ref[name]
        e = float(((t.double().reshape(r.shape) - r).abs().max() / r.abs().max().clamp_min(1e-30)))
        worst[name] = (float((torch.nan_to_num(ratio(t, r, bound[name], fmt), posinf=1e300)).max()) / C, e)
    if trend is not None:
        TREND[trend] = worst
    for name, t in got.items():
        record(dtype, f"long {name}/bound", check_bound(name, t, ref, bound, fmt), 1.0)
        if name in rel_only and float(ref[name].abs().max()) > 1e-6:
            tol = TOL_OUT[dtype] if name == "o" else TOL_GRAD[dtype]
            record(dtype, f"long {name}", worst[name][1], tol)
            assert worst[name][1] <= tol, (name, worst[name][1], tol)
    del ref, bound
    return worst


def randn(g, *shape, dtype):
    return torch.randn(*shape, generator=g, device="cuda").to(dtype)


def inputs(qs, kvs, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    q, k, v = randn(g, *qs, dtype=dtype), randn(g, *kvs, dtype=dtype), randn(g, *kvs, dtype=dtype)
    return q, k, v, randn(g, *qs, dtype=dtype)


def head(t, h):
    return t[:, h:h + 1]


def eta_share(q, k, v, do):
    """Median over elements of the share of the fp16 bound M that comes from its eta terms, per quantity."""
    kw = dict(causal=True, round_qk="f16", fmt="f16", shift=kernel_shift("f16", 8), device="cuda", chunk=CHUNK)
    _, full = attention_bounds(q, k, v, do, **kw)
    _, no_eta = attention_bounds(q, k, v, do, eta=0.0, **kw)
    share = {n: float(((full[n] - no_eta[n]) / full[n].clamp_min(1e-300)).median()) for n in ("o", "dq", "dk", "dv")}
    del full, no_eta
    return share


# ---- dense, MHA -----------------------------------------------------------------------------------------------------
# (D, N, causal): D = 64 at ragged lengths past 32k, and at 4096 and 16384 for the error-against-N trend
DENSE = [(64, 4096, True), (64, 16384, True), (64, 32769, True), (64, 65601, True), (64, 131071, True),
         (64, 65601, False), (128, 65537, True), (128, 65537, False)]


@pytest.mark.parametrize("D,N,causal", DENSE, ids=[f"D{d}-N{n}-{'causal' if c else 'full'}" for d, n, c in DENSE])
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "f16"])
def test_dense(fcsa, dtype, D, N, causal):
    q, k, v, do = inputs((1, 2, N, D), (1, 2, N, D), dtype, seed=N + D)
    got = run_dense(fcsa, q, k, v, do, dtype, causal=causal)
    trend = (FMT[dtype], N) if (D == 64 and causal) else None
    if trend is not None and dtype == torch.float16:
        ETA_SHARE[N] = eta_share(*(head(t, 1) for t in (q, k, v, do)))
    judge(dtype, {n: head(t, 1) for n, t in got.items()}, *(head(t, 1) for t in (q, k, v, do)), causal=causal,
          trend=trend)


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "f16"])
def test_short_backward_after_the_longest(fcsa, dtype):
    """The longest backward leaves its zeroed dq workspace behind: a short backward on the same stream reuses it and
    must give what it gives on a new workspace - dk, dv bitwise (one CTA per key tile), dq within its reduction-order
    spread - and pass the bound.  (The relative tolerance is held on dk and dv: this seed's fp16 dq is 4.7e-3 from the
    reference relative to its maximum on a new workspace too, against 4e-3, while its bound is at 0.31.)"""
    def short():
        q, k, v, do = inputs((1, 2, 1000, 64), (1, 2, 1000, 64), dtype, seed=7)
        qd, kd, vd = (t.clone().requires_grad_() for t in (q, k, v))
        fcsa.flash_cosine_sim_attention(qd, kd, vd, causal=True).backward(do)
        torch.cuda.synchronize()
        return (q, k, v, do), {"dq": qd.grad, "dk": kd.grad, "dv": vd.grad}
    fcsa.release_workspaces()
    _, fresh = short()
    N = max(n for _, n, _ in DENSE)
    q, k, v, do = inputs((1, 2, N, 64), (1, 2, N, 64), dtype, seed=N + 64)
    run_dense(fcsa, q, k, v, do, dtype, causal=True)       # poisons, then runs the longest backward
    del q, k, v, do
    args, after = short()
    assert torch.equal(after["dk"], fresh["dk"]) and torch.equal(after["dv"], fresh["dv"])
    fmt = FMT[dtype]
    _, b = attention_bounds(*args, causal=True, round_qk=fmt, fmt=fmt, shift=kernel_shift(fmt, 8), device="cuda")
    assert float((ratio(after["dq"], fresh["dq"].double(), b["dq"], fmt) / C).max()) <= 1.0
    judge(dtype, after, *args, causal=True, rel_only=("dk", "dv"))


@pytest.mark.parametrize("nq,nk", [(1000, 131072), (65536, 3000)])
@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "f16"])
def test_dense_cross(fcsa, dtype, causal, nq, nk):
    """Nq != Nk.  With (65536, 3000) causal the first 62536 rows see no key: o and dq exactly 0 there."""
    q, k, v, do = inputs((1, 2, nq, 64), (1, 2, nk, 64), dtype, seed=nq + causal)
    got = run_dense(fcsa, q, k, v, do, dtype, causal=causal)
    if causal and nq > nk:
        blind = nq - nk
        assert bool((got["o"][:, :, :blind] == 0).all()) and bool((got["dq"][:, :, :blind] == 0).all())
    judge(dtype, {n: head(t, 1) for n, t in got.items()}, *(head(t, 1) for t in (q, k, v, do)), causal=causal)


@pytest.mark.parametrize("family", ["aligned0.05", "one_peak"])
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "f16"])
def test_logit_range_families(fcsa, dtype, family):
    """Gaussian inputs make attention almost uniform at this length; these put a row's weight on a few keys.  dq and
    dk are held to the bound only (near P = 1 the cancellation in dS makes max|dq| small, tests/logit_range.py)."""
    N = 65601
    q, k, v, do, _ = logit_range.dense(family, 1, 1, 1, N, N, 64, dtype, causal=True, seed=11)
    q, k, v, do = (t.cuda() for t in (q, k, v, do))
    got = run_dense(fcsa, q, k, v, do, dtype, causal=True)
    judge(dtype, got, q, k, v, do, causal=True, rel_only=("o", "dv"))


# ---- grouped-query --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "f16"])
def test_gqa(fcsa, dtype):
    """(1, 8 heads, 2 kv heads, 32768, 64): B * kv_heads * key tiles = 512 CTAs fill the device, so the backward keeps
    each group in one CTA (the only side of the split rule this shape reaches; MQA below takes the other)."""
    B, H, Hk, N = 1, 8, 2, 32768
    assert group_split(B, H, Hk, N, sm_count()) == 1
    q, k, v, do = inputs((B, H, N, 64), (B, Hk, N, 64), dtype, seed=21)
    got = run_dense(fcsa, q, k, v, do, dtype, causal=True, launches="loop")
    sl = slice(4, 8)                                   # kv head 1 and its group of query heads
    judge(dtype, {"o": got["o"][:, sl], "dq": got["dq"][:, sl], "dk": head(got["dk"], 1), "dv": head(got["dv"], 1)},
          q[:, sl], head(k, 1), head(v, 1), do[:, sl], causal=True)


def test_mqa_3d_keys_groups4(fcsa):
    """Shared 3-D keys / values, l2norm over 4 groups: the backward splits the group over CTAs (fp32 dk / dv
    accumulators and finish passes)."""
    dtype, B, H, N = torch.bfloat16, 1, 4, 32768
    assert group_split(B, H, 1, N, sm_count()) == H
    q, k, v, do = inputs((B, H, N, 64), (B, N, 64), dtype, seed=22)
    got = run_dense(fcsa, q, k, v, do, dtype, causal=True, groups=4, launches="split")
    judge(dtype, got, q, k, v, do, causal=True, groups=4)


# ---- key mask, bias, float32 ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "f16"])
def test_key_mask_padding_suffix(fcsa, dtype):
    """40000 keys; batch element 1 masks its last 9000 (whole masked key tiles): its masked keys get dk = dv = 0."""
    B, H, N, pad = 2, 2, 40000, 9000
    q, k, v, do = inputs((B, H, N, 64), (B, H, N, 64), dtype, seed=31)
    mask = torch.ones(B, N, dtype=torch.bool, device="cuda")
    mask[1, N - pad:] = False
    got = run_dense(fcsa, q, k, v, do, dtype, mask=mask)
    assert bool((got["dk"][1, :, N - pad:] == 0).all()) and bool((got["dv"][1, :, N - pad:] == 0).all())
    s = (slice(1, 2), slice(1, 2))
    judge(dtype, {n: t[s] for n, t in got.items()}, *(t[s] for t in (q, k, v, do)), mask=mask[1:2])


def test_fp16_head_bias_with_d_bias(fcsa):
    """One per-head fp16 attn_bias with its gradient, causal, 12289 rows (the BIAS kernels and the fp32 d_bias).

    The bias path normalises q and k with `l2norm_tensors` first, whose fp32 arithmetic rounds a few dozen of the
    786k features one ulp away from round(x / ||x||) (the reference's q^, k^).  At this length that moves single
    logits enough to put d_bias, which is dS itself, past the bound at an element (2.04 u M), while on the q^, k^
    the attention kernels are given it stays at 0.47.  So o, dv and d_bias are judged on those q^, k^ (as the decode
    tests judge the cache), dq and dk, which carry the l2norm backward to the raw inputs, on the reference's."""
    dtype, N = torch.float16, 12289
    q, k, v, do = inputs((1, 1, N, 64), (1, 1, N, 64), dtype, seed=41)
    bias = torch.randn(1, N, N, generator=torch.Generator(device="cuda").manual_seed(42), device="cuda").to(dtype)
    got = run_dense(fcsa, q, k, v, do, dtype, causal=True, attn_bias=bias)
    judge(dtype, {n: got[n] for n in ("dq", "dk")}, q, k, v, do, causal=True, attn_bias=bias)
    qh, kh = fcsa.l2norm_tensors(q, k)
    fmt = FMT[dtype]
    ref, bound = attention_bounds(qh, kh, v, do, causal=True, attn_bias=bias, l2norm_qk=False, fmt=fmt,
                                  shift=kernel_shift(fmt, 8, 1, True, bias), device="cuda", chunk=CHUNK)
    for name in ("o", "dv", "d_bias"):
        record(dtype, f"long {name}/bound", check_bound(name, got[name], ref, bound, fmt), 1.0)
        e = float((got[name].double() - ref[name]).abs().max() / ref[name].abs().max())
        tol = TOL_OUT[dtype] if name == "o" else TOL_GRAD[dtype]
        record(dtype, f"long {name}", e, tol)
        assert e <= tol, (name, e, tol)


@pytest.mark.parametrize("D", [64, 96])
def test_float32(fcsa, D):
    """The float32 path (fp16 kernels; D = 96 zero-padded to 128), judged on the operands those kernels see.  The
    kernels run on v / sv and dO / pg, so their dS is the caller's / (sv pg) and the eta of its rounding is carried
    sv pg times over (`float32_ds_scale`): the last keys, seen by a few queries with P ~ 1/N, are bound by it."""
    q, k, v, do = inputs((1, 1, 32768, D), (1, 1, 32768, D), torch.float32, seed=51 + D)
    got = run_dense(fcsa, q, k, v, do, torch.float32, causal=True)
    judge(torch.float32, got, q, k, v, do, causal=True)


# ---- varlen ---------------------------------------------------------------------------------------------------------
VARLEN = [70001, 1, 0, 32768, 129, 40000]      # 142899 rows, one sequence past 65535


def per_seq(t, s, n):
    return t[s:s + n].transpose(0, 1).unsqueeze(0)


@pytest.mark.parametrize("heads,kv_heads", [(4, 4), (4, 2)])
@pytest.mark.parametrize("causal", [True, False])
def test_varlen(fcsa, causal, heads, kv_heads):
    """Each sequence against the reference (the query heads of kv head 0), o per sequence bitwise the dense op."""
    dtype = torch.float16 if causal else torch.bfloat16
    ls, D, T = VARLEN, 64, sum(VARLEN)
    g = torch.Generator(device="cuda").manual_seed(61 + heads + kv_heads)
    q, do = randn(g, T, heads, D, dtype=dtype), randn(g, T, heads, D, dtype=dtype)
    k, v = randn(g, T, kv_heads, D, dtype=dtype), randn(g, T, kv_heads, D, dtype=dtype)
    cu = torch.tensor([0] + list(torch.tensor(ls).cumsum(0).tolist()), dtype=torch.int32, device="cuda")
    qd, kd, vd = (t.clone().requires_grad_() for t in (q, k, v))
    poison([(q.shape, dtype), ((heads, T), torch.float32, True), (q.shape, dtype), (k.shape, dtype),
            ((heads, T, 1), torch.float32, True), ((kv_heads, T, 1), torch.float32, True)])
    o = fcsa.flash_cosine_sim_attention_varlen(qd, kd, vd, cu, cu, max(ls), max(ls), causal=causal)
    poison([(q.shape, dtype), (k.shape, dtype), (v.shape, dtype),
            ((varlen_scratch_bytes(dtype, cu, heads, kv_heads, max(ls), T, T, D),), torch.uint8)])
    o.backward(do)
    torch.cuda.synchronize()
    got = {"o": o.detach(), "dq": qd.grad, "dk": kd.grad, "dv": vd.grad}
    for name, t in got.items():
        finite(name, t)
    G, s = heads // kv_heads, 0
    for n in ls:
        if n:
            with torch.no_grad():
                od = fcsa.flash_cosine_sim_attention(*(per_seq(t, s, n) for t in (q, k, v)), causal=causal)
            assert torch.equal(per_seq(got["o"], s, n), od), ("o bitwise", n)
            qs = lambda t: per_seq(t, s, n)[:, :G]
            ks = lambda t: per_seq(t, s, n)[:, :1]
            judge(dtype, {"o": qs(got["o"]), "dq": qs(got["dq"]), "dk": ks(got["dk"]), "dv": ks(got["dv"])},
                  qs(q), ks(k), ks(v), qs(do), causal=causal)
        s += n


# ---- sliding window -------------------------------------------------------------------------------------------------
def run_window(fcsa, dtype, qs, kvs, window, causal, judge_q, judge_kv, seed):
    q, k, v, do = inputs(qs, kvs, dtype, seed)
    got = run_dense(fcsa, q, k, v, do, dtype, causal=causal, window=window)
    sq = lambda t: t[:, judge_q]
    skv = lambda t: t[:, judge_kv]
    judge(dtype, {"o": sq(got["o"]), "dq": sq(got["dq"]), "dk": skv(got["dk"]), "dv": skv(got["dv"])},
          sq(q), skv(k), skv(v), sq(do), bounds=window_attention_bounds, causal=causal, window=window)
    return got


@pytest.mark.parametrize("window,dtype", [(4096, torch.float16), (4097, torch.bfloat16), (1000, torch.float16)],
                         ids=["W4096-f16", "W4097-bf16", "W1000-f16"])
@pytest.mark.parametrize("causal", [True, False])
def test_window(fcsa, window, dtype, causal):
    run_window(fcsa, dtype, (1, 2, 65601, 64), (1, 2, 65601, 64), window, causal, slice(1, 2), slice(1, 2),
               seed=window + causal)


def test_window_d128(fcsa):
    run_window(fcsa, torch.bfloat16, (1, 2, 32768, 128), (1, 2, 32768, 128), 4096, True, slice(0, 1), slice(0, 1),
               seed=71)


def test_window_gqa(fcsa):
    run_window(fcsa, torch.float16, (1, 4, 32768, 64), (1, 2, 32768, 64), 4096, True, slice(2, 4), slice(1, 2),
               seed=72)


def test_window_keys_no_query_sees(fcsa):
    """(Nq, Nk) = (1000, 65601), W = 4096, causal: keys below 65601 - 1000 - 4096 + 1 = 60506 (whole key tiles of them)
    are seen by no query, so their dk and dv are exactly 0 on memory that started as NaN."""
    nq, nk, W = 1000, 65601, 4096
    got = run_window(fcsa, torch.bfloat16, (1, 2, nq, 64), (1, 2, nk, 64), W, True, slice(1, 2), slice(1, 2), seed=73)
    unseen = nk - nq - W + 1
    assert bool((got["dk"][:, :, :unseen] == 0).all()) and bool((got["dv"][:, :, :unseen] == 0).all())
    assert not bool((got["dv"][:, :, unseen:] == 0).all())


# ---- decode ---------------------------------------------------------------------------------------------------------
def decode_scratch_bytes(dtype, B, H, Hk, Nq, cap, D, causal, window, n_new):
    from flash_cosine_sim_attention_b200 import _abi
    p = _abi.FcsaProblem()
    p.dtype = _abi.FCSA_BF16 if dtype == torch.bfloat16 else _abi.FCSA_F16
    p.batch, p.heads, p.kv_heads, p.seq_q, p.seq_k, p.head_dim = B, H, Hk, Nq, cap, D
    p.causal, p.window, p.scale, p.shift = int(causal), window or 0, 8.0, 8.0
    n = _abi.load().fcsa_decode_workspace_bytes(_abi.ref(p), n_new)
    assert n > 0
    return n


def decode_check(fcsa, dtype, D, G, Nq, cap, append, window=None, seed=0):
    """One call over lengths [cap, cap - 1, 100003, 1, 0] (100003 clamps to the capacity of a 65536 cache) with one
    kv head: the append bitwise, the NaN sentinel past each T_b, o per batch element against the reference."""
    from flash_cosine_sim_attention_b200 import l2norm_tensors
    lens, Hk = [cap, cap - 1, 100003, 1, 0], 1
    B, H, n_new = len(lens), G, (Nq if append else 0)
    if window is None:
        # more than one key tile per split, and a tile count (T_b = capacity) that the splits do not divide
        s, nt = decode_split(B * Hk * math.ceil(G * Nq / 64), cap, sm_count()), cap // 128
        assert nt >= 2 * s and nt % s != 0, (nt, s)
    g = torch.Generator(device="cuda").manual_seed(seed)
    q = randn(g, B, H, Nq, D, dtype=dtype)
    kc = l2norm_tensors(randn(g, B, Hk, cap, D, dtype=dtype))[0]
    vc = randn(g, B, Hk, cap, D, dtype=dtype)
    T = [min(min(L, cap) + n_new, cap) for L in lens]
    for b, L in enumerate(lens):
        kc[b, :, L:].view(torch.int16).fill_(SENTINEL)
        vc[b, :, L:].view(torch.int16).fill_(SENTINEL)
    k = v = None
    if append:
        k, v = randn(g, B, Hk, n_new, D, dtype=dtype), randn(g, B, Hk, n_new, D, dtype=dtype)
    seqlens = torch.tensor(lens, dtype=torch.int32, device="cuda")
    poison([((B, H, Nq, D), dtype),
            ((decode_scratch_bytes(dtype, B, H, Hk, Nq, cap, D, True, window, n_new),), torch.uint8)])
    with torch.no_grad():
        o = fcsa.flash_cosine_sim_attention_with_kv_cache(q, kc, vc, seqlens, k, v, window=window)
    torch.cuda.synchronize()
    kn = l2norm_tensors(k)[0] if append else None
    qh = l2norm_tensors(q)[0]
    fmt = FMT[dtype]
    for b, L in enumerate(lens):
        L = min(L, cap)
        n = T[b] - L
        if n:
            assert torch.equal(kc[b, :, L:T[b]], kn[b, :, :n]) and torch.equal(vc[b, :, L:T[b]], v[b, :, :n])
        assert bool((kc[b, :, T[b]:].view(torch.int16) == SENTINEL).all()), ("k sentinel", b)
        assert bool((vc[b, :, T[b]:].view(torch.int16) == SENTINEL).all()), ("v sentinel", b)
        if T[b] == 0:
            assert bool((o[b] == 0).all())
            continue
        kw = dict(causal=True, l2norm_qk=False, fmt=fmt, shift=kernel_shift(fmt, 8), device="cuda")
        if window is None:
            ref, bound = attention_bounds(qh[b:b + 1], kc[b:b + 1, :, :T[b]], vc[b:b + 1, :, :T[b]], **kw)
        else:
            ref, bound = window_attention_bounds(qh[b:b + 1], kc[b:b + 1, :, :T[b]], vc[b:b + 1, :, :T[b]],
                                                 window=window, **kw)
        record(dtype, "long decode o/bound", check_bound("o", o[b:b + 1], ref, bound, fmt), 1.0)
        e = float((o[b:b + 1].double() - ref["o"]).abs().max() / ref["o"].abs().max())
        record(dtype, "long decode o", e, TOL_OUT[dtype])
        assert e <= TOL_OUT[dtype], (b, T[b], e)


# every (capacity, D, dtype, append) with one (G, Nq) each, so that every G and Nq meets both capacities
_DECODE = [(cap, D, dt, app) for cap in (65536, 262144) for D in (64, 128) for dt in DTYPES for app in (True, False)]
_GNQ = [(4, 1), (8, 5), (4, 17), (8, 1), (4, 5), (8, 17)]


@pytest.mark.parametrize("i", range(len(_DECODE)),
                         ids=[f"cap{c}-D{d}-{FMT[t]}-{'append' if a else 'noappend'}-G{_GNQ[i % 6][0]}-Nq{_GNQ[i % 6][1]}"
                              for i, (c, d, t, a) in enumerate(_DECODE)])
def test_decode(fcsa, i):
    cap, D, dtype, append = _DECODE[i]
    G, Nq = _GNQ[i % len(_GNQ)]
    decode_check(fcsa, dtype, D, G, Nq, cap, append, seed=i)


def test_decode_window(fcsa):
    decode_check(fcsa, torch.bfloat16, 128, 8, 5, 262144, True, window=4096, seed=99)


# ---- the file's cost and the error-against-N trend --------------------------------------------------------------------
def test_report_long_context(capsys):
    """Prints the worst err / (C u M) and relative error of the dense causal D = 64 cases per length, the eta share of
    the fp16 bound, the file's runtime and its peak device memory."""
    with capsys.disabled():
        for (fmt, N), w in sorted(TREND.items()):
            cells = "  ".join(f"{n} {w[n][0]:.2f} ({w[n][1]:.1e})" for n in ("o", "dq", "dk", "dv"))
            print(f"\n  long {fmt} N={N}: {cells}", end="")
        for N, s in sorted(ETA_SHARE.items()):
            print(f"\n  long f16 N={N} median eta share of M: " + "  ".join(f"{n} {x:.2f}" for n, x in s.items()),
                  end="")
        print(f"\n  long context file: {time.perf_counter() - _RUN['t0']:.0f} s, peak max_memory_allocated "
              f"{torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB, {torch.cuda.get_device_name()}", end="")
