"""GPU tests at the ends of the logit range (run on an H100 with `pytest -m gpu`): the input families of
tests/logit_range.py - queries aligned with keys in every l2norm group, tokens attending to themselves, one exact key
per row, runs of duplicate keys, opposed queries and all-zero rows - through every entry point, against the float64
reference of tests/elementwise_bounds.py on the same 16-bit operands.

The Gaussian inputs of the other GPU tests keep scale * q^.k^ far from the top of the shifted exponential's range (at
D = 64 the best match of a row is a cosine near 0.5); these reach it, and the bottom.

Judgement: every output under the element-wise bound |got - ref| <= C u M at C = 2 (the worst err / (C u M) is
recorded under '<dtype>:<name>/bound'), o and dv also under the relative tolerances of test_gpu_parity.py.  dq and dk
get the bound alone: when one key takes a row, dS = P (dP - delta) cancels to far below the rounding of its terms, so
max|dq| and max|dk| shrink while the rounding does not - the float32 emulation of the kernels' own arithmetic
(test_elementwise_bounds.emulate) is 10^4 times over the relative tolerance there and within half the bound.

Covering grids, not the full product: every family, (heads, kv_heads), causal flag and (groups, scale) appears with
both dtypes and both head dims.  fp16 runs at the (groups, scale) where exp(scale q.k - shift) fits its range; where it
does not (scale * (groups - 1) > ln 65504), the entry points warn, and the last tests pin exactly when."""
import importlib
import math
import warnings

import pytest
import torch

import logit_range
from elementwise_bounds import FMT, attention_bounds, check_bound, kernel_shift
from test_gpu_decode import n_split_of, sm_count
from test_gpu_parity import TOL_GRAD, TOL_OUT, fcsa, float32_operands, record, rel_err  # noqa: F401
from test_gpu_varlen import LONG, cu_of, per_seq, run_varlen

pytestmark = pytest.mark.gpu

GS = {torch.bfloat16: [(4, 8), (1, 32), (2, 16), (1, 8), (1, 10), (2, 5), (8, 1)],
      torch.float16: [(1, 8), (1, 10), (2, 5), (8, 1)]}
HEADS = [(4, 4), (4, 2), (4, 1)]
REL_TOL = {"bf16": {"o": TOL_OUT[torch.bfloat16], "dv": TOL_GRAD[torch.bfloat16]},
           "f16": {"o": TOL_OUT[torch.float16], "dv": TOL_GRAD[torch.float16]}}


def judge(dtype, got, q, k, v, do=None, what="", shift=None, **kw):
    """Every output in `got` ({name: tensor}) under the element-wise bound, o and dv also under the relative tolerance
    of the kernels' operand type.  float32 inputs are judged on the operands the 16-bit kernels see.  shift: the
    kernels' logit shift when it is not the one of these keywords (already-normalised operands)."""
    l2 = kw.get("l2norm_qk", True)
    bias = kw.get("attn_bias")
    if dtype == torch.float32:
        fmt, q, k, v, do, kw["attn_bias"] = float32_operands(q, k, v, do, bias, kw.get("scale", 8),
                                                             kw.get("groups", 1), l2)
    else:
        fmt = FMT[dtype]
    if shift is None:
        shift = kernel_shift(fmt, kw.get("scale", 8), kw.get("groups", 1), l2, bias)
    ref, bound = attention_bounds(q, k, v, do, round_qk=fmt if l2 else None, fmt=fmt, shift=shift, device="cuda", **kw)
    for name, t in got.items():
        if name in REL_TOL[fmt]:
            e = rel_err(t, ref[name].cpu().numpy())
            record(dtype, f"range{what} {name}", e, REL_TOL[fmt][name])
            assert e <= REL_TOL[fmt][name], (name, e)
        try:
            w = check_bound(name, t, ref, bound, fmt)
        except AssertionError:
            record(dtype, f"{name}/bound", float("inf"), 1.0)
            raise
        record(dtype, f"{name}/bound", w, 1.0)


def run_dense(fcsa, q, k, v, do, grads=True, **kw):
    qd, kd, vd = (t.cuda().requires_grad_(grads) for t in (q, k, v))
    bias = kw.pop("attn_bias", None)
    bd = None if bias is None else bias.cuda().requires_grad_(grads)
    o = fcsa.flash_cosine_sim_attention(qd, kd, vd, attn_bias=bd, **kw)
    assert o.shape == q.shape and o.dtype == q.dtype
    got = {"o": o.detach()}
    if grads:
        o.backward(do.cuda())
        got.update(dq=qd.grad, dk=kd.grad, dv=vd.grad)
        if bd is not None:
            got["d_bias"] = bd.grad
    return got


# ---- 1. dense forward and backward: every family ----------------------------------------------------------------
def _dense_cases():
    cases = []
    for dtype in (torch.float16, torch.bfloat16):
        gs = GS[dtype]
        for D in (64, 128):
            for i, fam in enumerate(logit_range.FAMILIES):
                for j in range(2):
                    g, s = gs[(2 * i + j + D // 64) % len(gs)]
                    H, Hk = HEADS[(i + j + D // 64) % len(HEADS)]
                    causal = (i + j) % 2 == 0
                    mode = "causal" if causal else "full"
                    cases.append(pytest.param(dtype, D, fam, g, s, H, Hk, causal,
                                              id=f"{FMT[dtype]}-D{D}-{fam}-g{g}s{s}-h{H}kv{Hk}-{mode}"))
    return cases


@pytest.mark.parametrize("dtype,D,family,groups,scale,H,Hk,causal", _dense_cases())
def test_dense_families(fcsa, dtype, D, family, groups, scale, H, Hk, causal):
    """Nq = Nk = 300: ragged last tiles.  fp16 zero rows: forward only (the l2norm backward of a zero row is x 1e12)."""
    q, k, v, do, _ = logit_range.dense(family, 1, H, Hk, 300, 300, D, dtype, causal=causal, seed=D + groups + scale)
    grads = not (family == "zero_rows" and dtype == torch.float16)
    kw = dict(groups=groups, scale=scale, causal=causal)
    got = run_dense(fcsa, q, k, v, do, grads=grads, **kw)
    judge(dtype, got, q, k, v, do if grads else None, **kw)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_dense_causal_diagonal_long(fcsa, dtype):
    """(1, 2, 2048, 64): every token attends to itself over 16 key tiles, through the D = 64 backward pipeline."""
    q, k, v, do, _ = logit_range.dense("diagonal", 1, 2, 2, 2048, 2048, 64, dtype, causal=True, seed=5)
    got = run_dense(fcsa, q, k, v, do, causal=True)
    judge(dtype, got, q, k, v, do, causal=True)


# ---- 2. the other kernels and paths on aligned and one-peak inputs ------------------------------------------------
@pytest.mark.parametrize("D,family,causal", [(64, "aligned0.05", True), (64, "one_peak", False),
                                             (128, "aligned0.05", False), (128, "one_peak", True)])
def test_bias_fp16_at_the_top(fcsa, D, family, causal):
    """BIAS kernels in fp16: +10 on each row's aligned key, so that key's logit minus the shift (which the bias maximum
    joins) is the top of the range, 15 ln 2; the other entries are 0.5 N(0, 1)."""
    dtype, H, Hk, N = torch.float16, 4, 2, 300
    q, k, v, do, peak = logit_range.dense(family, 1, H, Hk, N, N, D, dtype, causal=causal, seed=D + causal)
    g = torch.Generator().manual_seed(D)
    bias = torch.randn(H, N, N, generator=g) * 0.5
    hh, ii = torch.meshgrid(torch.arange(H), torch.arange(N), indexing="ij")
    ok = peak[0] >= 0
    bias[hh[ok], ii[ok], peak[0][ok]] = 10.0
    bias = bias.to(dtype)
    kw = dict(causal=causal, attn_bias=bias)
    got = run_dense(fcsa, q, k, v, do, **kw)
    judge(dtype, got, q, k, v, do, what=" bias", **kw)


@pytest.mark.parametrize("family,groups,scale,D", [("aligned0.05", 1, 8, 64), ("one_peak", 1, 8, 128),
                                                   ("aligned0.05", 4, 8, 128), ("one_peak", 4, 8, 64),
                                                   ("aligned0.05", 2, 16, 64), ("one_peak", 2, 16, 128)])
def test_float32_path(fcsa, family, groups, scale, D):
    """float32 inputs: the fp16 kernels at (1, 8), the bf16 kernels at (4, 8) and (2, 16)."""
    dtype = torch.float32
    causal = family == "one_peak"
    q, k, v, do, _ = logit_range.dense(family, 1, 4, 2, 300, 300, D, dtype, causal=causal, seed=D + scale)
    kw = dict(groups=groups, scale=scale, causal=causal)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")                  # the float32 path names its switch to the bf16 kernels
        got = run_dense(fcsa, q, k, v, do, **kw)
    assert all(t.dtype == torch.float32 for t in got.values())
    judge(dtype, got, q, k, v, do, what=" f32", **kw)


@pytest.mark.parametrize("family", ["aligned0.05", "one_peak"])
@pytest.mark.parametrize("D", [32, 96])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_padded_head_dims(fcsa, dtype, D, family):
    groups, scale = {(torch.float16, 32): (2, 5), (torch.float16, 96): (1, 8),
                     (torch.bfloat16, 32): (4, 8), (torch.bfloat16, 96): (2, 16)}[dtype, D]
    causal = family == "aligned0.05"
    q, k, v, do, _ = logit_range.dense(family, 1, 4, 2, 300, 300, D, dtype, causal=causal, seed=D)
    kw = dict(groups=groups, scale=scale, causal=causal)
    got = run_dense(fcsa, q, k, v, do, **kw)
    judge(dtype, got, q, k, v, do, what=" padded", **kw)


@pytest.mark.parametrize("heads,kv_heads", [(8, 8), (8, 2)])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_varlen_diagonal(fcsa, dtype, D, heads, kv_heads):
    """Packed sequences of test_gpu_varlen.py's LONG lengths, each token attending to itself; each sequence against the
    float64 reference on it alone."""
    groups, scale = {(torch.float16, 64): (1, 8), (torch.float16, 128): (2, 5),
                     (torch.bfloat16, 64): (4, 8), (torch.bfloat16, 128): (1, 32)}[dtype, D]
    causal = (D == 64) == (heads == kv_heads)
    ls = LONG
    q, k, v, do = logit_range.packed("diagonal", ls, ls, heads, kv_heads, D, dtype, causal=causal, seed=D + kv_heads)
    cu = cu_of(ls)
    kw = dict(groups=groups, scale=scale, causal=causal)
    o, dq, dk, dv, _ = run_varlen(fcsa, q, k, v, do, cu, cu, max(ls), max(ls), **kw)
    s = 0
    for n in ls:
        if n:
            got = {name: per_seq(t, s, n) for name, t in (("o", o), ("dq", dq), ("dk", dk), ("dv", dv))}
            judge(dtype, got, *(per_seq(t, s, n) for t in (q, k, v, do)), what=" varlen", **kw)
        s += n


def _decode(fcsa, family, dtype, D, H, Hk, Nq, lens, cap, groups, scale, launches=None, seed=0):
    """Append Nq new keys and attend with Nq new queries built with the whole key sequence; returns (o, q^, caches)."""
    from flash_cosine_sim_attention_b200 import l2norm_tensors
    q, kc, vc, k, v = (t.cuda() for t in logit_range.cache(family, lens, cap, Nq, H, Hk, Nq, D, dtype, seed=seed))
    kc = l2norm_tensors(kc, groups=groups)[0].contiguous()          # the cache holds normalised keys
    seqlens = torch.tensor(lens, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    before = fcsa.debug()
    with torch.no_grad():
        o = fcsa.flash_cosine_sim_attention_with_kv_cache(q, kc, vc, seqlens, k, v, scale=scale, groups=groups)
    torch.cuda.synchronize()
    if launches is not None:
        assert fcsa.debug() - before == launches
    return o, l2norm_tensors(q, groups=groups)[0], kc, vc


@pytest.mark.parametrize("side", ["split", "one"])
@pytest.mark.parametrize("Nq", [1, 33])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_decode_aligned_cache(fcsa, dtype, Nq, side):
    """New queries aligned with cache rows (and with the new keys), on both sides of the split rule: the launch count
    is append pass + decode kernel (+ the combine kernel when the keys are split)."""
    D = 64 if (Nq == 1) == (side == "split") else 128
    H, Hk, cap = (8, 8, 512) if Nq == 1 else (8, 2, 512)
    G = H // Hk
    B = {(1, "split"): 2, (1, "one"): math.ceil(sm_count() / Hk),
         (33, "split"): 1, (33, "one"): math.ceil(sm_count() / (Hk * math.ceil(G * Nq / 64)))}[Nq, side]
    s = n_split_of(B, H, Hk, Nq, cap)
    assert (s == 1) == (side == "one"), s
    groups, scale = (1, 8) if dtype == torch.float16 else (4, 8)
    family = "aligned0.05" if side == "split" else "one_peak"
    lens = [(131 * b + 97) % (cap - Nq) for b in range(B)]
    o, qh, kc, vc = _decode(fcsa, family, dtype, D, H, Hk, Nq, lens, cap, groups, scale,
                            launches=2 if s == 1 else 3, seed=Nq + D)
    for b, L in enumerate(lens):
        T = L + Nq
        judge(dtype, {"o": o[b:b + 1]}, qh[b:b + 1], kc[b:b + 1, :, :T], vc[b:b + 1, :, :T], what=" decode",
              shift=kernel_shift(FMT[dtype], scale, groups), scale=scale, causal=True, l2norm_qk=False)


# ---- 3. the fp16 regime where p can exceed 65504: a warning, exactly there, and finite outputs ---------------------
# (groups 3 runs on the dense op only, at head dim 96: varlen and decode take power-of-two groups of 64 or 128)
SATURATION = [(4, 8, True), (3, 8, True), (2, 16, True), (2, 8, False), (8, 1, False), (1, 10, False)]


def _overflow_warnings(call):
    m = importlib.import_module("flash_cosine_sim_attention_b200.flash_cosine_sim_attention")
    m._warned.discard("f16-overflow")
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        out = call()
    return out, sum("exceeds fp16's maximum" in str(x.message) for x in w)


@pytest.mark.parametrize("groups,scale,warns", SATURATION)
def test_fp16_overflow_dense(fcsa, groups, scale, warns, capsys):
    """(1, 1, 256, D), queries that are noisy copies of keys (sigma 0.3).  Where no overflow is possible the outputs are
    also under the bound; where it is, the error of o is printed (it is the reason for the warning)."""
    m = importlib.import_module("flash_cosine_sim_attention_b200.flash_cosine_sim_attention")
    dtype, D = torch.float16, (96 if groups == 3 else 64)
    assert m._fp16_overflows(dtype, scale, groups, True) == warns
    q, k, v, do, _ = logit_range.dense("aligned0.3", 1, 1, 1, 256, 256, D, dtype, seed=0)
    kw = dict(groups=groups, scale=scale)
    got, n = _overflow_warnings(lambda: run_dense(fcsa, q, k, v, do, **kw))
    assert n == (1 if warns else 0)
    for name, t in got.items():
        assert torch.isfinite(t).all(), name
    if not warns:
        judge(dtype, got, q, k, v, do, what=" f16 range", **kw)
        return
    ref, _ = attention_bounds(q, k, v, round_qk="f16", fmt="f16", device="cuda", **kw)
    err = float((got["o"].double() - ref["o"]).abs().max() / ref["o"].abs().max())
    with capsys.disabled():
        print(f"\n  fp16 groups {groups} scale {scale} (warned): o relative error {err:.3g}", end="")


@pytest.mark.parametrize("groups,scale,warns", [c for c in SATURATION if c[0] != 3])
def test_fp16_overflow_varlen(fcsa, groups, scale, warns):
    ls = [65, 0, 129, 300]
    q, k, v, do = logit_range.packed("aligned0.3", ls, ls, 4, 2, 64, torch.float16, seed=1)
    cu = cu_of(ls)
    got, n = _overflow_warnings(lambda: run_varlen(fcsa, q, k, v, do, cu, cu, max(ls), max(ls), groups=groups,
                                                   scale=scale))
    assert n == (1 if warns else 0)
    for t in got[:4]:
        assert torch.isfinite(t).all()


@pytest.mark.parametrize("groups,scale,warns", [c for c in SATURATION if c[0] != 3])
def test_fp16_overflow_decode(fcsa, groups, scale, warns):
    (o, *_), n = _overflow_warnings(lambda: _decode(fcsa, "aligned0.3", torch.float16, 64, 4, 2, 5, [100, 300], 512,
                                                    groups, scale, seed=2))
    assert n == (1 if warns else 0)
    assert torch.isfinite(o).all()
