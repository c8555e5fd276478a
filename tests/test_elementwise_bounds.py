"""CPU tests of the element-wise error bound (tests/elementwise_bounds.py), both ways: its reference part is the
oracle, it accepts an emulation of the kernels' roundings with margin, and it rejects the tile-shaped mistakes that
the relative-to-max metric of the GPU tests lets through."""
import numpy as np
import pytest
import torch

import logit_range
from elementwise_bounds import C, U, attention_bounds, check_bound, kernel_shift, ratio
from gqa_reference import gqa_attention
from oracle import cosine_sim_attention_oracle as oracle

# (q shape, k shape, kwargs, bias planes or None): bias with d_bias, mask, causal Nq != Nk, groups, GQA, MQA,
# merged batch-heads and l2norm_qk=False
CASES = {
    "bias_heads_mask_cross": ((2, 3, 70, 64), (2, 3, 90, 64), dict(mask_p=0.4), "heads"),
    "bias_batch_causal": ((2, 2, 80, 64), (2, 2, 80, 64), dict(causal=True), "batch"),
    "causal_q_lt_k": ((1, 2, 40, 64), (1, 2, 150, 64), dict(causal=True), None),
    "causal_q_gt_k": ((1, 2, 150, 128), (1, 2, 40, 128), dict(causal=True), None),
    "groups4_scale2": ((1, 2, 100, 64), (1, 2, 100, 64), dict(groups=4, scale=2), None),
    "gqa_6_3": ((2, 6, 60, 64), (2, 3, 90, 64), dict(mask_p=0.3), None),
    "gqa_bias_causal": ((1, 4, 64, 64), (1, 2, 64, 64), dict(causal=True), "heads"),
    "mqa": ((2, 4, 70, 64), (2, 70, 64), dict(causal=True), None),
    "merged": ((4, 90, 64), (4, 90, 64), dict(causal=True), None),
    "no_l2norm": ((1, 2, 80, 64), (1, 2, 80, 64), dict(l2norm_qk=False, scale=1, amp=0.2), None),
}


def make_case(name, fmt, seed=0):
    qs, ks, kw, bias_kind = CASES[name]
    kw = dict(kw)
    rng = np.random.default_rng(seed)
    rnd = lambda shape, amp=1.0: oracle.round_to(rng.standard_normal(shape) * amp, fmt)
    amp = kw.pop("amp", 1.0)
    q, k, v, do = rnd(qs, amp), rnd(ks, amp), rnd(ks), rnd(qs)
    mask_p = kw.pop("mask_p", None)
    if mask_p is not None:
        kw["mask"] = rng.random((qs[0], ks[-2])) > mask_p
        kw["mask"][:, 0] = True
    if bias_kind is not None:
        planes = qs[0] if bias_kind == "batch" else qs[1]
        kw["attn_bias"] = rnd((planes, qs[-2], ks[-2]))
        kw["attn_bias_batch_dim"] = bias_kind == "batch"
    return q, k, v, do, kw


def reference(q, k, v, do, kw, fmt):
    """oracle.attention (through gqa_attention for grouped keys/values) with the 16-bit q^, k^ of `fmt`."""
    rq = fmt if kw.get("l2norm_qk", True) else None
    f = gqa_attention if (k.ndim == 4 and q.ndim == 4 and k.shape[1] != q.shape[1]) else oracle.attention
    return f(q, k, v, d_out=do, empty_rows="zero", round_qk=rq, **kw)


@pytest.mark.parametrize("name", sorted(CASES))
def test_reference_matches_oracle(name):
    q, k, v, do, kw = make_case(name, "bf16")
    want = reference(q, k, v, do, kw, "bf16")
    ref, bound = attention_bounds(q, k, v, do, round_qk="bf16" if kw.get("l2norm_qk", True) else None, chunk=32,
                                  **kw)
    names = ("o", "dq", "dk", "dv", "d_bias")[:len(want)]
    assert sorted(ref) == sorted(names)
    for n, w in zip(names, want):
        got = ref[n].numpy()
        assert got.shape == w.shape, n
        assert np.abs(got - w).max() <= 1e-12 * max(1.0, np.abs(w).max()), n
        assert (bound[n].numpy() >= np.abs(w) - 1e-12).all(), n      # M is never below |ref| (it contains it)


# ---- a numpy emulation of the kernels' rounding points ---------------------------------------------------------
def emulate(q, k, v, do, fmt, mask=None, attn_bias=None, scale=8, groups=1, causal=False, l2norm_qk=True,
            attn_bias_batch_dim=False):
    """What the kernels compute, in float32 with every 16-bit rounding in its place: q^, k^ stored in T; S = q^ k^T
    and p = exp(scale S + bias - shift) in fp32; p -> T before P V, l summed in fp32, o -> T; in the backward
    delta from the stored o, P -> T before dV, dS -> T before dK / dQ, the l2norm backward on the stored q^, k^ with
    fp32 1/||x||, outputs -> T (d_bias summed in fp32).  p is packed with saturation in fp16 (65504, not inf) while l
    sums the unsaturated fp32 p, and 1/||x|| uses the l2norm's 1e-12 clamp, as in the kernels."""
    f32 = np.float32
    T = lambda x: oracle.round_to(x, fmt).astype(f32)
    Tp = (lambda x: T(np.minimum(x, f32(65504)))) if fmt == "f16" else T
    shift = f32(kernel_shift(fmt, scale, groups, l2norm_qk, attn_bias))
    merged, single = q.ndim == 3, k.ndim == 3
    if merged:
        q, k, v, do = q[:, None], k[:, None], v[:, None], do[:, None]
        attn_bias_batch_dim = True
    elif single:
        k, v = k[:, None], v[:, None]
    B, H, Nq, D = q.shape
    Hk, Nk = k.shape[1], k.shape[2]
    G = H // Hk
    if l2norm_qk:
        (qn, nq), (kn, nk) = oracle.l2norm(q, groups), oracle.l2norm(k, groups)
        qn, kn = T(qn), T(kn)
    else:
        qn, kn = q.astype(f32), k.astype(f32)
    v, do = v.astype(f32), do.astype(f32)
    bias = None if attn_bias is None else attn_bias.astype(f32)
    o = np.zeros(q.shape, f32)
    dqn, dkn, dv = np.zeros(q.shape, f32), np.zeros(k.shape, f32), np.zeros(v.shape, f32)
    db = None if bias is None else np.zeros(bias.shape, f32)
    for b in range(B):
        vis = oracle._visibility(b, Nq, Nk, mask, causal)
        for h in range(H):
            hk = h // G
            logit = f32(scale) * (qn[b, h] @ kn[b, hk].T)
            if bias is not None:
                logit = logit + bias[b if attn_bias_batch_dim else h]
            p = np.where(vis, np.exp(logit - shift), f32(0))
            l = p.sum(-1, dtype=f32)
            inv_l = f32(1) / np.maximum(l, f32(1e-37))
            o[b, h] = T((Tp(p) @ v[b, hk]) * inv_l[:, None])
            delta = (do[b, h] * o[b, h]).sum(-1, dtype=f32, keepdims=True)
            with np.errstate(over="ignore"):         # rows without a visible key: 0 * (1 / 1e-37), then masked
                P = np.where(vis, np.exp(logit - shift) * inv_l[:, None], f32(0))
            dv[b, hk] += T(P).T @ do[b, h]
            ds = P * (do[b, h] @ v[b, hk].T - delta)
            dsr = T(ds)
            dqn[b, h] = f32(scale) * (dsr @ kn[b, hk])
            dkn[b, hk] += f32(scale) * (dsr.T @ qn[b, h])
            if db is not None:
                db[b if attn_bias_batch_dim else h] += ds

    dq, dk = (_l2bwd(dqn, qn, nq, groups), _l2bwd(dkn, kn, nk, groups)) if l2norm_qk else (dqn, dkn)
    out = [T(o), T(dq), T(dk), T(dv)] + ([] if db is None else [T(db)])
    if merged:
        out[0], out[1], out[2], out[3] = out[0][:, 0], out[1][:, 0], out[2][:, 0], out[3][:, 0]
    elif single:
        out[2], out[3] = out[2][:, 0], out[3][:, 0]
    return out


def _l2bwd(dy, y, n, groups):
    """The l2norm backward in float32 on the stored y = x^ with 1/||x|| from the 1e-12 clamp."""
    f32 = np.float32
    g = y.reshape(*y.shape[:-1], groups, -1)
    d = dy.reshape(g.shape)
    rn = f32(1) / np.maximum(n, 1e-12).astype(f32)
    return ((d - g * (g * d).sum(-1, keepdims=True)) * rn[..., None]).reshape(y.shape)


def emulate_long_causal(q, k, v, do, fmt, rows=512, scale=8):
    """`emulate` for one causal (1, 1, N, D) problem at long N, in torch float32 on the CPU, chunked over query rows.
    The fp32 sums run as in the kernels: the row sum l, O = P~ V and dQ = dS~ K are summed tile by tile over 128 keys
    (each tile's partial in fp32, the tiles added one after another), dK and dV over the query rows.  Returns
    [o, dq, dk, dv] as (1, 1, N, D) float64 tensors."""
    dt = torch.bfloat16 if fmt == "bf16" else torch.float16
    T = lambda x: x.to(dt).float()
    Tp = (lambda x: T(x.clamp(max=65504.0))) if fmt == "f16" else T
    shift = float(kernel_shift(fmt, scale))
    f = lambda x: torch.from_numpy(np.ascontiguousarray(x[0, 0])).float()
    q, k, v, do = f(q), f(k), f(v), f(do)
    qn, kn = T(q / q.norm(dim=-1, keepdim=True)), T(k / k.norm(dim=-1, keepdim=True))
    N, D = q.shape
    o, dqn = torch.zeros(N, D), torch.zeros(N, D)
    dkn, dv = torch.zeros(N, D), torch.zeros(N, D)

    def tile_sum(x, y):
        """sum over the key tiles of x[:, tile] @ y[tile], one tile after another, in fp32"""
        nt = x.shape[1] // 128
        part = torch.bmm(x.reshape(-1, nt, 128).transpose(0, 1), y.reshape(nt, 128, -1))
        acc = torch.zeros_like(part[0])
        for t in range(nt):
            acc += part[t]
        return acc

    for r0 in range(0, N, rows):
        r1 = min(N, r0 + rows)
        ke = (r1 + 127) // 128 * 128                   # whole key tiles up to the chunk's last visible key
        kp = torch.zeros(ke, D)
        vp = torch.zeros(ke, D)
        kp[:min(ke, N)], vp[:min(ke, N)] = kn[:ke], v[:ke]
        cols = torch.arange(ke)
        vis = cols[None, :] <= torch.arange(r0, r1)[:, None]
        p = torch.where(vis, torch.exp(scale * (qn[r0:r1] @ kp.T) - shift), torch.zeros(()))
        lt = p.reshape(r1 - r0, -1, 128).sum(-1)
        l = torch.zeros(r1 - r0)
        for t in range(lt.shape[1]):
            l += lt[:, t]
        inv_l = 1.0 / l.clamp_min(1e-37)
        ob = T(tile_sum(Tp(p), vp) * inv_l[:, None])
        o[r0:r1] = ob
        dob = do[r0:r1]
        delta = (dob * ob).sum(-1, keepdim=True)
        P = p * inv_l[:, None]
        dv[:ke] += (T(P).T @ dob)[:min(ke, N)]
        dsr = T(P * (dob @ vp.T - delta))
        dqn[r0:r1] = scale * tile_sum(dsr, kp)
        dkn[:ke] += (scale * (dsr.T @ qn[r0:r1]))[:min(ke, N)]
    l2 = lambda dy, x, y: (dy - y * (y * dy).sum(-1, keepdim=True)) / x.norm(dim=-1, keepdim=True)
    out = [T(o), T(l2(dqn, q, qn)), T(l2(dkn, k, kn)), T(dv)]
    return [t.double()[None, None] for t in out]


@pytest.mark.parametrize("fmt", ["bf16", "f16"])
def test_emulated_rounding_within_bound_at_32k(fmt, capsys):
    """Causal (1, 1, 32768, 64): the emulation's worst err / (u M) stays within C / 2 where fp16 P ~ 1/N and dS are
    subnormal and the fp32 sums run over 256 key tiles, so C = 2 holds at long context too."""
    N = 32768
    rng = np.random.default_rng(5)
    q, k, v, do = (oracle.round_to(rng.standard_normal((1, 1, N, 64)), fmt) for _ in range(4))
    got = emulate_long_causal(q, k, v, do, fmt)
    ref, bound = attention_bounds(q, k, v, do, causal=True, round_qk=fmt, fmt=fmt, shift=kernel_shift(fmt, 8),
                                  chunk=512)
    worst = {}
    for n, g in zip(("o", "dq", "dk", "dv"), got):
        worst[n] = check_bound(n, g, ref, bound, fmt, c=C / 2) * C / 2
        EMULATION_WORST[f"{fmt}:{n}@32k"] = worst[n]
    with capsys.disabled():
        print(f"\n  emulation at causal 32768 x 64, {fmt}: worst err / (u M) "
              + "  ".join(f"{n} {w:.3f}" for n, w in worst.items()), end="")


EMULATION_WORST = {}


@pytest.mark.parametrize("fmt", ["bf16", "f16"])
@pytest.mark.parametrize("name", sorted(CASES) + ["long_causal"])
def test_emulated_rounding_within_bound(name, fmt):
    """The emulation stays within the bound with margin: its worst err / (u M) is at most C / 2."""
    if name == "long_causal":
        rng = np.random.default_rng(1)
        q, k, v, do = (oracle.round_to(rng.standard_normal((1, 1, 2048, 64)), fmt) for _ in range(4))
        kw = dict(causal=True)
    else:
        q, k, v, do, kw = make_case(name, fmt, seed=3)
    got = emulate(q, k, v, do, fmt, **kw)
    rq = fmt if kw.get("l2norm_qk", True) else None
    shift = kernel_shift(fmt, kw.get("scale", 8), kw.get("groups", 1), kw.get("l2norm_qk", True),
                         kw.get("attn_bias"))
    ref, bound = attention_bounds(q, k, v, do, round_qk=rq, fmt=fmt, shift=shift, chunk=512, **kw)
    for n, g in zip(("o", "dq", "dk", "dv", "d_bias"), got):
        w = check_bound(n, torch.from_numpy(g), ref, bound, fmt, c=C / 2) * C / 2
        EMULATION_WORST[f"{fmt}:{n}"] = max(EMULATION_WORST.get(f"{fmt}:{n}", 0.0), w)


# ---- the ends of the logit range (tests/logit_range.py): q^.k^ near +-groups, duplicate keys, zero rows -----------
# (groups, scale): fp16 only where p = exp(scale q.k - shift) fits its range; bf16 also at large scale * groups
LOGIT_RANGE_GS = {"bf16": [(1, 8), (1, 10), (2, 5), (8, 1), (4, 8), (1, 32), (2, 16)],
                  "f16": [(1, 8), (1, 10), (2, 5), (8, 1)]}
DTYPES = {"bf16": torch.bfloat16, "f16": torch.float16}


def _emulate_family(family, fmt, groups, scale, causal, seed, shape=(1, 4, 2, 300, 64)):
    B, H, Hk, N, D = shape
    q, k, v, do, _ = logit_range.dense(family, B, H, Hk, N, N, D, DTYPES[fmt], causal=causal, seed=seed)
    q, k, v, do = (t.double().numpy() for t in (q, k, v, do))
    kw = dict(groups=groups, scale=scale, causal=causal)
    with np.errstate(over="ignore"):                 # fp16 gradients of a zero row: x 1e12, out of range
        got = emulate(q, k, v, do, fmt, **kw)
    ref, bound = attention_bounds(q, k, v, do, round_qk=fmt, fmt=fmt, shift=kernel_shift(fmt, scale, groups), **kw)
    return got, ref, bound


@pytest.mark.parametrize("fmt,groups,scale", [(f, g, s) for f in LOGIT_RANGE_GS for g, s in LOGIT_RANGE_GS[f]])
@pytest.mark.parametrize("family", logit_range.FAMILIES)
def test_emulated_logit_range_within_bound(family, fmt, groups, scale):
    """Every input family at every (groups, scale) of its dtype, causal and not: the emulation stays within C / 2,
    the pin of the Gaussian cases.  fp16 gradients of the zero rows are out of range by construction (x 1e12)."""
    for causal in (False, True):
        got, ref, bound = _emulate_family(family, fmt, groups, scale, causal, seed=groups + scale + causal)
        names = ("o",) if (family == "zero_rows" and fmt == "f16") else ("o", "dq", "dk", "dv")
        for n, g in zip(names, got):
            w = check_bound(n, torch.from_numpy(g), ref, bound, fmt, c=C / 2) * C / 2
            EMULATION_WORST[f"{fmt}:{n}"] = max(EMULATION_WORST.get(f"{fmt}:{n}", 0.0), w)


def test_fp16_overflow_helper_matches_the_largest_p():
    """`_fp16_overflows` is exactly `exp(scale * groups - shift) > 65504` (the largest p, at q.k = groups) for fp16 with
    l2norm, and never true for bf16, float32 or without l2norm."""
    m = pytest.importorskip("flash_cosine_sim_attention_b200.flash_cosine_sim_attention")
    for groups in (1, 2, 3, 4, 8, 16, 32):
        for scale in (0.5, 1, 1.25, 2, 3, 4, 5, 6, 7, 8, 10, 11, 12, 16, 24, 32):
            shift = m._choose_shift(torch.float16, scale, groups, True)
            with np.errstate(over="ignore"):
                want = np.exp(np.float64(scale * groups - shift)) > 65504
            assert m._fp16_overflows(torch.float16, scale, groups, True) == want, (groups, scale)
            for dt, l2 in ((torch.bfloat16, True), (torch.float32, True), (torch.float16, False)):
                assert not m._fp16_overflows(dt, scale, groups, l2)
    for groups, scale, want in ((4, 8, True), (3, 8, True), (2, 16, True), (2, 8, False), (8, 1, False),
                                (1, 10, False), (1, 32, False)):
        assert m._fp16_overflows(torch.float16, scale, groups, True) == want, (groups, scale)


def test_emulated_fp16_overflow_breaks_the_bound(capsys):
    """Where `_fp16_overflows` warns, the kernels' arithmetic is wrong, not imprecise: at (1, 1, 256, 64), groups 4,
    scale 8, queries that are noisy copies of keys (sigma 0.3), every row's best p exceeds 65504 and the emulated o
    misses the bound by orders of magnitude; bf16 on the same input stays within C / 2."""
    out = {}
    for fmt in ("f16", "bf16"):
        got, ref, bound = _emulate_family("aligned0.3", fmt, 4, 8, False, seed=0, shape=(1, 1, 1, 256, 64))
        o = torch.from_numpy(got[0]).double()
        rel = float(((o - ref["o"]).norm(dim=-1) / ref["o"].norm(dim=-1)).max())
        worst = float(torch.nan_to_num(ratio(o, ref["o"], bound["o"], fmt), posinf=1e300).max()) / C
        out[fmt] = (rel, worst)
    assert out["f16"][1] > 10 and out["bf16"][1] <= 0.5, out
    with capsys.disabled():
        print(f"\n  emulated fp16 overflow (groups 4, scale 8, aligned0.3): o relative error {out['f16'][0]:.3g}, "
              f"worst err / (C u M) {out['f16'][1]:.3g}; bf16 {out['bf16'][1]:.3g}", end="")


# ---- context parallelism (context_parallel.py): key blocks, an additive merge, the backward per block --------------
def emulate_context_parallel(q, k, v, do, fmt, world, scale=8, groups=1, causal=False):
    """What the fused context-parallel path computes, in float32 with every 16-bit rounding in its place.  The sequence
    is cut into `world` blocks of queries and keys.  Query block r sees key blocks s <= r when causal (block r itself
    with the causal diagonal), all of them otherwise.  q^, k^ are stored in T (l2norm_tensors).  Per (r, s) the forward
    forms p = exp(scale S - shift) in fp32, the fp32 row sum l_s and o_s = (p~ V_s) / l_s, with p~ = p rounded to T (as
    in `emulate`) and o_s left in fp32 (out_f32).  The merge is o = sum_s o_s l_s / sum_s l_s in fp32, stored to T.  The
    backward per (r, s) uses the GLOBAL 1/l and the fp32 o (delta from it): P -> T before dV, dS -> T before dq^ and
    dk^.  dq^ is summed over the blocks in fp32, dk^ and dv over the query blocks in fp32 (the reduce-scatter), each
    rounded to T once; dq^ and dk^ then go through the separate l2norm backward, output -> T.
    q, k, v, do: (B, H, N, D) arrays of 16-bit values, N a multiple of `world`.  Returns [o, dq, dk, dv]."""
    f32 = np.float32
    T = lambda x: oracle.round_to(x, fmt).astype(f32)
    Tp = (lambda x: T(np.minimum(x, f32(65504)))) if fmt == "f16" else T
    shift = f32(kernel_shift(fmt, scale, groups))
    B, H, N, D = q.shape
    n = N // world
    (qn, nq), (kn, nk) = oracle.l2norm(q, groups), oracle.l2norm(k, groups)
    qn, kn = T(qn), T(kn)
    v, do = v.astype(f32), do.astype(f32)
    o, dqn, dkn, dv = (np.zeros(q.shape, f32) for _ in range(4))
    blk = [slice(r * n, (r + 1) * n) for r in range(world)]
    diag = np.tril(np.ones((n, n), bool))
    for b in range(B):
        for h in range(H):
            for r in range(world):
                qr, dor = qn[b, h, blk[r]], do[b, h, blk[r]]
                seen = [s for s in range(world) if not (causal and s > r)]
                p, num, den = {}, f32(0), f32(0)
                for s in seen:
                    vis = diag if (causal and s == r) else np.ones((n, n), bool)
                    p[s] = np.where(vis, np.exp(f32(scale) * (qr @ kn[b, h, blk[s]].T) - shift), f32(0))
                    inv_l_s = f32(1) / np.maximum(p[s].sum(-1, dtype=f32), f32(1e-37))
                    o_s = (Tp(p[s]) @ v[b, h, blk[s]]) * inv_l_s[:, None]
                    den_s = f32(1) / inv_l_s
                    num, den = num + o_s * den_s[:, None], den + den_s
                inv_l = f32(1) / den
                o_wide = num * inv_l[:, None]
                o[b, h, blk[r]] = o_wide
                delta = (dor * o_wide).sum(-1, dtype=f32, keepdims=True)
                for s in seen:
                    P = p[s] * inv_l[:, None]
                    dv[b, h, blk[s]] += T(P).T @ dor
                    ds = T(P * (dor @ v[b, h, blk[s]].T - delta))
                    dqn[b, h, blk[r]] += f32(scale) * (ds @ kn[b, h, blk[s]])
                    dkn[b, h, blk[s]] += f32(scale) * (ds.T @ qr)
    dq, dk = _l2bwd(T(dqn), qn, nq, groups), _l2bwd(T(dkn), kn, nk, groups)
    return [T(o), T(dq), T(dk), T(dv)]


# the (groups, scale) of the GPU grid (tests/test_gpu_context_parallel.py) at both ends: fp16 at (2, 8) is the
# shift = scale regime below the overflow threshold
CP_GS = {"bf16": [(1, 8), (4, 8), (2, 16)], "f16": [(1, 8), (2, 5), (2, 8)]}


@pytest.mark.parametrize("fmt,groups,scale", [(f, g, s) for f in CP_GS for g, s in CP_GS[f]])
@pytest.mark.parametrize("family", ["gaussian", "aligned0", "one_peak"])
def test_emulated_context_parallel_within_bound(family, fmt, groups, scale):
    """W = 3 blocks of 100 rows of (1, 2, 300, 64), causal and not: the context-parallel arrangement makes every 16-bit
    rounding of the dense kernels and otherwise fewer, plus one rounding of dq^ and dk^ before the l2norm backward (as
    on the BIAS path).  Its worst err / (u M) against the whole-sequence reference stays within C / 2, the pin of the
    dense emulation, so the GPU tests hold context parallelism to the same C."""
    for causal in (False, True):
        seed = groups + scale + causal
        if family == "gaussian":
            g = torch.Generator().manual_seed(seed)
            q, k, v, do = (torch.randn(1, 2, 300, 64, generator=g).to(DTYPES[fmt]) for _ in range(4))
        else:
            q, k, v, do, _ = logit_range.dense(family, 1, 2, 2, 300, 300, 64, DTYPES[fmt], causal=causal, seed=seed)
        q, k, v, do = (t.double().numpy() for t in (q, k, v, do))
        got = emulate_context_parallel(q, k, v, do, fmt, 3, scale=scale, groups=groups, causal=causal)
        ref, bound = attention_bounds(q, k, v, do, round_qk=fmt, fmt=fmt, shift=kernel_shift(fmt, scale, groups),
                                      groups=groups, scale=scale, causal=causal)
        for n, t in zip(("o", "dq", "dk", "dv"), got):
            w = check_bound(n, torch.from_numpy(t), ref, bound, fmt, c=C / 2) * C / 2
            EMULATION_WORST[f"{fmt}:cp {n}"] = max(EMULATION_WORST.get(f"{fmt}:cp {n}", 0.0), w)


# ---- planted errors: kernel-shaped mistakes, built from float64 results, that the bound must reject --------------
N = 2048


def rel_err(got, ref):
    return float(np.abs(got - ref).max() / np.abs(ref).max())


@pytest.fixture(scope="module")
def long_causal():
    """(1, 1, 2048, 64) bf16 causal: float64 reference and bound.  The same problem with a per-head bias gives
    d_bias ("biased")."""
    rng = np.random.default_rng(0)
    q, k, v, do = (oracle.round_to(rng.standard_normal((1, 1, N, 64)), "bf16") for _ in range(4))
    bias = oracle.round_to(rng.standard_normal((1, N, N)) * 0.5, "bf16")
    ref, bound = attention_bounds(q, k, v, do, causal=True, round_qk="bf16", fmt="bf16")
    bref, bbound = attention_bounds(q, k, v, do, causal=True, attn_bias=bias, round_qk="bf16", fmt="bf16")
    qn = oracle.round_to(oracle.l2norm(q)[0], "bf16")[0, 0]
    kn = oracle.round_to(oracle.l2norm(k)[0], "bf16")[0, 0]
    return dict(q=q, k=k, v=v, do=do, qn=qn, kn=kn, ref={n: t.numpy() for n, t in ref.items()}, tref=ref,
                bound=bound, biased=(bref, bbound))


def _rows(d, r0, r1, vis):
    """o and dS of query rows [r0, r1) of the long causal problem under a visibility of their own."""
    s = 8.0 * d["qn"][r0:r1] @ d["kn"].T
    s = np.where(vis, s, -np.inf)
    p = np.exp(s - s.max(-1, keepdims=True))
    p /= p.sum(-1, keepdims=True)
    v, do = d["v"][0, 0], d["do"][0, 0, r0:r1]
    o = p @ v
    ds = p * (do @ v.T - (do * o).sum(-1, keepdims=True))
    return o, ds


def _causal_vis(r0, r1, extra=0):
    return np.arange(N)[None, :] <= np.arange(r0, r1)[:, None] + extra


def _plant(d, what):
    ref = d["ref"]
    last_q, last_k = slice(N - 64, N), slice(N - 128, N)
    if what == "dv_last_key_tile_zero":
        g = ref["dv"].copy(); g[..., last_k, :] = 0
        return "dv", g
    if what == "dk_last_key_tile_x0.7":
        g = ref["dk"].copy(); g[..., last_k, :] *= 0.7
        return "dk", g
    if what == "dq_last_query_tile_x0.7":
        g = ref["dq"].copy(); g[..., last_q, :] *= 0.7
        return "dq", g
    if what == "o_last_query_tile_x0.7":
        g = ref["o"].copy(); g[..., last_q, :] *= 0.7
        return "o", g
    if what == "o_late_tile_without_key_tile_3":
        r0, r1 = N - 256, N - 128                      # forward query tile 14 drops keys 384..511
        vis = _causal_vis(r0, r1)
        vis[:, 384:512] = False
        g = ref["o"].copy(); g[0, 0, r0:r1] = _rows(d, r0, r1, vis)[0]
        return "o", g
    if what == "o_causal_diagonal_off_by_one":
        r0, r1 = N - 384, N - 256                      # forward query tile 13 sees one key past the diagonal
        g = ref["o"].copy(); g[0, 0, r0:r1] = _rows(d, r0, r1, _causal_vis(r0, r1, extra=1))[0]
        return "o", g
    if what == "dq_tile_missing_64_keys":
        r0, r1 = N - 128, N - 64                       # backward query tile 30 misses keys 1088..1151 (one half-tile)
        _, ds = _rows(d, r0, r1, _causal_vis(r0, r1))
        dqn = 8.0 * ds[:, 1088:1152] @ d["kn"][1088:1152]
        g = ref["dq"].copy()
        g[0, 0, r0:r1] -= oracle.l2norm_backward(dqn, d["q"][0, 0, r0:r1])
        return "dq", g
    if what == "d_bias_missing_query_tile":
        g = d["biased"][0]["d_bias"].numpy().copy(); g[0, N - 64:] = 0
        return "d_bias", g
    raise ValueError(what)


TOL = {"o": 1e-2, "dq": 2e-2, "dk": 2e-2, "dv": 2e-2, "d_bias": 2e-2}
PLANTS = ["dv_last_key_tile_zero", "dk_last_key_tile_x0.7", "dq_last_query_tile_x0.7", "o_last_query_tile_x0.7",
          "o_late_tile_without_key_tile_3", "o_causal_diagonal_off_by_one", "dq_tile_missing_64_keys",
          "d_bias_missing_query_tile"]


@pytest.mark.parametrize("what", PLANTS)
def test_planted_error_fails_the_bound(long_causal, what, capsys):
    name, got = _plant(long_causal, what)
    ref, bound = long_causal["biased"] if name == "d_bias" else (long_causal["tref"], long_causal["bound"])
    old = rel_err(got, ref[name].numpy())
    with pytest.raises(AssertionError, match="element-wise bound") as e:
        check_bound(name, torch.from_numpy(got), ref, bound, "bf16")
    with capsys.disabled():
        print(f"\n  planted {what}: rel_err {old:.3g} (tolerance {TOL[name]:g}: "
              f"{'passes' if old <= TOL[name] else 'fails'}); bound: {str(e.value).split(' at ')[0]}")


def test_bound_accepts_the_unplanted_reference(long_causal):
    for ref, bound in ((long_causal["tref"], long_causal["bound"]), long_causal["biased"]):
        for n, t in ref.items():
            assert check_bound(n, t, ref, bound, "bf16") == 0.0


def test_constants():
    assert U["bf16"] == 2.0 ** -8 and U["f16"] == 2.0 ** -11 and C == 2.0


def test_report_emulation_worst(capsys):
    """Prints the emulation's worst err / (u M) per format and quantity (what C is chosen from) when the emulation
    tests ran in the same session."""
    with capsys.disabled():
        for key in sorted(EMULATION_WORST):
            print(f"\n  emulation worst {key}: {EMULATION_WORST[key]:.3f} u M", end="")
