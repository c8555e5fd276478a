"""GPU tests at the tile edges of the kernels, judged by the element-wise bound (tests/elementwise_bounds.py) next to
the relative-to-max tolerances of test_gpu_parity.py:

* a sweep of sequence lengths around multiples of 64 that makes forward CTAs visit 1 to 7 key tiles (past both K/V
  rings) and backward CTAs visit 1 to 8 query tiles (past the 4- and 3-stage Q/dO rings, the D = 64 drain with
  either dQ owner), plus grouped-query loop-path CTAs whose flat (head, query tile) sequence restarts at every
  residue mod 2 and mod 3; the coverage is computed from the kernels' tile arithmetic (tests/tile_ranges.py) and
  asserted for each head dim's forward block;
* the BIAS instantiations past one ring, with d_bias;
* fp16 biases at the edges of the shifted exponent range;
* padding-suffix key masks, with whole masked key tiles;
* the float32 path past one ring."""
import pytest
import torch

from elementwise_bounds import C, U, attention_bounds, check_bound, kernel_shift
from gqa_reference import gqa_attention
from test_gpu_gqa import gqa_check, loop_batch, sm_count
from test_gpu_parity import (ROUND, TOL_GRAD, TOL_OUT, bound_check, check, fcsa, float32_operands,  # noqa: F401
                             make_inputs, record, rel_err)
from oracle import cosine_sim_attention_oracle as oracle
from tile_ranges import block_range, bwd_range, fwd_block_rows, group_split

gpu = pytest.mark.gpu        # every test here but the coverage check of the sweep needs the H100

KT = 128                  # key tile (forward and backward)


# ---- the tile counts of the kernels' work items -----------------------------------------------------------------
def fwd_key_tiles(Nq, Nk, causal, D):
    """Key tiles each forward CTA of head dim D visits (fcsa_fwd_kernel's NT)."""
    bm = fwd_block_rows(D)
    return [int(block_range(m0, bm, Nq, Nk, None, causal)[1][0]) for m0 in range(0, Nq, bm)]


def bwd_query_tiles(Nq, Nk, causal, hpc=1):
    """(NI, NT) of each backward CTA (one 128-key tile, hpc query heads): fcsa_bwd_kernel's NI / NT."""
    out = []
    for key0 in range(0, Nk, KT):
        i_lo, i_end = bwd_range(key0, Nq, Nk, None, causal)
        ni = max(0, int(i_end[0] - i_lo[0]))
        out.append((ni, hpc * ni))
    return out


def head_restarts(ni, hpc):
    """Flat tile indices i at which row0 restarts with the next query head."""
    return [hh * ni for hh in range(1, hpc)]


SWEEP = [  # (Nq, Nk, causal): lengths at 64k - 1, 64k and 64k + 1
    (767, 767, True), (384, 512, True), (513, 385, True), (511, 769, False), (65, 640, False)]
GQA_LOOP = [(ni, hpc) for hpc in (2, 3) for ni in (1, 2, 3)]      # Nq = 64 ni - 1 + (ni > 1): NI query tiles


def gqa_nq(ni):
    return 63 if ni == 1 else 64 * (ni - 1) + 1


def test_sweep_covers_every_tile_count():
    for D in (64, 128):                                      # 1 .. 6 key tiles: past the 4- and 2-stage rings
        fwd = {nt for nq, nk, c in SWEEP for nt in fwd_key_tiles(nq, nk, c, D)}
        assert set(range(1, 7)) <= fwd, (D, fwd)
    bwd = {nt for nq, nk, c in SWEEP for _, nt in bwd_query_tiles(nq, nk, c)}
    assert set(range(1, 9)) <= bwd, bwd                      # NT = 1 .. 8, both dQ owners of the last tile
    gqa = [bwd_query_tiles(gqa_nq(ni), 256, False, hpc) for ni, hpc in GQA_LOOP]
    assert all(len({ni_ for ni_, _ in t}) == 1 for t in gqa)
    assert {t[0][0] for t in gqa} == {1, 2, 3}
    restarts = [i for ni, hpc in GQA_LOOP for i in head_restarts(ni, hpc)]
    assert {i % 2 for i in restarts} == {0, 1} and {i % 3 for i in restarts} == {0, 1, 2}, restarts


@gpu
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("dim_head", [64, 128])
@pytest.mark.parametrize("nq,nk,causal", SWEEP)
def test_tile_count_sweep(fcsa, nq, nk, causal, dim_head, dtype):
    check(fcsa, (1, 2, nq, dim_head), (1, 2, nk, dim_head), dtype, seed=nq + nk + dim_head, causal=causal)


@gpu
@pytest.mark.parametrize("dim_head", [64, 128])
@pytest.mark.parametrize("ni,hpc", GQA_LOOP)
def test_gqa_loop_head_restarts(fcsa, ni, hpc, dim_head):
    """Loop-path CTAs with hpc = 2 or 3 query heads of NI = 1, 2, 3 tiles each: row0 restarts at flat tile
    indices of every residue mod 2 and mod 3, and the dQ owner parity of each head's first tile varies."""
    Hk, Nk = 2, 256
    B = loop_batch(Hk, Nk)
    assert group_split(B, Hk * hpc, Hk, Nk, sm_count()) == 1
    gqa_check(fcsa, (B, Hk * hpc, gqa_nq(ni), dim_head), (B, Hk, Nk, dim_head), torch.bfloat16, seed=ni + 7 * hpc,
              path="loop")


# ---- BIAS past one ring ----------------------------------------------------------------------------------------
def bias_check(fcsa, qs, kvs, dtype, seed, bias_kind, causal=False, mask_p=None, bias=None):
    q, k, v, do, m = make_inputs(qs, kvs, dtype, seed=seed, mask_p=mask_p)
    B, H, Nq = qs[0], qs[1], qs[2]
    Nk = kvs[-2]
    if bias is None:
        g = torch.Generator().manual_seed(seed + 1)
        bias = torch.randn((B if bias_kind == "batch" else H, Nq, Nk), generator=g).to(dtype)
    qd, kd, vd, bd = (t.cuda().requires_grad_() for t in (q, k, v, bias))
    o = fcsa.flash_cosine_sim_attention(qd, kd, vd, mask=None if m is None else m.cuda(), attn_bias=bd, causal=causal,
                                        attn_bias_batch_dim=bias_kind == "batch")
    o.backward(do.cuda())
    kw = dict(mask=m, attn_bias=bias, causal=causal, attn_bias_batch_dim=bias_kind == "batch")
    grouped = len(kvs) == 4 and kvs[1] != H
    f = gqa_attention if grouped else oracle.attention
    ref = f(q.float().numpy(), k.float().numpy(), v.float().numpy(), mask=None if m is None else m.numpy(),
            attn_bias=bias.float().numpy(), causal=causal, attn_bias_batch_dim=bias_kind == "batch",
            d_out=do.float().numpy(), empty_rows="zero", round_qk=ROUND[dtype])
    for name, t, r in (("o", o, ref[0]), ("dq", qd.grad, ref[1]), ("dk", kd.grad, ref[2]), ("dv", vd.grad, ref[3]),
                       ("d_bias", bd.grad, ref[4])):
        assert t.shape == (q.shape if name in ("o", "dq") else (bias.shape if name == "d_bias" else k.shape))
        e = rel_err(t, r)
        tol = TOL_OUT[dtype] if name == "o" else TOL_GRAD[dtype]
        record(dtype, name, e, tol)
        assert e <= tol, name
    return bound_check(dtype, {"o": o, "dq": qd.grad, "dk": kd.grad, "dv": vd.grad, "d_bias": bd.grad},
                       q, k, v, do, **kw)


@gpu
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("dim_head", [64, 128])
@pytest.mark.parametrize("bias_kind", ["heads", "batch"])
@pytest.mark.parametrize("masking", ["causal", "mask", "none"])
def test_bias_past_one_ring(fcsa, masking, bias_kind, dim_head, dtype):
    """(2, 3, 600, 700) and causal (2, 3, 640, 640): the forward visits 5 - 6 key tiles, the backward 9 - 10 query
    tiles per CTA (D = 64: the DS_EMPTY wait and the wrap of the Q/dO ring with a bias); d_bias on 600 x 700 planes."""
    n = (640, 640) if masking == "causal" else (600, 700)
    bias_check(fcsa, (2, 3, n[0], dim_head), (2, 3, n[1], dim_head), dtype, seed=dim_head + len(masking),
               bias_kind=bias_kind, causal=masking == "causal", mask_p=0.3 if masking == "mask" else None)


@gpu
@pytest.mark.parametrize("kv", ["gqa", "mqa"])
def test_bias_past_one_ring_grouped(fcsa, kv):
    kvs = (2, 3, 700, 64) if kv == "gqa" else (2, 700, 64)
    bias_check(fcsa, (2, 6, 600, 64), kvs, torch.bfloat16, seed=5, bias_kind="heads", mask_p=0.3)


# ---- fp16 bias range -------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("causal", [False, True])
def test_fp16_bias_with_large_entries(fcsa, causal):
    """A few bias entries at +10: the bias maximum added to the shift is all that keeps p = exp(logit - shift) below
    fp16's largest value; the other rows lose that much range.  Forward and backward within the bound."""
    H, N = 2, 520
    g = torch.Generator().manual_seed(61)
    bias = torch.randn(H, N, N, generator=g)
    idx = torch.randint(0, N, (2, 16), generator=g)
    bias[:, idx[0], idx[1]] = 10.0
    bias_check(fcsa, (1, H, N, 64), (1, H, N, 64), torch.float16, seed=61, bias_kind="heads", causal=causal,
               bias=bias.half())


@gpu
@pytest.mark.parametrize("slope", [0.25, 1.0])
def test_fp16_bias_alibi_like(fcsa, slope):
    """A distance bias -slope |i - j| (ALiBi-like): far keys get p deep in fp16's subnormals or 0."""
    H, N = 2, 640
    i = torch.arange(N)
    bias = (-slope * (i[:, None] - i[None, :]).abs().float() * torch.tensor([1.0, 0.5])[:, None, None]).half()
    bias_check(fcsa, (1, H, N, 64), (1, H, N, 64), torch.float16, seed=62, bias_kind="heads", causal=True,
               bias=bias)


# ---- padding-suffix key masks ---------------------------------------------------------------------------------
LENGTHS = (1, 63, 64, 65, 127, 128, 129, 255, 256, 257, 700)


@gpu
@pytest.mark.parametrize("dim_head", [64, 128])
@pytest.mark.parametrize("kv", ["mha", "mqa", "gqa"])
def test_padding_suffix_masks(fcsa, kv, dim_head, capsys):
    """Key-padding masks as a batch of sequences of lengths LENGTHS padded to Nk = 700: whole masked key tiles, and
    backward CTAs whose keys are all masked.  dk, dv of every masked key are exactly 0; o, dq are within the bound
    against the float64 reference and against the same call on k, v truncated to each length."""
    B, H, Nq, Nk, dt = len(LENGTHS), 4, 257, 700, torch.bfloat16
    kvs = {"mha": (B, H, Nk, dim_head), "mqa": (B, Nk, dim_head), "gqa": (B, 2, Nk, dim_head)}[kv]
    q, k, v, do, _ = make_inputs((B, H, Nq, dim_head), kvs, dt, seed=dim_head + len(kv))
    mask = torch.arange(Nk)[None, :] < torch.tensor(LENGTHS)[:, None]
    qd, kd, vd = (t.cuda().requires_grad_() for t in (q, k, v))
    o = fcsa.flash_cosine_sim_attention(qd, kd, vd, mask=mask.cuda())
    o.backward(do.cuda())
    ok, dk, dv = o.detach(), kd.grad, vd.grad
    for b, n in enumerate(LENGTHS):
        assert torch.all(dk[b, ..., n:, :] == 0) and torch.all(dv[b, ..., n:, :] == 0), (b, n)
    bound_check(dt, {"o": o, "dq": qd.grad, "dk": dk, "dv": dv}, q, k, v, do, mask=mask)
    ref, bound = attention_bounds(q, k, v, do, mask=mask, round_qk="bf16", fmt="bf16", shift=kernel_shift("bf16", 8),
                                  device="cuda")
    bitwise = []
    for b, n in enumerate(LENGTHS):
        sl = lambda t: t[b:b + 1, ..., :n, :].cuda().requires_grad_()
        qb = q[b:b + 1].cuda().requires_grad_()
        kb, vb = sl(k), sl(v)
        ob = fcsa.flash_cosine_sim_attention(qb, kb, vb)
        ob.backward(do[b:b + 1].cuda())
        one = lambda x: {n_: t[b:b + 1] for n_, t in x.items()}
        for name, full, trunc in (("o", ok[b:b + 1], ob), ("dq", qd.grad[b:b + 1], qb.grad)):
            w = check_bound(name, trunc, one(ref), one(bound), "bf16")       # the truncated call against the oracle
            # and the padded call against the truncated one, at the same scale
            d = (full.double() - trunc.double()).abs()
            lim = C * U["bf16"] * bound[name][b:b + 1]
            assert torch.all(d <= lim), (name, n, float((d / lim).max()))
            record(dt, f"{name}/bound", w, 1.0)
        bitwise.append(torch.equal(ok[b:b + 1], ob) and torch.equal(qd.grad[b:b + 1], qb.grad))
    with capsys.disabled():
        print(f"\n  padding suffix {kv} D={dim_head}: o, dq bitwise equal to the truncated call for lengths "
              f"{[n for n, e in zip(LENGTHS, bitwise) if e]} of {list(LENGTHS)}", end="")


# ---- float32 past one ring -------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("n,dim_head", [(1100, 64), (600, 128)])
def test_float32_past_one_ring(fcsa, n, dim_head, causal):
    """check() applies both float32 checks: 1e-3 / 2e-3 against the unrounded oracle, and the element-wise bound
    against the oracle on the operands the fp16 kernels see."""
    check(fcsa, (1, 2, n, dim_head), (1, 2, n, dim_head), torch.float32, seed=n + dim_head, causal=causal)


@gpu
def test_float32_bias_past_one_ring(fcsa):
    g = torch.Generator().manual_seed(71)
    q, k, v, do = (torch.randn(1, 2, 700, 64, generator=g) for _ in range(4))
    bias = torch.randn(2, 700, 700, generator=g)
    qd, kd, vd, bd = (t.cuda().requires_grad_() for t in (q, k, v, bias))
    o = fcsa.flash_cosine_sim_attention(qd, kd, vd, attn_bias=bd, causal=True, scale=4, groups=2)
    o.backward(do.cuda())
    ref = oracle.attention(q.numpy(), k.numpy(), v.numpy(), attn_bias=bias.numpy(), causal=True, scale=4, groups=2,
                           d_out=do.numpy())
    for name, t, r, tol in (("o", o, ref[0], 1e-3), ("dq", qd.grad, ref[1], 2e-3), ("dk", kd.grad, ref[2], 2e-3),
                            ("dv", vd.grad, ref[3], 2e-3), ("d_bias", bd.grad, ref[4], 2e-3)):
        e = rel_err(t, r)
        record(torch.float32, name, e, tol)
        assert e <= tol, name
    bound_check(torch.float32, {"o": o, "dq": qd.grad, "dk": kd.grad, "dv": vd.grad, "d_bias": bd.grad}, q, k, v, do,
                attn_bias=bias, causal=True, scale=4, groups=2)
