"""GPU: every kernel instantiation of libfcsa_b200.so runs inside a call whose outputs are judged against the float64
reference.

Each row below is one small judged call (or a few) through the public API, with the helpers of the deeper tests:
`wcheck` (window or not, float32, the backward's split rule by launch count), `repeated` + `bounded` (the
deterministic route), `run_varlen` / `varlen_repeated` + `seq_check` (packed sequences), `check_case` (decode), and
`run_dense` + `judge` (a bias).  Each row states, as data, the kernels it launches (tests/kernel_census.py names them
from their template arguments); torch.profiler records the kernels that ran, and the row asserts that exact set, so
the host dispatch is checked too: fp16 with a window must reach the WINDOW = true kernel, and so on.  A row whose
outputs pass adds its kernels to the census.

The last test compares the union of the rows' kernels with the library's list (read from the ELF file) and names every
kernel that no row judged.  It runs after the rows of this module and skips when some of them did not run."""
import math

import pytest
import torch

import kernel_census as kc
from kernel_census import (VARLEN_TAIL, bwd, combine, decode, dq, dq_finish, fwd, kv_finish, prep, row_bwd, row_fwd)
from test_gpu_decode import check_case, n_split_of
from test_gpu_deterministic import bounded, make, repeated, varlen_repeated
from test_gpu_gqa import loop_batch, sm_count
from test_gpu_long_context import inputs, judge, run_dense
from oracle import cosine_sim_attention_oracle as oracle
from test_gpu_parity import TOL_GRAD, TOL_OUT, bound_check, fcsa, make_inputs, rel_err  # noqa: F401  (fcsa: a fixture)
from test_gpu_row_passes import _l2norm_round_trip
from test_gpu_varlen import cu_of, make_packed, run_varlen, seq_check
from test_gpu_window import wcheck
from tile_ranges import group_split
from window_bounds import window_attention_bounds

pytestmark = pytest.mark.gpu

BF16, F16, F32 = torch.bfloat16, torch.float16, torch.float32
TD = [(t, D) for t in (BF16, F16) for D in (64, 128)]
NAME = {BF16: "bf16", F16: "f16"}

ROWS = []            # (id, fn(fcsa), expected kernels)


def row(rid, expected):
    def add(fn):
        ROWS.append((rid, fn, frozenset(expected)))
        return fn
    return add


# ---- per dtype and head dim: every attention kernel ------------------------------------------------------------------
def _attention_rows(t, D):
    p = f"{NAME[t]}-D{D}"
    fw = {row_fwd(t, D), fwd(t, D)}                                   # l2norm(q, k) + the forward
    fw_w = {row_fwd(t, D), fwd(t, D, window=True)}
    vfw = {row_fwd(t, D), fwd(t, D, varlen=True), VARLEN_TAIL}
    vfw_w = {row_fwd(t, D), fwd(t, D, varlen=True, window=True), VARLEN_TAIL}

    def back(varlen=False, **k):                                      # the default backward
        return {prep(t, D, varlen), bwd(t, D, varlen=varlen, **k), dq_finish(t, D, varlen)} | (
            {VARLEN_TAIL} if varlen else set())

    def det(varlen=False, window=False, head_loop=False):             # the deterministic backward
        return {prep(t, D, varlen), bwd(t, D, head_loop, varlen, window, dq=False), dq(t, D, varlen, window)} | (
            {VARLEN_TAIL} if varlen else set())

    # -- dense, default backward
    @row(f"{p}-mha", fw | back())
    def _(fcsa):
        wcheck(fcsa, (1, 2, 300, D), (1, 2, 300, D), t, None, seed=1, causal=True)

    @row(f"{p}-mha-window", fw_w | back(window=True))
    def _(fcsa):
        wcheck(fcsa, (1, 2, 300, D), (1, 2, 300, D), t, 65, seed=2)

    @row(f"{p}-gqa-loop", fw | back(head_loop=True))
    def _(fcsa):
        B = loop_batch(2, 300)
        wcheck(fcsa, (B, 4, 300, D), (B, 2, 300, D), t, None, seed=3, path="loop", causal=True)

    @row(f"{p}-gqa-loop-window", fw_w | back(head_loop=True, window=True))
    def _(fcsa):
        B = loop_batch(2, 300)
        wcheck(fcsa, (B, 4, 300, D), (B, 2, 300, D), t, 129, seed=4, path="loop", causal=True)

    @row(f"{p}-mqa-split", fw | back() | {kv_finish(t), row_bwd(t)})
    def _(fcsa):
        # keys shared by all heads: dk / dv summed over CTAs, then converted, then the l2norm backward of dk
        wcheck(fcsa, (2, 4, 300, D), (2, 300, D), t, None, seed=5, causal=True)

    @row(f"{p}-bias", {row_fwd(t, D), row_bwd(t), fwd(t, D, bias=True), prep(t, D), bwd(t, D, bias=True),
                       dq_finish(t, D)})
    def _(fcsa):
        q, k, v, do = inputs((1, 2, 150, D), (1, 2, 203, D), t, seed=6)
        bias = torch.randn(2, 150, 203, generator=torch.Generator(device="cuda").manual_seed(7), device="cuda").to(t)
        got = run_dense(fcsa, q, k, v, do, t, attn_bias=bias)
        judge(t, got, q, k, v, do, attn_bias=bias)

    # -- dense, deterministic backward
    for heads, kv_heads in ((4, 4), (4, 2)):
        for window in (None, 65):
            kind = ("mha" if heads == kv_heads else "gqa") + ("-window" if window else "")

            @row(f"{p}-det-{kind}", (fw_w if window else fw) | det(False, window is not None, heads != kv_heads))
            def _(fcsa, heads=heads, kv_heads=kv_heads, window=window):
                q, k, v, do = make(1, heads, kv_heads, 300, 300, D, t, seed=8 + kv_heads)
                kw = dict(causal=True) if window is None else dict(causal=False, window=window)
                got, _ = repeated(fcsa, q, k, v, do, **kw)
                bounded(t, got, q, k, v, do, **kw)

    # -- packed sequences, default backward
    for kind, heads, kv_heads, window in (("mha", 4, 4, None), ("mha-window", 4, 4, 65), ("gqa-loop", 8, 4, None),
                                          ("gqa-loop-window", 8, 4, 129)):
        hl = heads != kv_heads

        @row(f"{p}-varlen-{kind}", (vfw_w if window else vfw) | back(True, head_loop=hl, window=window is not None))
        def _(fcsa, heads=heads, kv_heads=kv_heads, window=window):
            # the loop rows: enough key tiles x sequences x kv heads that the groups stay in one CTA
            ls = [700, 65, 1, 300, 129, 0] if heads != kv_heads else [300, 0, 1, 65, 129]
            if heads != kv_heads:
                assert group_split(len(ls), heads, kv_heads, max(ls), sm_count()) == 1
            q, k, v, do = make_packed(ls, ls, heads, kv_heads, D, t, seed=10 + kv_heads)
            kw = dict(causal=True) if window is None else dict(causal=window > 100, window=window)
            *got, _ = run_varlen(fcsa, q, k, v, do, cu_of(ls), cu_of(ls), max(ls), max(ls), **kw)
            seq_check(t, got, q, k, v, do, ls, ls, **kw)

    # -- packed sequences, deterministic backward
    for heads, kv_heads in ((4, 4), (4, 2)):
        for window in (None, 65):
            kind = ("mha" if heads == kv_heads else "gqa") + ("-window" if window else "")

            @row(f"{p}-varlen-det-{kind}", (vfw_w if window else vfw) | det(True, window is not None, heads != kv_heads))
            def _(fcsa, heads=heads, kv_heads=kv_heads, window=window):
                ls = [300, 0, 1, 65, 129]
                q, k, v, do = make_packed(ls, ls, heads, kv_heads, D, t, seed=12 + kv_heads)
                kw = dict(causal=True) if window is None else dict(causal=False, window=window)
                *got, _ = varlen_repeated(fcsa, q, k, v, do, cu_of(ls), max(ls), **kw)
                seq_check(t, got, q, k, v, do, ls, ls, **kw)

    # -- decode (check_case normalises q and the new keys with l2norm_tensors for its reference: the 16-bit l2norm)
    dec = {row_fwd(t, D), row_fwd(t, D, append=True)}

    @row(f"{p}-decode-split", dec | {decode(t, D), combine(t, D)})
    def _(fcsa):
        assert n_split_of(4, 8, 2, 1, 1024) > 1
        check_case(fcsa, t, D, 8, 2, 1, [0, 131, 383, 1023], 1024, 1, seed=14, launches=3)

    @row(f"{p}-decode-window-split", dec | {decode(t, D, window=True), combine(t, D)})
    def _(fcsa):
        assert n_split_of(6, 8, 2, 3, 640, 65) > 1
        check_case(fcsa, t, D, 8, 2, 3, [0, 61, 62, 63, 300, 637], 640, 3, seed=15, launches=3, window=65)

    @row(f"{p}-decode-window-one", dec | {decode(t, D, window=True)})
    def _(fcsa):
        B = math.ceil(sm_count() / 8)
        assert n_split_of(B, 8, 8, 1, 1024, 200) == 1
        check_case(fcsa, t, D, 8, 8, 1, [(198 + 37 * b) % 1023 for b in range(B)], 1024, 1, seed=16, launches=2,
                   window=200)


for _t, _D in TD:
    _attention_rows(_t, _D)


# ---- float32 inputs: the cast passes (fp16 kernels, or bf16 ones past fp16's range) ------------------------------------
def _f32_row(half, D, **kw):
    Dk = 64 if D < 64 else D                    # the kernels' head dim (zero-padded features)
    # the backward of the l2norm cast reads the 16-bit q^, k^ (row_bwd<half, float>); the plain scaled cast's backward
    # (dv, and q, k without l2norm) reads no 16-bit tensor and runs row_bwd<__half, float> whatever the kernels' type
    expected = {row_fwd(half, D, x=F32), row_bwd(F16, F32), fwd(half, Dk), prep(half, Dk), bwd(half, Dk),
                dq_finish(half, Dk)}
    if kw.get("l2norm_qk", True):
        expected.add(row_bwd(half, F32))

    @row(f"f32-{NAME[half]}-D{D}", expected)
    def _(fcsa):
        if half == F16:
            wcheck(fcsa, (1, 2, 270, D), (1, 2, 270, D), F32, None, seed=D, causal=True, **kw)
            return
        # on the bf16 kernels the relative tolerances are bf16's; the element-wise bound models the bf16 operands
        # without the l2norm q.k is unbounded: small inputs, as test_gpu_parity.py's test_no_l2norm
        amp = 1.0 if kw.get("l2norm_qk", True) else 0.2
        q, k, v, do, _ = make_inputs((1, 2, 270, D), (1, 2, 270, D), F32, seed=D, amp=amp)
        qd, kd, vd = (x.cuda().requires_grad_() for x in (q, k, v))
        o = fcsa.flash_cosine_sim_attention(qd, kd, vd, causal=True, **kw)
        o.backward(do.cuda())
        got = {"o": o, "dq": qd.grad, "dk": kd.grad, "dv": vd.grad}
        assert all(x.dtype == F32 for x in got.values())
        bound_check(F32, got, q, k, v, do, causal=True, **kw)
        ref = oracle.attention(*(x.double().numpy() for x in (q, k, v)), causal=True, d_out=do.double().numpy(), **kw)
        for name, r in zip(("o", "dq", "dk", "dv"), ref):
            assert rel_err(got[name], r) <= (TOL_OUT if name == "o" else TOL_GRAD)[BF16], name


_f32_row(F16, 32)
_f32_row(F16, 64)
_f32_row(F16, 128)
_f32_row(BF16, 32, groups=2)                    # scale * groups > 10: the bf16 kernels
_f32_row(BF16, 64, l2norm_qk=False, scale=1)    # no l2norm: the bf16 kernels, no rnorm pointer
_f32_row(BF16, 128, groups=2)


# ---- runtime branches inside the kernels above ------------------------------------------------------------------------
@row("f32-window-det", {row_fwd(F16, 64, x=F32), row_bwd(F16, F32), fwd(F16, 64, window=True), prep(F16, 64),
                        bwd(F16, 64, head_loop=True, window=True, dq=False), dq(F16, 64, window=True)})
def _(fcsa):
    """float32 outputs (out_f32) of the dK / dV and dQ kernels with a window"""
    q, k, v, do = make(1, 4, 2, 300, 300, 64, F32, seed=20)
    got, _ = repeated(fcsa, q, k, v, do, causal=True, window=65)
    judge(F32, {n: x.cuda() for n, x in got.items()}, *(x.cuda() for x in (q, k, v, do)),
          bounds=window_attention_bounds, causal=True, window=65)


@row("f16-D128-det-mask-window", {row_fwd(F16, 128), fwd(F16, 128, window=True), prep(F16, 128),
                                  bwd(F16, 128, head_loop=True, window=True, dq=False), dq(F16, 128, window=True)})
def _(fcsa):
    """a key-padding mask together with a window in the dQ kernel"""
    q, k, v, do = make(2, 4, 2, 300, 700, 128, F16, seed=21)
    mask = torch.rand(2, 700, generator=torch.Generator().manual_seed(22)) > 0.3
    got, _ = repeated(fcsa, q, k, v, do, mask=mask.cuda(), window=129)
    bounded(F16, got, q, k, v, do, mask=mask, window=129)


@row("bf16-D64-det-no-l2norm", {fwd(BF16, 64), prep(BF16, 64), bwd(BF16, 64, dq=False), dq(BF16, 64)})
def _(fcsa):
    """l2norm_qk=False: no row pass and no rnorm pointer in the dQ kernel"""
    q, k, v, do = make(1, 4, 4, 300, 300, 64, BF16, seed=23)
    got, _ = repeated(fcsa, q, k, v, do, causal=True, l2norm_qk=False, scale=1)
    bounded(BF16, got, q, k, v, do, causal=True, l2norm_qk=False, scale=1)


# ---- the 16-bit l2norm at head dims other than 64 and 128 -------------------------------------------------------------
for _t in (BF16, F16):
    @row(f"l2norm-{NAME[_t]}-D32", {row_fwd(_t, 32), row_bwd(_t)})
    def _(fcsa, t=_t):
        g = torch.Generator().manual_seed(24)
        x, dy = (torch.randn(2, 3, 77, 32, generator=g).to(t) for _ in range(2))
        _l2norm_round_trip(fcsa, x, dy, 2)


# ---- the rows, then the census ------------------------------------------------------------------------------------------
JUDGED = {}          # row id -> kernels it ran, for the rows whose outputs passed
RAN = set()          # row ids that ran


@pytest.mark.parametrize("rid,fn,expected", ROWS, ids=[r[0] for r in ROWS])
def test_row(fcsa, rid, fn, expected):
    RAN.add(rid)
    _, ran = kc.launched_kernels(lambda: fn(fcsa))
    assert ran, "the profiler saw no fcsa kernel: the census cannot count this row"
    assert ran == expected, f"missing {sorted(expected - ran)}, unexpected {sorted(ran - expected)}"
    JUDGED[rid] = ran


def test_every_kernel_is_judged():
    from flash_cosine_sim_attention_b200 import _abi
    skipped = [r[0] for r in ROWS if r[0] not in RAN]
    if skipped:
        pytest.skip(f"{len(skipped)} of {len(ROWS)} census rows did not run in this session (deselected): "
                    f"{skipped[:5]}{' ...' if len(skipped) > 5 else ''}")
    library = set(kc.library_kernels(_abi.LIB_PATH))
    judged = set().union(*JUDGED.values()) if JUDGED else set()
    failed = [r[0] for r in ROWS if r[0] not in JUDGED]
    missing = sorted(library - judged)
    print(f"\nkernel census: {len(library & judged)} of {len(library)} kernels judged")
    assert not missing, (f"{len(missing)} of {len(library)} kernels ran in no judged call"
                         f"{f' (failed rows: {failed})' if failed else ''}:\n  " + "\n  ".join(missing))
    assert judged <= library, sorted(judged - library)
