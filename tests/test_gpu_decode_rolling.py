"""GPU tests of flash_cosine_sim_attention_with_kv_cache(..., rolling=True): rolling key/value caches for
sliding-window decoding, rings of C rows where absolute position p lives at row p mod C.

Every call is checked three ways against a full-length host copy of the keys (a cache of the same keys at their
absolute rows, the sentinel NaN past each element's length):
  * o against the float64 windowed reference over the absolute sequence (tests/window_bounds.py), with the relative
    tolerance of test_gpu_parity.py and the element-wise bound;
  * o bitwise against the same call on the full-length cache whenever both use the same number of key splits (the
    kernel reads the same tiles in the same order; rows outside the window get P = 0 exactly);
  * the ring after the call bitwise against the last C positions of the full-length cache after its append, and the
    sentinel in every ring row that never held a position.
Rings start as the sentinel, so a ring row never written that leaked into P V would show up as a NaN."""
import math

import pytest
import torch

from elementwise_bounds import FMT, check_bound, kernel_shift
from kernel_census import VARLEN_TAIL, combine, decode, library_kernels, row_fwd
from test_gpu_decode import SENTINEL, make_cache, n_split_of, sm_count
from test_gpu_decode_varlen import make_pack, packed_split
from test_gpu_parity import TOL_OUT, fcsa, record, rel_err  # noqa: F401
from window_bounds import window_attention_bounds

pytestmark = pytest.mark.gpu


def ring_of(full, C, T):
    """The ring of C rows a rolling cache holds once positions [0, T) of `full` (one batch element, (1, Hk, N, D))
    have been appended: positions [max(0, T - C), T) at rows p mod C, the sentinel in the rows never written."""
    ring = torch.empty(*full.shape[:2], C, full.shape[3], dtype=full.dtype, device=full.device)
    ring.view(torch.int16).fill_(SENTINEL)
    p = torch.arange(max(0, T - C), T, device=full.device)
    ring[:, :, p % C] = full[:, :, p]
    return ring


def rings_of(full, C, lens):
    return torch.cat([ring_of(full[b:b + 1], C, L) for b, L in enumerate(lens)]).contiguous()


def bitwise(a, b):
    return torch.equal(a.view(torch.int16), b.view(torch.int16))


def check_o(dtype, o_b, qh_b, kf_b, vf_b, T, W, scale, causal, groups, l2norm_qk, what):
    """o of one batch element ((1, H, n, D)) against the windowed float64 reference over keys [0, T)."""
    if T == 0:
        assert int(o_b.count_nonzero()) == 0
        return
    fmt = FMT[dtype]
    shift = kernel_shift(fmt, scale, groups, l2norm_qk)
    ref, bound = window_attention_bounds(qh_b, kf_b[:, :, :T], vf_b[:, :, :T], window=W, scale=scale, causal=causal,
                                         l2norm_qk=False, fmt=fmt, shift=shift, device="cuda")
    r = ref["o"].cpu().numpy()
    e = rel_err(o_b, r) if abs(r).max() > 0 else float(o_b.abs().max())
    record(dtype, what, e, TOL_OUT[dtype])
    assert e <= TOL_OUT[dtype], f"{what}: T = {T}"
    record(dtype, what + "/bound", check_bound("o", o_b, ref, bound, fmt), 1.0)


def _setup(dtype, l2norm_qk, groups):
    amp = 1.0 if l2norm_qk else 0.15
    scale = 1 if (not l2norm_qk or groups > 1) else 8
    return amp, scale


def run_dense(fcsa, dtype, D, H, Hk, Nq, lens, C, W, causal=True, groups=1, l2norm_qk=True, append=True, seed=0):
    """One dense rolling call on rings holding L_b = lens[b] positions, checked as the module docstring says."""
    from flash_cosine_sim_attention_b200 import l2norm_tensors
    B = len(lens)
    g = torch.Generator().manual_seed(seed)
    amp, scale = _setup(dtype, l2norm_qk, groups)
    n = Nq if append else 0
    cap = max(lens) + Nq
    q = (torch.randn(B, H, Nq, D, generator=g) * amp).to(dtype).cuda()
    kf, vf = make_cache(B, Hk, cap, D, dtype, lens, g, l2norm_qk, groups, amp)
    kr, vr = rings_of(kf, C, lens), rings_of(vf, C, lens)
    k = v = None
    if append:
        k = (torch.randn(B, Hk, Nq, D, generator=g) * amp).to(dtype).cuda()
        v = torch.randn(B, Hk, Nq, D, generator=g).to(dtype).cuda()
    sl = torch.tensor(lens, dtype=torch.int32, device="cuda")
    kw = dict(scale=scale, groups=groups, causal=causal, l2norm_qk=l2norm_qk, window=W)
    with torch.no_grad():
        o = fcsa.flash_cosine_sim_attention_with_kv_cache(q, kr, vr, sl, k, v, rolling=True, **kw)
        o_full = fcsa.flash_cosine_sim_attention_with_kv_cache(q, kf, vf, sl, k, v, **kw)
    torch.cuda.synchronize()
    assert sl.tolist() == list(lens)
    assert torch.isfinite(o.float()).all()
    for b, L in enumerate(lens):
        assert bitwise(kr[b:b + 1], ring_of(kf[b:b + 1], C, L + n)), f"k ring {b}"
        assert bitwise(vr[b:b + 1], ring_of(vf[b:b + 1], C, L + n)), f"v ring {b}"
    qh = l2norm_tensors(q, groups=groups)[0] if l2norm_qk else q
    for b, L in enumerate(lens):
        check_o(dtype, o[b:b + 1], qh[b:b + 1], kf[b:b + 1], vf[b:b + 1], L + n, W, scale, causal, groups, l2norm_qk,
                "decode rolling o")
    same_split = n_split_of(B, H, Hk, Nq, C, W, causal) == n_split_of(B, H, Hk, Nq, cap, W, causal)
    if same_split:
        assert bitwise(o, o_full)
    return same_split


# ---- dense parity over the covering grid --------------------------------------------------------------------------
# L_b on both sides of multiples of C (the append wraps inside a call), far past C, and 0; W not a multiple of 128
_BASE = dict(H=8, Hk=2, Nq=4, C=384, W=300, causal=True, groups=1, l2norm_qk=True, append=True)
_VARIANTS = [dict(), dict(C=256, W=253), dict(causal=False), dict(causal=False, C=256, W=253), dict(H=8, Hk=1),
             dict(H=8, Hk=8), dict(groups=8), dict(l2norm_qk=False), dict(append=False), dict(Nq=1, W=128, C=128),
             dict(Nq=70, W=59, C=128)]


def _case_id(v):
    return "-".join(f"{k}{int(x) if isinstance(x, bool) else x}" for k, x in v.items()) or "base"


@pytest.mark.parametrize("variant", _VARIANTS, ids=_case_id)
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_dense_grid(fcsa, variant, D, dtype):
    c = {**_BASE, **variant}
    C, n = c["C"], c["Nq"]
    lens = [0, 3, C - n, C - 1, C, C + 1, 2 * C - 2, 5 * C + 77]
    run_dense(fcsa, dtype, D, c["H"], c["Hk"], n, lens, C, c["W"], causal=c["causal"], groups=c["groups"],
              l2norm_qk=c["l2norm_qk"], append=c["append"], seed=_VARIANTS.index(variant) + D)


@pytest.mark.parametrize("side", ["split", "one"])
@pytest.mark.parametrize("D", [64, 128])
def test_split_sides(fcsa, side, D):
    """One key split (a grid of at least one CTA per SM) and several; both equal the full-length call bitwise."""
    H, Hk, C, W = 8, 8, 512, 300
    B = 2 if side == "split" else math.ceil(sm_count() / Hk)
    s = n_split_of(B, H, Hk, 1, C, W)
    assert (s == 1) == (side == "one"), s
    lens = [C - 1, 40000] if side == "split" else [(C - 1, 3 * C + 5)[b % 2] for b in range(B)]
    assert run_dense(fcsa, torch.bfloat16, D, H, Hk, 1, lens, C, W, seed=D)


# ---- packed new tokens ----------------------------------------------------------------------------------------------
def run_packed(fcsa, dtype, D, H, Hk, ns, lens, C, W, causal=True, append=True, seed=0):
    """One packed rolling call: element b brings ns[b] tokens (some 0) onto L_b = lens[b] positions."""
    from flash_cosine_sim_attention_b200 import l2norm_tensors
    B = len(ns)
    g = torch.Generator().manual_seed(seed)
    amp, scale = _setup(dtype, True, 1)
    cu, total = make_pack(ns, 2, 3)
    max_q = max(ns)
    cap = max(L + m for L, m in zip(lens, ns))
    q = torch.randn(total, H, D, generator=g).to(dtype).cuda()
    kf, vf = make_cache(B, Hk, cap, D, dtype, lens, g, True, 1, amp)
    kr, vr = rings_of(kf, C, lens), rings_of(vf, C, lens)
    k = v = None
    if append:
        k = torch.randn(total, Hk, D, generator=g).to(dtype).cuda()
        v = torch.randn(total, Hk, D, generator=g).to(dtype).cuda()
    sl = torch.tensor(lens, dtype=torch.int32, device="cuda")
    cu_t = torch.tensor(cu, dtype=torch.int32, device="cuda")
    kw = dict(scale=scale, causal=causal, window=W, cu_seqlens_q=cu_t, max_seqlen_q=max_q)
    with torch.no_grad():
        o = fcsa.flash_cosine_sim_attention_with_kv_cache(q, kr, vr, sl, k, v, rolling=True, **kw)
        o_full = fcsa.flash_cosine_sim_attention_with_kv_cache(q, kf, vf, sl, k, v, **kw)
    torch.cuda.synchronize()
    assert int(o[:cu[0]].count_nonzero()) == 0 and int(o[cu[-1]:].count_nonzero()) == 0
    qh = l2norm_tensors(q)[0]
    for b, L in enumerate(lens):
        T = L + (ns[b] if append else 0)
        assert bitwise(kr[b:b + 1], ring_of(kf[b:b + 1], C, T)), f"k ring {b}"
        assert bitwise(vr[b:b + 1], ring_of(vf[b:b + 1], C, T)), f"v ring {b}"
        if ns[b]:
            check_o(dtype, o[cu[b]:cu[b + 1]].transpose(0, 1)[None], qh[cu[b]:cu[b + 1]].transpose(0, 1)[None],
                    kf[b:b + 1], vf[b:b + 1], T, W, scale, causal, 1, True, "decode rolling packed o")
    if packed_split(B, H, Hk, max_q, C, W, causal) == packed_split(B, H, Hk, max_q, cap, W, causal):
        assert bitwise(o, o_full)


@pytest.mark.parametrize("append", [True, False], ids=["append", "no_append"])
@pytest.mark.parametrize("causal", [True, False], ids=["causal", "noncausal"])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_packed(fcsa, dtype, D, causal, append):
    C, W = 384, 250
    ns = [0, 1, 7, 130, 3, 0, 135]                  # C = W + max n - 1
    lens = [5, C - 1, C - 7, 2 * C + 1, 0, 3 * C, 4 * C - 60]
    run_packed(fcsa, dtype, D, 8, 2, ns, lens, C, W, causal=causal, append=append, seed=D + 2 * causal + append)


# ---- streaming through several wraps ---------------------------------------------------------------------------------
@pytest.mark.parametrize("schedule", ["tokens", "chunks"])
def test_streaming_through_wraps(fcsa, schedule):
    """Decode token by token, or in chunks of 1 to 285 tokens, through more than two wraps of a ring that starts as the
    sentinel.  Each step's o equals the full-length cache's bitwise (the same split count: C and the full capacity both
    exceed the window's key bound), and the ring equals the last C positions of the full-length cache, bitwise."""
    from flash_cosine_sim_attention_b200 import l2norm_tensors
    dt, B, H, Hk, D, C, W = torch.bfloat16, 2, 8, 2, 64, 384, 100
    total = 2 * C + 130
    sizes = [1] * total if schedule == "tokens" else [1, 7, 64, 285, 3, 130, 1, 200, 77, 64, 1, 59, 70]
    assert sum(sizes) >= total and max(sizes) <= C - W + 1
    assert n_split_of(B, H, Hk, max(sizes), C, W) == n_split_of(B, H, Hk, max(sizes), total + 300, W)
    g = torch.Generator(device="cuda").manual_seed(5)
    kf = torch.empty(B, Hk, total + 300, D, dtype=dt, device="cuda")
    kf.view(torch.int16).fill_(SENTINEL)
    vf = kf.clone()
    kr = torch.empty(B, Hk, C, D, dtype=dt, device="cuda")
    kr.view(torch.int16).fill_(SENTINEL)
    vr = kr.clone()
    sl_r = torch.zeros(B, dtype=torch.int32, device="cuda")
    sl_f = sl_r.clone()
    L = 0
    with torch.no_grad():
        for step, n in enumerate(sizes):
            q = torch.randn(B, H, n, D, generator=g, device="cuda").to(dt)
            k = torch.randn(B, Hk, n, D, generator=g, device="cuda").to(dt)
            v = torch.randn(B, Hk, n, D, generator=g, device="cuda").to(dt)
            o = fcsa.flash_cosine_sim_attention_with_kv_cache(q, kr, vr, sl_r, k, v, window=W, rolling=True)
            o_full = fcsa.flash_cosine_sim_attention_with_kv_cache(q, kf, vf, sl_f, k, v, window=W)
            sl_r += n
            sl_f += n
            L += n
            assert torch.isfinite(o.float()).all(), step
            assert bitwise(o, o_full), f"step {step}: L = {L}"
            assert bitwise(kr, rings_of(kf, C, [L] * B)) and bitwise(vr, rings_of(vf, C, [L] * B)), f"step {step}"
            if step % 97 == 0 or L >= total:
                check_o(dt, o, l2norm_tensors(q)[0], kf, vf, L, W, 8, True, 1, True, "decode rolling stream o")
            if L >= total:
                break
    assert L >= 2 * C


def test_rows_never_written_nan(fcsa):
    """A ring that is all NaN but for the positions a call sees: o is finite and the reference's, for lengths that
    leave most of the ring unwritten and for a tile past T_b that reaches rows never written."""
    run_dense(fcsa, torch.float16, 128, 8, 2, 3, [0, 1, 100, 130], 512, 200, seed=3)
    run_dense(fcsa, torch.bfloat16, 64, 8, 2, 3, [0, 1, 100, 130], 512, 200, causal=False, append=False, seed=4)


# ---- CUDA graph -----------------------------------------------------------------------------------------------------
def test_cuda_graph_across_a_wrap(fcsa):
    """One step captured once, replayed 12 times with cache_seqlens advanced on the device: elements cross the wrap
    at different replays.  Each replay equals the eager call on a copy of the rings, bitwise."""
    dt, B, H, Hk, D, C, W = torch.float16, 3, 8, 2, 64, 256, 150
    g = torch.Generator().manual_seed(21)
    kr, vr = (torch.randn(B, Hk, C, D, generator=g).to(dt).cuda() for _ in range(2))
    sq = torch.zeros(B, H, 1, D, dtype=dt, device="cuda")
    sk, sv = (torch.zeros(B, Hk, 1, D, dtype=dt, device="cuda") for _ in range(2))
    seqlens = torch.tensor([250, 3 * C - 4, 7000], dtype=torch.int32, device="cuda")

    def step(kr_, vr_, sl):
        return fcsa.flash_cosine_sim_attention_with_kv_cache(sq, kr_, vr_, sl, sk, sv, window=W, rolling=True)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.no_grad(), torch.cuda.stream(side):
        step(kr.clone(), vr.clone(), seqlens.clone())
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.no_grad(), torch.cuda.graph(graph, stream=side):
        out = step(kr, vr, seqlens)
    for _ in range(12):
        with torch.no_grad():
            sq.copy_(torch.randn(sq.shape, generator=g).to(dt))
            sk.copy_(torch.randn(sk.shape, generator=g).to(dt))
            sv.copy_(torch.randn(sv.shape, generator=g).to(dt))
            kre, vre, sle = kr.clone(), vr.clone(), seqlens.clone()
            want = step(kre, vre, sle)
            graph.replay()
            torch.cuda.synchronize()
            assert bitwise(out, want)
            assert bitwise(kr, kre) and bitwise(vr, vre)
            seqlens += 1


# ---- no new kernels -------------------------------------------------------------------------------------------------
# The ring calls run under torch.profiler in a child process.  Run in the pytest process, this session came before the
# other GPU test files, and test_gpu_kernel_census.py's sessions later in that process then saw no kernel at all; the
# census passed alone and right after this file.
_LAUNCHES = """
import json, torch
from flash_cosine_sim_attention_b200 import flash_cosine_sim_attention_with_kv_cache as f
from kernel_census import launched_kernels
dt, D, C, W = torch.bfloat16, 128, 256, 200
kr = torch.zeros(2, 2, C, D, dtype=dt, device="cuda")
vr = torch.zeros_like(kr)
sl = torch.tensor([300, 5], dtype=torch.int32, device="cuda")
q, k = torch.randn(2, 8, 2, D, dtype=dt, device="cuda"), torch.randn(2, 2, 2, D, dtype=dt, device="cuda")
qp, kp = torch.randn(5, 8, D, dtype=dt, device="cuda"), torch.randn(5, 2, D, dtype=dt, device="cuda")
cu = torch.tensor([0, 2, 5], dtype=torch.int32, device="cuda")
with torch.no_grad():
    _, names = launched_kernels(lambda: (f(q, kr, vr, sl, k, k, window=W, rolling=True),
                                         f(qp, kr, vr, sl, kp, kp, window=W, cu_seqlens_q=cu, max_seqlen_q=3,
                                           rolling=True)))
print(json.dumps(sorted(names)))
"""


def test_launches_only_existing_instantiations(fcsa):
    """Dense and packed ring calls, with key splits, launch the windowed decode kernel, the combine, the append pass
    and the varlen tail: instantiations the library already holds."""
    import json
    import os
    import subprocess
    import sys
    from flash_cosine_sim_attention_b200._abi import LIB_PATH
    dt, D = torch.bfloat16, 128
    assert n_split_of(2, 8, 2, 2, 256, 200) > 1
    here = os.path.dirname(os.path.abspath(__file__))
    env = {**os.environ, "PYTHONPATH": os.pathsep.join([here, os.path.dirname(here), os.environ.get("PYTHONPATH", "")])}
    out = subprocess.run([sys.executable, "-c", _LAUNCHES], capture_output=True, text=True, env=env, timeout=600)
    assert out.returncode == 0, out.stderr[-4000:]
    names = set(json.loads(out.stdout.strip().splitlines()[-1]))
    expected = {decode(dt, D, window=True), combine(dt, D), row_fwd(dt, D, append=True), VARLEN_TAIL}
    assert names == expected, names
    assert names <= set(library_kernels(LIB_PATH))


# ---- the transformer --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_transformer_rolling_cache(dtype):
    """Window 40: rings of 256 rows and prefill chunks of 217 tokens.  A 300-token prompt, then single tokens past 2 C
    positions: the logits match the full-length cache's and the full forward's, and generate runs on rolling caches."""
    from flash_cosine_sim_attention_b200.transformer import CosineSimCausalTransformer
    torch.manual_seed(0)
    m = CosineSimCausalTransformer(num_tokens=256, dim=128, max_seq_len=640, depth=2, heads=4, dim_head=64,
                                   kv_heads=2, pre_norm=True, use_cuda_kernel=True, window=40).cuda().eval()
    x = torch.randint(0, 256, (2, 560), device="cuda")
    with torch.no_grad(), torch.autocast("cuda", dtype=dtype):
        full = m(x).float()
        ring, flat = m.new_cache(rolling=True), m.new_cache()
        steps_r, steps_f = [m(x[:, :300], cache=ring)], [m(x[:, :300], cache=flat)]
        for i in range(300, 560):
            steps_r.append(m(x[:, i:i + 1], cache=ring))
            steps_f.append(m(x[:, i:i + 1], cache=flat))
        inc_r, inc_f = torch.cat(steps_r, 1).float(), torch.cat(steps_f, 1).float()
    assert ring[0].k.shape[2] == 256 and ring[0].length == 560
    assert torch.isfinite(inc_r).all()
    assert (inc_r - inc_f).abs().max() <= 5e-2 * inc_f.abs().max() + 1e-6
    assert (inc_r - full).abs().max() <= 5e-2 * full.abs().max() + 1e-6
    with torch.no_grad(), torch.autocast("cuda", dtype=dtype):
        out = m.generate(x[:, :300], 300, kv_cache=True, rolling_cache=True)
    assert out.shape == (2, 300)
