"""GPU tests of the deterministic backward (`deterministic=True`).

Three forward + backward calls give bitwise-equal dq, dk, dv; batch element b of a batch of three is bitwise the same
as the element alone; a packed sequence's gradients do not depend on the rest of the pack.  Every output is within the
float64 reference's element-wise bound at C = 2 (tests/elementwise_bounds.py, tests/window_bounds.py) and the relative
tolerances of test_gpu_parity.py; dk, dv are bitwise the default backward's wherever that keeps each kv group in one
CTA.  Also: the launches (preprocess, dK / dV, dQ), no zeroed workspace, CUDA graph replay, two training steps of the
transformer, and two long causal problems on memory that starts as NaN."""
import pytest
import torch

from elementwise_bounds import FMT, attention_bounds, check_bound, kernel_shift
from test_gpu_gqa import sm_count
from test_gpu_long_context import inputs, judge, run_dense
from test_gpu_parity import TOL_GRAD, TOL_OUT, fcsa, record, rel_err  # noqa: F401
from test_gpu_varlen import cu_of, make_packed, per_seq, run_varlen, seq_check
from tile_ranges import group_split
from window_bounds import window_attention_bounds

pytestmark = pytest.mark.gpu

DET = True              # the keyword under test (False runs the same assertions on the default backward)
NAMES = ("o", "dq", "dk", "dv")


def run(fcsa, q, k, v, do, **kw):
    """fwd + bwd through the public API on CUDA copies; returns ({o, dq, dk, dv}, kernels launched by the backward)."""
    qd, kd, vd = (t.cuda().clone().requires_grad_() for t in (q, k, v))
    o = fcsa.flash_cosine_sim_attention(qd, kd, vd, **kw)
    torch.cuda.synchronize()
    before = fcsa.debug()
    o.backward(do.cuda())
    torch.cuda.synchronize()
    return dict(o=o.detach(), dq=qd.grad, dk=kd.grad, dv=vd.grad), fcsa.debug() - before


def repeated(fcsa, q, k, v, do, **kw):
    """Three calls: asserts dq, dk, dv (and o) bitwise equal; returns the first call's outputs and launches."""
    first, launched = run(fcsa, q, k, v, do, deterministic=DET, **kw)
    for _ in range(2):
        again, _ = run(fcsa, q, k, v, do, deterministic=DET, **kw)
        for n in NAMES:
            assert torch.equal(first[n], again[n]), f"{n} differs between identical calls"
    return first, launched


def bounded(dtype, got, q, k, v, do, window=None, **kw):
    """Every output against the float64 reference: element-wise bound at C = 2 and the relative tolerance."""
    fmt = FMT[dtype]
    l2 = kw.get("l2norm_qk", True)
    shift = kernel_shift(fmt, kw.get("scale", 8), kw.get("groups", 1), l2)
    common = dict(round_qk=fmt if l2 else None, fmt=fmt, shift=shift, device="cuda", **kw)
    if window is None:
        ref, bound = attention_bounds(q, k, v, do, **common)
    else:
        ref, bound = window_attention_bounds(q, k, v, do, window=window, **common)
    for n in NAMES:
        record(dtype, f"deterministic {n}/bound", check_bound(n, got[n], ref, bound, fmt), 1.0)
        if float(ref[n].abs().max()) > 1e-6:
            e = rel_err(got[n], ref[n].cpu().numpy())
            tol = TOL_OUT[dtype] if n == "o" else TOL_GRAD[dtype]
            record(dtype, f"deterministic {n}", e, tol)
            assert e <= tol, (n, e, tol)
    return ref, bound


def make(B, H, Hk, Nq, Nk, D, dtype, seed, q3=False, k3=False):
    g = torch.Generator().manual_seed(seed)
    qs = (B, Nq, D) if q3 else (B, H, Nq, D)
    ks = (B, Nk, D) if (q3 or k3) else (B, Hk, Nk, D)
    return tuple(torch.randn(*s, generator=g).to(dtype) for s in (qs, ks, ks, qs))


def default_agrees(fcsa, got, q, k, v, do, **kw):
    """dk, dv bitwise the default backward's when it keeps each group in one CTA."""
    dflt, _ = run(fcsa, q, k, v, do, **kw)
    assert torch.equal(dflt["o"], got["o"])
    B, H = q.shape[0], (q.shape[1] if q.ndim == 4 else 1)
    Hk = k.shape[1] if k.ndim == 4 else 1
    if group_split(B, H, Hk, k.shape[-2], sm_count()) == 1:
        assert torch.equal(dflt["dk"], got["dk"]) and torch.equal(dflt["dv"], got["dv"])
    return dflt


# ---- 1. the grid: dtypes, head dims, causal, lengths, heads ---------------------------------------------------------
SHAPES = [(300, 300), (300, 700), (700, 300)]


@pytest.mark.parametrize("nq,nk", SHAPES, ids=[f"{a}x{b}" for a, b in SHAPES])
@pytest.mark.parametrize("causal", [False, True], ids=["full", "causal"])
@pytest.mark.parametrize("heads,kv_heads", [(4, 4), (4, 2)])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "f16"])
def test_grid(fcsa, dtype, D, heads, kv_heads, causal, nq, nk):
    q, k, v, do = make(1, heads, kv_heads, nq, nk, D, dtype, seed=nq + 3 * nk + D + kv_heads)
    got, launched = repeated(fcsa, q, k, v, do, causal=causal)
    assert launched == 3, launched            # preprocess, dK / dV, dQ: no dq finish, no dk / dv finish
    ref, bound = bounded(dtype, got, q, k, v, do, causal=causal)
    dflt = default_agrees(fcsa, got, q, k, v, do, causal=causal)
    check_bound("dq", dflt["dq"], ref, bound, FMT[dtype])
    if causal and nq > nk:
        # rows whose causal limit lies before key 0 see no key
        assert (got["dq"][:, :, :nq - nk] == 0).all()


# ---- 2. batch invariance --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("causal", [False, True], ids=["full", "causal"])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "f16"])
def test_batch_element_alone(fcsa, dtype, D, causal):
    q, k, v, do = make(3, 4, 2, 300, 700, D, dtype, seed=5 + D)
    got, _ = repeated(fcsa, q, k, v, do, causal=causal)
    for b in range(3):
        one, _ = run(fcsa, *(t[b:b + 1] for t in (q, k, v, do)), causal=causal, deterministic=DET)
        for n in NAMES:
            assert torch.equal(got[n][b:b + 1], one[n]), (b, n)


# ---- 3. grouped grids the default backward splits, MQA, 3-D keys, merged heads ----------------------------------------
@pytest.mark.parametrize("D", [64, 128])
def test_split_group(fcsa, D):
    dtype, B, H, Hk, N = torch.bfloat16, 1, 8, 2, 300
    assert group_split(B, H, Hk, N, sm_count()) > 1          # the default sums dk / dv over CTAs here
    q, k, v, do = make(B, H, Hk, N, N, D, dtype, seed=11)
    got, launched = repeated(fcsa, q, k, v, do, causal=True)
    assert launched == 3, launched
    bounded(dtype, got, q, k, v, do, causal=True)


@pytest.mark.parametrize("layout", ["mqa", "k3", "q3"])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("causal", [False, True], ids=["full", "causal"])
def test_layouts(fcsa, layout, D, causal):
    dtype = torch.bfloat16
    q, k, v, do = make(2, 4, 1, 300, 300, D, dtype, seed=13 + D, q3=layout == "q3", k3=layout == "k3")
    got, launched = repeated(fcsa, q, k, v, do, causal=causal)
    assert launched == 3, launched
    bounded(dtype, got, q, k, v, do, causal=causal)
    default_agrees(fcsa, got, q, k, v, do, causal=causal)


# ---- 4. key mask, windows, l2norm options -----------------------------------------------------------------------------
@pytest.mark.parametrize("D", [64, 128])
def test_key_mask(fcsa, D):
    dtype = torch.float16
    q, k, v, do = make(2, 4, 2, 300, 700, D, dtype, seed=17)
    mask = torch.rand(2, 700, generator=torch.Generator().manual_seed(1)) > 0.3
    mask[1, :] = False                                       # batch element 1 sees no key: dq = 0 there
    got, _ = repeated(fcsa, q, k, v, do, mask=mask.cuda())
    bounded(dtype, got, q, k, v, do, mask=mask)
    assert (got["dq"][1] == 0).all()
    default_agrees(fcsa, got, q, k, v, do, mask=mask.cuda())


def window_case(fcsa, dtype, heads, kv_heads, window, causal, D):
    q, k, v, do = make(1, heads, kv_heads, 700, 300, D, dtype, seed=window + D)
    got, launched = repeated(fcsa, q, k, v, do, causal=causal, window=window)
    assert launched == 3, launched
    bounded(dtype, got, q, k, v, do, window=window, causal=causal)
    default_agrees(fcsa, got, q, k, v, do, causal=causal, window=window)


@pytest.mark.parametrize("window", [1, 65, 200])
@pytest.mark.parametrize("causal", [False, True], ids=["full", "causal"])
@pytest.mark.parametrize("D", [64, 128])
def test_window(fcsa, window, causal, D):
    window_case(fcsa, torch.bfloat16, 4, 2, window, causal, D)


# the other dtype and MHA (one query head per CTA: no head loop in the dK / dV kernel)
@pytest.mark.parametrize("window", [1, 65, 200])
@pytest.mark.parametrize("causal", [False, True], ids=["full", "causal"])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("dtype,heads,kv_heads", [(torch.float16, 4, 4), (torch.float16, 4, 2),
                                                  (torch.bfloat16, 4, 4)], ids=["f16-4:4", "f16-4:2", "bf16-4:4"])
def test_window_dtypes_and_heads(fcsa, dtype, heads, kv_heads, window, causal, D):
    window_case(fcsa, dtype, heads, kv_heads, window, causal, D)


@pytest.mark.parametrize("opts", [dict(groups=1), dict(groups=8, scale=1), dict(l2norm_qk=False, scale=1)],
                         ids=["groups1", "groups8", "no-l2norm"])
@pytest.mark.parametrize("D", [64, 128])
def test_l2norm_options(fcsa, opts, D):
    dtype = torch.bfloat16
    q, k, v, do = make(1, 4, 2, 300, 300, D, dtype, seed=23)
    got, _ = repeated(fcsa, q, k, v, do, causal=True, **opts)
    bounded(dtype, got, q, k, v, do, causal=True, **opts)


# ---- 5. float32 and zero-padded head dims -----------------------------------------------------------------------------
@pytest.mark.parametrize("dtype,D,window", [(torch.float32, 32, None), (torch.float32, 64, None),
                                            (torch.float32, 96, None), (torch.bfloat16, 32, None),
                                            (torch.bfloat16, 96, None), (torch.float32, 64, 65)],
                         ids=["f32-32", "f32-64", "f32-96", "bf16-32", "bf16-96", "f32-64-window65"])
def test_other_dtypes_and_head_dims(fcsa, dtype, D, window):
    q, k, v, do = make(1, 4, 2, 300, 300, D, dtype, seed=29 + D)
    kw = dict(causal=True) if window is None else dict(causal=True, window=window)
    got, _ = repeated(fcsa, q, k, v, do, **kw)
    if dtype == torch.float32:
        bounds = attention_bounds if window is None else window_attention_bounds
        judge(dtype, {n: t.cuda() for n, t in got.items()}, *(t.cuda() for t in (q, k, v, do)), bounds=bounds, **kw)
    else:
        bounded(dtype, got, q, k, v, do, **kw)
    default_agrees(fcsa, got, q, k, v, do, **kw)


# ---- 6. packed sequences ------------------------------------------------------------------------------------------------
SKEWED = [700, 0, 1, 65, 129, 300]


def varlen_repeated(fcsa, q, k, v, do, cu, m, **kw):
    first = run_varlen(fcsa, q, k, v, do, cu, cu, m, m, deterministic=DET, **kw)
    for _ in range(2):
        again = run_varlen(fcsa, q, k, v, do, cu, cu, m, m, deterministic=DET, **kw)
        for n, a, b in zip(NAMES, first[:4], again[:4]):
            assert torch.equal(a, b), n
    return first


def varlen_case(fcsa, dtype, heads, kv_heads, D, causal, window=None):
    ls = SKEWED
    q, k, v, do = make_packed(ls, ls, heads, kv_heads, D, dtype, seed=31 + D + kv_heads)
    cu = cu_of(ls)
    kw = dict(causal=causal) if window is None else dict(causal=causal, window=window)
    *got, launched = varlen_repeated(fcsa, q, k, v, do, cu, max(ls), **kw)
    assert launched == 4, launched            # preprocess, dK / dV, dQ, the rows outside every sequence
    seq_check(dtype, got, q, k, v, do, ls, ls, **kw)
    # the same sequences in another order: each sequence's gradients bitwise unchanged
    order = [3, 5, 0, 2, 1, 4]
    starts = cu.tolist()
    pick = lambda t: torch.cat([t[starts[i]:starts[i + 1]] for i in order])
    ls2 = [ls[i] for i in order]
    cu2 = cu_of(ls2)
    got2 = varlen_repeated(fcsa, *(pick(t) for t in (q, k, v, do)), cu2, max(ls), **kw)
    starts2 = cu2.tolist()
    for j, i in enumerate(order):
        for n, a, b in zip(NAMES, got, got2[:4]):
            assert torch.equal(a[starts[i]:starts[i + 1]], b[starts2[j]:starts2[j + 1]]), (i, n)
    if heads == kv_heads:
        # MHA: each sequence bitwise as the dense deterministic op on it alone
        for i, n in enumerate(ls):
            if n == 0:
                continue
            s = starts[i]
            dense, _ = run(fcsa, *(per_seq(t, s, n) for t in (q, k, v, do)), deterministic=DET, **kw)
            for name, t in zip(NAMES, got):
                assert torch.equal(per_seq(t, s, n), dense[name]), (i, name)


@pytest.mark.parametrize("heads,kv_heads", [(4, 4), (4, 2)])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("causal", [False, True], ids=["full", "causal"])
def test_varlen(fcsa, heads, kv_heads, D, causal):
    varlen_case(fcsa, torch.bfloat16, heads, kv_heads, D, causal)


# fp16, and a sliding window in both dtypes (the packed, windowed dK / dV and dQ kernels)
@pytest.mark.parametrize("heads,kv_heads", [(4, 4), (4, 2)])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("causal", [False, True], ids=["full", "causal"])
@pytest.mark.parametrize("dtype,window", [(torch.float16, None), (torch.float16, 65), (torch.bfloat16, 65)],
                         ids=["f16", "f16-window65", "bf16-window65"])
def test_varlen_dtypes_and_windows(fcsa, dtype, window, heads, kv_heads, D, causal):
    varlen_case(fcsa, dtype, heads, kv_heads, D, causal, window)


def test_varlen_rows_outside_sequences(fcsa):
    dtype, H, D = torch.bfloat16, 4, 64
    ls = [65, 0, 300]
    q, k, v, do = make_packed([10] + ls + [37], [10] + ls + [37], H, H, D, dtype, seed=37)
    cu = cu_of(ls) + 10                                      # rows [0, 10) and the last 37 belong to no sequence
    o, dq, dk, dv, _ = varlen_repeated(fcsa, q, k, v, do, cu, 300, causal=True)
    for t in (o, dq, dk, dv):
        assert (t[:10] == 0).all() and (t[-37:] == 0).all()
    seq_check(dtype, (o[10:-37], dq[10:-37], dk[10:-37], dv[10:-37]), *(t[10:-37] for t in (q, k, v, do)), ls, ls,
              causal=True)


# ---- 7. workspaces, graphs, the transformer ----------------------------------------------------------------------------
def test_no_zeroed_workspace(fcsa):
    from flash_cosine_sim_attention_b200 import _abi
    dtype, D = torch.bfloat16, 64
    q, k, v, do = make(2, 4, 2, 300, 700, D, dtype, seed=41)
    fcsa.release_workspaces()
    got, _ = run(fcsa, q, k, v, do, causal=True, deterministic=True)
    torch.cuda.synchronize()
    p = _abi.FcsaProblem()
    p.dtype, p.batch, p.heads, p.kv_heads, p.seq_q, p.seq_k, p.head_dim = _abi.FCSA_BF16, 2, 4, 2, 300, 700, D
    scratch = _abi.load().fcsa_backward_fused_deterministic_workspace_bytes(_abi.ref(p))
    assert fcsa.release_workspaces() == scratch              # the scratch alone was allocated
    # a default backward after a deterministic one still finds its zeroed workspace zero
    run(fcsa, q, k, v, do, causal=True, deterministic=True)
    dflt, _ = run(fcsa, q, k, v, do, causal=True)
    ref, bound = bounded(dtype, dflt, q, k, v, do, causal=True)
    check_bound("dq", got["dq"], ref, bound, FMT[dtype])


def test_cuda_graph(fcsa):
    dtype, H, Hk, N, D = torch.bfloat16, 8, 2, 300, 64
    q, k, v, do = (t.cuda() for t in make(1, H, Hk, N, N, D, dtype, seed=43))
    qs, ks, vs = (t.clone().requires_grad_() for t in (q, k, v))
    out = {}

    def step():
        for t in (qs, ks, vs):
            t.grad = None
        o = fcsa.flash_cosine_sim_attention(qs, ks, vs, causal=True, deterministic=DET)
        o.backward(do)
        out["o"] = o.detach()

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        step()
    eager, _ = run(fcsa, q, k, v, do, causal=True, deterministic=DET)
    for _ in range(3):
        graph.replay()
        torch.cuda.synchronize()
        for n, t in (("o", out["o"]), ("dq", qs.grad), ("dk", ks.grad), ("dv", vs.grad)):
            assert torch.equal(t, eager[n]), n


@pytest.mark.parametrize("packed", [False, True], ids=["dense", "packed"])
def test_transformer_training_steps(fcsa, packed):
    from flash_cosine_sim_attention_b200.transformer import CosineSimCausalTransformer

    def train():
        torch.manual_seed(0)
        model = CosineSimCausalTransformer(num_tokens=64, dim=128, max_seq_len=512, depth=2, heads=4, dim_head=64,
                                           kv_heads=2, use_cuda_kernel=True, deterministic=DET).cuda().to(torch.bfloat16)
        opt = torch.optim.SGD(model.parameters(), lr=1e-2)
        g = torch.Generator(device="cuda").manual_seed(1)
        for _ in range(2):
            opt.zero_grad()
            if packed:
                docs = [200, 1, 300]
                x = torch.randint(0, 64, (1, sum(docs)), device="cuda", generator=g)
                logits = model(x, cu_seqlens=cu_of(docs).cuda(), max_seqlen=max(docs))
                loss = logits.float().square().mean()
            else:
                x = torch.randint(0, 64, (2, 301), device="cuda", generator=g)
                loss = model(x, return_loss=True)
            loss.backward()
            opt.step()
        return [p.detach().clone() for p in model.parameters()]

    a, b = train(), train()
    for i, (x, y) in enumerate(zip(a, b)):
        assert torch.equal(x, y), i


# ---- 8. long causal problems on memory that starts as NaN ------------------------------------------------------------
@pytest.mark.parametrize("D,N", [(64, 32769), (128, 16385)], ids=["D64-N32769", "D128-N16385"])
def test_long_causal(fcsa, D, N):
    dtype = torch.bfloat16
    q, k, v, do = inputs((1, 1, N, D), (1, 1, N, D), dtype, seed=N)
    got = run_dense(fcsa, q, k, v, do, dtype, causal=True, deterministic=DET)
    judge(dtype, got, q, k, v, do, causal=True)
