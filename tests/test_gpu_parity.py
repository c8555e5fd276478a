"""GPU parity tests (run on an H100 with `pytest -m gpu`): the CUDA path - reached through the
public Python API, i.e. ctypes -> C ABI -> sm_90a kernels - against the float64 oracle on the
same (already rounded) inputs, against the committed reference golden vectors, and through
size-independent properties at BASELINE.json's full sizes.

Tolerance policy (floating point; stated per test):
  max |got - ref| <= tol * max |ref|, tol = 1e-2 for bf16 and 2e-3 for f16 outputs, 2e-2 / 4e-3
  for gradients (they pass through two more 16-bit roundings: P/dS operands and the stored
  normalised q, k).  The reference's own tests allow 1e-1 absolute in f16 (tests/test.py:12-18,49).
Next to it, element-wise: |got - ref| <= C u M for every element of every output, M modelling the kernels'
roundings (tests/elementwise_bounds.py); the worst err / (C u M) is recorded under '<dtype>:<name>/bound'.
"""
import ast
import glob
import os

import numpy as np
import pytest
import torch

from elementwise_bounds import FMT, attention_bounds, check_bound, kernel_shift, round_to
from oracle import cosine_sim_attention_oracle as oracle

pytestmark = pytest.mark.gpu

TOL_OUT = {torch.bfloat16: 1e-2, torch.float16: 2e-3, torch.float32: 1e-3}
TOL_GRAD = {torch.bfloat16: 2e-2, torch.float16: 4e-3, torch.float32: 2e-3}
BWD_HEAD_DIMS = (16, 32, 64, 96, 128)   # 16, 32 and 96 run the 64 / 128 kernels on zero-padded features
# the op stores normalised q, k in the input dtype; float32 inputs are compared with the UNROUNDED oracle
ROUND = {torch.bfloat16: "bf16", torch.float16: "f16", torch.float32: None}

# achieved errors, per dtype and quantity: the worst seen over the whole run, written to
# gpurun_out/parity_errors.json and printed in the pytest summary (conftest.py)
ERRORS = {}


def record(dtype, what, err, tol):
    key = f"{str(dtype).replace('torch.', '')}:{what}"
    cur = ERRORS.get(key)
    if cur is None or err > cur["max_err"]:
        ERRORS[key] = {"max_err": float(err), "tol": float(tol)}


@pytest.fixture(scope="module")
def fcsa():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import flash_cosine_sim_attention_b200 as pkg
    from flash_cosine_sim_attention_b200 import _abi
    _abi.load()            # fail loudly if the native library did not travel
    return pkg


def rel_err(got, ref):
    got = got.detach().float().cpu().numpy().astype(np.float64)
    assert np.isfinite(got).all(), "NaN/Inf in CUDA result"
    mag = np.abs(ref).max()
    if mag < 1e-6:
        # the exact answer is identically zero (e.g. dq with a single key: softmax over one
        # element): only 16-bit rounding noise may remain, judged on an absolute scale
        return np.abs(got).max() / 5.0
    return np.abs(got - ref).max() / mag


def float32_operands(q, k, v, do, attn_bias=None, scale=8, groups=1, l2norm_qk=True):
    """What the float32 path hands the 16-bit kernels (_float32_on_half_kernels): the operand type, and v, dO
    divided by their `_pow2_scale` factors, rounded and scaled back (exact), the bias rounded, q, k rounded when
    they are not normalised inside the op.  Returns (fmt, q, k, v, do, bias) as float64 CPU tensors."""
    from flash_cosine_sim_attention_b200.flash_cosine_sim_attention import _FP16_GROUPED_RANGE, _pow2_scale
    fmt = "f16" if (l2norm_qk and scale * groups <= _FP16_GROUPED_RANGE) else "bf16"
    t64 = lambda t: None if t is None else torch.as_tensor(t).detach().cpu().double()
    q, k, v, do, attn_bias = (t64(t) for t in (q, k, v, do, attn_bias))

    def scaled(t):
        s = _pow2_scale(t.float(), 1).double()
        return round_to(t / s, fmt) * s
    if not l2norm_qk:
        q, k = round_to(q, fmt), round_to(k, fmt)
    return fmt, q, k, scaled(v), None if do is None else scaled(do), round_to(attn_bias, fmt)


def float32_ds_scale(v, do):
    """sv * pg: the float32 path runs the kernels on v / sv and dO / pg (`_pow2_scale`), so the dS they round to 16 bit
    is the caller's dS / (sv pg), and the absolute eta of that rounding counts sv pg times over in the caller's units."""
    if do is None:
        return 1.0
    from flash_cosine_sim_attention_b200.flash_cosine_sim_attention import _pow2_scale
    f = lambda t: torch.as_tensor(t).detach().float()
    return float(_pow2_scale(f(v), 1) * _pow2_scale(f(do), 1))


def bound_check(dtype, got, q, k, v, do=None, mask=None, **kw):
    """The element-wise bound of every output in `got` ({name: tensor}) against the float64 reference of the same
    inputs, computed on the GPU; records the worst err / (C u M) per dtype and quantity under '<name>/bound'.
    float32 inputs are judged on the operands the 16-bit kernels really see (float32_operands)."""
    l2 = kw.get("l2norm_qk", True)
    bias = kw.get("attn_bias")
    if dtype == torch.float32:
        kw["ds_scale"] = float32_ds_scale(v, do)
        fmt, q, k, v, do, kw["attn_bias"] = float32_operands(q, k, v, do, bias, kw.get("scale", 8),
                                                             kw.get("groups", 1), l2)
    else:
        fmt = FMT[dtype]
    shift = kernel_shift(fmt, kw.get("scale", 8), kw.get("groups", 1), l2, bias)
    ref, bound = attention_bounds(q, k, v, do, mask=mask, round_qk=fmt if l2 else None, fmt=fmt, shift=shift,
                                  device="cuda", **kw)
    worst = {}
    for name, t in got.items():
        try:
            worst[name] = check_bound(name, t, ref, bound, fmt)
        except AssertionError:
            record(dtype, f"{name}/bound", float("inf"), 1.0)
            raise
        record(dtype, f"{name}/bound", worst[name], 1.0)
    return worst


def make_inputs(qs, kvs, dtype, seed, mask_p=None, amp=1.0):
    g = torch.Generator().manual_seed(seed)
    q = (torch.randn(qs, generator=g) * amp).to(dtype)
    k = (torch.randn(kvs, generator=g) * amp).to(dtype)
    v = torch.randn(kvs, generator=g).to(dtype)
    do = torch.randn(qs, generator=g).to(dtype)
    mask = None
    if mask_p is not None:
        mask = torch.rand((qs[0], kvs[-2]), generator=g) > mask_p
        mask[:, 0] = True
    return q, k, v, do, mask


def check(fcsa, qs, kvs, dtype, seed=0, mask_p=None, grads=True, amp=1.0, **kw):
    q, k, v, do, mask = make_inputs(qs, kvs, dtype, seed, mask_p, amp)
    dev = "cuda"
    grads = grads and qs[-1] in BWD_HEAD_DIMS
    qd, kd, vd = (t.to(dev).requires_grad_(grads) for t in (q, k, v))
    o = fcsa.flash_cosine_sim_attention(qd, kd, vd, mask=None if mask is None else mask.to(dev), **kw)
    assert o.shape == q.shape and o.dtype == dtype
    ref = oracle.attention(q.float().numpy(), k.float().numpy(), v.float().numpy(),
                           mask=None if mask is None else mask.numpy(),
                           d_out=do.float().numpy() if grads else None, empty_rows="zero",
                           round_qk=ROUND[dtype], **kw)
    if not grads:
        e = rel_err(o, ref)
        record(dtype, "o", e, TOL_OUT[dtype])
        assert e <= TOL_OUT[dtype]
        bound_check(dtype, {"o": o}, q, k, v, mask=mask, **kw)
        return
    o.backward(do.to(dev))
    e = rel_err(o, ref[0])
    record(dtype, "o", e, TOL_OUT[dtype])
    assert e <= TOL_OUT[dtype], "o"
    for name, t, r in (("dq", qd, ref[1]), ("dk", kd, ref[2]), ("dv", vd, ref[3])):
        assert t.grad.shape == t.shape and t.grad.dtype == dtype
        e = rel_err(t.grad, r)
        record(dtype, name, e, TOL_GRAD[dtype])
        assert e <= TOL_GRAD[dtype], name
    bound_check(dtype, {"o": o, "dq": qd.grad, "dk": kd.grad, "dv": vd.grad}, q, k, v, do, mask=mask, **kw)


# ---- the reference's own test grid (tests/test.py:31-125), on the dtypes/head dims the kernels cover,
# ---- plus bf16 and MQA gradients which the reference never tested -----------------------------------
@pytest.mark.parametrize("causal,mask", [(True, False), (False, True), (False, False)])
@pytest.mark.parametrize("seq_len", [63, 127])
@pytest.mark.parametrize("dim_head", [64, 128])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("single_head_kv", [False, True])
def test_reference_grid(fcsa, causal, mask, seq_len, dim_head, dtype, single_head_kv):
    batch, heads = 4, 8
    kvs = (batch, seq_len, dim_head) if single_head_kv else (batch, heads, seq_len, dim_head)
    check(fcsa, (batch, heads, seq_len, dim_head), kvs, dtype, seed=seq_len + dim_head,
          mask_p=0.5 if mask else None, causal=causal)


# ---- the remaining head dims of the reference grid (tests/test.py:33): zero-padded onto the same kernels
@pytest.mark.parametrize("causal,mask", [(True, False), (False, True)])
@pytest.mark.parametrize("dim_head,groups", [(32, 1), (96, 1), (32, 2), (96, 3)])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_padded_head_dims(fcsa, causal, mask, dim_head, groups, dtype):
    check(fcsa, (2, 4, 127, dim_head), (2, 4, 127, dim_head), dtype, seed=dim_head + groups,
          mask_p=0.5 if mask else None, causal=causal, groups=groups,
          scale=8 if groups == 1 or dtype == torch.bfloat16 else 4)


# ---- attn_bias (reference tests/test.py:32,58-61): the BIAS instantiations of both kernels, d_bias ----
@pytest.mark.parametrize("causal,mask", [(True, False), (False, True), (False, False)])
@pytest.mark.parametrize("dim_head", [64, 128])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("batch_dim", [False, True])
def test_attn_bias(fcsa, causal, mask, dim_head, dtype, batch_dim):
    B, H, Nq, Nk = 2, 3, 150, 203            # ragged on both axes, Nk not a multiple of 8
    if causal:
        Nk = Nq
    q, k, v, do, m = make_inputs((B, H, Nq, dim_head), (B, H, Nk, dim_head), dtype, seed=dim_head + 7 * batch_dim,
                                 mask_p=0.4 if mask else None)
    g = torch.Generator().manual_seed(99)
    bias = torch.randn((B if batch_dim else H, Nq, Nk), generator=g).to(dtype)
    if batch_dim:
        # the reference's batch-dim bias is (batch, i, j): one plane shared by the heads of a batch element
        pass
    qd, kd, vd, bd = (t.cuda().requires_grad_() for t in (q, k, v, bias))
    o = fcsa.flash_cosine_sim_attention(qd, kd, vd, mask=None if m is None else m.cuda(), attn_bias=bd,
                                        causal=causal, attn_bias_batch_dim=batch_dim)
    o.backward(do.cuda())
    nb = bias.float().numpy()
    if batch_dim:
        # oracle indexes a batch-dim bias as bias[b]; it applies to every head of that batch element
        ref = oracle.attention(q.float().numpy(), k.float().numpy(), v.float().numpy(),
                               mask=None if m is None else m.numpy(), attn_bias=nb, attn_bias_batch_dim=True,
                               causal=causal, d_out=do.float().numpy(), empty_rows="zero", round_qk=ROUND[dtype])
    else:
        ref = oracle.attention(q.float().numpy(), k.float().numpy(), v.float().numpy(),
                               mask=None if m is None else m.numpy(), attn_bias=nb, causal=causal,
                               d_out=do.float().numpy(), empty_rows="zero", round_qk=ROUND[dtype])
    assert rel_err(o, ref[0]) <= TOL_OUT[dtype], "o"
    for name, t, r in (("dq", qd, ref[1]), ("dk", kd, ref[2]), ("dv", vd, ref[3]), ("d_bias", bd, ref[4])):
        assert t.grad is not None and t.grad.shape == t.shape and t.grad.dtype == dtype, name
        assert rel_err(t.grad, r) <= TOL_GRAD[dtype], name
    bound_check(dtype, {"o": o, "dq": qd.grad, "dk": kd.grad, "dv": vd.grad, "d_bias": bd.grad}, q, k, v, do,
                mask=m, attn_bias=bias, causal=causal, attn_bias_batch_dim=batch_dim)


def test_attn_bias_single_head_kv_grouped_l2norm(fcsa):
    """bias together with shared keys/values (dk, dv summed over heads) and grouped l2norm, bf16."""
    dtype = torch.bfloat16
    B, H, Nq, Nk, D = 2, 4, 96, 136, 64
    q, k, v, do, m = make_inputs((B, H, Nq, D), (B, Nk, D), dtype, seed=5, mask_p=0.3)
    g = torch.Generator().manual_seed(6)
    bias = torch.randn((H, Nq, Nk), generator=g).to(dtype)
    qd, kd, vd, bd = (t.cuda().requires_grad_() for t in (q, k, v, bias))
    o = fcsa.flash_cosine_sim_attention(qd, kd, vd, mask=m.cuda(), attn_bias=bd, groups=2, scale=6)
    o.backward(do.cuda())
    ref = oracle.attention(q.float().numpy(), k.float().numpy(), v.float().numpy(), mask=m.numpy(),
                           attn_bias=bias.float().numpy(), groups=2, scale=6, d_out=do.float().numpy(),
                           empty_rows="zero", round_qk=ROUND[dtype])
    assert rel_err(o, ref[0]) <= TOL_OUT[dtype], "o"
    for name, t, r in (("dq", qd, ref[1]), ("dk", kd, ref[2]), ("dv", vd, ref[3]), ("d_bias", bd, ref[4])):
        assert t.grad.shape == t.shape
        assert rel_err(t.grad, r) <= TOL_GRAD[dtype], name


def test_attn_bias_without_grad_and_forward_only(fcsa):
    """a bias that needs no gradient takes the no-accumulator path; forward-only under no_grad."""
    dtype = torch.float16
    q, k, v, do, _ = make_inputs((1, 2, 200, 128), (1, 2, 200, 128), dtype, seed=8)
    bias = torch.randn((2, 200, 200), generator=torch.Generator().manual_seed(9)).to(dtype)
    ref = oracle.attention(q.float().numpy(), k.float().numpy(), v.float().numpy(), attn_bias=bias.float().numpy(),
                           causal=True, d_out=do.float().numpy(), empty_rows="zero", round_qk=ROUND[dtype])
    with torch.no_grad():
        o = fcsa.flash_cosine_sim_attention(q.cuda(), k.cuda(), v.cuda(), attn_bias=bias.cuda(), causal=True)
    assert rel_err(o, ref[0]) <= TOL_OUT[dtype]
    qd, kd, vd = (t.cuda().requires_grad_() for t in (q, k, v))
    o = fcsa.flash_cosine_sim_attention(qd, kd, vd, attn_bias=bias.cuda(), causal=True)
    o.backward(do.cuda())
    for name, t, r in (("dq", qd, ref[1]), ("dk", kd, ref[2]), ("dv", vd, ref[3])):
        assert rel_err(t.grad, r) <= TOL_GRAD[dtype], name


# ---- committed golden vectors produced by the unmodified reference --------------------------------
GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "*.npz")))


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[:-4] for p in GOLDEN])
def test_reference_golden_vectors(fcsa, path):
    z = np.load(path)
    kw = ast.literal_eval(str(z["kwargs"]))
    mask = torch.from_numpy(z["mask"]).cuda() if z["mask"].size else None
    dt = torch.bfloat16     # the golden inputs are bf16-representable by construction
    grads = z["q"].shape[-1] in BWD_HEAD_DIMS
    q, k, v = (torch.from_numpy(z[n]).to(dt).cuda().requires_grad_(grads) for n in ("q", "k", "v"))
    assert np.array_equal(q.detach().float().cpu().numpy(), z["q"])
    bias = None
    if "attn_bias" in z.files:
        bias = torch.from_numpy(z["attn_bias"]).to(dt).cuda().requires_grad_(grads)
        kw = dict(kw, attn_bias=bias)
    o = fcsa.flash_cosine_sim_attention(q, k, v, mask=mask, **kw)
    want = {n: z[n] for n in ("o", "dq", "dk", "dv")}
    if kw.get("causal") and z["q"].shape[-2] > z["k"].shape[-2]:
        # queries that see no key: the naive reference averages v, the fused kernels (reference's
        # included, cu:1239) give 0.  Compare with the oracle's "zero" variant, which test_oracle.py
        # pins to these same golden vectors in its "mean" variant.
        ref = oracle.attention(z["q"], z["k"], z["v"], d_out=z["d_out"], empty_rows="zero", **kw)
        want = dict(zip(("o", "dq", "dk", "dv"), ref))
    assert rel_err(o, want["o"]) <= TOL_OUT[dt]
    if grads:
        o.backward(torch.from_numpy(z["d_out"]).to(dt).cuda())
        for name, t in (("dq", q), ("dk", k), ("dv", v)):
            assert rel_err(t.grad, want[name]) <= TOL_GRAD[dt], name
        if bias is not None:
            assert bias.grad is not None and bias.grad.shape == bias.shape
            assert rel_err(bias.grad, z["d_bias"]) <= TOL_GRAD[dt], "d_bias"


# ---- features the reference never tested ------------------------------------------------------------
@pytest.mark.parametrize("qn,kn", [(200, 456), (456, 200), (129, 129), (1, 300), (257, 1)])
def test_causal_cross_lengths(fcsa, qn, kn):
    check(fcsa, (2, 2, qn, 64), (2, 2, kn, 64), torch.bfloat16, seed=qn, causal=True)


@pytest.mark.parametrize("groups,scale", [(2, 8), (4, 10), (8, 1), (16, 4)])
def test_groups_and_scales(fcsa, groups, scale):
    check(fcsa, (1, 4, 300, 64), (1, 4, 300, 64), torch.bfloat16, seed=groups, groups=groups, scale=scale)


@pytest.mark.parametrize("groups,scale", [(1, 10), (2, 8), (8, 1)])
def test_groups_and_scales_fp16(fcsa, groups, scale):
    """fp16 holds exp(scale*q.k) only while scale*groups stays moderate (see _choose_shift)."""
    check(fcsa, (1, 4, 300, 64), (1, 4, 300, 64), torch.float16, seed=groups, groups=groups, scale=scale)


def test_merged_batch_heads(fcsa):
    check(fcsa, (6, 260, 64), (6, 260, 64), torch.bfloat16, seed=7, causal=True)


def test_no_l2norm(fcsa):
    check(fcsa, (1, 2, 200, 64), (1, 2, 200, 64), torch.bfloat16, seed=8, amp=0.2, l2norm_qk=False, scale=1)


def test_l2norm_groups_alias(fcsa):
    q, k, v, _, _ = make_inputs((1, 2, 130, 64), (1, 2, 130, 64), torch.float16, 9)
    a = fcsa.flash_cosine_sim_attention(q.cuda(), k.cuda(), v.cuda(), groups=4)
    b = fcsa.flash_cosine_sim_attention(q.cuda(), k.cuda(), v.cuda(), l2norm_groups=4)
    assert torch.equal(a, b)


def test_strided_inputs_as_in_transformer(fcsa):
    """transformer.py hands the op 'b n (h d) -> b h n d' views (reference transformer.py:100)."""
    g = torch.Generator().manual_seed(10)
    dt = torch.bfloat16
    base = [torch.randn(2, 300, 4 * 64, generator=g).to(dt) for _ in range(3)]
    views = [t.view(2, 300, 4, 64).permute(0, 2, 1, 3) for t in base]
    assert not views[0].is_contiguous()
    qd, kd, vd = (t.cuda().view(2, 300, 4, 64).permute(0, 2, 1, 3).requires_grad_() for t in base)
    do = torch.randn(2, 4, 300, 64, generator=g).to(dt)
    o = fcsa.flash_cosine_sim_attention(qd, kd, vd, causal=True)
    o.backward(do.cuda())
    ref = oracle.attention(*(t.float().numpy() for t in views), causal=True, d_out=do.float().numpy())
    assert rel_err(o, ref[0]) <= TOL_OUT[dt]
    for t, r in zip((qd, kd, vd), ref[1:]):
        assert rel_err(t.grad, r) <= TOL_GRAD[dt]


def test_sum_backward_broadcast_grad(fcsa):
    """`o.sum().backward()` (reference tests and benchmark helper) delivers a stride-0 grad."""
    q, k, v, _, _ = make_inputs((1, 2, 150, 64), (1, 2, 150, 64), torch.float16, 11)
    qd, kd, vd = (t.cuda().requires_grad_() for t in (q, k, v))
    fcsa.flash_cosine_sim_attention(qd, kd, vd).sum().backward()
    ref = oracle.attention(q.float().numpy(), k.float().numpy(), v.float().numpy(),
                           d_out=np.ones((1, 2, 150, 64)))
    for t, r in zip((qd, kd, vd), ref[1:]):
        assert rel_err(t.grad, r) <= TOL_GRAD[torch.float16]


def test_expanded_stride0_views(fcsa):
    """ADVICE r1 (high): head-expanded keys/values and a head-expanded upstream gradient (what `o.sum(1)`
    style reductions hand back: strides (N*D, 0, D, 1)) are stride-0 views a TMA tensor map cannot
    express - they must be materialised, never mis-addressed."""
    dt = torch.bfloat16
    g = torch.Generator().manual_seed(21)
    B, H, N = 3, 4, 200
    q = torch.randn(B, H, N, 64, generator=g).to(dt)
    k1, v1 = (torch.randn(B, N, 64, generator=g).to(dt) for _ in range(2))
    d1 = torch.randn(B, N, 64, generator=g).to(dt)
    qd = q.cuda().requires_grad_()
    kd, vd = k1.cuda().requires_grad_(), v1.cuda().requires_grad_()
    ke, ve = kd[:, None].expand(-1, H, -1, -1), vd[:, None].expand(-1, H, -1, -1)      # stride 0 over heads
    assert ke.stride(1) == 0
    o = fcsa.flash_cosine_sim_attention(qd, ke, ve, causal=True)
    do = d1.cuda()[:, None].expand(-1, H, -1, -1)                                       # stride-0 grad
    o.backward(do)
    kf, vf, df = (t[:, None].expand(-1, H, -1, -1).float().numpy() for t in (k1, v1, d1))
    ref = oracle.attention(q.float().numpy(), kf, vf, causal=True, d_out=df, round_qk="bf16")
    assert rel_err(o, ref[0]) <= TOL_OUT[dt]
    assert rel_err(qd.grad, ref[1]) <= TOL_GRAD[dt]
    assert rel_err(kd.grad, ref[2].sum(1)) <= TOL_GRAD[dt]        # expand's backward sums over heads
    assert rel_err(vd.grad, ref[3].sum(1)) <= TOL_GRAD[dt]


def test_c_abi_refuses_stride0_tensor(fcsa):
    """Behind the C ABI a stride-0 dimension of extent > 1 is an error, not a silent dense stride."""
    from flash_cosine_sim_attention_b200 import _abi
    lib = _abi.load()
    x = torch.zeros(2, 4, 128, 64, dtype=torch.bfloat16, device="cuda")
    p = _abi.FcsaProblem()
    p.dtype, p.batch, p.heads, p.kv_heads, p.seq_q, p.seq_k, p.head_dim = _abi.FCSA_BF16, 2, 4, 4, 128, 128, 64
    p.scale, p.shift = 8.0, 8.0
    good = _abi.FcsaTensor(x.data_ptr(), x.stride(0), x.stride(1), x.stride(2))
    bad = _abi.FcsaTensor(x.data_ptr(), x.stride(0), 0, x.stride(2))
    rc = lib.fcsa_forward(_abi.ref(p), _abi.ref(good), _abi.ref(bad), _abi.ref(good), _abi.ref(good), None, None)
    assert rc == _abi.FCSA_ERR_INVALID and b"stride-0" in lib.fcsa_last_error()
    # the backward's maps say the same, naming the operand: here a head-expanded d_o
    inv_l = torch.ones(2, 4, 128, dtype=torch.float32, device="cuda")
    grads = [torch.empty_like(x) for _ in range(3)]
    tg = [_abi.FcsaTensor(t.data_ptr(), t.stride(0), t.stride(1), t.stride(2)) for t in grads]
    ws = torch.empty(lib.fcsa_backward_workspace_bytes(_abi.ref(p)), dtype=torch.uint8, device="cuda")
    zs = torch.zeros(lib.fcsa_backward_zeroed_bytes(_abi.ref(p)), dtype=torch.uint8, device="cuda")
    rc = lib.fcsa_backward(_abi.ref(p), *([_abi.ref(good)] * 4), _abi.ref(bad), inv_l.data_ptr(),
                           *(_abi.ref(t) for t in tg), ws.data_ptr(), ws.numel(), zs.data_ptr(), zs.numel(), None)
    err = lib.fcsa_last_error()
    assert rc == _abi.FCSA_ERR_INVALID and b"stride-0" in err and err.startswith(b"d_o:")
    torch.cuda.synchronize()
    assert int(zs.count_nonzero()) == 0           # the zeroed workspace is left zero


def test_zeroed_workspace_is_left_clean_across_shapes(fcsa):
    """The fp32 dq accumulator lives in a persistent buffer that every backward must leave zero (the
    finish pass converts and clears it).  Interleave shapes, head dims, masks and repeat: any dirt left
    behind shows up as a wrong dq in a later call."""
    cases = [((2, 3, 300, 64), dict(causal=True)), ((1, 2, 130, 128), dict(causal=True)),
             ((1, 2, 700, 64), dict()), ((2, 3, 300, 64), dict(causal=True)),
             ((1, 2, 64, 128), dict()), ((1, 4, 456, 64), dict(causal=True))]
    for rep in range(2):
        for i, (shape, kw) in enumerate(cases):
            check(fcsa, shape, shape, torch.bfloat16, seed=100 + i, **kw)
    m = __import__("flash_cosine_sim_attention_b200.flash_cosine_sim_attention", fromlist=["x"])
    torch.cuda.synchronize()
    # white box: the extension's buffers are not reachable from Python, so check through one more call whose
    # exact answer is known to be zero wherever nothing contributes (causal, more queries than keys)
    check(fcsa, (1, 2, 456, 64), (1, 2, 200, 64), torch.bfloat16, seed=7, causal=True)


def test_release_workspaces(fcsa):
    check(fcsa, (1, 2, 256, 64), (1, 2, 256, 64), torch.bfloat16, seed=71, causal=True)
    assert fcsa.release_workspaces() > 0
    assert fcsa.release_workspaces() == 0
    check(fcsa, (1, 2, 256, 64), (1, 2, 256, 64), torch.bfloat16, seed=72, causal=True)      # re-created on demand


def test_many_batch_heads_merged(fcsa):
    """ADVICE r1: batch*heads > 65535 (merged 3-D layout) must run forward AND backward."""
    dt = torch.float16
    g = torch.Generator().manual_seed(22)
    BH, N = 66000, 16
    q, k, v, do = (torch.randn(BH, N, 64, generator=g).to(dt) for _ in range(4))
    qd, kd, vd = (t.cuda().requires_grad_() for t in (q, k, v))
    o = fcsa.flash_cosine_sim_attention(qd, kd, vd, causal=True)
    o.backward(do.cuda())
    sl = slice(65530, 65560)                      # across the old grid.y limit
    ref = oracle.attention(q[sl].float().numpy(), k[sl].float().numpy(), v[sl].float().numpy(), causal=True,
                           d_out=do[sl].float().numpy(), round_qk="f16")
    assert rel_err(o[sl], ref[0]) <= TOL_OUT[dt]
    for t, r in zip((qd, kd, vd), ref[1:]):
        assert rel_err(t.grad[sl], r) <= TOL_GRAD[dt]
    assert torch.isfinite(qd.grad).all()


@pytest.mark.parametrize("shape", [(2, 300, 520, 260), (1, 1500, 300, 300), (3, 200, 16, 1024), (1, 700, 700, 300)])
def test_persistent_ctas_many_short_work_items(fcsa, shape):
    """Many short work items, including query blocks with no visible key (causal, more queries than keys: items
    without any key tile) and half-empty query blocks."""
    dt = torch.bfloat16
    B, H, Nq, Nk = shape
    g = torch.Generator().manual_seed(41)
    q, do = (torch.randn(B, H, Nq, 64, generator=g).to(dt) for _ in range(2))
    k, v = (torch.randn(B, H, Nk, 64, generator=g).to(dt) for _ in range(2))
    qd, kd, vd = (t.cuda().requires_grad_() for t in (q, k, v))
    for _ in range(2):                                 # twice: the zeroed workspace must come back clean
        for t in (qd, kd, vd):
            t.grad = None
        o = fcsa.flash_cosine_sim_attention(qd, kd, vd, causal=True)
        o.backward(do.cuda())
        torch.cuda.synchronize()
    for hh in (0, H // 2, H - 1):
        sl = (slice(B - 1, B), slice(hh, hh + 1))
        ref = oracle.attention(q[sl].float().numpy(), k[sl].float().numpy(), v[sl].float().numpy(), causal=True,
                               d_out=do[sl].float().numpy(), round_qk="bf16", empty_rows="zero")
        assert rel_err(o[sl], ref[0]) <= TOL_OUT[dt]
        for t, r in zip((qd, kd, vd), ref[1:]):
            assert rel_err(t.grad[sl], r) <= TOL_GRAD[dt]
    assert torch.isfinite(qd.grad).all() and torch.isfinite(kd.grad).all()


def test_two_streams_have_their_own_workspaces(fcsa):
    """Backward calls on two streams must not share the persistent accumulator."""
    dt = torch.bfloat16
    q, k, v, do, _ = make_inputs((2, 2, 384, 64), (2, 2, 384, 64), dt, 23)
    ref = oracle.attention(q.float().numpy(), k.float().numpy(), v.float().numpy(), causal=True,
                           d_out=do.float().numpy(), round_qk="bf16")
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    grads = []
    torch.cuda.synchronize()
    for s in streams:
        with torch.cuda.stream(s):
            qd, kd, vd = (t.cuda().requires_grad_() for t in (q, k, v))
            for _ in range(3):
                qd.grad = None
                o = fcsa.flash_cosine_sim_attention(qd, kd, vd, causal=True)
                o.backward(do.cuda())
            grads.append(qd.grad)
    torch.cuda.synchronize()
    for gq in grads:
        assert rel_err(gq, ref[1]) <= TOL_GRAD[dt]


def test_cuda_graph_capture_of_a_training_step(fcsa):
    """The whole fwd+bwd (5 launches with programmatic dependent launch, persistent workspaces, no host
    synchronisation anywhere) can be captured in a CUDA graph and replayed on new data - the launch-bound
    regime of small problems."""
    dt = torch.bfloat16
    g = torch.Generator().manual_seed(51)
    shape = (2, 4, 384, 64)
    sq, sk, sv, sdo = (torch.zeros(shape, dtype=dt, device="cuda") for _ in range(4))
    sq.requires_grad_(), sk.requires_grad_(), sv.requires_grad_()

    def step():
        o = fcsa.flash_cosine_sim_attention(sq, sk, sv, causal=True)
        return (o,) + torch.autograd.grad(o, (sq, sk, sv), sdo)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            step()                                         # warm-up: workspaces of this stream exist before capture
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=side):
        outs = step()
    for trial in range(2):
        q, k, v, do = (torch.randn(shape, generator=g).to(dt) for _ in range(4))
        with torch.no_grad():
            sq.copy_(q); sk.copy_(k); sv.copy_(v); sdo.copy_(do)
        graph.replay()
        torch.cuda.synchronize()
        ref = oracle.attention(q.float().numpy(), k.float().numpy(), v.float().numpy(), causal=True,
                               d_out=do.float().numpy(), round_qk="bf16")
        assert rel_err(outs[0], ref[0]) <= TOL_OUT[dt]
        for got, want in zip(outs[1:], ref[1:]):
            assert rel_err(got, want) <= TOL_GRAD[dt]


def test_fully_masked_rows_give_zero(fcsa):
    """Documented divergence from the naive formulation (reference cu:1239): o = 0, grads = 0."""
    q, k, v, do, _ = make_inputs((2, 2, 70, 64), (2, 2, 90, 64), torch.bfloat16, 12)
    mask = torch.ones(2, 90, dtype=torch.bool)
    mask[1] = False
    qd, kd, vd = (t.cuda().requires_grad_() for t in (q, k, v))
    o = fcsa.flash_cosine_sim_attention(qd, kd, vd, mask=mask.cuda())
    o.backward(do.cuda())
    assert torch.all(o[1] == 0) and torch.isfinite(o).all()
    for t in (qd, kd, vd):
        assert torch.isfinite(t.grad).all() and torch.all(t.grad[1] == 0)


def test_forward_only_under_no_grad_and_ragged_generate_lengths(fcsa):
    """`generate` calls the op with a different, unaligned N every step (transformer.py:167-181)."""
    for n in (1, 7, 64, 65, 255, 256, 257):
        check(fcsa, (1, 2, n, 64), (1, 2, n, 64), torch.float16, seed=n, grads=False, causal=True)


def test_reference_extension_surface(fcsa):
    """forward / backward / debug with the reference's pybind signatures (cu:1630, 1752, 1921)."""
    from importlib import import_module
    m = import_module("flash_cosine_sim_attention_b200.flash_cosine_sim_attention")
    q, k, v, do, _ = make_inputs((1, 2, 140, 64), (1, 2, 140, 64), torch.float16, 13)
    qn, kn = fcsa.l2norm_tensors(q.cuda(), k.cuda())
    qn.requires_grad_()
    o, inv_l, should_backwards = m.forward(qn, kn, v.cuda(), None, None, False, 8.0, True)
    assert should_backwards and inv_l.shape == (1, 2, 140) and inv_l.dtype == torch.float32
    dq, dk, dv, db = m.backward(do.cuda(), o, inv_l, qn.detach(), kn, v.cuda(), None, None, False, 8.0, True)
    assert db is None and dq.shape == q.shape
    qn64, kn64 = (oracle.l2norm(t.float().numpy())[0] for t in (q, k))
    ref = oracle.attention(qn.detach().float().cpu().numpy(), kn.float().cpu().numpy(), v.float().numpy(),
                           causal=True, l2norm_qk=False, d_out=do.float().numpy())
    assert rel_err(o, ref[0]) <= TOL_OUT[torch.float16]
    assert rel_err(dq, ref[1]) <= TOL_GRAD[torch.float16]
    assert np.abs(qn.detach().float().cpu().numpy() - qn64).max() < 1e-3
    assert m.debug() > 0


def test_reference_named_extension_module(fcsa):
    """The torch extension carries the reference's module name (version.py:3) and pybind surface
    (cu:1928-1933): `import flash_cosine_sim_attention_cuda_0_1_40` gives forward/backward/debug with the
    reference's positional signatures - what the reference's own flash_cosine_sim_attention.py binds."""
    import importlib
    import sys
    fcsa.debug()                                            # loads + registers the module
    m = importlib.import_module("flash_cosine_sim_attention_cuda_0_1_40")
    assert m.__file__.endswith(".so") and "flash_cosine_sim_attention_b200" in m.__file__
    q, k, v, do, mask = make_inputs((2, 2, 100, 64), (2, 2, 100, 64), torch.float16, 31, mask_p=0.3)
    qn, kn = (torch.nn.functional.normalize(t.float(), dim=-1).half().cuda() for t in (q, k))
    qn.requires_grad_()
    bias = (torch.randn(2, 100, 100) * 0.5).half().cuda().requires_grad_()
    o, l, should = m.forward(qn, kn, v.cuda(), mask.cuda(), bias, False, 8.0, False)
    assert should is True and o.shape == q.shape and l.shape == (2, 2, 100)
    dq, dk, dv, db = m.backward(do.cuda(), o, l, qn.detach(), kn, v.cuda(), mask.cuda(), bias, False, 8.0, False)
    ref = oracle.attention(qn.detach().float().cpu().numpy(), kn.float().cpu().numpy(), v.float().numpy(),
                           mask=mask.numpy(), attn_bias=bias.detach().float().cpu().numpy(), l2norm_qk=False,
                           d_out=do.float().numpy(), empty_rows="zero")
    assert rel_err(o, ref[0]) <= TOL_OUT[torch.float16]
    for got, want in zip((dq, dk, dv, db), ref[1:5]):
        assert rel_err(got, want) <= 2 * TOL_GRAD[torch.float16]
    assert db.dtype == bias.dtype and db.shape == bias.shape
    assert isinstance(m.debug(), int)


def test_l2norm_tensors_kernel_and_its_backward(fcsa):
    g = torch.Generator().manual_seed(14)
    x = torch.randn(2, 3, 77, 64, generator=g).to(torch.bfloat16)
    dy = torch.randn(2, 3, 77, 64, generator=g).to(torch.bfloat16)
    for groups in (1, 2, 8, 16):
        xd = x.cuda().requires_grad_()
        (y,) = fcsa.l2norm_tensors(xd, groups=groups)
        y.backward(dy.cuda())
        assert rel_err(y, oracle.l2norm(x.float().numpy(), groups)[0]) < 5e-3
        # the kernel differentiates through the ROUNDED y it stored, like autograd on 16-bit tensors
        assert rel_err(xd.grad, oracle.l2norm_backward(dy.float().numpy(), x.float().numpy(), groups)) < 2e-2


# ---- float32 inputs and head dim 16 (reference: Float dispatched fwd + bwd, cu:1702-1703 / 1832-1834; the f32 half
# ---- of its grid, tests/test.py:33-35).  north_star tolerance for f32: 1e-3 - against the UNROUNDED oracle.
@pytest.mark.parametrize("causal,mask", [(True, False), (False, True), (False, False)])
@pytest.mark.parametrize("seq_len", [63, 127])
@pytest.mark.parametrize("dim_head", [16, 32, 64, 96, 128])
@pytest.mark.parametrize("single_head_kv", [False, True])
def test_reference_grid_float32(fcsa, causal, mask, seq_len, dim_head, single_head_kv):
    qs = (2, 4, seq_len, dim_head)
    kvs = (2, seq_len, dim_head) if single_head_kv else qs
    check(fcsa, qs, kvs, torch.float32, seed=seq_len + dim_head, mask_p=0.5 if mask else None, causal=causal)


def test_float32_value_and_gradient_ranges(fcsa):
    """v and d_out far outside fp16's exponent range: the power-of-two scaling around the fp16 kernels
    must make the result independent of their magnitude."""
    g = torch.Generator().manual_seed(41)
    q, k = (torch.randn(1, 2, 200, 64, generator=g) for _ in range(2))
    v0, d0 = (torch.randn(1, 2, 200, 64, generator=g) for _ in range(2))
    for vs, ds in ((1.0, 1.0), (3e6, 2e-9), (1e-7, 4e5)):
        v, do = v0 * vs, d0 * ds
        qd, kd, vd = (t.cuda().requires_grad_() for t in (q, k, v))
        o = fcsa.flash_cosine_sim_attention(qd, kd, vd, causal=True)
        assert o.dtype == torch.float32
        o.backward(do.cuda())
        ref = oracle.attention(q.numpy(), k.numpy(), v.numpy(), causal=True, d_out=do.numpy())
        assert rel_err(o, ref[0]) <= TOL_OUT[torch.float32]
        for t, r in zip((qd, kd, vd), ref[1:]):
            assert rel_err(t.grad, r) <= TOL_GRAD[torch.float32]


@pytest.mark.parametrize("scale,groups,tol_o,tol_g", [(4, 2, 1e-3, 2e-3), (8, 2, 1e-2, 2e-2)])
def test_float32_attn_bias_and_groups(fcsa, scale, groups, tol_o, tol_g):
    """scale*groups <= 10: fp16 kernels (north_star's 1e-3); above: exp(scale*q.k) needs more exponent range than
    fp16 has, the float32 path switches to the bf16 kernels (bf16 tolerances) instead of producing garbage rows."""
    import warnings
    g = torch.Generator().manual_seed(42)
    q, k, v, do = (torch.randn(2, 3, 90, 64, generator=g) for _ in range(4))
    bias = torch.randn(3, 90, 90, generator=g)
    qd, kd, vd, bd = (t.cuda().requires_grad_() for t in (q, k, v, bias))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        o = fcsa.flash_cosine_sim_attention(qd, kd, vd, attn_bias=bd, causal=True, groups=groups, scale=scale)
    o.backward(do.cuda())
    ref = oracle.attention(q.numpy(), k.numpy(), v.numpy(), attn_bias=bias.numpy(), causal=True, groups=groups,
                           scale=scale, d_out=do.numpy())
    assert rel_err(o, ref[0]) <= tol_o
    for t, r in zip((qd, kd, vd, bd), ref[1:5]):
        assert t.grad.dtype == torch.float32
        assert rel_err(t.grad, r) <= tol_g


def test_no_unfused_fallback_is_reachable(fcsa):
    """Unsupported inputs raise; nothing routes to plain_cosine_sim_attention or the CPU."""
    x = torch.zeros(1, 2, 8, 64)
    with pytest.raises(RuntimeError):
        fcsa.flash_cosine_sim_attention(x, x, x)                                   # CPU tensors
    y = torch.zeros(1, 2, 8, 72, device="cuda", dtype=torch.float64)
    with pytest.raises(TypeError):
        fcsa.flash_cosine_sim_attention(y, y, y)                                   # float64
    z = torch.zeros(1, 2, 8, 132, device="cuda", dtype=torch.float16)
    with pytest.raises(NotImplementedError):
        fcsa.flash_cosine_sim_attention(z, z, z)                                   # head dim not a multiple of 8
    import inspect
    src = inspect.getsource(fcsa.flash_cosine_sim_attention)
    assert "plain_cosine_sim_attention(" not in src


# ---- BASELINE.json configs ------------------------------------------------------------------------
def test_config2_self_attn_1x8x1024x64_bf16_fwd(fcsa):
    check(fcsa, (1, 8, 1024, 64), (1, 8, 1024, 64), torch.bfloat16, seed=2, grads=False)


def test_config4_cross_attn_mask_single_head_kv_grouped(fcsa):
    check(fcsa, (1, 8, 1024, 64), (1, 2048, 64), torch.bfloat16, seed=4, mask_p=0.25, groups=2)


def _slice_check(fcsa, shape, dtype, slices, grads=True):
    """Full-size run on the GPU; oracle on a few (batch, head) slices (each is an independent
    attention problem, reference cu:1091-1092)."""
    q, k, v, do, _ = make_inputs(shape, shape, dtype, seed=3)
    grads = grads and shape[-1] in BWD_HEAD_DIMS
    qd, kd, vd = (t.cuda().requires_grad_(grads) for t in (q, k, v))
    o = fcsa.flash_cosine_sim_attention(qd, kd, vd, causal=True)
    if grads:
        o.backward(do.cuda())
    for b, h in slices:
        sl = lambda t: t[b:b + 1, h:h + 1].float().numpy()
        ref = oracle.attention(sl(q), sl(k), sl(v), causal=True, d_out=sl(do) if grads else None)
        ref = ref if grads else (ref,)
        assert rel_err(o[b:b + 1, h:h + 1], ref[0]) <= TOL_OUT[dtype]
        if grads:
            for t, r in zip((qd, kd, vd), ref[1:]):
                assert rel_err(t.grad[b:b + 1, h:h + 1], r) <= TOL_GRAD[dtype]
        ts = lambda t: t[b:b + 1, h:h + 1]
        got = {"o": ts(o)}
        if grads:
            got.update(dq=ts(qd.grad), dk=ts(kd.grad), dv=ts(vd.grad))
        bound_check(dtype, got, ts(q), ts(k), ts(v), ts(do) if grads else None, causal=True)
    return qd, kd, vd, o


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_config3_causal_4x8x4096x64_fwd_bwd(fcsa, dtype):
    qd, kd, vd, o = _slice_check(fcsa, (4, 8, 4096, 64), dtype, [(0, 0), (3, 7)])
    # size-independent properties at full size
    ones = torch.ones_like(vd)
    o1 = fcsa.flash_cosine_sim_attention(qd.detach(), kd.detach(), ones, causal=True)
    assert (o1.float() - 1).abs().max() < 1e-2             # rows are convex combinations of v
    o2 = fcsa.flash_cosine_sim_attention(qd.detach(), kd.detach(), vd.detach(), causal=True)
    assert torch.equal(o2, o.detach())                      # forward is deterministic
    # causality: perturbing the last key/value must leave all earlier rows untouched
    k2, v2 = kd.detach().clone(), vd.detach().clone()
    k2[:, :, -1] += 1
    v2[:, :, -1] += 1
    o3 = fcsa.flash_cosine_sim_attention(qd.detach(), k2, v2, causal=True)
    assert torch.equal(o3[:, :, :-1], o.detach()[:, :, :-1])


def _f64_attention_on_gpu(q, k, v, do, scale=8.0):
    """The oracle formula (py:75-126) for ONE (batch, head), causal, evaluated in float64 on the GPU with autograd;
    q, k are l2-normalised in float64 and rounded to the input dtype first, as py:64 does.  Test infrastructure."""
    dt = q.dtype
    q64, k64, v64 = (t.double().detach().requires_grad_() for t in (q, k, v))
    qn = torch.nn.functional.normalize(q64, dim=-1)
    kn = torch.nn.functional.normalize(k64, dim=-1)
    qn = qn + (qn.to(dt).double() - qn).detach()          # value rounded to the storage dtype, gradient straight through
    kn = kn + (kn.to(dt).double() - kn).detach()
    sim = (qn @ kn.t()) * scale
    n = sim.shape[0]
    sim = sim.masked_fill(torch.ones(n, n, dtype=torch.bool, device=q.device).triu(1), float("-inf"))
    o = sim.softmax(dim=-1) @ v64
    o.backward(do.double())
    return o.detach(), q64.grad, k64.grad, v64.grad


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_config3_every_batch_head_against_float64_on_gpu(fcsa, dtype):
    """ALL 32 (batch, head) problems of the metric configuration, outputs and the three gradients, against a float64
    evaluation of the oracle formula on the same GPU (the numpy oracle checks two of them in
    test_config3_causal_4x8x4096x64_fwd_bwd; 32 x 4096^2 float64 similarity matrices are too slow on the host)."""
    g = torch.Generator(device="cuda").manual_seed(33)
    q, k, v, do = (torch.randn(4, 8, 4096, 64, generator=g, device="cuda").to(dtype) for _ in range(4))
    qd, kd, vd = (t.clone().requires_grad_() for t in (q, k, v))
    o = fcsa.flash_cosine_sim_attention(qd, kd, vd, causal=True)
    o.backward(do)
    worst = {"o": 0.0, "dq": 0.0, "dk": 0.0, "dv": 0.0}
    for b in range(4):
        for h in range(8):
            ref = _f64_attention_on_gpu(q[b, h], k[b, h], v[b, h], do[b, h])
            for name, got, want in zip(worst, (o[b, h], qd.grad[b, h], kd.grad[b, h], vd.grad[b, h]), ref):
                err = float((got.double() - want).abs().max() / want.abs().max())
                worst[name] = max(worst[name], err)
    for name, err in worst.items():
        tol = TOL_OUT[dtype] if name == "o" else TOL_GRAD[dtype]
        record(dtype, f"{name}@C3x32", err, tol)
        assert err <= tol, (name, err)
    # every element of all 32 problems under the element-wise bound, its float64 reference computed on the GPU
    bound_check(dtype, {"o": o, "dq": qd.grad, "dk": kd.grad, "dv": vd.grad}, q, k, v, do, causal=True)


def test_config5_long_context_slice_16384x128(fcsa):
    """One rank's share of config 5 is (1, 16, 16384, 128); two heads checked against the oracle."""
    _slice_check(fcsa, (1, 2, 16384, 128), torch.bfloat16, [(0, 1)], grads=True)
