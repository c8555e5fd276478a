"""GPU tests of context parallelism (`context_parallel.py`) and of the sharded operator (`sharding.py`) on the fused
kernels (run on an H100 with `pytest -m gpu`).  W ranks run as W processes on the current CUDA device, joined by a gloo
process group (gloo stages CUDA tensors through the host for its all-gather and all-reduce), so no second GPU is
needed.  The NCCL branch of the collectives is what tests/gpu_sharding_nccl.py runs on two or more GPUs.

Context parallelism uses the kernels in a way no other caller does: one forward per key block returning an fp32
partial o (out_f32) and 1/l, and one backward per block with the MERGED 1/l and fp32 o, so a block's P rows do not sum
to 1 and delta comes from the merged o.

Harness: one `torch.multiprocessing.spawn` per world size for the whole module.  Every rank builds the full tensors
from a seeded CPU generator (identical on every rank), slices its block, runs every case of its world size in turn
and saves its block of o and its gradients under a temporary directory.  The tests below load them per case and
judge them in this process against the float64 reference of the whole problem (tests/elementwise_bounds.py): the
element-wise bound at C = 2 (pinned on the CPU by test_elementwise_bounds.test_emulated_context_parallel_within_bound)
on o, dq, dk and dv, and the relative tolerances of test_gpu_parity.py on o and dv, and on dq and dk except for the
aligned families, where one key takes a row and dS = P (dP - delta) cancels (as in test_gpu_logit_range.py).

Context-parallel covering grid (not the full product).  Every input family (Gaussian; aligned0 and one_peak, whose
row peaks often lie in another rank's block; diagonal, peaks in the diagonal block; opposed) runs with both dtypes
at both W in {2, 3}, causal at one W and not at the other.  Every (groups, scale) of its dtype, bf16 (1, 8), (8, 1), (2, 5),
(4, 8), (2, 16) and fp16 (1, 8), (8, 1), (2, 5), (2, 8), runs at both W.  Every family meets both head dims, every
(W, dtype) pair all three local lengths n in {128, 300, 1000} (300: ragged tiles in every block call, the diagonal
block included; 1000: past the forward ring), and the merged 3-D layout (B*H = 6) appears with both dtypes at both W,
causal and not.  At W = 3 causal, rank 1 has a fully visible earlier block, its diagonal block and a skipped later
block.  fp16 at (2, 8) is the shift = scale regime below the overflow threshold, where p of poorly matching keys
flushes to 0 in P V; it runs with every family but the opposed one.  With opposed inputs there, every p of a row is
about exp(-scale (groups + 1)) = e^-24, below fp16's smallest subnormal, so P V and o are 0 and delta = 0 makes dq
wrong: the dense op gives the same (o = 0 on every row), a limit of the fp16 shift, not of this path (DESIGN 6).
l2norm_qk=False runs at scale 1 with Gaussian inputs x 0.2, once per W."""
import contextlib
import importlib
import os
import socket
import traceback
import warnings
from collections import namedtuple
from datetime import timedelta

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import logit_range
from elementwise_bounds import FMT, attention_bounds, check_bound, kernel_shift
from test_gpu_parity import ERRORS, TOL_GRAD, TOL_OUT, fcsa, record, rel_err  # noqa: F401

pytestmark = pytest.mark.gpu

BF16, F16 = torch.bfloat16, torch.float16
FAMILIES = ("gaussian", "aligned0", "one_peak", "diagonal", "opposed")
ALIGNED = ("aligned0", "one_peak", "diagonal")
GS = {BF16: [(1, 8), (8, 1), (2, 5), (4, 8), (2, 16)], F16: [(1, 8), (8, 1), (2, 5), (2, 8)]}
NS = (128, 300, 1000)
TIMEOUT = timedelta(seconds=120)

Cp = namedtuple("Cp", "id W n dtype D causal groups scale l2norm merged family seed")
Sh = namedtuple("Sh", "id qs kvs dtype kw mask presharded seed")


def _cp_cases():
    cases = []
    for W in (2, 3):
        for di, dtype in enumerate((BF16, F16)):
            for j, fam in enumerate(FAMILIES):
                g, s = GS[dtype][(j + W) % len(GS[dtype])]
                if fam == "opposed" and (dtype, g, s) == (F16, 2, 8):
                    g, s = 2, 5                      # p below fp16's subnormals: o = 0 in every kernel (docstring)
                n, D = NS[(j + di + W) % 3], (64, 128)[(j + di) % 2]
                causal, merged = (j + W) % 2 == 1, (j + 2 * di + W) % 3 == 0
                cases.append(Cp(f"w{W}-{FMT[dtype]}-{fam}-n{n}-D{D}-g{g}s{s}-{'causal' if causal else 'full'}"
                                f"{'-bh' if merged else ''}", W, n, dtype, D, causal, g, s, True, merged, fam,
                                100 * W + 10 * di + j))
        dtype, n, D, causal = (BF16, 300, 64, True) if W == 2 else (F16, 128, 128, False)
        cases.append(Cp(f"w{W}-{FMT[dtype]}-no_l2norm-n{n}-D{D}-{'causal' if causal else 'full'}", W, n, dtype, D,
                        causal, 1, 1, False, W == 3, "gaussian", 100 * W + 50))
    return cases


CP_CASES = _cp_cases()

# the sharded operator at W = 2, even splits only (gloo has no all-gather of unequal blocks)
SH_CASES = [
    Sh("batch_gather", (4, 3, 300, 64), (4, 3, 300, 64), BF16, dict(causal=True), False, False, 1),
    Sh("heads_shared_kv_mask", (1, 4, 256, 64), (1, 256, 64), F16, dict(), True, False, 2),
    Sh("heads_gqa", (1, 8, 300, 128), (1, 4, 300, 128), BF16, dict(causal=True, groups=2), False, False, 3),
    Sh("presharded_gather", (4, 2, 200, 128), (4, 2, 200, 128), F16, dict(causal=True), False, True, 4),
]


# ---- inputs: the same on every rank and in this process -------------------------------------------------------------
def cp_inputs(c):
    """Full (2, 3, N, D) q, k, v, dO of a context-parallel case (merged: (6, N, D)), N = W n."""
    N = c.W * c.n
    if c.family == "gaussian":
        g = torch.Generator().manual_seed(c.seed)
        amp = 1.0 if c.l2norm else 0.2
        q, k = (torch.randn(2, 3, N, c.D, generator=g) * amp for _ in range(2))
        v, do = (torch.randn(2, 3, N, c.D, generator=g) for _ in range(2))
        q, k, v, do = (t.to(c.dtype) for t in (q, k, v, do))
    else:
        q, k, v, do, _ = logit_range.dense(c.family, 2, 3, 3, N, N, c.D, c.dtype, causal=c.causal, seed=c.seed)
    if c.merged:
        q, k, v, do = (t.reshape(6, N, c.D) for t in (q, k, v, do))
    return q, k, v, do


def sh_inputs(c):
    g = torch.Generator().manual_seed(c.seed)
    q, do = (torch.randn(c.qs, generator=g).to(c.dtype) for _ in range(2))
    k, v = (torch.randn(c.kvs, generator=g).to(c.dtype) for _ in range(2))
    mask = None
    if c.mask:
        mask = torch.rand((c.qs[0], c.kvs[-2]), generator=g) > 0.3
        mask[:, 0] = True
    return q, k, v, do, mask


# ---- the ranks ----------------------------------------------------------------------------------------------------------
def _run_cp(c, rank):
    from flash_cosine_sim_attention_b200.context_parallel import context_parallel_cosine_sim_attention
    q, k, v, do = cp_inputs(c)
    sl = slice(rank * c.n, (rank + 1) * c.n)
    ql, kl, vl = (t[..., sl, :].contiguous().cuda().requires_grad_() for t in (q, k, v))
    o = context_parallel_cosine_sim_attention(ql, kl, vl, scale=c.scale, groups=c.groups, causal=c.causal,
                                              l2norm_qk=c.l2norm)
    assert o.shape == ql.shape and o.dtype == ql.dtype, (tuple(o.shape), o.dtype)
    o.backward(do[..., sl, :].contiguous().cuda())
    return {"o": o.detach().cpu(), "dq": ql.grad.cpu(), "dk": kl.grad.cpu(), "dv": vl.grad.cpu()}


def _run_sharded(c, rank, world):
    from flash_cosine_sim_attention_b200.sharding import local_shard, sharded_flash_cosine_sim_attention
    q, k, v, do, mask = sh_inputs(c)
    if c.presharded:
        q, k, v, mask = (None if t is None else local_shard(t, rank, world) for t in (q, k, v, mask))
    qd, kd, vd = (t.cuda().requires_grad_() for t in (q, k, v))
    o = sharded_flash_cosine_sim_attention(qd, kd, vd, mask=None if mask is None else mask.cuda(), gather=True,
                                           presharded=c.presharded, **c.kw)
    o.backward(do.cuda())                                        # o is the gathered whole-batch output
    return {"o": o.detach().cpu(), "dq": qd.grad.cpu(), "dk": kd.grad.cpu(), "dv": vd.grad.cpu()}


def _worker(rank, world, port, device, out_dir):
    torch.cuda.set_device(device)
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world,
                            timeout=TIMEOUT)
    try:
        jobs = [(c, lambda c=c: _run_cp(c, rank)) for c in CP_CASES if c.W == world]
        if world == 2:
            jobs += [(c, lambda c=c: _run_sharded(c, rank, world)) for c in SH_CASES]
        for c, job in jobs:
            try:
                res = job()
            except Exception:                               # noqa: BLE001 - reported by the case's test
                res = {"error": traceback.format_exc()}
            torch.save(res, os.path.join(out_dir, f"{c.id}-r{rank}.pt"))
    finally:
        dist.destroy_process_group()


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


@pytest.fixture(scope="module")
def ranks(fcsa, tmp_path_factory):
    """ranks(W, case) -> the W ranks' saved results of the case; one spawn of W processes per world size."""
    dirs = {}

    def get(world, case):
        if world not in dirs:
            d = tmp_path_factory.mktemp(f"world{world}")
            mp.spawn(_worker, args=(world, _free_port(), torch.cuda.current_device(), str(d)), nprocs=world,
                     join=True)
            dirs[world] = d
        res = [torch.load(os.path.join(dirs[world], f"{case.id}-r{r}.pt")) for r in range(world)]
        for r, x in enumerate(res):
            assert "error" not in x, f"rank {r}:\n{x['error']}"
        return res
    return get


# ---- judgement ----------------------------------------------------------------------------------------------------------
def judge(tag, dtype, got, q, k, v, do, rel=("o", "dq", "dk", "dv"), scale=8, groups=1, l2norm_qk=True, **kw):
    """Every output in `got` under the element-wise bound at C = 2, those in `rel` also under the relative tolerance;
    the worst values are recorded under '<tag> <name>' and '<tag> <name>/bound'."""
    fmt = FMT[dtype]
    ref, bound = attention_bounds(q, k, v, do, scale=scale, groups=groups, l2norm_qk=l2norm_qk,
                                  round_qk=fmt if l2norm_qk else None, fmt=fmt,
                                  shift=kernel_shift(fmt, scale, groups, l2norm_qk), device="cuda", **kw)
    for name, t in got.items():
        if name in rel:
            tol = (TOL_OUT if name == "o" else TOL_GRAD)[dtype]
            e = rel_err(t, ref[name].cpu().numpy())
            record(dtype, f"{tag} {name}", e, tol)
            assert e <= tol, (name, e, tol)
        try:
            w = check_bound(name, t, ref, bound, fmt)
        except AssertionError:
            record(dtype, f"{tag} {name}/bound", float("inf"), 1.0)
            raise
        record(dtype, f"{tag} {name}/bound", w, 1.0)


# ---- 1. context parallelism ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", CP_CASES, ids=[c.id for c in CP_CASES])
def test_context_parallel(ranks, case):
    res = ranks(case.W, case)
    got = {name: torch.cat([r[name] for r in res], dim=-2) for name in ("o", "dq", "dk", "dv")}
    q, k, v, do = cp_inputs(case)
    rel = ("o", "dv") if case.family in ALIGNED else ("o", "dq", "dk", "dv")
    judge("cp", case.dtype, got, q, k, v, do, rel=rel, scale=case.scale, groups=case.groups,
          l2norm_qk=case.l2norm, causal=case.causal)


# ---- 2. the sharded operator --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", SH_CASES, ids=[c.id for c in SH_CASES])
def test_sharded(fcsa, ranks, case):
    """Every rank's gathered o under the bound and bitwise equal to the unsharded fused op; the gradients summed over
    the ranks (shared keys / values: one rank's, the all-reduce has summed them) under the bound, and dk, dv of the
    MHA splits bitwise equal to the unsharded op's."""
    res = ranks(2, case)
    q, k, v, do, mask = sh_inputs(case)
    if case.presharded:
        grads = {n: torch.cat([r[n] for r in res]) for n in ("dq", "dk", "dv")}
    else:
        grads = {n: res[0][n] + res[1][n] for n in ("dq", "dk", "dv")}
    if len(case.kvs) == 3:
        for n in ("dk", "dv"):
            assert torch.equal(res[0][n], res[1][n]), n
            grads[n] = res[0][n]
    qd, kd, vd = (t.cuda().requires_grad_() for t in (q, k, v))
    o = fcsa.flash_cosine_sim_attention(qd, kd, vd, mask=None if mask is None else mask.cuda(), **case.kw)
    o.backward(do.cuda())
    for r in res:
        assert torch.equal(r["o"], o.detach().cpu())
    if len(case.kvs) == 4 and case.kvs[1] == case.qs[1]:
        assert torch.equal(grads["dk"], kd.grad.cpu()) and torch.equal(grads["dv"], vd.grad.cpu())
    kw = dict(case.kw)
    if mask is not None:
        kw["mask"] = mask
    for r in res:
        judge("sharded", case.dtype, {"o": r["o"]}, q, k, v, None, **kw)
    judge("sharded", case.dtype, grads, q, k, v, do, **kw)


# ---- 3. one rank in this process: the fp16 overflow warning and the rejections, before any collective ------------------
@contextlib.contextmanager
def world_of_one():
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{_free_port()}", rank=0, world_size=1,
                            timeout=TIMEOUT)
    try:
        yield
    finally:
        dist.destroy_process_group()


SATURATION = [(4, 8, True), (3, 8, True), (2, 16, True), (2, 8, False), (8, 1, False), (1, 10, False)]


@pytest.mark.parametrize("groups,scale,warns", SATURATION)
def test_fp16_overflow_warning(fcsa, groups, scale, warns):
    """Warns exactly where the dense op does (test_gpu_logit_range.test_fp16_overflow_dense).  Groups of 3 cannot
    divide head dim 64 or 128: the warning still comes, before the l2norm refuses the groups."""
    from flash_cosine_sim_attention_b200.context_parallel import context_parallel_cosine_sim_attention
    m = importlib.import_module("flash_cosine_sim_attention_b200.flash_cosine_sim_attention")
    assert m._fp16_overflows(F16, scale, groups, True) == warns
    q, k, v, _, _ = logit_range.dense("aligned0.3", 1, 2, 2, 128, 128, 64, F16, seed=0)
    m._warned.discard("f16-overflow")
    with world_of_one(), warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        call = lambda: context_parallel_cosine_sim_attention(q.cuda(), k.cuda(), v.cuda(), scale=scale, groups=groups)
        if groups == 3:
            with pytest.raises(AssertionError, match="groups must divide"):
                call()
        else:
            assert torch.isfinite(call()).all()
    assert sum("exceeds fp16's maximum" in str(x.message) for x in w) == (1 if warns else 0)


@pytest.mark.parametrize("dtype,D,exc,match", [(torch.float32, 64, TypeError, "float16 or all bfloat16"),
                                               (BF16, 96, NotImplementedError, "64 or 128"),
                                               (F16, 32, NotImplementedError, "64 or 128")])
def test_rejected_before_any_collective(fcsa, monkeypatch, dtype, D, exc, match):
    from flash_cosine_sim_attention_b200.context_parallel import context_parallel_cosine_sim_attention

    def collective(*args, **kwargs):
        raise AssertionError("a collective ran before the arguments were checked")
    monkeypatch.setattr(dist, "all_gather", collective)
    g = torch.Generator().manual_seed(D)
    q, k, v = (torch.randn(1, 2, 64, D, generator=g).to(dtype).cuda() for _ in range(3))
    with world_of_one(), pytest.raises(exc, match=match):
        context_parallel_cosine_sim_attention(q, k, v, causal=True)


def test_report_worst(capsys):
    """Prints the worst recorded values of this file (relative error, and err / (C u M) under '/bound')."""
    with capsys.disabled():
        for key in sorted(ERRORS):
            if ":cp " in key or ":sharded " in key:
                e = ERRORS[key]
                print(f"\n  {key:24s} {e['max_err']:.3e}   (limit {e['tol']:g})", end="")
