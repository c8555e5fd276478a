"""GPU parity of the D = 64 backward's 192-key work items (three key warpgroups, one dQ tile per query tile and CTA),
judged element-wise against the float64 reference (tests/elementwise_bounds.py, C = 2) with the relative-to-max
tolerances next to it.

The key lengths put the end of the keys at every warpgroup of a work item: 63 / 64 / 65 keys leave one warpgroup with
keys, 191 / 192 / 193 three, then one, 383 / 385 a full item and a short last one, 4096 a last item of 64 keys.  Causal
problems with Nq != Nk move the diagonal against the items both ways; the window moves both ends of each
warpgroup's query-tile range."""
import pytest
import torch

from test_gpu_gqa import loop_batch
from test_gpu_parity import fcsa  # noqa: F401
from test_gpu_varlen import cu_of, make_packed, run_varlen, seq_check
from test_gpu_window import wcheck

gpu = pytest.mark.gpu

NK = [63, 64, 65, 191, 192, 193, 383, 385, 4096]


@gpu
@pytest.mark.parametrize("nk", NK)
@pytest.mark.parametrize("causal", [False, True], ids=["full", "causal"])
def test_dense(fcsa, nk, causal):
    nq = min(nk, 1000)
    wcheck(fcsa, (1, 2, nq, 64), (1, 2, nk, 64), torch.bfloat16, None, seed=nk, causal=causal)


@gpu
@pytest.mark.parametrize("nq,nk", [(100, 385), (385, 100), (64, 193), (193, 64), (700, 191), (191, 700)])
def test_causal_cross(fcsa, nq, nk):
    wcheck(fcsa, (2, 2, nq, 64), (2, 2, nk, 64), torch.bfloat16, None, seed=nq + nk, causal=True)


@gpu
@pytest.mark.parametrize("nk", [65, 193, 385])
def test_gqa_split(fcsa, nk):
    """Grouped-query problems split into one query head per CTA (192-key items, dk / dv summed in fp32); the head-loop
    kernels keep 128-key items."""
    wcheck(fcsa, (1, 6, 200, 64), (1, 2, nk, 64), torch.bfloat16, None, seed=nk + 1, causal=True, path="split")


@gpu
@pytest.mark.parametrize("nk", [65, 193, 385])
def test_gqa_head_loop(fcsa, nk):
    """Grouped-query problems whose groups stay in one CTA (the head-loop kernels, 128-key items)."""
    B = loop_batch(2, nk)
    wcheck(fcsa, (B, 6, 200, 64), (B, 2, nk, 64), torch.bfloat16, None, seed=nk + 1, causal=True, path="loop")


@gpu
@pytest.mark.parametrize("nk", [65, 191, 385])
def test_key_mask(fcsa, nk):
    wcheck(fcsa, (2, 2, 300, 64), (2, 2, nk, 64), torch.bfloat16, None, seed=nk + 2, mask_p=0.3)


@gpu
@pytest.mark.parametrize("window", [1, 40, 65, 200])
@pytest.mark.parametrize("causal", [False, True], ids=["full", "causal"])
@pytest.mark.parametrize("nq,nk", [(385, 385), (200, 450), (450, 200)])
def test_window(fcsa, window, causal, nq, nk):
    wcheck(fcsa, (1, 2, nq, 64), (1, 2, nk, 64), torch.bfloat16, window, seed=window + nq, causal=causal)


@gpu
@pytest.mark.parametrize("heads,kv_heads", [(4, 4), (6, 2)])
@pytest.mark.parametrize("window", [None, 70])
def test_varlen(fcsa, heads, kv_heads, window):
    ls = [63, 64, 65, 191, 192, 193, 383, 385, 1, 0]
    q, k, v, do = make_packed(ls, ls, heads, kv_heads, 64, torch.bfloat16, seed=heads + (window or 0))
    kw = dict(causal=True) if window is None else dict(causal=False, window=window)
    *got, _ = run_varlen(fcsa, q, k, v, do, cu_of(ls), cu_of(ls), max(ls), max(ls), **kw)
    seq_check(torch.bfloat16, got, q, k, v, do, ls, ls, **kw)
