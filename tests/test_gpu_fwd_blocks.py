"""GPU: the forward kernel's query blocks (192 rows and three consumer warpgroups at D = 64, 128 rows and two at
D = 128) at lengths around one and two 192-row blocks and at 4096, on the dense, grouped-query loop, packed (varlen)
and windowed paths, causal with Nq != Nk included.  Every output is judged against the float64 reference with the
element-wise bound at C = 2 and the relative tolerances of test_gpu_parity.py.  The tile arithmetic itself is
checked on the CPU by tests/test_fwd_blocks_host.py."""
import pytest
import torch

from test_gpu_gqa import gqa_check, loop_batch
from test_gpu_parity import check, fcsa  # noqa: F401
from test_gpu_varlen import cu_of, make_packed, per_seq, run_varlen, seq_check
from test_gpu_window import wcheck

pytestmark = pytest.mark.gpu

LENGTHS = (191, 192, 193, 383, 385)
CROSS = [(191, 385), (385, 191), (193, 576), (576, 193), (1, 385), (385, 1)]      # (Nq, Nk)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("dim_head", [64, 128])
@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("n", LENGTHS)
def test_dense_block_edges(fcsa, n, causal, dim_head, dtype):
    check(fcsa, (2, 3, n, dim_head), (2, 3, n, dim_head), dtype, seed=n + dim_head, causal=causal)


@pytest.mark.parametrize("dim_head", [64, 128])
@pytest.mark.parametrize("nq,nk", CROSS)
def test_dense_causal_cross_lengths(fcsa, nq, nk, dim_head):
    """Bottom-right aligned causal masks whose diagonal falls anywhere in a block: Nq > Nk leaves the first Nq - Nk
    rows with no key (o = 0), and whole warpgroups of a block past the diagonal."""
    check(fcsa, (2, 3, nq, dim_head), (2, 3, nk, dim_head), torch.bfloat16, seed=nq + 2 * nk, causal=True)


@pytest.mark.parametrize("causal", [True, False])
def test_dense_4096(fcsa, causal):
    """The benchmark's sequence length: 21 full blocks and one of 64 rows (two warpgroups with no row)."""
    check(fcsa, (1, 2, 4096, 64), (1, 2, 4096, 64), torch.bfloat16, seed=4096, causal=causal, grads=causal)


@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("n", [193, 385])
def test_gqa_loop_block_edges(fcsa, n, causal):
    Hk = 2
    gqa_check(fcsa, (loop_batch(Hk, n), 2 * Hk, n, 64), (loop_batch(Hk, n), Hk, n, 64), torch.bfloat16, seed=n,
              path="loop", causal=causal)


@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("heads,kv_heads", [(4, 4), (4, 2)])
def test_varlen_block_edges(fcsa, causal, heads, kv_heads):
    """Packed sequences around one and two blocks, each against the reference on it alone and o bitwise against the
    dense op on it (blocks past a sequence's end exit; a tile past it reads the next sequence's rows)."""
    ls = [191, 1, 192, 193, 0, 383, 64, 385]
    q, k, v, do = make_packed(ls, ls, heads, kv_heads, 64, torch.bfloat16, seed=heads + kv_heads)
    cu = cu_of(ls)
    o, dq, dk, dv, _ = run_varlen(fcsa, q, k, v, do, cu, cu, max(ls), max(ls), causal=causal)
    seq_check(torch.bfloat16, (o, dq, dk, dv), q, k, v, do, ls, ls, causal=causal)
    s = 0
    for n in ls:
        if n:
            od = fcsa.flash_cosine_sim_attention(*(per_seq(t, s, n).cuda() for t in (q, k, v)), causal=causal)
            assert torch.equal(per_seq(o, s, n), od), n
        s += n


@pytest.mark.parametrize("window", [1, 64, 129, 193, 385])
@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("nq,nk", [(385, 385), (193, 576), (576, 193)])
def test_window_block_edges(fcsa, window, causal, nq, nk):
    """A band whose edges fall inside a block: warpgroups start at different key tiles and stop at different ones."""
    wcheck(fcsa, (1, 2, nq, 64), (1, 2, nk, 64), torch.bfloat16, window, seed=nq + nk + window, causal=causal)
