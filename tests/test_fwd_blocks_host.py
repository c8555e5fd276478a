"""CPU: the forward kernel's work split, mirrored from csrc/fwd_kernel.cuh and checked against the visibility rule.

D = 64 runs blocks of 192 query rows (three consumer warpgroups of 64 rows), D = 128 blocks of 128 rows (two).  A
block visits the key tiles [j_lo, NT) of 128 keys; each warpgroup computes the tiles [jw_lo, jw_hi) of that range that
its own rows see and passes the other ring slots on.  For Nq, Nk around multiples of 64, 128 and 192, causal and not,
unwindowed and with every window from 1 to Nq + Nk - 1: every visible (query, key) pair lies in a tile its warpgroup
computes, every computed tile holds one, and the block's range is exactly the union of the tiles its rows see (a
block that sees nothing may visit nothing)."""
import numpy as np
import pytest

from test_window_host import band, check_tiles, tiles_hit, visited

KT, WG = 128, 64                     # key tile, query rows per consumer warpgroup
BLOCK_M = {64: 192, 128: 128}        # FwdCfg<D>::kBlockM
LENGTHS = (1, 2, 63, 64, 65, 127, 128, 129, 191, 192, 193, 255, 256, 257, 383, 384, 385)


def n_qblk(nq, bm):
    """launch_forward: the query blocks per (batch, head); a VARLEN block starting past its sequence exits."""
    return (nq + bm - 1) // bm


# ---- mirror of fcsa_fwd_kernel (numpy arrays over the window w, or w = None for the unwindowed kernels) -------------
def block_range(m0, bm, nq, nk, w, causal):
    """Key tiles [j_lo, NT) of the block of bm query rows starting at m0."""
    off = nk - nq
    if w is None:
        NT = (nk + 127) >> 7
        if causal:
            last_col = min(m0 + bm - 1, nq - 1) + off
            NT = 0 if last_col < 0 else min(NT, (last_col >> 7) + 1)
        return np.zeros(1, dtype=np.int64), np.full(1, NT)
    last_col = min(m0 + bm - 1, nq - 1) + off + (0 if causal else w - 1)
    NT = np.where(last_col < 0, 0, np.minimum((nk + 127) >> 7, np.maximum(last_col, 0) // 128 + 1))
    first_col = m0 + off - w + 1
    j_lo = np.where(first_col <= 0, 0, np.minimum(np.maximum(first_col, 0) // 128, NT))
    return j_lo, NT


def warpgroup_range(r0, nq, nk, w, causal, j_lo, NT):
    """Tiles [jw_lo, jw_hi) of the warpgroup whose rows start at r0; it computes j in [j_lo, NT) inside them."""
    off = nk - nq
    jw_lo, jw_hi = j_lo, NT
    if r0 >= nq:
        jw_hi = np.zeros_like(NT)
    elif causal or w is not None:
        last_col = min(r0 + 63, nq - 1) + off + (0 if causal else w - 1)
        jw_hi = np.where(last_col < 0, 0, np.maximum(last_col, 0) // 128 + 1)
    if w is not None:
        first_col = r0 + off - w + 1
        jw_lo = np.where(first_col > 0, np.maximum(j_lo, np.maximum(first_col, 0) // 128), j_lo)
    return np.maximum(j_lo, jw_lo), np.minimum(NT, jw_hi)


def check_split(nq, nk, causal, windowed, bm):
    w = np.arange(1, nq + nk) if windowed else None
    vis = band(nq, nk, w if windowed else np.array([nq + nk]), causal)        # (W, nq, nk)
    nt = (nk + KT - 1) // KT
    nb = n_qblk(nq, bm)
    assert (nb - 1) * bm < nq <= nb * bm
    for m0 in range(0, nb * bm, bm):
        j_lo, NT = block_range(m0, bm, nq, nk, w, causal)
        check_tiles(tiles_hit(vis[:, m0:m0 + bm], 2, KT), j_lo, NT)
        for r0 in range(m0, m0 + bm, WG):
            lo, hi = warpgroup_range(r0, nq, nk, w, causal, j_lo, NT)
            rows = vis[:, r0:r0 + WG]                                          # empty past the end
            want = tiles_hit(rows, 2, KT) if rows.shape[1] else np.zeros((vis.shape[0], nt), bool)
            got = visited(np.broadcast_to(lo, (vis.shape[0],)), np.broadcast_to(hi, (vis.shape[0],)), nt)
            assert (got == want).all(), (m0, r0, np.argwhere(got != want)[:4])


@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("nq", LENGTHS)
def test_forward_block_and_warpgroup_tiles(nq, causal, D):
    for nk in LENGTHS:
        check_split(nq, nk, causal, False, BLOCK_M[D])
        check_split(nq, nk, causal, True, BLOCK_M[D])


def test_causal_square_work_matches_64_row_groups():
    """Causal Nq = Nk = 4096 at D = 64: the warpgroups compute 1056 tiles of 64 x 128, as many as 128-row blocks do;
    visiting the whole block range with every warpgroup would compute 1152."""
    nq = nk = 4096
    total = whole = 0
    for m0 in range(0, n_qblk(nq, 192) * 192, 192):
        j_lo, NT = block_range(m0, 192, nq, nk, None, True)
        for r0 in range(m0, m0 + 192, WG):
            lo, hi = warpgroup_range(r0, nq, nk, None, True, j_lo, NT)
            total += int(max(0, hi[0] - lo[0]))
            whole += int(NT[0] - j_lo[0])
    assert (total, whole) == (1056, 1152)
