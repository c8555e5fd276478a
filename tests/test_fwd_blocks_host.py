"""CPU: the forward kernel's work split (csrc/tile_ranges.h through tests/tile_ranges.py), checked against the
visibility rule.

D = 64 runs blocks of 192 query rows (three consumer warpgroups of 64 rows), D = 128 blocks of 128 rows (two).  A
block visits the key tiles [j_lo, NT) of 128 keys; each warpgroup computes the tiles [jw_lo, jw_hi) of that range that
its own rows see and passes the other ring slots on.  For Nq, Nk around multiples of 64, 128 and 192, causal and not,
unwindowed and with every window from 1 to Nq + Nk - 1: every visible (query, key) pair lies in a tile its warpgroup
computes, every computed tile holds one, and the block's range is exactly the union of the tiles its rows see (a
block that sees nothing may visit nothing)."""
import numpy as np
import pytest

from test_window_host import band, check_tiles, tiles_hit, visited
from tile_ranges import block_range, fwd_block_rows, n_qblk, warpgroup_range

KT, WG = 128, 64                     # key tile, query rows per consumer warpgroup
LENGTHS = (1, 2, 63, 64, 65, 127, 128, 129, 191, 192, 193, 200, 255, 256, 257, 383, 384, 385, 400)


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
        check_split(nq, nk, causal, False, fwd_block_rows(D))
        check_split(nq, nk, causal, True, fwd_block_rows(D))


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
