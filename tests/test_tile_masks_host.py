"""CPU: the masks of the forward and decode exp stages (csrc/tile_ranges.h through tests/tile_ranges.py), checked
against the visibility rule.

A masked tile selects, per element, the key columns [lo, hi] of each row (row_key_cols); a tile whose rows see every
one of its keys (tile_visible) skips the selects.  Both are checked both ways: a wrong "visible" would add keys past Nk,
above the diagonal or outside the window into the row sums and O, and a wrong "not visible" costs the selects.  For Nq,
Nk around multiples of 64, 128 and 192, causal and not, unwindowed and with every window from 1 to Nq + Nk - 1:
* column c lies in [lo, hi] of query i iff i sees c;
* tile_visible holds iff every (query, key) pair of the rectangle is visible, for the forward's 64-row warpgroup ranges
  and for decode's row blocks, whose rows r = query * G + head map 64 rows onto the queries [r0 / G, r_last / G];
* the forward's warpgroup range unclipped at Nq (as the kernel passes it) is visible only where the clipped one is."""
import numpy as np
import pytest

from test_fwd_blocks_host import LENGTHS
from test_window_host import band
from tile_ranges import row_key_cols, tile_visible

KT = 128


def windows(nq, nk, windowed):
    """The windows to check, and those band() takes (no window: one wider than every distance)."""
    return (np.arange(1, nq + nk), np.arange(1, nq + nk)) if windowed else (None, np.array([nq + nk]))


def whole_tiles(vis, q_first, q_last):
    """(W, ranges, key tiles): every pair of rows [q_first, q_last] x the tile is visible, keys past Nk invisible."""
    nk = vis.shape[2]
    nt = (nk + KT - 1) // KT
    v = np.pad(vis, [(0, 0), (0, 0), (0, nt * KT - nk)])
    return np.stack([v[:, f:l + 1].reshape(v.shape[0], l + 1 - f, nt, KT).all(axis=(1, 3))
                     for f, l in zip(q_first, q_last)], axis=1)


@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("nq", LENGTHS)
def test_row_key_cols_are_the_band(nq, causal):
    for nk in LENGTHS:
        for windowed in (False, True):
            w, wb = windows(nq, nk, windowed)
            lo, hi = row_key_cols(nq, nk, w, causal)
            c = np.arange(nk)
            inside = (c >= lo[..., None]) & (c <= hi[..., None])
            vis = band(nq, nk, wb, causal)
            assert (inside == vis).all(), (nk, windowed, np.argwhere(inside != vis)[:4])


@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("nq", LENGTHS)
def test_tile_visible_iff_every_pair_is(nq, causal):
    for nk in LENGTHS:
        for windowed in (False, True):
            w, wb = windows(nq, nk, windowed)
            vis = band(nq, nk, wb, causal)
            r0 = np.arange(0, nq, 64)                                      # the forward's warpgroups
            last = np.minimum(r0 + 63, nq - 1)
            got = tile_visible(r0, last, nq, nk, w, causal)
            assert (got == whole_tiles(vis, r0, last)).all(), (nk, windowed)
            # the kernel passes r0 + 63 also past Nq: that only ever masks more
            assert not (tile_visible(r0, r0 + 63, nq, nk, w, causal) & ~got).any(), (nk, windowed)


@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("G,nq", [(2, 1), (2, 70), (3, 1), (3, 43), (4, 33), (4, 65), (7, 20)])
def test_tile_visible_for_decode_row_blocks(G, nq, causal):
    for Tb in LENGTHS:
        for windowed in (False, True):
            w, wb = windows(nq, Tb, windowed)
            R = G * nq
            r0 = np.arange(0, R, 64)
            first, last = r0 // G, np.minimum(r0 + 63, R - 1) // G
            got = tile_visible(first, last, nq, Tb, w, causal)
            assert (got == whole_tiles(band(nq, Tb, wb, causal), first, last)).all(), (Tb, windowed)
