"""CPU checks of the D = 64 backward's 192-key work items (csrc/tile_ranges.h through tests/bwd_blocks_host.cpp):
the query tiles each of an item's three key warpgroups computes, against brute-force visibility.

* every visible (query, key) pair lies in a query tile that its key's warpgroup computes;
* every tile a warpgroup computes holds at least one pair it sees;
* the item's range is the union of its warpgroups' (the loop visits no tile that no warpgroup computes);
for causal and non-causal problems, Nq != Nk both ways, sliding windows and the lengths of packed sequences (each
sequence is its own (Nq, Nk) problem on the device)."""
import ctypes
import functools
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
_INTS = np.ctypeslib.ndpointer(np.int32, flags="C_CONTIGUOUS")
KEYS = 192


@functools.lru_cache(maxsize=None)
def _lib():
    cxx = os.environ.get("FCSA_CXX") or shutil.which("g++") or "g++"
    tmp = tempfile.TemporaryDirectory(prefix="fcsa_bwd_blocks_")
    out = os.path.join(tmp.name, "bwd_blocks_host.so")
    subprocess.run([cxx, "-O1", "-std=c++17", "-Wall", "-fPIC", "-shared", os.path.join(HERE, "bwd_blocks_host.cpp"),
                    "-o", out], check=True)
    lib = ctypes.CDLL(out)
    lib._tmp = tmp
    i = ctypes.c_int
    lib.fcsa_bwd_block_keys.argtypes, lib.fcsa_bwd_block_keys.restype = [i, i, i, i], i
    lib.fcsa_key_block_query_tiles.argtypes = [i, i, i, i, i, i, i, _INTS, _INTS]
    lib.fcsa_key_block_query_tiles.restype = None
    return lib


def tiles(key0, keys, nq, nk, causal, window):
    lo, hi = np.empty(1, np.int32), np.empty(1, np.int32)
    wb, we = (0, 1) if window is None else (window, window + 1)
    _lib().fcsa_key_block_query_tiles(key0, keys, nq, nk, int(causal), wb, we, lo, hi)
    return int(lo[0]), int(hi[0])


def visible(nq, nk, causal, window):
    """(nq, nk) bool: query i sees key j (bottom-right aligned diagonal, optional window)."""
    d = np.arange(nq)[:, None] + (nk - nq) - np.arange(nk)[None, :]
    v = d >= 0 if causal else np.ones_like(d, bool)
    if window is not None:
        v &= (d < window) if causal else (np.abs(d) < window)
    return v


def check(nq, nk, causal, window):
    vis = visible(nq, nk, causal, window)
    qtile = np.arange(nq) // 64
    for key0 in range(0, nk, KEYS):
        blk = tiles(key0, KEYS, nq, nk, causal, window)
        covered = set()
        for w in range(3):
            k0 = key0 + 64 * w
            lo, hi = tiles(k0, 64, nq, nk, causal, window)
            seen = vis[:, k0:min(k0 + 64, nk)].any(axis=1) if k0 < nk else np.zeros(nq, bool)
            need = set(qtile[seen].tolist())
            got = set(range(lo, hi))
            assert need <= got, (nq, nk, causal, window, key0, w, sorted(need - got))
            assert got <= need, (nq, nk, causal, window, key0, w, sorted(got - need))
            covered |= got
        assert covered == set(range(*blk)) or (not covered and blk[0] >= blk[1]), (nq, nk, causal, window, key0)


SIZES = [1, 63, 64, 65, 127, 191, 192, 193, 383, 385, 450]


def test_block_keys():
    lib = _lib()
    assert lib.fcsa_bwd_block_keys(64, 0, 1, 0) == 192
    assert lib.fcsa_bwd_block_keys(64, 0, 1, 1) == 128      # head loop
    assert lib.fcsa_bwd_block_keys(64, 1, 1, 0) == 128      # bias
    assert lib.fcsa_bwd_block_keys(64, 0, 0, 0) == 128      # dK / dV only
    assert lib.fcsa_bwd_block_keys(128, 0, 1, 0) == 128


@pytest.mark.parametrize("causal", [False, True])
def test_unwindowed(causal):
    for nq in SIZES:
        for nk in SIZES:
            check(nq, nk, causal, None)


@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("window", [1, 2, 40, 64, 65, 129, 200, 500])
def test_windowed(causal, window):
    for nq in (1, 65, 193, 385, 450):
        for nk in (1, 64, 192, 193, 385, 450):
            check(nq, nk, causal, window)


@pytest.mark.parametrize("window", [None, 70])
def test_packed_lengths(window):
    """Packed sequences: every (Nq, Nk) pair of a batch's lengths, each item of the longest key length that lies in
    the sequence (the device returns early for the others)."""
    lq, lk = [0, 1, 63, 300, 193], [5, 64, 385, 191, 0]
    for a, b in zip(lq, lk):
        if a and b:
            check(a, b, True, window)
            check(a, b, False, window)
