"""The kernels' tile ranges and grid rules for the CPU tests: csrc/tile_ranges.h itself, through the extern "C"
wrappers of tests/tile_ranges_host.cpp.  The first use compiles that file with the host C++ compiler (FCSA_CXX, or g++
on PATH, as build.py) into a temporary directory and loads it with ctypes: no nvcc, no built library, no GPU.

Functions over a window take `w`, an np.arange of windows (one result per window, from the WINDOW instantiations), or
None for the unwindowed instantiations (arrays of one element)."""
import ctypes
import functools
import itertools
import os
import shutil
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
_INTS = np.ctypeslib.ndpointer(np.int32, flags="C_CONTIGUOUS")


@functools.lru_cache(maxsize=None)
def _lib():
    cxx = os.environ.get("FCSA_CXX") or shutil.which("g++") or "g++"
    tmp = tempfile.TemporaryDirectory(prefix="fcsa_tile_ranges_")
    out = os.path.join(tmp.name, "tile_ranges_host.so")
    subprocess.run([cxx, "-O1", "-std=c++17", "-Wall", "-fPIC", "-shared", os.path.join(HERE, "tile_ranges_host.cpp"),
                    "-o", out], check=True)
    lib = ctypes.CDLL(out)
    lib._tmp = tmp                                  # removed when the library goes
    i, p = ctypes.c_int, _INTS
    for name, argtypes in {
        "fcsa_block_key_tiles": [i, i, i, i, i, i, i, p, p],
        "fcsa_warpgroup_key_tiles": [i, p, p, i, i, i, i, i, p, p],
        "fcsa_decode_chunk": [i, i, i, i, i, i, i, i, i, p, p],
        "fcsa_query_tiles": [i, i, i, i, i, i, p, p],
        "fcsa_bwd_row0_sequence": [i, i, i, i, i, i, i, i, p, p],
        "fcsa_row_key_cols": [i, i, i, i, i, p, p],
        "fcsa_tile_visible": [p, p, i, i, i, i, i, i, p],
        "fcsa_varlen_tile_base": [i, i],
        "fcsa_varlen_tiles": [i, ctypes.c_longlong],
        "fcsa_fwd_block_rows": [i],
        "fcsa_row_blocks": [i, i],
        "fcsa_decode_split": [ctypes.c_longlong, i, i],
        "fcsa_decode_window_keys": [i, i, i],
        "fcsa_bwd_group_split": [i, i, i, i, i, i],
    }.items():
        f = getattr(lib, name)
        f.argtypes, f.restype = argtypes, (None if p in argtypes else i)
    return lib


def _span(w):
    """(w_begin, w_end) of an np.arange of windows; (0, 1) = unwindowed."""
    if w is None:
        return 0, 1
    assert w[0] >= 1 and (np.diff(w) == 1).all()
    return int(w[0]), int(w[-1]) + 1


def _ranges(fn, w, *args):
    b, e = _span(w)
    lo, hi = np.empty(e - b, np.int32), np.empty(e - b, np.int32)
    fn(*args, b, e, lo, hi)
    return lo, hi


def fwd_block_rows(D):
    """Query rows of one forward CTA."""
    return _lib().fcsa_fwd_block_rows(D)


def n_qblk(nq, bm):
    """The query blocks of bm rows per (batch, head)."""
    return _lib().fcsa_row_blocks(nq, bm)


def block_range(m0, bm, nq, nk, w, causal):
    """fcsa_fwd_kernel: key tiles [j_lo, NT) of the block of bm query rows starting at m0."""
    return _ranges(_lib().fcsa_block_key_tiles, w, m0, bm, nq, nk, int(causal))


def warpgroup_range(r0, nq, nk, w, causal, j_lo, NT):
    """fcsa_fwd_kernel: tiles [jw_lo, jw_hi) of the warpgroup whose rows start at r0; it computes the j of its block's
    [j_lo, NT) inside them."""
    lo, hi = _ranges(_lib().fcsa_warpgroup_key_tiles, w, r0, np.ascontiguousarray(j_lo, np.int32),
                     np.ascontiguousarray(NT, np.int32), nq, nk, int(causal))
    return np.maximum(j_lo, lo), np.minimum(NT, hi)


def bwd_range(key0, nq, nk, w, causal):
    """fcsa_bwd_kernel: query tiles [i_lo, i_end) of the key tile starting at key0."""
    return _ranges(_lib().fcsa_query_tiles, w, key0, nq, nk, int(causal))


def bwd_row0_sequence(key0, nq, nk, w, causal, hpc):
    """The STAGED consumer loop's row0 over the flat (head, query tile) sequence, as the kernel steps it, and the
    dQ reducer's query tile: lists of per-window arrays (-1 past a window's hpc * NI tiles), then i_lo and NI."""
    i_lo, i_end = bwd_range(key0, nq, nk, w, causal)
    NI = np.maximum(0, i_end - i_lo)
    steps = int((hpc * NI).max(initial=0))
    b, e = _span(w)
    rows, qts = np.empty((e - b, steps), np.int32), np.empty((e - b, steps), np.int32)
    _lib().fcsa_bwd_row0_sequence(key0, nq, nk, int(causal), hpc, b, e, steps, rows, qts)
    return list(rows.T), list(qts.T), i_lo, NI


def decode_range(r0, R, G, Tb, nq, w, causal, n_split):
    """fcsa_decode_kernel: the [j0, j1) of every split of the row block starting at row r0 (rows r = query * G + head)."""
    r_last = min(r0 + 63, R - 1)
    return [_ranges(_lib().fcsa_decode_chunk, w, r0 // G, r_last // G, nq, Tb, int(causal), s, n_split)
            for s in range(n_split)]


def row_key_cols(nq, nk, w, causal):
    """The forward's and decode's per-element limits: the key columns [lo, hi] each query sees, as (W, nq) arrays."""
    b, e = _span(w)
    lo, hi = np.empty((e - b, nq), np.int32), np.empty((e - b, nq), np.int32)
    _lib().fcsa_row_key_cols(nq, nk, int(causal), b, e, lo, hi)
    return lo, hi


def tile_visible(q_first, q_last, nq, nk, w, causal):
    """Whether query rows [q_first[r], q_last[r]] see every key of each 128-key tile (the tile needs no masks):
    (W, ranges, key tiles) bool."""
    b, e = _span(w)
    q_first, q_last = np.ascontiguousarray(q_first, np.int32), np.ascontiguousarray(q_last, np.int32)
    out = np.empty((e - b, len(q_first), (nk + 127) // 128), np.int32)
    _lib().fcsa_tile_visible(q_first, q_last, len(q_first), nq, nk, int(causal), b, e, out)
    return out.astype(bool)


def decode_window_keys(cap, window, causal):
    """The keys whose tiles bound a decode row block under each window of `window`."""
    return np.array([_lib().fcsa_decode_window_keys(cap, int(x), int(causal)) for x in np.atleast_1d(window)])


def decode_split(items, cap, sms):
    """Key splits per decode work item."""
    return _lib().fcsa_decode_split(items, cap, sms)


def group_split(B, H, Hk, Nk, sms, bias=False):
    """Slices per key/value-head group the backward chooses."""
    return _lib().fcsa_bwd_group_split(B, H, Hk, Nk, int(bias), sms)


def tiles(lengths):
    """The backward's packed layout: (the query-tile range of every sequence from its base, tiles per head)."""
    cu = [0] + list(itertools.accumulate(lengths))
    base = [_lib().fcsa_varlen_tile_base(cu[b], b) for b in range(len(lengths))]
    return [(t, t + n_qblk(n, 64)) for t, n in zip(base, lengths)], _lib().fcsa_varlen_tiles(len(lengths), cu[-1])
