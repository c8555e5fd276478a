"""CPU: sliding-window attention on the host side.

* The tile ranges the backward and decode kernels visit under a window (csrc/tile_ranges.h through
  tests/tile_ranges.py; the forward's are in test_fwd_blocks_host.py), checked against the band rule for every window up to Nq + Nk, causal and not: every visible
  (query, key) pair lies in a visited tile, and every visited tile holds at least one visible pair (a work item that
  visits nothing is the one exception).  The backward's HEAD_LOOP row0 sequence and the decode split are included.
* plain_cosine_sim_attention(window=...) in float64 against an explicit band mask, with GQA and merged 3-D layouts.
* Every rejection of the keyword, the ABI's argument checks through ctypes, and a sharded CPU run.
* The transformer's window on the plain path: cached decoding against the full forward, packed documents against
  per-document calls.
* The float32 emulation of the kernels' roundings with windows stays within C / 2 of the element-wise bound.
* The windowed float64 reference (tests/window_bounds.py) is elementwise_bounds.attention_bounds bitwise when the band
  hides nothing, and the op on each row's band otherwise."""
import numpy as np
import pytest
import torch

from elementwise_bounds import C, attention_bounds, check_bound, kernel_shift
from tile_ranges import bwd_range, bwd_row0_sequence, decode_range, decode_window_keys
from window_bounds import window_attention_bounds

QT = 64
LENGTHS = (1, 2, 63, 64, 65, 127, 128, 129, 200, 255, 256, 257, 383, 384, 385, 400)


def band(nq, nk, w, causal):
    """(W, nq, nk) visibility for every window w (an array) - the rule of the public docstring."""
    d = np.arange(nq)[None, :, None] + (nk - nq) - np.arange(nk)[None, None, :]
    w = w[:, None, None]
    return ((d >= 0) & (d < w)) if causal else (np.abs(d) < w)


def tiles_hit(vis, axis, size):
    """vis (W, rows, cols) -> (W, ntiles) bool: which tiles of `size` along `axis` (1 rows, 2 cols) hold a pair."""
    n = vis.shape[axis]
    nt = (n + size - 1) // size
    pad = nt * size - n
    widths = [(0, 0)] * 3
    widths[axis] = (0, pad)
    v = np.pad(vis, widths)
    if axis == 2:
        return v.reshape(v.shape[0], v.shape[1], nt, size).any(axis=(1, 3))
    return v.reshape(v.shape[0], nt, size, v.shape[2]).any(axis=(2, 3))


def visited(lo, hi, nt):
    """(W, nt) bool of tiles [lo, hi) per window."""
    t = np.arange(nt)[None, :]
    return (t >= lo[:, None]) & (t < hi[:, None])


def check_tiles(vis_tiles, lo, hi):
    """Visited tiles == tiles with a visible pair, except that a work item with no visible pair may visit nothing."""
    n, nt = vis_tiles.shape
    got = visited(np.broadcast_to(lo, (n,)), np.broadcast_to(hi, (n,)), nt)
    empty = ~vis_tiles.any(1)
    assert ((got == vis_tiles) | (empty[:, None] & ~got)).all()


@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("nq", LENGTHS)
def test_backward_tile_range_and_row0_sequence(nq, causal):
    for nk in LENGTHS:
        w = np.arange(1, nq + nk)
        vis = band(nq, nk, w, causal)
        for key0 in range(0, nk, 128):
            cols = vis[:, :, key0:key0 + 128]
            i_lo, i_end = bwd_range(key0, nq, nk, w, causal)
            check_tiles(tiles_hit(cols, 1, QT), i_lo, i_end)
            for hpc in (2, 3):                    # HEAD_LOOP: row0 restarts at the window's first tile with every head
                rows, qts, lo, NI = bwd_row0_sequence(key0, nq, nk, w, causal, hpc)
                for i, (r, qt) in enumerate(zip(rows, qts)):
                    live = r >= 0
                    want = (lo + i % np.maximum(NI, 1)) * QT
                    assert (r[live] == want[live]).all() and (qt[live] * QT == r[live]).all()


@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("G,nq", [(1, 1), (1, 5), (3, 1), (4, 33), (2, 70)])
def test_decode_tile_split(G, nq, causal):
    for Tb in (1, 63, 64, 65, 127, 128, 129, 200, 256, 257, 399, 400):
        R = G * nq
        w = np.arange(1, nq + Tb)
        vis = band(nq, Tb, w, causal)                           # (W, query, key)
        for r0 in range(0, R, 64):
            rows = np.arange(r0, min(r0 + 64, R)) // G
            blk = vis[:, rows]
            hit = tiles_hit(blk, 2, 128)
            # the tiles a block sees fit in the window's tile bound used by the split rule
            assert (hit.sum(1) <= -(-decode_window_keys(1 << 30, w, causal) // 128)).all()
            for n_split in (1, 2, 3, 7):
                parts = decode_range(r0, R, G, Tb, nq, w, causal, n_split)
                for (a0, a1), (b0, b1) in zip(parts, parts[1:]):
                    assert (a1 == b0).all() and (a0 <= a1).all()
                check_tiles(hit, parts[0][0], parts[-1][1])


# ---- the plain path ------------------------------------------------------------------------------------------------
def _qkv(shape_q, shape_k, seed=0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape_q, generator=g, dtype=torch.float64), torch.randn(shape_k, generator=g, dtype=torch.float64),
            torch.randn(shape_k, generator=g, dtype=torch.float64))


@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("layout", ["mha", "gqa", "single", "merged"])
@pytest.mark.parametrize("nq,nk,w", [(50, 50, 1), (50, 50, 7), (30, 70, 16), (70, 30, 9), (40, 40, 200)])
def test_plain_window_is_a_band_mask(layout, causal, nq, nk, w):
    from flash_cosine_sim_attention_b200 import plain_cosine_sim_attention
    shapes = {"mha": ((2, 4, nq, 16), (2, 4, nk, 16)), "gqa": ((2, 4, nq, 16), (2, 2, nk, 16)),
              "single": ((2, 4, nq, 16), (2, nk, 16)), "merged": ((6, nq, 16), (6, nk, 16))}
    q, k, v = _qkv(*shapes[layout], seed=w)
    got = plain_cosine_sim_attention(q, k, v, causal=causal, window=w, groups=2)
    d = torch.arange(nq)[:, None] + (nk - nq) - torch.arange(nk)[None, :]
    keep = ((d >= 0) & (d < w)) if causal else (d.abs() < w)
    # the band as an additive bias on the unwindowed formulation (-inf-like where a key is outside it)
    ref_k, ref_v = k, v
    if layout == "gqa":
        ref_k, ref_v = k.repeat_interleave(2, 1), v.repeat_interleave(2, 1)
    heads = 1 if layout == "merged" else 4
    bias = torch.zeros(nq, nk, dtype=torch.float64).masked_fill(~keep, -torch.finfo(torch.float64).max)
    bias = bias.expand(6 if layout == "merged" else heads, nq, nk)
    want = plain_cosine_sim_attention(q, ref_k, ref_v, attn_bias=bias, causal=causal, groups=2)
    assert torch.allclose(got, want, rtol=0, atol=1e-12)
    if w >= nq + nk:
        assert torch.equal(got, plain_cosine_sim_attention(q, k, v, causal=causal, groups=2))


# ---- rejections ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bad,exc", [(0, ValueError), (-3, ValueError), (True, TypeError), (2.0, TypeError),
                                     ("8", TypeError)])
def test_window_must_be_a_positive_int(bad, exc):
    import flash_cosine_sim_attention_b200 as m
    q = torch.zeros(1, 2, 8, 64)
    with pytest.raises(exc, match="window"):
        m.plain_cosine_sim_attention(q, q, q, window=bad)
    with pytest.raises(exc, match="window"):
        m.flash_cosine_sim_attention(q, q, q, window=bad)
    with pytest.raises(exc, match="window"):
        m.flash_cosine_sim_attention_varlen(q[0].transpose(0, 1).half(), q[0].transpose(0, 1).half(),
                                            q[0].transpose(0, 1).half(), torch.tensor([0, 8], dtype=torch.int32),
                                            torch.tensor([0, 8], dtype=torch.int32), 8, 8, window=bad)
    with pytest.raises(exc, match="window"):
        m.flash_cosine_sim_attention_with_kv_cache(q.half(), q.half(), q.half(), torch.zeros(1, dtype=torch.int32),
                                                   window=bad)


def test_window_with_attn_bias_is_rejected():
    import flash_cosine_sim_attention_b200 as m
    q = torch.zeros(1, 2, 8, 64)
    bias = torch.zeros(2, 8, 8)
    with pytest.raises(NotImplementedError, match="window with attn_bias"):
        m.flash_cosine_sim_attention(q, q, q, attn_bias=bias, window=4)
    with pytest.raises(NotImplementedError, match="window with attn_bias"):
        m.flash_cosine_sim_attention(q, q, q, attn_bias=bias, window=4, causal=True)


def test_context_parallel_rejects_window_before_any_collective():
    from flash_cosine_sim_attention_b200.context_parallel import context_parallel_cosine_sim_attention
    q = torch.zeros(1, 2, 8, 64, dtype=torch.bfloat16)
    with pytest.raises(NotImplementedError, match="window"):
        context_parallel_cosine_sim_attention(q, q, q, window=4)      # no process group exists here


def test_transformer_rejects_window_with_softmax_attention():
    from flash_cosine_sim_attention_b200.transformer import Attention
    with pytest.raises(NotImplementedError, match="window"):
        Attention(64, dim_head=16, heads=2, non_cosine_sim_attn=True, window=8)


# ---- the C ABI -----------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    from flash_cosine_sim_attention_b200 import _abi
    if not __import__("os").path.exists(_abi.LIB_PATH):
        from flash_cosine_sim_attention_b200.build import build_library
        build_library()
    return _abi.load()


def test_abi_window_field_and_checks(lib):
    from flash_cosine_sim_attention_b200 import _abi
    assert _abi.FcsaProblem.window.offset == 60 and lib.fcsa_version() == 300
    p = _abi.FcsaProblem()
    p.dtype, p.batch, p.heads, p.kv_heads, p.seq_q, p.seq_k, p.head_dim = _abi.FCSA_BF16, 1, 2, 2, 16, 16, 64
    t = _abi.FcsaTensor(None, 0, 0, 0)
    r = _abi.ref
    p.window = -1
    calls = {
        "forward": lambda: lib.fcsa_forward(r(p), r(t), r(t), r(t), r(t), None, None),
        "backward": lambda: lib.fcsa_backward(r(p), *([r(t)] * 5), None, *([r(t)] * 3), None, 0, None, 0, None),
        "decode": lambda: lib.fcsa_decode(r(p), r(t), r(t), r(t), None, r(t), r(t), 0, 1, r(t), None, 0, None),
    }
    for name, call in calls.items():
        assert call() == _abi.FCSA_ERR_INVALID and b"window -1" in lib.fcsa_last_error(), name
    assert lib.fcsa_backward_workspace_bytes(r(p)) == 0
    # a nonzero window on the bias entry points
    p.window = 4
    b = _abi.FcsaBias(4096, 0, 16 * 16, 16, None)
    good = _abi.FcsaTensor(4096, 2 * 16 * 64, 16 * 64, 64)
    assert lib.fcsa_forward_bias(r(p), r(good), r(good), r(good), r(b), r(good), None, None) == _abi.FCSA_ERR_INVALID
    assert b"no sliding window with a bias" in lib.fcsa_last_error()
    # workspace sizes do not depend on the window
    sizes = []
    for w in (0, 1, 5, 1000):
        p.window = w
        sizes.append((lib.fcsa_backward_workspace_bytes(r(p)), lib.fcsa_backward_zeroed_bytes(r(p))))
    assert len(set(sizes)) == 1 and sizes[0][0] > 0


# ---- sharding (gloo, CPU) ------------------------------------------------------------------------------------------
def test_sharded_plain_attention_with_a_window():
    import os
    import torch.distributed as dist
    from flash_cosine_sim_attention_b200 import plain_cosine_sim_attention
    from flash_cosine_sim_attention_b200.sharding import sharded_flash_cosine_sim_attention
    if dist.is_initialized():
        pytest.skip("a process group already exists")
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "29533")
    dist.init_process_group("gloo", rank=0, world_size=1)
    try:
        q, k, v = _qkv((2, 4, 40, 16), (2, 4, 40, 16), seed=5)
        got = sharded_flash_cosine_sim_attention(q, k, v, attn_fn=plain_cosine_sim_attention, causal=True, window=6,
                                                 gather=True)
        want = plain_cosine_sim_attention(q, k, v, causal=True, window=6)
        assert torch.allclose(got, want, rtol=0, atol=1e-12)
        assert not torch.allclose(want, plain_cosine_sim_attention(q, k, v, causal=True), atol=1e-3)
    finally:
        dist.destroy_process_group()


# ---- the transformer on the plain path -----------------------------------------------------------------------------
def _model(window, seed=0):
    from flash_cosine_sim_attention_b200.transformer import CosineSimCausalTransformer
    torch.manual_seed(seed)
    return CosineSimCausalTransformer(num_tokens=50, dim=32, max_seq_len=64, depth=2, heads=4, dim_head=8,
                                      kv_heads=2, window=window).double().eval()


def test_transformer_window_cached_logits_match_the_full_forward():
    m = _model(window=5)
    x = torch.randint(0, 50, (2, 24))
    with torch.no_grad():
        full = m(x)
        cache = m.new_cache()
        steps = [m(x[:, :10], cache=cache)] + [m(x[:, t:t + 1], cache=cache) for t in range(10, 24)]
    assert torch.allclose(torch.cat(steps, 1), full, rtol=0, atol=1e-10)
    with torch.no_grad():
        assert not torch.allclose(_model(window=None)(x), full, atol=1e-6)     # the window changes the result


def test_transformer_window_packed_documents_match_per_document_calls():
    m = _model(window=4, seed=1)
    docs = [torch.randint(0, 50, (1, n)) for n in (7, 12, 1, 9)]
    cu = torch.tensor(np.cumsum([0] + [d.shape[1] for d in docs]), dtype=torch.int32)
    with torch.no_grad():
        packed = m(torch.cat(docs, 1), cu_seqlens=cu)
        each = torch.cat([m(d) for d in docs], 1)
    assert torch.allclose(packed, each, rtol=0, atol=1e-10)


# ---- the float32 emulation of the kernels' roundings, with windows ------------------------------------------------
@pytest.mark.parametrize("fmt", ["bf16", "f16"])
@pytest.mark.parametrize("causal,w", [(True, 1), (True, 65), (False, 33), (False, 130)])
def test_emulated_rounding_with_window_within_bound(fmt, causal, w, monkeypatch):
    """test_elementwise_bounds.emulate with the band added to its visibility: within C / 2, so C = 2 stands."""
    import test_elementwise_bounds as teb
    oracle = teb.oracle
    nq, nk = 200, 260
    d = np.arange(nq)[:, None] + (nk - nq) - np.arange(nk)[None, :]
    keep = ((d >= 0) & (d < w)) if causal else (np.abs(d) < w)
    vis0 = oracle._visibility
    monkeypatch.setattr(oracle, "_visibility", lambda *a, **kw: vis0(*a, **kw) & keep)
    rng = np.random.default_rng(w)
    q, do = (oracle.round_to(rng.standard_normal((1, 4, nq, 64)), fmt) for _ in range(2))
    k, v = (oracle.round_to(rng.standard_normal((1, 2, nk, 64)), fmt) for _ in range(2))
    got = teb.emulate(q, k, v, do, fmt, causal=causal)
    ref, bound = window_attention_bounds(q, k, v, do, causal=causal, round_qk=fmt, fmt=fmt,
                                         shift=kernel_shift(fmt, 8), chunk=256, window=w)
    for n, g in zip(("o", "dq", "dk", "dv"), got):
        check_bound(n, torch.from_numpy(g), ref, bound, fmt, c=C / 2)


# ---- the windowed float64 reference (tests/window_bounds.py) -------------------------------------------------------
@pytest.mark.parametrize("layout,kw", [("gqa", dict(causal=True)), ("single", dict(mask=True)),
                                       ("merged", dict(causal=True, groups=2)), ("mha", dict(l2norm_qk=False))])
def test_window_reference_without_a_band_is_attention_bounds(layout, kw):
    """With no window (and with one that hides nothing) it is elementwise_bounds.attention_bounds, bitwise."""
    shapes = {"mha": ((2, 2, 70, 32), (2, 2, 90, 32)), "gqa": ((2, 4, 70, 32), (2, 2, 90, 32)),
              "single": ((2, 4, 70, 32), (2, 90, 32)), "merged": ((4, 90, 32), (4, 70, 32))}
    q, k, v = _qkv(*shapes[layout], seed=3)
    do = torch.randn(q.shape, generator=torch.Generator().manual_seed(4), dtype=torch.float64)
    kw = dict(kw)
    if kw.pop("mask", False):
        kw["mask"] = torch.rand(2, 90, generator=torch.Generator().manual_seed(5)) > 0.4
    common = dict(fmt="f16", round_qk="f16" if kw.get("l2norm_qk", True) else None, shift=4.0, chunk=32)
    want = attention_bounds(q, k, v, do, **common, **kw)
    for window in (None, 160):
        got = window_attention_bounds(q, k, v, do, window=window, **common, **kw)
        for part in range(2):
            assert set(got[part]) == set(want[part])
            for name in want[part]:
                assert torch.equal(got[part][name], want[part][name]), (window, part, name)


@pytest.mark.parametrize("causal", [True, False])
def test_window_reference_is_the_op_on_each_rows_band(causal):
    """o of every query row equals attention_bounds on that row alone with the keys outside its band dropped; rows
    that see no key give 0."""
    nq, nk, w = 40, 25, 9
    q, k, v = _qkv((1, 2, nq, 16), (1, 2, nk, 16), seed=6)
    ref, _ = window_attention_bounds(q, k, v, window=w, causal=causal, fmt="bf16")
    for i in range(nq):
        d = i + nk - nq - torch.arange(nk)
        keep = ((d >= 0) & (d < w)) if causal else (d.abs() < w)
        if not keep.any():
            assert (ref["o"][:, :, i] == 0).all()
            continue
        one, _ = attention_bounds(q[:, :, i:i + 1], k[:, :, keep], v[:, :, keep], fmt="bf16")
        assert torch.allclose(ref["o"][:, :, i], one["o"][:, :, 0], rtol=0, atol=1e-12)
