// Which tiles a work item visits, which of them the forward and decode must mask per element, and the host rules that
// size the grids from the same quantities: the one definition, for the three attention kernels (device), the launch
// code (host) and the CPU tests
// (tests/tile_ranges_host.cpp compiles this header with the host compiler alone).
//
// Visibility is the public rule: query i sees key j iff j <= i + (Nk - Nq) when causal (bottom-right aligned), and,
// with a window W, iff 0 <= i + (Nk - Nq) - j < W (causal) or |i + (Nk - Nq) - j| < W.  Keys come in tiles of 128,
// the backward's query rows in tiles of 64.
//
// Plain C++17, no CUDA includes.  Every function takes and returns integers and inlines into its caller; WINDOW is a
// template parameter so that the unwindowed instantiations contain no window arithmetic.
#pragma once

#if defined(__CUDACC__)
#define FCSA_TILE_FN __host__ __device__ __forceinline__
#else
#define FCSA_TILE_FN inline
#endif

namespace fcsa {

struct TileRange {
  int lo, hi;          // tiles [lo, hi)
};

FCSA_TILE_FN int tile_min(int a, int b) { return a < b ? a : b; }
FCSA_TILE_FN int tile_max(int a, int b) { return a > b ? a : b; }
FCSA_TILE_FN int tile_count(TileRange t) { return tile_max(0, t.hi - t.lo); }

// The diagonal's offset: query i sits at column i + off.  The kernels compute it once and use the same value for their
// mask limits, so the functions below take it rather than Nq.
FCSA_TILE_FN int diag_off(int Nq, int Nk) { return Nk - Nq; }

// ---- key tiles of a range of query rows (forward, decode) ----------------------------------------------------------
// The 128-key tiles that query rows [r_first, r_last] (0 <= r_first <= r_last < Nq, off = diag_off) can see, inside [0, ceil(Nk / 128)):
// up to the tile of the last row's last column, from the tile of the smallest lower limit (the first row's).  The
// last column moves up by W - 1 when the window is not causal.  A range that sees no key has hi = 0 or lo = hi.
template <bool WINDOW>
FCSA_TILE_FN int last_key_col(int r_last, int off, int causal, int W) {         // causal or WINDOW
  return r_last + off + (WINDOW && !causal ? W - 1 : 0);
}
FCSA_TILE_FN int first_key_col(int r_first, int off, int W) {                   // WINDOW: the first row's lower limit
  return r_first + off - W + 1;
}
template <bool WINDOW>
FCSA_TILE_FN TileRange key_tiles(int r_first, int r_last, int off, int Nk, int causal, int W) {
  TileRange t = {0, (Nk + 127) >> 7};
  if (causal || WINDOW) {
    const int last_col = last_key_col<WINDOW>(r_last, off, causal, W);
    t.hi = last_col < 0 ? 0 : tile_min(t.hi, (last_col >> 7) + 1);
  }
  if constexpr (WINDOW) {
    const int first_col = first_key_col(r_first, off, W);
    t.lo = first_col <= 0 ? 0 : tile_min(first_col >> 7, t.hi);
  }
  return t;
}

// The forward's blocks: `rows` query rows from r0 (r0 < Nq), the last block ending with the sequence.
template <bool WINDOW>
FCSA_TILE_FN TileRange block_key_tiles(int r0, int rows, int Nq, int Nk, int off, int causal, int W) {
  return key_tiles<WINDOW>(r0, tile_min(r0 + rows - 1, Nq - 1), off, Nk, causal, W);
}

// The key tiles a forward warpgroup's own 64 rows (from r0) see, of its block's [blk_lo, blk_hi): the block's rules
// applied to its first and last row (the block's clip to Nk holds for them too).  On the block's other tiles every p
// of these rows is 0 (with 192-row blocks, the trailing causal tiles of the first warpgroups and all tiles of rows
// past the end), so the warpgroup only passes their ring slots on.
template <bool WINDOW>
FCSA_TILE_FN TileRange warpgroup_key_tiles(int r0, int blk_lo, int blk_hi, int Nq, int off, int causal, int W) {
  TileRange t = {blk_lo, blk_hi};
  if (r0 >= Nq) {
    t.hi = 0;
  } else if (causal || WINDOW) {
    const int last_col = last_key_col<WINDOW>(tile_min(r0 + 63, Nq - 1), off, causal, W);
    t.hi = last_col < 0 ? 0 : (last_col >> 7) + 1;
  }
  if constexpr (WINDOW) {
    const int first_col = first_key_col(r0, off, W);
    if (first_col > 0) t.lo = tile_max(blk_lo, first_col >> 7);
  }
  return t;
}

// Decode: the split-th of n_split contiguous chunks of a row block's tiles.
FCSA_TILE_FN TileRange split_chunk(TileRange t, int split, int n_split) {
  return {t.lo + (int)((long long)(t.hi - t.lo) * split / n_split),
          t.lo + (int)((long long)(t.hi - t.lo) * (split + 1) / n_split)};
}

// ---- the masks of the forward and decode exp stages --------------------------------------------------------------
// The key columns [lo, hi] (inclusive) that query i sees among Nk keys: the per-element limits of a masked tile.
struct ColRange {
  int lo, hi;
};
template <bool WINDOW>
FCSA_TILE_FN ColRange row_key_cols(int i, int off, int Nk, int causal, int W) {
  ColRange c = {0, causal ? tile_min(Nk - 1, i + off) : Nk - 1};
  if constexpr (WINDOW) {
    c.lo = i + off - W + 1;
    if (!causal) c.hi = tile_min(Nk - 1, i + off + W - 1);
  }
  return c;
}

// True iff every key of [k_first, k_last] exists and is visible to every query of [q_first, q_last]: such a tile
// needs no per-element selects.  Only the corners decide: the causal limit and the window's upper side are smallest
// for the first query, the window's lower side largest for the last.
template <bool WINDOW>
FCSA_TILE_FN bool tile_visible(int q_first, int q_last, int k_first, int k_last, int off, int Nk, int causal, int W) {
  bool all = k_last < Nk && !(causal && k_last > q_first + off);
  if constexpr (WINDOW) all = all && !(k_first < q_last + off - W + 1 || k_last > q_first + off + W - 1);
  return all;
}

// ---- query tiles of a key tile (backward) --------------------------------------------------------------------------
// With a window, the visible query rows of key j are [j + lo_off, j + window_hi_off]; the backward's consumers keep
// this one offset for both of a thread's key rows.
FCSA_TILE_FN int window_hi_off(int off, int W) { return W - 1 - off; }

// The 64-row query tiles [lo, hi) that the `keys` keys from key0 (128: a key tile) are visible to, nqt = ceil(Nq / 64)
// tiles in all: from the first tile with a row that can see key0 (causal: 64 i + 63 + off >= key0; a non-causal
// window: whose band reaches key0) to, with a window, the tile of the last query row whose lower limit is at most
// key0 + keys - 1.
template <bool WINDOW>
FCSA_TILE_FN TileRange query_tiles(int key0, int off, int nqt, int causal, int W, int keys = 128) {
  TileRange t = {0, nqt};
  if (causal || WINDOW) {
    const int x = key0 - off - 63 - (WINDOW && !causal ? W - 1 : 0);
    t.lo = x <= 0 ? 0 : (x + 63) / 64;
  }
  if constexpr (WINDOW) {
    const int last_row = key0 + keys - 1 - off + W - 1;
    t.hi = last_row < 0 ? 0 : tile_min(nqt, last_row / 64 + 1);
  }
  return t;
}

// Keys of one backward work item: three consumer warpgroups of 64 keys for the D = 64 kernels that compute dQ without
// a bias or a head loop (BwdCfg), two for the others.  A head loop runs where the split rule (bwd_group_split) sizes
// the grid to about fill the device with 128-key CTAs: 192-key items would leave it at 1.33 waves.
constexpr int bwd_block_keys(int D, bool bias, bool dq, bool head_loop = false) {
  return D == 64 && !bias && dq && !head_loop ? 192 : 128;
}

// The query tiles that the existing keys among the `keys` from key0 see, Nk keys in all: a 192-key work item's
// (keys = 192) or one of its warpgroups' (key0 + 64 w, keys = 64).  Empty when key0 >= Nk.  The warpgroups' ranges
// tile the item's: a key's visible rows form one interval that moves up by one row per key, so the item's range is the
// first warpgroup's lower end to the last existing warpgroup's upper end, and a tile between them is some warpgroup's.
template <bool WINDOW>
FCSA_TILE_FN TileRange key_block_query_tiles(int key0, int keys, int Nk, int off, int nqt, int causal, int W) {
  const int n = tile_min(keys, Nk - key0);
  if (n <= 0) return {0, 0};
  return query_tiles<WINDOW>(key0, off, nqt, causal, W, n);
}

// A backward CTA with several query heads works through one flat sequence of hpc * NI tiles, NI = max(0, hi - lo) per
// head: flat index i is query tile lo + i % NI of head i / NI.
struct HeadTile {
  int head, qt;
};
FCSA_TILE_FN HeadTile head_tile(int i, int i_lo, int NI, bool head_loop) {
  const int hh = head_loop ? i / NI : 0;
  return {hh, i_lo + i - hh * NI};
}

// The same sequence as the consumers step it, by first row: row0 restarts at i_lo * 64 with every head, after the
// head's last tile - the one that ends the q_end rows (the padded length, or the sequence's: a head's last tile ends
// at ceil(Nq / 64) * 64, so row0 + 64 < Nq says whether row0 is before it) or, with a window, once row0 + 64 passes
// key0 + 127 + hi_off, the last row seeing a key of the tile (hi_off = window_hi_off; this is tile hi - 1 of
// query_tiles, told from the offset the consumers hold anyway rather than from hi kept live through their loop).
template <bool WINDOW>
FCSA_TILE_FN int next_row0(int row0, int i_lo, int q_end, int key0, int hi_off) {
  const bool in_head = row0 + 64 < q_end && (!WINDOW || row0 + 64 <= key0 + 127 + hi_off);
  return in_head ? row0 + 64 : i_lo * 64;
}

// ---- packed sequences ----------------------------------------------------------------------------------------------
// The stats and the dq accumulator hold, per query head, varlen_tiles tiles of 64 rows.  Sequence b starts at tile
// varlen_tile_base (start = its first query row), which needs no prefix sum on the device and leaves room for
// ceil(len_b / 64) tiles before the base of b + 1; every tile index stays below total_q / 64 + B + 1.
FCSA_TILE_FN int varlen_tile_base(int start, int b) { return start / 64 + b; }
inline int varlen_tiles(int B, long long total_q) { return (int)(total_q / 64 + B + 1); }

// ---- host: the grids ------------------------------------------------------------------------------------------------
// Query rows of one forward CTA: three consumer warpgroups of 64 rows for D = 64, two for D = 128 (FwdCfg).
constexpr int fwd_block_rows(int D) { return D == 64 ? 192 : 128; }

// Query rows of one CTA of the deterministic backward's dQ kernel: two consumer warpgroups of 64 rows.
constexpr int dq_block_rows = 128;

// Blocks of `rows` rows that cover n rows: the forward's query blocks, the dQ kernel's, decode's row blocks.
inline int row_blocks(int n, int rows) { return (n + rows - 1) / rows; }

// Decode splits per work item: 1 when the items alone fill the SMs, otherwise the fewest that do, at most one per key
// tile of the capacity.  With a window, `cap` is decode_window_keys.
inline int decode_split(long long items, int cap, int sm_count) {
  if (items >= sm_count) return 1;
  const long long want = (sm_count + items - 1) / items;
  const long long tiles = (cap + 127) / 128;
  return (int)(want < tiles ? want : tiles);
}

// A bound on the keys whose tiles one row block can see under a window W: its rows span at most 64 queries, so its
// keys lie in a range of 64 + W - 2 (causal) or 64 + 2 W - 3 keys, which touches at most ceil(range / 128) + 1 tiles.
// The split rule then bounds a block's tiles by the window instead of the capacity.
inline int decode_window_keys(int cap, int window, bool causal) {
  const long long range = 64LL + (causal ? 1 : 2) * (long long)window;
  const long long keys = range + 128;
  return (int)(keys < cap ? keys : cap);
}

// Slices per key/value-head group (query heads per CTA = G / split).  One CTA per group keeps dk / dv in registers
// (no accumulator, no finish pass, bitwise reproducible), but the grid then has B * kv_heads * key tiles CTAs; below
// one CTA per SM the group is split into the fewest slices that fill the device.  Keys/values shared by all heads
// (kv_heads == 1) and the BIAS kernels (no registers to spare for the head loop) take one query head per CTA.
// The rule counts 128-key CTAs for every kernel, so which path a shape takes does not depend on the head dim; a grid of
// 192-key items that stays unsplit between 2/3 of a wave and one wave still keeps dk / dv in registers.
inline int bwd_group_split(int B, int H, int kv_heads, int Nk, bool bias, int sm_count) {
  const int G = H / kv_heads;
  if (G == 1) return 1;
  if (bias || kv_heads == 1) return G;
  const long long unsplit = (long long)((Nk + 127) / 128) * B * kv_heads;
  if (unsplit >= sm_count) return 1;
  for (int s = 2; s < G; ++s)
    if (G % s == 0 && unsplit * s >= sm_count) return s;
  return G;
}

}  // namespace fcsa
