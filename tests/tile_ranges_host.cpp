// extern "C" wrappers over csrc/tile_ranges.h for the CPU tests (tests/tile_ranges.py builds this file with the host
// compiler and loads it with ctypes).  A wrapper with [w_begin, w_end) fills one array entry per window W of that range
// with the WINDOW instantiation; w_begin = 0 asks for the unwindowed instantiation (one entry).
#include <type_traits>

#include "../flash_cosine_sim_attention_b200/csrc/tile_ranges.h"

using namespace fcsa;

namespace {
template <typename F>
void per_window(int w_begin, int w_end, int* lo, int* hi, F f) {
  if (w_begin == 0) {
    const TileRange t = f(std::false_type{}, 0);
    lo[0] = t.lo, hi[0] = t.hi;
    return;
  }
  for (int w = w_begin; w < w_end; ++w) {
    const TileRange t = f(std::true_type{}, w);
    lo[w - w_begin] = t.lo, hi[w - w_begin] = t.hi;
  }
}
}  // namespace

extern "C" {

void fcsa_block_key_tiles(int r0, int rows, int nq, int nk, int causal, int w_begin, int w_end, int* lo, int* hi) {
  per_window(w_begin, w_end, lo, hi,
             [&](auto win, int w) { return block_key_tiles<decltype(win)::value>(r0, rows, nq, nk, diag_off(nq, nk), causal, w); });
}

// blk_lo, blk_hi: the block's range per window (what fcsa_block_key_tiles filled)
void fcsa_warpgroup_key_tiles(int r0, const int* blk_lo, const int* blk_hi, int nq, int nk, int causal, int w_begin,
                              int w_end, int* lo, int* hi) {
  per_window(w_begin, w_end, lo, hi, [&](auto win, int w) {
    const int k = w ? w - w_begin : 0;
    return warpgroup_key_tiles<decltype(win)::value>(r0, blk_lo[k], blk_hi[k], nq, diag_off(nq, nk), causal, w);
  });
}

// the split-th chunk of the tiles queries [q_first, q_last] see among Tb keys
void fcsa_decode_chunk(int q_first, int q_last, int nq, int Tb, int causal, int split, int n_split, int w_begin,
                       int w_end, int* lo, int* hi) {
  per_window(w_begin, w_end, lo, hi, [&](auto win, int w) {
    return split_chunk(key_tiles<decltype(win)::value>(q_first, q_last, diag_off(nq, Tb), Tb, causal, w), split, n_split);
  });
}

void fcsa_query_tiles(int key0, int nq, int nk, int causal, int w_begin, int w_end, int* lo, int* hi) {
  per_window(w_begin, w_end, lo, hi, [&](auto win, int w) {
    return query_tiles<decltype(win)::value>(key0, diag_off(nq, nk), row_blocks(nq, 64), causal, w);
  });
}

// The flat (head, query tile) sequence of a backward CTA with hpc heads under every window of [w_begin, w_end), as the
// consumers step row0 and as head_tile splits the index: rows[w][i], qts[w][i] for i < steps, -1 past hpc * NI.
void fcsa_bwd_row0_sequence(int key0, int nq, int nk, int causal, int hpc, int w_begin, int w_end, int steps,
                            int* rows, int* qts) {
  for (int w = w_begin; w < w_end; ++w) {
    const TileRange qr = query_tiles<true>(key0, diag_off(nq, nk), row_blocks(nq, 64), causal, w);
    const int NI = tile_count(qr), NT = hpc * NI;
    int* r = rows + (long long)(w - w_begin) * steps;
    int* q = qts + (long long)(w - w_begin) * steps;
    for (int i = 0, row0 = qr.lo * 64; i < steps;
         ++i, row0 = next_row0<true>(row0, qr.lo, nq, key0, window_hi_off(diag_off(nq, nk), w))) {
      r[i] = i < NT ? row0 : -1;
      q[i] = i < NT ? head_tile(i, qr.lo, NI, true).qt : -1;
    }
  }
}

int fcsa_varlen_tile_base(int start, int b) { return varlen_tile_base(start, b); }
int fcsa_varlen_tiles(int B, long long total_q) { return varlen_tiles(B, total_q); }
int fcsa_fwd_block_rows(int D) { return fwd_block_rows(D); }
int fcsa_row_blocks(int n, int rows) { return row_blocks(n, rows); }
int fcsa_decode_split(long long items, int cap, int sm_count) { return decode_split(items, cap, sm_count); }
int fcsa_decode_window_keys(int cap, int window, int causal) { return decode_window_keys(cap, window, causal != 0); }
int fcsa_bwd_group_split(int B, int H, int kv_heads, int Nk, int bias, int sm_count) {
  return bwd_group_split(B, H, kv_heads, Nk, bias != 0, sm_count);
}

}  // extern "C"
