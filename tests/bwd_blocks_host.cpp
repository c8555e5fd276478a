// extern "C" wrappers over the backward's work-item rules of csrc/tile_ranges.h for tests/test_bwd_blocks_host.py,
// which builds this file with the host compiler and loads it with ctypes.  w_begin = 0 asks for the unwindowed
// instantiation (one entry); otherwise one entry per window of [w_begin, w_end).
#include "../flash_cosine_sim_attention_b200/csrc/tile_ranges.h"

using namespace fcsa;

extern "C" {

int fcsa_bwd_block_keys(int D, int bias, int dq, int head_loop) {
  return bwd_block_keys(D, bias != 0, dq != 0, head_loop != 0);
}

// The query tiles of the `keys` keys from key0 (a work item's, or one warpgroup's with keys = 64), Nk keys in all.
void fcsa_key_block_query_tiles(int key0, int keys, int nq, int nk, int causal, int w_begin, int w_end, int* lo,
                                int* hi) {
  const int off = diag_off(nq, nk), nqt = row_blocks(nq, 64);
  if (w_begin == 0) {
    const TileRange t = key_block_query_tiles<false>(key0, keys, nk, off, nqt, causal, 0);
    lo[0] = t.lo, hi[0] = t.hi;
    return;
  }
  for (int w = w_begin; w < w_end; ++w) {
    const TileRange t = key_block_query_tiles<true>(key0, keys, nk, off, nqt, causal, w);
    lo[w - w_begin] = t.lo, hi[w - w_begin] = t.hi;
  }
}

}  // extern "C"
