// Decode kernel: Nq >= 1 new queries per (batch, head) against a key/value cache whose valid length differs per
// batch element and is read on the device (no reference counterpart: the reference has no inference path).
//
// The math is the forward's (fixed shift, no row max), and that is what makes a split over keys cheap: the partial
// results (sum_j p_j v_j, sum_j p_j) of disjoint key ranges simply add, with no rescaling.
//
//   * work item = (batch, kv head, row block, split).  The rows of a (batch, kv head) are its G * Nq (query, head in
//     group) pairs, numbered r = i * G + g (query-major: a block's causal limits stay close together), in blocks of
//     64 = one wgmma M tile.  All G query heads of a group therefore share every K / V tile load.
//   * warpgroup 0 : TMA producer (one thread): 128-key K and V tiles of the split's key range through mbarrier rings
//   * warpgroup 1 : the 64 rows.  Q (8 or 16 KB) is loaded with ordinary loads into the 128-byte-swizzled layout;
//                   per key tile the forward's step (key_tile.cuh): S = Q K^T -> P = exp2(S*c1 - c2) -> O += P V
//   * visible length T_b = min(cache_seqlens[b] + n_new, capacity); query i sees key j iff j < T_b and, causal,
//     j <= i + T_b - Nq (the forward's bottom-right rule with Nk = T_b).  The ceil(T_b / 128) tiles a block can see
//     are cut into n_split contiguous chunks on the device, so a cache allocated at full length costs nothing.
//   * n_split = 1: o is written directly.  Otherwise each split writes fp32 partials (O_s, l_s) and
//     decode_combine_kernel forms o = sum_s O_s / max(sum_s l_s, 1e-37) in split order: o is bitwise reproducible.
//   * packed new tokens (cu_q set): batch element b brings n_b = cu_q[b + 1] - cu_q[b] queries at packed rows
//     [cu_q[b], cu_q[b + 1]) of q and o (q_sb = o_sb = 0), read on the device after pdl_wait (seq_span).  Nq and R of
//     the rules above become n_b and R_b = G * n_b; the grid is sized by the maximum (a.Nq), and a row block at or past
//     R_b has no work.
//   * rolling cache (ring = C > 0, WINDOW kernels only): the cache is a ring of C rows, absolute position p at row
//     p mod C.  cache_seqlens[b] counts every token the element has seen and may exceed C; L_b and T_b are not clamped,
//     and the tile ranges, split chunks and masks stay in absolute positions.  Absolute tile t is read from ring row
//     (128 t) mod C (C is a multiple of 128, so a tile never straddles the wrap).  The host checks C >= W + Nq - 1: the
//     keys a call sees, [T_b - Nq - W + 1, T_b), then still hold their own positions after its append.  A ring row
//     past T_b in a tile holds an older position or was never written: the select gives P = 0 there, and V's rows
//     past T_b are zeroed as before.
#pragma once

#include "key_tile.cuh"

namespace fcsa {

struct DecodeArgs {
  int B, H, KVH, G;          // G = H / KVH query heads per kv head
  int Nq, cap, n_new;        // new queries, cache rows (capacity), rows the append pass added at cache_seqlens[b]
                             // (packed: 1 = each sequence appended its own n_b rows, 0 = none); Nq: packed, the maximum
  int causal;
  int R, n_rb, n_split;      // R = G * Nq rows per (batch, kv head) (packed: of the longest), in n_rb blocks of 64;
                             // key splits
  float c1;                  // scale * log2(e)
  float c2;                  // shift * log2(e)
  int ring;                  // rolling cache (WINDOW kernels only): C = cap ring rows, position p at row p mod C; 0 = none
  const int32_t* seqlens;    // (B,) valid cache rows before the call
  const void* q;             // (B, H, Nq, D), element strides, feature dim contiguous
  long long q_sb, q_sh, q_sn;
  void* o;
  long long o_sb, o_sh, o_sn;
  float* part;               // n_split > 1: O_s [item][split][64][D], then l_s [item][split][64] (fp32)
  const int32_t* cu_q;       // packed new tokens: (B + 1,) cumulative counts over q's and o's rows; nullptr = dense
  int total_q;               // packed: rows of q and o
};

// The queries of batch element b: dense, the a.Nq rows of q's batch b; packed, the n_b rows of sequence b from packed
// row `start` (clamped as seq_span does).  The rows of the (batch, kv head) are R = G * Nq.
struct DecodeRows {
  int Nq, start;
};
__device__ __forceinline__ DecodeRows decode_rows(const DecodeArgs& a, int b) {
  if (a.cu_q == nullptr) return {a.Nq, 0};
  const SeqSpan s = seq_span(a.cu_q, b, a.Nq, a.total_q);
  return {s.len, s.start};
}

template <int D>
struct DecodeCfg {
  static constexpr int kTile = 128 * D * 2;           // bytes of one 128-key operand tile
  static constexpr int kQ = 64 * D * 2;               // the 64-row Q tile
  static constexpr int kStages = 3;                   // K / V ring depth
  static constexpr int kOffQ = 0;
  static constexpr int kOffK = kQ;
  static constexpr int kOffV = kOffK + kStages * kTile;
  static constexpr int kOffBar = kOffV + kStages * kTile;
  static constexpr int kSmem = kOffBar + 256 + 1024;  // + alignment slack
  static constexpr int kThreads = 256;                // producer warpgroup + one consumer warpgroup
  // D = 64: two CTAs per SM (105 KB of shared memory each), the consumer takes most of the register pool
  static constexpr int kCtasPerSm = D == 64 ? 2 : 1;
  static_assert(kSmem * kCtasPerSm <= 232448, "decode kernel shared memory");
};

// WINDOW: sliding-window attention (Windowed<DecodeArgs>::window = W).  A row block's visible tiles start at the tile of
// its smallest lower limit; the split cuts [t_lo, t_hi) into n_split chunks.
template <typename T, int D, bool WINDOW = false>
__global__ void __launch_bounds__(256, DecodeCfg<D>::kCtasPerSm)
fcsa_decode_kernel(const __grid_constant__ CUtensorMap tm_k, const __grid_constant__ CUtensorMap tm_v,
                   const std::conditional_t<WINDOW, Windowed<DecodeArgs>, DecodeArgs> a) {
  using Cfg = DecodeCfg<D>;
  constexpr int S = Cfg::kStages, TILE = Cfg::kTile, DCH = D / 64;

  uint8_t* smem = smem_1024();
  const uint32_t sQ = smem_u32(smem + Cfg::kOffQ);
  const uint32_t sK = smem_u32(smem + Cfg::kOffK);
  const uint32_t sV = smem_u32(smem + Cfg::kOffV);
  const uint32_t bar0 = smem_u32(smem + Cfg::kOffBar);
  auto BAR = [&](int i) { return bar0 + 8u * i; };
  constexpr int K_FULL = 0, K_EMPTY = K_FULL + S, V_FULL = K_EMPTY + S, V_EMPTY = V_FULL + S, NBARS = V_EMPTY + S;
  static_assert(NBARS * 8 <= 256, "barrier area");
  const Ring<S> kr = {BAR(K_FULL), BAR(K_EMPTY)}, vr = {BAR(V_FULL), BAR(V_EMPTY)};

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg = warp >> 2;
  pdl_launch_dependents();

  // ---- work item: (batch, kv head, row block, split), split fastest ------------------------
  const int item = blockIdx.x / a.n_split;
  const int split = blockIdx.x - item * a.n_split;
  const int bh = item / a.n_rb;
  const int rb = item - bh * a.n_rb;
  const int b = bh / a.KVH, hk = bh - b * a.KVH;
  const int r0 = rb * 64;

  if (threadIdx.x == 0) {
    kr.init(1, 128);
    vr.init(1, 128);
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();          // q (normalised by the append pass), the caches, cache_seqlens and cu_q are read from here on

  // this element's queries: a block past its rows has no work (packed; the combine skips its rows)
  const DecodeRows qs = decode_rows(a, b);
  const int R = a.G * qs.Nq;
  if (r0 >= R) return;
  const int r_last = min(r0 + 63, R - 1);

  // visible keys and this split's key tiles (uniform over the CTA); a ring's lengths are absolute and not clamped
  int ring = 0;
  if constexpr (WINDOW) ring = a.ring;
  const int L0 = max(a.seqlens[b], 0), L = ring ? L0 : min(L0, a.cap);
  const int Tn = L + (a.cu_q != nullptr ? (a.n_new ? qs.Nq : 0) : a.n_new);
  const int Tb = ring ? Tn : min(Tn, a.cap);
  const int off = diag_off(qs.Nq, Tb);
  int W = 0;                                  // the window
  if constexpr (WINDOW) W = a.window;
  // the tiles the block's queries r0 / G .. r_last / G see (the forward's rule with Nk = T_b), and this split's chunk
  const TileRange chunk =
      split_chunk(key_tiles<WINDOW>(r0 / a.G, r_last / a.G, off, Tb, a.causal, W), split, a.n_split);
  const int j0 = chunk.lo, j1 = chunk.hi;

  if (wg == 0) {
    // =============================== TMA producer ===============================
    if constexpr (Cfg::kCtasPerSm == 2) reg_dealloc<40>();
    if (warp == 0 && elect_one() && j1 > j0) {
      tma_prefetch_desc(&tm_k);
      tma_prefetch_desc(&tm_v);
      if (ring) load_kv_tiles<D>(&tm_k, &tm_v, kr, vr, sK, sV, j0, j1, [=](int j) { return (j * 128) % ring; }, hk, b);
      else load_kv_tiles<D>(&tm_k, &tm_v, kr, vr, sK, sV, j0, j1, TileRows{0}, hk, b);
    }
    return;
  }

  // =============================== consumer warpgroup ============================
  if constexpr (Cfg::kCtasPerSm == 2) reg_alloc<216>();     // 128 x 40 + 128 x 216 = 256 x 128
  const int t = threadIdx.x - 128;
  const int wl = warp & 3;
  const int row_a = 16 * wl + (lane >> 2);    // this thread's rows of the block: row_a and row_a + 8
  const int cq = 2 * (lane & 3);

  if (j1 > j0) {
    // Q: row r of the block is query i = r / G of head hk * G + r % G; rows past R are zero (and not read: packed,
    // they belong to the next sequence).  Every 64-feature chunk is a 64 x 128-byte SWIZZLE_128B tile (8 KB), the
    // layout a TMA box would leave.
    constexpr int CH = D / 8;                 // 16-byte pieces per row
    const T* qb = static_cast<const T*>(a.q) + b * a.q_sb + (long long)qs.start * a.q_sn;
#pragma unroll
    for (int k = 0; k < 64 * CH / 128; ++k) {
      const int idx = t + 128 * k, row = idx / CH, c = idx - (idx / CH) * CH;
      const int r = r0 + row;
      uint4 v = make_uint4(0, 0, 0, 0);
      if (r < R) {
        const int i = r / a.G, h = hk * a.G + (r - i * a.G);
        v = __ldg(reinterpret_cast<const uint4*>(qb + h * a.q_sh + (long long)i * a.q_sn + c * 8));
      }
      *reinterpret_cast<uint4*>(smem + Cfg::kOffQ + (c >> 3) * 8192 + sw128_offset(row, c & 7)) = v;
    }
    fence_proxy_async_smem();
    named_bar_sync(1, 128);
  }

  // the visible key columns of each of the thread's rows (none for a padding row past R)
  ColRange lim[2];
#pragma unroll
  for (int hf = 0; hf < 2; ++hf) {
    const int r = r0 + row_a + 8 * hf;
    lim[hf] = r >= R ? ColRange{0, -1} : row_key_cols<WINDOW>(r / a.G, off, Tb, a.causal, W);
  }
  const float c1 = a.c1;

  float o[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) o[i] = 0.f;
  float l[2] = {0.f, 0.f};

  for (int j = j0; j < j1; ++j) {
    const int n = j - j0;                     // the rings' use
    float sacc[64];
    const int s = kr.wait(n);
    qk_tile<T, D>(sacc, sQ, 8192, sK + s * TILE);
    kr.release(n);

    // (a select: cache rows past T_b may hold anything)
    const int col0 = j * 128;
    const bool need_mask = !tile_visible<WINDOW>(r0 / a.G, r_last / a.G, col0, col0 + 127, off, Tb, a.causal, W);
    uint32_t pf[32];
    exp_tile<T, WINDOW>(need_mask, sacc, pf, l, c1, col0, cq, lim, ShiftOnly{-a.c2}, AllKeys{});

    vr.wait(n);
    if (col0 + 128 > Tb) {
      // the tile runs past T_b: its rows there are zeroed (P = 0 there, but 0 * NaN would not be 0)
      const int valid = Tb - col0;
      for (int idx = t; idx < (128 - valid) * 8 * DCH; idx += 128) {
        const int row = valid + idx / (8 * DCH), rem = idx % (8 * DCH);
        *reinterpret_cast<uint4*>(smem + Cfg::kOffV + s * TILE + (rem >> 3) * 16384 + row * 128 + (rem & 7) * 16) =
            make_uint4(0, 0, 0, 0);
      }
      fence_proxy_async_smem();
      named_bar_sync(1, 128);
    }
    pv_tile<T>(o, pf, sV + s * TILE);
    vr.release(n);
  }

  // ---- epilogue --------------------------------------------------------------------------
#pragma unroll
  for (int hf = 0; hf < 2; ++hf) l[hf] = quad_sum(l[hf]);
  if (a.n_split == 1) {
    // (the span read again: volatile loads, not kept live through the key loop)
    const DecodeRows qe = decode_rows(a, b);
    T* ob = static_cast<T*>(a.o) + b * a.o_sb + (long long)qe.start * a.o_sn;
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
      const int r = r0 + row_a + 8 * hf;
      if (r >= a.G * qe.Nq) continue;
      const int i = r / a.G, h = hk * a.G + (r - i * a.G);
      store_row(ob + h * a.o_sh + (long long)i * a.o_sn, o, hf, cq, 1.0f / fmaxf(l[hf], 1e-37f));
    }
    return;
  }
  // every split writes its partials, an empty one zeros
  const long long slot = (long long)item * a.n_split + split;
  const long long n_slots = (long long)a.B * a.KVH * a.n_rb * a.n_split;
  float* po = a.part + slot * 64 * D;
  float* pl = a.part + n_slots * 64 * D + slot * 64;
#pragma unroll
  for (int hf = 0; hf < 2; ++hf) {
    const int row = row_a + 8 * hf;
    store_row(po + row * D, o, hf, cq, 1.f);
    if ((lane & 3) == 0) pl[row] = l[hf];
  }
}

// o = sum_s O_s / max(sum_s l_s, 1e-37), the splits summed in order.  One thread per 4 features of a row.
template <typename T, int D>
__global__ void __launch_bounds__(256) decode_combine_kernel(const DecodeArgs a) {
  pdl_launch_dependents();
  pdl_wait();
  constexpr int QD = D / 4;
  const long long n_items = (long long)a.B * a.KVH * a.n_rb;
  const long long idx = (long long)blockIdx.x * 256 + threadIdx.x;
  if (idx >= n_items * 64 * QD) return;
  const int qd = (int)(idx % QD);
  const int row = (int)((idx / QD) % 64);
  const long long item = idx / (64 * QD);
  const int rb = (int)(item % a.n_rb);
  const int bh = (int)(item / a.n_rb);
  const int b = bh / a.KVH, hk = bh - b * a.KVH;
  const int r = rb * 64 + row;
  const DecodeRows qs = decode_rows(a, b);
  if (r >= a.G * qs.Nq) return;
  const float* po = a.part + (item * a.n_split * 64 + row) * D + 4 * qd;
  const float* pl = a.part + n_items * a.n_split * 64 * D + item * a.n_split * 64 + row;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  float l = 0.f;
  // the loop is latency-bound (few rows, many splits): eight splits' loads are issued before they are summed, in
  // split order as one at a time would
  constexpr int SB = 8;
  int s = 0;
  for (; s + SB <= a.n_split; s += SB) {
    float4 v[SB];
    float lv[SB];
#pragma unroll
    for (int u = 0; u < SB; ++u) {
      v[u] = *reinterpret_cast<const float4*>(po + (long long)(s + u) * 64 * D);
      lv[u] = pl[(s + u) * 64];
    }
#pragma unroll
    for (int u = 0; u < SB; ++u) {
      acc.x += v[u].x; acc.y += v[u].y; acc.z += v[u].z; acc.w += v[u].w;
      l += lv[u];
    }
  }
  for (; s < a.n_split; ++s) {
    const float4 v = *reinterpret_cast<const float4*>(po + (long long)s * 64 * D);
    acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    l += pl[s * 64];
  }
  const float inv = 1.0f / fmaxf(l, 1e-37f);
  const int i = r / a.G, h = hk * a.G + (r - i * a.G);
  T* orow = static_cast<T*>(a.o) + b * a.o_sb + h * a.o_sh + (long long)(qs.start + i) * a.o_sn + 4 * qd;
  *reinterpret_cast<uint2*>(orow) = make_uint2(pack2<T>(acc.x * inv, acc.y * inv), pack2<T>(acc.z * inv, acc.w * inv));
}

// bytes of the partials of n_split > 1
inline size_t decode_partial_bytes(long long items, int n_split, int D) {
  return n_split > 1 ? (size_t)items * n_split * 64 * (D + 1) * sizeof(float) : 0;
}

}  // namespace fcsa
