// dQ of the deterministic backward: the forward's loop over a query block's key tiles, with one more product.
//
// One CTA = 128 query rows of one (batch, query head), or of one sequence (VARLEN).  Warpgroup 0 is the TMA producer:
// Q and dO of the block once, then the K and V tiles of block_key_tiles through two Rings (load_kv_tiles).  Warpgroups
// 1 and 2 own 64 rows each and visit their warpgroup_key_tiles in ascending order; per key tile:
//     S  = Q K^T, dP = dO V^T                    qk_tile (both operands in shared memory)
//     P  = exp2(S*c1 + c3), masked               fp32, with the forward's selects (row_key_cols / tile_visible,
//                                                the key-padding mask, the window)
//     dS = P (dP - delta)                        fp32, rounded to T once, as the A fragments of
//     dQ += dS K                                 pv_tile with the K slot as the B operand
// c3 and -delta are the stats bwd_prep_kernel wrote.  These are the rounding points of fcsa_bwd_kernel, and every sum
// has a fixed order: dq is bitwise the same from run to run, whatever the grid.  The epilogue writes scale * dQ once
// (with q_rnorm: the l2norm backward w.r.t. the raw q, from the resident Q tile), as T or float32, for every row below
// Nq; a row that sees no key gets 0.
#pragma once

#include "bwd_kernel.cuh"
#include "fwd_kernel.cuh"

namespace fcsa {

template <int D>
struct DqCfg {
  static constexpr int kBlockM = dq_block_rows;         // query rows of one CTA: two consumer warpgroups of 64
  static constexpr int kTile = 128 * D * 2;             // bytes of one 128-row K / V tile
  static constexpr int kQ = kBlockM * D * 2;            // bytes of the Q (or dO) tile
  static constexpr int kStages = (D == 64) ? 4 : 2;     // K / V ring depth
  static constexpr int kOffQ = 0;
  static constexpr int kOffDO = kQ;
  static constexpr int kOffK = 2 * kQ;
  static constexpr int kOffV = kOffK + kStages * kTile;
  static constexpr int kOffBar = kOffV + kStages * kTile;
  static constexpr int kSmem = kOffBar + 256 + 1024;    // + alignment slack
  static constexpr int kThreads = 384;                  // producer warpgroup + 2 consumer warpgroups
  static_assert(kQ % 1024 == 0, "operand tiles start on 1024-byte swizzle atoms");
  static_assert(kSmem <= 232448, "dQ kernel shared memory");
};

struct DqArgs {
  int B, H, Nq, Nk, causal, has_mask;
  int group;                        // query heads per key/value head: head h reads kv head h / group
  int n_qblk;                       // ceil(Nq / 128)
  int nqt;                          // stats tiles per (batch, head) (bwd_workspace_layout)
  float c1;                         // scale * log2e
  float scale;
  const uint8_t* mask; long long mask_sb;
  const float* stats;
  int out_f32;                      // 1: dq is float32 (strides in float32 elements)
  void* dq; long long dq_sb, dq_sh, dq_sn;
  // fused l2norm: q is the normalised q_hat and dq the gradient w.r.t. the raw queries; q_rnorm (B, H, Nq, groups)
  // or nullptr
  const float* q_rnorm;
  int groups;
};

// Packed sequences: q, d_o, dq are (total_q, H, D) and k, v (total_k, kv_heads, D) (dq_sb unused); the stats of head h,
// sequence b start at tile h * ntile + base(b) (bwd_varlen_workspace_layout) and q_rnorm is [H][total_q][groups].
struct DqVarlenArgs : DqArgs {
  const int* cu_q;
  const int* cu_k;
  int total_q, total_k, ntile;
};

template <bool VARLEN, bool WINDOW>
using DqArgsOf = std::conditional_t<WINDOW, Windowed<std::conditional_t<VARLEN, DqVarlenArgs, DqArgs>>,
                                    std::conditional_t<VARLEN, DqVarlenArgs, DqArgs>>;

template <typename T, int D, bool VARLEN = false, bool WINDOW = false>
__global__ void __launch_bounds__(384, 1)
fcsa_dq_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_k,
               const __grid_constant__ CUtensorMap tm_v, const __grid_constant__ CUtensorMap tm_do,
               const DqArgsOf<VARLEN, WINDOW> a) {
  static_assert(D == 64 || D == 128, "head dim 64 or 128");
  using Cfg = DqCfg<D>;
  constexpr int S = Cfg::kStages, TILE = Cfg::kTile, DCH = D / 64, BM = Cfg::kBlockM;

  uint8_t* smem = smem_1024();
  const uint32_t sQ = smem_u32(smem + Cfg::kOffQ);
  const uint32_t sDO = smem_u32(smem + Cfg::kOffDO);
  const uint32_t sK = smem_u32(smem + Cfg::kOffK);
  const uint32_t sV = smem_u32(smem + Cfg::kOffV);
  const uint32_t bar0 = smem_u32(smem + Cfg::kOffBar);
  auto BAR = [&](int i) { return bar0 + 8u * i; };
  constexpr int Q_FULL = 0, K_FULL = 1, K_EMPTY = K_FULL + S, V_FULL = K_EMPTY + S, V_EMPTY = V_FULL + S,
                NBARS = V_EMPTY + S;
  static_assert(NBARS * 8 <= 256, "barrier area");
  const Ring<S> kr = {BAR(K_FULL), BAR(K_EMPTY)}, vr = {BAR(V_FULL), BAR(V_EMPTY)};

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg = warp >> 2;
  pdl_launch_dependents();

  // ---- work item: BM query rows of one (batch, head), numbered as the forward's: heaviest causal blocks first, the
  // query heads of one kv group in consecutive CTAs ----
  const int bh_count = a.B * a.H;
  const int rank = blockIdx.x / bh_count;
  const int bh = blockIdx.x - rank * bh_count;
  const int qblk = a.causal ? (a.n_qblk - 1 - rank) : rank;
  const int b = bh / a.H, h = bh - b * a.H;
  const int hk = h / a.group;
  const int m0 = qblk * BM;
  const int tb = VARLEN ? 0 : b;
  int Nq = a.Nq, Nk = a.Nk, q_row0 = 0, k_row0 = 0;
  long long tile0 = ((long long)b * a.H + h) * a.nqt;      // the stats tile of query row 0
  long long rrow0 = ((long long)b * a.H + h) * a.Nq;       // the q_rnorm row of query row 0

  if (threadIdx.x == 0) {
    mbar_init(BAR(Q_FULL), 1);
    kr.init(1, 256);
    vr.init(1, 256);
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();          // the stats (preprocess kernel) and the lengths are read from here on
  if constexpr (VARLEN) {
    const SeqSpan sq = seq_span(a.cu_q, b, a.Nq, a.total_q), sk = seq_span(a.cu_k, b, a.Nk, a.total_k);
    Nq = sq.len; Nk = sk.len; q_row0 = sq.start; k_row0 = sk.start;
    if (m0 >= Nq) return;                                     // a query block past the end of its sequence
    tile0 = (long long)h * a.ntile + varlen_tile_base(q_row0, b);
    rrow0 = (long long)h * a.total_q + q_row0;
  }
  const int off = diag_off(Nq, Nk);
  int W = 0;                                                  // the window
  if constexpr (WINDOW) W = a.window;
  const TileRange blk = block_key_tiles<WINDOW>(m0, BM, Nq, Nk, off, a.causal, W);
  const int j_lo = blk.lo, NT = blk.hi;                       // the key tiles [j_lo, NT) this block visits

  if (wg == 0) {
    // =============================== TMA producer ===============================
    reg_dealloc<kProducerRegs>();
    if (warp == 0 && elect_one() && NT > j_lo) {
      tma_prefetch_desc(&tm_q);
      tma_prefetch_desc(&tm_do);
      tma_prefetch_desc(&tm_k);
      tma_prefetch_desc(&tm_v);
      mbar_expect_tx(BAR(Q_FULL), 2 * Cfg::kQ);
#pragma unroll
      for (int ch = 0; ch < DCH; ++ch) {
        tma_load_4d(sQ + ch * BM * 128, &tm_q, BAR(Q_FULL), ch * 64, q_row0 + m0, h, tb);
        tma_load_4d(sDO + ch * BM * 128, &tm_do, BAR(Q_FULL), ch * 64, q_row0 + m0, h, tb);
      }
      load_kv_tiles<D>(&tm_k, &tm_v, kr, vr, sK, sV, j_lo, NT, k_row0, hk, tb);
    }
    return;
  }

  // =============================== consumer warpgroups =========================
  reg_alloc<kConsumerRegs>();
  const int w = wg - 1;                       // which 64 of the block's BM query rows
  const int wl = warp & 3;
  const int r_blk = 64 * w + 16 * wl + (lane >> 2);   // the thread's rows inside the block: r_blk and r_blk + 8
  const int row_a = m0 + r_blk;
  const int cq = 2 * (lane & 3);              // first of the thread's two columns inside every 8-column block
  const float c1 = a.c1;
  // c3 and -delta of the thread's two rows (rows at or past Nq are never stored: 0)
  float c3[2], ndl[2];
#pragma unroll
  for (int hf = 0; hf < 2; ++hf) {
    const int row = row_a + 8 * hf;
    c3[hf] = ndl[hf] = 0.f;
    if (row < Nq) {
      const float* st = a.stats + (tile0 + (row >> 6)) * 128 + (row & 63);
      c3[hf] = __ldg(st);
      ndl[hf] = __ldg(st + 64);
    }
  }
  ColRange lim[2];
#pragma unroll
  for (int hf = 0; hf < 2; ++hf) lim[hf] = row_key_cols<WINDOW>(row_a + 8 * hf, off, Nk, a.causal, W);
  const PaddingMask keys = {a.mask + (long long)b * a.mask_sb, a.has_mask != 0};
  // the key tiles this warpgroup's own 64 rows see; it only passes the ring slots of the others on
  const TileRange wgt = warpgroup_key_tiles<WINDOW>(m0 + 64 * w, j_lo, NT, Nq, off, a.causal, W);

  // P = exp2(S*c1 + c3) (masked: a select, S may be anything there), dS = P (dP - delta) as 16-bit A fragments.
  // Element pair i: row hf = i & 1 of the thread's two, columns col0 + 8 (i >> 1) + cq and + 1.
  auto ds_tile = [&](auto masked_tag, const float (&s)[64], const float (&dp)[64], uint32_t (&dsf)[32], int col0) {
    constexpr bool MASKED = decltype(masked_tag)::value;
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int hf = i & 1;
      const int col = col0 + 8 * (i >> 1) + cq;
      float p0 = ex2_approx(fmaf(s[2 * i], c1, c3[hf]));
      float p1 = ex2_approx(fmaf(s[2 * i + 1], c1, c3[hf]));
      if constexpr (MASKED) {
        bool v0 = col <= lim[hf].hi, v1 = col + 1 <= lim[hf].hi;
        if constexpr (WINDOW) {
          v0 = v0 && col >= lim[hf].lo;
          v1 = v1 && col + 1 >= lim[hf].lo;
        }
        if (keys.on()) {
          v0 = v0 && keys(col);
          v1 = v1 && keys(col + 1);
        }
        p0 = v0 ? p0 : 0.f;
        p1 = v1 ? p1 : 0.f;
      }
      dsf[i] = pack2<T>(p0 * (dp[2 * i] + ndl[hf]), p1 * (dp[2 * i + 1] + ndl[hf]));
    }
  };

  float dq[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) dq[i] = 0.f;
  if (NT > j_lo) mbar_wait(BAR(Q_FULL), 0);
  const uint32_t sQw = sQ + w * 64 * 128, sDOw = sDO + w * 64 * 128;   // the warpgroup's rows of every chunk

  for (int j = j_lo; j < NT; ++j) {
    const int n = j - j_lo;                   // the rings' use
    if (j < wgt.lo || j >= wgt.hi) {
      kr.pass(n);
      vr.pass(n);
      continue;
    }
    float s[64], dp[64];
    const int st = kr.wait(n);
    qk_tile<T, D>(s, sQw, BM * 128, sK + st * TILE);
    vr.wait(n);
    qk_tile<T, D>(dp, sDOw, BM * 128, sV + st * TILE);
    vr.release(n);

    // (the warpgroup's 64 rows unclipped, as in the forward: rows past Nq are never stored)
    const int col0 = j * 128;
    const bool need_mask =
        a.has_mask || !tile_visible<WINDOW>(m0 + 64 * w, m0 + 64 * w + 63, col0, col0 + 127, off, Nk, a.causal, W);
    uint32_t dsf[32];
    if (need_mask) ds_tile(std::true_type{}, s, dp, dsf, col0);
    else ds_tile(std::false_type{}, s, dp, dsf, col0);

    pv_tile<T>(dq, dsf, sK + st * TILE);      // dQ += dS K: K is the MN-major B operand, as V is in P V
    kr.release(n);
  }

  // ---- epilogue: scale * dQ (+ the l2norm backward) -> global ------------------------------------------------
  // (no early exit for rows at or past Nq: the l2norm backward shuffles within the quad of a row)
#pragma unroll
  for (int hf = 0; hf < 2; ++hf) {
    const int row = row_a + 8 * hf;
    const bool in = row < Nq;
    // g[2 jb + e] = dq_hat of feature 8 jb + cq + e
    float g[D / 4];
#pragma unroll
    for (int jb = 0; jb < D / 8; ++jb) {
      g[2 * jb] = dq[4 * jb + 2 * hf] * a.scale;
      g[2 * jb + 1] = dq[4 * jb + 2 * hf + 1] * a.scale;
    }
    // (a block that visits no key tile has not loaded Q; its dq is 0 either way)
    if (a.q_rnorm != nullptr && NT > j_lo)
      l2norm_bwd_key_row<T, D>(g, a.q_rnorm, a.groups, sQ + (r_blk + 8 * hf) * 128, rrow0, row, in);
    if (!in) continue;
    const long long o_off = (long long)tb * a.dq_sb + (long long)h * a.dq_sh + (long long)(q_row0 + row) * a.dq_sn + cq;
    if (a.out_f32) {
      float* p = reinterpret_cast<float*>(a.dq) + o_off;
#pragma unroll
      for (int jb = 0; jb < D / 8; ++jb) *reinterpret_cast<float2*>(p + 8 * jb) = make_float2(g[2 * jb], g[2 * jb + 1]);
    } else {
      T* p = reinterpret_cast<T*>(a.dq) + o_off;
#pragma unroll
      for (int jb = 0; jb < D / 8; ++jb) *reinterpret_cast<uint32_t*>(p + 8 * jb) = pack2<T>(g[2 * jb], g[2 * jb + 1]);
    }
  }
}

}  // namespace fcsa
