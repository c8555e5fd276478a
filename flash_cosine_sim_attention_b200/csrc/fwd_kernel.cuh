// Forward kernel: o = (sum_j exp(scale*q.k_j - shift) v_j) / max(sum_j exp(..), 1e-37)
//
// Replaces the reference's forward_kernel (flash_cosine_sim_attention_cuda.cu:1072-1247).
// Same math (fixed shift instead of a running row max, cu:1216; running row sum, cu:1236;
// final 1/max(l, eps) scaling, cu:1239-1246; bottom-right aligned causal mask, cu:1097/1210;
// key-padding mask, cu:1198-1212) - a different machine mapping:
//
//   * one CTA = BM query rows of one (batch, head) (FwdCfg: 192 for D = 64, 128 for D = 128); CTAs are
//     numbered heaviest first (causal: the last query blocks see the most keys), so the block scheduler
//     starts the long ones first
//   * warpgroup 0 : TMA producer (one thread): Q once, then K and V tiles of 128 keys through
//                   mbarrier rings; the warpgroup gives most of its registers to the consumers
//   * warpgroups 1 .. BM / 64: 64 query rows each.  Per key tile: S = Q K^T (wgmma, both operands in
//                   shared memory) -> P = exp2(S*c1 - c2) in registers -> O += P V (wgmma with P as the
//                   register A operand).  Because there is no row max there is no rescaling of O: the
//                   accumulator stays in registers until the epilogue.  The consumers share every K / V tile
//                   and run independently of each other, each waiting on its own products; three of them
//                   (D = 64) drift out of phase, so one's exps overlap another's products more often than two do.
#pragma once

#include "key_tile.cuh"

namespace fcsa {

struct FwdArgs {
  int B, H, Nq, Nk;
  int causal;        // bottom-right aligned: key j visible to query i iff j <= i + (Nk - Nq)
  int has_mask;      // key padding mask (B, Nk), nonzero = keep
  int group;         // query heads per key/value head (H / kv_heads): head h reads kv head h / group
  int n_qblk;        // ceil(Nq / FwdCfg<D>::kBlockM)
  float c1;          // scale * log2(e)
  float c2;          // shift * log2(e)
  const uint8_t* mask;
  long long mask_sb;
  void* o;
  long long o_sb, o_sh, o_sn;   // element strides of o (feature dim contiguous)
  int o_f32;                    // 1: o is float32 (strides in float32 elements), else the operand type
  float* inv_l;                 // (B, H, Nq) fp32, contiguous
  // additive bias on the logits (reference py:312, cu:1168,1214): element type = q's, [b][h][i][j] with
  // element strides (bias_sb = 0 when the bias has no batch dimension); rows are 16-byte aligned and
  // hold at least ceil8(Nk) elements.  Only read by the BIAS instantiation.
  const void* bias;
  long long bias_sb, bias_sh, bias_sn;
  const float* bias_amax;       // optional device scalar: shift += max(*bias_amax, 0)  (fp16 range guard)
};

// Packed sequences (VARLEN instantiation): B sequences, Nq / Nk = the maximum lengths (they size the grid and clamp
// the device lengths).  q is (total_q, H, D) and k, v (total_k, kv_heads, D), addressed by tensor maps of batch extent
// 1; sequence b owns query rows [cu_q[b], cu_q[b + 1]) and key rows [cu_k[b], cu_k[b + 1]).  o has q's layout (o_sb is
// unused) and inv_l is (H, total_q).
struct FwdVarlenArgs : FwdArgs {
  const int* cu_q;
  const int* cu_k;
  int total_q, total_k;
};

// D = 64 runs three consumer warpgroups over 192 query rows: their S, O and P fit 160 registers, and three
// independent consumers of the same K / V tiles cannot all stay in the same phase, so one's exponentials overlap
// another's products more often than with two (DESIGN.md 4.1).  D = 128 (O alone is 64 registers) keeps two.
template <int D>
struct FwdCfg {
  static constexpr int kBlockM = fwd_block_rows(D);                    // query rows of one CTA
  static constexpr int kConsumers = kBlockM / 64;                      // consumer warpgroups, 64 query rows each
  static constexpr int kThreads = 128 * (1 + kConsumers);              // + the producer warpgroup
  static constexpr int kProducerRegs = kConsumers == 3 ? kProducerRegs3 : fcsa::kProducerRegs;
  static constexpr int kConsumerRegs = kConsumers == 3 ? kConsumerRegs3 : fcsa::kConsumerRegs;
  static constexpr int kTile = 128 * D * 2;          // bytes of one 128-row K / V tile
  static constexpr int kQ = kBlockM * D * 2;         // bytes of the Q tile (kBlockM rows per 64-feature chunk)
  static constexpr int kStages = (D == 64) ? 4 : 2;   // K / V ring depth
  static constexpr int kOffQ = 0;
  static constexpr int kOffK = kQ;
  static constexpr int kOffV = kOffK + kStages * kTile;
  static constexpr int kOffBar = kOffV + kStages * kTile;
  static constexpr int kSmem = kOffBar + 256 + 1024;  // + alignment slack
  static_assert(kQ % 1024 == 0, "operand tiles start on 1024-byte swizzle atoms");
  static_assert(kSmem <= 232448, "forward kernel shared memory");
};

// The exp stage's key padding mask (key_tile.cuh): key col is kept iff its byte in the batch's mask row is nonzero.
struct PaddingMask {
  const uint8_t* row;
  bool has;
  __device__ __forceinline__ bool on() const { return has; }
  __device__ __forceinline__ bool operator()(int col) const { return row[col] != 0; }
};

template <bool VARLEN, bool WINDOW>
using FwdArgsOf = std::conditional_t<WINDOW, Windowed<std::conditional_t<VARLEN, FwdVarlenArgs, FwdArgs>>,
                                     std::conditional_t<VARLEN, FwdVarlenArgs, FwdArgs>>;

// WINDOW: sliding-window attention (Windowed<>::window = W).  A block visits key tiles [j_lo, NT) instead of
// [0, NT): j_lo is the tile of the smallest lower limit of its rows, and NT moves up by W - 1 when not causal.
template <typename T, int D, bool BIAS = false, bool VARLEN = false, bool WINDOW = false>
__global__ void __launch_bounds__(FwdCfg<D>::kThreads, 1)
fcsa_fwd_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_k,
                const __grid_constant__ CUtensorMap tm_v, const FwdArgsOf<VARLEN, WINDOW> a) {
  static_assert(!(BIAS && VARLEN), "packed sequences take no bias");
  static_assert(!(BIAS && WINDOW), "a window takes no bias");
  using Cfg = FwdCfg<D>;
  constexpr int S = Cfg::kStages, TILE = Cfg::kTile, DCH = D / 64, BM = Cfg::kBlockM;

  uint8_t* smem = smem_1024();
  const uint32_t sQ = smem_u32(smem + Cfg::kOffQ);
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

  // ---- work item: BM query rows of one (batch, head) ------------------------------------
  // (the heads of one (batch, query block) are consecutive CTAs: the `group` heads sharing a key/value head
  // stream the same K / V tiles close together in time and meet in L2)
  const int bh_count = a.B * a.H;
  const int rank = blockIdx.x / bh_count;
  const int bh = blockIdx.x - rank * bh_count;
  const int qblk = a.causal ? (a.n_qblk - 1 - rank) : rank;   // heaviest causal blocks first
  const int b = bh / a.H, h = bh - b * a.H;
  const int hk = h / a.group;
  const int m0 = qblk * BM;
  // the (batch) coordinate of the tensor maps and the first query / key row of the sequence: packed sequences are
  // row offsets into maps of batch extent 1; their lengths are read after pdl_wait (a previous kernel may write them)
  const int tb = VARLEN ? 0 : b;
  int Nq = a.Nq, Nk = a.Nk, q_row0 = 0, k_row0 = 0;

  if (threadIdx.x == 0) {
    mbar_init(BAR(Q_FULL), 1);
    kr.init(1, 128 * Cfg::kConsumers);
    vr.init(1, 128 * Cfg::kConsumers);
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();          // q, k (normalised by the previous kernel), v, mask are read from here on
  if constexpr (VARLEN) {
    const SeqSpan sq = seq_span(a.cu_q, b, a.Nq, a.total_q), sk = seq_span(a.cu_k, b, a.Nk, a.total_k);
    Nq = sq.len; Nk = sk.len; q_row0 = sq.start; k_row0 = sk.start;
    if (m0 >= Nq) return;                                     // a query block past the end of its sequence
  }
  const int off = diag_off(Nq, Nk);
  int W = 0;                                                  // the window
  if constexpr (WINDOW) W = a.window;
  const TileRange blk = block_key_tiles<WINDOW>(m0, BM, Nq, Nk, off, a.causal, W);
  const int j_lo = blk.lo, NT = blk.hi;                       // the key tiles [j_lo, NT) this block visits

  if (wg == 0) {
    // =============================== TMA producer ===============================
    reg_dealloc<Cfg::kProducerRegs>();
    if (warp == 0 && elect_one() && NT > j_lo) {
      tma_prefetch_desc(&tm_q);
      tma_prefetch_desc(&tm_k);
      tma_prefetch_desc(&tm_v);
      mbar_expect_tx(BAR(Q_FULL), Cfg::kQ);
#pragma unroll
      for (int ch = 0; ch < DCH; ++ch) tma_load_4d(sQ + ch * BM * 128, &tm_q, BAR(Q_FULL), ch * 64, q_row0 + m0, h, tb);
      load_kv_tiles<D>(&tm_k, &tm_v, kr, vr, sK, sV, j_lo, NT, k_row0, hk, tb);
    }
    return;
  }

  // =============================== consumer warpgroups =========================
  reg_alloc<Cfg::kConsumerRegs>();
  const int w = wg - 1;                       // which 64 of the block's BM query rows
  const int wl = warp & 3;
  // this thread's two rows (accumulator layout, sm90_primitives.cuh): row_a and row_a + 8
  const int row_a = m0 + 64 * w + 16 * wl + (lane >> 2);
  const int cq = 2 * (lane & 3);              // first of the thread's two columns inside every 8-column block
  float nc2 = -a.c2;
  if constexpr (BIAS) {
    if (a.bias_amax != nullptr) nc2 -= fmaxf(__ldg(a.bias_amax), 0.f) * 1.4426950408889634f;
  }
  const float c1 = a.c1;
  const T* brow[2] = {nullptr, nullptr};
  if constexpr (BIAS) {
#pragma unroll
    for (int hf = 0; hf < 2; ++hf)          // (clamped for the padding rows of the last block, never stored)
      brow[hf] = reinterpret_cast<const T*>(a.bias) + (long long)b * a.bias_sb + (long long)h * a.bias_sh +
                 (long long)min(row_a + 8 * hf, a.Nq - 1) * a.bias_sn;
  }
  // the visible key columns of each of the thread's rows (the selects of a masked tile)
  ColRange lim[2];
#pragma unroll
  for (int hf = 0; hf < 2; ++hf) lim[hf] = row_key_cols<WINDOW>(row_a + 8 * hf, off, Nk, a.causal, W);
  // the additive term (with BIAS: + bias * log2e) and the key padding mask of the exp stage
  auto add = [&](int hf, int col) {
    if constexpr (BIAS) {
      uint32_t bw = 0;
      if (col < a.Nk) bw = __ldg(reinterpret_cast<const unsigned int*>(brow[hf] + col));
      const float2 bf = unpack2<T>(bw);
      return make_float2(fmaf(bf.x, 1.4426950408889634f, nc2), fmaf(bf.y, 1.4426950408889634f, nc2));
    } else {
      return make_float2(nc2, nc2);
    }
  };
  const PaddingMask keys = {a.mask + (long long)b * a.mask_sb, a.has_mask != 0};
  // the key tiles [jw_lo, jw_hi) this warpgroup's own 64 rows see; it only passes the ring slots of the others on
  const TileRange wgt = warpgroup_key_tiles<WINDOW>(m0 + 64 * w, j_lo, NT, Nq, off, a.causal, W);
  const int jw_lo = wgt.lo, jw_hi = wgt.hi;

  float o[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) o[i] = 0.f;
  float l[2] = {0.f, 0.f};
  if (NT > j_lo) mbar_wait(BAR(Q_FULL), 0);
  const uint32_t sQw = sQ + w * 64 * 128;     // this warpgroup's 64 rows inside every 64-feature chunk of Q

  for (int j = j_lo; j < NT; ++j) {
    const int n = j - j_lo;                   // the rings' use
    if (j < jw_lo || j >= jw_hi) {
      kr.pass(n);
      vr.pass(n);
      continue;
    }
    float sacc[64];
    const int s = kr.wait(n);
    qk_tile<T, D>(sacc, sQw, BM * 128, sK + s * TILE);
    kr.release(n);

    // (the warpgroup's 64 rows unclipped: rows past Nq are never stored, and a later last row only masks more)
    const int col0 = j * 128;
    const bool need_mask =
        a.has_mask || !tile_visible<WINDOW>(m0 + 64 * w, m0 + 64 * w + 63, col0, col0 + 127, off, Nk, a.causal, W);
    uint32_t pf[32];
    exp_tile<T, WINDOW>(need_mask, sacc, pf, l, c1, col0, cq, lim, add, keys);

    vr.wait(n);
    pv_tile<T>(o, pf, sV + s * TILE);
    vr.release(n);
  }

  // ---- epilogue: O * 1/max(l, eps) -> global ----------------------------------------------
  // The four lanes of a row hold its partial sums.  The clamp only guards rows with no visible key
  // (l == 0, O == 0 -> o = 0; reference: cu:1239 uses 1e-10, too large here because shift = scale*groups
  // makes legitimately tiny row sums).
  float inv[2];
#pragma unroll
  for (int hf = 0; hf < 2; ++hf) inv[hf] = 1.0f / fmaxf(quad_sum(l[hf]), 1e-37f);
#pragma unroll
  for (int hf = 0; hf < 2; ++hf) {
    const int row = row_a + 8 * hf;
    if (row >= Nq) continue;
    const long long o_off = (long long)tb * a.o_sb + (long long)h * a.o_sh + (long long)(q_row0 + row) * a.o_sn;
    if (a.o_f32) store_row(reinterpret_cast<float*>(a.o) + o_off, o, hf, cq, inv[hf]);
    else store_row(reinterpret_cast<T*>(a.o) + o_off, o, hf, cq, inv[hf]);
    if ((lane & 3) == 0 && a.inv_l != nullptr) {
      if constexpr (VARLEN) a.inv_l[(long long)h * a.total_q + q_row0 + row] = inv[hf];
      else a.inv_l[((long long)b * a.H + h) * a.Nq + row] = inv[hf];
    }
  }
}

// ------------------------------------------------------------------------------------------
// Packed sequences: the rows that belong to no sequence
// ------------------------------------------------------------------------------------------
// With cumulative lengths cu[0 .. B] the sequences own rows [cu[0], cu[B]) of a packed tensor; rows [0, cu[0]) and
// [cu[B], total) belong to none (e.g. a fixed-size packing buffer that is not full).  The attention kernels never
// write them, so this pass sets them to zero in the outputs: o = 0 there, and zero gradients.  The bounds are read on
// the device (clamped to [0, total]); when the sequences fill the tensor every block exits after two loads.
struct TailArgs {
  struct Tensor {
    void* ptr;               // 16-bit (total, H, D) tensor, element strides sh, sn, features contiguous
    long long sh, sn;
    int H, total;
    const int* cu;           // its cumulative lengths (B + 1 entries)
  } t[3];
  int B, D;
};

__global__ void __launch_bounds__(256) varlen_tail_kernel(const __grid_constant__ TailArgs a) {
  pdl_launch_dependents();
  pdl_wait();                          // the lengths may come from a previous kernel; the outputs are written after it
  const TailArgs::Tensor& t = a.t[blockIdx.y];
  const int lo = min(max(ld_cu(t.cu), 0), t.total);                  // rows [0, lo) and [hi, total) are cleared
  const int hi = max(min(max(ld_cu(t.cu + a.B), 0), t.total), lo);
  const int vpr = a.D / 8;                                           // 16-byte vectors per row
  const long long n = (long long)(lo + t.total - hi) * t.H * vpr;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    const int c = (int)(i % vpr);
    const long long rh = i / vpr;
    const int h = (int)(rh % t.H);
    long long r = rh / t.H;
    if (r >= lo) r += hi - lo;
    *reinterpret_cast<uint4*>(static_cast<uint16_t*>(t.ptr) + h * t.sh + r * t.sn + c * 8) = make_uint4(0, 0, 0, 0);
  }
}

}  // namespace fcsa
