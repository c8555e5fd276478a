// Forward kernel: o = (sum_j exp(scale*q.k_j - shift) v_j) / max(sum_j exp(..), 1e-37)
//
// Replaces the reference's forward_kernel (flash_cosine_sim_attention_cuda.cu:1072-1247).
// Same math (fixed shift instead of a running row max, cu:1216; running row sum, cu:1236;
// final 1/max(l, eps) scaling, cu:1239-1246; bottom-right aligned causal mask, cu:1097/1210;
// key-padding mask, cu:1198-1212) - a different machine mapping:
//
//   * one CTA = 128 query rows of one (batch, head); CTAs are numbered heaviest first (causal: the last
//     query blocks see the most keys), so the block scheduler starts the long ones first
//   * warpgroup 0 : TMA producer (one thread): Q once, then K and V tiles of 128 keys through
//                   mbarrier rings; the warpgroup gives most of its registers to the other two
//   * warpgroups 1, 2: 64 query rows each.  Per key tile: S = Q K^T (wgmma, both operands in shared
//                   memory) -> P = exp2(S*c1 - c2) in registers -> O += P V (wgmma with P as the register
//                   A operand).  Because there is no row max there is no rescaling of O: the accumulator
//                   stays in registers until the epilogue.  The two warpgroups share every K / V tile and
//                   interleave on the tensor cores: one runs its exps while the other's MMAs run.
#pragma once

#include "sm90_primitives.cuh"

namespace fcsa {

struct FwdArgs {
  int B, H, Nq, Nk;
  int causal;        // bottom-right aligned: key j visible to query i iff j <= i + (Nk - Nq)
  int has_mask;      // key padding mask (B, Nk), nonzero = keep
  int group;         // query heads per key/value head (H / kv_heads): head h reads kv head h / group
  int n_qblk;        // ceil(Nq / 128)
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

template <int D>
struct FwdCfg {
  static constexpr int kTile = 128 * D * 2;          // bytes of one 128-row operand tile
  static constexpr int kStages = (D == 64) ? 4 : 2;   // K / V ring depth
  static constexpr int kOffQ = 0;
  static constexpr int kOffK = kTile;
  static constexpr int kOffV = kOffK + kStages * kTile;
  static constexpr int kOffBar = kOffV + kStages * kTile;
  static constexpr int kSmem = kOffBar + 256 + 1024;  // + alignment slack
  static constexpr int kThreads = 384;                // producer warpgroup + 2 consumer warpgroups
  static_assert(kSmem <= 232448, "forward kernel shared memory");
};

template <typename T, int D, bool BIAS = false>
__global__ void __launch_bounds__(384, 1)
fcsa_fwd_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_k,
                const __grid_constant__ CUtensorMap tm_v, const FwdArgs a) {
  using Cfg = FwdCfg<D>;
  constexpr int S = Cfg::kStages, TILE = Cfg::kTile, DCH = D / 64;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~uintptr_t(1023));
  const uint32_t sQ = smem_u32(smem + Cfg::kOffQ);
  const uint32_t sK = smem_u32(smem + Cfg::kOffK);
  const uint32_t sV = smem_u32(smem + Cfg::kOffV);
  const uint32_t bar0 = smem_u32(smem + Cfg::kOffBar);
  auto BAR = [&](int i) { return bar0 + 8u * i; };
  constexpr int Q_FULL = 0, K_FULL = 1, K_EMPTY = K_FULL + S, V_FULL = K_EMPTY + S, V_EMPTY = V_FULL + S,
                NBARS = V_EMPTY + S;
  static_assert(NBARS * 8 <= 256, "barrier area");

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg = warp >> 2;
  pdl_launch_dependents();

  // ---- work item: 128 query rows of one (batch, head) ------------------------------------
  // (the heads of one (batch, query block) are consecutive CTAs: the `group` heads sharing a key/value head
  // stream the same K / V tiles close together in time and meet in L2)
  const int bh_count = a.B * a.H;
  const int rank = blockIdx.x / bh_count;
  const int bh = blockIdx.x - rank * bh_count;
  const int qblk = a.causal ? (a.n_qblk - 1 - rank) : rank;   // heaviest causal blocks first
  const int b = bh / a.H, h = bh - b * a.H;
  const int hk = h / a.group;
  const int m0 = qblk * 128;
  const int off = a.Nk - a.Nq;
  int NT = (a.Nk + 127) >> 7;                                 // key tiles this block visits
  if (a.causal) {
    const int last_col = min(m0 + 127, a.Nq - 1) + off;
    NT = last_col < 0 ? 0 : min(NT, (last_col >> 7) + 1);
  }

  if (threadIdx.x == 0) {
    mbar_init(BAR(Q_FULL), 1);
    for (int s = 0; s < S; ++s) {
      mbar_init(BAR(K_FULL + s), 1);
      mbar_init(BAR(K_EMPTY + s), 256);
      mbar_init(BAR(V_FULL + s), 1);
      mbar_init(BAR(V_EMPTY + s), 256);
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();          // q, k (normalised by the previous kernel), v, mask are read from here on

  if (wg == 0) {
    // =============================== TMA producer ===============================
    reg_dealloc<kProducerRegs>();
    if (warp == 0 && elect_one() && NT > 0) {
      tma_prefetch_desc(&tm_q);
      tma_prefetch_desc(&tm_k);
      tma_prefetch_desc(&tm_v);
      mbar_expect_tx(BAR(Q_FULL), TILE);
#pragma unroll
      for (int ch = 0; ch < DCH; ++ch) tma_load_4d(sQ + ch * 16384, &tm_q, BAR(Q_FULL), ch * 64, m0, h, b);
      for (int j = 0; j < NT; ++j) {
        const int s = j % S;
        const uint32_t par = ((j / S) & 1) ^ 1;
        mbar_wait(BAR(K_EMPTY + s), par);
        mbar_expect_tx(BAR(K_FULL + s), TILE);
#pragma unroll
        for (int ch = 0; ch < DCH; ++ch)
          tma_load_4d(sK + s * TILE + ch * 16384, &tm_k, BAR(K_FULL + s), ch * 64, j * 128, hk, b);
        mbar_wait(BAR(V_EMPTY + s), par);
        mbar_expect_tx(BAR(V_FULL + s), TILE);
#pragma unroll
        for (int ch = 0; ch < DCH; ++ch)
          tma_load_4d(sV + s * TILE + ch * 16384, &tm_v, BAR(V_FULL + s), ch * 64, j * 128, hk, b);
      }
    }
    return;
  }

  // =============================== consumer warpgroups =========================
  reg_alloc<kConsumerRegs>();
  const int w = wg - 1;                       // which 64 of the block's 128 query rows
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
  // last visible column of each row (causal / ragged end)
  int lim[2];
#pragma unroll
  for (int hf = 0; hf < 2; ++hf) lim[hf] = a.causal ? min(a.Nk - 1, row_a + 8 * hf + off) : a.Nk - 1;

  float o[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) o[i] = 0.f;
  float l[2] = {0.f, 0.f};
  if (NT > 0) mbar_wait(BAR(Q_FULL), 0);
  const uint32_t sQw = sQ + w * 64 * 128;     // this warpgroup's 64 rows inside every 64-feature chunk of Q

  for (int j = 0; j < NT; ++j) {
    const int s = j % S;
    const uint32_t par = (j / S) & 1;
    // ---- S = Q K^T (64 x 128, fp32) ----
    float sacc[64];
    mbar_wait(BAR(K_FULL + s), par);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk) {
      const uint32_t ko = (kk >> 2) * 16384 + (kk & 3) * 32;
      wgmma_ss_n128<T, 0, 0>(sacc, gmma_desc_sw128(sQw + ko, 16, 1024),
                             gmma_desc_sw128(sK + s * TILE + ko, 16, 1024), kk > 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(sacc);
    mbar_arrive(BAR(K_EMPTY + s));

    // ---- P = exp2(S*c1 - c2 [+ bias*log2e]), masked; row sums in fp32; 16-bit P as A fragments ----
    const int col0 = j * 128;
    const bool need_mask = a.has_mask || (col0 + 127 >= a.Nk) || (a.causal && col0 + 127 > m0 + 64 * w + off);
    uint32_t pf[32];
    auto exp_tile = [&](auto masked_tag) {
      constexpr bool MASKED = decltype(masked_tag)::value;
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        const int hf = i & 1;                                 // row_a or row_a + 8
        const int col = col0 + 8 * (i >> 1) + cq;
        float add0 = nc2, add1 = nc2;
        if constexpr (BIAS) {
          uint32_t bw = 0;
          if (col < a.Nk) bw = __ldg(reinterpret_cast<const unsigned int*>(brow[hf] + col));
          const float2 bf = unpack2<T>(bw);
          add0 = fmaf(bf.x, 1.4426950408889634f, nc2);
          add1 = fmaf(bf.y, 1.4426950408889634f, nc2);
        }
        float p0 = ex2_approx(fmaf(sacc[2 * i], c1, add0));
        float p1 = ex2_approx(fmaf(sacc[2 * i + 1], c1, add1));
        if constexpr (MASKED) {
          bool v0 = col <= lim[hf], v1 = col + 1 <= lim[hf];
          if (a.has_mask) {
            v0 = v0 && a.mask[(long long)b * a.mask_sb + col] != 0;
            v1 = v1 && a.mask[(long long)b * a.mask_sb + col + 1] != 0;
          }
          p0 = v0 ? p0 : 0.f;
          p1 = v1 ? p1 : 0.f;
        }
        l[hf] += p0 + p1;
        pf[i] = pack2<T>(p0, p1);
      }
    };
    if (need_mask) exp_tile(std::true_type{});
    else exp_tile(std::false_type{});

    // ---- O += P V ----
    mbar_wait(BAR(V_FULL + s), par);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
      const uint32_t af[4] = {pf[4 * kk], pf[4 * kk + 1], pf[4 * kk + 2], pf[4 * kk + 3]};
      const uint64_t dv = gmma_desc_sw128(sV + s * TILE + kk * 2048, 16384, 1024);
      if constexpr (D == 64) wgmma_rs_n64<T, 1>(o, af, dv, 1u);
      else wgmma_rs_n128<T, 1>(o, af, dv, 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(o);
    fence_regs(pf);
    mbar_arrive(BAR(V_EMPTY + s));
  }

  // ---- epilogue: O * 1/max(l, eps) -> global ----------------------------------------------
  // The four lanes of a row hold its partial sums.  The clamp only guards rows with no visible key
  // (l == 0, O == 0 -> o = 0; reference: cu:1239 uses 1e-10, too large here because shift = scale*groups
  // makes legitimately tiny row sums).
  float inv[2];
#pragma unroll
  for (int hf = 0; hf < 2; ++hf) {
    float x = l[hf];
    x += __shfl_xor_sync(0xFFFFFFFFu, x, 1);
    x += __shfl_xor_sync(0xFFFFFFFFu, x, 2);
    inv[hf] = 1.0f / fmaxf(x, 1e-37f);
  }
#pragma unroll
  for (int hf = 0; hf < 2; ++hf) {
    const int row = row_a + 8 * hf;
    if (row >= a.Nq) continue;
    const long long o_off = (long long)b * a.o_sb + (long long)h * a.o_sh + (long long)row * a.o_sn;
    if (a.o_f32) {
      float* orow = reinterpret_cast<float*>(a.o) + o_off;
#pragma unroll
      for (int jb = 0; jb < D / 8; ++jb)
        *reinterpret_cast<float2*>(orow + 8 * jb + cq) =
            make_float2(o[4 * jb + 2 * hf] * inv[hf], o[4 * jb + 2 * hf + 1] * inv[hf]);
    } else {
      T* orow = reinterpret_cast<T*>(a.o) + o_off;
#pragma unroll
      for (int jb = 0; jb < D / 8; ++jb)
        *reinterpret_cast<uint32_t*>(orow + 8 * jb + cq) =
            pack2<T>(o[4 * jb + 2 * hf] * inv[hf], o[4 * jb + 2 * hf + 1] * inv[hf]);
    }
    if ((lane & 3) == 0 && a.inv_l != nullptr) a.inv_l[((long long)b * a.H + h) * a.Nq + row] = inv[hf];
  }
}

}  // namespace fcsa
