// Backward: dq, dk, dv of the fixed-shift cosine-sim attention.
//
// Replaces the reference's backward_preprocess (flash_cosine_sim_attention_cuda.cu:1256-1335)
// and backward_kernel (cu:1339-1626).  The math is the reference's (restated in DESIGN.md par. 2):
//     P_ij  = exp(scale*s_ij - shift) * inv_l_i          cu:1513-1526
//     delta = rowsum(dO * O)                               cu:1293-1334
//     dV    = P^T dO          dP = dO V^T                  cu:1534-1553
//     dS    = P * (dP - delta)                             cu:1564-1570
//     dK    = scale * dS^T q  dQ = scale * dS k            cu:1580-1610
// The machine mapping is new.  Three kernels:
//   1. bwd_prep_kernel    : per query row {c3 = log2(inv_l) - shift*log2e, -delta} (fp32, never
//                           rounded to 16 bit as the reference does at cu:1260/1820)
//   2. fcsa_bwd_kernel    : one CTA = one 128-key tile of one (batch, kv head), K and V stationary in shared memory,
//                           loop over the query tiles of QT = 64 rows that can see it, for each query head of the
//                           CTA's slice of the kv head's group (grouped-query attention; one head for MHA): the
//                           (head, query tile) pairs form one flat sequence of tiles.  Warpgroup 0 is the TMA
//                           producer (K, V once; Q, dO and the per-query constants through an mbarrier ring);
//                           warpgroups 1 and 2 own 64 keys each and run, per query tile, independently of each other:
//                             S^T = K Q^T, dP^T = V dO^T            (wgmma, both operands in shared memory)
//                             P^T, dS^T in registers                 (16-bit A fragments for the next two products)
//                             dV += P^T dO, dK += dS^T Q             (wgmma, A from registers)
//                             dQ = dS K                              (wgmma; dS^T through shared memory)
//                           Everything is computed TRANSPOSED (rows = keys) so that P^T and dS^T come out of the
//                           accumulators in the register layout of a wgmma A operand.  The dQ tile is added to an
//                           fp32 accumulator in global memory: D = 64 computes it once per query tile over all
//                           128 keys (the warpgroups take turns), stages it in shared memory for TMA reduce-adds
//                           issued by producer warps 1 and 2 and pipelines the products of consecutive query
//                           tiles; D = 128 adds a partial over each warpgroup's 64 keys with vector reductions
//                           from registers.  dK / dV accumulate in registers over all the CTA's heads; when the
//                           CTA covers its whole group the epilogue writes them (with the fused l2norm: the
//                           gradient w.r.t. the raw keys), otherwise it adds them to fp32 accumulators.
//   3. bwd_dq_finish_kernel: fp32 accumulator * scale -> 16-bit dq (+ l2norm backward of q); writes the accumulator
//                           back as zeros (the "zeroed" workspace is zero on entry and on exit of every call).
// BIAS instantiation: additive attention bias (16-bit loads along the query axis) and d_bias = dS
// (fp32 reductions), reference cu:1474-1476 / 1574-1576.
#pragma once

#include <stdlib.h>
#include <algorithm>
#include <type_traits>

#include "../../include/fcsa_b200.h"
#include "key_tile.cuh"
#include "l2norm_kernels.cuh"
#include "tensor_map.h"

namespace fcsa {

// D = 64 computes one dQ tile per query tile and CTA (a contraction over all 128 keys, shared by the two
// warpgroups through shared memory), stages it for TMA reduce-adds and pipelines the products of consecutive
// query tiles; D = 128 has neither the shared memory (two 32 KB staging tiles on top of 194 KB) nor the
// registers (a second S^T / dP^T pair next to 128 dV / dK accumulators) for that, and keeps the in-order loop
// with a dQ partial per warpgroup and vector reductions from registers.
template <int D>
struct BwdCfg {
  static constexpr bool kStaged = (D == 64);
  static constexpr int QT = 64;                           // query rows per tile
  static constexpr int kKV = 128 * D * 2;                 // bytes of the K (or V) tile
  static constexpr int kQ = QT * D * 2;                   // bytes of one Q (or dO) stage
  static constexpr int NST = kStaged ? 4 : 3;             // Q / dO / stats ring depth
  static constexpr int kDS = 64 * QT * 2;                 // one warpgroup's dS^T: 64 keys x QT queries, 16-bit
  static constexpr int NDS = kStaged ? 3 : 2;             // dS^T slots (one buffer per warpgroup each)
  static constexpr int NDQ = kStaged ? 1 : 0;             // dQ staging buffers per warpgroup
  static constexpr int kDQ = kStaged ? QT * D * 4 : 0;    // one fp32 dQ staging tile: D / 32 boxes of 32 x QT
  static constexpr int kOffK = 0;
  static constexpr int kOffV = kOffK + kKV;
  static constexpr int kOffQ = kOffV + kKV;
  static constexpr int kOffDO = kOffQ + NST * kQ;
  static constexpr int kOffDS = kOffDO + NST * kQ;        // NDS slots x 2 warpgroups (slot-major: 128 keys each)
  static constexpr int kOffDQ = kOffDS + 2 * NDS * kDS;   // 2 warpgroups x NDQ buffers (1024-byte aligned)
  static constexpr int kOffStats = kOffDQ + 2 * NDQ * kDQ;  // NST stages x {c3, -delta} x QT floats
  static constexpr int kOffBar = kOffStats + NST * 8 * QT;
  static constexpr int kSmem = kOffBar + 256 + 1024;
  static_assert(kSmem <= 232448, "backward kernel shared memory");
  static_assert(kOffDQ % 1024 == 0, "128B-swizzled staging tiles");
  static constexpr int kThreads = 384;                    // producer warpgroup + 2 consumer warpgroups
};

// ------------------------------------------------------------------------------------------
// Two caller-provided device buffers:
//
// SCRATCH workspace (contents irrelevant on entry, garbage on exit):
//   stats : fp32 [B*H][nqt][2][QT]   c3 then -delta for each query tile (padded rows = 0)
//   dkv_acc (kv_heads < heads only): fp32 dk [B][kv_heads][Nk][D] then dv [B][kv_heads][Nk][D]; used when a
//            group's query heads are split over several CTAs (BwdArgs::split > 1)
//
// ZEROED workspace (all zero on entry - the caller zero-fills it ONCE, fcsa_zeroed_init - and all
// zero again on exit: the dq conversion pass clears every accumulator row it converts, so no per-call
// memset / zeroing pass is needed; reference: a 33.5 MB cudaMemset of dq per backward, cu:1818):
//   dq_acc: fp32 [B*H][nqt*QT][D], row-major
// ------------------------------------------------------------------------------------------
struct BwdWorkspace {
  size_t stats_off, dkv_off, total;     // scratch
  size_t dq_off, ztotal;                // zeroed
  int nqt, QT;
};

inline BwdWorkspace bwd_workspace_layout(int B, int H, int kv_heads, int Nq, int Nk, int D) {
  BwdWorkspace w;
  w.QT = 64;
  w.nqt = (Nq + w.QT - 1) / w.QT;
  size_t stats = (size_t)B * H * w.nqt * 2 * w.QT * 4;
  size_t dq = (size_t)B * H * w.nqt * w.QT * D * 4;
  size_t dkv = kv_heads < H ? (size_t)2 * B * kv_heads * Nk * D * 4 : 0;
  auto up = [](size_t x) { return (x + 255) & ~size_t(255); };
  w.stats_off = 0;
  w.dkv_off = up(stats);
  w.total = w.dkv_off + up(dkv);
  w.dq_off = 0;
  w.ztotal = up(dq);
  return w;
}

// Packed sequences: the stats and the dq accumulator hold, per query head, varlen_tiles tiles of QT rows, sequence b
// from tile base(b) = varlen_tile_base (tile_ranges.h).  dkv_acc is [kv_heads][total_k][D] (dk, then dv).
inline BwdWorkspace bwd_varlen_workspace_layout(int B, int H, int kv_heads, long long total_q, long long total_k,
                                                int D) {
  BwdWorkspace w;
  w.QT = 64;
  w.nqt = varlen_tiles(B, total_q);
  size_t stats = (size_t)H * w.nqt * 2 * w.QT * 4;
  size_t dq = (size_t)H * w.nqt * w.QT * D * 4;
  size_t dkv = kv_heads < H ? (size_t)2 * kv_heads * total_k * D * 4 : 0;
  auto up = [](size_t x) { return (x + 255) & ~size_t(255); };
  w.stats_off = 0;
  w.dkv_off = up(stats);
  w.total = w.dkv_off + up(dkv);
  w.dq_off = 0;
  w.ztotal = up(dq);
  return w;
}

inline size_t bwd_workspace_bytes(int B, int H, int kv_heads, int Nq, int Nk, int D) {
  return bwd_workspace_layout(B, H, kv_heads, Nq, Nk, D).total;
}
inline size_t bwd_zeroed_workspace_bytes(int B, int H, int kv_heads, int Nq, int Nk, int D) {
  return bwd_workspace_layout(B, H, kv_heads, Nq, Nk, D).ztotal;
}

// ------------------------------------------------------------------------------------------
// 1. preprocess
// ------------------------------------------------------------------------------------------
struct PrepArgs {
  int B, H, Nq, Nk, D, nqt, QT, causal;
  int bpb;                          // blocks per (batch, head): the grid is 1-D (no 65535 limit on batch*heads)
  float c2;                         // shift * log2e
  const float* shift_extra;         // optional device scalar: shift += max(*shift_extra, 0) (bias range guard)
  int o_f32;                        // 1: o is float32 (strides in float32 elements)
  const void* o;  long long o_sb, o_sh, o_sn;
  const void* d_o; long long do_sb, do_sh, do_sn;
  const float* inv_l;               // (B, H, Nq)
  float* stats;
};

// Packed sequences: B sequences, Nq = the maximum length and nqt = ceil(Nq / QT) (the grid); o, d_o are
// (total_q, H, D) (o_sb, do_sb unused), inv_l is (H, total_q) and the stats of head h, sequence b start at tile
// h * ntile + base(b) (bwd_varlen_workspace_layout).
struct PrepVarlenArgs : PrepArgs {
  const int* cu_q;
  int total_q, ntile;
};

__device__ __forceinline__ float lg2_approx(float x) {
  float y;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// TPR = threads per row = D / 8 (8 or 16); QT = 64.
template <typename T, int TPR, bool VARLEN = false>
__global__ void __launch_bounds__(256) bwd_prep_kernel(const std::conditional_t<VARLEN, PrepVarlenArgs, PrepArgs> a) {
  // 1-D grid = batch*heads x (row blocks of the padded sequence); TPR threads per row, two rows per
  // thread (four 16-byte loads in flight), shuffle reduce.  The pass must stay memory-bound: no
  // runtime-divisor divisions, MUFU log2.
  pdl_launch_dependents();
  pdl_wait();
  constexpr int RPB = 256 / TPR;             // rows per block and pass
  constexpr int QT = 64, QSH = 6;
  const int bh = blockIdx.x / a.bpb;
  const int blk = blockIdx.x - bh * a.bpb;
  const int b = bh / a.H, h = bh - b * a.H;
  const int tr = threadIdx.x % TPR;
  int padded = a.nqt * QT, Nq = a.Nq;
  long long tile0 = (long long)bh * a.nqt, row_off = 0;     // the stats tile of query row 0, o / d_o rows before it
  if constexpr (VARLEN) {
    // the sequence's rows, then zeros up to its last tile's end
    const SeqSpan sq = seq_span(a.cu_q, b, a.Nq, a.total_q);
    Nq = sq.len;
    padded = (Nq + QT - 1) / QT * QT;
    tile0 = (long long)h * a.ntile + varlen_tile_base(sq.start, b);
    row_off = sq.start;
  }
  const float c2 = a.c2 + (a.shift_extra != nullptr ? fmaxf(__ldg(a.shift_extra), 0.f) * 1.4426950408889634f : 0.f);
  const long long o_off = (VARLEN ? 0 : b * a.o_sb) + h * a.o_sh + row_off * a.o_sn + tr * 8;
  const T* obase = reinterpret_cast<const T*>(a.o) + o_off;
  const float* obase32 = reinterpret_cast<const float*>(a.o) + o_off;
  const T* dbase = reinterpret_cast<const T*>(a.d_o) + (VARLEN ? 0 : b * a.do_sb) + h * a.do_sh + row_off * a.do_sn + tr * 8;
  int row[2];
  bool in[2], valid[2];
  uint4 ro[2], rd[2];
  float4 rof[2][2];                           // o as float32 (o_f32 problems): 8 features = two float4
  float il[2];
#pragma unroll
  for (int u = 0; u < 2; ++u) {
    row[u] = (blk * 2 + u) * RPB + threadIdx.x / TPR;     // row inside the padded (nqt*QT) range
    in[u] = row[u] < padded;
    valid[u] = in[u] && row[u] < Nq;
    ro[u] = rd[u] = make_uint4(0, 0, 0, 0);
    rof[u][0] = rof[u][1] = make_float4(0.f, 0.f, 0.f, 0.f);
    il[u] = 1.f;
    if (valid[u]) {
      if (a.o_f32) {
        rof[u][0] = __ldg(reinterpret_cast<const float4*>(obase32 + (long long)row[u] * a.o_sn));
        rof[u][1] = __ldg(reinterpret_cast<const float4*>(obase32 + (long long)row[u] * a.o_sn + 4));
      } else {
        ro[u] = ldg_stream128(obase + (long long)row[u] * a.o_sn);
      }
      rd[u] = ldg_stream128(dbase + (long long)row[u] * a.do_sn);
      if (tr == 0) {
        if constexpr (VARLEN) il[u] = __ldg(a.inv_l + (long long)h * a.total_q + row_off + row[u]);
        else il[u] = __ldg(a.inv_l + (long long)bh * a.Nq + row[u]);
      }
    }
  }
#pragma unroll
  for (int u = 0; u < 2; ++u) {
    float2 a0 = unpack2<T>(ro[u].x), a1 = unpack2<T>(ro[u].y), a2 = unpack2<T>(ro[u].z), a3 = unpack2<T>(ro[u].w);
    if (a.o_f32) {
      a0 = make_float2(rof[u][0].x, rof[u][0].y); a1 = make_float2(rof[u][0].z, rof[u][0].w);
      a2 = make_float2(rof[u][1].x, rof[u][1].y); a3 = make_float2(rof[u][1].z, rof[u][1].w);
    }
    const float2 b0 = unpack2<T>(rd[u].x), b1 = unpack2<T>(rd[u].y), b2 = unpack2<T>(rd[u].z), b3 = unpack2<T>(rd[u].w);
    float dot = a0.x * b0.x + a0.y * b0.y + a1.x * b1.x + a1.y * b1.y + a2.x * b2.x + a2.y * b2.y +
                a3.x * b3.x + a3.y * b3.y;
#pragma unroll
    for (int m = 1; m < TPR; m <<= 1) dot += __shfl_xor_sync(0xFFFFFFFFu, dot, m);
    // lane tr == 0 of the row holds inv_l: c3 = log2(inv_l) - shift*log2e
    const float c3 = valid[u] ? lg2_approx(il[u]) - c2 : 0.f;
    const float ndl = valid[u] ? -dot : 0.f;      // stored negated: the dS stage computes P * (dP + (-delta))
    if (!in[u] || tr != 0) continue;
    const int qt = row[u] >> QSH, r = row[u] & (QT - 1);
    float* st = a.stats + (tile0 + qt) * 2 * QT;
    st[r] = c3;
    st[QT + r] = ndl;
  }
}

// ------------------------------------------------------------------------------------------
// 2. main kernel
// ------------------------------------------------------------------------------------------
struct BwdArgs {
  int B, H, Nq, Nk, kv_heads, causal, has_mask, nqt;
  // query heads per CTA: the group of kv head hk (query heads hk * G .. + G - 1, G = H / kv_heads) is split into
  // `split` slices of `hpc` = G / split consecutive heads, one slice per CTA.  split > 1: dk / dv are reduced over
  // the slices in the fp32 accumulators.  BIAS launches have hpc = 1.
  int split, hpc;
  float c1;                         // scale * log2e
  float scale;
  const uint8_t* mask; long long mask_sb;
  const float* stats;
  float* dq_acc;
  float* dk_acc; float* dv_acc;     // fp32 (B, kv_heads, Nk, D) accumulators when split > 1
  void* dk; long long dk_sb, dk_sh, dk_sn;
  void* dv; long long dv_sb, dv_sh, dv_sn;
  // additive bias on the logits (BIAS instantiation only): element type T, [b][h][query][key], element
  // strides (bias_sb = 0: no batch dimension), keys contiguous.  dbias: fp32 accumulator of dS in the same
  // index space ([.][.][Nq][Nk] planes, strides dbias_sb (0 = summed over the batch) / dbias_sh) or nullptr.
  const void* bias; long long bias_sb, bias_sh, bias_sn;
  float* dbias; long long dbias_sb, dbias_sh;
  int out_f32;                      // 1: dk, dv are float32 tensors (strides in float32 elements)
  // fused l2norm: k is the normalised k_hat and dk the gradient w.r.t. the raw keys (written by the epilogue
  // when split == 1); k_rnorm (B, kv_heads, Nk, groups) or nullptr
  const float* k_rnorm;
  int groups;
};

// Packed sequences (VARLEN instantiations): B sequences, Nq / Nk = the maximum lengths (nqt unused).  q, d_o are
// (total_q, H, D), k, v, dk, dv (total_k, kv_heads, D), addressed at batch 0 of their maps (dk_sb, dv_sb unused);
// sequence b owns query rows [cu_q[b], cu_q[b + 1]) and key rows [cu_k[b], cu_k[b + 1]).  The stats and the dq
// accumulator of head h, sequence b start at tile h * ntile + base(b) (bwd_varlen_workspace_layout); dk_acc / dv_acc
// and k_rnorm are [kv_heads][total_k][.].
struct BwdVarlenArgs : BwdArgs {
  const int* cu_q;
  const int* cu_k;
  int total_q, total_k, ntile;
};

// 16-bit global load through the read-only path (bias elements along the query axis are strided)
__device__ __forceinline__ uint32_t ldg_u16(const void* p) {
  uint16_t v;
  asm volatile("ld.global.nc.u16 %0, [%1];" : "=h"(v) : "l"(p));
  return v;
}
__device__ __forceinline__ void red_add_f32(float* p, float v) {
  asm volatile("red.global.add.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}
__device__ __forceinline__ void red_add_f32x2(float* p, float x, float y) {
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(x), "f"(y) : "memory");
}
// 16-byte load served by L2 (never a stale L1 line): accumulator rows other CTAs have reduced into
__device__ __forceinline__ float4 ldg_cg128f(const float* p) {
  float4 v;
  asm volatile("ld.global.cg.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(p)
               : "memory");
  return v;
}

// l2norm backward of one key row in the backward epilogue: dk = (dk_hat - k_hat <k_hat, dk_hat>_group) * rnorm_group.
// The thread holds features 8 jb + cq + {0, 1} (g[2 jb], g[2 jb + 1]) of the row; the row's other features are in the
// other three lanes of its quad.  k_hat comes from the resident K tile (row address sk_row, 128B swizzle, 64-feature
// chunks 16 KB apart).  All lanes of the warp must call it (quad shuffles); `in` = the key exists.  k_rnorm has
// `groups` floats per row; the key's row is krow0 + key.  (The dQ kernel applies it to a row of its resident Q tile.)
template <typename T, int D>
__device__ __forceinline__ void l2norm_bwd_key_row(float (&g)[D / 4], const float* k_rnorm, int groups, uint32_t sk_row,
                                                   long long krow0, int key, bool in) {
  const int lane = threadIdx.x & 31;
  const int r8 = (lane >> 2) & 7, cq = 2 * (lane & 3);
  const int gs = D / groups;                    // features per group (a power of two)
  float y[D / 4], dot[D / 4];
#pragma unroll
  for (int jb = 0; jb < D / 8; ++jb) {
    const float2 v = unpack2<T>(lds32(sk_row + (jb >> 3) * 16384 + ((((jb & 7) ^ r8)) << 4) + 2 * cq));
    y[2 * jb] = v.x;
    y[2 * jb + 1] = v.y;
  }
  if (gs == 1) {
#pragma unroll
    for (int e = 0; e < D / 4; ++e) dot[e] = y[e] * g[e];
  } else {
    float q[D / 8];                             // sums over the thread's feature pairs, then over the group
#pragma unroll
    for (int jb = 0; jb < D / 8; ++jb) q[jb] = y[2 * jb] * g[2 * jb] + y[2 * jb + 1] * g[2 * jb + 1];
    // groups wider than 8 features: aligned blocks of gs / 8 pairs (compile-time register indices only)
#pragma unroll
    for (int m = 1; m < D / 8; m <<= 1) {
      float t[D / 8];
#pragma unroll
      for (int jb = 0; jb < D / 8; ++jb) t[jb] = q[jb] + q[jb ^ m];
      if (8 * m < gs) {
#pragma unroll
        for (int jb = 0; jb < D / 8; ++jb) q[jb] = t[jb];
      }
    }
    // across the quad: gs = 4 spans lane pairs, gs >= 8 all four lanes
    if (gs >= 4) {
#pragma unroll
      for (int jb = 0; jb < D / 8; ++jb) q[jb] += __shfl_xor_sync(0xFFFFFFFFu, q[jb], 1);
    }
    if (gs >= 8) {
#pragma unroll
      for (int jb = 0; jb < D / 8; ++jb) q[jb] += __shfl_xor_sync(0xFFFFFFFFu, q[jb], 2);
    }
#pragma unroll
    for (int jb = 0; jb < D / 8; ++jb) dot[2 * jb] = dot[2 * jb + 1] = q[jb];
  }
  const int lg = __ffs(gs) - 1;
  const float* rn = k_rnorm + (krow0 + (in ? key : 0)) * groups;         // k_rnorm row krow0 + key
  // one load per feature pair (a pair shares its group unless gs = 1); the pairs of one group hit the same L1 line
#pragma unroll
  for (int jb = 0; jb < D / 8; ++jb) {
    const int f = 8 * jb + cq;
    const float r0 = in ? __ldg(rn + (f >> lg)) : 0.f;
    const float r1 = gs == 1 && in ? __ldg(rn + f + 1) : r0;
    g[2 * jb] = (g[2 * jb] - y[2 * jb] * dot[2 * jb]) * r0;
    g[2 * jb + 1] = (g[2 * jb + 1] - y[2 * jb + 1] * dot[2 * jb + 1]) * r1;
  }
}

template <bool VARLEN, bool WINDOW>
using BwdArgsOf = std::conditional_t<WINDOW, Windowed<std::conditional_t<VARLEN, BwdVarlenArgs, BwdArgs>>,
                                     std::conditional_t<VARLEN, BwdVarlenArgs, BwdArgs>>;

// HEAD_LOOP: the CTA works through several query heads (hpc > 1, grouped-query launches); otherwise hpc = 1 is a
// compile-time constant and the loops below are those of one query head (MHA, MQA, BIAS and split groups of one head).
// VARLEN: packed sequences (BwdVarlenArgs); `b` is then the sequence, and its lengths replace Nq / Nk.
// WINDOW: sliding-window attention (Windowed<>::window = W): a key tile visits query tiles [i_lo, i_end) instead of
// [i_lo, nqt), i_end being the tile after the last query row whose lower limit reaches key0 + 127.
// DQ = false: dK and dV only (the deterministic backward, whose dq comes from fcsa_dq_kernel).  No dS^T in shared
// memory, no dQ product, no reducer warps, no dq accumulator; both head dims run the in-order loop, and the host
// launches it with split = 1, so dk / dv always leave through the direct epilogue.
template <typename T, int D, bool BIAS = false, bool HEAD_LOOP = false, bool VARLEN = false, bool WINDOW = false,
          bool DQ = true>
__global__ void __launch_bounds__(384, 1)
fcsa_bwd_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_k,
                const __grid_constant__ CUtensorMap tm_v, const __grid_constant__ CUtensorMap tm_do,
                const __grid_constant__ CUtensorMap tm_dq, const BwdArgsOf<VARLEN, WINDOW> a) {
  static_assert(D == 64 || D == 128, "head dim 64 or 128");
  static_assert(!(BIAS && HEAD_LOOP), "BIAS launches have one query head per CTA");
  static_assert(!(BIAS && VARLEN), "packed sequences take no bias");
  static_assert(!(BIAS && WINDOW), "a window takes no bias");
  static_assert(DQ || !BIAS, "the dK / dV-only kernel takes no bias");
  using Cfg = BwdCfg<D>;
  constexpr bool STAGED = Cfg::kStaged && DQ;
  constexpr int QT = Cfg::QT;              // query rows per tile
  constexpr int KCH = D / 64;              // 64-feature chunks of every operand tile
  constexpr int QCHUNK = QT * 128;         // bytes of one 64-feature chunk of a Q / dO stage
  constexpr int NST = Cfg::NST;

  uint8_t* smem = smem_1024();
  const uint32_t sK = smem_u32(smem + Cfg::kOffK);
  const uint32_t sV = smem_u32(smem + Cfg::kOffV);
  const uint32_t sQ = smem_u32(smem + Cfg::kOffQ);
  const uint32_t sDO = smem_u32(smem + Cfg::kOffDO);
  const uint32_t sDS = smem_u32(smem + Cfg::kOffDS);
  const uint32_t sDQ = smem_u32(smem + Cfg::kOffDQ);
  const uint32_t sStats = smem_u32(smem + Cfg::kOffStats);
  const uint32_t bar0 = smem_u32(smem + Cfg::kOffBar);
  auto BAR = [&](int i) { return bar0 + 8u * i; };
  // STAGED only: DQ_FULL / DQ_EMPTY + NDQ w + buffer: warpgroup w's dQ staging tiles; DS_FULL / DS_EMPTY + slot:
  // the dS^T slot holds both halves of the tile that uses it / the dQ product reading the slot has retired
  constexpr int NDQ = STAGED ? Cfg::NDQ : 1, NDS = Cfg::NDS;    // (a divisor even where the staging is compiled out)
  constexpr int KV_FULL = 0, FULL = 1, EMPTY = FULL + NST, DQ_FULL = EMPTY + NST, DQ_EMPTY = DQ_FULL + 2 * NDQ,
                DS_FULL = DQ_EMPTY + 2 * NDQ, DS_EMPTY = DS_FULL + NDS, NBARS = DS_EMPTY + NDS;
  static_assert(NBARS * 8 <= 256, "barrier area");
  const Ring<NST> qring = {BAR(FULL), BAR(EMPTY)};            // Q, dO and the stats of a query tile
  const Ring<NDS> dsr = {BAR(DS_FULL), BAR(DS_EMPTY)};        // STAGED: the dS^T slots
  auto dq_ring = [&](int wg_) { return Ring<NDQ>{BAR(DQ_FULL + NDQ * wg_), BAR(DQ_EMPTY + NDQ * wg_)}; };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg = warp >> 2;
  pdl_launch_dependents();

  // ---- work item: one 128-key tile of one (batch, kv head) and a slice of hpc query heads of its group, numbered
  // (key tile, batch, kv head, slice) = (key tile, batch, first query head h0 / hpc); key tiles ascending = heaviest
  // first (causal) ----
  const int slices = HEAD_LOOP ? a.kv_heads * a.split : a.H;     // one query head per CTA: a slice per head
  const int bs_count = a.B * slices;
  const int jt = blockIdx.x / bs_count;
  const int bs = blockIdx.x - jt * bs_count;
  const int b = bs / slices, sl = bs - b * slices;
  const int hk = (HEAD_LOOP || a.split > 1) ? sl / a.split : sl;
  const int hpc = HEAD_LOOP ? a.hpc : 1;
  const int h0 = sl * hpc;                    // = hk * G + (slice within the group) * hpc
  const int key0 = jt * 128;
  // packed sequences: the tensor maps' batch coordinate is 0, the sequence starts at query row q_row0 and key row
  // k_row0, and its stats / dq accumulator at tile qbase of each head; the lengths are read after pdl_wait
  const int tb = VARLEN ? 0 : b;
  int Nq = a.Nq, Nk = a.Nk, nqt = a.nqt, q_row0 = 0, k_row0 = 0, qbase = 0;

  if (threadIdx.x == 0) {
    mbar_init(BAR(KV_FULL), 1);
    qring.init(1, 256);
    dq_ring(0).init(128, 1);                  // filled by a consumer warpgroup, emptied by its reducer thread
    dq_ring(1).init(128, 1);
    dsr.init(128, 128);
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();          // stats come from the preprocess kernel; the dq accumulator is zero on entry
  if constexpr (VARLEN) {
    const SeqSpan sq = seq_span(a.cu_q, b, a.Nq, a.total_q), sk = seq_span(a.cu_k, b, a.Nk, a.total_k);
    Nq = sq.len; Nk = sk.len; q_row0 = sq.start; k_row0 = sk.start;
    nqt = (Nq + QT - 1) / QT;
    qbase = varlen_tile_base(q_row0, b);
    if (key0 >= Nk) return;                   // a key tile past the end of its sequence
  }
  const int off = diag_off(Nq, Nk);
  int W = 0;                                  // the window
  if constexpr (WINDOW) W = a.window;
  const TileRange qr = query_tiles<WINDOW>(key0, off, nqt, a.causal, W);
  const int i_lo = qr.lo, i_end = qr.hi;      // the query tiles [i_lo, i_end) visited per query head
  const int NI = tile_count(qr);              // number of query tiles to visit per query head
  const int NT = hpc * NI;                    // flat tile index i: head h0 + i / NI, query tile i_lo + i % NI

  if (wg == 0) {
    // =============================== TMA producer ===============================
    reg_dealloc<kProducerRegs>();
    if (warp == 0 && elect_one()) {
      tma_prefetch_desc(&tm_q);
      tma_prefetch_desc(&tm_k);
      tma_prefetch_desc(&tm_v);
      tma_prefetch_desc(&tm_do);
      mbar_expect_tx(BAR(KV_FULL), 2 * Cfg::kKV);
#pragma unroll
      for (int ch = 0; ch < KCH; ++ch) {
        tma_load_4d(sK + ch * 16384, &tm_k, BAR(KV_FULL), ch * 64, k_row0 + key0, hk, tb);
        tma_load_4d(sV + ch * 16384, &tm_v, BAR(KV_FULL), ch * 64, k_row0 + key0, hk, tb);
      }
      for (int i = 0, h = h0; h < h0 + hpc; ++h) {
        long long tile0 = ((long long)b * a.H + h) * a.nqt;     // the stats tile of query tile 0
        if constexpr (VARLEN) tile0 = (long long)h * a.ntile + qbase;
        const float* stats_h = a.stats + tile0 * 2 * QT;
        for (int qt = i_lo; qt < i_end; ++qt, ++i) {
          const int st = qring.acquire(i);
          const uint32_t full = qring.full_bar(st);
          mbar_expect_tx(full, 2 * Cfg::kQ + 8 * QT);
#pragma unroll
          for (int ch = 0; ch < KCH; ++ch) {
            tma_load_4d(sQ + st * Cfg::kQ + ch * QCHUNK, &tm_q, full, ch * 64, q_row0 + qt * QT, h, tb);
            tma_load_4d(sDO + st * Cfg::kQ + ch * QCHUNK, &tm_do, full, ch * 64, q_row0 + qt * QT, h, tb);
          }
          bulk_load_1d(sStats + st * 8 * QT, stats_h + (long long)qt * 2 * QT, 8 * QT, full);
        }
      }
    } else if (STAGED && (warp == 1 || warp == 2) && elect_one()) {
      // dQ reducer of consumer warpgroup warp - 1, which owns the query tiles i = warp - 1 (mod 2): each staged
      // 64 x D fp32 tile is added into the accumulator by TMA (rows at or beyond Nq lie outside the tensor map
      // and are not written; with packed sequences the rows of a tail tile past the sequence's end are inside it,
      // and the dq finish kernel clears them)
      const int rw = warp - 1;
      const Ring<NDQ> dqr = dq_ring(rw);
      if (rw == 0) tma_prefetch_desc(&tm_dq);
      for (int i = rw; i < NT; i += 2) {
        const int n = i >> 1;                      // the warpgroup's n-th tile
        const HeadTile ht = head_tile(i, i_lo, NI, HEAD_LOOP);
        const int hh = ht.head, qt = ht.qt;
        const uint32_t src = sDQ + (NDQ * rw + dqr.wait(n)) * Cfg::kDQ;
#pragma unroll
        for (int c = 0; c < D / 32; ++c)
          tma_reduce_add_4d(&tm_dq, src + c * (QT * 128), c * 32, (qbase + qt) * QT, h0 + hh, tb);
        bulk_commit();
        bulk_wait_read<0>();
        dqr.release(n);
      }
      bulk_wait<0>();                          // every reduction performed before the dq finish kernel reads
    }
    return;
  }

  // =============================== consumer warpgroups =============================
  reg_alloc<kConsumerRegs>();
  const int w = wg - 1;                       // keys key0 + 64 w .. + 63
  const int wl = warp & 3;
  const int r8 = lane >> 2;                   // row inside every 8-row group of an accumulator
  const int kr = 16 * wl + r8;                // this thread's key rows inside the warpgroup's 64: kr, kr + 8
  const int cq = 2 * (lane & 3);              // first of the thread's two columns inside every 8-column block
  // key_lo[hf]: the first query row that sees key row kr + 8 hf (causal: key - (Nk - Nq), else 0), or Nq + QT when
  // the key does not exist or is masked - one register per row for the masked elementwise stage.  WINDOW: a key's
  // visible query rows are [key + lo_off, key + hi_off], lo_off = -off (causal) or -off - W + 1, hi_off = W - 1 - off;
  // one register each for both rows (the D = 64 consumers have none to spare)
  int key_g[2], key_lo[2];
  int lo_off = 0, hi_off = 0;
  if constexpr (WINDOW) {
    lo_off = a.causal ? -off : -off - W + 1;
    hi_off = window_hi_off(off, W);
  }
#pragma unroll
  for (int hf = 0; hf < 2; ++hf) {
    key_g[hf] = key0 + 64 * w + kr + 8 * hf;
    bool ok = key_g[hf] < Nk;
    if (a.has_mask && ok) ok = a.mask[(long long)b * a.mask_sb + key_g[hf]] != 0;
    key_lo[hf] = !ok ? Nq + QT : (a.causal ? key_g[hf] - off : 0);
    if constexpr (WINDOW) {
      if (ok) key_lo[hf] = key_g[hf] + lo_off;
    }
  }
  // the warpgroup's keys are all real and unmasked: only query tiles crossing the causal diagonal or the end
  // of the sequence need per-element selects
  const bool keys_full = !a.has_mask && key0 + 64 * w + 64 <= Nk;
  const uint32_t sKw = sK + w * 64 * 128, sVw = sV + w * 64 * 128;    // the warpgroup's 64 rows of every chunk
  const uint32_t ds_thr = kr * 128 + cq * 2;  // the thread's dS^T words: + 1024 hf + 16 (column block ^ r8)
  const float c1 = a.c1;

  // S^T = K Q^T and dP^T = V dO^T (64 keys x QT queries each), one commit group
  auto issue_s_dp = [&](float (&s)[QT / 2], float (&dp)[QT / 2], uint32_t sQs, uint32_t sDOs) {
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk) {
      const uint32_t ka = (kk >> 2) * 16384 + (kk & 3) * 32, kb = (kk >> 2) * QCHUNK + (kk & 3) * 32;
      wgmma_ss_n64<T, 0, 0>(s, gmma_desc_sw128(sKw + ka, 16, 1024), gmma_desc_sw128(sQs + kb, 16, 1024),
                            kk > 0 ? 1u : 0u);
    }
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk) {
      const uint32_t ka = (kk >> 2) * 16384 + (kk & 3) * 32, kb = (kk >> 2) * QCHUNK + (kk & 3) * 32;
      wgmma_ss_n64<T, 0, 0>(dp, gmma_desc_sw128(sVw + ka, 16, 1024), gmma_desc_sw128(sDOs + kb, 16, 1024),
                            kk > 0 ? 1u : 0u);
    }
    wgmma_commit();
  };

  // P^T = exp2(S^T*c1 + c3 [+ bias*log2e]) (masked), dS^T = P^T * (dP^T - delta): 16-bit A fragments in
  // pf / dsf, dS^T also to shared memory (row = key, 128-byte rows of QT = 64 queries, 128B swizzle).
  // Element pair e = 2 j + hf: key row kr + 8 hf, query columns 8 j + cq + {0, 1}.
  auto elementwise = [&](const bool MASKED, const float (&s)[QT / 2], const float (&dp)[QT / 2],
                         uint32_t (&pf)[QT / 4], uint32_t (&dsf)[QT / 4], int row0, uint32_t stc3, uint32_t dsbuf) {
    int hi = QT - 1, lo[2] = {0, 0}, hi_k[2];
    if (MASKED) {
      hi = min(QT - 1, Nq - 1 - row0);                        // last valid query column of the tile
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) {                        // first visible query column of each key row
        lo[hf] = max(0, key_lo[hf] - row0);
        if constexpr (WINDOW) hi_k[hf] = min(hi, key_g[hf] + hi_off - row0);   // ... and the last, with the window
      }
    }
#pragma unroll
    for (int j = 0; j < QT / 8; ++j) {
      const int cc = 8 * j + cq;
      // {c3, -delta} of the two columns, loaded once for both key rows (per key row in the BIAS kernels, whose
      // bias loads leave no registers to hold them)
      float2 c3, ndl;
      if constexpr (!BIAS) {
        c3 = lds64f(stc3 + 4 * cc);
        ndl = lds64f(stc3 + 4 * QT + 4 * cc);
      }
      const uint32_t ds_addr = dsbuf + ds_thr + ((j ^ r8) << 4);
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) {
        const int e = 2 * j + hf;
        if constexpr (BIAS) {
          c3 = lds64f(stc3 + 4 * cc);
          ndl = lds64f(stc3 + 4 * QT + 4 * cc);
        }
        float x0 = fmaf(s[2 * e], c1, c3.x), x1 = fmaf(s[2 * e + 1], c1, c3.y);
        if constexpr (BIAS) {
          // (BIAS launches have one query head per CTA: h0)
          const uint8_t* bcol = reinterpret_cast<const uint8_t*>(a.bias) +
                                2 * ((long long)b * a.bias_sb + (long long)h0 * a.bias_sh + min(key_g[hf], a.Nk - 1));
          const int q0 = min(row0 + cc, a.Nq - 1), q1 = min(row0 + cc + 1, a.Nq - 1);
          const float2 bv = unpack2<T>(ldg_u16(bcol + 2 * (long long)q0 * a.bias_sn) |
                                       (ldg_u16(bcol + 2 * (long long)q1 * a.bias_sn) << 16));
          x0 = fmaf(bv.x, 1.4426950408889634f, x0);
          x1 = fmaf(bv.y, 1.4426950408889634f, x1);
        }
        const int hk_ = WINDOW ? hi_k[hf] : hi;
        const bool v0 = !MASKED || (cc >= lo[hf] && cc <= hk_), v1 = !MASKED || (cc + 1 >= lo[hf] && cc + 1 <= hk_);
        const float p0 = v0 ? ex2_approx(x0) : 0.f;
        const float p1 = v1 ? ex2_approx(x1) : 0.f;
        const float ds0 = p0 * (dp[2 * e] + ndl.x), ds1 = p1 * (dp[2 * e + 1] + ndl.y);
        pf[e] = pack2<T>(p0, p1);
        dsf[e] = pack2<T>(ds0, ds1);
        if constexpr (DQ) sts32(ds_addr + 1024 * hf, dsf[e]);
        if constexpr (BIAS) {
          // d bias = dS (reference cu:1574-1576): fp32 reduction
          if (a.dbias != nullptr) {
            float* dst = a.dbias + (long long)b * a.dbias_sb + (long long)h0 * a.dbias_sh + key_g[hf];
            if (v0) red_add_f32(dst + (long long)(row0 + cc) * a.Nk, ds0);
            if (v1) red_add_f32(dst + (long long)(row0 + cc + 1) * a.Nk, ds1);
          }
        }
      }
    }
  };
  auto elementwise_tile = [&](const float (&s)[QT / 2], const float (&dp)[QT / 2], uint32_t (&pf)[QT / 4],
                              uint32_t (&dsf)[QT / 4], int row0, uint32_t stc3, uint32_t dsbuf) {
    // interior tile: every key of the warpgroup sees every query row (no causal diagonal, no ragged end)
    bool interior = keys_full && row0 + QT <= Nq && (!a.causal || key0 + 64 * w + 63 - off <= row0);
    // (window: the tile's rows lie between the last key's first visible row and the first key's last one)
    if constexpr (WINDOW)
      interior = keys_full && row0 + QT <= Nq && key0 + 64 * w + 63 + lo_off <= row0 &&
                 row0 + QT - 1 <= key0 + 64 * w + hi_off;
    if (!BIAS && interior) elementwise(false, s, dp, pf, dsf, row0, stc3, dsbuf);
    else elementwise(true, s, dp, pf, dsf, row0, stc3, dsbuf);
    if constexpr (DQ) {
      fence_proxy_async_smem();
      named_bar_sync(1 + w, 128);             // the warpgroup's whole dS^T tile is in shared memory
    }
  };

  // dV += P^T dO, dK += dS^T Q (A from registers)
  auto issue_dv_dk = [&](const uint32_t (&pf)[QT / 4], const uint32_t (&dsf)[QT / 4], uint32_t sQs, uint32_t sDOs,
                         float (&dv)[D / 2], float (&dk)[D / 2]) {
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < QT / 16; ++kk) {
      const uint32_t af[4] = {pf[4 * kk], pf[4 * kk + 1], pf[4 * kk + 2], pf[4 * kk + 3]};
      wgmma_rs<T, 1>(dv, af, gmma_desc_sw128(sDOs + kk * 2048, QCHUNK, 1024), 1u);
    }
#pragma unroll
    for (int kk = 0; kk < QT / 16; ++kk) {
      const uint32_t af[4] = {dsf[4 * kk], dsf[4 * kk + 1], dsf[4 * kk + 2], dsf[4 * kk + 3]};
      wgmma_rs<T, 1>(dk, af, gmma_desc_sw128(sQs + kk * 2048, QCHUNK, 1024), 1u);
    }
  };
  // dQ = dS K.  STAGED: contraction over all 128 keys of the CTA (dsbuf = a dS^T slot, whose two warpgroup halves
  // are contiguous: 16 keys = 2048 bytes throughout); otherwise a partial over the warpgroup's 64 keys.
  auto issue_dq = [&](float (&dq)[D / 2], uint32_t dsbuf) {
    constexpr int NKK = STAGED ? 8 : 4;
    const uint32_t sKd = STAGED ? sK : sKw;
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < NKK; ++kk) {
      const uint64_t da = gmma_desc_sw128(dsbuf + kk * 2048, 8192, 1024);     // dS: queries contiguous (MN-major)
      const uint64_t db = gmma_desc_sw128(sKd + kk * 2048, 16384, 1024);      // K: features contiguous (MN-major)
      wgmma_ss<T, 1, 1>(dq, da, db, kk > 0 ? 1u : 0u);
    }
  };

  float dv[D / 2], dk[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) dv[i] = dk[i] = 0.f;
  // the producer loads K and V whatever NI; the epilogue reads K (l2norm backward) even when no query tile is visited
  mbar_wait(BAR(KV_FULL), 0);

  if constexpr (STAGED) {
    // One dQ tile per query tile and CTA, dQ(i) = [dS_0(i) | dS_1(i)] K over all 128 keys, owned by warpgroup i & 1
    // (i = loop index, so both warpgroups agree; the last tile has one owner whatever NI).  The owner issues it one
    // tile late, in the batch of tile i + 1 behind dV / dK(i + 1) and ahead of S^T / dP^T(i + 2) (20 wgmmas, one
    // wait per tile); the other warpgroup has then almost always written its half of dS^T(i).  Tile i's dS^T lives
    // in slot i % NDS (both halves, slot-major):
    //   DS_FULL  : the non-owner fences its half to the async proxy and arrives (128 threads) after writing it;
    //              the owner waits before issuing dQ(i)
    //   DS_EMPTY : the owner arrives (128 threads) after the wait that retires dQ(i); the owner of tile
    //              i + NDS (the other warpgroup, NDS being odd) waits before writing its half of the slot again.
    //              The non-owner of i + NDS owns i and has retired dQ(i) itself.
    // dQ(i) is retired by the owner's wait at iteration i + 2 and leaves through shared memory: the warpgroup
    // stores the fp32 tile (128B swizzle, the layout of a 32-feature TMA box) and its reducer warp adds it into
    // the accumulator.  Each warpgroup stages every other tile.
    // Staging word of accumulator pair (jb, hf): box jb / 4, row 16 wl + r8 + 8 hf, 16-byte chunk
    // (2 (jb & 3) + (lane & 3) / 2) ^ r8, 8-byte half lane & 1.  Each warp store covers all 32 banks twice.
    static_assert(NDS % 2 == 1, "consecutive users of a dS^T slot must have different owners");
    const uint32_t dq_thr = (16 * wl + r8) * 128 + (lane & 1) * 8;
    const int dq_sx = ((lane & 3) >> 1) ^ r8;
    float s[QT / 2], dp[QT / 2], dq[D / 2];
    uint32_t pf[QT / 4], dsf[QT / 4];
#pragma unroll
    for (int k = 0; k < D / 2; ++k) dq[k] = 0.f;
    auto ds_slot = [&](int i) { return sDS + 2 * (i % NDS) * Cfg::kDS; };
    const Ring<NDQ> dqr = dq_ring(w);
    auto stage_dq = [&](int i) {              // i & 1 == w
      const int n = i >> 1;
      const int sb = dqr.acquire(n);          // the reducer has read the buffer's last tile
      const uint32_t dst = sDQ + (NDQ * w + sb) * Cfg::kDQ + dq_thr;
#pragma unroll
      for (int jb = 0; jb < D / 8; ++jb) {
        const uint32_t o = dst + (jb >> 2) * (QT * 128) + (((2 * (jb & 3)) ^ dq_sx) << 4);
        sts64f(o, dq[4 * jb], dq[4 * jb + 1]);
        sts64f(o + 1024, dq[4 * jb + 2], dq[4 * jb + 3]);
      }
      fence_proxy_async_smem();
      dqr.commit(n);
    };
    // dQ(i) retired: release its dS^T slot, stage the tile
    auto retire_dq = [&](int i) {
      dsr.release(i);
      stage_dq(i);
    };
    auto issue_owned_dq = [&](int i) {        // i & 1 == w
      dsr.wait(i);
      issue_dq(dq, ds_slot(i));
    };

    // The zero accumulators are pinned before the first issue: a register move of dV / dK / dQ that the compiler
    // schedules while a wgmma is in flight makes ptxas serialise every wgmma of the kernel.
    fence_regs(dv);
    fence_regs(dk);
    fence_regs(dq);
    if (NT > 0) {
      qring.wait(0);
      issue_s_dp(s, dp, sQ, sDO);
      // i runs over the flat (head, query tile) sequence; row0 restarts at i_lo * QT with every head (next_row0)
      for (int i = 0, row0 = i_lo * QT; i < NT; ++i,
               row0 = HEAD_LOOP ? next_row0<WINDOW>(row0, i_lo, VARLEN ? Nq : a.nqt * QT, key0, hi_off) : row0 + QT) {
        const int st = i % NST;
        const uint32_t sQs = sQ + st * Cfg::kQ, sDOs = sDO + st * Cfg::kQ;
        wgmma_wait<0>();                        // S^T, dP^T of tile i; dV, dK of tile i - 1; dQ of tile i - 2
        fence_regs(s);
        fence_regs(dp);
        fence_regs(dv);
        fence_regs(dk);
        fence_regs(dq);
        fence_regs(pf);
        fence_regs(dsf);
        if (i >= 2 && ((i - 2) & 1) == w) retire_dq(i - 2);
        if (i > 0) qring.release(i - 1);        // Q, dO and the stats of tile i - 1 are no longer read
        const bool own = (i & 1) == w;
        if (own && i >= NDS) dsr.acquire(i);
        elementwise_tile(s, dp, pf, dsf, row0, sStats + st * 8 * QT, ds_slot(i) + w * Cfg::kDS);
        // the slot arithmetic below is redone from an opaque copy of i rather than kept live through the elementwise
        // stage (the BIAS kernels have no register to spare there)
        int io = i;
        asm volatile("" : "+r"(io));
        if ((io & 1) != w) dsr.commit(io);
        issue_dv_dk(pf, dsf, sQs, sDOs, dv, dk);
        if (io >= 1 && (io & 1) != w) issue_owned_dq(io - 1);
        wgmma_commit();
        if (i + 1 < NT) {
          const int sn = qring.wait(i + 1);
          issue_s_dp(s, dp, sQ + sn * Cfg::kQ, sDO + sn * Cfg::kQ);
        }
      }
      // drain: dQ(NT - 2) is in flight if this warpgroup owns it, dQ(NT - 1) is not issued yet
      wgmma_wait<0>();
      fence_regs(dv);
      fence_regs(dk);
      fence_regs(dq);
      if (NT >= 2 && ((NT - 2) & 1) == w) retire_dq(NT - 2);
      qring.release(NT - 1);
      if (((NT - 1) & 1) == w) {
        issue_owned_dq(NT - 1);
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(dq);
        retire_dq(NT - 1);
      }
    }
  } else {
    for (int i = 0; i < NT; ++i) {
      const HeadTile ht = head_tile(i, i_lo, NI, HEAD_LOOP);
      const int hh = ht.head, row0 = ht.qt * QT;
      const int st = qring.wait(i);
      const uint32_t sQs = sQ + st * Cfg::kQ, sDOs = sDO + st * Cfg::kQ;
      float s[QT / 2], dp[QT / 2];
      issue_s_dp(s, dp, sQs, sDOs);
      wgmma_wait<0>();
      fence_regs(s);
      fence_regs(dp);

      const uint32_t dsbuf = sDS + (2 * (i & 1) + w) * Cfg::kDS;
      uint32_t pf[QT / 4], dsf[QT / 4];
      elementwise_tile(s, dp, pf, dsf, row0, sStats + st * 8 * QT, dsbuf);
      issue_dv_dk(pf, dsf, sQs, sDOs, dv, dk);
      wgmma_commit();
      wgmma_wait<0>();                          // the dQ accumulator only fits once the A fragments are dead
      fence_regs(pf);
      fence_regs(dsf);
      if constexpr (!DQ) {
        fence_regs(dv);
        fence_regs(dk);
        qring.release(i);                       // Q, dO and the stats of this stage are no longer read
        continue;
      }
      float dq[D / 2];
      issue_dq(dq, dsbuf);
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs(dv);
      fence_regs(dk);
      fence_regs(dq);
      qring.release(i);                         // Q, dO and the stats of this stage are no longer read

      // ---- dQ partial tile -> fp32 accumulator (rows = queries, columns = features) ----
      long long tile0 = ((long long)b * a.H + h0 + hh) * a.nqt;     // the accumulator tile of query tile 0
      if constexpr (VARLEN) tile0 = (long long)(h0 + hh) * a.ntile + qbase;
      float* acc = a.dq_acc + (tile0 * QT + row0) * D + cq;
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) {
        const int q = 16 * wl + r8 + 8 * hf;
        if (row0 + q < Nq) {
#pragma unroll
          for (int jb = 0; jb < D / 8; ++jb)
            red_add_f32x2(acc + (long long)q * D + 8 * jb, dq[4 * jb + 2 * hf], dq[4 * jb + 2 * hf + 1]);
        }
      }
    }
  }

  // ---- epilogue: dV and dK * scale of the warpgroup's 64 keys ---------------------------------
  // (no early exit for keys at or beyond Nk: the l2norm backward below shuffles within the quad of a key row)
  const bool to_acc = DQ && a.split > 1;
  long long krow0 = ((long long)b * a.kv_heads + hk) * a.Nk;     // the row of key 0 in k_rnorm and dk_acc / dv_acc
  if constexpr (VARLEN) {
    // the key span is read again rather than kept in registers through the main loop
    const SeqSpan sk = seq_span(a.cu_k, b, a.Nk, a.total_k);
    Nk = sk.len;
    k_row0 = sk.start;
    krow0 = (long long)hk * a.total_k + k_row0;
  }
#pragma unroll
  for (int hf = 0; hf < 2; ++hf) {
    const int key = key_g[hf];
    const bool in = key < Nk;
    if (to_acc) {
      // the group's heads are split over several CTAs: sum over them in fp32 (reference: cu:1613-1619)
      float* pv = a.dv_acc + (krow0 + key) * D + cq;
      float* pk = a.dk_acc + (krow0 + key) * D + cq;
      if (in) {
#pragma unroll
        for (int jb = 0; jb < D / 8; ++jb) {
          red_add_f32x2(pv + 8 * jb, dv[4 * jb + 2 * hf], dv[4 * jb + 2 * hf + 1]);
          red_add_f32x2(pk + 8 * jb, dk[4 * jb + 2 * hf] * a.scale, dk[4 * jb + 2 * hf + 1] * a.scale);
        }
      }
    } else if (!VARLEN && a.out_f32) {
      float* pv = reinterpret_cast<float*>(a.dv) + b * a.dv_sb + hk * a.dv_sh + (long long)key * a.dv_sn + cq;
      float* pk = reinterpret_cast<float*>(a.dk) + b * a.dk_sb + hk * a.dk_sh + (long long)key * a.dk_sn + cq;
      if (in) {
#pragma unroll
        for (int jb = 0; jb < D / 8; ++jb) {
          *reinterpret_cast<float2*>(pv + 8 * jb) = make_float2(dv[4 * jb + 2 * hf], dv[4 * jb + 2 * hf + 1]);
          *reinterpret_cast<float2*>(pk + 8 * jb) =
              make_float2(dk[4 * jb + 2 * hf] * a.scale, dk[4 * jb + 2 * hf + 1] * a.scale);
        }
      }
    } else {
      T* pv = reinterpret_cast<T*>(a.dv) + tb * a.dv_sb + hk * a.dv_sh + (long long)(k_row0 + key) * a.dv_sn + cq;
      T* pk = reinterpret_cast<T*>(a.dk) + tb * a.dk_sb + hk * a.dk_sh + (long long)(k_row0 + key) * a.dk_sn + cq;
      if (in) {
#pragma unroll
        for (int jb = 0; jb < D / 8; ++jb)
          *reinterpret_cast<uint32_t*>(pv + 8 * jb) = pack2<T>(dv[4 * jb + 2 * hf], dv[4 * jb + 2 * hf + 1]);
      }
      // g[2 jb + e] = dk_hat of feature 8 jb + cq + e
      float g[D / 4];
#pragma unroll
      for (int jb = 0; jb < D / 8; ++jb) {
        g[2 * jb] = dk[4 * jb + 2 * hf] * a.scale;
        g[2 * jb + 1] = dk[4 * jb + 2 * hf + 1] * a.scale;
      }
      if (a.k_rnorm != nullptr)
        l2norm_bwd_key_row<T, D>(g, a.k_rnorm, a.groups, sK + (64 * w + kr + 8 * hf) * 128, krow0, key, in);
      if (in) {
#pragma unroll
        for (int jb = 0; jb < D / 8; ++jb)
          *reinterpret_cast<uint32_t*>(pk + 8 * jb) = pack2<T>(g[2 * jb], g[2 * jb + 1]);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// 3. finish kernels (dq; shared-kv dk/dv)
// ------------------------------------------------------------------------------------------
struct DqFinishArgs {
  int B, H, Nq, D, nqt, padded;     // padded = nqt * QT rows per (batch, head) in the accumulator
  float scale;
  int out_f32;                      // 1: dq is float32
  float* dq_acc;
  void* dq; long long sb, sh, sn;
  // when q_rnorm is set, dq is the gradient w.r.t. the RAW queries (l2norm backward applied here)
  const void* q_hat; long long q_sb, q_sh, q_sn;
  const float* q_rnorm;             // (B, H, Nq, G) or nullptr
  int G;
};

// Packed sequences: B sequences, Nq = the maximum length, padded = ceil(Nq / QT) * QT (the grid covers that many rows
// of every (sequence, head)); dq, q_hat are (total_q, H, D) (sb, q_sb unused), q_rnorm is (H, total_q, G) and the
// accumulator of head h, sequence b starts at tile h * ntile + base(b).
struct DqFinishVarlenArgs : DqFinishArgs {
  const int* cu_q;
  int total_q, ntile;
};

// dq conversion (reference: the fp32 -> scalar_t cast of dq after its atomics, cu:1904): TPR = D / 8 consecutive lanes
// per query row, 8 features each, and two rows per thread in the dense kernels (one in the VARLEN ones).  The accumulator is read from L2 (the reductions of the main kernel have just
// produced it there), converted, and written back as zeros: it is zero between launches.
// VARLEN: every row of a sequence's tiles is cleared, the padding rows past its end included.  Those lie inside the
// accumulator's tensor map and receive dS K for masked queries: exact zeros for finite K, NaN when the neighbouring rows
// the tail tile reads hold non-finite values - cleared here, so the zeroed workspace stays zero for every later call.
template <typename T, int D, bool VARLEN = false>
__global__ void __launch_bounds__(256)
bwd_dq_finish_kernel(const std::conditional_t<VARLEN, DqFinishVarlenArgs, DqFinishArgs> a) {
  pdl_launch_dependents();
  pdl_wait();
  constexpr int TPR = D / 8;
  if constexpr (VARLEN) {
    constexpr int QT = 64;
    const long long t = (long long)blockIdx.x * 256 + threadIdx.x;
    const long long rowid = t / TPR;                       // over (sequences*heads) x padded
    const int c8 = (int)(t % TPR);
    const bool in_grid = rowid < (long long)a.B * a.H * a.padded;
    const long long bh = in_grid ? rowid / a.padded : 0;
    const int r = (int)(rowid - bh * a.padded);
    const int b = (int)(bh / a.H), h = (int)(bh % a.H);
    const SeqSpan sq = seq_span(a.cu_q, b, a.Nq, a.total_q);
    const bool own = in_grid && r < (sq.len + QT - 1) / QT * QT;    // a row of the sequence's tiles
    const bool ok = in_grid && r < sq.len;                          // ... and of the sequence (whole rows of lanes)
    float* src = a.dq_acc + (((long long)h * a.ntile + varlen_tile_base(sq.start, b)) * QT + r) * D + c8 * 8;
    const long long row = (long long)sq.start + r;                  // the packed row
    float4 lo = make_float4(0.f, 0.f, 0.f, 0.f), hi = lo;
    if (own) {
      lo = ldg_cg128f(src);
      hi = ldg_cg128f(src + 4);
      *reinterpret_cast<float4*>(src) = make_float4(0.f, 0.f, 0.f, 0.f);
      *reinterpret_cast<float4*>(src + 4) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    float g[8] = {lo.x * a.scale, lo.y * a.scale, lo.z * a.scale, lo.w * a.scale,
                  hi.x * a.scale, hi.y * a.scale, hi.z * a.scale, hi.w * a.scale};
    if (a.q_rnorm != nullptr) {
      float y[8];
      unpack16B<T>(ok ? ldg_stream128(reinterpret_cast<const T*>(a.q_hat) + h * a.q_sh + row * a.q_sn + c8 * 8)
                      : make_uint4(0, 0, 0, 0), y);
      l2norm_bwd_group<8>(g, y, D / a.G, c8, ok ? a.q_rnorm + ((long long)h * a.total_q + row) * a.G : nullptr, 1.f);
    }
    if (!ok) return;
    T* dst = reinterpret_cast<T*>(a.dq) + h * a.sh + row * a.sn + c8 * 8;
    *reinterpret_cast<uint4*>(dst) = pack16B<T>(g);
    return;
  }
  // Two rows per thread, 256 / TPR rows apart (a block covers 2 x 256 / TPR consecutive rows): every load of both rows
  // is issued before any of them is used.  Row indices in 32 bits whenever the grid's rows fit (the divisions by Nq
  // and H are then a few instructions instead of a 64-bit division routine each).
  constexpr int RPB = 256 / TPR;
  const long long nrows = (long long)a.B * a.H * a.Nq;
  const bool small = nrows < 0x7FFFFFFFLL;
  const int c8 = threadIdx.x % TPR;
  long long bhs[2];
  int rows[2];
  bool oks[2];
  float4 lo[2], hi[2];
  uint4 yq[2];
  float rn[2];
#pragma unroll
  for (int u = 0; u < 2; ++u) {
    const long long rowid = ((long long)blockIdx.x * 2 + u) * RPB + threadIdx.x / TPR;    // over (batch*heads) x Nq
    const bool ok = rowid < nrows;                         // whole rows of TPR lanes (shuffles stay in them)
    long long bh = 0;
    int row = 0;
    if (ok) {
      if (small) {
        const unsigned r32 = (unsigned)rowid, q32 = r32 / (unsigned)a.Nq;
        bh = q32;
        row = (int)(r32 - q32 * (unsigned)a.Nq);
      } else {
        bh = rowid / a.Nq;
        row = (int)(rowid - bh * a.Nq);
      }
    }
    bhs[u] = bh;
    rows[u] = row;
    oks[u] = ok;
    lo[u] = hi[u] = make_float4(0.f, 0.f, 0.f, 0.f);
    yq[u] = make_uint4(0, 0, 0, 0);
    rn[u] = 0.f;
    if (ok) {
      const float* src = a.dq_acc + (bh * a.padded + row) * D + c8 * 8;
      lo[u] = ldg_cg128f(src);
      hi[u] = ldg_cg128f(src + 4);
    }
  }
#pragma unroll
  for (int u = 0; u < 2; ++u) {
    if (!oks[u] || a.q_rnorm == nullptr) continue;
    const int b = (int)(bhs[u] / a.H), h = (int)(bhs[u] - (long long)b * a.H);
    yq[u] = ldg_stream128(reinterpret_cast<const T*>(a.q_hat) + b * a.q_sb + h * a.q_sh + (long long)rows[u] * a.q_sn +
                          c8 * 8);
  }
#pragma unroll
  for (int u = 0; u < 2; ++u) {
    const bool ok = oks[u];
    const long long bh = bhs[u];
    const int row = rows[u];
    const int b = (int)(bh / a.H), h = (int)(bh - (long long)b * a.H);
    if (ok) {
      float* src = a.dq_acc + (bh * a.padded + row) * D + c8 * 8;
      *reinterpret_cast<float4*>(src) = make_float4(0.f, 0.f, 0.f, 0.f);
      *reinterpret_cast<float4*>(src + 4) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    float g[8] = {lo[u].x * a.scale, lo[u].y * a.scale, lo[u].z * a.scale, lo[u].w * a.scale,
                  hi[u].x * a.scale, hi[u].y * a.scale, hi[u].z * a.scale, hi[u].w * a.scale};
    if (a.q_rnorm != nullptr) {                           // uniform across the grid
      float y[8];
      unpack16B<T>(yq[u], y);
      l2norm_bwd_group<8>(g, y, D / a.G, c8, ok ? a.q_rnorm + (((long long)b * a.H + h) * a.Nq + row) * a.G : nullptr,
                          1.f);
    }
    if (!ok) continue;
    if (a.out_f32) {
      float* dst = reinterpret_cast<float*>(a.dq) + b * a.sb + h * a.sh + (long long)row * a.sn + c8 * 8;
      *reinterpret_cast<float4*>(dst) = make_float4(g[0], g[1], g[2], g[3]);
      *reinterpret_cast<float4*>(dst + 4) = make_float4(g[4], g[5], g[6], g[7]);
    } else {
      T* dst = reinterpret_cast<T*>(a.dq) + b * a.sb + h * a.sh + (long long)row * a.sn + c8 * 8;
      *reinterpret_cast<uint4*>(dst) = pack16B<T>(g);
    }
  }
}

struct KvFinishArgs {
  int B, Hk, Nk, D, out_f32;
  const float* acc;                 // (B, Hk, Nk, D) fp32
  void* out; long long sb, sh, sn;
};
template <typename T>
__global__ void __launch_bounds__(256) bwd_kv_finish_kernel(const KvFinishArgs a) {
  const int tpr = a.D >> 3;
  const long long idx = (long long)blockIdx.x * 256 + threadIdx.x;
  const long long total = (long long)a.B * a.Hk * a.Nk * tpr;
  if (idx >= total) return;
  const int c8 = (int)(idx % tpr);
  const long long rowid = idx / tpr;
  const int n = (int)(rowid % a.Nk);
  const long long bh = rowid / a.Nk;
  const int b = (int)(bh / a.Hk), h = (int)(bh % a.Hk);
  const float* src = a.acc + rowid * a.D + c8 * 8;
  const float4 lo = *reinterpret_cast<const float4*>(src);
  const float4 hi = *reinterpret_cast<const float4*>(src + 4);
  const long long doff = b * a.sb + h * a.sh + (long long)n * a.sn + c8 * 8;
  if (a.out_f32) {
    float* dst = reinterpret_cast<float*>(a.out) + doff;
    *reinterpret_cast<float4*>(dst) = lo;
    *reinterpret_cast<float4*>(dst + 4) = hi;
    return;
  }
  uint4 o4;
  o4.x = pack2<T>(lo.x, lo.y);
  o4.y = pack2<T>(lo.z, lo.w);
  o4.z = pack2<T>(hi.x, hi.y);
  o4.w = pack2<T>(hi.z, hi.w);
  T* dst = reinterpret_cast<T*>(a.out) + doff;
  *reinterpret_cast<uint4*>(dst) = o4;
}

}  // namespace fcsa
