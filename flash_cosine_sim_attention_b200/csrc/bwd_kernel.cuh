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
#include "l2norm_kernels.cuh"
#include "sm90_primitives.cuh"
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

__device__ __forceinline__ float lg2_approx(float x) {
  float y;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// TPR = threads per row = D / 8 (8 or 16); QT = 64.
template <typename T, int TPR>
__global__ void __launch_bounds__(256) bwd_prep_kernel(const PrepArgs a) {
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
  const int padded = a.nqt * QT;
  const float c2 = a.c2 + (a.shift_extra != nullptr ? fmaxf(__ldg(a.shift_extra), 0.f) * 1.4426950408889634f : 0.f);
  const long long o_off = b * a.o_sb + h * a.o_sh + tr * 8;
  const T* obase = reinterpret_cast<const T*>(a.o) + o_off;
  const float* obase32 = reinterpret_cast<const float*>(a.o) + o_off;
  const T* dbase = reinterpret_cast<const T*>(a.d_o) + b * a.do_sb + h * a.do_sh + tr * 8;
  int row[2];
  bool in[2], valid[2];
  uint4 ro[2], rd[2];
  float4 rof[2][2];                           // o as float32 (o_f32 problems): 8 features = two float4
  float il[2];
#pragma unroll
  for (int u = 0; u < 2; ++u) {
    row[u] = (blk * 2 + u) * RPB + threadIdx.x / TPR;     // row inside the padded (nqt*QT) range
    in[u] = row[u] < padded;
    valid[u] = in[u] && row[u] < a.Nq;
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
      if (tr == 0) il[u] = __ldg(a.inv_l + (long long)bh * a.Nq + row[u]);
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
    float* st = a.stats + ((long long)bh * a.nqt + qt) * 2 * QT;
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
// chunks 16 KB apart).  All lanes of the warp must call it (quad shuffles); `in` = the key exists.
template <typename T, int D>
__device__ __forceinline__ void l2norm_bwd_key_row(float (&g)[D / 4], const BwdArgs& a, uint32_t sk_row, int b, int hk,
                                                   int key, bool in) {
  const int lane = threadIdx.x & 31;
  const int r8 = (lane >> 2) & 7, cq = 2 * (lane & 3);
  const int gs = D / a.groups;                  // features per group (a power of two)
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
  const float* rn = a.k_rnorm + (((long long)b * a.kv_heads + hk) * a.Nk + (in ? key : 0)) * a.groups;
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

// HEAD_LOOP: the CTA works through several query heads (hpc > 1, grouped-query launches); otherwise hpc = 1 is a
// compile-time constant and the loops below are those of one query head (MHA, MQA, BIAS and split groups of one head).
template <typename T, int D, bool BIAS = false, bool HEAD_LOOP = false>
__global__ void __launch_bounds__(384, 1)
fcsa_bwd_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_k,
                const __grid_constant__ CUtensorMap tm_v, const __grid_constant__ CUtensorMap tm_do,
                const __grid_constant__ CUtensorMap tm_dq, const BwdArgs a) {
  static_assert(D == 64 || D == 128, "head dim 64 or 128");
  static_assert(!(BIAS && HEAD_LOOP), "BIAS launches have one query head per CTA");
  using Cfg = BwdCfg<D>;
  constexpr bool STAGED = Cfg::kStaged;
  constexpr int QT = Cfg::QT;              // query rows per tile
  constexpr int KCH = D / 64;              // 64-feature chunks of every operand tile
  constexpr int QCHUNK = QT * 128;         // bytes of one 64-feature chunk of a Q / dO stage
  constexpr int NST = Cfg::NST;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~uintptr_t(1023));
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
  const int off = a.Nk - a.Nq;
  int i_lo = 0;
  if (a.causal) {
    // first query tile with a row that can see key0: QT*i + QT-1 + off >= key0
    const int x = key0 - off - (QT - 1);
    i_lo = x <= 0 ? 0 : (x + QT - 1) / QT;
  }
  const int NI = max(0, a.nqt - i_lo);        // number of query tiles to visit per query head
  const int NT = hpc * NI;                    // flat tile index i: head h0 + i / NI, query tile i_lo + i % NI

  if (threadIdx.x == 0) {
    mbar_init(BAR(KV_FULL), 1);
    for (int s = 0; s < NST; ++s) {
      mbar_init(BAR(FULL + s), 1);
      mbar_init(BAR(EMPTY + s), 256);
    }
    for (int s = 0; s < 2 * NDQ; ++s) {
      mbar_init(BAR(DQ_FULL + s), 128);
      mbar_init(BAR(DQ_EMPTY + s), 1);
    }
    for (int s = 0; s < NDS; ++s) {
      mbar_init(BAR(DS_FULL + s), 128);
      mbar_init(BAR(DS_EMPTY + s), 128);
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();          // stats come from the preprocess kernel; the dq accumulator is zero on entry

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
        tma_load_4d(sK + ch * 16384, &tm_k, BAR(KV_FULL), ch * 64, key0, hk, b);
        tma_load_4d(sV + ch * 16384, &tm_v, BAR(KV_FULL), ch * 64, key0, hk, b);
      }
      for (int i = 0, h = h0; h < h0 + hpc; ++h) {
        const float* stats_h = a.stats + ((long long)b * a.H + h) * a.nqt * 2 * QT;
        for (int qt = i_lo; qt < a.nqt; ++qt, ++i) {
          const int st = i % NST;
          mbar_wait(BAR(EMPTY + st), ((i / NST) & 1) ^ 1);
          mbar_expect_tx(BAR(FULL + st), 2 * Cfg::kQ + 8 * QT);
#pragma unroll
          for (int ch = 0; ch < KCH; ++ch) {
            tma_load_4d(sQ + st * Cfg::kQ + ch * QCHUNK, &tm_q, BAR(FULL + st), ch * 64, qt * QT, h, b);
            tma_load_4d(sDO + st * Cfg::kQ + ch * QCHUNK, &tm_do, BAR(FULL + st), ch * 64, qt * QT, h, b);
          }
          bulk_load_1d(sStats + st * 8 * QT, stats_h + (long long)qt * 2 * QT, 8 * QT, BAR(FULL + st));
        }
      }
    } else if (STAGED && (warp == 1 || warp == 2) && elect_one()) {
      // dQ reducer of consumer warpgroup warp - 1, which owns the query tiles i = warp - 1 (mod 2): each staged
      // 64 x D fp32 tile is added into the accumulator by TMA (rows at or beyond Nq lie outside the tensor map
      // and are not written)
      const int rw = warp - 1;
      if (rw == 0) tma_prefetch_desc(&tm_dq);
      for (int i = rw; i < NT; i += 2) {
        const int n = i >> 1, sb = n % NDQ;        // the warpgroup's n-th tile
        const int hh = HEAD_LOOP ? i / NI : 0, qt = i_lo + i - hh * NI;
        const uint32_t src = sDQ + (NDQ * rw + sb) * Cfg::kDQ;
        mbar_wait(BAR(DQ_FULL + NDQ * rw + sb), (n / NDQ) & 1);
#pragma unroll
        for (int c = 0; c < D / 32; ++c) tma_reduce_add_4d(&tm_dq, src + c * (QT * 128), c * 32, qt * QT, h0 + hh, b);
        bulk_commit();
        bulk_wait_read<0>();
        mbar_arrive(BAR(DQ_EMPTY + NDQ * rw + sb));
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
  // the key does not exist or is masked - one register per row for the masked elementwise stage
  int key_g[2], key_lo[2];
#pragma unroll
  for (int hf = 0; hf < 2; ++hf) {
    key_g[hf] = key0 + 64 * w + kr + 8 * hf;
    bool ok = key_g[hf] < a.Nk;
    if (a.has_mask && ok) ok = a.mask[(long long)b * a.mask_sb + key_g[hf]] != 0;
    key_lo[hf] = !ok ? a.Nq + QT : (a.causal ? key_g[hf] - off : 0);
  }
  // the warpgroup's keys are all real and unmasked: only query tiles crossing the causal diagonal or the end
  // of the sequence need per-element selects
  const bool keys_full = !a.has_mask && key0 + 64 * w + 64 <= a.Nk;
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
    int hi = QT - 1, lo[2] = {0, 0};
    if (MASKED) {
      hi = min(QT - 1, a.Nq - 1 - row0);                      // last valid query column of the tile
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) {                        // first visible query column of each key row
        lo[hf] = max(0, key_lo[hf] - row0);
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
        const bool v0 = !MASKED || (cc >= lo[hf] && cc <= hi), v1 = !MASKED || (cc + 1 >= lo[hf] && cc + 1 <= hi);
        const float p0 = v0 ? ex2_approx(x0) : 0.f;
        const float p1 = v1 ? ex2_approx(x1) : 0.f;
        const float ds0 = p0 * (dp[2 * e] + ndl.x), ds1 = p1 * (dp[2 * e + 1] + ndl.y);
        pf[e] = pack2<T>(p0, p1);
        dsf[e] = pack2<T>(ds0, ds1);
        sts32(ds_addr + 1024 * hf, dsf[e]);
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
    const bool interior = keys_full && row0 + QT <= a.Nq && (!a.causal || key0 + 64 * w + 63 - off <= row0);
    if (!BIAS && interior) elementwise(false, s, dp, pf, dsf, row0, stc3, dsbuf);
    else elementwise(true, s, dp, pf, dsf, row0, stc3, dsbuf);
    fence_proxy_async_smem();
    named_bar_sync(1 + w, 128);               // the warpgroup's whole dS^T tile is in shared memory
  };

  // dV += P^T dO, dK += dS^T Q (A from registers)
  auto issue_dv_dk = [&](const uint32_t (&pf)[QT / 4], const uint32_t (&dsf)[QT / 4], uint32_t sQs, uint32_t sDOs,
                         float (&dv)[D / 2], float (&dk)[D / 2]) {
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < QT / 16; ++kk) {
      const uint32_t af[4] = {pf[4 * kk], pf[4 * kk + 1], pf[4 * kk + 2], pf[4 * kk + 3]};
      const uint64_t db = gmma_desc_sw128(sDOs + kk * 2048, QCHUNK, 1024);
      if constexpr (D == 64) wgmma_rs_n64<T, 1>(dv, af, db, 1u);
      else wgmma_rs_n128<T, 1>(dv, af, db, 1u);
    }
#pragma unroll
    for (int kk = 0; kk < QT / 16; ++kk) {
      const uint32_t af[4] = {dsf[4 * kk], dsf[4 * kk + 1], dsf[4 * kk + 2], dsf[4 * kk + 3]};
      const uint64_t db = gmma_desc_sw128(sQs + kk * 2048, QCHUNK, 1024);
      if constexpr (D == 64) wgmma_rs_n64<T, 1>(dk, af, db, 1u);
      else wgmma_rs_n128<T, 1>(dk, af, db, 1u);
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
      if constexpr (D == 64) wgmma_ss_n64<T, 1, 1>(dq, da, db, kk > 0 ? 1u : 0u);
      else wgmma_ss_n128<T, 1, 1>(dq, da, db, kk > 0 ? 1u : 0u);
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
    auto stage_dq = [&](int i) {              // i & 1 == w
      const int n = i >> 1, sb = n % NDQ;
      mbar_wait(BAR(DQ_EMPTY + NDQ * w + sb), ((n / NDQ) & 1) ^ 1);   // the reducer has read the buffer's last tile
      const uint32_t dst = sDQ + (NDQ * w + sb) * Cfg::kDQ + dq_thr;
#pragma unroll
      for (int jb = 0; jb < D / 8; ++jb) {
        const uint32_t o = dst + (jb >> 2) * (QT * 128) + (((2 * (jb & 3)) ^ dq_sx) << 4);
        sts64f(o, dq[4 * jb], dq[4 * jb + 1]);
        sts64f(o + 1024, dq[4 * jb + 2], dq[4 * jb + 3]);
      }
      fence_proxy_async_smem();
      mbar_arrive(BAR(DQ_FULL + NDQ * w + sb));
    };
    // dQ(i) retired: release its dS^T slot, stage the tile
    auto retire_dq = [&](int i) {
      mbar_arrive(BAR(DS_EMPTY + i % NDS));
      stage_dq(i);
    };
    auto issue_owned_dq = [&](int i) {        // i & 1 == w
      mbar_wait(BAR(DS_FULL + i % NDS), (i / NDS) & 1);
      issue_dq(dq, ds_slot(i));
    };

    // The zero accumulators are pinned before the first issue: a register move of dV / dK / dQ that the compiler
    // schedules while a wgmma is in flight makes ptxas serialise every wgmma of the kernel.
    fence_regs(dv);
    fence_regs(dk);
    fence_regs(dq);
    if (NT > 0) {
      mbar_wait(BAR(FULL), 0);
      issue_s_dp(s, dp, sQ, sDO);
      // i runs over the flat (head, query tile) sequence; row0 restarts at i_lo * QT with every head
      for (int i = 0, row0 = i_lo * QT; i < NT; ++i, row0 = (!HEAD_LOOP || row0 + QT < a.nqt * QT) ? row0 + QT : i_lo * QT) {
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
        if (i > 0) mbar_arrive(BAR(EMPTY + (i - 1) % NST));   // Q, dO and the stats of tile i - 1 are no longer read
        const bool own = (i & 1) == w;
        if (own && i >= NDS) mbar_wait(BAR(DS_EMPTY + i % NDS), ((i - NDS) / NDS) & 1);
        elementwise_tile(s, dp, pf, dsf, row0, sStats + st * 8 * QT, ds_slot(i) + w * Cfg::kDS);
        // the slot arithmetic below is redone from an opaque copy of i rather than kept live through the elementwise
        // stage (the BIAS kernels have no register to spare there)
        int io = i;
        asm volatile("" : "+r"(io));
        if ((io & 1) != w) mbar_arrive(BAR(DS_FULL + io % NDS));
        issue_dv_dk(pf, dsf, sQs, sDOs, dv, dk);
        if (io >= 1 && (io & 1) != w) issue_owned_dq(io - 1);
        wgmma_commit();
        if (i + 1 < NT) {
          const int sn = (i + 1) % NST;
          mbar_wait(BAR(FULL + sn), ((i + 1) / NST) & 1);
          issue_s_dp(s, dp, sQ + sn * Cfg::kQ, sDO + sn * Cfg::kQ);
        }
      }
      // drain: dQ(NT - 2) is in flight if this warpgroup owns it, dQ(NT - 1) is not issued yet
      wgmma_wait<0>();
      fence_regs(dv);
      fence_regs(dk);
      fence_regs(dq);
      if (NT >= 2 && ((NT - 2) & 1) == w) retire_dq(NT - 2);
      mbar_arrive(BAR(EMPTY + (NT - 1) % NST));
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
      const int st = i % NST;
      const int hh = HEAD_LOOP ? i / NI : 0;    // head h0 + hh, query tile i_lo + i % NI
      const int row0 = (i_lo + i - hh * NI) * QT;
      const uint32_t sQs = sQ + st * Cfg::kQ, sDOs = sDO + st * Cfg::kQ;
      mbar_wait(BAR(FULL + st), (i / NST) & 1);
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
      float dq[D / 2];
      issue_dq(dq, dsbuf);
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs(dv);
      fence_regs(dk);
      fence_regs(dq);
      mbar_arrive(BAR(EMPTY + st));             // Q, dO and the stats of this stage are no longer read

      // ---- dQ partial tile -> fp32 accumulator (rows = queries, columns = features) ----
      float* acc = a.dq_acc + (((long long)b * a.H + h0 + hh) * a.nqt * QT + row0) * D + cq;
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) {
        const int q = 16 * wl + r8 + 8 * hf;
        if (row0 + q < a.Nq) {
#pragma unroll
          for (int jb = 0; jb < D / 8; ++jb)
            red_add_f32x2(acc + (long long)q * D + 8 * jb, dq[4 * jb + 2 * hf], dq[4 * jb + 2 * hf + 1]);
        }
      }
    }
  }

  // ---- epilogue: dV and dK * scale of the warpgroup's 64 keys ---------------------------------
  // (no early exit for keys at or beyond Nk: the l2norm backward below shuffles within the quad of a key row)
  const bool to_acc = a.split > 1;
#pragma unroll
  for (int hf = 0; hf < 2; ++hf) {
    const int key = key_g[hf];
    const bool in = key < a.Nk;
    if (to_acc) {
      // the group's heads are split over several CTAs: sum over them in fp32 (reference: cu:1613-1619)
      float* pv = a.dv_acc + (((long long)b * a.kv_heads + hk) * a.Nk + key) * D + cq;
      float* pk = a.dk_acc + (((long long)b * a.kv_heads + hk) * a.Nk + key) * D + cq;
      if (in) {
#pragma unroll
        for (int jb = 0; jb < D / 8; ++jb) {
          red_add_f32x2(pv + 8 * jb, dv[4 * jb + 2 * hf], dv[4 * jb + 2 * hf + 1]);
          red_add_f32x2(pk + 8 * jb, dk[4 * jb + 2 * hf] * a.scale, dk[4 * jb + 2 * hf + 1] * a.scale);
        }
      }
    } else if (a.out_f32) {
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
      T* pv = reinterpret_cast<T*>(a.dv) + b * a.dv_sb + hk * a.dv_sh + (long long)key * a.dv_sn + cq;
      T* pk = reinterpret_cast<T*>(a.dk) + b * a.dk_sb + hk * a.dk_sh + (long long)key * a.dk_sn + cq;
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
      if (a.k_rnorm != nullptr) l2norm_bwd_key_row<T, D>(g, a, sK + (64 * w + kr + 8 * hf) * 128, b, hk, key, in);
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

// (dq_hat - q_hat <q_hat, dq_hat>_group) * rnorm_group on the 8 features one thread owns; the
// `tpr` threads of a row are consecutive lanes, groups are aligned sub-blocks of them.
template <typename T>
__device__ __forceinline__ void finish_l2norm_bwd(float (&g)[8], const DqFinishArgs& a, bool ok, uint4 raw, int b,
                                                  int h, int row, int c8) {
  if (a.q_rnorm == nullptr) return;            // uniform across the grid
  float y[8];
  {
    const float2 u0 = unpack2<T>(raw.x), u1 = unpack2<T>(raw.y), u2 = unpack2<T>(raw.z), u3 = unpack2<T>(raw.w);
    y[0] = u0.x; y[1] = u0.y; y[2] = u1.x; y[3] = u1.y; y[4] = u2.x; y[5] = u2.y; y[6] = u3.x; y[7] = u3.y;
  }
  const int gs = a.D / a.G;
  const long long rbase = (((long long)b * a.H + h) * a.Nq + row) * a.G;
  if (gs >= 8) {
    float dot = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) dot += y[i] * g[i];
    const int tpg = gs >> 3;
    for (int m = 1; m < tpg; m <<= 1) dot += __shfl_xor_sync(0xFFFFFFFFu, dot, m);
    const float rn = ok ? a.q_rnorm[rbase + c8 / tpg] : 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) g[i] = (g[i] - y[i] * dot) * rn;
  } else {
    float pr[8], dot[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) pr[i] = y[i] * g[i];
    subgroup_sums8(pr, gs, dot);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float rn = ok ? a.q_rnorm[rbase + (c8 * 8 + i) / gs] : 0.f;
      g[i] = (g[i] - y[i] * dot[i]) * rn;
    }
  }
}

// dq conversion (reference: the fp32 -> scalar_t cast of dq after its atomics, cu:1904): TPR = D / 8 consecutive lanes
// per query row, 8 features each.  The accumulator is read from L2 (the reductions of the main kernel have just
// produced it there), converted, and written back as zeros: it is zero between launches.
template <typename T, int D>
__global__ void __launch_bounds__(256) bwd_dq_finish_kernel(const DqFinishArgs a) {
  pdl_launch_dependents();
  pdl_wait();
  constexpr int TPR = D / 8;
  const long long t = (long long)blockIdx.x * 256 + threadIdx.x;
  const long long rowid = t / TPR;                         // over (batch*heads) x Nq
  const int c8 = (int)(t % TPR);
  const bool ok = rowid < (long long)a.B * a.H * a.Nq;     // whole rows of TPR lanes (shuffles stay in them)
  const long long bh = ok ? rowid / a.Nq : 0;
  const int row = ok ? (int)(rowid - bh * a.Nq) : 0;
  const int b = (int)(bh / a.H), h = (int)(bh % a.H);
  float* src = a.dq_acc + (bh * a.padded + row) * D + c8 * 8;
  float4 lo = make_float4(0.f, 0.f, 0.f, 0.f), hi = lo;
  if (ok) {
    lo = ldg_cg128f(src);
    hi = ldg_cg128f(src + 4);
    *reinterpret_cast<float4*>(src) = make_float4(0.f, 0.f, 0.f, 0.f);
    *reinterpret_cast<float4*>(src + 4) = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  float g[8] = {lo.x * a.scale, lo.y * a.scale, lo.z * a.scale, lo.w * a.scale,
                hi.x * a.scale, hi.y * a.scale, hi.z * a.scale, hi.w * a.scale};
  uint4 qraw = make_uint4(0, 0, 0, 0);
  if (ok && a.q_rnorm != nullptr)
    qraw = ldg_stream128(reinterpret_cast<const T*>(a.q_hat) + b * a.q_sb + h * a.q_sh + (long long)row * a.q_sn +
                         c8 * 8);
  finish_l2norm_bwd<T>(g, a, ok, qraw, b, h, row, c8);
  if (!ok) return;
  if (a.out_f32) {
    float* dst = reinterpret_cast<float*>(a.dq) + b * a.sb + h * a.sh + (long long)row * a.sn + c8 * 8;
    *reinterpret_cast<float4*>(dst) = make_float4(g[0], g[1], g[2], g[3]);
    *reinterpret_cast<float4*>(dst + 4) = make_float4(g[4], g[5], g[6], g[7]);
  } else {
    uint4 o4;
    o4.x = pack2<T>(g[0], g[1]);
    o4.y = pack2<T>(g[2], g[3]);
    o4.z = pack2<T>(g[4], g[5]);
    o4.w = pack2<T>(g[6], g[7]);
    T* dst = reinterpret_cast<T*>(a.dq) + b * a.sb + h * a.sh + (long long)row * a.sn + c8 * 8;
    *reinterpret_cast<uint4*>(dst) = o4;
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

// ------------------------------------------------------------------------------------------
// host runner
// ------------------------------------------------------------------------------------------
struct BwdHostArgs {
  bool dtype_bf16;
  int B, H, kv_heads, Nq, Nk, D, causal;
  float scale, shift;
  const uint8_t* mask; long long mask_sb;
  fcsa_tensor q, k, v, o, d_o, dq, dk, dv;
  const float* inv_l;
  bool out_f32 = false;             // o (read), dq, dk, dv (written) are float32
  void* workspace;                  // scratch
  void* zeroed;                     // zero on entry, zero again on exit (dq accumulator)
  cudaEvent_t ev_start = nullptr, ev_stop = nullptr;   // optional: recorded around the main kernel
  cudaEvent_t ev_prep[2] = {nullptr, nullptr}, ev_finish[2] = {nullptr, nullptr};   // ... the preprocess / dq finish
  // fused l2norm backward (q, k above are then the NORMALISED tensors and dq, dk the gradients
  // w.r.t. the raw ones); both null = plain backward
  const float* q_rnorm = nullptr;
  const float* k_rnorm = nullptr;
  int groups = 1;
  // additive bias (nullptr = none) and its fp32 gradient accumulator (nullptr = not needed)
  const void* bias = nullptr; long long bias_sb = 0, bias_sh = 0, bias_sn = 0;
  const float* bias_amax = nullptr;           // optional device scalar added (if positive) to the shift
  float* dbias = nullptr; long long dbias_sb = 0, dbias_sh = 0;
};

// Slices per key/value-head group (query heads per CTA = G / split).  One CTA per group keeps dk / dv in registers
// (no accumulator, no finish pass, bitwise reproducible), but the grid then has B * kv_heads * key tiles CTAs; below
// one CTA per SM the group is split into the fewest slices that fill the device.  Keys/values shared by all heads
// (kv_heads == 1) and the BIAS kernels (no registers to spare for the head loop) take one query head per CTA.
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

template <typename T, int D, bool BIAS = false>
int run_backward_t(const BwdHostArgs& h, cudaStream_t stream, int* launches, const char** err,
                   cudaError_t* ce) {
  using Cfg = BwdCfg<D>;
  const BwdWorkspace w = bwd_workspace_layout(h.B, h.H, h.kv_heads, h.Nq, h.Nk, D);
  uint8_t* ws = reinterpret_cast<uint8_t*>(h.workspace);
  uint8_t* zs = reinterpret_cast<uint8_t*>(h.zeroed);
  float* stats = reinterpret_cast<float*>(ws + w.stats_off);
  float* dq_acc = reinterpret_cast<float*>(zs + w.dq_off);
  float* dkv_acc = reinterpret_cast<float*>(ws + w.dkv_off);
  const float log2e = 1.4426950408889634f;
  cudaError_t e;
  int split = 1;
  if (h.kv_heads < h.H) {
    int sms = 0;
    e = device_sm_count(&sms);
    if (e != cudaSuccess) { *err = "cudaDeviceGetAttribute(multiProcessorCount)"; *ce = e; return FCSA_ERR_CUDA; }
    split = bwd_group_split(h.B, h.H, h.kv_heads, h.Nk, BIAS, sms);
  }
  const bool to_acc = split > 1;
  const size_t dkv_elems = (size_t)h.B * h.kv_heads * h.Nk * D;

  // dk/dv accumulators of split groups are per call (the dq accumulator is self-cleaning)
  if (to_acc) {
    e = cudaMemsetAsync(dkv_acc, 0, 2 * dkv_elems * 4, stream);
    if (e != cudaSuccess) { *err = "cudaMemsetAsync(workspace)"; *ce = e; return FCSA_ERR_CUDA; }
  }

  // 1. preprocess
  {
    PrepArgs pa;
    pa.B = h.B; pa.H = h.H; pa.Nq = h.Nq; pa.Nk = h.Nk; pa.D = D; pa.nqt = w.nqt; pa.QT = Cfg::QT; pa.causal = h.causal;
    pa.c2 = h.shift * log2e;
    pa.shift_extra = h.bias_amax;
    pa.o_f32 = h.out_f32 ? 1 : 0;
    pa.o = h.o.ptr; pa.o_sb = h.o.sb; pa.o_sh = h.o.sh; pa.o_sn = h.o.sn;
    pa.d_o = h.d_o.ptr; pa.do_sb = h.d_o.sb; pa.do_sh = h.d_o.sh; pa.do_sn = h.d_o.sn;
    pa.inv_l = h.inv_l; pa.stats = stats;
    const int rows_per_block = 2 * (256 / (D / 8));
    const int padded = w.nqt * Cfg::QT;
    pa.bpb = (padded + rows_per_block - 1) / rows_per_block;
    const long long grid = (long long)pa.bpb * h.B * h.H;
    if (grid > 0x7FFFFFFFLL) { *err = "problem too large for one launch"; return FCSA_ERR_INVALID; }
    if (h.ev_prep[0]) cudaEventRecord(h.ev_prep[0], stream);
    e = launch_pdl(bwd_prep_kernel<T, D / 8>, dim3((unsigned)grid), dim3(256), 0, stream, pa);
    if (h.ev_prep[1]) cudaEventRecord(h.ev_prep[1], stream);
    if (e != cudaSuccess) { *err = "backward preprocess launch"; *ce = e; return FCSA_ERR_CUDA; }
    ++*launches;
  }
  // 2. main
  {
    CUtensorMap tq, tk, tv, tdo, tdq;
    const CUtensorMapDataType dt = tma_dtype16(h.dtype_bf16);
    if (make_tensor_map_bhnd(&tq, h.q.ptr, dt, h.B, h.H, h.Nq, D, h.q.sb, h.q.sh, h.q.sn, Cfg::QT) ||
        make_tensor_map_bhnd(&tk, h.k.ptr, dt, h.B, h.kv_heads, h.Nk, D, h.k.sb, h.k.sh, h.k.sn, 128) ||
        make_tensor_map_bhnd(&tv, h.v.ptr, dt, h.B, h.kv_heads, h.Nk, D, h.v.sb, h.v.sh, h.v.sn, 128) ||
        make_tensor_map_bhnd(&tdo, h.d_o.ptr, dt, h.B, h.H, h.Nq, D, h.d_o.sb, h.d_o.sh, h.d_o.sn, Cfg::QT)) {
      *err = "cuTensorMapEncodeTiled failed (backward): q, k, v, d_o must be views a TMA tensor map can express "
             "(positive strides, 16-byte aligned)";
      return FCSA_ERR_INVALID;
    }
    // the dq accumulator as [B][H][Nq][D] fp32 over its padded rows: boxes of 32 features x QT rows
    memset(&tdq, 0, sizeof(tdq));
    const long long acc_sh = (long long)w.nqt * Cfg::QT * D;
    if (Cfg::kStaged &&
        make_tensor_map_bhnd(&tdq, dq_acc, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, h.B, h.H, h.Nq, D, h.H * acc_sh, acc_sh, D,
                             Cfg::QT, 32)) {
      *err = "cuTensorMapEncodeTiled failed (backward dq accumulator)";
      return FCSA_ERR_CUDA;
    }
    BwdArgs a;
    a.B = h.B; a.H = h.H; a.Nq = h.Nq; a.Nk = h.Nk; a.kv_heads = h.kv_heads; a.causal = h.causal;
    a.has_mask = h.mask ? 1 : 0; a.nqt = w.nqt;
    a.split = split; a.hpc = h.H / h.kv_heads / split;
    a.c1 = h.scale * log2e; a.scale = h.scale;
    a.mask = h.mask; a.mask_sb = h.mask_sb;
    a.stats = stats; a.dq_acc = dq_acc;
    a.dk_acc = dkv_acc; a.dv_acc = dkv_acc + dkv_elems;
    a.dk = h.dk.ptr; a.dk_sb = h.dk.sb; a.dk_sh = h.dk.sh; a.dk_sn = h.dk.sn;
    a.dv = h.dv.ptr; a.dv_sb = h.dv.sb; a.dv_sh = h.dv.sh; a.dv_sn = h.dv.sn;
    a.bias = h.bias; a.bias_sb = h.bias_sb; a.bias_sh = h.bias_sh; a.bias_sn = h.bias_sn;
    a.dbias = h.dbias; a.dbias_sb = h.dbias_sb; a.dbias_sh = h.dbias_sh;
    a.out_f32 = h.out_f32 ? 1 : 0;
    a.k_rnorm = h.k_rnorm; a.groups = h.groups;
    constexpr bool kLoop = !BIAS;
    auto kern = a.hpc > 1 ? fcsa_bwd_kernel<T, D, BIAS, kLoop> : fcsa_bwd_kernel<T, D, BIAS>;
    e = a.hpc > 1 ? ensure_dynamic_smem<fcsa_bwd_kernel<T, D, BIAS, kLoop>>(Cfg::kSmem)
                  : ensure_dynamic_smem<fcsa_bwd_kernel<T, D, BIAS>>(Cfg::kSmem);
    if (e != cudaSuccess) { *err = "cudaFuncSetAttribute(bwd)"; *ce = e; return FCSA_ERR_CUDA; }
    // one CTA per (key tile, batch, kv head, slice of its group)
    const long long items = (long long)((h.Nk + 127) / 128) * h.B * h.kv_heads * split;
    if (items > 0x7FFFFFFFLL) { *err = "problem too large for one launch"; return FCSA_ERR_INVALID; }
    if (h.ev_start) cudaEventRecord(h.ev_start, stream);
    e = launch_pdl(kern, dim3((unsigned)items), dim3(Cfg::kThreads), Cfg::kSmem, stream, tq, tk, tv, tdo, tdq, a);
    if (h.ev_stop) cudaEventRecord(h.ev_stop, stream);
    if (e != cudaSuccess) { *err = "backward kernel launch"; *ce = e; return FCSA_ERR_CUDA; }
    ++*launches;
  }
  // 3. finish
  {
    DqFinishArgs fa;
    fa.B = h.B; fa.H = h.H; fa.Nq = h.Nq; fa.D = D; fa.nqt = w.nqt; fa.padded = w.nqt * Cfg::QT; fa.scale = h.scale;
    fa.dq_acc = dq_acc; fa.dq = h.dq.ptr; fa.sb = h.dq.sb; fa.sh = h.dq.sh; fa.sn = h.dq.sn;
    fa.q_hat = h.q.ptr; fa.q_sb = h.q.sb; fa.q_sh = h.q.sh; fa.q_sn = h.q.sn;
    fa.q_rnorm = h.q_rnorm; fa.G = h.groups; fa.out_f32 = h.out_f32 ? 1 : 0;
    const long long threads = (long long)h.B * h.H * h.Nq * (D / 8);
    const long long blocks = (threads + 255) / 256;
    if (blocks > 0x7FFFFFFFLL) { *err = "problem too large for one launch"; return FCSA_ERR_INVALID; }
    if (h.ev_finish[0]) cudaEventRecord(h.ev_finish[0], stream);
    e = launch_pdl(bwd_dq_finish_kernel<T, D>, dim3((unsigned)blocks), dim3(256), 0, stream, fa);
    if (h.ev_finish[1]) cudaEventRecord(h.ev_finish[1], stream);
    if (e != cudaSuccess) { *err = "dq finish launch"; *ce = e; return FCSA_ERR_CUDA; }
    ++*launches;
    if (to_acc) {
      for (int which = 0; which < 2; ++which) {
        KvFinishArgs ka;
        ka.B = h.B; ka.Hk = h.kv_heads; ka.Nk = h.Nk; ka.D = D; ka.out_f32 = h.out_f32 ? 1 : 0;
        ka.acc = dkv_acc + (which ? dkv_elems : 0);
        const fcsa_tensor& t = which ? h.dv : h.dk;
        ka.out = t.ptr; ka.sb = t.sb; ka.sh = t.sh; ka.sn = t.sn;
        const long long tot = (long long)dkv_elems / 8;
        bwd_kv_finish_kernel<T><<<(unsigned)((tot + 255) / 256), 256, 0, stream>>>(ka);
        e = cudaGetLastError();
        if (e != cudaSuccess) { *err = "dk/dv finish launch"; *ce = e; return FCSA_ERR_CUDA; }
        ++*launches;
      }
    }
    if (h.k_rnorm != nullptr && to_acc) {
      // l2norm backward of dk (gradient w.r.t. the raw keys) as its own pass over the head-summed dk; otherwise
      // the main kernel's epilogue applies it
      L2Args la;
      la.B = h.B; la.H = h.kv_heads; la.N = h.Nk; la.D = D; la.G = h.groups;
      la.x_sb = h.dk.sb; la.x_sh = h.dk.sh; la.x_sn = h.dk.sn;
      la.y_sb = h.k.sb; la.y_sh = h.k.sh; la.y_sn = h.k.sn;
      la.o_sb = h.dk.sb; la.o_sh = h.dk.sh; la.o_sn = h.dk.sn;
      la.x = h.dk.ptr; la.y = h.k.ptr; la.dx = h.dk.ptr; la.rnorm = const_cast<float*>(h.k_rnorm);
      const int rows_per_block = 256 / (D / 8);
      const long long rows = (long long)la.B * la.H * la.N;
      l2norm_bwd_kernel<T><<<(unsigned)((rows + rows_per_block - 1) / rows_per_block), 256, 0, stream>>>(la);
      e = cudaGetLastError();
      if (e != cudaSuccess) { *err = "l2norm backward (dk) launch"; *ce = e; return FCSA_ERR_CUDA; }
      ++*launches;
    }
  }
  return FCSA_OK;
}

inline int run_backward(const BwdHostArgs& h, cudaStream_t stream, int* launches, const char** err,
                        cudaError_t* ce) {
  if (h.bias != nullptr) {
    if (h.D == 64) {
      if (h.dtype_bf16) return run_backward_t<__nv_bfloat16, 64, true>(h, stream, launches, err, ce);
      return run_backward_t<__half, 64, true>(h, stream, launches, err, ce);
    }
    if (h.dtype_bf16) return run_backward_t<__nv_bfloat16, 128, true>(h, stream, launches, err, ce);
    return run_backward_t<__half, 128, true>(h, stream, launches, err, ce);
  }
  if (h.D == 64) {
    if (h.dtype_bf16) return run_backward_t<__nv_bfloat16, 64>(h, stream, launches, err, ce);
    return run_backward_t<__half, 64>(h, stream, launches, err, ce);
  }
  if (h.dtype_bf16) return run_backward_t<__nv_bfloat16, 128>(h, stream, launches, err, ce);
  return run_backward_t<__half, 128>(h, stream, launches, err, ce);
}

}  // namespace fcsa
