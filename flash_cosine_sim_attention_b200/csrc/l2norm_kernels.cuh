// Grouped l2-normalisation of q / k rows and its backward, and the float32 front end.
//
// Replaces the PyTorch ops the reference runs outside its kernels
// (flash_cosine_sim_attention.py:38-65: F.normalize per `groups` chunk of the head dim, cast
// back to the input dtype; backward left to autograd).  One pass each way, HBM-bound:
// 16-byte vector loads, fp32 reduction with warp shuffles.
//
// float32 callers (reference: Float is dispatched in forward and backward, cu:1702-1703 / 1832-1834) run on the
// 16-bit tensor-core kernels; the same two row kernels are the only extra work around them:
//   row_fwd_kernel : y(16 bit) = round( x / max(||x||_group, 1e-12) * mul )   G > 0: l2norm over G groups
//                                round( x * mul )                              G = 0: plain scaled cast
//   row_bwd_kernel : dx = (dy - y <y, dy>_group) * rnorm_group * mul           G > 0   (dy: gradient w.r.t. y;
//                         dy * mul                                             G = 0    y: 16 bit)
// x / dy / dx are 16-bit or float32.  `mul` is an optional DEVICE scalar (the power-of-two range scale of v / dO,
// chosen on the device - no host synchronisation) taken by the float32 passes; rnorm (fp32, per group) is kept for
// the backward.
#pragma once

#include "../../include/fcsa_b200.h"
#include "sm90_primitives.cuh"
#include "tensor_map.h"

namespace fcsa {

// One (B, H, N, D) tensor of a row pass; views with element strides and contiguous features.
struct RowTensor {
  int H, N;                       // heads (0: no tensor), rows
  fcsa_tensor x;                  // forward: input; backward: dy (16-bit or float32)
  fcsa_tensor y;                  // the 16-bit normalised tensor: output of forward, input of backward
  fcsa_tensor dx;                 // backward only: output, the type of dy (may be dy itself: in-place passes)
  float* rnorm;                   // (B, H, N, G) fp32; forward: nullptr = not kept
  // read by the append pass only (row_fwd_kernel<..., APPEND = true>, the key/value-cache decode):
  const int32_t* row0;            // device (B,): row n of x goes to row row0[b] + n of y; nullptr = row n
  int rows_y;                     // rows of y: a destination row outside [0, rows_y) is not written
  // (raw and ring share the four bytes raw once had alone: every row pass keeps its parameter block)
  uint8_t raw;                    // 1: y = x, no l2norm whatever G (the values)
  uint8_t ring;                   // 1: y is a rolling cache of rows_y rows, row r goes to row r mod rows_y
  // packed sequences (with row0): x is one batch of N packed rows, sequence s owns rows [cu[s], cu[s + 1]) (clamped as
  // seq_span does, at most max_n rows) and its row n goes to row row0[s] + n - cu[s] of y's batch s; rows outside
  // every sequence are not written.  nullptr = row n of batch b goes to row row0[b] + n of y's batch b.
  const int32_t* cu;
  int n_seq, max_n;               // sequences (cu has n_seq + 1 entries), the longest
};

struct RowArgs {
  int B, D, G;                    // G = 0: plain scaled cast (float32 passes)
  const float* mul;               // device scalar or nullptr (= 1); read by the float32 passes only
  int mul_reciprocal;             // 1: use 1 / *mul
  RowTensor t[3];                 // forward: one to three tensors (t[i].H = 0 ends the list); backward: t[0]
};

// The sequence s of packed row n (cu[s] <= n < cu[s + 1], with seq_span's clamp to max_n rows and [0, total)) and
// its first row, or s = -1 for a row outside every sequence: a binary search over the n_seq + 1 entries.
__device__ __forceinline__ int row_sequence(const int32_t* cu, int n_seq, int max_n, int total, int n, int* start) {
  int lo = 0, hi = n_seq;                             // the last s in [0, n_seq] with cu[s] <= n
  if (ld_cu(cu) > n) return -1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (ld_cu(cu + mid) <= n) lo = mid;
    else hi = mid - 1;
  }
  if (lo == n_seq) return -1;
  const SeqSpan sp = seq_span(cu, lo, max_n, total);
  if (n < sp.start || n - sp.start >= sp.len) return -1;
  *start = sp.start;
  return lo;
}

// 1 / max(sqrt(ss), 1e-12)  (py:38-55: F.normalize's eps) = min(rsqrt(ss), 1e12): one MUFU.RSQ instead of an
// IEEE sqrt + divide (~60 instructions per row and thread in a pass that must stay HBM-bound); the
// approximation error (2^-22) vanishes under the 16-bit rounding of the normalised output
__device__ __forceinline__ float rnorm_of(float ss) {
  float r;
  asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(ss));
  return fminf(r, 1e12f);
}

// sum over the `tpg` consecutive lanes that share a group (tpg is a power of two <= 16)
__device__ __forceinline__ float group_reduce(float v, int tpg) {
  for (int m = 1; m < tpg; m <<= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, m);
  return v;
}

// Groups narrower than 8 features (group size gs = 1, 2 or 4): for every feature, the sum of v over the aligned
// gs-wide block it belongs to.  Written with compile-time register indices only - a `for (i < gs)` loop over the
// arrays would push them to local memory.
__device__ __forceinline__ void subgroup_sums8(const float (&v)[8], int gs, float (&out)[8]) {
  float p2[8], p4[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) p2[i] = v[i] + v[i ^ 1];
#pragma unroll
  for (int i = 0; i < 8; ++i) p4[i] = p2[i] + p2[i ^ 2];
#pragma unroll
  for (int i = 0; i < 8; ++i) out[i] = gs == 1 ? v[i] : (gs == 2 ? p2[i] : p4[i]);
}

// The group arithmetic of the F features (8 or 16) one thread owns.  The threads of a row are consecutive lanes,
// tr is this thread's index in its row, gs the power-of-two group size; every lane of a row must take part (the
// shuffles).  rnorm_row points at the row's G rnorm values, or is nullptr (forward: not kept; backward: a row past
// the end, whose result is not stored).  A group of gs >= F features spans gs / F lanes; a 16-feature thread with
// smaller groups works on each 8-feature half as a thread of its own.
//
// Forward: rn[i] = 1 / ||group of feature i||; the thread holding a group's first feature stores it.
template <int F>
__device__ __forceinline__ void l2norm_fwd_group(const float (&f)[F], int gs, int tr, float* rnorm_row,
                                                 float (&rn)[F]) {
  if (gs >= F) {
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < F; ++i) ss += f[i] * f[i];
    const int tpg = gs / F;                           // threads per group
    const float r = rnorm_of(group_reduce(ss, tpg));
#pragma unroll
    for (int i = 0; i < F; ++i) rn[i] = r;
    if (rnorm_row && (tr & (tpg - 1)) == 0) rnorm_row[tr / tpg] = r;
  } else if constexpr (F == 16) {
#pragma unroll
    for (int s = 0; s < 2; ++s) {
      float h[8], r8[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) h[i] = f[8 * s + i];
      l2norm_fwd_group<8>(h, gs, 2 * tr + s, rnorm_row, r8);
#pragma unroll
      for (int i = 0; i < 8; ++i) rn[8 * s + i] = r8[i];
    }
  } else {
    float sq[8], ss[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) sq[i] = f[i] * f[i];
    subgroup_sums8(sq, gs, ss);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      rn[i] = rnorm_of(ss[i]);
      if (rnorm_row && (i & (gs - 1)) == 0) rnorm_row[(tr * 8 + i) / gs] = rn[i];
    }
  }
}

// Backward, in place on g (dy in, dx out): g = (g - y <y, g>_group) * rnorm_group * mul.
template <int F>
__device__ __forceinline__ void l2norm_bwd_group(float (&g)[F], const float (&y)[F], int gs, int tr,
                                                 const float* rnorm_row, float mul) {
  if (gs >= F) {
    float dot = 0.f;
#pragma unroll
    for (int i = 0; i < F; ++i) dot += y[i] * g[i];
    const int tpg = gs / F;
    dot = group_reduce(dot, tpg);
    const float r = (rnorm_row ? rnorm_row[tr / tpg] : 0.f) * mul;
#pragma unroll
    for (int i = 0; i < F; ++i) g[i] = (g[i] - y[i] * dot) * r;
  } else if constexpr (F == 16) {
#pragma unroll
    for (int s = 0; s < 2; ++s) {
      float h[8], y8[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) { h[i] = g[8 * s + i]; y8[i] = y[8 * s + i]; }
      l2norm_bwd_group<8>(h, y8, gs, 2 * tr + s, rnorm_row, mul);
#pragma unroll
      for (int i = 0; i < 8; ++i) g[8 * s + i] = h[i];
    }
  } else {
    float pr[8], dot[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) pr[i] = y[i] * g[i];
    subgroup_sums8(pr, gs, dot);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float r = (rnorm_row ? rnorm_row[(tr * 8 + i) / gs] : 0.f) * mul;
      g[i] = (g[i] - y[i] * dot[i]) * r;
    }
  }
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

// One 16-byte vector of X (16-bit: 8 elements, float: 4) to and from fp32.
template <typename X>
__device__ __forceinline__ void unpack16B(uint4 r, float* f) {
  if constexpr (std::is_same<X, float>::value) {
    f[0] = __uint_as_float(r.x); f[1] = __uint_as_float(r.y); f[2] = __uint_as_float(r.z); f[3] = __uint_as_float(r.w);
  } else {
    const float2 t0 = unpack2<X>(r.x), t1 = unpack2<X>(r.y), t2 = unpack2<X>(r.z), t3 = unpack2<X>(r.w);
    f[0] = t0.x; f[1] = t0.y; f[2] = t1.x; f[3] = t1.y; f[4] = t2.x; f[5] = t2.y; f[6] = t3.x; f[7] = t3.y;
  }
}
template <typename X>
__device__ __forceinline__ uint4 pack16B(const float* f) {
  if constexpr (std::is_same<X, float>::value)
    return make_uint4(__float_as_uint(f[0]), __float_as_uint(f[1]), __float_as_uint(f[2]), __float_as_uint(f[3]));
  else
    return make_uint4(pack2<X>(f[0], f[1]), pack2<X>(f[2], f[3]), pack2<X>(f[4], f[5]), pack2<X>(f[6], f[7]));
}

// the scale of the float32 passes (1 without `mul`); the 16-bit passes take none
template <typename X>
__device__ __forceinline__ float row_mul(const RowArgs& a) {
  if (!std::is_same<X, float>::value || a.mul == nullptr) return 1.f;
  const float m = __ldg(a.mul);
  return a.mul_reciprocal ? 1.f / m : m;
}

// Forward: T is the 16-bit type of y, X the type of x (T or float).  grid = (row blocks, tensor): blockIdx.y
// selects t[0] or t[1], and the blocks run over that tensor's (batch, head, row) rows as one flat sequence, so a
// short sequence does not leave most of a block idle and any number of (batch, head) pairs fits.  Row indices are
// 32-bit: 2^31 rows of at least 64 bytes do not fit in device memory.  One thread owns 16 features of U rows and
// issues its loads of all U rows before the first reduction; TPR = threads per row (D / 16) when known at compile
// time (4 or 8), 0 = read it from the arguments.  x is read with coherent loads: it may alias y.  The 16-bit passes
// keep four blocks per SM (at most 64 registers).  APPEND (16-bit only): grid.y runs over up to three tensors, each
// row lands at the per-batch offset row0[b] (rows falling outside y are skipped) and `raw` tensors are copied; with
// packed sequences (RowTensor::cu) at the offset of the row's sequence; in a rolling cache (`ring`) at that row modulo
// rows_y.
template <typename T, typename X, int TPR, int U, bool APPEND = false>
__global__ void __launch_bounds__(256, 8 / sizeof(X)) row_fwd_kernel(const RowArgs a) {
  // SIXTEEN features per thread: the pass is issue-bound before it is memory-bound (ncu: 84 % issue-slot
  // utilisation with 8 features per thread), so the per-row bookkeeping (addresses, shuffle steps, predicates) is
  // spread over twice the bytes.
  pdl_launch_dependents();
  pdl_wait();
  constexpr int E = 16 / sizeof(X);                   // elements of x per 16-byte vector
  const RowTensor& t = a.t[blockIdx.y];
  const int tpr = TPR ? TPR : (a.D >> 4);
  const int rpp = 256 / tpr;                          // rows per pass
  const int tr = threadIdx.x % tpr;
  const int rows = a.B * t.H * t.N;
  if (blockIdx.x * (U * rpp) >= rows) return;         // the grid is sized for the longer of the two tensors
  const int row0 = blockIdx.x * (U * rpp) + threadIdx.x / tpr;
  const int gs = (a.G && !(APPEND && t.raw)) ? a.D / a.G : 0;
  const float mul = row_mul<X>(a);
  uint4 raw[U][16 / E];
  long long yoff[U];
#pragma unroll
  for (int u = 0; u < U; ++u) {
    const int row = row0 + u * rpp;
    const int bh = row / t.N, n = row - bh * t.N, b = bh / t.H, h = bh - b * t.H;
    const X* xp = static_cast<const X*>(t.x.ptr) + b * t.x.sb + h * t.x.sh + (long long)n * t.x.sn + tr * 16;
    if constexpr (!APPEND) yoff[u] = b * t.y.sb + h * t.y.sh + (long long)n * t.y.sn + tr * 16;
#pragma unroll
    for (int v = 0; v < 16 / E; ++v) raw[u][v] = row < rows ? ld_stream128(xp + v * E) : make_uint4(0, 0, 0, 0);
  }
  if constexpr (APPEND) {
    // the destinations, while the loads are in flight (the sequence search of packed rows is a loop of its own)
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int row = row0 + u * rpp;
      const int bh = row / t.N, n = row - bh * t.N, b = bh / t.H, h = bh - b * t.H;
      long long ny = n;
      int yb = b;
      if (t.row0 != nullptr && row < rows) {
        if (t.cu != nullptr) {
          int start = 0;
          yb = row_sequence(t.cu, t.n_seq, t.max_n, t.N, n, &start);
          ny = yb < 0 ? -1 : (long long)t.row0[yb] + n - start;
        } else {
          ny += t.row0[b];
        }
        if (t.ring && ny >= 0) ny %= t.rows_y;
      }
      yoff[u] = (ny >= 0 && ny < t.rows_y) ? yb * t.y.sb + h * t.y.sh + ny * t.y.sn + tr * 16 : -1;
    }
  }
#pragma unroll
  for (int u = 0; u < U; ++u) {
    const int row = row0 + u * rpp;
    const bool ok = row < rows;
    float f[16], rn[16];
#pragma unroll
    for (int v = 0; v < 16 / E; ++v) unpack16B<X>(raw[u][v], f + v * E);
    if (gs == 0) {
#pragma unroll
      for (int i = 0; i < 16; ++i) rn[i] = 1.f;
    } else {
      l2norm_fwd_group<16>(f, gs, tr, ok && t.rnorm ? t.rnorm + (long long)row * a.G : nullptr, rn);
    }
#pragma unroll
    for (int i = 0; i < 16; ++i) f[i] *= rn[i] * mul;
    if (ok && (!APPEND || yoff[u] >= 0)) {
#pragma unroll
      for (int s = 0; s < 2; ++s)
        *reinterpret_cast<uint4*>(static_cast<T*>(t.y.ptr) + yoff[u] + 8 * s) = pack16B<T>(f + 8 * s);
    }
  }
}

// Backward over a.t[0]: T is the 16-bit type of y, X the type of dy and dx (T or float).  One thread owns 8
// features of one row, rows are flat over (batch, head, row).  dy is read with coherent loads: the dk pass of the
// attention backward runs in place (dy == dx).
template <typename T, typename X>
__global__ void __launch_bounds__(256) row_bwd_kernel(const RowArgs a) {
  constexpr int E = 16 / sizeof(X);                   // elements of dy / dx per 16-byte vector
  const RowTensor& t = a.t[0];
  const int tpr = a.D >> 3;
  const long long row = (long long)blockIdx.x * (256 / tpr) + threadIdx.x / tpr;
  const int tr = threadIdx.x % tpr;
  const bool ok = row < (long long)a.B * t.H * t.N;
  const long long rr = ok ? row : 0;
  const int n = (int)(rr % t.N);
  const int h = (int)((rr / t.N) % t.H);
  const int b = (int)(rr / ((long long)t.N * t.H));
  const X* dyp = static_cast<const X*>(t.x.ptr) + b * t.x.sb + h * t.x.sh + (long long)n * t.x.sn + tr * 8;
  uint4 rdy[8 / E], ry = make_uint4(0, 0, 0, 0);
#pragma unroll
  for (int v = 0; v < 8 / E; ++v) rdy[v] = ok ? ld_stream128(dyp + v * E) : make_uint4(0, 0, 0, 0);
  if (ok && a.G > 0)
    ry = ldg_stream128(static_cast<const T*>(t.y.ptr) + b * t.y.sb + h * t.y.sh + (long long)n * t.y.sn + tr * 8);
  float g[8];
#pragma unroll
  for (int v = 0; v < 8 / E; ++v) unpack16B<X>(rdy[v], g + v * E);
  const float mul = row_mul<X>(a);
  if (a.G == 0) {
#pragma unroll
    for (int i = 0; i < 8; ++i) g[i] *= mul;
  } else {
    float y[8];
    unpack16B<T>(ry, y);
    l2norm_bwd_group<8>(g, y, a.D / a.G, tr, ok ? t.rnorm + row * a.G : nullptr, mul);
  }
  if (!ok) return;
  X* dxp = static_cast<X*>(t.dx.ptr) + b * t.dx.sb + h * t.dx.sh + (long long)n * t.dx.sn + tr * 8;
#pragma unroll
  for (int v = 0; v < 8 / E; ++v) *reinterpret_cast<uint4*>(dxp + v * E) = pack16B<X>(g + v * E);
}

// ------------------------------------------------------------------------------------------------
// launchers: the grid, the instantiation and the launch error of each direction
// ------------------------------------------------------------------------------------------------
constexpr int kRowFwdU = 2;                           // forward: rows per thread (16 features each)

template <typename T, typename X>
cudaError_t launch_row_fwd_t(const RowArgs& a, dim3 grid, cudaStream_t stream) {
  constexpr int U = kRowFwdU;
  if (a.D == 64) return launch_pdl(row_fwd_kernel<T, X, 4, U>, grid, dim3(256), 0, stream, a);
  if (a.D == 128) return launch_pdl(row_fwd_kernel<T, X, 8, U>, grid, dim3(256), 0, stream, a);
  return launch_pdl(row_fwd_kernel<T, X, 0, U>, grid, dim3(256), 0, stream, a);
}

// forward over a.t[0] and, when a.t[1].H > 0, a.t[1]; x is float32 when f32_in, else of y's type
inline cudaError_t launch_row_fwd(const RowArgs& a, bool bf16, bool f32_in, cudaStream_t stream) {
  const int rows_per_block = kRowFwdU * (256 / (a.D / 16));
  const long long rows = (long long)a.B * (a.t[0].H * a.t[0].N > a.t[1].H * a.t[1].N ? a.t[0].H * a.t[0].N
                                                                                     : a.t[1].H * a.t[1].N);
  const dim3 grid((unsigned)((rows + rows_per_block - 1) / rows_per_block), a.t[1].H ? 2 : 1);
  if (bf16)
    return f32_in ? launch_row_fwd_t<__nv_bfloat16, float>(a, grid, stream)
                  : launch_row_fwd_t<__nv_bfloat16, __nv_bfloat16>(a, grid, stream);
  return f32_in ? launch_row_fwd_t<__half, float>(a, grid, stream) : launch_row_fwd_t<__half, __half>(a, grid, stream);
}

// the append pass of the key/value-cache decode over a.t[0 .. n): 16-bit x and y, head dim 64 or 128
inline cudaError_t launch_row_append(const RowArgs& a, int n, bool bf16, cudaStream_t stream) {
  constexpr int U = kRowFwdU;
  const int rows_per_block = U * (256 / (a.D / 16));
  long long rows = 0;
  for (int i = 0; i < n; ++i) {
    const long long r = (long long)a.B * a.t[i].H * a.t[i].N;
    rows = r > rows ? r : rows;
  }
  const dim3 grid((unsigned)((rows + rows_per_block - 1) / rows_per_block), n);
  if (bf16)
    return a.D == 64 ? launch_pdl(row_fwd_kernel<__nv_bfloat16, __nv_bfloat16, 4, U, true>, grid, dim3(256), 0, stream, a)
                     : launch_pdl(row_fwd_kernel<__nv_bfloat16, __nv_bfloat16, 8, U, true>, grid, dim3(256), 0, stream, a);
  return a.D == 64 ? launch_pdl(row_fwd_kernel<__half, __half, 4, U, true>, grid, dim3(256), 0, stream, a)
                   : launch_pdl(row_fwd_kernel<__half, __half, 8, U, true>, grid, dim3(256), 0, stream, a);
}

// backward over a.t[0]; dy and dx are float32 when f32_grad, else of y's type
inline cudaError_t launch_row_bwd(const RowArgs& a, bool bf16, bool f32_grad, cudaStream_t stream) {
  const int rows_per_block = 256 / (a.D / 8);
  const long long rows = (long long)a.B * a.t[0].H * a.t[0].N;
  const unsigned grid = (unsigned)((rows + rows_per_block - 1) / rows_per_block);
  if (bf16) {
    if (f32_grad) row_bwd_kernel<__nv_bfloat16, float><<<grid, 256, 0, stream>>>(a);
    else row_bwd_kernel<__nv_bfloat16, __nv_bfloat16><<<grid, 256, 0, stream>>>(a);
  } else {
    if (f32_grad) row_bwd_kernel<__half, float><<<grid, 256, 0, stream>>>(a);
    else row_bwd_kernel<__half, __half><<<grid, 256, 0, stream>>>(a);
  }
  return cudaGetLastError();
}

}  // namespace fcsa
