// The pipeline the forward and decode kernels share, and the mbarrier ring all three attention kernels use.
//
// Per 128-key tile a consumer warpgroup of 64 query rows computes S = Q K^T (64 x 128, fp32) -> P = exp2(S*c1 + add),
// masked where the tile needs it, row sums in fp32, 16-bit P as wgmma A fragments -> O += P V.  The kernels keep what
// differs: how Q gets into shared memory, the additive term and key mask (the forward's bias and padding mask), what
// happens to V before P V (decode zeroes rows past its valid length) and what the epilogue writes.
#pragma once

#include "sm90_primitives.cuh"
#include "tile_ranges.h"

namespace fcsa {

// A ring of S slots, each with a FULL barrier (the producer has filled it) and an EMPTY one (its consumers are done
// with it), at FULL + s and EMPTY + s of the kernel's barrier array.  Use n of the ring (0, 1, ...) is slot n % S in
// phase n / S: its consumers wait for that phase of FULL; its producer waits for the previous phase of EMPTY, which a
// fresh barrier counts as complete, so the first S uses do not wait.
template <int S>
struct Ring {
  uint32_t full, empty;            // shared addresses of FULL[0], EMPTY[0]

  __device__ __forceinline__ uint32_t full_bar(int s) const { return full + 8u * s; }
  __device__ __forceinline__ uint32_t empty_bar(int s) const { return empty + 8u * s; }
  __device__ __forceinline__ void init(uint32_t full_count, uint32_t empty_count) const {
    for (int s = 0; s < S; ++s) {
      mbar_init(full_bar(s), full_count);
      mbar_init(empty_bar(s), empty_count);
    }
  }
  // producer: wait until use n's slot is free; returns the slot
  __device__ __forceinline__ int acquire(int n) const {
    mbar_wait(empty_bar(n % S), ((n / S) & 1) ^ 1);
    return n % S;
  }
  // producer without TMA: use n's slot is filled
  __device__ __forceinline__ void commit(int n) const { mbar_arrive(full_bar(n % S)); }
  // consumer: wait until use n's slot is filled; returns the slot
  __device__ __forceinline__ int wait(int n) const {
    mbar_wait(full_bar(n % S), (n / S) & 1);
    return n % S;
  }
  // consumer: done with use n's slot
  __device__ __forceinline__ void release(int n) const { mbar_arrive(empty_bar(n % S)); }
  // a consumer that does not read use n still takes part in it (an arrival must count for this use of the slot)
  __device__ __forceinline__ void pass(int n) const {
    wait(n);
    release(n);
  }
};

// ---- producer: K and V tiles [j0, j1) through the two rings (tile j is use j - j0) --------------------------------
// Tile j is rows row0 + 128 j of kv head hk at batch coordinate tb, D / 64 TMA boxes of 64 features each.
template <int D, int S>
__device__ __forceinline__ void load_kv_tiles(const CUtensorMap* tm_k, const CUtensorMap* tm_v, Ring<S> kr, Ring<S> vr,
                                              uint32_t sK, uint32_t sV, int j0, int j1, int row0, int hk, int tb) {
  constexpr int TILE = 128 * D * 2;
  for (int j = j0; j < j1; ++j) {
    const int s = kr.acquire(j - j0);
    mbar_expect_tx(kr.full_bar(s), TILE);
#pragma unroll
    for (int ch = 0; ch < D / 64; ++ch)
      tma_load_4d(sK + s * TILE + ch * 16384, tm_k, kr.full_bar(s), ch * 64, row0 + j * 128, hk, tb);
    vr.acquire(j - j0);
    mbar_expect_tx(vr.full_bar(s), TILE);
#pragma unroll
    for (int ch = 0; ch < D / 64; ++ch)
      tma_load_4d(sV + s * TILE + ch * 16384, tm_v, vr.full_bar(s), ch * 64, row0 + j * 128, hk, tb);
  }
}

// ---- consumer: S = Q K^T (64 x 128, fp32) ----------------------------------------------------------------------
// sQ: the warpgroup's 64 rows of the first 64-feature chunk of Q, q_chunk bytes to the next; sKs: the K tile's slot.
template <typename T, int D>
__device__ __forceinline__ void qk_tile(float (&sacc)[64], uint32_t sQ, uint32_t q_chunk, uint32_t sKs) {
  wgmma_fence();
#pragma unroll
  for (int kk = 0; kk < D / 16; ++kk) {
    const uint32_t ko = (kk & 3) * 32;         // + the 64-feature chunk (kk >> 2)
    wgmma_ss<T, 0, 0>(sacc, gmma_desc_sw128(sQ + (kk >> 2) * q_chunk + ko, 16, 1024),
                      gmma_desc_sw128(sKs + (kk >> 2) * 16384 + ko, 16, 1024), kk > 0 ? 1u : 0u);
  }
  wgmma_commit();
  wgmma_wait<0>();
  fence_regs(sacc);
}

// ---- consumer: P = exp2(S*c1 + add), masked; row sums in fp32; 16-bit P as A fragments ----------------------------
// Element pair i of S (sacc[2 i], sacc[2 i + 1]) is row hf = i & 1 of the thread's two rows (accumulator layout,
// sm90_primitives.cuh), columns col = col0 + 8 (i >> 1) + cq and col + 1.  add(hf, col) returns the additive terms of
// the pair.  On a tile that needs masks (tile_visible is false) a column outside the row's lim (row_key_cols), or one
// that keys(col) refuses when keys.on(), gives p = 0: a select, since S may be anything there.
struct ShiftOnly {                   // the additive term without a bias: -shift * log2(e)
  float nc2;
  __device__ __forceinline__ float2 operator()(int, int) const { return make_float2(nc2, nc2); }
};
struct AllKeys {                     // no key padding mask
  __device__ __forceinline__ bool on() const { return false; }
  __device__ __forceinline__ bool operator()(int) const { return true; }
};
template <typename T, bool WINDOW, class Add, class Keys>
__device__ __forceinline__ void exp_tile(bool need_mask, const float (&sacc)[64], uint32_t (&pf)[32], float (&l)[2],
                                         float c1, int col0, int cq, const ColRange (&lim)[2], Add add, Keys keys) {
  auto run = [&](auto masked_tag) {
    constexpr bool MASKED = decltype(masked_tag)::value;
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int hf = i & 1;
      const int col = col0 + 8 * (i >> 1) + cq;
      const float2 ad = add(hf, col);
      float p0 = ex2_approx(fmaf(sacc[2 * i], c1, ad.x));
      float p1 = ex2_approx(fmaf(sacc[2 * i + 1], c1, ad.y));
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
      l[hf] += p0 + p1;
      pf[i] = pack2<T>(p0, p1);
    }
  };
  if (need_mask) run(std::true_type{});
  else run(std::false_type{});
}

// ---- consumer: O += P V ----------------------------------------------------------------------------------------
// sVs: the V tile's slot.
template <typename T, int N>
__device__ __forceinline__ void pv_tile(float (&o)[N], uint32_t (&pf)[32], uint32_t sVs) {
  wgmma_fence();
#pragma unroll
  for (int kk = 0; kk < 8; ++kk) {
    const uint32_t af[4] = {pf[4 * kk], pf[4 * kk + 1], pf[4 * kk + 2], pf[4 * kk + 3]};
    wgmma_rs<T, 1>(o, af, gmma_desc_sw128(sVs + kk * 2048, 16384, 1024), 1u);
  }
  wgmma_commit();
  wgmma_wait<0>();
  fence_regs(o);
  fence_regs(pf);
}

// ---- epilogue ---------------------------------------------------------------------------------------------------
// A row's sum over the four lanes that hold its columns.
__device__ __forceinline__ float quad_sum(float x) {
  x += __shfl_xor_sync(0xFFFFFFFFu, x, 1);
  x += __shfl_xor_sync(0xFFFFFFFFu, x, 2);
  return x;
}

// The thread's columns of row hf of a 64 x 4N accumulator, times scale, to row (float32 or 16-bit Out): columns
// 8 jb + cq and + 1 are acc[4 jb + 2 hf] and acc[4 jb + 2 hf + 1].
template <typename Out, int N>
__device__ __forceinline__ void store_row(Out* row, const float (&acc)[N], int hf, int cq, float scale) {
#pragma unroll
  for (int jb = 0; jb < N / 4; ++jb) {
    const float x = acc[4 * jb + 2 * hf] * scale, y = acc[4 * jb + 2 * hf + 1] * scale;
    if constexpr (std::is_same<Out, float>::value) *reinterpret_cast<float2*>(row + 8 * jb + cq) = make_float2(x, y);
    else *reinterpret_cast<uint32_t*>(row + 8 * jb + cq) = pack2<Out>(x, y);
  }
}

}  // namespace fcsa
