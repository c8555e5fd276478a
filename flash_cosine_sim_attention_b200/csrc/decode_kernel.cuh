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
//                   per key tile S = Q K^T -> P = exp2(S*c1 - c2), masked -> O += P V, all as in the forward
//   * visible length T_b = min(cache_seqlens[b] + n_new, capacity); query i sees key j iff j < T_b and, causal,
//     j <= i + T_b - Nq (the forward's bottom-right rule with Nk = T_b).  The ceil(T_b / 128) tiles a block can see
//     are cut into n_split contiguous chunks on the device, so a cache allocated at full length costs nothing.
//   * n_split = 1: o is written directly.  Otherwise each split writes fp32 partials (O_s, l_s) and
//     decode_combine_kernel forms o = sum_s O_s / max(sum_s l_s, 1e-37) in split order: o is bitwise reproducible.
#pragma once

#include "sm90_primitives.cuh"

namespace fcsa {

struct DecodeArgs {
  int B, H, KVH, G;          // G = H / KVH query heads per kv head
  int Nq, cap, n_new;        // new queries, cache rows (capacity), rows the append pass added at cache_seqlens[b]
  int causal;
  int R, n_rb, n_split;      // R = G * Nq rows per (batch, kv head), in n_rb blocks of 64; key splits
  float c1;                  // scale * log2(e)
  float c2;                  // shift * log2(e)
  const int32_t* seqlens;    // (B,) valid cache rows before the call
  const void* q;             // (B, H, Nq, D), element strides, feature dim contiguous
  long long q_sb, q_sh, q_sn;
  void* o;
  long long o_sb, o_sh, o_sn;
  float* part;               // n_split > 1: O_s [item][split][64][D], then l_s [item][split][64] (fp32)
};

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

// Splits per work item: 1 when the items alone fill the SMs, otherwise the fewest that do, at most one per key tile
// of the capacity.  (tests/test_decode_host.py mirrors this rule.)
inline int decode_split(long long items, int cap, int sm_count) {
  if (items >= sm_count) return 1;
  const long long want = (sm_count + items - 1) / items;
  const long long tiles = (cap + 127) / 128;
  return (int)(want < tiles ? want : tiles);
}

template <typename T, int D>
__global__ void __launch_bounds__(256, DecodeCfg<D>::kCtasPerSm)
fcsa_decode_kernel(const __grid_constant__ CUtensorMap tm_k, const __grid_constant__ CUtensorMap tm_v,
                   const DecodeArgs a) {
  using Cfg = DecodeCfg<D>;
  constexpr int S = Cfg::kStages, TILE = Cfg::kTile, DCH = D / 64;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~uintptr_t(1023));
  const uint32_t sQ = smem_u32(smem + Cfg::kOffQ);
  const uint32_t sK = smem_u32(smem + Cfg::kOffK);
  const uint32_t sV = smem_u32(smem + Cfg::kOffV);
  const uint32_t bar0 = smem_u32(smem + Cfg::kOffBar);
  auto BAR = [&](int i) { return bar0 + 8u * i; };
  constexpr int K_FULL = 0, K_EMPTY = K_FULL + S, V_FULL = K_EMPTY + S, V_EMPTY = V_FULL + S, NBARS = V_EMPTY + S;
  static_assert(NBARS * 8 <= 256, "barrier area");

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
  const int r_last = min(r0 + 63, a.R - 1);

  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(BAR(K_FULL + s), 1);
      mbar_init(BAR(K_EMPTY + s), 128);
      mbar_init(BAR(V_FULL + s), 1);
      mbar_init(BAR(V_EMPTY + s), 128);
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();          // q (normalised by the append pass), the caches and cache_seqlens are read from here on

  // visible keys and this split's key tiles (uniform over the CTA)
  const int L = min(max(a.seqlens[b], 0), a.cap);
  const int Tb = min(L + a.n_new, a.cap);
  const int off = Tb - a.Nq;
  int nt = (Tb + 127) >> 7;
  if (a.causal) {
    const int last_col = r_last / a.G + off;
    nt = last_col < 0 ? 0 : min(nt, (last_col >> 7) + 1);
  }
  const int j0 = (int)((long long)nt * split / a.n_split);
  const int j1 = (int)((long long)nt * (split + 1) / a.n_split);

  if (wg == 0) {
    // =============================== TMA producer ===============================
    if constexpr (Cfg::kCtasPerSm == 2) reg_dealloc<40>();
    if (warp == 0 && elect_one() && j1 > j0) {
      tma_prefetch_desc(&tm_k);
      tma_prefetch_desc(&tm_v);
      for (int j = j0; j < j1; ++j) {
        const int s = (j - j0) % S;
        const uint32_t par = (((j - j0) / S) & 1) ^ 1;
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

  // =============================== consumer warpgroup ============================
  if constexpr (Cfg::kCtasPerSm == 2) reg_alloc<216>();     // 128 x 40 + 128 x 216 = 256 x 128
  const int t = threadIdx.x - 128;
  const int wl = warp & 3;
  const int row_a = 16 * wl + (lane >> 2);    // this thread's rows of the block: row_a and row_a + 8
  const int cq = 2 * (lane & 3);

  if (j1 > j0) {
    // Q: row r of the block is query i = r / G of head hk * G + r % G; rows past R are zero.  Every 64-feature
    // chunk is a 64 x 128-byte SWIZZLE_128B tile (8 KB), the layout a TMA box would leave.
    constexpr int CH = D / 8;                 // 16-byte pieces per row
#pragma unroll
    for (int k = 0; k < 64 * CH / 128; ++k) {
      const int idx = t + 128 * k, row = idx / CH, c = idx - (idx / CH) * CH;
      const int r = r0 + row;
      uint4 v = make_uint4(0, 0, 0, 0);
      if (r < a.R) {
        const int i = r / a.G, h = hk * a.G + (r - i * a.G);
        v = __ldg(reinterpret_cast<const uint4*>(static_cast<const T*>(a.q) + b * a.q_sb + h * a.q_sh +
                                                 (long long)i * a.q_sn + c * 8));
      }
      *reinterpret_cast<uint4*>(smem + Cfg::kOffQ + (c >> 3) * 8192 + sw128_offset(row, c & 7)) = v;
    }
    fence_proxy_async_smem();
    named_bar_sync(1, 128);
  }

  // last visible column of each of the thread's rows (-1: a padding row past R)
  int lim[2];
#pragma unroll
  for (int hf = 0; hf < 2; ++hf) {
    const int r = r0 + row_a + 8 * hf;
    lim[hf] = r >= a.R ? -1 : (a.causal ? min(Tb - 1, r / a.G + off) : Tb - 1);
  }
  const int first_lim = r0 / a.G + off;       // the block's smallest causal limit
  const float c1 = a.c1, nc2 = -a.c2;

  float o[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) o[i] = 0.f;
  float l[2] = {0.f, 0.f};

  for (int j = j0; j < j1; ++j) {
    const int s = (j - j0) % S;
    const uint32_t par = ((j - j0) / S) & 1;
    // ---- S = Q K^T (64 x 128, fp32) ----
    float sacc[64];
    mbar_wait(BAR(K_FULL + s), par);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk) {
      const uint32_t qo = (kk >> 2) * 8192 + (kk & 3) * 32;
      const uint32_t ko = (kk >> 2) * 16384 + (kk & 3) * 32;
      wgmma_ss_n128<T, 0, 0>(sacc, gmma_desc_sw128(sQ + qo, 16, 1024), gmma_desc_sw128(sK + s * TILE + ko, 16, 1024),
                             kk > 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(sacc);
    mbar_arrive(BAR(K_EMPTY + s));

    // ---- P = exp2(S*c1 - c2), masked (a select: cache rows past T_b may hold anything); 16-bit P as A fragments --
    const int col0 = j * 128;
    const bool need_mask = (col0 + 127 >= Tb) || (a.causal && col0 + 127 > first_lim);
    uint32_t pf[32];
    auto exp_tile = [&](auto masked_tag) {
      constexpr bool MASKED = decltype(masked_tag)::value;
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        const int hf = i & 1;
        const int col = col0 + 8 * (i >> 1) + cq;
        float p0 = ex2_approx(fmaf(sacc[2 * i], c1, nc2));
        float p1 = ex2_approx(fmaf(sacc[2 * i + 1], c1, nc2));
        if constexpr (MASKED) {
          p0 = col <= lim[hf] ? p0 : 0.f;
          p1 = col + 1 <= lim[hf] ? p1 : 0.f;
        }
        l[hf] += p0 + p1;
        pf[i] = pack2<T>(p0, p1);
      }
    };
    if (need_mask) exp_tile(std::true_type{});
    else exp_tile(std::false_type{});

    // ---- O += P V ----
    mbar_wait(BAR(V_FULL + s), par);
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

  // ---- epilogue --------------------------------------------------------------------------
#pragma unroll
  for (int hf = 0; hf < 2; ++hf) {
    l[hf] += __shfl_xor_sync(0xFFFFFFFFu, l[hf], 1);
    l[hf] += __shfl_xor_sync(0xFFFFFFFFu, l[hf], 2);
  }
  if (a.n_split == 1) {
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
      const int r = r0 + row_a + 8 * hf;
      if (r >= a.R) continue;
      const int i = r / a.G, h = hk * a.G + (r - i * a.G);
      const float inv = 1.0f / fmaxf(l[hf], 1e-37f);
      T* orow = static_cast<T*>(a.o) + b * a.o_sb + h * a.o_sh + (long long)i * a.o_sn;
#pragma unroll
      for (int jb = 0; jb < D / 8; ++jb)
        *reinterpret_cast<uint32_t*>(orow + 8 * jb + cq) = pack2<T>(o[4 * jb + 2 * hf] * inv, o[4 * jb + 2 * hf + 1] * inv);
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
#pragma unroll
    for (int jb = 0; jb < D / 8; ++jb)
      *reinterpret_cast<float2*>(po + row * D + 8 * jb + cq) = make_float2(o[4 * jb + 2 * hf], o[4 * jb + 2 * hf + 1]);
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
  if (r >= a.R) return;
  const float* po = a.part + (item * a.n_split * 64 + row) * D + 4 * qd;
  const float* pl = a.part + n_items * a.n_split * 64 * D + item * a.n_split * 64 + row;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  float l = 0.f;
  for (int s = 0; s < a.n_split; ++s) {
    const float4 v = *reinterpret_cast<const float4*>(po + (long long)s * 64 * D);
    acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    l += pl[s * 64];
  }
  const float inv = 1.0f / fmaxf(l, 1e-37f);
  const int i = r / a.G, h = hk * a.G + (r - i * a.G);
  T* orow = static_cast<T*>(a.o) + b * a.o_sb + h * a.o_sh + (long long)i * a.o_sn + 4 * qd;
  *reinterpret_cast<uint2*>(orow) = make_uint2(pack2<T>(acc.x * inv, acc.y * inv), pack2<T>(acc.z * inv, acc.w * inv));
}

// bytes of the partials of n_split > 1
inline size_t decode_partial_bytes(long long items, int n_split, int D) {
  return n_split > 1 ? (size_t)items * n_split * 64 * (D + 1) * sizeof(float) : 0;
}

}  // namespace fcsa
