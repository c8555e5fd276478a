// Host-side construction of TMA tensor maps for (batch, head, row, feature) tensors whose
// feature dimension is contiguous.  The driver entry point is resolved at run time through
// cudaGetDriverEntryPoint so the library does not link against libcuda.
//
// This is what replaces the reference's strided PackedTensorAccessor32 indexing
// (flash_cosine_sim_attention_cuda.cu:30-35): arbitrary (b, h, n) strides are encoded in
// the tensor map, the kernels never compute element addresses for q/k/v/do themselves.
#pragma once

#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <atomic>

namespace fcsa {

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                    const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                    const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline PFN_encodeTiled get_encode_tiled() {
  static PFN_encodeTiled fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult qres;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
  if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || p == nullptr) return nullptr;
  fn = reinterpret_cast<PFN_encodeTiled>(p);
  return fn;
}

// Tensor map over a 16-bit or fp32 tensor addressed as [b][h][n][d] with element strides
// (sb, sh, sn, 1).  The box is box_cols features x box_rows rows: 64 16-bit features = one 128-byte swizzle
// span for the operand tiles, 32 fp32 features = one 128-byte span for the dq accumulator tiles, 16 16-bit
// features = one 32-byte span (swizzle_bytes = 32) for the K = 16 slivers.
// A dimension of extent 1 gets a dummy stride (the driver rejects zero strides); a zero or negative
// stride on a dimension of extent > 1 (an expanded / broadcast view) cannot be expressed by a tensor
// map and is refused (-2) - callers make such tensors contiguous first.
// Returns 0 on success, -1 if the driver entry point is missing, -2 for an inexpressible view, else
// the CUresult.
struct TensorMapKey {
  const void* base;
  int64_t B, H, N, D, sb, sh, sn;
  int32_t dtype, box_rows, box_cols, swizzle_bytes;     // dtype: a CUtensorMapDataType
};

inline CUtensorMapDataType tma_dtype16(bool is_bf16) {
  return is_bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
}

inline int encode_tensor_map_bhnd(CUtensorMap* tm, const TensorMapKey& k) {
  PFN_encodeTiled enc = get_encode_tiled();
  if (!enc) return -1;
  cuuint64_t dims[4] = {(cuuint64_t)k.D, (cuuint64_t)k.N, (cuuint64_t)k.H, (cuuint64_t)k.B};
  const CUtensorMapDataType dt = (CUtensorMapDataType)k.dtype;
  const int64_t es = dt == CU_TENSOR_MAP_DATA_TYPE_FLOAT32 ? 4 : 2;     // element bytes
  // strides in bytes for dims 1..3
  int64_t sn_b = k.sn * es, sh_b = k.sh * es, sb_b = k.sb * es;
  if ((k.N > 1 && sn_b <= 0) || (k.H > 1 && sh_b <= 0) || (k.B > 1 && sb_b <= 0)) return -2;
  if (k.N == 1) sn_b = k.D * es;
  if (k.H == 1) sh_b = sn_b * k.N;
  if (k.B == 1) sb_b = sh_b * k.H;
  cuuint64_t strides[3] = {(cuuint64_t)sn_b, (cuuint64_t)sh_b, (cuuint64_t)sb_b};
  cuuint32_t box[4] = {(cuuint32_t)k.box_cols, (cuuint32_t)k.box_rows, 1, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = enc(tm, dt, 4, const_cast<void*>(k.base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE,
                   k.swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                                          : (k.swizzle_bytes == 32 ? CU_TENSOR_MAP_SWIZZLE_32B : CU_TENSOR_MAP_SWIZZLE_NONE),
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return (int)r;
}

// A tensor map is a pure function of (pointer, shape, strides, box): training loops present the same
// few views again and again, so each thread keeps the last few encodings.  32 entries x 8 maps per step (3 forward, 5 backward) cover several layers' worth of views.
inline int make_tensor_map_bhnd(CUtensorMap* tm, const void* base, CUtensorMapDataType dtype, int64_t B,
                                int64_t H, int64_t N, int64_t D, int64_t sb, int64_t sh, int64_t sn,
                                int box_rows, int box_cols = 64, int swizzle_bytes = 128) {
  struct Entry {
    TensorMapKey key;
    CUtensorMap map;
    bool used;
  };
  constexpr int kEntries = 32;
  thread_local Entry cache[kEntries];
  thread_local int next_victim = 0;
  TensorMapKey key;
  memset(&key, 0, sizeof(key));
  key.base = base; key.B = B; key.H = H; key.N = N; key.D = D; key.sb = sb; key.sh = sh; key.sn = sn;
  key.dtype = (int32_t)dtype; key.box_rows = box_rows; key.box_cols = box_cols; key.swizzle_bytes = swizzle_bytes;
  for (int i = 0; i < kEntries; ++i)
    if (cache[i].used && memcmp(&cache[i].key, &key, sizeof(key)) == 0) {
      *tm = cache[i].map;
      return 0;
    }
  const int r = encode_tensor_map_bhnd(tm, key);
  if (r == 0) {
    Entry& e = cache[next_victim];
    next_victim = (next_victim + 1) % kEntries;
    e.key = key; e.map = *tm; e.used = true;
  }
  return r;
}

// cudaFuncAttributeMaxDynamicSharedMemorySize is a per-DEVICE attribute of a kernel: set it once per
// (kernel, device), thread-safe (autograd runs the backward on its own thread; one process may drive
// several GPUs).
template <auto Kern>
inline cudaError_t ensure_dynamic_smem(int bytes) {
  static std::atomic<uint64_t> done[4];          // devices 0..255
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  if (dev < 0 || dev >= 256) return cudaFuncSetAttribute(Kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  const uint64_t bit = 1ull << (dev & 63);
  if (done[dev >> 6].load(std::memory_order_acquire) & bit) return cudaSuccess;
  e = cudaFuncSetAttribute(Kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e == cudaSuccess) done[dev >> 6].fetch_or(bit, std::memory_order_release);
  return e;
}

// Number of SMs of the current device, read once per device (0 = not read yet).
inline cudaError_t device_sm_count(int* n) {
  static std::atomic<int> count[256];
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  if (dev >= 0 && dev < 256 && (*n = count[dev].load(std::memory_order_relaxed)) > 0) return cudaSuccess;
  e = cudaDeviceGetAttribute(n, cudaDevAttrMultiProcessorCount, dev);
  if (e == cudaSuccess && dev >= 0 && dev < 256) count[dev].store(*n, std::memory_order_relaxed);
  return e;
}

// Launch with programmatic dependent launch enabled (see pdl_wait / pdl_launch_dependents).
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                              Args... args) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

}  // namespace fcsa
