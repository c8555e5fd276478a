// Host side of libfcsa_b200.so: argument validation, TMA tensor-map construction, the
// {f16, bf16} x {64, 128} switch and the kernel launches behind the C ABI of
// include/fcsa_b200.h.
//
// Replaces the reference's host op + pybind layer (flash_cosine_sim_attention_cuda.cu:1630-1933)
// and its dispatch macros (dispatch.h:38-73).  Differences by design: launches go to the
// caller's stream and never synchronise (reference: legacy stream + cudaDeviceSynchronize,
// cu:1720/1745/1889); errors are returned, not printed (cu:17-28); sm_90a only.
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <atomic>

#include "../../include/fcsa_b200.h"
#include "bwd_kernel.cuh"
#include "decode_kernel.cuh"
#include "fwd_kernel.cuh"
#include "l2norm_kernels.cuh"
#include "tensor_map.h"

namespace {

thread_local char g_err[512] = "";
cudaEvent_t g_ev[5][2] = {};   // 0 forward, 1 backward, 2 l2norm(q,k), 3 backward preprocess, 4 dq finish
std::atomic<long long> g_launches{0};

int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

int cuda_fail(cudaError_t e, const char* what) {
  return fail(FCSA_ERR_CUDA, "%s: %s", what, cudaGetErrorString(e));
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

int check_tensor(const fcsa_tensor* t, const char* name) {
  if (!t || !t->ptr) return fail(FCSA_ERR_INVALID, "%s: null tensor", name);
  if (!aligned16(t->ptr)) return fail(FCSA_ERR_INVALID, "%s: pointer not 16-byte aligned", name);
  if ((t->sb % 8) || (t->sh % 8) || (t->sn % 8))
    return fail(FCSA_ERR_INVALID, "%s: strides must be multiples of 8 elements (16 bytes)", name);
  if (t->sb < 0 || t->sh < 0 || t->sn < 0)
    return fail(FCSA_ERR_INVALID, "%s: negative strides are not supported", name);
  return FCSA_OK;
}

int check_problem(const fcsa_problem* p) {
  if (!p) return fail(FCSA_ERR_INVALID, "null problem");
  if (p->dtype != FCSA_F16 && p->dtype != FCSA_BF16)
    return fail(FCSA_ERR_UNSUPPORTED, "dtype %d: only f16 and bf16 are implemented", p->dtype);
  if (p->head_dim != 64 && p->head_dim != 128)
    return fail(FCSA_ERR_UNSUPPORTED, "head_dim %d: only 64 and 128 are implemented", p->head_dim);
  if (p->batch <= 0 || p->heads <= 0 || p->seq_q <= 0 || p->seq_k <= 0)
    return fail(FCSA_ERR_INVALID, "empty problem (batch %d heads %d seq_q %d seq_k %d)", p->batch,
                p->heads, p->seq_q, p->seq_k);
  if (p->kv_heads <= 0 || p->heads % p->kv_heads != 0)
    return fail(FCSA_ERR_INVALID, "kv_heads must divide heads (got %d kv_heads for %d heads)", p->kv_heads,
                p->heads);
  if (p->causal && p->key_mask)
    return fail(FCSA_ERR_INVALID, "mask should not be supplied if causality is needed");
  return FCSA_OK;
}

int check_bias(const fcsa_problem* p, const fcsa_bias* bias) {
  if (!bias || !bias->ptr) return fail(FCSA_ERR_INVALID, "attn_bias: null");
  if (!aligned16(bias->ptr) || (bias->sn % 8) != 0 || (bias->sh % 8) != 0 || (bias->sb % 8) != 0)
    return fail(FCSA_ERR_INVALID, "attn_bias: rows must be 16-byte aligned (strides multiples of 8 elements)");
  if (bias->sn < ((p->seq_k + 7) / 8) * 8)
    return fail(FCSA_ERR_INVALID, "attn_bias: row stride %lld shorter than seq_k rounded up to 8", (long long)bias->sn);
  return FCSA_OK;
}

template <typename T, int D, bool BIAS = false>
int launch_forward(const fcsa_problem* p, const fcsa_tensor* q, const fcsa_tensor* k,
                   const fcsa_tensor* v, const fcsa_tensor* o, float* inv_l, cudaStream_t stream,
                   const fcsa_bias* bias = nullptr) {
  using Cfg = fcsa::FwdCfg<D>;
  const bool bf = p->dtype == FCSA_BF16;
  CUtensorMap tq, tk, tv;
  int r;
  if ((r = fcsa::make_tensor_map_bhnd(&tq, q->ptr, fcsa::tma_dtype16(bf), p->batch, p->heads, p->seq_q, D, q->sb, q->sh,
                                      q->sn, 128)))
    return fail(r == -2 ? FCSA_ERR_INVALID : FCSA_ERR_CUDA, "q: %s (%d)", r == -2 ? "expanded (stride-0) views of extent > 1 cannot be addressed by a tensor map - make the tensor contiguous" : "cuTensorMapEncodeTiled failed", r);
  if ((r = fcsa::make_tensor_map_bhnd(&tk, k->ptr, fcsa::tma_dtype16(bf), p->batch, p->kv_heads, p->seq_k, D, k->sb,
                                      k->sh, k->sn, 128)))
    return fail(r == -2 ? FCSA_ERR_INVALID : FCSA_ERR_CUDA, "k: %s (%d)", r == -2 ? "expanded (stride-0) views of extent > 1 cannot be addressed by a tensor map - make the tensor contiguous" : "cuTensorMapEncodeTiled failed", r);
  if ((r = fcsa::make_tensor_map_bhnd(&tv, v->ptr, fcsa::tma_dtype16(bf), p->batch, p->kv_heads, p->seq_k, D, v->sb,
                                      v->sh, v->sn, 128)))
    return fail(r == -2 ? FCSA_ERR_INVALID : FCSA_ERR_CUDA, "v: %s (%d)", r == -2 ? "expanded (stride-0) views of extent > 1 cannot be addressed by a tensor map - make the tensor contiguous" : "cuTensorMapEncodeTiled failed", r);

  fcsa::FwdArgs a;
  a.B = p->batch;
  a.H = p->heads;
  a.Nq = p->seq_q;
  a.Nk = p->seq_k;
  a.causal = p->causal ? 1 : 0;
  a.has_mask = p->key_mask ? 1 : 0;
  a.group = p->heads / p->kv_heads;
  a.n_qblk = (p->seq_q + 127) / 128;
  const float log2e = 1.4426950408889634f;
  a.c1 = p->scale * log2e;
  a.c2 = p->shift * log2e;
  a.mask = p->key_mask;
  a.mask_sb = p->key_mask_stride;
  a.o = o->ptr;
  a.o_sb = o->sb;
  a.o_sh = o->sh;
  a.o_sn = o->sn;
  a.o_f32 = p->out_f32 ? 1 : 0;
  a.inv_l = inv_l;
  a.bias = BIAS ? bias->ptr : nullptr;
  a.bias_sb = BIAS ? bias->sb : 0;
  a.bias_sh = BIAS ? bias->sh : 0;
  a.bias_sn = BIAS ? bias->sn : 0;
  a.bias_amax = BIAS ? bias->amax : nullptr;

  auto kern = fcsa::fcsa_fwd_kernel<T, D, BIAS>;
  {
    cudaError_t e = fcsa::ensure_dynamic_smem<fcsa::fcsa_fwd_kernel<T, D, BIAS>>(Cfg::kSmem);
    if (e != cudaSuccess) return cuda_fail(e, "cudaFuncSetAttribute(fwd)");
  }
  // one CTA per (query block of 128 rows, batch, head)
  const long long grid = (long long)a.n_qblk * p->batch * p->heads;
  if (grid > 0x7FFFFFFFLL) return fail(FCSA_ERR_INVALID, "problem too large for one launch");
  if (g_ev[0][0]) cudaEventRecord(g_ev[0][0], stream);
  cudaError_t e = fcsa::launch_pdl(kern, dim3((unsigned)grid), dim3(Cfg::kThreads), Cfg::kSmem, stream, tq, tk, tv, a);
  if (g_ev[0][1]) cudaEventRecord(g_ev[0][1], stream);
  if (e != cudaSuccess) return cuda_fail(e, "forward kernel launch");
  g_launches.fetch_add(1);
  return FCSA_OK;
}

// error and launch count of one row pass
int row_pass_launched(cudaError_t e, const char* what) {
  if (e != cudaSuccess) return cuda_fail(e, what);
  g_launches.fetch_add(1);
  return FCSA_OK;
}

// Shapes of the row passes.  The 16-bit l2norm takes head dims 32 to 256 and groups > 0; the float32 cast takes
// head dims 16 to 128, and groups = 0 for a plain cast.  Head dims are powers of two, so every group size is too.
int check_rows(bool f32, int32_t dtype, int32_t B, int32_t H, int32_t N, int32_t D, int32_t G) {
  const char* what = f32 ? "f32 cast" : "l2norm";
  if (dtype != FCSA_F16 && dtype != FCSA_BF16)
    return fail(FCSA_ERR_UNSUPPORTED, "%s: %sdtype %d not implemented", what, f32 ? "16-bit " : "", dtype);
  if (B <= 0 || H <= 0 || N <= 0) return fail(FCSA_ERR_INVALID, "%s: empty tensor", what);
  if (D < (f32 ? 16 : 32) || D > (f32 ? 128 : 256) || (D & (D - 1)) != 0)
    return fail(FCSA_ERR_UNSUPPORTED, "%s: head_dim %d not implemented", what, D);
  if (G < 0 || (G == 0 && !f32) || (G > 0 && D % G != 0))
    return fail(FCSA_ERR_INVALID, f32 ? "f32 cast: groups %d must divide %d into power-of-two chunks"
                                      : "l2norm: groups %d does not divide %d", G, D);
  return FCSA_OK;
}

// a float32 view whose rows start 16-byte aligned
bool f32_rows(const fcsa_tensor* t) {
  return t && t->ptr && aligned16(t->ptr) && t->sb % 4 == 0 && t->sh % 4 == 0 && t->sn % 4 == 0;
}

fcsa::RowArgs row_args(int32_t B, int32_t D, int32_t G, const float* mul = nullptr, int32_t mul_reciprocal = 0) {
  fcsa::RowArgs a = {};
  a.B = B; a.D = D; a.G = G; a.mul = mul; a.mul_reciprocal = mul_reciprocal;
  return a;
}

// ---- key/value-cache decode --------------------------------------------------------------------
// The problem of a decode call: seq_q = new queries, seq_k = cache capacity; no key mask, 16-bit output.
int check_decode_problem(const fcsa_problem* p, int32_t n_new) {
  int r;
  if ((r = check_problem(p))) return r;
  if (p->key_mask) return fail(FCSA_ERR_UNSUPPORTED, "decode: no key mask (cache_seqlens gives the valid rows)");
  if (p->out_f32) return fail(FCSA_ERR_UNSUPPORTED, "decode: out_f32 is not implemented");
  if (n_new < 0) return fail(FCSA_ERR_INVALID, "decode: n_new %d < 0", n_new);
  if ((long long)(p->heads / p->kv_heads) * p->seq_q > 0x7FFFFFFFLL - 64)
    return fail(FCSA_ERR_INVALID, "decode: heads per kv head x seq_q too large");
  return FCSA_OK;
}

struct DecodeShape {
  int R, n_rb, n_split;
  long long items;
};

// rows, row blocks, work items and splits of a decode problem on the current device
int decode_shape(const fcsa_problem* p, DecodeShape* s) {
  int sms = 0;
  const cudaError_t e = fcsa::device_sm_count(&sms);
  if (e != cudaSuccess) return cuda_fail(e, "cudaDeviceGetAttribute(multiProcessorCount)");
  s->R = (p->heads / p->kv_heads) * p->seq_q;
  s->n_rb = (s->R + 63) / 64;
  s->items = (long long)p->batch * p->kv_heads * s->n_rb;
  s->n_split = fcsa::decode_split(s->items, p->seq_k, sms);
  return FCSA_OK;
}

size_t align16(size_t n) { return (n + 15) & ~size_t(15); }

size_t decode_qhat_bytes(const fcsa_problem* p) {
  return align16((size_t)p->batch * p->heads * p->seq_q * p->head_dim * 2);
}

template <typename T, int D>
int launch_decode(const fcsa_problem* p, const DecodeShape& sh, const fcsa_tensor* q, const fcsa_tensor* kc,
                  const fcsa_tensor* vc, const int32_t* seqlens, int32_t n_new, const fcsa_tensor* o, float* part,
                  cudaStream_t stream) {
  using Cfg = fcsa::DecodeCfg<D>;
  const bool bf = p->dtype == FCSA_BF16;
  CUtensorMap tk, tv;
  int r;
  if ((r = fcsa::make_tensor_map_bhnd(&tk, kc->ptr, fcsa::tma_dtype16(bf), p->batch, p->kv_heads, p->seq_k, D, kc->sb,
                                      kc->sh, kc->sn, 128)))
    return fail(r == -2 ? FCSA_ERR_INVALID : FCSA_ERR_CUDA, "k_cache: %s (%d)", r == -2 ? "expanded (stride-0) views of extent > 1 cannot be addressed by a tensor map" : "cuTensorMapEncodeTiled failed", r);
  if ((r = fcsa::make_tensor_map_bhnd(&tv, vc->ptr, fcsa::tma_dtype16(bf), p->batch, p->kv_heads, p->seq_k, D, vc->sb,
                                      vc->sh, vc->sn, 128)))
    return fail(r == -2 ? FCSA_ERR_INVALID : FCSA_ERR_CUDA, "v_cache: %s (%d)", r == -2 ? "expanded (stride-0) views of extent > 1 cannot be addressed by a tensor map" : "cuTensorMapEncodeTiled failed", r);
  fcsa::DecodeArgs a;
  a.B = p->batch; a.H = p->heads; a.KVH = p->kv_heads; a.G = p->heads / p->kv_heads;
  a.Nq = p->seq_q; a.cap = p->seq_k; a.n_new = n_new;
  a.causal = p->causal ? 1 : 0;
  a.R = sh.R; a.n_rb = sh.n_rb; a.n_split = sh.n_split;
  const float log2e = 1.4426950408889634f;
  a.c1 = p->scale * log2e;
  a.c2 = p->shift * log2e;
  a.seqlens = seqlens;
  a.q = q->ptr; a.q_sb = q->sb; a.q_sh = q->sh; a.q_sn = q->sn;
  a.o = o->ptr; a.o_sb = o->sb; a.o_sh = o->sh; a.o_sn = o->sn;
  a.part = part;
  {
    cudaError_t e = fcsa::ensure_dynamic_smem<fcsa::fcsa_decode_kernel<T, D>>(Cfg::kSmem);
    if (e != cudaSuccess) return cuda_fail(e, "cudaFuncSetAttribute(decode)");
  }
  const long long grid = sh.items * sh.n_split;
  if (grid > 0x7FFFFFFFLL) return fail(FCSA_ERR_INVALID, "decode: problem too large for one launch");
  cudaError_t e = fcsa::launch_pdl(fcsa::fcsa_decode_kernel<T, D>, dim3((unsigned)grid), dim3(Cfg::kThreads),
                                   Cfg::kSmem, stream, tk, tv, a);
  if (e != cudaSuccess) return cuda_fail(e, "decode kernel launch");
  g_launches.fetch_add(1);
  if (sh.n_split == 1) return FCSA_OK;
  const long long threads = sh.items * 64 * (D / 4);
  e = fcsa::launch_pdl(fcsa::decode_combine_kernel<T, D>, dim3((unsigned)((threads + 255) / 256)), dim3(256), 0,
                       stream, a);
  if (e != cudaSuccess) return cuda_fail(e, "decode combine launch");
  g_launches.fetch_add(1);
  return FCSA_OK;
}

}  // namespace

extern "C" {

int fcsa_version(void) { return 300; }

const char* fcsa_last_error(void) { return g_err; }

int64_t fcsa_debug(void) { return g_launches.load(); }

int fcsa_set_kernel_events(int32_t which, void* start_event, void* stop_event) {
  if (which < 0 || which > 4)
    return fail(FCSA_ERR_INVALID, "which must be 0 (forward), 1 (backward), 2 (l2norm), 3 (preprocess) or 4 (dq finish)");
  g_ev[which][0] = reinterpret_cast<cudaEvent_t>(start_event);
  g_ev[which][1] = reinterpret_cast<cudaEvent_t>(stop_event);
  return FCSA_OK;
}

int fcsa_forward(const fcsa_problem* p, const fcsa_tensor* q, const fcsa_tensor* k,
                 const fcsa_tensor* v, const fcsa_tensor* o, float* inv_l, void* stream) {
  int r;
  if ((r = check_problem(p))) return r;
  if ((r = check_tensor(q, "q")) || (r = check_tensor(k, "k")) || (r = check_tensor(v, "v")) ||
      (r = check_tensor(o, "o")))
    return r;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (p->dtype == FCSA_BF16) {
    if (p->head_dim == 64) return launch_forward<__nv_bfloat16, 64>(p, q, k, v, o, inv_l, s);
    return launch_forward<__nv_bfloat16, 128>(p, q, k, v, o, inv_l, s);
  } else {
    if (p->head_dim == 64) return launch_forward<__half, 64>(p, q, k, v, o, inv_l, s);
    return launch_forward<__half, 128>(p, q, k, v, o, inv_l, s);
  }
}

int fcsa_forward_bias(const fcsa_problem* p, const fcsa_tensor* q, const fcsa_tensor* k,
                      const fcsa_tensor* v, const fcsa_bias* bias, const fcsa_tensor* o, float* inv_l,
                      void* stream) {
  int r;
  if ((r = check_problem(p))) return r;
  if ((r = check_tensor(q, "q")) || (r = check_tensor(k, "k")) || (r = check_tensor(v, "v")) ||
      (r = check_tensor(o, "o")) || (r = check_bias(p, bias)))
    return r;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (p->dtype == FCSA_BF16) {
    if (p->head_dim == 64) return launch_forward<__nv_bfloat16, 64, true>(p, q, k, v, o, inv_l, s, bias);
    return launch_forward<__nv_bfloat16, 128, true>(p, q, k, v, o, inv_l, s, bias);
  } else {
    if (p->head_dim == 64) return launch_forward<__half, 64, true>(p, q, k, v, o, inv_l, s, bias);
    return launch_forward<__half, 128, true>(p, q, k, v, o, inv_l, s, bias);
  }
}

size_t fcsa_backward_workspace_bytes(const fcsa_problem* p) {
  if (check_problem(p)) return 0;
  return fcsa::bwd_workspace_bytes(p->batch, p->heads, p->kv_heads, p->seq_q, p->seq_k, p->head_dim);
}

size_t fcsa_backward_zeroed_bytes(const fcsa_problem* p) {
  if (check_problem(p)) return 0;
  return fcsa::bwd_zeroed_workspace_bytes(p->batch, p->heads, p->kv_heads, p->seq_q, p->seq_k, p->head_dim);
}

int fcsa_zeroed_init(void* zeroed, size_t bytes, void* stream) {
  if (!zeroed || bytes == 0) return fail(FCSA_ERR_INVALID, "zeroed workspace: null / empty");
  cudaError_t e = cudaMemsetAsync(zeroed, 0, bytes, reinterpret_cast<cudaStream_t>(stream));
  if (e != cudaSuccess) return cuda_fail(e, "cudaMemsetAsync(zeroed workspace)");
  return FCSA_OK;
}

static int backward_impl(const fcsa_problem* p, const fcsa_tensor* q, const fcsa_tensor* k,
                         const fcsa_tensor* v, const fcsa_tensor* o, const fcsa_tensor* d_o,
                         const float* inv_l, const fcsa_tensor* dq, const fcsa_tensor* dk,
                         const fcsa_tensor* dv, void* workspace, size_t workspace_bytes, void* zeroed,
                         size_t zeroed_bytes, void* stream,
                         const float* q_rnorm, const float* k_rnorm, int groups,
                         const fcsa_bias* bias = nullptr, float* d_bias_acc = nullptr, int64_t dsb = 0,
                         int64_t dsh = 0) {
  int r;
  if ((r = check_problem(p))) return r;
  if (bias && (r = check_bias(p, bias))) return r;
  if ((r = check_tensor(q, "q")) || (r = check_tensor(k, "k")) || (r = check_tensor(v, "v")) ||
      (r = check_tensor(o, "o")) || (r = check_tensor(d_o, "d_o")) || (r = check_tensor(dq, "dq")) ||
      (r = check_tensor(dk, "dk")) || (r = check_tensor(dv, "dv")))
    return r;
  if (!inv_l) return fail(FCSA_ERR_INVALID, "inv_l: null");
  const size_t need = fcsa_backward_workspace_bytes(p);
  if (!workspace || workspace_bytes < need)
    return fail(FCSA_ERR_WORKSPACE, "workspace too small: need %zu bytes, got %zu", need, workspace_bytes);
  if (!aligned16(workspace)) return fail(FCSA_ERR_INVALID, "workspace not 16-byte aligned");
  const size_t zneed = fcsa_backward_zeroed_bytes(p);
  if (!zeroed || zeroed_bytes < zneed)
    return fail(FCSA_ERR_WORKSPACE, "zeroed workspace too small: need %zu bytes, got %zu", zneed, zeroed_bytes);
  if (!aligned16(zeroed)) return fail(FCSA_ERR_INVALID, "zeroed workspace not 16-byte aligned");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  fcsa::BwdHostArgs h;
  h.dtype_bf16 = p->dtype == FCSA_BF16;
  h.B = p->batch; h.H = p->heads; h.kv_heads = p->kv_heads; h.Nq = p->seq_q; h.Nk = p->seq_k;
  h.D = p->head_dim; h.causal = p->causal ? 1 : 0;
  h.scale = p->scale; h.shift = p->shift;
  h.mask = p->key_mask; h.mask_sb = p->key_mask_stride;
  h.q = *q; h.k = *k; h.v = *v; h.o = *o; h.d_o = *d_o; h.dq = *dq; h.dk = *dk; h.dv = *dv;
  h.inv_l = inv_l;
  h.out_f32 = p->out_f32 != 0;
  if (h.out_f32 && (q_rnorm || k_rnorm))
    return fail(FCSA_ERR_UNSUPPORTED, "out_f32 with the fused l2norm backward is not implemented (normalise outside)");
  h.workspace = workspace;
  h.zeroed = zeroed;
  h.ev_start = g_ev[1][0];
  h.ev_stop = g_ev[1][1];
  h.ev_prep[0] = g_ev[3][0]; h.ev_prep[1] = g_ev[3][1];
  h.ev_finish[0] = g_ev[4][0]; h.ev_finish[1] = g_ev[4][1];
  h.q_rnorm = q_rnorm;
  h.k_rnorm = k_rnorm;
  h.groups = groups;
  if (bias) {
    h.bias = bias->ptr; h.bias_sb = bias->sb; h.bias_sh = bias->sh; h.bias_sn = bias->sn;
    h.bias_amax = bias->amax;
    h.dbias = d_bias_acc; h.dbias_sb = dsb; h.dbias_sh = dsh;
  }
  int launches = 0;
  const char* err = nullptr;
  cudaError_t ce = cudaSuccess;
  r = fcsa::run_backward(h, s, &launches, &err, &ce);
  g_launches.fetch_add(launches);
  if (r == FCSA_ERR_CUDA) return fail(r, "%s: %s", err ? err : "backward", cudaGetErrorString(ce));
  if (r != FCSA_OK) return fail(r, "%s", err ? err : "backward failed");
  return FCSA_OK;
}

int fcsa_backward(const fcsa_problem* p, const fcsa_tensor* q, const fcsa_tensor* k,
                  const fcsa_tensor* v, const fcsa_tensor* o, const fcsa_tensor* d_o,
                  const float* inv_l, const fcsa_tensor* dq, const fcsa_tensor* dk,
                  const fcsa_tensor* dv, void* workspace, size_t workspace_bytes, void* zeroed,
                  size_t zeroed_bytes, void* stream) {
  return backward_impl(p, q, k, v, o, d_o, inv_l, dq, dk, dv, workspace, workspace_bytes, zeroed, zeroed_bytes,
                       stream, nullptr, nullptr, 1);
}

int fcsa_backward_bias(const fcsa_problem* p, const fcsa_tensor* q, const fcsa_tensor* k,
                       const fcsa_tensor* v, const fcsa_tensor* o, const fcsa_tensor* d_o,
                       const float* inv_l, const fcsa_bias* bias, float* d_bias_acc, int64_t dsb,
                       int64_t dsh, const fcsa_tensor* dq, const fcsa_tensor* dk, const fcsa_tensor* dv,
                       void* workspace, size_t workspace_bytes, void* zeroed, size_t zeroed_bytes, void* stream) {
  if (!bias) return fail(FCSA_ERR_INVALID, "attn_bias: null");
  return backward_impl(p, q, k, v, o, d_o, inv_l, dq, dk, dv, workspace, workspace_bytes, zeroed, zeroed_bytes,
                       stream, nullptr, nullptr, 1, bias, d_bias_acc, dsb, dsh);
}

int fcsa_forward_fused(const fcsa_problem* p, const fcsa_tensor* q, const fcsa_tensor* k,
                       const fcsa_tensor* v, const fcsa_l2norm* n, const fcsa_tensor* o, float* inv_l,
                       void* stream) {
  int r;
  if ((r = check_problem(p))) return r;
  if (!n) return fail(FCSA_ERR_INVALID, "null fcsa_l2norm");
  if ((r = check_rows(false, p->dtype, p->batch, p->heads, p->seq_q, p->head_dim, n->groups))) return r;
  if ((r = check_tensor(q, "q")) || (r = check_tensor(k, "k")) || (r = check_tensor(&n->q_hat, "q_hat")) ||
      (r = check_tensor(&n->k_hat, "k_hat")))
    return r;
  if (!n->q_rnorm || !n->k_rnorm) return fail(FCSA_ERR_INVALID, "q_rnorm / k_rnorm: null");
  fcsa::RowArgs a = row_args(p->batch, p->head_dim, n->groups);
  a.t[0] = {p->heads, p->seq_q, *q, n->q_hat, {}, n->q_rnorm};
  a.t[1] = {p->kv_heads, p->seq_k, *k, n->k_hat, {}, n->k_rnorm};
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (g_ev[2][0]) cudaEventRecord(g_ev[2][0], s);
  const cudaError_t e = fcsa::launch_row_fwd(a, p->dtype == FCSA_BF16, false, s);
  if (g_ev[2][1]) cudaEventRecord(g_ev[2][1], s);
  if ((r = row_pass_launched(e, "l2norm (q, k) launch"))) return r;
  return fcsa_forward(p, &n->q_hat, &n->k_hat, v, o, inv_l, stream);
}

int fcsa_backward_fused(const fcsa_problem* p, const fcsa_l2norm* n, const fcsa_tensor* v,
                        const fcsa_tensor* o, const fcsa_tensor* d_o, const float* inv_l,
                        const fcsa_tensor* dq, const fcsa_tensor* dk, const fcsa_tensor* dv,
                        void* workspace, size_t workspace_bytes, void* zeroed, size_t zeroed_bytes,
                        void* stream) {
  if (!n) return fail(FCSA_ERR_INVALID, "null fcsa_l2norm");
  int r;
  if ((r = check_problem(p))) return r;
  if ((r = check_rows(false, p->dtype, p->batch, p->heads, p->seq_q, p->head_dim, n->groups))) return r;
  if (!n->q_rnorm || !n->k_rnorm) return fail(FCSA_ERR_INVALID, "q_rnorm / k_rnorm: null");
  return backward_impl(p, &n->q_hat, &n->k_hat, v, o, d_o, inv_l, dq, dk, dv, workspace, workspace_bytes,
                       zeroed, zeroed_bytes, stream, n->q_rnorm, n->k_rnorm, n->groups);
}

int fcsa_f32_cast(int32_t dtype, int32_t batch, int32_t heads, int32_t rows, int32_t head_dim, int32_t groups,
                  const fcsa_tensor* x, const fcsa_tensor* y, float* rnorm, const float* mul, int32_t mul_reciprocal,
                  void* stream) {
  int r;
  if ((r = check_rows(true, dtype, batch, heads, rows, head_dim, groups))) return r;
  if (!x || !x->ptr || !y) return fail(FCSA_ERR_INVALID, "f32 cast: null tensor");
  if (!f32_rows(x)) return fail(FCSA_ERR_INVALID, "f32 cast: float32 rows must be 16-byte aligned");
  if ((r = check_tensor(y, "y"))) return r;
  if (groups > 0 && !rnorm) return fail(FCSA_ERR_INVALID, "f32 cast: rnorm is null");
  fcsa::RowArgs a = row_args(batch, head_dim, groups, mul, mul_reciprocal);
  a.t[0] = {heads, rows, *x, *y, {}, rnorm};
  return row_pass_launched(fcsa::launch_row_fwd(a, dtype == FCSA_BF16, true, reinterpret_cast<cudaStream_t>(stream)),
                           "f32 cast launch");
}

int fcsa_f32_cast_backward(int32_t dtype, int32_t batch, int32_t heads, int32_t rows, int32_t head_dim,
                           int32_t groups, const fcsa_tensor* dy, const fcsa_tensor* y, const float* rnorm,
                           const fcsa_tensor* dx, const float* mul, int32_t mul_reciprocal, void* stream) {
  int r;
  if ((r = check_rows(true, dtype, batch, heads, rows, head_dim, groups))) return r;
  if (!dy || !dy->ptr || (groups > 0 && !y)) return fail(FCSA_ERR_INVALID, "f32 cast: null tensor");
  if (!f32_rows(dy)) return fail(FCSA_ERR_INVALID, "f32 cast: float32 rows must be 16-byte aligned");
  if (groups > 0 && (r = check_tensor(y, "y"))) return r;
  if (groups > 0 && !rnorm) return fail(FCSA_ERR_INVALID, "f32 cast backward: rnorm is null");
  if (!f32_rows(dx)) return fail(FCSA_ERR_INVALID, "f32 cast backward: dx rows must be 16-byte aligned float32");
  fcsa::RowArgs a = row_args(batch, head_dim, groups, mul, mul_reciprocal);
  a.t[0] = {heads, rows, *dy, groups > 0 ? *y : fcsa_tensor{}, *dx, const_cast<float*>(rnorm)};
  return row_pass_launched(fcsa::launch_row_bwd(a, dtype == FCSA_BF16, true, reinterpret_cast<cudaStream_t>(stream)),
                           "f32 cast backward launch");
}

int fcsa_l2norm_forward(int32_t dtype, int32_t batch, int32_t heads, int32_t rows, int32_t head_dim,
                        int32_t groups, const fcsa_tensor* x, const fcsa_tensor* y, float* rnorm,
                        void* stream) {
  int r;
  if ((r = check_rows(false, dtype, batch, heads, rows, head_dim, groups))) return r;
  if ((r = check_tensor(x, "x")) || (r = check_tensor(y, "y"))) return r;
  fcsa::RowArgs a = row_args(batch, head_dim, groups);
  a.t[0] = {heads, rows, *x, *y, {}, rnorm};
  return row_pass_launched(fcsa::launch_row_fwd(a, dtype == FCSA_BF16, false, reinterpret_cast<cudaStream_t>(stream)),
                           "l2norm forward launch");
}

int fcsa_l2norm_backward(int32_t dtype, int32_t batch, int32_t heads, int32_t rows,
                         int32_t head_dim, int32_t groups, const fcsa_tensor* dy,
                         const fcsa_tensor* y, const float* rnorm, const fcsa_tensor* dx,
                         void* stream) {
  int r;
  if ((r = check_rows(false, dtype, batch, heads, rows, head_dim, groups))) return r;
  if ((r = check_tensor(dy, "dy")) || (r = check_tensor(y, "y")) || (r = check_tensor(dx, "dx")))
    return r;
  if (!rnorm) return fail(FCSA_ERR_INVALID, "rnorm: null");
  fcsa::RowArgs a = row_args(batch, head_dim, groups);
  a.t[0] = {heads, rows, *dy, *y, *dx, const_cast<float*>(rnorm)};
  return row_pass_launched(fcsa::launch_row_bwd(a, dtype == FCSA_BF16, false, reinterpret_cast<cudaStream_t>(stream)),
                           "l2norm backward launch");
}

size_t fcsa_decode_workspace_bytes(const fcsa_problem* p, int32_t n_new) {
  DecodeShape sh;
  if (check_decode_problem(p, n_new) || decode_shape(p, &sh)) return 0;
  return decode_qhat_bytes(p) + fcsa::decode_partial_bytes(sh.items, sh.n_split, p->head_dim);
}

int fcsa_decode(const fcsa_problem* p, const fcsa_tensor* q, const fcsa_tensor* k_cache, const fcsa_tensor* v_cache,
                const int32_t* cache_seqlens, const fcsa_tensor* k_new, const fcsa_tensor* v_new, int32_t n_new,
                int32_t groups, const fcsa_tensor* o, void* workspace, size_t workspace_bytes, void* stream) {
  int r;
  if ((r = check_decode_problem(p, n_new))) return r;
  if ((r = check_tensor(q, "q")) || (r = check_tensor(k_cache, "k_cache")) || (r = check_tensor(v_cache, "v_cache")) ||
      (r = check_tensor(o, "o")))
    return r;
  if (n_new > 0 && ((r = check_tensor(k_new, "k")) || (r = check_tensor(v_new, "v")))) return r;
  if (groups != 0 && (r = check_rows(false, p->dtype, p->batch, p->heads, p->seq_q, p->head_dim, groups))) return r;
  if (!cache_seqlens) return fail(FCSA_ERR_INVALID, "cache_seqlens: null");
  DecodeShape sh;
  if ((r = decode_shape(p, &sh))) return r;
  const size_t qbytes = decode_qhat_bytes(p);
  const size_t need = qbytes + fcsa::decode_partial_bytes(sh.items, sh.n_split, p->head_dim);
  if (!workspace || workspace_bytes < need)
    return fail(FCSA_ERR_WORKSPACE, "workspace too small: need %zu bytes, got %zu", need, workspace_bytes);
  if (!aligned16(workspace)) return fail(FCSA_ERR_INVALID, "workspace not 16-byte aligned");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);

  // append pass: q_hat to the workspace (groups > 0), then k (normalised when groups > 0) and v into the caches at
  // row cache_seqlens[b]
  const int64_t H = p->heads, N = p->seq_q, D = p->head_dim;
  const fcsa_tensor qhat = {workspace, H * N * D, N * D, D};
  fcsa::RowArgs a = row_args(p->batch, p->head_dim, groups);
  int n = 0;
  if (groups > 0) a.t[n++] = {p->heads, p->seq_q, *q, qhat, {}, nullptr, nullptr, p->seq_q, 0};
  if (n_new > 0) {
    a.t[n++] = {p->kv_heads, n_new, *k_new, *k_cache, {}, nullptr, cache_seqlens, p->seq_k, groups == 0 ? 1 : 0};
    a.t[n++] = {p->kv_heads, n_new, *v_new, *v_cache, {}, nullptr, cache_seqlens, p->seq_k, 1};
  }
  if (n > 0 && (r = row_pass_launched(fcsa::launch_row_append(a, n, p->dtype == FCSA_BF16, s), "append pass launch")))
    return r;

  const fcsa_tensor* qa = groups > 0 ? &qhat : q;
  float* part = reinterpret_cast<float*>(static_cast<char*>(workspace) + qbytes);
  if (p->dtype == FCSA_BF16) {
    if (p->head_dim == 64) return launch_decode<__nv_bfloat16, 64>(p, sh, qa, k_cache, v_cache, cache_seqlens, n_new, o, part, s);
    return launch_decode<__nv_bfloat16, 128>(p, sh, qa, k_cache, v_cache, cache_seqlens, n_new, o, part, s);
  }
  if (p->head_dim == 64) return launch_decode<__half, 64>(p, sh, qa, k_cache, v_cache, cache_seqlens, n_new, o, part, s);
  return launch_decode<__half, 128>(p, sh, qa, k_cache, v_cache, cache_seqlens, n_new, o, part, s);
}

}  // extern "C"
