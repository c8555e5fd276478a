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

template <typename T>
int launch_l2norm_fwd(const fcsa::L2Args& a, cudaStream_t stream) {
  const int tpr = a.D / 8;
  const int rows_per_block = 256 / tpr;
  const long long rows = (long long)a.B * a.H * a.N;
  const long long grid = (rows + rows_per_block - 1) / rows_per_block;
  fcsa::l2norm_fwd_kernel<T><<<(unsigned)grid, 256, 0, stream>>>(a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "l2norm forward launch");
  g_launches.fetch_add(1);
  return FCSA_OK;
}
template <typename T>
int launch_l2norm_bwd(const fcsa::L2Args& a, cudaStream_t stream) {
  const int tpr = a.D / 8;
  const int rows_per_block = 256 / tpr;
  const long long rows = (long long)a.B * a.H * a.N;
  const long long grid = (rows + rows_per_block - 1) / rows_per_block;
  fcsa::l2norm_bwd_kernel<T><<<(unsigned)grid, 256, 0, stream>>>(a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "l2norm backward launch");
  g_launches.fetch_add(1);
  return FCSA_OK;
}

int check_l2(int32_t dtype, int32_t B, int32_t H, int32_t N, int32_t D, int32_t G) {
  if (dtype != FCSA_F16 && dtype != FCSA_BF16)
    return fail(FCSA_ERR_UNSUPPORTED, "l2norm: dtype %d not implemented", dtype);
  if (B <= 0 || H <= 0 || N <= 0) return fail(FCSA_ERR_INVALID, "l2norm: empty tensor");
  if (D != 32 && D != 64 && D != 128 && D != 256)
    return fail(FCSA_ERR_UNSUPPORTED, "l2norm: head_dim %d not implemented", D);
  if (G <= 0 || D % G != 0) return fail(FCSA_ERR_INVALID, "l2norm: groups %d does not divide %d", G, D);
  const int gs = D / G;
  if ((gs & (gs - 1)) != 0) return fail(FCSA_ERR_UNSUPPORTED, "l2norm: group size %d must be a power of two", gs);
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
  if ((r = check_l2(p->dtype, p->batch, p->heads, p->seq_q, p->head_dim, n->groups))) return r;
  if ((r = check_tensor(q, "q")) || (r = check_tensor(k, "k")) || (r = check_tensor(&n->q_hat, "q_hat")) ||
      (r = check_tensor(&n->k_hat, "k_hat")))
    return r;
  if (!n->q_rnorm || !n->k_rnorm) return fail(FCSA_ERR_INVALID, "q_rnorm / k_rnorm: null");
  fcsa::L2PairArgs pa;
  memset(&pa, 0, sizeof(pa));
  const fcsa_tensor* src[2] = {q, k};
  const fcsa_tensor* dst[2] = {&n->q_hat, &n->k_hat};
  float* rn[2] = {n->q_rnorm, n->k_rnorm};
  const int heads[2] = {p->heads, p->kv_heads};
  const int rows[2] = {p->seq_q, p->seq_k};
  int max_rows = 0;
  for (int t = 0; t < 2; ++t) {
    fcsa::L2Args& a = pa.t[t];
    a.B = p->batch; a.H = heads[t]; a.N = rows[t]; a.D = p->head_dim; a.G = n->groups;
    a.x_sb = src[t]->sb; a.x_sh = src[t]->sh; a.x_sn = src[t]->sn;
    a.y_sb = dst[t]->sb; a.y_sh = dst[t]->sh; a.y_sn = dst[t]->sn;
    a.x = src[t]->ptr; a.y = dst[t]->ptr; a.rnorm = rn[t];
    if (a.N > max_rows) max_rows = a.N;
  }
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  constexpr int U = 2;                                       // rows per thread (16 features each)
  const int rows_per_block = U * (256 / (p->head_dim / 16));
  const long long bhs = (long long)pa.t[0].B * pa.t[0].H + (long long)pa.t[1].B * pa.t[1].H;
  if (bhs > 65535) {
    // more (batch, head) pairs than grid.y holds (merged batch-heads layouts): one 1-D-grid launch per tensor
    const bool bf16 = p->dtype == FCSA_BF16;
    for (int t = 0; t < 2; ++t)
      if ((r = bf16 ? launch_l2norm_fwd<__nv_bfloat16>(pa.t[t], s) : launch_l2norm_fwd<__half>(pa.t[t], s))) return r;
    return fcsa_forward(p, &n->q_hat, &n->k_hat, v, o, inv_l, stream);
  }
  dim3 grid((unsigned)((max_rows + rows_per_block - 1) / rows_per_block), (unsigned)bhs);
  cudaError_t e;
  const bool bf = p->dtype == FCSA_BF16;
  if (g_ev[2][0]) cudaEventRecord(g_ev[2][0], s);
  if (p->head_dim == 64)
    e = bf ? fcsa::launch_pdl(fcsa::l2norm_fwd_pair_kernel<__nv_bfloat16, 4, U>, grid, dim3(256), 0, s, pa)
           : fcsa::launch_pdl(fcsa::l2norm_fwd_pair_kernel<__half, 4, U>, grid, dim3(256), 0, s, pa);
  else if (p->head_dim == 128)
    e = bf ? fcsa::launch_pdl(fcsa::l2norm_fwd_pair_kernel<__nv_bfloat16, 8, U>, grid, dim3(256), 0, s, pa)
           : fcsa::launch_pdl(fcsa::l2norm_fwd_pair_kernel<__half, 8, U>, grid, dim3(256), 0, s, pa);
  else
    e = bf ? fcsa::launch_pdl(fcsa::l2norm_fwd_pair_kernel<__nv_bfloat16, 0, U>, grid, dim3(256), 0, s, pa)
           : fcsa::launch_pdl(fcsa::l2norm_fwd_pair_kernel<__half, 0, U>, grid, dim3(256), 0, s, pa);
  if (g_ev[2][1]) cudaEventRecord(g_ev[2][1], s);
  if (e != cudaSuccess) return cuda_fail(e, "l2norm (q, k) launch");
  g_launches.fetch_add(1);
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
  if ((r = check_l2(p->dtype, p->batch, p->heads, p->seq_q, p->head_dim, n->groups))) return r;
  if (!n->q_rnorm || !n->k_rnorm) return fail(FCSA_ERR_INVALID, "q_rnorm / k_rnorm: null");
  return backward_impl(p, &n->q_hat, &n->k_hat, v, o, d_o, inv_l, dq, dk, dv, workspace, workspace_bytes,
                       zeroed, zeroed_bytes, stream, n->q_rnorm, n->k_rnorm, n->groups);
}

static int f32_cast_common(fcsa::F32CastArgs& a, int32_t dtype, int32_t B, int32_t H, int32_t N, int32_t D, int32_t G,
                           const fcsa_tensor* x, const fcsa_tensor* y) {
  if (dtype != FCSA_F16 && dtype != FCSA_BF16) return fail(FCSA_ERR_UNSUPPORTED, "f32 cast: 16-bit dtype %d not implemented", dtype);
  if (B <= 0 || H <= 0 || N <= 0) return fail(FCSA_ERR_INVALID, "f32 cast: empty tensor");
  if (D != 16 && D != 32 && D != 64 && D != 128) return fail(FCSA_ERR_UNSUPPORTED, "f32 cast: head_dim %d not implemented", D);
  if (G < 0 || (G > 0 && (D % G != 0 || ((D / G) & (D / G - 1)) != 0)))
    return fail(FCSA_ERR_INVALID, "f32 cast: groups %d must divide %d into power-of-two chunks", G, D);
  if (!x || !x->ptr || !y) return fail(FCSA_ERR_INVALID, "f32 cast: null tensor");
  if ((reinterpret_cast<uintptr_t>(x->ptr) & 15u) || (x->sb % 4) || (x->sh % 4) || (x->sn % 4))
    return fail(FCSA_ERR_INVALID, "f32 cast: float32 rows must be 16-byte aligned");
  memset(&a, 0, sizeof(a));
  a.B = B; a.H = H; a.N = N; a.D = D; a.G = G;
  a.x = reinterpret_cast<const float*>(x->ptr); a.x_sb = x->sb; a.x_sh = x->sh; a.x_sn = x->sn;
  a.y = y->ptr; a.y_sb = y->sb; a.y_sh = y->sh; a.y_sn = y->sn;
  return FCSA_OK;
}

int fcsa_f32_cast(int32_t dtype, int32_t batch, int32_t heads, int32_t rows, int32_t head_dim, int32_t groups,
                  const fcsa_tensor* x, const fcsa_tensor* y, float* rnorm, const float* mul, int32_t mul_reciprocal,
                  void* stream) {
  fcsa::F32CastArgs a;
  int r;
  if ((r = f32_cast_common(a, dtype, batch, heads, rows, head_dim, groups, x, y))) return r;
  if ((r = check_tensor(y, "y"))) return r;
  if (groups > 0 && !rnorm) return fail(FCSA_ERR_INVALID, "f32 cast: rnorm is null");
  a.rnorm = rnorm; a.mul = mul; a.mul_reciprocal = mul_reciprocal;
  const int rpb = 256 / (head_dim / 8);
  const long long total = (long long)batch * heads * rows;
  const unsigned grid = (unsigned)((total + rpb - 1) / rpb);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (dtype == FCSA_BF16) fcsa::f32_cast_kernel<__nv_bfloat16><<<grid, 256, 0, s>>>(a);
  else fcsa::f32_cast_kernel<__half><<<grid, 256, 0, s>>>(a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "f32 cast launch");
  g_launches.fetch_add(1);
  return FCSA_OK;
}

int fcsa_f32_cast_backward(int32_t dtype, int32_t batch, int32_t heads, int32_t rows, int32_t head_dim,
                           int32_t groups, const fcsa_tensor* dy, const fcsa_tensor* y, const float* rnorm,
                           const fcsa_tensor* dx, const float* mul, int32_t mul_reciprocal, void* stream) {
  fcsa::F32CastArgs a;
  int r;
  fcsa_tensor ynull = {nullptr, 0, 0, 0};
  if ((r = f32_cast_common(a, dtype, batch, heads, rows, head_dim, groups, dy, groups > 0 ? y : &ynull))) return r;
  if (groups > 0 && ((r = check_tensor(y, "y")) || !rnorm)) return r ? r : fail(FCSA_ERR_INVALID, "f32 cast backward: rnorm is null");
  if (!dx || !dx->ptr || (reinterpret_cast<uintptr_t>(dx->ptr) & 15u) || (dx->sb % 4) || (dx->sh % 4) || (dx->sn % 4))
    return fail(FCSA_ERR_INVALID, "f32 cast backward: dx rows must be 16-byte aligned float32");
  a.dx = reinterpret_cast<float*>(dx->ptr); a.o_sb = dx->sb; a.o_sh = dx->sh; a.o_sn = dx->sn;
  a.rnorm = const_cast<float*>(rnorm); a.mul = mul; a.mul_reciprocal = mul_reciprocal;
  const int rpb = 256 / (head_dim / 8);
  const long long total = (long long)batch * heads * rows;
  const unsigned grid = (unsigned)((total + rpb - 1) / rpb);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (dtype == FCSA_BF16) fcsa::f32_cast_bwd_kernel<__nv_bfloat16><<<grid, 256, 0, s>>>(a);
  else fcsa::f32_cast_bwd_kernel<__half><<<grid, 256, 0, s>>>(a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cuda_fail(e, "f32 cast backward launch");
  g_launches.fetch_add(1);
  return FCSA_OK;
}

int fcsa_l2norm_forward(int32_t dtype, int32_t batch, int32_t heads, int32_t rows, int32_t head_dim,
                        int32_t groups, const fcsa_tensor* x, const fcsa_tensor* y, float* rnorm,
                        void* stream) {
  int r;
  if ((r = check_l2(dtype, batch, heads, rows, head_dim, groups))) return r;
  if ((r = check_tensor(x, "x")) || (r = check_tensor(y, "y"))) return r;
  fcsa::L2Args a;
  memset(&a, 0, sizeof(a));
  a.B = batch; a.H = heads; a.N = rows; a.D = head_dim; a.G = groups;
  a.x_sb = x->sb; a.x_sh = x->sh; a.x_sn = x->sn;
  a.y_sb = y->sb; a.y_sh = y->sh; a.y_sn = y->sn;
  a.x = x->ptr; a.y = y->ptr; a.rnorm = rnorm;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  return dtype == FCSA_BF16 ? launch_l2norm_fwd<__nv_bfloat16>(a, s) : launch_l2norm_fwd<__half>(a, s);
}

int fcsa_l2norm_backward(int32_t dtype, int32_t batch, int32_t heads, int32_t rows,
                         int32_t head_dim, int32_t groups, const fcsa_tensor* dy,
                         const fcsa_tensor* y, const float* rnorm, const fcsa_tensor* dx,
                         void* stream) {
  int r;
  if ((r = check_l2(dtype, batch, heads, rows, head_dim, groups))) return r;
  if ((r = check_tensor(dy, "dy")) || (r = check_tensor(y, "y")) || (r = check_tensor(dx, "dx")))
    return r;
  if (!rnorm) return fail(FCSA_ERR_INVALID, "rnorm: null");
  fcsa::L2Args a;
  memset(&a, 0, sizeof(a));
  a.B = batch; a.H = heads; a.N = rows; a.D = head_dim; a.G = groups;
  a.x_sb = dy->sb; a.x_sh = dy->sh; a.x_sn = dy->sn;
  a.y_sb = y->sb; a.y_sh = y->sh; a.y_sn = y->sn;
  a.o_sb = dx->sb; a.o_sh = dx->sh; a.o_sn = dx->sn;
  a.x = dy->ptr; a.y = y->ptr; a.dx = dx->ptr; a.rnorm = const_cast<float*>(rnorm);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  return dtype == FCSA_BF16 ? launch_l2norm_bwd<__nv_bfloat16>(a, s) : launch_l2norm_bwd<__half>(a, s);
}

}  // extern "C"
