// Host side of libfcsa_b200.so: argument validation, TMA tensor-map construction, the
// {f16, bf16} x {64, 128} dispatch and the forward, decode, backward and row-pass launches behind
// the C ABI of include/fcsa_b200.h.
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
#include <type_traits>

#include "../../include/fcsa_b200.h"
#include "bwd_kernel.cuh"
#include "decode_kernel.cuh"
#include "dq_kernel.cuh"
#include "fwd_kernel.cuh"
#include "l2norm_kernels.cuh"
#include "tensor_map.h"

namespace {

thread_local char g_err[512] = "";
cudaEvent_t g_ev[5][2] = {};   // 0 forward, 1 backward, 2 l2norm(q,k), 3 backward preprocess, 4 dq finish / dQ kernel
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
  if (p->window < 0) return fail(FCSA_ERR_INVALID, "window %d < 0 (0 = no window)", p->window);
  return FCSA_OK;
}

// The window the kernels apply: 0 (the unwindowed kernels) when there is none, or when it is at least seq_q + seq_k and
// so hides no key (seq_q / seq_k bound every length the problem covers: varlen maxima, the decode capacity).
int kernel_window(const fcsa_problem* p) {
  return (long long)p->window >= (long long)p->seq_q + p->seq_k ? 0 : p->window;
}

int check_bias(const fcsa_problem* p, const fcsa_bias* bias) {
  if (!bias || !bias->ptr) return fail(FCSA_ERR_INVALID, "attn_bias: null");
  if (p->window != 0) return fail(FCSA_ERR_INVALID, "attn_bias: no sliding window with a bias (window %d)", p->window);
  if (!aligned16(bias->ptr) || (bias->sn % 8) != 0 || (bias->sh % 8) != 0 || (bias->sb % 8) != 0)
    return fail(FCSA_ERR_INVALID, "attn_bias: rows must be 16-byte aligned (strides multiples of 8 elements)");
  if (bias->sn < ((p->seq_k + 7) / 8) * 8)
    return fail(FCSA_ERR_INVALID, "attn_bias: row stride %lld shorter than seq_k rounded up to 8", (long long)bias->sn);
  return FCSA_OK;
}

template <typename T>
struct type_tag {
  using type = T;
};

// Calls f(type_tag<T>{}, std::integral_constant<int, D>{}) with the element type and head dim of a checked problem:
// the one place where the host code turns (dtype, head_dim) into template arguments.
template <typename F>
int dispatch(const fcsa_problem* p, F&& f) {
  using D64 = std::integral_constant<int, 64>;
  using D128 = std::integral_constant<int, 128>;
  if (p->dtype == FCSA_BF16)
    return p->head_dim == 64 ? f(type_tag<__nv_bfloat16>{}, D64{}) : f(type_tag<__nv_bfloat16>{}, D128{});
  return p->head_dim == 64 ? f(type_tag<__half>{}, D64{}) : f(type_tag<__half>{}, D128{});
}

// The TMA map of a [b][h][n][D] operand of element type T (boxes of box_rows rows x 64 features).  A failure names
// the operand.
template <typename T, int D>
int map_operand(CUtensorMap* tm, const char* name, const fcsa_tensor& t, int64_t B, int64_t H, int64_t N, int box_rows) {
  const int r = fcsa::make_tensor_map_bhnd(tm, t.ptr, fcsa::tma_dtype16(std::is_same<T, __nv_bfloat16>::value), B, H,
                                           N, D, t.sb, t.sh, t.sn, box_rows);
  if (r == -2)
    return fail(FCSA_ERR_INVALID, "%s: expanded (stride-0) views of extent > 1 cannot be addressed by a tensor map - "
                "make the tensor contiguous (%d)", name, r);
  if (r) return fail(FCSA_ERR_CUDA, "%s: cuTensorMapEncodeTiled failed (%d)", name, r);
  return FCSA_OK;
}

// error and launch count of one launch
int launched(cudaError_t e, const char* what) {
  if (e != cudaSuccess) return cuda_fail(e, what);
  g_launches.fetch_add(1);
  return FCSA_OK;
}

// launch() between the events ev[0] / ev[1] of fcsa_set_kernel_events when they are set (ev = nullptr: untimed)
template <typename L>
cudaError_t timed(const cudaEvent_t* ev, cudaStream_t stream, L&& launch) {
  if (ev && ev[0]) cudaEventRecord(ev[0], stream);
  const cudaError_t e = launch();
  if (ev && ev[1]) cudaEventRecord(ev[1], stream);
  return e;
}

// A kernel as a type, so that a site can pick one of several variants and pass it to a single launch
template <auto Kern>
using kernel_c = std::integral_constant<decltype(Kern), Kern>;

// Launch of an attention kernel: its dynamic shared memory set once per (kernel, device), then a timed PDL launch.
// A kernel whose parameter is the base of `args`' window arguments (the unwindowed variants) receives that base.
template <auto Kern, typename... Args>
int launch_attention(const char* what, const cudaEvent_t* ev, long long grid, int threads, int smem,
                     cudaStream_t stream, const Args&... args) {
  cudaError_t e = fcsa::ensure_dynamic_smem<Kern>(smem);
  if (e != cudaSuccess) return fail(FCSA_ERR_CUDA, "cudaFuncSetAttribute(%s): %s", what, cudaGetErrorString(e));
  e = timed(ev, stream,
            [&] { return fcsa::launch_pdl(Kern, dim3((unsigned)grid), dim3(threads), smem, stream, args...); });
  if (e != cudaSuccess) return fail(FCSA_ERR_CUDA, "%s kernel launch: %s", what, cudaGetErrorString(e));
  g_launches.fetch_add(1);
  return FCSA_OK;
}

// VARLEN: packed sequences (vl); q, k, v, o are then one batch of total_q / total_k rows
template <typename T, int D, bool BIAS = false, bool VARLEN = false>
int launch_forward(const fcsa_problem* p, const fcsa_tensor* q, const fcsa_tensor* k,
                   const fcsa_tensor* v, const fcsa_tensor* o, float* inv_l, cudaStream_t stream,
                   const fcsa_bias* bias = nullptr, const fcsa_varlen* vl = nullptr) {
  using Cfg = fcsa::FwdCfg<D>;
  const int tB = VARLEN ? 1 : p->batch, tNq = VARLEN ? vl->total_q : p->seq_q, tNk = VARLEN ? vl->total_k : p->seq_k;
  CUtensorMap tq, tk, tv;
  int r;
  if ((r = map_operand<T, D>(&tq, "q", *q, tB, p->heads, tNq, Cfg::kBlockM)) ||   // Q: one box of the CTA's query rows
      (r = map_operand<T, D>(&tk, "k", *k, tB, p->kv_heads, tNk, 128)) ||
      (r = map_operand<T, D>(&tv, "v", *v, tB, p->kv_heads, tNk, 128)))
    return r;

  // (the window's arguments extend the kernel's)
  fcsa::ArgsOf<fcsa::FwdArgs, fcsa::FwdVarlenArgs, VARLEN, true> a;
  a.window = kernel_window(p);
  if constexpr (VARLEN) {
    a.cu_q = vl->cu_seqlens_q; a.cu_k = vl->cu_seqlens_k; a.total_q = vl->total_q; a.total_k = vl->total_k;
  }
  a.B = p->batch;
  a.H = p->heads;
  a.Nq = p->seq_q;
  a.Nk = p->seq_k;
  a.causal = p->causal ? 1 : 0;
  a.has_mask = p->key_mask ? 1 : 0;
  a.group = p->heads / p->kv_heads;
  a.n_qblk = fcsa::row_blocks(p->seq_q, Cfg::kBlockM);
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

  // one CTA per (query block of kBlockM rows, batch, head); packed sequences: blocks of the longest sequence
  const long long grid = (long long)a.n_qblk * p->batch * p->heads;
  if (grid > 0x7FFFFFFFLL) return fail(FCSA_ERR_INVALID, "problem too large for one launch");
  const auto launch = [&](auto kern) {
    return launch_attention<decltype(kern)::value>("forward", g_ev[0], grid, Cfg::kThreads, Cfg::kSmem, stream, tq, tk,
                                                   tv, a);
  };
  if constexpr (BIAS)   // (a bias takes no window)
    return launch(kernel_c<fcsa::fcsa_fwd_kernel<T, D, true>>{});
  else
    return a.window > 0 ? launch(kernel_c<fcsa::fcsa_fwd_kernel<T, D, false, VARLEN, true>>{})
                        : launch(kernel_c<fcsa::fcsa_fwd_kernel<T, D, false, VARLEN>>{});
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

// The fused l2norm n of a checked problem over rows_batch x rows_n query rows (packed sequences: 1 x total_q): its
// groups and rnorms.  The forward's pre-pass (prepass) also checks its inputs q, k and the q^, k^ it writes.
int check_l2norm(const fcsa_problem* p, const fcsa_l2norm* n, int32_t rows_batch, int32_t rows_n, bool prepass = false,
                 const fcsa_tensor* q = nullptr, const fcsa_tensor* k = nullptr) {
  int r;
  if ((r = check_rows(false, p->dtype, rows_batch, p->heads, rows_n, p->head_dim, n->groups))) return r;
  if (prepass && ((r = check_tensor(q, "q")) || (r = check_tensor(k, "k")) || (r = check_tensor(&n->q_hat, "q_hat")) ||
                  (r = check_tensor(&n->k_hat, "k_hat"))))
    return r;
  if (!n->q_rnorm || !n->k_rnorm) return fail(FCSA_ERR_INVALID, "q_rnorm / k_rnorm: null");
  return FCSA_OK;
}

// The q / k l2norm pre-pass of the fused forwards: q^, k^ and their rnorms over B batches of Nq query and Nk key rows
// (packed sequences: one batch of total_q / total_k)
int l2norm_qk(const fcsa_problem* p, const fcsa_l2norm* n, const fcsa_tensor* q, const fcsa_tensor* k, int32_t B,
              int32_t Nq, int32_t Nk, cudaStream_t s) {
  int r;
  if ((r = check_l2norm(p, n, B, Nq, true, q, k))) return r;
  fcsa::RowArgs a = row_args(B, p->head_dim, n->groups);
  a.t[0] = {p->heads, Nq, *q, n->q_hat, {}, n->q_rnorm};
  a.t[1] = {p->kv_heads, Nk, *k, n->k_hat, {}, n->k_rnorm};
  return launched(timed(g_ev[2], s, [&] { return fcsa::launch_row_fwd(a, p->dtype == FCSA_BF16, false, s); }),
                  "l2norm (q, k) launch");
}

// ---- key/value-cache decode --------------------------------------------------------------------
// A decode call (fcsa_decode, fcsa_decode_varlen, fcsa_decode_rolling): seq_q = new queries (packed: the longest
// sequence's), seq_k = cache capacity.
struct DecodeCall {
  const char* who;        // the route's message prefix
  bool packed;            // total_q new rows, sequence b owning [cu[b], cu[b + 1]); dense: batch x seq_q
  const int32_t* cu;
  int32_t total_q;
  int32_t n_new;          // fcsa_decode: rows appended per sequence; the other routes append when k_new, v_new are set
  bool ring;              // rolling caches of seq_k rows
};

// The checks of decode call c, in the order the routes report them.  A workspace-size query (query = true) has no
// cu_seqlens_q or k_new / v_new to check.
int check_decode(const fcsa_problem* p, const DecodeCall& c, bool query, const fcsa_tensor* k_new = nullptr,
                 const fcsa_tensor* v_new = nullptr) {
  if (c.packed && p && p->seq_q < 0)
    return fail(FCSA_ERR_INVALID, "decode varlen: max_seqlen_q (seq_q) %d < 0", p->seq_q);
  int r;
  if ((r = check_problem(p))) return r;
  if (p->key_mask) return fail(FCSA_ERR_UNSUPPORTED, "decode: no key mask (cache_seqlens gives the valid rows)");
  if (p->out_f32) return fail(FCSA_ERR_UNSUPPORTED, "decode: out_f32 is not implemented");
  if (c.n_new < 0) return fail(FCSA_ERR_INVALID, "decode: n_new %d < 0", c.n_new);
  if ((long long)(p->heads / p->kv_heads) * p->seq_q > 0x7FFFFFFFLL - 64)
    return fail(FCSA_ERR_INVALID, "decode: heads per kv head x seq_q too large");
  if (c.packed && c.total_q < 0) return fail(FCSA_ERR_INVALID, "decode varlen: total_q %d < 0", c.total_q);
  // A rolling cache of C = seq_k rows needs a window, whole 128-row tiles (a tile never straddles the wrap), and
  // C >= W + seq_q - 1, so that the keys a call sees, [T_b - seq_q - W + 1, T_b), are not overwritten by its own
  // append.
  if (c.ring && p->window <= 0) return fail(FCSA_ERR_INVALID, "decode rolling: a rolling cache needs a window");
  if (c.ring && p->seq_k % 128 != 0)
    return fail(FCSA_ERR_INVALID, "decode rolling: cache rows %d must be a multiple of 128", p->seq_k);
  if (c.ring && (long long)p->seq_k < (long long)p->window + p->seq_q - 1)
    return fail(FCSA_ERR_INVALID, "decode rolling: cache rows %d < window %d + new queries %d - 1", p->seq_k,
                p->window, p->seq_q);
  if (query) return FCSA_OK;
  if (c.packed && !c.cu) return fail(FCSA_ERR_INVALID, "%snull cu_seqlens_q", c.who);
  if (reinterpret_cast<uintptr_t>(c.cu) & 3)
    return fail(FCSA_ERR_INVALID, "%scu_seqlens_q must be a 4-byte aligned int32 array", c.who);
  if ((c.packed || c.ring) && (k_new == nullptr) != (v_new == nullptr))
    return fail(FCSA_ERR_INVALID, "%spass both k_new and v_new, or neither", c.who);
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
  s->n_rb = fcsa::row_blocks(s->R, 64);
  s->items = (long long)p->batch * p->kv_heads * s->n_rb;
  const int w = kernel_window(p);
  s->n_split = fcsa::decode_split(s->items, w > 0 ? fcsa::decode_window_keys(p->seq_k, w, p->causal != 0) : p->seq_k, sms);
  return FCSA_OK;
}

size_t align16(size_t n) { return (n + 15) & ~size_t(15); }

// The scratch of decode call c: q^ of its query rows, then the partials of its splits
size_t decode_qhat_bytes(const fcsa_problem* p, const DecodeCall& c) {
  const size_t rows = c.packed ? (size_t)c.total_q : (size_t)p->batch * p->seq_q;
  return align16(rows * p->heads * p->head_dim * 2);
}

size_t decode_bytes(const fcsa_problem* p, const DecodeCall& c, const DecodeShape& sh) {
  return decode_qhat_bytes(p, c) + fcsa::decode_partial_bytes(sh.items, sh.n_split, p->head_dim);
}

// The workspace-size query of decode call c: 0 for a refused problem
size_t decode_workspace_bytes(const fcsa_problem* p, const DecodeCall& c) {
  DecodeShape sh;
  if (check_decode(p, c, true) || decode_shape(p, &sh)) return 0;
  return decode_bytes(p, c, sh);
}

// n_new: rows appended per sequence (packed: 1 when appending, else 0)
template <typename T, int D>
int launch_decode(const fcsa_problem* p, const DecodeCall& c, const DecodeShape& sh, const fcsa_tensor* q,
                  const fcsa_tensor* kc, const fcsa_tensor* vc, const int32_t* seqlens, int32_t n_new,
                  const fcsa_tensor* o, float* part, cudaStream_t stream) {
  using Cfg = fcsa::DecodeCfg<D>;
  CUtensorMap tk, tv;
  int r;
  if ((r = map_operand<T, D>(&tk, "k_cache", *kc, p->batch, p->kv_heads, p->seq_k, 128)) ||
      (r = map_operand<T, D>(&tv, "v_cache", *vc, p->batch, p->kv_heads, p->seq_k, 128)))
    return r;
  fcsa::Windowed<fcsa::DecodeArgs> a;
  a.window = kernel_window(p);
  a.B = p->batch; a.H = p->heads; a.KVH = p->kv_heads; a.G = p->heads / p->kv_heads;
  a.Nq = p->seq_q; a.cap = p->seq_k; a.n_new = n_new;
  a.causal = p->causal ? 1 : 0;
  a.R = sh.R; a.n_rb = sh.n_rb; a.n_split = sh.n_split;
  const float log2e = 1.4426950408889634f;
  a.c1 = p->scale * log2e;
  a.c2 = p->shift * log2e;
  a.ring = c.ring ? p->seq_k : 0;
  a.seqlens = seqlens;
  a.q = q->ptr; a.q_sb = q->sb; a.q_sh = q->sh; a.q_sn = q->sn;
  a.o = o->ptr; a.o_sb = o->sb; a.o_sh = o->sh; a.o_sn = o->sn;
  a.part = part;
  a.cu_q = c.cu; a.total_q = c.total_q;
  if (c.cu) a.q_sb = a.o_sb = 0;
  const long long grid = sh.items * sh.n_split;
  if (grid > 0x7FFFFFFFLL) return fail(FCSA_ERR_INVALID, "decode: problem too large for one launch");
  const auto launch = [&](auto kern) {
    return launch_attention<decltype(kern)::value>("decode", nullptr, grid, Cfg::kThreads, Cfg::kSmem, stream, tk, tv, a);
  };
  r = a.window > 0 ? launch(kernel_c<fcsa::fcsa_decode_kernel<T, D, true>>{})
                   : launch(kernel_c<fcsa::fcsa_decode_kernel<T, D>>{});
  if (r || sh.n_split == 1) return r;
  const long long threads = sh.items * 64 * (D / 4);
  return launched(fcsa::launch_pdl(fcsa::decode_combine_kernel<T, D>, dim3((unsigned)((threads + 255) / 256)),
                                   dim3(256), 0, stream, a),
                  "decode combine launch");
}

// ---- packed sequences ----------------------------------------------------------------------------
// The problem of a varlen call: batch = sequences, seq_q / seq_k = the maximum lengths; no key mask, 16-bit outputs.
int check_varlen(const fcsa_problem* p, const fcsa_varlen* vl) {
  int r;
  if ((r = check_problem(p))) return r;
  if (p->key_mask) return fail(FCSA_ERR_UNSUPPORTED, "varlen: no key mask (cu_seqlens give the valid rows)");
  if (p->out_f32) return fail(FCSA_ERR_UNSUPPORTED, "varlen: out_f32 is not implemented");
  if (!vl) return fail(FCSA_ERR_INVALID, "varlen: null fcsa_varlen");
  if (!vl->cu_seqlens_q || !vl->cu_seqlens_k) return fail(FCSA_ERR_INVALID, "varlen: null cu_seqlens");
  if ((reinterpret_cast<uintptr_t>(vl->cu_seqlens_q) & 3) || (reinterpret_cast<uintptr_t>(vl->cu_seqlens_k) & 3))
    return fail(FCSA_ERR_INVALID, "varlen: cu_seqlens must be 4-byte aligned int32 arrays");
  if (vl->total_q <= 0 || vl->total_k <= 0)
    return fail(FCSA_ERR_INVALID, "varlen: empty packed tensors (total_q %d total_k %d)", vl->total_q, vl->total_k);
  if ((long long)vl->total_q / 64 + p->batch + 1 > 0x7FFFFFFFLL / 64)
    return fail(FCSA_ERR_INVALID, "varlen: too many query rows and sequences for one call");
  return FCSA_OK;
}

// Zero the rows of up to three packed outputs that belong to no sequence (fcsa::varlen_tail_kernel), after the
// attention kernels on the same stream.  t[i].cu / total say which cumulative lengths each tensor follows.
int launch_varlen_tail(const fcsa_problem* p, fcsa::TailArgs a, int n, cudaStream_t stream) {
  a.B = p->batch;
  a.D = p->head_dim;
  long long vecs = 0;
  for (int i = 0; i < n; ++i) vecs = std::max(vecs, (long long)a.t[i].total * a.t[i].H * (p->head_dim / 8));
  // a grid-stride loop: a few waves of blocks at most, whatever the tail's length
  const unsigned blocks = (unsigned)std::max(1LL, std::min((vecs + 255) / 256, 1024LL));
  return launched(fcsa::launch_pdl(fcsa::varlen_tail_kernel, dim3(blocks, n), dim3(256), 0, stream, a),
                  "varlen tail launch");
}

// ---- backward ------------------------------------------------------------------------------------
// The backward's workspace layout, dense or packed sequences (vl), and the scratch and zeroed bytes its route needs.
// The deterministic route takes the stats alone as scratch (no dq accumulator, and no dk / dv accumulators:
// split = 1) and no zeroed workspace.
struct BwdNeed {
  fcsa::BwdWorkspace w;
  size_t scratch, zeroed;
};

BwdNeed bwd_need(const fcsa_problem* p, const fcsa_varlen* vl, bool deterministic) {
  const fcsa::BwdWorkspace w =
      vl ? fcsa::bwd_varlen_workspace_layout(p->batch, p->heads, p->kv_heads, vl->total_q, vl->total_k, p->head_dim)
         : fcsa::bwd_workspace_layout(p->batch, p->heads, p->kv_heads, p->seq_q, p->seq_k, p->head_dim);
  return {w, deterministic ? w.dkv_off : w.total, deterministic ? 0 : w.ztotal};
}

// The backward's arguments, filled from the problem and the caller's tensors by backward_impl
struct BwdHostArgs {
  int B, H, kv_heads, Nq, Nk, causal;
  int window;                       // sliding window W (0 = none; never with a bias)
  float scale, shift;
  const uint8_t* mask; long long mask_sb;
  fcsa_tensor q, k, v, o, d_o, dq, dk, dv;
  const float* inv_l;
  bool out_f32;                     // o (read), dq, dk, dv (written) are float32
  void* workspace;                  // scratch
  void* zeroed;                     // zero on entry, zero again on exit (dq accumulator); unused when deterministic
  // the deterministic route: dK / dV with split = 1 (fcsa_bwd_kernel<DQ = false>), then fcsa_dq_kernel
  bool deterministic = false;
  // fused l2norm backward (q, k above are then the NORMALISED tensors and dq, dk the gradients
  // w.r.t. the raw ones); both null = plain backward
  const float* q_rnorm;
  const float* k_rnorm;
  int groups;
  // additive bias (nullptr = none) and its fp32 gradient accumulator (nullptr = not needed)
  const void* bias = nullptr; long long bias_sb = 0, bias_sh = 0, bias_sn = 0;
  const float* bias_amax = nullptr;           // optional device scalar added (if positive) to the shift
  float* dbias = nullptr; long long dbias_sb = 0, dbias_sh = 0;
  // packed sequences (VARLEN): B sequences, Nq / Nk the maximum lengths, q, d_o, o, dq (total_q, H, D)
  // and k, v, dk, dv (total_k, kv_heads, D) with sb unused, inv_l (H, total_q), the rnorms [heads][total][groups]
  const int* cu_q = nullptr;
  const int* cu_k = nullptr;
  int total_q = 0, total_k = 0;
};

// The dQ kernel of the deterministic backward, after the dK / dV kernel: one CTA per (block of dq_block_rows query
// rows, batch, query head); packed sequences: blocks of the longest sequence.
template <typename T, int D, bool VARLEN>
int launch_dq(const BwdHostArgs& h, const fcsa::BwdWorkspace& w, const float* stats, cudaStream_t stream) {
  using Cfg = fcsa::DqCfg<D>;
  const int tB = VARLEN ? 1 : h.B, tNq = VARLEN ? h.total_q : h.Nq, tNk = VARLEN ? h.total_k : h.Nk;
  CUtensorMap tq, tk, tv, tdo;
  int r;
  if ((r = map_operand<T, D>(&tq, "q", h.q, tB, h.H, tNq, Cfg::kBlockM)) ||
      (r = map_operand<T, D>(&tk, "k", h.k, tB, h.kv_heads, tNk, 128)) ||
      (r = map_operand<T, D>(&tv, "v", h.v, tB, h.kv_heads, tNk, 128)) ||
      (r = map_operand<T, D>(&tdo, "d_o", h.d_o, tB, h.H, tNq, Cfg::kBlockM)))
    return r;
  fcsa::ArgsOf<fcsa::DqArgs, fcsa::DqVarlenArgs, VARLEN, true> a;
  a.window = h.window;
  if constexpr (VARLEN) {
    a.cu_q = h.cu_q; a.cu_k = h.cu_k; a.total_q = h.total_q; a.total_k = h.total_k; a.ntile = w.nqt;
  }
  a.B = h.B; a.H = h.H; a.Nq = h.Nq; a.Nk = h.Nk; a.causal = h.causal; a.has_mask = h.mask ? 1 : 0;
  a.group = h.H / h.kv_heads;
  a.n_qblk = fcsa::row_blocks(h.Nq, Cfg::kBlockM);
  a.nqt = w.nqt;
  a.c1 = h.scale * 1.4426950408889634f; a.scale = h.scale;
  a.mask = h.mask; a.mask_sb = h.mask_sb;
  a.stats = stats;
  a.out_f32 = h.out_f32 ? 1 : 0;
  a.dq = h.dq.ptr; a.dq_sb = h.dq.sb; a.dq_sh = h.dq.sh; a.dq_sn = h.dq.sn;
  a.q_rnorm = h.q_rnorm; a.groups = h.groups;
  const long long grid = (long long)a.n_qblk * h.B * h.H;
  if (grid > 0x7FFFFFFFLL) return fail(FCSA_ERR_INVALID, "problem too large for one launch");
  const auto launch = [&](auto kern) {
    return launch_attention<decltype(kern)::value>("dQ", g_ev[4], grid, Cfg::kThreads, Cfg::kSmem, stream, tq, tk, tv,
                                                   tdo, a);
  };
  return a.window > 0 ? launch(kernel_c<fcsa::fcsa_dq_kernel<T, D, VARLEN, true>>{})
                      : launch(kernel_c<fcsa::fcsa_dq_kernel<T, D, VARLEN>>{});
}

// The backward's launches: preprocess, main kernel, dq finish, and for split groups the dk / dv finish (and the l2norm
// backward of dk).  Deterministic: preprocess, the dK / dV kernel with split = 1, the dQ kernel.  w: the workspaces'
// layout (bwd_need).
template <typename T, int D, bool BIAS = false, bool VARLEN = false>
int run_backward_t(const BwdHostArgs& h, const fcsa::BwdWorkspace& w, cudaStream_t stream) {
  using namespace fcsa;
  using Cfg = BwdCfg<D>;
  // the batch, key rows and query tiles of the tensors as addressed: packed sequences are one batch of total rows
  const int tB = VARLEN ? 1 : h.B, tNq = VARLEN ? h.total_q : h.Nq, tNk = VARLEN ? h.total_k : h.Nk;
  const int nqt = (h.Nq + Cfg::QT - 1) / Cfg::QT;     // query tiles of the longest sequence
  uint8_t* ws = reinterpret_cast<uint8_t*>(h.workspace);
  uint8_t* zs = reinterpret_cast<uint8_t*>(h.zeroed);
  float* stats = reinterpret_cast<float*>(ws + w.stats_off);
  float* dq_acc = reinterpret_cast<float*>(zs + w.dq_off);
  float* dkv_acc = reinterpret_cast<float*>(ws + w.dkv_off);
  const float log2e = 1.4426950408889634f;
  cudaError_t e;
  int r;
  int split = 1;
  if (h.kv_heads < h.H && !h.deterministic) {
    int sms = 0;
    e = device_sm_count(&sms);
    if (e != cudaSuccess) return cuda_fail(e, "cudaDeviceGetAttribute(multiProcessorCount)");
    split = bwd_group_split(h.B, h.H, h.kv_heads, h.Nk, BIAS, sms);
  }
  const bool to_acc = split > 1;
  const size_t dkv_elems = (size_t)tB * h.kv_heads * tNk * D;

  // dk/dv accumulators of split groups are per call (the dq accumulator is self-cleaning)
  if (to_acc) {
    e = cudaMemsetAsync(dkv_acc, 0, 2 * dkv_elems * 4, stream);
    if (e != cudaSuccess) return cuda_fail(e, "cudaMemsetAsync(workspace)");
  }

  // 1. preprocess
  {
    std::conditional_t<VARLEN, PrepVarlenArgs, PrepArgs> pa;
    pa.B = h.B; pa.H = h.H; pa.Nq = h.Nq; pa.Nk = h.Nk; pa.D = D; pa.nqt = nqt; pa.QT = Cfg::QT; pa.causal = h.causal;
    if constexpr (VARLEN) { pa.cu_q = h.cu_q; pa.total_q = h.total_q; pa.ntile = w.nqt; }
    pa.c2 = h.shift * log2e;
    pa.shift_extra = h.bias_amax;
    pa.o_f32 = h.out_f32 ? 1 : 0;
    pa.o = h.o.ptr; pa.o_sb = h.o.sb; pa.o_sh = h.o.sh; pa.o_sn = h.o.sn;
    pa.d_o = h.d_o.ptr; pa.do_sb = h.d_o.sb; pa.do_sh = h.d_o.sh; pa.do_sn = h.d_o.sn;
    pa.inv_l = h.inv_l; pa.stats = stats;
    const int rows_per_block = 2 * (256 / (D / 8));
    const int padded = nqt * Cfg::QT;
    pa.bpb = (padded + rows_per_block - 1) / rows_per_block;
    const long long grid = (long long)pa.bpb * h.B * h.H;
    if (grid > 0x7FFFFFFFLL) return fail(FCSA_ERR_INVALID, "problem too large for one launch");
    e = timed(g_ev[3], stream, [&] {
      return launch_pdl(bwd_prep_kernel<T, D / 8, VARLEN>, dim3((unsigned)grid), dim3(256), 0, stream, pa);
    });
    if ((r = launched(e, "backward preprocess launch"))) return r;
  }
  // 2. main
  {
    CUtensorMap tq, tk, tv, tdo, tdq;
    // keys of one work item (BwdCfg::kKeys of the kernel launched below): one K / V box each
    const bool head_loop = !BIAS && h.H / h.kv_heads / split > 1;
    const int keys = h.deterministic ? BwdCfg<D, BIAS, false>::kKeys
                                     : head_loop ? BwdCfg<D, BIAS, true, true>::kKeys : BwdCfg<D, BIAS, true>::kKeys;
    if ((r = map_operand<T, D>(&tq, "q", h.q, tB, h.H, tNq, Cfg::QT)) ||
        (r = map_operand<T, D>(&tk, "k", h.k, tB, h.kv_heads, tNk, keys)) ||
        (r = map_operand<T, D>(&tv, "v", h.v, tB, h.kv_heads, tNk, keys)) ||
        (r = map_operand<T, D>(&tdo, "d_o", h.d_o, tB, h.H, tNq, Cfg::QT)))
      return r;
    // the dq accumulator as [B][H][Nq][D] fp32 over its padded rows: boxes of 32 features x QT rows (packed
    // sequences: [1][H][ntile * QT][D], every tile inside the map)
    memset(&tdq, 0, sizeof(tdq));
    const long long acc_sh = (long long)w.nqt * Cfg::QT * D;
    if (Cfg::kStaged && !h.deterministic &&
        (r = make_tensor_map_bhnd(&tdq, dq_acc, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, tB, h.H, VARLEN ? w.nqt * Cfg::QT : h.Nq,
                                  D, h.H * acc_sh, acc_sh, D, Cfg::QT, 32)))
      return fail(FCSA_ERR_CUDA, "dq accumulator: cuTensorMapEncodeTiled failed (%d)", r);
    // (the window's arguments extend the kernel's)
    ArgsOf<BwdArgs, BwdVarlenArgs, VARLEN, true> a;
    a.window = h.window;
    a.B = h.B; a.H = h.H; a.Nq = h.Nq; a.Nk = h.Nk; a.kv_heads = h.kv_heads; a.causal = h.causal;
    a.has_mask = h.mask ? 1 : 0; a.nqt = w.nqt;
    if constexpr (VARLEN) {
      a.cu_q = h.cu_q; a.cu_k = h.cu_k; a.total_q = h.total_q; a.total_k = h.total_k; a.ntile = w.nqt;
    }
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
    // one CTA per (block of `keys` keys, batch, kv head, slice of its group), heaviest blocks first; packed
    // sequences: key blocks of the longest one
    const long long items = (long long)((h.Nk + keys - 1) / keys) * h.B * h.kv_heads * split;
    if (items > 0x7FFFFFFFLL) return fail(FCSA_ERR_INVALID, "problem too large for one launch");
    // (kern, its config)
    const auto launch = [&](auto kern, auto cfg) {
      using KCfg = decltype(cfg);
      return launch_attention<decltype(kern)::value>("backward", g_ev[1], items, KCfg::kThreads, KCfg::kSmem, stream,
                                                     tq, tk, tv, tdo, tdq, a);
    };
    // DQ = false: the dK / dV kernel of the deterministic route
    const auto launch_main = [&](auto dq) {
      constexpr bool DQ = decltype(dq)::value;
      if (a.hpc > 1)   // HEAD_LOOP
        return a.window > 0 ? launch(kernel_c<fcsa_bwd_kernel<T, D, false, true, VARLEN, true, DQ>>{},
                                     BwdCfg<D, false, DQ, true>{})
                            : launch(kernel_c<fcsa_bwd_kernel<T, D, false, true, VARLEN, false, DQ>>{},
                                     BwdCfg<D, false, DQ, true>{});
      const BwdCfg<D, false, DQ> cfg;
      return a.window > 0 ? launch(kernel_c<fcsa_bwd_kernel<T, D, false, false, VARLEN, true, DQ>>{}, cfg)
                          : launch(kernel_c<fcsa_bwd_kernel<T, D, false, false, VARLEN, false, DQ>>{}, cfg);
    };
    if constexpr (BIAS)   // (one query head per CTA, no window)
      r = launch(kernel_c<fcsa_bwd_kernel<T, D, true>>{}, BwdCfg<D, true>{});
    else
      r = h.deterministic ? launch_main(std::false_type{}) : launch_main(std::true_type{});
    if (r) return r;
  }
  if constexpr (!BIAS) {
    if (h.deterministic) return launch_dq<T, D, VARLEN>(h, w, stats, stream);
  }
  // 3. finish
  {
    std::conditional_t<VARLEN, DqFinishVarlenArgs, DqFinishArgs> fa;
    fa.B = h.B; fa.H = h.H; fa.Nq = h.Nq; fa.D = D; fa.nqt = w.nqt; fa.padded = w.nqt * Cfg::QT; fa.scale = h.scale;
    if constexpr (VARLEN) { fa.padded = nqt * Cfg::QT; fa.cu_q = h.cu_q; fa.total_q = h.total_q; fa.ntile = w.nqt; }
    fa.dq_acc = dq_acc; fa.dq = h.dq.ptr; fa.sb = h.dq.sb; fa.sh = h.dq.sh; fa.sn = h.dq.sn;
    fa.q_hat = h.q.ptr; fa.q_sb = h.q.sb; fa.q_sh = h.q.sh; fa.q_sn = h.q.sn;
    fa.q_rnorm = h.q_rnorm; fa.G = h.groups; fa.out_f32 = h.out_f32 ? 1 : 0;
    const long long threads = (long long)h.B * h.H * (VARLEN ? fa.padded : h.Nq) * (D / 8);
    const long long blocks = VARLEN ? (threads + 255) / 256 : (threads + 511) / 512;   // dense: two rows per thread
    if (blocks > 0x7FFFFFFFLL) return fail(FCSA_ERR_INVALID, "problem too large for one launch");
    e = timed(g_ev[4], stream, [&] {
      return launch_pdl(bwd_dq_finish_kernel<T, D, VARLEN>, dim3((unsigned)blocks), dim3(256), 0, stream, fa);
    });
    if ((r = launched(e, "dq finish launch"))) return r;
    if (to_acc) {
      for (int which = 0; which < 2; ++which) {
        KvFinishArgs ka;
        ka.B = tB; ka.Hk = h.kv_heads; ka.Nk = tNk; ka.D = D; ka.out_f32 = h.out_f32 ? 1 : 0;
        ka.acc = dkv_acc + (which ? dkv_elems : 0);
        const fcsa_tensor& t = which ? h.dv : h.dk;
        ka.out = t.ptr; ka.sb = t.sb; ka.sh = t.sh; ka.sn = t.sn;
        const long long tot = (long long)dkv_elems / 8;
        bwd_kv_finish_kernel<T><<<(unsigned)((tot + 255) / 256), 256, 0, stream>>>(ka);
        if ((r = launched(cudaGetLastError(), "dk/dv finish launch"))) return r;
      }
    }
    if (h.k_rnorm != nullptr && to_acc) {
      // l2norm backward of dk (gradient w.r.t. the raw keys) as its own pass over the head-summed dk; otherwise
      // the main kernel's epilogue applies it
      RowArgs la = {};
      la.B = tB; la.D = D; la.G = h.groups;
      la.t[0] = {h.kv_heads, tNk, h.dk, h.k, h.dk, const_cast<float*>(h.k_rnorm)};
      if ((r = launched(launch_row_bwd(la, std::is_same<T, __nv_bfloat16>::value, false, stream),
                        "l2norm backward (dk) launch")))
        return r;
    }
  }
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
  return dispatch(p, [&](auto t, auto d) {
    return launch_forward<typename decltype(t)::type, decltype(d)::value>(p, q, k, v, o, inv_l,
                                                                          reinterpret_cast<cudaStream_t>(stream));
  });
}

int fcsa_forward_bias(const fcsa_problem* p, const fcsa_tensor* q, const fcsa_tensor* k,
                      const fcsa_tensor* v, const fcsa_bias* bias, const fcsa_tensor* o, float* inv_l,
                      void* stream) {
  int r;
  if ((r = check_problem(p))) return r;
  if ((r = check_tensor(q, "q")) || (r = check_tensor(k, "k")) || (r = check_tensor(v, "v")) ||
      (r = check_tensor(o, "o")) || (r = check_bias(p, bias)))
    return r;
  return dispatch(p, [&](auto t, auto d) {
    return launch_forward<typename decltype(t)::type, decltype(d)::value, true>(
        p, q, k, v, o, inv_l, reinterpret_cast<cudaStream_t>(stream), bias);
  });
}

size_t fcsa_backward_workspace_bytes(const fcsa_problem* p) {
  return check_problem(p) ? 0 : bwd_need(p, nullptr, false).scratch;
}

size_t fcsa_backward_zeroed_bytes(const fcsa_problem* p) {
  return check_problem(p) ? 0 : bwd_need(p, nullptr, false).zeroed;
}

int fcsa_zeroed_init(void* zeroed, size_t bytes, void* stream) {
  if (!zeroed || bytes == 0) return fail(FCSA_ERR_INVALID, "zeroed workspace: null / empty");
  cudaError_t e = cudaMemsetAsync(zeroed, 0, bytes, reinterpret_cast<cudaStream_t>(stream));
  if (e != cudaSuccess) return cuda_fail(e, "cudaMemsetAsync(zeroed workspace)");
  return FCSA_OK;
}

// Every backward entry point: dense or packed sequences (vl), with the fused l2norm backward over `groups` when
// q_rnorm / k_rnorm are set (q, k are then the normalised tensors), or with a bias.  deterministic: the route without
// atomics, which needs the stats alone as scratch and no zeroed workspace (zeroed is ignored).  Packed sequences end
// with zero gradients in the rows outside every sequence.
static int backward_impl(const fcsa_problem* p, const fcsa_varlen* vl, const fcsa_tensor* q, const fcsa_tensor* k,
                         const fcsa_tensor* v, const fcsa_tensor* o, const fcsa_tensor* d_o,
                         const float* inv_l, const fcsa_tensor* dq, const fcsa_tensor* dk,
                         const fcsa_tensor* dv, void* workspace, size_t workspace_bytes, void* zeroed,
                         size_t zeroed_bytes, void* stream,
                         const float* q_rnorm, const float* k_rnorm, int groups, bool deterministic,
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
  const BwdNeed need = bwd_need(p, vl, deterministic);
  if (!workspace || workspace_bytes < need.scratch)
    return fail(FCSA_ERR_WORKSPACE, "workspace too small: need %zu bytes, got %zu", need.scratch, workspace_bytes);
  if (!aligned16(workspace)) return fail(FCSA_ERR_INVALID, "workspace not 16-byte aligned");
  if (!deterministic) {
    if (!zeroed || zeroed_bytes < need.zeroed)
      return fail(FCSA_ERR_WORKSPACE, "zeroed workspace too small: need %zu bytes, got %zu", need.zeroed, zeroed_bytes);
    if (!aligned16(zeroed)) return fail(FCSA_ERR_INVALID, "zeroed workspace not 16-byte aligned");
  }
  if (p->out_f32 && (q_rnorm || k_rnorm))
    return fail(FCSA_ERR_UNSUPPORTED, "out_f32 with the fused l2norm backward is not implemented (normalise outside)");
  BwdHostArgs h;
  h.B = p->batch; h.H = p->heads; h.kv_heads = p->kv_heads; h.Nq = p->seq_q; h.Nk = p->seq_k;
  h.causal = p->causal ? 1 : 0;
  h.window = kernel_window(p);
  h.scale = p->scale; h.shift = p->shift;
  h.mask = p->key_mask; h.mask_sb = p->key_mask_stride;
  h.q = *q; h.k = *k; h.v = *v; h.o = *o; h.d_o = *d_o; h.dq = *dq; h.dk = *dk; h.dv = *dv;
  h.inv_l = inv_l;
  h.out_f32 = p->out_f32 != 0;
  h.workspace = workspace;
  h.zeroed = deterministic ? nullptr : zeroed;
  h.deterministic = deterministic;
  h.q_rnorm = q_rnorm;
  h.k_rnorm = k_rnorm;
  h.groups = groups;
  if (bias) {
    h.bias = bias->ptr; h.bias_sb = bias->sb; h.bias_sh = bias->sh; h.bias_sn = bias->sn;
    h.bias_amax = bias->amax;
    h.dbias = d_bias_acc; h.dbias_sb = dsb; h.dbias_sh = dsh;
  }
  if (vl) {
    h.cu_q = vl->cu_seqlens_q; h.cu_k = vl->cu_seqlens_k;
    h.total_q = vl->total_q; h.total_k = vl->total_k;
  }
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  r = dispatch(p, [&](auto t, auto d) {
    using T = typename decltype(t)::type;
    constexpr int D = decltype(d)::value;
    if (vl) return run_backward_t<T, D, false, true>(h, need.w, s);   // (packed sequences take no bias)
    if (bias) return run_backward_t<T, D, true>(h, need.w, s);
    return run_backward_t<T, D>(h, need.w, s);
  });
  if (r || !vl) return r;
  fcsa::TailArgs ta = {};
  ta.t[0] = {dq->ptr, dq->sh, dq->sn, p->heads, vl->total_q, vl->cu_seqlens_q};
  ta.t[1] = {dk->ptr, dk->sh, dk->sn, p->kv_heads, vl->total_k, vl->cu_seqlens_k};
  ta.t[2] = {dv->ptr, dv->sh, dv->sn, p->kv_heads, vl->total_k, vl->cu_seqlens_k};
  return launch_varlen_tail(p, ta, 3, s);
}

// The backward entry points that take the fused l2norm's outputs n (q^, k^ and their rnorms): dense, or packed
// sequences (the varlen entry points, whose vl must be set).  groups = 0 is the plain backward of q^, k^, except in
// fcsa_backward_fused.
static int backward_l2norm(const fcsa_problem* p, bool packed, const fcsa_varlen* vl, const fcsa_l2norm* n,
                           const fcsa_tensor* v, const fcsa_tensor* o, const fcsa_tensor* d_o, const float* inv_l,
                           const fcsa_tensor* dq, const fcsa_tensor* dk, const fcsa_tensor* dv, void* workspace,
                           size_t workspace_bytes, void* zeroed, size_t zeroed_bytes, void* stream,
                           bool deterministic) {
  int r;
  if (packed && (r = check_varlen(p, vl))) return r;
  if (!n) return fail(FCSA_ERR_INVALID, "null fcsa_l2norm");
  if (!packed && (r = check_problem(p))) return r;
  const bool fused = n->groups != 0 || (!vl && !deterministic);
  if (fused && (r = check_l2norm(p, n, vl ? 1 : p->batch, vl ? vl->total_q : p->seq_q))) return r;
  return backward_impl(p, vl, &n->q_hat, &n->k_hat, v, o, d_o, inv_l, dq, dk, dv, workspace, workspace_bytes, zeroed,
                       zeroed_bytes, stream, fused ? n->q_rnorm : nullptr, fused ? n->k_rnorm : nullptr,
                       fused ? n->groups : 1, deterministic);
}

int fcsa_backward(const fcsa_problem* p, const fcsa_tensor* q, const fcsa_tensor* k,
                  const fcsa_tensor* v, const fcsa_tensor* o, const fcsa_tensor* d_o,
                  const float* inv_l, const fcsa_tensor* dq, const fcsa_tensor* dk,
                  const fcsa_tensor* dv, void* workspace, size_t workspace_bytes, void* zeroed,
                  size_t zeroed_bytes, void* stream) {
  return backward_impl(p, nullptr, q, k, v, o, d_o, inv_l, dq, dk, dv, workspace, workspace_bytes, zeroed,
                       zeroed_bytes, stream, nullptr, nullptr, 1, false);
}

int fcsa_backward_bias(const fcsa_problem* p, const fcsa_tensor* q, const fcsa_tensor* k,
                       const fcsa_tensor* v, const fcsa_tensor* o, const fcsa_tensor* d_o,
                       const float* inv_l, const fcsa_bias* bias, float* d_bias_acc, int64_t dsb,
                       int64_t dsh, const fcsa_tensor* dq, const fcsa_tensor* dk, const fcsa_tensor* dv,
                       void* workspace, size_t workspace_bytes, void* zeroed, size_t zeroed_bytes, void* stream) {
  if (!bias) return fail(FCSA_ERR_INVALID, "attn_bias: null");
  return backward_impl(p, nullptr, q, k, v, o, d_o, inv_l, dq, dk, dv, workspace, workspace_bytes, zeroed,
                       zeroed_bytes, stream, nullptr, nullptr, 1, false, bias, d_bias_acc, dsb, dsh);
}

int fcsa_forward_fused(const fcsa_problem* p, const fcsa_tensor* q, const fcsa_tensor* k,
                       const fcsa_tensor* v, const fcsa_l2norm* n, const fcsa_tensor* o, float* inv_l,
                       void* stream) {
  int r;
  if ((r = check_problem(p))) return r;
  if (!n) return fail(FCSA_ERR_INVALID, "null fcsa_l2norm");
  if ((r = l2norm_qk(p, n, q, k, p->batch, p->seq_q, p->seq_k, reinterpret_cast<cudaStream_t>(stream)))) return r;
  return fcsa_forward(p, &n->q_hat, &n->k_hat, v, o, inv_l, stream);
}

int fcsa_backward_fused(const fcsa_problem* p, const fcsa_l2norm* n, const fcsa_tensor* v,
                        const fcsa_tensor* o, const fcsa_tensor* d_o, const float* inv_l,
                        const fcsa_tensor* dq, const fcsa_tensor* dk, const fcsa_tensor* dv,
                        void* workspace, size_t workspace_bytes, void* zeroed, size_t zeroed_bytes,
                        void* stream) {
  return backward_l2norm(p, false, nullptr, n, v, o, d_o, inv_l, dq, dk, dv, workspace, workspace_bytes, zeroed,
                         zeroed_bytes, stream, false);
}

size_t fcsa_backward_fused_deterministic_workspace_bytes(const fcsa_problem* p) {
  return check_problem(p) ? 0 : bwd_need(p, nullptr, true).scratch;
}

int fcsa_backward_fused_deterministic(const fcsa_problem* p, const fcsa_l2norm* n, const fcsa_tensor* v,
                                      const fcsa_tensor* o, const fcsa_tensor* d_o, const float* inv_l,
                                      const fcsa_tensor* dq, const fcsa_tensor* dk, const fcsa_tensor* dv,
                                      void* workspace, size_t workspace_bytes, void* stream) {
  return backward_l2norm(p, false, nullptr, n, v, o, d_o, inv_l, dq, dk, dv, workspace, workspace_bytes, nullptr, 0,
                         stream, true);
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
  return launched(fcsa::launch_row_fwd(a, dtype == FCSA_BF16, true, reinterpret_cast<cudaStream_t>(stream)),
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
  return launched(fcsa::launch_row_bwd(a, dtype == FCSA_BF16, true, reinterpret_cast<cudaStream_t>(stream)),
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
  return launched(fcsa::launch_row_fwd(a, dtype == FCSA_BF16, false, reinterpret_cast<cudaStream_t>(stream)),
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
  return launched(fcsa::launch_row_bwd(a, dtype == FCSA_BF16, false, reinterpret_cast<cudaStream_t>(stream)),
                  "l2norm backward launch");
}

// fcsa_decode, fcsa_decode_varlen and fcsa_decode_rolling: decode call c (packed: q, o, k_new, v_new are total_q rows)
static int decode_impl(const fcsa_problem* p, const DecodeCall& c, const fcsa_tensor* q, const fcsa_tensor* k_cache,
                       const fcsa_tensor* v_cache, const int32_t* cache_seqlens, const fcsa_tensor* k_new,
                       const fcsa_tensor* v_new, int32_t groups, const fcsa_tensor* o, void* workspace,
                       size_t workspace_bytes, void* stream) {
  int r;
  if ((r = check_decode(p, c, false, k_new, v_new))) return r;
  const bool append = c.packed || c.ring ? k_new != nullptr : c.n_new > 0;
  // rows appended per sequence (packed: 1, each sequence appending its own rows); a dense rolling call one per query
  const int32_t n_new = !append ? 0 : c.packed ? 1 : c.ring ? p->seq_q : c.n_new;
  if ((r = check_tensor(q, "q")) || (r = check_tensor(k_cache, "k_cache")) || (r = check_tensor(v_cache, "v_cache")) ||
      (r = check_tensor(o, "o")))
    return r;
  if (append && ((r = check_tensor(k_new, "k")) || (r = check_tensor(v_new, "v")))) return r;
  if (c.packed && c.total_q == 0) return FCSA_OK;
  // the row pass's shape: the batch's rows, or the packed rows as one batch
  const int32_t rB = c.packed ? 1 : p->batch, rN = c.packed ? c.total_q : p->seq_q;
  if (groups != 0 && (r = check_rows(false, p->dtype, rB, p->heads, rN, p->head_dim, groups))) return r;
  if (!cache_seqlens) return fail(FCSA_ERR_INVALID, "cache_seqlens: null");
  DecodeShape sh;
  if ((r = decode_shape(p, &sh))) return r;
  const size_t need = decode_bytes(p, c, sh);
  if (!workspace || workspace_bytes < need)
    return fail(FCSA_ERR_WORKSPACE, "workspace too small: need %zu bytes, got %zu", need, workspace_bytes);
  if (!aligned16(workspace)) return fail(FCSA_ERR_INVALID, "workspace not 16-byte aligned");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);

  // append pass: q_hat to the workspace (groups > 0), then k (normalised when groups > 0) and v into the caches at
  // row cache_seqlens[b] (packed: the row's sequence b, at cache_seqlens[b] + its row within the sequence), modulo
  // the rows of a rolling cache
  const int64_t H = p->heads, N = rN, D = p->head_dim;
  const fcsa_tensor qhat = {workspace, H * N * D, N * D, D};
  fcsa::RowArgs a = row_args(rB, p->head_dim, groups);
  const int32_t n_app = c.packed ? c.total_q : n_new;
  int n = 0;
  if (groups > 0) a.t[n++] = {p->heads, rN, *q, qhat, {}, nullptr, nullptr, rN, 0};
  if (append) {
    const uint8_t k_raw = groups == 0 ? 1 : 0, rolling = c.ring ? 1 : 0;
    a.t[n++] = {p->kv_heads, n_app, *k_new, *k_cache, {}, nullptr, cache_seqlens, p->seq_k, k_raw, rolling, c.cu,
                p->batch, p->seq_q};
    a.t[n++] = {p->kv_heads, n_app, *v_new, *v_cache, {}, nullptr, cache_seqlens, p->seq_k, 1, rolling, c.cu,
                p->batch, p->seq_q};
  }
  if (n > 0 && (r = launched(fcsa::launch_row_append(a, n, p->dtype == FCSA_BF16, s), "append pass launch")))
    return r;

  const fcsa_tensor* qa = groups > 0 ? &qhat : q;
  float* part = reinterpret_cast<float*>(static_cast<char*>(workspace) + decode_qhat_bytes(p, c));
  r = dispatch(p, [&](auto t, auto d) {
    return launch_decode<typename decltype(t)::type, decltype(d)::value>(p, c, sh, qa, k_cache, v_cache, cache_seqlens,
                                                                         n_new, o, part, s);
  });
  if (r || !c.packed) return r;
  // o = 0 in the rows outside every sequence
  fcsa::TailArgs ta = {};
  ta.t[0] = {o->ptr, o->sh, o->sn, p->heads, c.total_q, c.cu};
  return launch_varlen_tail(p, ta, 1, s);
}

size_t fcsa_decode_workspace_bytes(const fcsa_problem* p, int32_t n_new) {
  return decode_workspace_bytes(p, {"decode: ", false, nullptr, 0, n_new, false});
}

int fcsa_decode(const fcsa_problem* p, const fcsa_tensor* q, const fcsa_tensor* k_cache, const fcsa_tensor* v_cache,
                const int32_t* cache_seqlens, const fcsa_tensor* k_new, const fcsa_tensor* v_new, int32_t n_new,
                int32_t groups, const fcsa_tensor* o, void* workspace, size_t workspace_bytes, void* stream) {
  return decode_impl(p, {"decode: ", false, nullptr, 0, n_new, false}, q, k_cache, v_cache, cache_seqlens, k_new, v_new,
                     groups, o, workspace, workspace_bytes, stream);
}

size_t fcsa_decode_varlen_workspace_bytes(const fcsa_problem* p, int32_t total_q) {
  return decode_workspace_bytes(p, {"decode varlen: ", true, nullptr, total_q, 0, false});
}

int fcsa_decode_varlen(const fcsa_problem* p, const int32_t* cu_seqlens_q, int32_t total_q, const fcsa_tensor* q,
                       const fcsa_tensor* k_cache, const fcsa_tensor* v_cache, const int32_t* cache_seqlens,
                       const fcsa_tensor* k_new, const fcsa_tensor* v_new, int32_t groups, const fcsa_tensor* o,
                       void* workspace, size_t workspace_bytes, void* stream) {
  return decode_impl(p, {"decode varlen: ", true, cu_seqlens_q, total_q, 0, false}, q, k_cache, v_cache, cache_seqlens,
                     k_new, v_new, groups, o, workspace, workspace_bytes, stream);
}

size_t fcsa_decode_rolling_workspace_bytes(const fcsa_problem* p, const int32_t* cu_seqlens_q, int32_t total_q) {
  return decode_workspace_bytes(p, {"decode rolling: ", cu_seqlens_q != nullptr, cu_seqlens_q, total_q, 0, true});
}

int fcsa_decode_rolling(const fcsa_problem* p, const int32_t* cu_seqlens_q, int32_t total_q, const fcsa_tensor* q,
                        const fcsa_tensor* k_cache, const fcsa_tensor* v_cache, const int32_t* cache_seqlens,
                        const fcsa_tensor* k_new, const fcsa_tensor* v_new, int32_t groups, const fcsa_tensor* o,
                        void* workspace, size_t workspace_bytes, void* stream) {
  return decode_impl(p, {"decode rolling: ", cu_seqlens_q != nullptr, cu_seqlens_q, total_q, 0, true}, q, k_cache,
                     v_cache, cache_seqlens, k_new, v_new, groups, o, workspace, workspace_bytes, stream);
}

int fcsa_forward_fused_varlen(const fcsa_problem* p, const fcsa_varlen* vl, const fcsa_tensor* q, const fcsa_tensor* k,
                              const fcsa_tensor* v, const fcsa_l2norm* n, const fcsa_tensor* o, float* inv_l,
                              void* stream) {
  int r;
  if ((r = check_varlen(p, vl))) return r;
  if (!n) return fail(FCSA_ERR_INVALID, "null fcsa_l2norm");
  if ((r = check_tensor(q, "q")) || (r = check_tensor(k, "k")) || (r = check_tensor(v, "v")) ||
      (r = check_tensor(o, "o")))
    return r;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  // the row pass runs over the packed rows as one batch: rnorm is [heads][total][groups]
  const bool fused = n->groups != 0;
  if (fused && (r = l2norm_qk(p, n, q, k, 1, vl->total_q, vl->total_k, s))) return r;
  const fcsa_tensor *qa = fused ? &n->q_hat : q, *ka = fused ? &n->k_hat : k;
  r = dispatch(p, [&](auto t, auto d) {
    return launch_forward<typename decltype(t)::type, decltype(d)::value, false, true>(p, qa, ka, v, o, inv_l, s,
                                                                                       nullptr, vl);
  });
  if (r) return r;
  // o = 0 in the rows outside every sequence
  fcsa::TailArgs ta = {};
  ta.t[0] = {o->ptr, o->sh, o->sn, p->heads, vl->total_q, vl->cu_seqlens_q};
  return launch_varlen_tail(p, ta, 1, s);
}

size_t fcsa_backward_fused_varlen_workspace_bytes(const fcsa_problem* p, const fcsa_varlen* vl) {
  return check_varlen(p, vl) ? 0 : bwd_need(p, vl, false).scratch;
}

size_t fcsa_backward_fused_varlen_zeroed_bytes(const fcsa_problem* p, const fcsa_varlen* vl) {
  return check_varlen(p, vl) ? 0 : bwd_need(p, vl, false).zeroed;
}

int fcsa_backward_fused_varlen(const fcsa_problem* p, const fcsa_varlen* vl, const fcsa_l2norm* n,
                               const fcsa_tensor* v, const fcsa_tensor* o, const fcsa_tensor* d_o, const float* inv_l,
                               const fcsa_tensor* dq, const fcsa_tensor* dk, const fcsa_tensor* dv, void* workspace,
                               size_t workspace_bytes, void* zeroed, size_t zeroed_bytes, void* stream) {
  return backward_l2norm(p, true, vl, n, v, o, d_o, inv_l, dq, dk, dv, workspace, workspace_bytes, zeroed,
                         zeroed_bytes, stream, false);
}

size_t fcsa_backward_fused_deterministic_varlen_workspace_bytes(const fcsa_problem* p, const fcsa_varlen* vl) {
  return check_varlen(p, vl) ? 0 : bwd_need(p, vl, true).scratch;
}

int fcsa_backward_fused_deterministic_varlen(const fcsa_problem* p, const fcsa_varlen* vl, const fcsa_l2norm* n,
                                             const fcsa_tensor* v, const fcsa_tensor* o, const fcsa_tensor* d_o,
                                             const float* inv_l, const fcsa_tensor* dq, const fcsa_tensor* dk,
                                             const fcsa_tensor* dv, void* workspace, size_t workspace_bytes,
                                             void* stream) {
  return backward_l2norm(p, true, vl, n, v, o, d_o, inv_l, dq, dk, dv, workspace, workspace_bytes, nullptr, 0, stream,
                         true);
}

}  // extern "C"
