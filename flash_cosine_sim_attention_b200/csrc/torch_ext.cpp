// PyTorch extension module over the C ABI of libfcsa_b200.so.
//
// This is the module the reference builds from its .cu with setup.py (setup.py:30-39) and imports
// by its versioned name (flash_cosine_sim_attention.py:15-20, version.py:3):
//     flash_cosine_sim_attention_cuda_0_1_40 . forward / backward / debug      (cu:1928-1933)
// with the reference's exact signatures (cu:1630-1639, 1752-1764, 1921), so that even the reference's
// own unmodified flash_cosine_sim_attention.py loads it.  All compute happens behind
// include/fcsa_b200.h; this file only does what the reference's host op did around its launches
// (cu:1640-1700, 1766-1830): shape canonicalisation, allocation of the outputs, the current stream.
// Extra entry points (forward_ex / backward_ex / l2norm_*) expose the fused-l2norm and explicit-shift
// variants the Python operator layer uses; they keep the per-call host cost at a few microseconds.
//
// No kernels, no CUDA code here: this file is compiled by the host C++ compiler only.
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include <map>
#include <mutex>
#include <tuple>

#include "../../include/fcsa_b200.h"

namespace {

using at::Tensor;
using c10::optional;

#define FCSA_CHECK(call)                                                                      \
  do {                                                                                        \
    const int rc_ = (call);                                                                   \
    TORCH_CHECK(rc_ == FCSA_OK, "libfcsa_b200 error ", rc_, ": ", fcsa_last_error());          \
  } while (0)

int32_t dtype_code(const Tensor& t) {
  if (t.scalar_type() == at::kHalf) return FCSA_F16;
  if (t.scalar_type() == at::kBFloat16) return FCSA_BF16;
  TORCH_CHECK(false, "flash_cosine_sim_attention (sm_90a): dtype ", t.scalar_type(),
              " has no fused kernel behind this entry point (float16 / bfloat16 only)");
}

// Tensor usable behind a TMA tensor map as is: feature dim contiguous, 16-byte aligned base and
// (batch, head, row) strides, no stride-0 (expanded) dimension of extent > 1.  Otherwise a contiguous
// copy (e.g. the expanded grad of `o.sum().backward()`, head-expanded keys).
Tensor tma_ready(const Tensor& t) {
  const int64_t nd = t.dim();
  bool ok = t.stride(nd - 1) == 1 && (reinterpret_cast<uintptr_t>(t.data_ptr()) % 16) == 0;
  for (int64_t d = 0; ok && d < nd - 1; ++d) {
    const int64_t s = t.stride(d);
    ok = (s % 8 == 0) && (s > 0 || t.size(d) == 1);
  }
  return ok ? t : t.contiguous();
}

// canonical (batch, head, row, feature) addressing: 4-D as is, 3-D (batch, row, feature) = one head
fcsa_tensor view4(const Tensor& t) {
  fcsa_tensor v;
  v.ptr = t.data_ptr();
  if (t.dim() == 4) {
    v.sb = t.stride(0); v.sh = t.stride(1); v.sn = t.stride(2);
  } else {
    v.sb = t.stride(0); v.sh = 0; v.sn = t.stride(1);
  }
  return v;
}

// shape canonicalisation of the reference's host op (cu:1647-1660, cu:1679)
struct Shapes {
  bool merged;
  int64_t B, H, kv_heads, Nq, Nk, D;
  Shapes(const Tensor& q, const Tensor& k, const Tensor& v) {
    merged = q.dim() == 3;
    if (merged) {
      TORCH_CHECK(k.dim() == 3 && v.dim() == 3,
                  "if batch and heads are merged for queries, keys and values must also similarly have only 3 dimensions");
      B = q.size(0); Nq = q.size(1); D = q.size(2); H = 1; kv_heads = 1;
    } else {
      TORCH_CHECK(q.dim() == 4, "queries must be (batch, heads, seq, dim) or (batch*heads, seq, dim)");
      B = q.size(0); H = q.size(1); Nq = q.size(2); D = q.size(3);
      if (k.dim() == 3) {
        TORCH_CHECK(v.dim() == 3, "keys and values must both be single-headed");
        kv_heads = 1;
      } else {
        TORCH_CHECK(k.dim() == 4 && v.dim() == 4, "keys and values must be 3- or 4-dimensional");
        // grouped-query attention: query head h reads key/value head h / (H / kv_heads)
        kv_heads = k.size(1);
        TORCH_CHECK(v.size(1) == kv_heads, "keys and values must have the same number of heads (kv_heads ", kv_heads,
                    " vs ", v.size(1), ")");
        TORCH_CHECK(kv_heads > 0 && H % kv_heads == 0, "kv_heads (", kv_heads, ") must divide the query heads (", H,
                    ")");
      }
    }
    Nk = k.size(-2);
    TORCH_CHECK(k.size(-1) == D && v.size(-1) == D, "head dimensions of q, k, v must match");
    TORCH_CHECK(k.size(0) == B && v.size(0) == B, "batch sizes of q, k, v must match");
    TORCH_CHECK(v.size(-2) == Nk, "keys and values must have the same length");
    TORCH_CHECK(q.is_cuda() && k.is_cuda() && v.is_cuda(),
                "flash_cosine_sim_attention: CUDA tensors required - this build has no CPU path");
    TORCH_CHECK(k.scalar_type() == q.scalar_type() && v.scalar_type() == q.scalar_type(),
                "q, k, v must share one dtype");
  }
};

// The problem of every entry point; `who` prefixes the message of a window out of range ("" / "decode: " / "varlen: ").
// dtype: q's; window: sliding-window attention (0 = none); the library rejects a negative one.
fcsa_problem build_problem(const char* who, const Tensor& q, int64_t B, int64_t H, int64_t kv_heads, int64_t Nq,
                           int64_t Nk, int64_t D, double scale, double shift, bool causal,
                           const optional<Tensor>& mask_u8, bool out_f32, int64_t window) {
  TORCH_CHECK(window >= 0 && window <= 0x7FFFFFFF, who, "window must be a non-negative int32 (0 = none), got ", window);
  fcsa_problem p;
  p.out_f32 = out_f32 ? 1 : 0;
  p.window = (int32_t)window;
  p.dtype = dtype_code(q);
  p.batch = (int32_t)B; p.heads = (int32_t)H; p.kv_heads = (int32_t)kv_heads;
  p.seq_q = (int32_t)Nq; p.seq_k = (int32_t)Nk; p.head_dim = (int32_t)D;
  p.causal = causal ? 1 : 0;
  p.scale = (float)scale; p.shift = (float)shift;
  if (mask_u8.has_value()) {
    p.key_mask = reinterpret_cast<const uint8_t*>(mask_u8->data_ptr());
    p.key_mask_stride = mask_u8->stride(0);
  } else {
    p.key_mask = nullptr;
    p.key_mask_stride = 0;
  }
  return p;
}

// the problem of q, k, v as Shapes canonicalised them
fcsa_problem make_problem(const Shapes& sh,const Tensor& q, double scale, double shift, bool causal,
                          const optional<Tensor>& mask_u8, bool out_f32, int64_t window) {
  return build_problem("", q, sh.B, sh.H, sh.kv_heads, sh.Nq, sh.Nk, sh.D, scale, shift, causal, mask_u8, out_f32,
                       window);
}

// key-padding mask (batch, seq_k), True = attend -> contiguous bytes
optional<Tensor> prep_mask(const optional<Tensor>& mask, const Shapes& sh) {
  if (!mask.has_value() || !mask->defined()) return c10::nullopt;
  TORCH_CHECK(mask->dim() == 2 && mask->size(0) == sh.B && mask->size(1) == sh.Nk, "mask must be (batch, seq_k) = (",
              sh.B, ", ", sh.Nk, ")");
  return mask->to(at::kBool).contiguous();
}

// (heads, i, j) - or (batch, i, j) when batch_dim - bias -> tensor in q's dtype whose rows are 16-byte
// aligned (row length padded to a multiple of 8) + the fcsa_bias addressing it as [batch][head][i][j]
Tensor prep_bias(const Tensor& bias, const Shapes& sh, at::ScalarType dtype, bool batch_dim) {
  const int64_t lead = batch_dim ? sh.B : sh.H;
  TORCH_CHECK(bias.dim() == 3 && bias.size(0) == lead && bias.size(1) == sh.Nq && bias.size(2) == sh.Nk,
              "attn_bias must be (", lead, ", ", sh.Nq, ", ", sh.Nk, ") (", batch_dim ? "batch" : "heads", ", i, j)");
  TORCH_CHECK(bias.is_cuda(), "attn_bias must be a CUDA tensor");
  Tensor t = bias.detach().to(dtype);
  const int64_t pad = (8 - sh.Nk % 8) % 8;
  if (pad) t = at::constant_pad_nd(t, {0, pad});
  t = t.contiguous();
  if (reinterpret_cast<uintptr_t>(t.data_ptr()) % 16) t = t.clone();
  return t;
}

fcsa_bias bias_struct(const Tensor& t, bool batch_dim, const optional<Tensor>& amax) {
  fcsa_bias b;
  b.ptr = t.data_ptr();
  const int64_t plane = t.stride(0);
  if (batch_dim) { b.sb = plane; b.sh = 0; } else { b.sb = 0; b.sh = plane; }
  b.sn = t.stride(1);
  b.amax = (amax.has_value() && amax->defined()) ? amax->data_ptr<float>() : nullptr;
  return b;
}

// Backward workspaces, one pair per (device, stream): `scratch` (contents irrelevant) and `zeroed`
// (fp32 dq accumulator + tile counters; zero-filled once, left zero by every backward).  Only grow.
struct Workspaces {
  Tensor scratch, zeroed;
};
std::mutex g_ws_mutex;
std::map<std::pair<int, void*>, Workspaces> g_ws;

// The workspaces of (like's device, stream), grown to need_s scratch and need_z zeroed bytes.  A size of 0 is the
// library's refusal of the problem.  with_zeroed = false (decode) needs the scratch only.
Workspaces workspaces_of_size(size_t need_s, size_t need_z, const Tensor& like, cudaStream_t stream,
                              bool with_zeroed = true) {
  TORCH_CHECK(need_s > 0 && (need_z > 0 || !with_zeroed), "libfcsa_b200: ", fcsa_last_error());
  std::lock_guard<std::mutex> lock(g_ws_mutex);
  Workspaces& w = g_ws[{(int)like.get_device(), (void*)stream}];
  const auto opts = like.options().dtype(at::kByte);
  if (!w.scratch.defined() || (size_t)w.scratch.numel() < need_s) w.scratch = at::empty({(int64_t)need_s}, opts);
  if (with_zeroed && (!w.zeroed.defined() || (size_t)w.zeroed.numel() < need_z)) {
    w.zeroed = at::empty({(int64_t)need_z}, opts);
    FCSA_CHECK(fcsa_zeroed_init(w.zeroed.data_ptr(), need_z, stream));
  }
  return w;
}

Workspaces backward_workspaces(const fcsa_problem& p, const Tensor& like, cudaStream_t stream) {
  return workspaces_of_size(fcsa_backward_workspace_bytes(&p), fcsa_backward_zeroed_bytes(&p), like, stream);
}

// ------------------------------------------------------------------------------------------------
// l2norm (flash_cosine_sim_attention.py:38-65)
// ------------------------------------------------------------------------------------------------
std::tuple<Tensor, Tensor> l2norm_forward(const Tensor& x_in, int64_t groups) {
  TORCH_CHECK(x_in.is_cuda() && (x_in.dim() == 3 || x_in.dim() == 4), "l2norm: 3-D or 4-D CUDA tensor expected");
  const c10::cuda::CUDAGuard guard(x_in.device());
  const Tensor x = tma_ready(x_in);
  const int64_t B = x.size(0), H = x.dim() == 4 ? x.size(1) : 1, N = x.size(-2), D = x.size(-1);
  Tensor y = at::empty(x.sizes(), x.options());
  Tensor rnorm = at::empty({B, H, N, groups}, x.options().dtype(at::kFloat));
  const fcsa_tensor tx = view4(x), ty = view4(y);
  FCSA_CHECK(fcsa_l2norm_forward(dtype_code(x), (int32_t)B, (int32_t)H, (int32_t)N, (int32_t)D, (int32_t)groups, &tx,
                                 &ty, rnorm.data_ptr<float>(), at::cuda::getCurrentCUDAStream().stream()));
  return {y, rnorm};
}

Tensor l2norm_backward(const Tensor& dy_in, const Tensor& y_in, const Tensor& rnorm, int64_t groups) {
  const c10::cuda::CUDAGuard guard(y_in.device());
  const Tensor dy = tma_ready(dy_in), y = tma_ready(y_in);
  const int64_t B = y.size(0), H = y.dim() == 4 ? y.size(1) : 1, N = y.size(-2), D = y.size(-1);
  Tensor dx = at::empty(y.sizes(), y.options());
  const fcsa_tensor tdy = view4(dy), ty = view4(y), tdx = view4(dx);
  FCSA_CHECK(fcsa_l2norm_backward(dtype_code(y), (int32_t)B, (int32_t)H, (int32_t)N, (int32_t)D, (int32_t)groups,
                                  &tdy, &ty, rnorm.data_ptr<float>(), &tdx,
                                  at::cuda::getCurrentCUDAStream().stream()));
  return dx;
}

// ------------------------------------------------------------------------------------------------
// float32 front end: (l2norm +) cast of a float32 tensor to the 16-bit operand dtype, and its backward
// ------------------------------------------------------------------------------------------------
// x: float32 (b, h, n, d) or (b, n, d); returns y (16 bit, `pad_to` >= d features, zero-padded) and rnorm (groups > 0)
std::tuple<Tensor, Tensor> f32_cast(const Tensor& x_in, bool to_bf16, int64_t groups, const optional<Tensor>& mul,
                                    bool mul_reciprocal, int64_t pad_to) {
  TORCH_CHECK(x_in.is_cuda() && x_in.scalar_type() == at::kFloat && (x_in.dim() == 3 || x_in.dim() == 4),
              "f32_cast: 3-D or 4-D float32 CUDA tensor expected");
  const c10::cuda::CUDAGuard guard(x_in.device());
  const Tensor x = (x_in.stride(-1) == 1 && reinterpret_cast<uintptr_t>(x_in.data_ptr()) % 16 == 0) ? x_in : x_in.contiguous();
  const int64_t B = x.size(0), H = x.dim() == 4 ? x.size(1) : 1, N = x.size(-2), D = x.size(-1);
  std::vector<int64_t> shape = x.sizes().vec();
  shape.back() = std::max(pad_to, D);
  const auto hopt = x.options().dtype(to_bf16 ? at::kBFloat16 : at::kHalf);
  Tensor y = shape.back() == D ? at::empty(shape, hopt) : at::zeros(shape, hopt);
  Tensor rnorm;
  if (groups > 0) rnorm = at::empty({B, H, N, groups}, x.options());
  const fcsa_tensor tx = view4(x), ty = view4(y);
  FCSA_CHECK(fcsa_f32_cast(to_bf16 ? FCSA_BF16 : FCSA_F16, (int32_t)B, (int32_t)H, (int32_t)N, (int32_t)D, (int32_t)groups,
                           &tx, &ty, groups > 0 ? rnorm.data_ptr<float>() : nullptr,
                           (mul.has_value() && mul->defined()) ? mul->data_ptr<float>() : nullptr, mul_reciprocal ? 1 : 0,
                           at::cuda::getCurrentCUDAStream().stream()));
  return {y, rnorm};
}

// dy: float32 gradient w.r.t. y (may carry padded features: only the first d are read); y / rnorm: what f32_cast
// returned (groups > 0); returns the float32 gradient w.r.t. x with d features
Tensor f32_cast_backward(const Tensor& dy_in, const optional<Tensor>& y, const optional<Tensor>& rnorm, int64_t groups,
                         const optional<Tensor>& mul, bool mul_reciprocal, int64_t d) {
  TORCH_CHECK(dy_in.is_cuda() && dy_in.scalar_type() == at::kFloat, "f32_cast_backward: float32 CUDA gradient expected");
  const c10::cuda::CUDAGuard guard(dy_in.device());
  const Tensor dy = (dy_in.stride(-1) == 1 && reinterpret_cast<uintptr_t>(dy_in.data_ptr()) % 16 == 0) ? dy_in : dy_in.contiguous();
  const int64_t B = dy.size(0), H = dy.dim() == 4 ? dy.size(1) : 1, N = dy.size(-2);
  std::vector<int64_t> shape = dy.sizes().vec();
  shape.back() = d;
  Tensor dx = at::empty(shape, dy.options());
  const fcsa_tensor tdy = view4(dy), tdx = view4(dx);
  fcsa_tensor ty = {nullptr, 0, 0, 0};
  bool bf = false;
  if (groups > 0) {
    TORCH_CHECK(y.has_value() && y->defined() && rnorm.has_value() && rnorm->defined(), "f32_cast_backward: y and rnorm needed");
    ty = view4(*y);
    bf = y->scalar_type() == at::kBFloat16;
  }
  FCSA_CHECK(fcsa_f32_cast_backward(bf ? FCSA_BF16 : FCSA_F16, (int32_t)B, (int32_t)H, (int32_t)N, (int32_t)d,
                                    (int32_t)groups, &tdy, &ty, groups > 0 ? rnorm->data_ptr<float>() : nullptr, &tdx,
                                    (mul.has_value() && mul->defined()) ? mul->data_ptr<float>() : nullptr,
                                    mul_reciprocal ? 1 : 0, at::cuda::getCurrentCUDAStream().stream()));
  return dx;
}

// ------------------------------------------------------------------------------------------------
// forward_ex: the general forward.
//   l2norm_groups > 0 : q, k are RAW; they are normalised over that many groups by the fused pre-pass
//                       (returns q_hat, k_hat, q_rnorm, k_rnorm for the backward); no bias on this path
//   l2norm_groups == 0: q, k are used as given (already normalised, or l2norm_qk=False)
//   bias_prepared     : the tensor prep_bias() made (saved by the caller for the backward), optional
//   bias_amax         : optional fp32 device scalar; the kernels add max(amax, 0) to `shift` (fp16 range)
//   out_f32           : o is returned as float32 (fp32 accumulator, no rounding to 16 bit) - float32 callers
// returns (o, inv_l, q_hat, k_hat, q_rnorm, k_rnorm) - the last four undefined when l2norm_groups == 0
// ------------------------------------------------------------------------------------------------
std::tuple<Tensor, Tensor, Tensor, Tensor, Tensor, Tensor> forward_ex(
    const Tensor& q_in, const Tensor& k_in, const Tensor& v_in, const optional<Tensor>& mask,
    const optional<Tensor>& bias_prepared, bool bias_batch_dim, const optional<Tensor>& bias_amax, double scale,
    double shift, bool causal, int64_t l2norm_groups, bool need_inv_l, bool out_f32, int64_t window) {
  const Shapes sh(q_in, k_in, v_in);
  TORCH_CHECK(!(causal && mask.has_value() && mask->defined()), "mask should not be supplied if causality is needed");
  const c10::cuda::CUDAGuard guard(q_in.device());
  const Tensor q = tma_ready(q_in), k = tma_ready(k_in), v = tma_ready(v_in);
  const optional<Tensor> mask_u8 = prep_mask(mask, sh);
  const fcsa_problem p = make_problem(sh, q, scale, shift, causal, mask_u8, out_f32, window);
  Tensor o = at::empty(q.sizes(), out_f32 ? q.options().dtype(at::kFloat) : q.options());   // out_f32: no final rounding
  Tensor inv_l;
  if (need_inv_l) inv_l = at::empty({sh.B, sh.H, sh.Nq}, q.options().dtype(at::kFloat));
  float* inv_l_ptr = need_inv_l ? inv_l.data_ptr<float>() : nullptr;
  const fcsa_tensor tq = view4(q), tk = view4(k), tv = view4(v), to = view4(o);
  cudaStream_t stream = at::cuda::getCurrentCUDAStream().stream();
  const bool has_bias = bias_prepared.has_value() && bias_prepared->defined();
  Tensor qn, kn, rq, rk;
  if (l2norm_groups > 0) {
    TORCH_CHECK(!has_bias, "forward_ex: the fused-l2norm path takes no attn_bias (normalise first)");
    qn = at::empty(q.sizes(), q.options());
    kn = at::empty(k.sizes(), k.options());
    rq = at::empty({sh.B, sh.H, sh.Nq, l2norm_groups}, q.options().dtype(at::kFloat));
    rk = at::empty({sh.B, sh.kv_heads, sh.Nk, l2norm_groups}, q.options().dtype(at::kFloat));
    fcsa_l2norm n;
    n.groups = (int32_t)l2norm_groups;
    n.q_hat = view4(qn); n.k_hat = view4(kn);
    n.q_rnorm = rq.data_ptr<float>(); n.k_rnorm = rk.data_ptr<float>();
    FCSA_CHECK(fcsa_forward_fused(&p, &tq, &tk, &tv, &n, &to, inv_l_ptr, stream));
  } else if (has_bias) {
    const fcsa_bias b = bias_struct(*bias_prepared, bias_batch_dim, bias_amax);
    FCSA_CHECK(fcsa_forward_bias(&p, &tq, &tk, &tv, &b, &to, inv_l_ptr, stream));
  } else {
    FCSA_CHECK(fcsa_forward(&p, &tq, &tk, &tv, &to, inv_l_ptr, stream));
  }
  return {o, inv_l, qn, kn, rq, rk};
}

// ------------------------------------------------------------------------------------------------
// backward_ex: gradients of forward_ex.
//   groups > 0 (with q_rnorm, k_rnorm): q, k are the NORMALISED tensors forward_ex returned and dq, dk
//                       are gradients w.r.t. the raw ones (l2norm backward fused)
//   bias_prepared + bias_grad: d_bias accumulated in fp32, returned in `bias_dtype_like`'s dtype / shape
//   deterministic     : the backward without atomics (fcsa_backward_fused_deterministic): bitwise reproducible
//                       dq, dk, dv; scratch only, no zeroed workspace; no bias
// returns (dq, dk, dv, d_bias or undefined)
// ------------------------------------------------------------------------------------------------
std::tuple<Tensor, Tensor, Tensor, Tensor> backward_ex(
    const Tensor& d_out, const Tensor& o_in, const Tensor& inv_l, const Tensor& q_in, const Tensor& k_in,
    const Tensor& v_in, const optional<Tensor>& q_rnorm, const optional<Tensor>& k_rnorm,
    const optional<Tensor>& mask, const optional<Tensor>& bias_prepared, bool bias_batch_dim,
    const optional<Tensor>& bias_amax, bool bias_grad, const optional<Tensor>& bias_like, double scale, double shift,
    bool causal, int64_t groups, bool out_f32, int64_t window, bool deterministic) {
  const Shapes sh(q_in, k_in, v_in);
  const c10::cuda::CUDAGuard guard(q_in.device());
  const Tensor q = tma_ready(q_in), k = tma_ready(k_in), v = tma_ready(v_in), o = tma_ready(o_in),
               d_o = tma_ready(d_out);
  TORCH_CHECK(d_o.sizes() == q.sizes() && d_o.scalar_type() == q.scalar_type(),
              "d_out must have the shape and dtype of the queries");
  const optional<Tensor> mask_u8 = prep_mask(mask, sh);
  const fcsa_problem p = make_problem(sh, q, scale, shift, causal, mask_u8, out_f32, window);
  TORCH_CHECK(o.scalar_type() == (out_f32 ? at::kFloat : q.scalar_type()), "backward_ex: `o` must be ",
              out_f32 ? "float32 (out_f32)" : "in the operand dtype");
  const auto gopt = out_f32 ? q.options().dtype(at::kFloat) : q.options();     // out_f32: float32 gradients
  Tensor dq = at::empty(q.sizes(), gopt);
  Tensor dk = at::empty(k.sizes(), gopt);
  Tensor dv = at::empty(v.sizes(), gopt);
  cudaStream_t stream = at::cuda::getCurrentCUDAStream().stream();
  const fcsa_tensor tq = view4(q), tk = view4(k), tv = view4(v), to = view4(o), tdo = view4(d_o), tdq = view4(dq),
                    tdk = view4(dk), tdv = view4(dv);
  const bool has_bias = bias_prepared.has_value() && bias_prepared->defined();
  const bool fused = q_rnorm.has_value() && q_rnorm->defined();
  Tensor db;
  if (deterministic) {
    TORCH_CHECK(!has_bias, "backward_ex: the deterministic backward takes no attn_bias");
    const Tensor scratch =
        workspaces_of_size(fcsa_backward_fused_deterministic_workspace_bytes(&p), 0, q, stream, false).scratch;
    fcsa_l2norm n;
    n.groups = fused ? (int32_t)groups : 0;
    n.q_hat = tq; n.k_hat = tk;
    n.q_rnorm = n.k_rnorm = nullptr;
    if (fused) {
      TORCH_CHECK(k_rnorm.has_value() && k_rnorm->defined() && groups > 0, "backward_ex: bad fused-l2norm arguments");
      n.q_rnorm = q_rnorm->data_ptr<float>(); n.k_rnorm = k_rnorm->data_ptr<float>();
    }
    FCSA_CHECK(fcsa_backward_fused_deterministic(&p, &n, &tv, &to, &tdo, inv_l.data_ptr<float>(), &tdq, &tdk, &tdv,
                                                 scratch.data_ptr(), (size_t)scratch.numel(), stream));
    return {dq, dk, dv, db};
  }
  const Workspaces ws = backward_workspaces(p, q, stream);
  void* wsp = ws.scratch.data_ptr();
  void* zsp = ws.zeroed.data_ptr();
  const size_t wsn = (size_t)ws.scratch.numel(), zsn = (size_t)ws.zeroed.numel();
  if (fused) {
    TORCH_CHECK(!has_bias && k_rnorm.has_value() && k_rnorm->defined() && groups > 0, "backward_ex: bad fused-l2norm arguments");
    fcsa_l2norm n;
    n.groups = (int32_t)groups;
    n.q_hat = tq; n.k_hat = tk;
    n.q_rnorm = q_rnorm->data_ptr<float>(); n.k_rnorm = k_rnorm->data_ptr<float>();
    FCSA_CHECK(fcsa_backward_fused(&p, &n, &tv, &to, &tdo, inv_l.data_ptr<float>(), &tdq, &tdk, &tdv, wsp, wsn, zsp,
                                   zsn, stream));
  } else if (has_bias) {
    const fcsa_bias b = bias_struct(*bias_prepared, bias_batch_dim, bias_amax);
    Tensor db_acc;
    float* db_ptr = nullptr;
    const int64_t plane = sh.Nq * sh.Nk;
    if (bias_grad) {
      db_acc = at::zeros({bias_batch_dim ? sh.B : sh.H, sh.Nq, sh.Nk}, q.options().dtype(at::kFloat));
      db_ptr = db_acc.data_ptr<float>();
    }
    FCSA_CHECK(fcsa_backward_bias(&p, &tq, &tk, &tv, &to, &tdo, inv_l.data_ptr<float>(), &b, db_ptr,
                                  bias_batch_dim ? plane : 0, bias_batch_dim ? 0 : plane, &tdq, &tdk, &tdv, wsp, wsn,
                                  zsp, zsn, stream));
    if (bias_grad)
      db = (bias_like.has_value() && bias_like->defined()) ? db_acc.to(bias_like->scalar_type()) : db_acc;
  } else {
    FCSA_CHECK(fcsa_backward(&p, &tq, &tk, &tv, &to, &tdo, inv_l.data_ptr<float>(), &tdq, &tdk, &tdv, wsp, wsn, zsp,
                             zsn, stream));
  }
  return {dq, dk, dv, db};
}

// ------------------------------------------------------------------------------------------------
// the reference's surface (cu:1630-1639, 1752-1764, 1921): q, k already normalised, shift = scale
// ------------------------------------------------------------------------------------------------
std::tuple<Tensor, Tensor, bool> forward(const Tensor& q, const Tensor& k, const Tensor& v,
                                         const optional<Tensor>& mask, const optional<Tensor>& attn_bias,
                                         bool attn_bias_batch_dim, double scale, bool causal) {
  const Shapes sh(q, k, v);
  if (sh.merged) attn_bias_batch_dim = true;   // cu:1647-1654
  const bool has_bias = attn_bias.has_value() && attn_bias->defined();
  const bool should_backwards =
      q.requires_grad() || k.requires_grad() || v.requires_grad() || (has_bias && attn_bias->requires_grad());
  optional<Tensor> bias_prepared;
  if (has_bias) bias_prepared = prep_bias(*attn_bias, sh, q.scalar_type(), attn_bias_batch_dim);
  auto r = forward_ex(q, k, v, mask, bias_prepared, attn_bias_batch_dim, c10::nullopt, scale, scale, causal, 0, true,
                      false, 0);
  return {std::get<0>(r), std::get<1>(r), should_backwards};
}

std::tuple<Tensor, Tensor, Tensor, optional<Tensor>> backward(
    const Tensor& d_out, const Tensor& o, const Tensor& l, const Tensor& q, const Tensor& k, const Tensor& v,
    const optional<Tensor>& mask, const optional<Tensor>& attn_bias, bool attn_bias_batch_dim, double scale,
    bool causal) {
  const Shapes sh(q, k, v);
  if (sh.merged) attn_bias_batch_dim = true;
  const bool has_bias = attn_bias.has_value() && attn_bias->defined();
  optional<Tensor> bias_prepared;
  if (has_bias) bias_prepared = prep_bias(*attn_bias, sh, q.scalar_type(), attn_bias_batch_dim);
  auto r = backward_ex(d_out, o, l, q, k, v, c10::nullopt, c10::nullopt, mask, bias_prepared, attn_bias_batch_dim,
                       c10::nullopt, has_bias && attn_bias->requires_grad(), attn_bias, scale, scale, causal, 0, false, 0,
                       false);
  optional<Tensor> db;
  if (std::get<3>(r).defined()) db = std::get<3>(r);
  return {std::get<0>(r), std::get<1>(r), std::get<2>(r), db};
}

// ------------------------------------------------------------------------------------------------
// decode: new queries against a key/value cache, appending k / v at row cache_seqlens[b] (fcsa_decode).
//   q (B, H, Nq, D); k_cache, v_cache (B, kv_heads, capacity, D), written in place, so they must be usable as they
//   are (no copy); cache_seqlens int32 on q's device; k, v (B, kv_heads, n_new, D) or both None; groups > 0:
//   l2-normalise q and k over that many groups.  Returns o (B, H, Nq, D).  Scratch comes from the per-(device,
//   stream) workspace of the backward, whose contents are irrelevant on entry.
// ------------------------------------------------------------------------------------------------
Tensor decode(const Tensor& q_in, const Tensor& k_cache, const Tensor& v_cache, const Tensor& cache_seqlens,
              const optional<Tensor>& k_in, const optional<Tensor>& v_in, double scale, double shift, bool causal,
              int64_t groups, int64_t window) {
  TORCH_CHECK(q_in.dim() == 4 && k_cache.dim() == 4 && v_cache.dim() == 4,
              "decode: q, k_cache, v_cache must be (batch, heads, seq, head_dim)");
  TORCH_CHECK(q_in.is_cuda() && k_cache.is_cuda() && v_cache.is_cuda(), "decode: CUDA tensors required");
  TORCH_CHECK(k_cache.scalar_type() == q_in.scalar_type() && v_cache.scalar_type() == q_in.scalar_type(),
              "decode: q and the caches must share one dtype");
  TORCH_CHECK(k_cache.sizes() == v_cache.sizes(), "decode: k_cache and v_cache must have the same shape");
  const int64_t B = q_in.size(0), H = q_in.size(1), Nq = q_in.size(2), D = q_in.size(3);
  const int64_t Hk = k_cache.size(1), cap = k_cache.size(2);
  TORCH_CHECK(k_cache.size(0) == B && k_cache.size(3) == D, "decode: caches must be (", B, ", kv_heads, capacity, ", D,
              ")");
  TORCH_CHECK(Hk > 0 && H % Hk == 0, "decode: kv_heads (", Hk, ") must divide the query heads (", H, ")");
  TORCH_CHECK(cache_seqlens.is_cuda() && cache_seqlens.get_device() == q_in.get_device() &&
                  cache_seqlens.scalar_type() == at::kInt && cache_seqlens.dim() == 1 && cache_seqlens.size(0) == B,
              "decode: cache_seqlens must be an int32 tensor of shape (", B, ") on q's device");
  // the kernels index it as a dense array; a copy would also break graph capture (a replay must read the caller's
  // buffer), so a strided or expanded view is refused
  TORCH_CHECK(cache_seqlens.is_contiguous(), "decode: cache_seqlens must be contiguous (not a strided or expanded view)");
  TORCH_CHECK(tma_ready(k_cache).data_ptr() == k_cache.data_ptr() && tma_ready(v_cache).data_ptr() == v_cache.data_ptr(),
              "decode: the caches are written in place and must be usable as they are: contiguous head dim, "
              "16-byte aligned base and strides, no expanded dimension");
  const bool has_new = k_in.has_value() && k_in->defined();
  TORCH_CHECK(has_new == (v_in.has_value() && v_in->defined()), "decode: pass both k and v, or neither");
  int64_t n_new = 0;
  Tensor k, v;
  if (has_new) {
    TORCH_CHECK(k_in->dim() == 4 && k_in->sizes() == v_in->sizes() && k_in->size(0) == B && k_in->size(1) == Hk &&
                    k_in->size(3) == D,
                "decode: k and v must be (", B, ", ", Hk, ", n_new, ", D, ")");
    TORCH_CHECK(k_in->scalar_type() == q_in.scalar_type() && v_in->scalar_type() == q_in.scalar_type() &&
                    k_in->is_cuda() && v_in->is_cuda(),
                "decode: k and v must be CUDA tensors of q's dtype");
    k = tma_ready(*k_in);
    v = tma_ready(*v_in);
    n_new = k.size(2);
  }
  const c10::cuda::CUDAGuard guard(q_in.device());
  const Tensor q = tma_ready(q_in);
  const fcsa_problem p =
      build_problem("decode: ", q, B, H, Hk, Nq, cap, D, scale, shift, causal, c10::nullopt, false, window);
  Tensor o = at::empty({B, H, Nq, D}, q.options());
  cudaStream_t stream = at::cuda::getCurrentCUDAStream().stream();
  const Tensor scratch =
      workspaces_of_size(fcsa_decode_workspace_bytes(&p, (int32_t)n_new), 0, q, stream, false).scratch;
  const fcsa_tensor tq = view4(q), tkc = view4(k_cache), tvc = view4(v_cache), to = view4(o);
  fcsa_tensor tk = {nullptr, 0, 0, 0}, tv = {nullptr, 0, 0, 0};
  if (has_new) { tk = view4(k); tv = view4(v); }
  FCSA_CHECK(fcsa_decode(&p, &tq, &tkc, &tvc, cache_seqlens.data_ptr<int32_t>(), &tk, &tv, (int32_t)n_new,
                         (int32_t)groups, &to, scratch.data_ptr(), (size_t)scratch.numel(), stream));
  return o;
}

// ------------------------------------------------------------------------------------------------
// packed variable-length sequences (fcsa_forward_fused_varlen / fcsa_backward_fused_varlen)
//   q (total_q, H, D), k, v (total_k, kv_heads, D); cu_q, cu_k int32 (B + 1) on q's device, read by the kernels
//   only (never copied: a CUDA graph replay must read the caller's buffers); max_q, max_k >= every length.
// ------------------------------------------------------------------------------------------------
// (total, heads, feature) -> the (batch, head, row) addressing of the ABI: one batch, rows = the packed rows
fcsa_tensor view_packed(const Tensor& t) {
  fcsa_tensor v;
  v.ptr = t.data_ptr();
  v.sb = 0; v.sh = t.stride(1); v.sn = t.stride(0);
  return v;
}

struct Varlen {
  fcsa_problem p;
  fcsa_varlen vl;
};

Varlen varlen_problem(const Tensor& q, const Tensor& k, const Tensor& v, const Tensor& cu_q, const Tensor& cu_k,
                      int64_t max_q, int64_t max_k, double scale, double shift, bool causal, int64_t window) {
  TORCH_CHECK(q.dim() == 3 && k.dim() == 3 && v.dim() == 3,
              "varlen: q must be (total_q, heads, head_dim) and k, v (total_k, kv_heads, head_dim)");
  TORCH_CHECK(q.is_cuda() && k.is_cuda() && v.is_cuda(), "varlen: CUDA tensors required - this build has no CPU path");
  TORCH_CHECK(k.scalar_type() == q.scalar_type() && v.scalar_type() == q.scalar_type(), "varlen: q, k, v must share one dtype");
  TORCH_CHECK(k.sizes() == v.sizes(), "varlen: k and v must have the same shape");
  const int64_t H = q.size(1), Hk = k.size(1), D = q.size(2);
  TORCH_CHECK(k.size(2) == D, "varlen: head dimensions of q, k, v must match");
  TORCH_CHECK(Hk > 0 && H % Hk == 0, "varlen: kv_heads (", Hk, ") must divide the query heads (", H, ")");
  for (const Tensor* c : {&cu_q, &cu_k}) {
    TORCH_CHECK(c->is_cuda() && c->get_device() == q.get_device() && c->scalar_type() == at::kInt && c->dim() == 1 &&
                    c->size(0) >= 2,
                "varlen: cu_seqlens must be int32 tensors of shape (batch + 1,) on q's device");
    TORCH_CHECK(c->is_contiguous(), "varlen: cu_seqlens must be contiguous (not a strided or expanded view)");
  }
  TORCH_CHECK(cu_q.size(0) == cu_k.size(0), "varlen: cu_seqlens_q and cu_seqlens_k must have the same length");
  TORCH_CHECK(max_q >= 1 && max_k >= 1 && max_q <= 0x7FFFFFFF && max_k <= 0x7FFFFFFF,
              "varlen: max_seqlen_q / max_seqlen_k must be positive int32 values");
  TORCH_CHECK(q.size(0) <= 0x7FFFFFFF && k.size(0) <= 0x7FFFFFFF, "varlen: too many packed rows");
  Varlen r;
  r.p = build_problem("varlen: ", q, cu_q.size(0) - 1, H, Hk, max_q, max_k, D, scale, shift, causal, c10::nullopt,
                      false, window);
  r.vl.cu_seqlens_q = cu_q.data_ptr<int32_t>();
  r.vl.cu_seqlens_k = cu_k.data_ptr<int32_t>();
  r.vl.total_q = (int32_t)q.size(0);
  r.vl.total_k = (int32_t)k.size(0);
  return r;
}

// groups > 0: q, k are RAW and l2-normalised inside; returns (o, inv_l, q_hat, k_hat, q_rnorm, k_rnorm), the last four
// undefined when groups == 0, inv_l undefined unless need_inv_l
std::tuple<Tensor, Tensor, Tensor, Tensor, Tensor, Tensor> forward_varlen(
    const Tensor& q_in, const Tensor& k_in, const Tensor& v_in, const Tensor& cu_q, const Tensor& cu_k, int64_t max_q,
    int64_t max_k, double scale, double shift, bool causal, int64_t groups, bool need_inv_l, int64_t window) {
  const c10::cuda::CUDAGuard guard(q_in.device());
  const Tensor q = tma_ready(q_in), k = tma_ready(k_in), v = tma_ready(v_in);
  const Varlen vr = varlen_problem(q, k, v, cu_q, cu_k, max_q, max_k, scale, shift, causal, window);
  const int64_t H = q.size(1), Hk = k.size(1), Tq = q.size(0), Tk = k.size(0);
  Tensor o = at::empty(q.sizes(), q.options());
  Tensor inv_l;
  if (need_inv_l) inv_l = at::empty({H, Tq}, q.options().dtype(at::kFloat));
  Tensor qn, kn, rq, rk;
  fcsa_l2norm n;
  n.groups = (int32_t)groups;
  n.q_hat = n.k_hat = fcsa_tensor{nullptr, 0, 0, 0};
  n.q_rnorm = n.k_rnorm = nullptr;
  if (groups > 0) {
    qn = at::empty(q.sizes(), q.options());
    kn = at::empty(k.sizes(), k.options());
    rq = at::empty({H, Tq, groups}, q.options().dtype(at::kFloat));
    rk = at::empty({Hk, Tk, groups}, q.options().dtype(at::kFloat));
    n.q_hat = view_packed(qn); n.k_hat = view_packed(kn);
    n.q_rnorm = rq.data_ptr<float>(); n.k_rnorm = rk.data_ptr<float>();
  }
  const fcsa_tensor tq = view_packed(q), tk = view_packed(k), tv = view_packed(v), to = view_packed(o);
  FCSA_CHECK(fcsa_forward_fused_varlen(&vr.p, &vr.vl, &tq, &tk, &tv, &n, &to, need_inv_l ? inv_l.data_ptr<float>() : nullptr,
                                       at::cuda::getCurrentCUDAStream().stream()));
  return {o, inv_l, qn, kn, rq, rk};
}

// gradients of forward_varlen w.r.t. the raw q, k (groups > 0: q, k are the normalised tensors it returned) and v;
// deterministic: fcsa_backward_fused_deterministic_varlen (scratch only)
std::tuple<Tensor, Tensor, Tensor> backward_varlen(
    const Tensor& d_out, const Tensor& o_in, const Tensor& inv_l, const Tensor& q_in, const Tensor& k_in,
    const Tensor& v_in, const optional<Tensor>& q_rnorm, const optional<Tensor>& k_rnorm, const Tensor& cu_q,
    const Tensor& cu_k, int64_t max_q, int64_t max_k, double scale, double shift, bool causal, int64_t groups,
    int64_t window, bool deterministic) {
  const c10::cuda::CUDAGuard guard(q_in.device());
  const Tensor q = tma_ready(q_in), k = tma_ready(k_in), v = tma_ready(v_in), o = tma_ready(o_in),
               d_o = tma_ready(d_out);
  const Varlen vr = varlen_problem(q, k, v, cu_q, cu_k, max_q, max_k, scale, shift, causal, window);
  TORCH_CHECK(d_o.sizes() == q.sizes() && d_o.scalar_type() == q.scalar_type() && o.sizes() == q.sizes() &&
                  o.scalar_type() == q.scalar_type(),
              "backward_varlen: o and d_out must have the shape and dtype of the queries");
  TORCH_CHECK(inv_l.scalar_type() == at::kFloat && inv_l.is_contiguous() && inv_l.numel() == q.size(0) * q.size(1),
              "backward_varlen: inv_l must be the (heads, total_q) float32 tensor of the forward");
  Tensor dq = at::empty(q.sizes(), q.options());
  Tensor dk = at::empty(k.sizes(), k.options());
  Tensor dv = at::empty(v.sizes(), v.options());
  cudaStream_t stream = at::cuda::getCurrentCUDAStream().stream();
  fcsa_l2norm n;
  n.groups = (int32_t)groups;
  n.q_hat = view_packed(q); n.k_hat = view_packed(k);
  n.q_rnorm = n.k_rnorm = nullptr;
  if (groups > 0) {
    TORCH_CHECK(q_rnorm.has_value() && q_rnorm->defined() && k_rnorm.has_value() && k_rnorm->defined(),
                "backward_varlen: q_rnorm and k_rnorm are needed with groups > 0");
    n.q_rnorm = q_rnorm->data_ptr<float>(); n.k_rnorm = k_rnorm->data_ptr<float>();
  }
  const fcsa_tensor tv = view_packed(v), to = view_packed(o), tdo = view_packed(d_o), tdq = view_packed(dq),
                    tdk = view_packed(dk), tdv = view_packed(dv);
  if (deterministic) {
    const Tensor scratch = workspaces_of_size(fcsa_backward_fused_deterministic_varlen_workspace_bytes(&vr.p, &vr.vl), 0,
                                              q, stream, false).scratch;
    FCSA_CHECK(fcsa_backward_fused_deterministic_varlen(&vr.p, &vr.vl, &n, &tv, &to, &tdo, inv_l.data_ptr<float>(),
                                                        &tdq, &tdk, &tdv, scratch.data_ptr(),
                                                        (size_t)scratch.numel(), stream));
    return {dq, dk, dv};
  }
  const Workspaces ws = workspaces_of_size(fcsa_backward_fused_varlen_workspace_bytes(&vr.p, &vr.vl),
                                           fcsa_backward_fused_varlen_zeroed_bytes(&vr.p, &vr.vl), q, stream);
  FCSA_CHECK(fcsa_backward_fused_varlen(&vr.p, &vr.vl, &n, &tv, &to, &tdo, inv_l.data_ptr<float>(), &tdq, &tdk, &tdv,
                                        ws.scratch.data_ptr(), (size_t)ws.scratch.numel(), ws.zeroed.data_ptr(),
                                        (size_t)ws.zeroed.numel(), stream));
  return {dq, dk, dv};
}

// Drops the cached backward workspaces of every (device, stream) (they only ever grow: a long-context call leaves a
// 1 GB accumulator behind).  Returns the number of bytes released to the caching allocator.  Safe at any time between
// calls: buffers still referenced by enqueued kernels stay alive through the allocator's stream semantics.
int64_t release_workspaces() {
  std::lock_guard<std::mutex> lock(g_ws_mutex);
  int64_t bytes = 0;
  for (auto& kv : g_ws) {
    if (kv.second.scratch.defined()) bytes += kv.second.scratch.numel();
    if (kv.second.zeroed.defined()) bytes += kv.second.zeroed.numel();
  }
  g_ws.clear();
  return bytes;
}

// the reference's debug() is an empty hook (cu:1921); this one reports the library's launch counter
int64_t debug() { return fcsa_debug(); }

Tensor prepare_bias(const Tensor& q, const Tensor& k, const Tensor& v, const Tensor& attn_bias, bool batch_dim) {
  const Shapes sh(q, k, v);
  return prep_bias(attn_bias, sh, q.scalar_type(), batch_dim || sh.merged);
}

}  // namespace

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.doc() = "H100 (sm_90a) fused cosine-similarity attention: torch binding of libfcsa_b200.so";
  m.def("forward", &forward, "Flash Cosine-Sim Attention Forward");
  m.def("backward", &backward, "Flash Cosine-Sim Attention Backward");
  m.def("debug", &debug, "Debug");
  namespace py = pybind11;
  // (window, deterministic: trailing arguments, default 0 = no window / false, after the positional ones every caller
  // passes)
  m.def("forward_ex", &forward_ex, "forward with explicit shift / fused l2norm / prepared bias", py::arg("q"),
        py::arg("k"), py::arg("v"), py::arg("mask"), py::arg("bias_prepared"), py::arg("bias_batch_dim"),
        py::arg("bias_amax"), py::arg("scale"), py::arg("shift"), py::arg("causal"), py::arg("l2norm_groups"),
        py::arg("need_inv_l"), py::arg("out_f32"), py::arg("window") = 0);
  m.def("backward_ex", &backward_ex, "backward of forward_ex", py::arg("d_out"), py::arg("o"), py::arg("inv_l"),
        py::arg("q"), py::arg("k"), py::arg("v"), py::arg("q_rnorm"), py::arg("k_rnorm"), py::arg("mask"),
        py::arg("bias_prepared"), py::arg("bias_batch_dim"), py::arg("bias_amax"), py::arg("bias_grad"),
        py::arg("bias_like"), py::arg("scale"), py::arg("shift"), py::arg("causal"), py::arg("groups"),
        py::arg("out_f32"), py::arg("window") = 0, py::arg("deterministic") = false);
  m.def("prepare_bias", &prepare_bias, "attn_bias -> padded, aligned tensor in the problem dtype");
  m.def("f32_cast", &f32_cast, "float32 -> (l2norm +) scaled cast to the 16-bit operand dtype");
  m.def("f32_cast_backward", &f32_cast_backward, "backward of f32_cast: float32 gradient w.r.t. the float32 input");
  m.def("l2norm_forward", &l2norm_forward, "grouped l2norm: x -> (y, 1/norm)");
  m.def("l2norm_backward", &l2norm_backward, "grouped l2norm backward from the normalised y");
  m.def("forward_varlen", &forward_varlen, "packed variable-length sequences: forward (fused l2norm when groups > 0)",
        py::arg("q"), py::arg("k"), py::arg("v"), py::arg("cu_q"), py::arg("cu_k"), py::arg("max_q"), py::arg("max_k"),
        py::arg("scale"), py::arg("shift"), py::arg("causal"), py::arg("groups"), py::arg("need_inv_l"),
        py::arg("window") = 0);
  m.def("backward_varlen", &backward_varlen, "backward of forward_varlen", py::arg("d_out"), py::arg("o"),
        py::arg("inv_l"), py::arg("q"), py::arg("k"), py::arg("v"), py::arg("q_rnorm"), py::arg("k_rnorm"),
        py::arg("cu_q"), py::arg("cu_k"), py::arg("max_q"), py::arg("max_k"), py::arg("scale"), py::arg("shift"),
        py::arg("causal"), py::arg("groups"), py::arg("window") = 0, py::arg("deterministic") = false);
  m.def("decode", &decode, "new queries against a key/value cache, appending k / v at cache_seqlens", py::arg("q"),
        py::arg("k_cache"), py::arg("v_cache"), py::arg("cache_seqlens"), py::arg("k"), py::arg("v"), py::arg("scale"),
        py::arg("shift"), py::arg("causal"), py::arg("groups"), py::arg("window") = 0);
  m.def("release_workspaces", &release_workspaces, "free the cached backward workspaces; returns the bytes released");
  m.def("abi_version", []() { return fcsa_version(); });
  m.def("_error_path_selftest", []() { FCSA_CHECK(fcsa_forward(nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr)); },
        "raises the library's error for a null problem (exercises the C ABI error -> Python exception path)");
}
