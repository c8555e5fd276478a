/*
 * fcsa_b200.h - C ABI of libfcsa_b200.so, the H100 (sm_90a) fused cosine-similarity
 * attention library.
 *
 * This is the drop-in boundary for the reference's CUDA extension
 * (lucidrains/flash-cosine-sim-attention @ v0.1.40).  Each entry point names the reference
 * interface it replaces (file:line, paths relative to the reference repository):
 *
 *   fcsa_forward            <- flash_cosine_sim_attention_forward   flash_cosine_sim_attention_cuda.cu:1630-1748
 *                              (pybind `forward`, cu:1928-1933; called from flash_cosine_sim_attention.py:247-256)
 *   fcsa_backward           <- flash_cosine_sim_attention_backward  cu:1752-1917
 *                              (pybind `backward`; called from flash_cosine_sim_attention.py:281-302)
 *   fcsa_debug              <- debug()                              cu:1921
 *   fcsa_l2norm_forward /   <- l2norm / grouped_l2norm / l2norm_tensors  flash_cosine_sim_attention.py:38-65
 *   fcsa_l2norm_backward       (PyTorch F.normalize + autograd in the reference; fused kernels here)
 *
 * Conventions
 *   - plain pointers and sizes only; no torch / C++ types cross this boundary
 *   - every tensor is a DEVICE pointer to 16-bit data (FCSA_F16 / FCSA_BF16) addressed as
 *     [batch][head][row][feature] with element strides (sb, sh, sn) and a contiguous feature
 *     dimension; pointers and strides*2 must be multiples of 16 bytes (TMA requirement)
 *   - `stream` is a cudaStream_t; all work is enqueued on it and nothing synchronises
 *     (the reference device-synchronised after every call, cu:1745/1889 - deliberately not kept)
 *   - inputs are borrowed and never written; outputs are caller-allocated
 *   - return value: FCSA_OK or an error code; fcsa_last_error() returns a thread-local message
 *     (the reference only printed CUDA errors to stderr, cu:17-28)
 *   - there is NO CPU fallback: without a CUDA device every compute entry point fails
 */
#ifndef FCSA_B200_H
#define FCSA_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum { FCSA_F16 = 0, FCSA_BF16 = 1 };

enum {
  FCSA_OK = 0,
  FCSA_ERR_INVALID = 1,      /* bad argument (shape, alignment, null pointer)           */
  FCSA_ERR_UNSUPPORTED = 2,  /* valid request this build has no kernel for              */
  FCSA_ERR_CUDA = 3,         /* a CUDA runtime / driver call failed                     */
  FCSA_ERR_WORKSPACE = 4     /* workspace too small                                     */
};

/* A (batch, head, row, feature) view with a contiguous feature dimension. */
typedef struct fcsa_tensor {
  void* ptr;
  int64_t sb, sh, sn; /* element strides of batch, head, row */
} fcsa_tensor;

/*
 * One attention problem.  Mirrors the argument list of the reference's forward/backward
 * (cu:1630-1639, cu:1752-1764) after its shape canonicalisation (cu:1647-1660):
 *   - merged batch-heads (3-D q) is expressed as heads = 1
 *   - single-head keys/values (3-D k, v with 4-D q; cu:1679) is kv_heads = 1
 *   - grouped-query attention (no reference counterpart): kv_heads divides heads and query head h reads
 *     key/value head h / (heads / kv_heads); k, v (and dk, dv) then have kv_heads heads
 */
typedef struct fcsa_problem {
  int32_t dtype;     /* FCSA_F16 | FCSA_BF16 (q, k, v, o, do, dq, dk, dv all share it)        */
  int32_t batch;
  int32_t heads;
  int32_t kv_heads;  /* divides heads: == heads (one per query head), 1 (shared by all), or a
                        grouped-query count in between; anything else is FCSA_ERR_INVALID      */
  int32_t seq_q;
  int32_t seq_k;
  int32_t head_dim;  /* 64 or 128                                                             */
  int32_t causal;    /* bottom-right aligned (cu:1097, cu:1210): key j visible iff j <= i + seq_k - seq_q */
  float scale;       /* logits = scale * <q, k>                                               */
  float shift;       /* p = exp(logit - shift); the reference uses shift = scale (cu:1216)    */
  const uint8_t* key_mask;   /* (batch, seq_k) bytes, nonzero = attend; NULL = no mask (cu:1198-1212) */
  int64_t key_mask_stride;   /* bytes between batches                                         */
  int32_t out_f32;   /* 0: o (forward; also the `o` the backward reads), dq, dk, dv have the problem dtype.
                        1: they are float32 tensors (strides then count float32 elements) - the accumulators are
                        fp32 anyway, this only skips the final rounding to 16 bit.  q, k, v, d_o stay 16-bit
                        operands.  Used for float32 callers (reference: Float dispatch, cu:1702-1703)        */
  int32_t window;    /* sliding-window (local) attention; 0 = none.  With off = seq_k - seq_q and d = i + off - j, key j
                        is visible to query i iff 0 <= d < window (causal) or |d| < window (not causal), on top of the
                        key mask.  Rows that see no key give o = 0 and zero gradients.  Negative: FCSA_ERR_INVALID;
                        nonzero on the _bias entry points: FCSA_ERR_INVALID.  Taken by fcsa_forward, fcsa_backward,
                        the _fused and _fused_varlen pairs (lengths per sequence) and fcsa_decode (seq_k = T_b there).
                        The backward's workspace sizes do not depend on it; the decode workspace can only shrink
                        (fewer key splits).  This field was `reserved_` before; a library built
                        before it existed ignores it (fcsa_version() is 300 either way)                      */
} fcsa_problem;

/* Library / ABI version: major*10000 + minor*100 + patch. */
int fcsa_version(void);

/* Message describing the last error on the calling thread ("" if none). */
const char* fcsa_last_error(void);

/* Reference `debug()` (cu:1921): a no-op hook.  Here it returns the number of kernels this
 * library has launched in the current process (bench.py reports it as gpu_launches). */
int64_t fcsa_debug(void);

/*
 * o = softmax-like(q k^T) v with the fixed-shift formulation; inv_l[b][h][i] = 1 / max(l_i, 1e-37)
 * is the saved normaliser the backward needs (the reference's `l` output, cu:1698/1239).
 * inv_l: (batch, heads, seq_q) fp32 contiguous, may be NULL when no backward will follow.
 * mask and causal are mutually exclusive (flash_cosine_sim_attention.py:88, cu:1675).
 * Rows with no visible key produce o = 0 (cu:1239, reference behaviour of the fused kernel).
 */
int fcsa_forward(const fcsa_problem* p, const fcsa_tensor* q, const fcsa_tensor* k,
                 const fcsa_tensor* v, const fcsa_tensor* o, float* inv_l, void* stream);

/* Bytes of SCRATCH fcsa_backward needs for this problem (per-row constants; when kv_heads < heads also
 * 2 * batch * kv_heads * seq_k * head_dim * 4 bytes of fp32 dk/dv accumulators): contents irrelevant on entry,
 * garbage on exit.  A pure function of the problem. */
size_t fcsa_backward_workspace_bytes(const fcsa_problem* p);

/* Bytes of the ZEROED workspace of fcsa_backward (the fp32 dq accumulator tiles).
 * Contract: every byte is zero when a backward call starts and zero again when its kernels have
 * finished - the pass that converts an accumulator tile to dq also clears it - so one buffer,
 * zero-filled ONCE (fcsa_zeroed_init), serves any number of calls of any shape enqueued on the same
 * stream.  This is what replaces the reference's per-call 33.5 MB memset of its fp32 dq (cu:1818).
 * Do not share one buffer between streams that may run concurrently.
 * CUDA graphs: a workspace (scratch or zeroed, of any entry point) passed to a call that is being captured belongs to
 * the graph until the graph is destroyed, since every replay uses it; do not free it, reuse it for other calls, or
 * share it with a graph that may replay concurrently.  Capture the zero fill too (fcsa_zeroed_init on the capturing
 * stream), so that the replay does not depend on what ran before it. */
size_t fcsa_backward_zeroed_bytes(const fcsa_problem* p);

/* Zero-fill a freshly allocated (or grown) zeroed workspace: cudaMemsetAsync on `stream`. */
int fcsa_zeroed_init(void* zeroed, size_t bytes, void* stream);

/*
 * Gradients of fcsa_forward w.r.t. q, k, v (the q, k given are the already-normalised ones,
 * exactly as in the reference: cu:1487-1626).  dq/dk/dv are caller-allocated in the problem
 * dtype; with kv_heads < heads, dk/dv have kv_heads heads and each receives the sum over the query
 * heads that read it (cu:1613-1619 for kv_heads == 1).  `workspace` must hold
 * fcsa_backward_workspace_bytes(p) bytes, `zeroed` fcsa_backward_zeroed_bytes(p) bytes that are all
 * zero (see above).
 * Reproducibility: o, dk, dv are bitwise reproducible from run to run when kv_heads == heads, and for
 * grouped-query problems whose backward grid keeps each group in one CTA (enough batch * kv_heads *
 * key tiles to fill the device, no bias).  Otherwise dk/dv are summed over CTAs with fp32 atomics and
 * may differ in the last bits between runs, like dq always may.  fcsa_backward_fused_deterministic and
 * fcsa_backward_fused_deterministic_varlen (below) have no such reduction: dq, dk, dv are bitwise
 * reproducible for every problem they take.
 */
int fcsa_backward(const fcsa_problem* p, const fcsa_tensor* q, const fcsa_tensor* k,
                  const fcsa_tensor* v, const fcsa_tensor* o, const fcsa_tensor* d_o,
                  const float* inv_l, const fcsa_tensor* dq, const fcsa_tensor* dk,
                  const fcsa_tensor* dv, void* workspace, size_t workspace_bytes, void* zeroed,
                  size_t zeroed_bytes, void* stream);

/*
 * y = x / max(||x||_2, 1e-12) over `groups` equal chunks of the feature dimension
 * (flash_cosine_sim_attention.py:38-55).  x: strided view; y: same shape (any strides);
 * rnorm: (batch, heads, rows, groups) fp32 contiguous = 1 / max(||x||, eps), may be NULL.
 */
int fcsa_l2norm_forward(int32_t dtype, int32_t batch, int32_t heads, int32_t rows, int32_t head_dim,
                        int32_t groups, const fcsa_tensor* x, const fcsa_tensor* y, float* rnorm,
                        void* stream);

/*
 * dx = (dy - y <y, dy>_group) * rnorm_group : the l2norm backward given the NORMALISED y.
 * dy, y, dx: 16-bit strided views.
 */
int fcsa_l2norm_backward(int32_t dtype, int32_t batch, int32_t heads, int32_t rows,
                         int32_t head_dim, int32_t groups, const fcsa_tensor* dy,
                         const fcsa_tensor* y, const float* rnorm, const fcsa_tensor* dx,
                         void* stream);

/*
 * Fused variants: the grouped l2-normalisation of q and k that the reference performs with PyTorch
 * ops around its kernels (flash_cosine_sim_attention.py:320-321, l2norm_tensors py:57-65) and its
 * autograd backward run inside the same call.
 *   q_hat, k_hat : normalised q / k in the problem dtype - outputs of fcsa_forward_fused, inputs of
 *                  fcsa_backward_fused (the reference saves exactly these for its backward, py:270)
 *   q_rnorm      : (batch, heads, seq_q, groups)    fp32 = 1 / max(||q||_group, 1e-12)
 *   k_rnorm      : (batch, kv_heads, seq_k, groups) fp32
 * head_dim / groups must be a power of two.
 */
typedef struct fcsa_l2norm {
  int32_t groups;
  fcsa_tensor q_hat, k_hat;
  float* q_rnorm;
  float* k_rnorm;
} fcsa_l2norm;

/* q_hat, k_hat = l2norm(q), l2norm(k); o, inv_l = fcsa_forward(q_hat, k_hat, v). */
int fcsa_forward_fused(const fcsa_problem* p, const fcsa_tensor* q, const fcsa_tensor* k,
                       const fcsa_tensor* v, const fcsa_l2norm* n, const fcsa_tensor* o, float* inv_l,
                       void* stream);

/* Gradients w.r.t. the RAW q, k (and v): fcsa_backward followed by the l2norm backward, the latter
 * folded into the dq conversion and the dk epilogue.  Same workspaces as fcsa_backward. */
int fcsa_backward_fused(const fcsa_problem* p, const fcsa_l2norm* n, const fcsa_tensor* v,
                        const fcsa_tensor* o, const fcsa_tensor* d_o, const float* inv_l,
                        const fcsa_tensor* dq, const fcsa_tensor* dk, const fcsa_tensor* dv,
                        void* workspace, size_t workspace_bytes, void* zeroed, size_t zeroed_bytes,
                        void* stream);

/* ---- deterministic backward ------------------------------------------------------------------------
 * The gradients of fcsa_backward_fused without a floating-point reduction whose order depends on
 * scheduling: dq, dk, dv are bitwise the same from run to run, and batch element b's are the same
 * whatever the batch around it.  Three launches: the preprocess, a dK / dV kernel with one CTA per
 * (key tile, batch, kv head) that keeps every query head of the group (no dk / dv accumulators), and a
 * dQ kernel that sums each query block's key tiles in ascending order in registers (no dq accumulator).
 * The rounding points are fcsa_backward's, so the results agree with it within its error bounds; dk, dv
 * are bitwise fcsa_backward's wherever that keeps each group in one CTA.
 *   n->groups == 0: q, k (n->q_hat, n->k_hat) are used as given and the rnorms are ignored; > 0: the
 *                   l2norm backward is applied as in fcsa_backward_fused.
 * Takes out_f32 (with groups == 0), window and key_mask as fcsa_backward does; no bias.  `workspace`:
 * fcsa_backward_fused_deterministic_workspace_bytes(p) bytes of scratch (the per-row constants only),
 * contents irrelevant on entry.  No zeroed workspace.
 */
size_t fcsa_backward_fused_deterministic_workspace_bytes(const fcsa_problem* p);
int fcsa_backward_fused_deterministic(const fcsa_problem* p, const fcsa_l2norm* n, const fcsa_tensor* v,
                                      const fcsa_tensor* o, const fcsa_tensor* d_o, const float* inv_l,
                                      const fcsa_tensor* dq, const fcsa_tensor* dk, const fcsa_tensor* dv,
                                      void* workspace, size_t workspace_bytes, void* stream);

/* ---- float32 front end ---------------------------------------------------------------------------
 * The reference dispatches Float in forward and backward (cu:1702-1703, 1832-1834).  Here float32 callers run the
 * 16-bit tensor-core kernels (fp32 accumulation, `out_f32` results); these two passes are all that surrounds them.
 * `x` / `dy` / `dx` are FLOAT32 tensors (fcsa_tensor with float32 element strides, feature dim contiguous, rows
 * 16-byte aligned), `y` is the 16-bit tensor (`dtype`), which may be wider than head_dim (zero-padded features are
 * the caller's business: only head_dim features per row are written / read).
 *   fcsa_f32_cast          y = round16( l2norm_groups(x) * m )   groups > 0 ;  round16( x * m )   groups == 0
 *   fcsa_f32_cast_backward dx = (dy - y <y,dy>_group) * rnorm_group * m   groups > 0 ;  dy * m   groups == 0
 * m = 1 if `mul` is NULL, else *mul (a DEVICE scalar - e.g. a power-of-two range scale chosen on the device, the
 * host never reads it), or 1 / *mul when mul_reciprocal != 0.  rnorm: (batch, heads, rows, groups) fp32.
 * head_dim must be 16, 32, 64 or 128 and head_dim / groups a power of two. */
int fcsa_f32_cast(int32_t dtype, int32_t batch, int32_t heads, int32_t rows, int32_t head_dim, int32_t groups,
                  const fcsa_tensor* x, const fcsa_tensor* y, float* rnorm, const float* mul, int32_t mul_reciprocal,
                  void* stream);
int fcsa_f32_cast_backward(int32_t dtype, int32_t batch, int32_t heads, int32_t rows, int32_t head_dim,
                           int32_t groups, const fcsa_tensor* dy, const fcsa_tensor* y, const float* rnorm,
                           const fcsa_tensor* dx, const float* mul, int32_t mul_reciprocal, void* stream);

/* ---- additive attention bias -------------------------------------------------------------------
 * Replaces the `attn_bias` / `attn_bias_batch_dim` arguments of the reference's forward / backward
 * (flash_cosine_sim_attention_cuda.cu:1630-1639, 1752-1764; added to the logits at cu:1168,1214 and
 * cu:1474-1476, gradient cu:1574-1576).  Elements have the problem's dtype; the bias is addressed as
 * [batch][head][query][key] with ELEMENT strides sb (0 when the bias has no batch dimension -
 * attn_bias_batch_dim == false), sh, sn and contiguous keys.  Rows must be 16-byte aligned: sb, sh, sn
 * multiples of 8 and sn >= seq_k rounded up to 8 (pad the rows; the padding is never used). */
typedef struct fcsa_bias {
  const void* ptr;
  int64_t sb, sh, sn;
  /* Optional DEVICE pointer to one fp32: an upper bound of the bias values (e.g. its max).  The kernels
   * add max(*amax, 0) to the problem's `shift`, which keeps p = exp(logit - shift) inside the fp16 range
   * whatever the bias adds - without the host ever reading the bias (no device synchronisation).
   * Pass the same pointer to the forward and the backward; NULL = use `shift` as is. */
  const float* amax;
} fcsa_bias;

/* fcsa_forward with the bias added to scale * q.k before the exponential. */
int fcsa_forward_bias(const fcsa_problem* p, const fcsa_tensor* q, const fcsa_tensor* k,
                      const fcsa_tensor* v, const fcsa_bias* bias, const fcsa_tensor* o, float* inv_l,
                      void* stream);

/* fcsa_backward with the bias.  d_bias_acc: fp32, zero-filled by the caller, same index space as the bias
 * with element strides (dsb, dsh) over batch / head and contiguous [seq_q][seq_k] planes (dsb = 0 sums
 * the gradient over the batch, as the reference does for a bias without batch dimension, cu:1574-1576);
 * NULL when the bias needs no gradient (reference: db is empty unless it requires grad, cu:1827). */
int fcsa_backward_bias(const fcsa_problem* p, const fcsa_tensor* q, const fcsa_tensor* k,
                       const fcsa_tensor* v, const fcsa_tensor* o, const fcsa_tensor* d_o,
                       const float* inv_l, const fcsa_bias* bias, float* d_bias_acc, int64_t dsb,
                       int64_t dsh, const fcsa_tensor* dq, const fcsa_tensor* dk, const fcsa_tensor* dv,
                       void* workspace, size_t workspace_bytes, void* zeroed, size_t zeroed_bytes,
                       void* stream);

/*
 * Measurement hook (bench.py roofline line; no reference counterpart - the reference only timed
 * whole calls, flash_cosine_sim_attention/benchmark.py:7-58).  While set, fcsa_forward (which = 0)
 * or fcsa_backward (which = 1) records the cudaEvent_t `start` / `stop` on the launch stream
 * immediately before / after its dominant kernel (the wgmma attention kernel, not the
 * pre/post passes); which = 2, 3, 4 do the same for the l2norm(q,k) pass of fcsa_forward_fused, the
 * backward preprocess and the dq finish pass (the dQ kernel in the deterministic backward).  An event between two launches suspends their programmatic
 * dependent launch, so a hooked run is for attribution, not for the headline time.  Pass NULL, NULL to clear.  State is process-wide (autograd calls the
 * backward from its own thread), so use it from single-stream measurement code only.
 */
int fcsa_set_kernel_events(int32_t which, void* start_event, void* stop_event);

/* ---- key/value-cache decode (no reference counterpart: the reference has no inference path) ----------------------
 * Attends seq_q >= 1 new queries per (batch, head) to a key/value cache and appends new keys / values to it, in at
 * most three launches (append pass, attention, combine of the key splits) that never synchronise: a decode step can
 * be captured in a CUDA graph.
 *   p              : seq_q = new queries, seq_k = the cache CAPACITY, kv_heads as in fcsa_problem; no key_mask,
 *                    out_f32 = 0.  scale / shift / causal as in fcsa_forward.
 *   q, o           : (batch, heads, seq_q, head_dim)
 *   k_cache,v_cache: (batch, kv_heads, capacity, head_dim), any TMA-legal strides; written in place
 *   cache_seqlens  : DEVICE int32 (batch,): valid cache rows L_b before the call; never read by the host, never
 *                    changed (the caller advances it by n_new afterwards)
 *   k_new, v_new   : (batch, kv_heads, n_new, head_dim), appended at cache rows [L_b, L_b + n_new); ignored when
 *                    n_new == 0
 *   groups         : > 0: q and k_new are l2-normalised over `groups` chunks of the head dim (as fcsa_forward_fused)
 *                    and the cache stores normalised keys rounded to the dtype; 0: q and k_new are used as given
 * Visible length T_b = min(L_b + n_new, capacity).  Query i sees key j iff j < T_b and, causal, j <= i + T_b - seq_q
 * (fcsa_forward's bottom-right rule with seq_k = T_b); rows with no visible key give o = 0.  Nothing is written
 * outside the cache: appended rows at or past the capacity are dropped (L_b + n_new > capacity is a caller error).
 * o is bitwise reproducible from run to run.  `workspace`: fcsa_decode_workspace_bytes(p, n_new) bytes of scratch,
 * contents irrelevant on entry.
 */
size_t fcsa_decode_workspace_bytes(const fcsa_problem* p, int32_t n_new);
int fcsa_decode(const fcsa_problem* p, const fcsa_tensor* q, const fcsa_tensor* k_cache, const fcsa_tensor* v_cache,
                const int32_t* cache_seqlens, const fcsa_tensor* k_new, const fcsa_tensor* v_new, int32_t n_new,
                int32_t groups, const fcsa_tensor* o, void* workspace, size_t workspace_bytes, void* stream);

/* Packed decode: a different number of new tokens per batch element (speculative verification, chunked prefill,
 * ragged prompts), in one call of the same kernels.  Arguments as fcsa_decode's, except:
 *   p              : seq_q = max_seqlen_q, at least every n_b (it sizes the grid and the key splits; larger lengths are
 *                    clamped to it).  batch = B, the cache's batch.
 *   cu_seqlens_q   : DEVICE int32 (B + 1,), non-decreasing, never read by the host.  Batch element b brings the
 *                    n_b = cu[b + 1] - cu[b] new tokens at packed rows [cu[b], cu[b + 1]).
 *   total_q        : rows of the packed tensors (0: nothing is launched)
 *   q, o           : (total_q, heads, head_dim) as fcsa_tensor with sh, sn set (sb unused)
 *   k_new, v_new   : (total_q, kv_heads, head_dim), packed with the same boundaries, or both NULL (nothing appended).
 *                    Row cu[b] + n goes to cache row L_b + n of batch element b; rows at or past the capacity and
 *                    rows outside every sequence are not written.
 * T_b = min(L_b + (n_b if appending, else 0), capacity); query i of element b sees key j iff j < T_b and, causal,
 * j <= i + T_b - n_b (fcsa_decode's rule per element; the window likewise).  Rows with no visible key give o = 0, and
 * so do the rows outside every sequence ([0, cu[0]) and [cu[B], total_q)).  Launches: the append pass, the decode
 * kernel, the combine kernel when the keys are split, and the pass that zeroes the rows outside every sequence.  With
 * cu = (0, n, 2n, ...) and seq_q = n, o and the caches are bitwise fcsa_decode's on the same data.  `workspace`:
 * fcsa_decode_varlen_workspace_bytes(p, total_q) bytes of scratch (0 for a problem it rejects).  Rejected: a null
 * cu_seqlens_q, total_q < 0, seq_q < 0, a key mask or out_f32.
 */
size_t fcsa_decode_varlen_workspace_bytes(const fcsa_problem* p, int32_t total_q);
int fcsa_decode_varlen(const fcsa_problem* p, const int32_t* cu_seqlens_q, int32_t total_q, const fcsa_tensor* q,
                       const fcsa_tensor* k_cache, const fcsa_tensor* v_cache, const int32_t* cache_seqlens,
                       const fcsa_tensor* k_new, const fcsa_tensor* v_new, int32_t groups, const fcsa_tensor* o,
                       void* workspace, size_t workspace_bytes, void* stream);

/* Rolling caches for sliding-window decoding: k_cache and v_cache are rings of C = seq_k rows that keep the window's
 * keys only, so their memory is bounded by the window instead of the sequence.  Arguments as fcsa_decode_varlen's,
 * except that cu_seqlens_q may be NULL: the dense form, with q, o (batch, heads, seq_q, head_dim) and k_new, v_new
 * (batch, kv_heads, seq_q, head_dim) or both NULL; total_q is then unused.
 *   - Absolute position p lives at ring row p mod C.
 *   - cache_seqlens[b] = L_b counts every token element b has seen, and may be far larger than C.
 *   - The visible length is T_b = L_b + n_b with no clamp (n_b = seq_q dense, the packed length otherwise, 0 when
 *     nothing is appended in the packed form).  The windowed rule of fcsa_decode holds over absolute positions: query i
 *     sees key j iff 0 <= i + T_b - n_b - j < window (causal) or |i + T_b - n_b - j| < window.
 *   - New row n of element b is written to ring row (L_b + n) mod C.
 * Rejected with FCSA_ERR_INVALID, besides fcsa_decode_varlen's rejections: no window, C not a multiple of 128, and
 * C < window + seq_q - 1 (seq_q = max_seqlen_q in the packed form), below which a call's append would overwrite a key
 * that one of its own queries still sees.  L_b + n_b must stay below 2^31 - 128; the host never reads the lengths and
 * cannot check it.  With the same number of key splits, o is bitwise what fcsa_decode or fcsa_decode_varlen give on a
 * full-length cache holding the same keys.  `workspace`: fcsa_decode_rolling_workspace_bytes(p, cu_seqlens_q, total_q)
 * bytes of scratch (0 for a problem it rejects).
 */
size_t fcsa_decode_rolling_workspace_bytes(const fcsa_problem* p, const int32_t* cu_seqlens_q, int32_t total_q);
int fcsa_decode_rolling(const fcsa_problem* p, const int32_t* cu_seqlens_q, int32_t total_q, const fcsa_tensor* q,
                        const fcsa_tensor* k_cache, const fcsa_tensor* v_cache, const int32_t* cache_seqlens,
                        const fcsa_tensor* k_new, const fcsa_tensor* v_new, int32_t groups, const fcsa_tensor* o,
                        void* workspace, size_t workspace_bytes, void* stream);

/* ---- packed variable-length sequences (no reference counterpart) ------------------------------------------------------
 * Training attention over B sequences of different lengths packed along the row dimension, without padding:
 *   p              : batch = B (sequences), seq_q / seq_k = maximum lengths (they size the grids and clamp the device
 *                    lengths), heads / kv_heads / head_dim / causal / scale / shift as in fcsa_problem; no key_mask,
 *                    out_f32 = 0
 *   vl             : the cumulative lengths, DEVICE int32 arrays of B + 1 entries, non-decreasing from 0, never read by
 *                    the host (a step can be captured in a CUDA graph).  Sequence b owns query rows
 *                    [cu_seqlens_q[b], cu_seqlens_q[b + 1]) and key rows [cu_seqlens_k[b], cu_seqlens_k[b + 1]).
 *                    total_q / total_k: the rows of the packed tensors
 *   q, o, d_o, dq  : (total_q, heads, head_dim) as fcsa_tensor with sh, sn set (sb unused)
 *   k, v, dk, dv   : (total_k, kv_heads, head_dim), likewise
 *   inv_l          : (heads, total_q) fp32
 *   n              : groups > 0: q, k are l2-normalised as in fcsa_forward_fused; q_hat / k_hat are (total, heads,
 *                    head_dim) and q_rnorm / k_rnorm [heads][total][groups].  groups == 0: q, k are used as given (the
 *                    forward ignores q_hat, k_hat and the rnorms; the backward reads q, k from q_hat, k_hat).
 * Each sequence gets what fcsa_forward_fused / fcsa_backward_fused give on it alone, with the causal rule applied to
 * its own lengths (key j visible to query i iff j <= i + len_k - len_q); rows with no visible key give o = 0.
 * Rows that belong to no sequence ([0, cu[0]) and [cu[B], total), e.g. the unused end of a fixed-size packing buffer)
 * get o = 0 and zero dq, dk, dv.  Out-of-contract lengths (above the maxima, or rows past the totals) are clamped:
 * nothing is accessed outside the tensors, and the rows past the clamp are unspecified.
 * Workspaces: the backward's scratch and zeroed buffers (same contract as fcsa_backward's: the zeroed one is zero on
 * entry and on exit) are pure functions of B, heads, kv_heads, the totals and head_dim.
 */
typedef struct fcsa_varlen {
  const int32_t* cu_seqlens_q;
  const int32_t* cu_seqlens_k;
  int32_t total_q;
  int32_t total_k;
} fcsa_varlen;

int fcsa_forward_fused_varlen(const fcsa_problem* p, const fcsa_varlen* vl, const fcsa_tensor* q, const fcsa_tensor* k,
                              const fcsa_tensor* v, const fcsa_l2norm* n, const fcsa_tensor* o, float* inv_l,
                              void* stream);
size_t fcsa_backward_fused_varlen_workspace_bytes(const fcsa_problem* p, const fcsa_varlen* vl);
size_t fcsa_backward_fused_varlen_zeroed_bytes(const fcsa_problem* p, const fcsa_varlen* vl);
int fcsa_backward_fused_varlen(const fcsa_problem* p, const fcsa_varlen* vl, const fcsa_l2norm* n,
                               const fcsa_tensor* v, const fcsa_tensor* o, const fcsa_tensor* d_o, const float* inv_l,
                               const fcsa_tensor* dq, const fcsa_tensor* dk, const fcsa_tensor* dv, void* workspace,
                               size_t workspace_bytes, void* zeroed, size_t zeroed_bytes, void* stream);
/* The deterministic backward (see fcsa_backward_fused_deterministic) over packed sequences: a sequence's gradients are
 * bitwise the same whatever the other sequences of the pack.  Scratch only, a pure function like the above. */
size_t fcsa_backward_fused_deterministic_varlen_workspace_bytes(const fcsa_problem* p, const fcsa_varlen* vl);
int fcsa_backward_fused_deterministic_varlen(const fcsa_problem* p, const fcsa_varlen* vl, const fcsa_l2norm* n,
                                             const fcsa_tensor* v, const fcsa_tensor* o, const fcsa_tensor* d_o,
                                             const float* inv_l, const fcsa_tensor* dq, const fcsa_tensor* dk,
                                             const fcsa_tensor* dv, void* workspace, size_t workspace_bytes,
                                             void* stream);

#ifdef __cplusplus
}
#endif

#endif /* FCSA_B200_H */
