"""Python operator API - the host-side mirror of the reference's
flash_cosine_sim_attention/flash_cosine_sim_attention.py, kept name-for-name so callers
(benchmark.py, train.py, transformer.py, the reference's tests) switch over unchanged:

    flash_cosine_sim_attention(q, k, v, mask, attn_bias, scale, groups, causal, l2norm_qk,
                               attn_bias_batch_dim)                     reference py:308-334
    l2norm_tensors(*tensors, groups)                                    reference py:57-65
    flash_cosine_sim_attention_with_kv_cache(q, k_cache, v_cache, cache_seqlens, k, v, ...)
                                      decoding with a key/value cache (no reference counterpart)
    flash_cosine_sim_attention_varlen(q, k, v, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k, ...)
                                      packed variable-length sequences (no reference counterpart)
    plain_cosine_sim_attention(...)   naive un-fused formulation        reference py:75-126
    FlashCosineSimAttention (autograd.Function) / forward / backward / debug   py:245-304, cu:1928-1933

What differs, on purpose:
  * the compute is libfcsa_b200.so (hand-written sm_90a kernels behind a C ABI), reached
    through ctypes with raw device pointers and the current CUDA stream;
  * with l2norm_qk=True the normalisation and its backward run as fused CUDA kernels inside
    one autograd node instead of PyTorch ops around it (reference py:320-321);
  * CUDA tensors only: the reference's tiled CPU forward (py:130-241) is not reproduced (it is
    wrong for causal N > 512, py:215) - CPU tensors raise;
  * the exponent shift is scale*groups (not scale): mathematically identical (softmax shift
    invariance), but safe in 16 bit when groups > 1 (q.k can reach `groups`).
"""
import math
import warnings

import torch
from torch.autograd import Function

from . import _abi

__all__ = [
    "flash_cosine_sim_attention",
    "flash_cosine_sim_attention_with_kv_cache",
    "flash_cosine_sim_attention_varlen",
    "plain_cosine_sim_attention",
    "l2norm_tensors",
    "FlashCosineSimAttention",
    "flash_cosine_sim_attention_cuda",
    "forward",
    "backward",
    "debug",
    "release_workspaces",
]

_KERNEL_DTYPES = {torch.float16: _abi.FCSA_F16, torch.bfloat16: _abi.FCSA_BF16}
_KERNEL_HEAD_DIMS = (64, 128)


def exists(val):
    return val is not None


# --------------------------------------------------------------------------------------------
# host-side helpers mirrored in csrc/torch_ext.cpp (kept here for the sharding layer and the tests)
# --------------------------------------------------------------------------------------------

def _tma_ready(t):
    """Tensor usable behind a TMA tensor map as is: feature dim contiguous, 16-byte aligned
    base and (batch, head, row) strides, no stride-0 (expanded) dimension of extent > 1 - a tensor
    map cannot express a broadcast.  Otherwise a contiguous copy is made - e.g. for the stride-0
    expanded grad that `o.sum().backward()` / `o.sum(1)` produce, or head-expanded keys."""
    ok = (t.stride(-1) == 1 and t.data_ptr() % 16 == 0
          and all(s % 8 == 0 and (s > 0 or n == 1) for s, n in zip(t.stride()[:-1], t.shape[:-1])))
    return t if ok else t.contiguous()


def _kernel_supported(q, k, v, attn_bias):
    return (q.is_cuda and q.dtype in _KERNEL_DTYPES and k.dtype == q.dtype and v.dtype == q.dtype
            and q.shape[-1] in _KERNEL_HEAD_DIMS and not exists(attn_bias))


def _check_kv_heads(q, k, v):
    """4-D q, k, v: k and v have the same number of heads, and it divides q's (grouped-query attention)."""
    if q.ndim != 4 or k.ndim != 4:
        return
    hk = k.shape[1]
    if v.ndim != 4 or v.shape[1] != hk:
        raise ValueError(f"keys and values must have the same number of heads (kv_heads {hk} vs "
                         f"{v.shape[1] if v.ndim == 4 else 'a 3-D v'})")
    if hk <= 0 or q.shape[1] % hk != 0:
        raise ValueError(f"kv_heads ({hk}) must divide the query heads ({q.shape[1]})")


class _Shapes:
    """Shape canonicalisation of the reference's host op (cu:1647-1660, cu:1679)."""

    def __init__(self, q, k, v):
        self.merged = q.ndim == 3
        if self.merged:
            assert k.ndim == 3 and v.ndim == 3, (
                "if batch and heads are merged for queries, keys and values must also similarly "
                "have only 3 dimensions")
            self.B, self.Nq, self.D = q.shape
            self.H = 1
            self.kv_heads = 1
            self.qkind = "bnd"
            self.kkind = "bnd"
        else:
            assert q.ndim == 4, "queries must be (batch, heads, seq, dim) or (batch*heads, seq, dim)"
            self.B, self.H, self.Nq, self.D = q.shape
            self.qkind = "bhnd"
            if k.ndim == 3:
                assert v.ndim == 3, "keys and values must both be single-headed"
                self.kv_heads = 1
                self.kkind = "bnd"
            else:
                # grouped-query attention: query head h reads key/value head h // (H // kv_heads)
                _check_kv_heads(q, k, v)
                self.kv_heads = k.shape[1]
                self.kkind = "bhnd"
        self.Nk = k.shape[-2]
        assert k.shape[-1] == self.D and v.shape[-1] == self.D, "head dimensions of q, k, v must match"
        assert k.shape[0] == self.B and v.shape[0] == self.B, "batch sizes of q, k, v must match"
        assert v.shape[-2] == self.Nk


# --------------------------------------------------------------------------------------------
# the compiled host layer: flash_cosine_sim_attention_cuda_0_1_40 (csrc/torch_ext.cpp), the
# module the reference imports by this very name (py:15-20, version.py:3).  It canonicalises shapes,
# allocates outputs and calls the C ABI on the current stream - a few microseconds per call.
# --------------------------------------------------------------------------------------------
_ext_module = None


def _ext():
    """Load (once) the torch extension module; registers it under its top-level name so that
    `importlib.import_module('flash_cosine_sim_attention_cuda_0_1_40')` - what the reference's own
    flash_cosine_sim_attention.py does - finds it too.  A missing build raises: no fallback."""
    global _ext_module
    if _ext_module is not None:
        return _ext_module
    import importlib
    import importlib.machinery
    import importlib.util
    import os
    import sys
    from .version import __cuda_pkg_name__ as name
    if name in sys.modules:
        _ext_module = sys.modules[name]
        return _ext_module
    here = os.path.dirname(os.path.abspath(__file__))
    for suffix in importlib.machinery.EXTENSION_SUFFIXES:
        path = os.path.join(here, name + suffix)
        if os.path.exists(path):
            break
    else:
        try:                                     # pip-installed: the module sits top-level, like the reference's
            _abi.load()
            _ext_module = importlib.import_module(name)
            return _ext_module
        except ImportError:
            pass
        raise ImportError(
            f"{name} (the torch extension module over libfcsa_b200.so) is not built in {here}: run "
            "`python -m flash_cosine_sim_attention_b200.build` (needs nvcc and g++; sm_90a only).  "
            "There is no CPU fallback.")
    _abi.load()                                  # fail with the library's own message if the .so is missing
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    sys.modules[name] = mod
    _ext_module = mod
    return mod


# --------------------------------------------------------------------------------------------
# the reference's extension-module surface: forward / backward / debug (cu:1630, 1752, 1921)
# --------------------------------------------------------------------------------------------

def forward(q, k, v, mask, attn_bias, attn_bias_batch_dim, scale, causal, shift=None):
    """Same contract as the reference's pybind `forward`: returns (o, inv_l, should_backwards).
    `shift` (extra, optional): the constant subtracted from the logits; the reference's is `scale`."""
    assert not (causal and exists(mask)), "mask should not be supplied if causality is needed"
    ext = _ext()
    if shift is None:
        return ext.forward(q, k, v, mask, attn_bias, bool(attn_bias_batch_dim), float(scale), bool(causal))
    should_backwards = any(t.requires_grad for t in (q, k, v)) or (exists(attn_bias) and attn_bias.requires_grad)
    bias = ext.prepare_bias(q, k, v, attn_bias, bool(attn_bias_batch_dim)) if exists(attn_bias) else None
    o, inv_l = ext.forward_ex(q, k, v, mask, bias, bool(attn_bias_batch_dim) or q.ndim == 3, None, float(scale),
                              float(shift), bool(causal), 0, True, False)[:2]
    return o, inv_l, should_backwards


def backward(d_out, o, inv_l, q, k, v, mask, attn_bias, attn_bias_batch_dim, scale, causal, shift=None):
    """Same contract as the reference's pybind `backward`: returns (dq, dk, dv, db)."""
    ext = _ext()
    if shift is None:
        return ext.backward(d_out, o, inv_l, q, k, v, mask, attn_bias, bool(attn_bias_batch_dim), float(scale),
                            bool(causal))
    bias = ext.prepare_bias(q, k, v, attn_bias, bool(attn_bias_batch_dim)) if exists(attn_bias) else None
    dq, dk, dv, db = ext.backward_ex(d_out, o, inv_l, q, k, v, None, None, mask, bias,
                                     bool(attn_bias_batch_dim) or q.ndim == 3, None,
                                     exists(attn_bias) and attn_bias.requires_grad, attn_bias, float(scale),
                                     float(shift), bool(causal), 0, False)
    return dq, dk, dv, db


def debug():
    """Reference: a no-op hook (cu:1921).  Here: number of kernels launched by the library."""
    return int(_ext().debug())


def release_workspaces():
    """Free the workspaces cached per (device, stream) for eager backward and decode calls - the fp32 dq accumulator
    and the scratch area only ever grow with the largest problem seen.  Returns the number of bytes handed back to the
    allocator.  Safe at any time, also while CUDA graphs are alive: a call captured into a graph allocates workspaces
    of its own from the graph's memory pool, kept until the graph is destroyed, so a replay never uses the cache."""
    return int(_ext().release_workspaces())


class FlashCosineSimAttention(Function):
    """The reference's autograd.Function (py:245-304) on already-normalised q, k.  Extra optional
    arguments: `shift` (constant subtracted from the logits, default = scale as in the reference) and
    `bias_amax` (fp32 device scalar >= the bias values; added to the shift inside the kernels)."""

    @staticmethod
    def forward(ctx, q, k, v, mask, attn_bias, scale, causal, attn_bias_batch_dim, shift=None, bias_amax=None):
        assert not (causal and exists(mask)), "mask should not be supplied if causality is needed"
        ext = _ext()
        batch_dim = bool(attn_bias_batch_dim) or q.ndim == 3          # reference cu:1647-1654
        should_backwards = any(t.requires_grad for t in (q, k, v)) or (exists(attn_bias) and attn_bias.requires_grad)
        bias = ext.prepare_bias(q, k, v, attn_bias, batch_dim) if exists(attn_bias) else None
        sft = float(scale if shift is None else shift)
        o, inv_l = ext.forward_ex(q, k, v, mask, bias, batch_dim, bias_amax, float(scale), sft, bool(causal), 0,
                                  should_backwards, False)[:2]
        if not should_backwards:
            return o
        ctx.should_backwards = should_backwards
        # the padded / aligned bias is saved, not rebuilt in the backward
        ctx.save_for_backward(o, inv_l, q, k, v, mask, bias, bias_amax)
        ctx.params = (float(scale), bool(causal), batch_dim, sft,
                      exists(attn_bias) and attn_bias.requires_grad, attn_bias.dtype if exists(attn_bias) else None)
        return o

    @staticmethod
    def backward(ctx, do):
        assert ctx.should_backwards
        o, inv_l, q, k, v, mask, bias, bias_amax = ctx.saved_tensors
        scale, causal, batch_dim, shift, bias_grad, bias_dtype = ctx.params
        like = torch.empty(0, dtype=bias_dtype, device=q.device) if bias_grad else None
        dq, dk, dv, db = _ext().backward_ex(do, o, inv_l, q, k, v, None, None, mask, bias, batch_dim, bias_amax,
                                            bias_grad, like, scale, shift, causal, 0, False)
        return dq, dk, dv, None, db, None, None, None, None, None


flash_cosine_sim_attention_cuda = FlashCosineSimAttention.apply


_FP16_GROUPED_RANGE = 10.0      # scale * groups up to which exp(scale * q.k) fits fp16's normal range, see below


def _choose_shift(dtype, scale, groups, l2norm_qk):
    """Constant subtracted from the logits before exp (any constant gives the same attention;
    the reference hard-codes `scale`, cu:1216).  p = exp(logit - shift) is stored in 16 bit:
      bf16: shift = scale*groups - p <= 1 for every possible q.k (<= groups); bf16 has fp32's range.
      fp16: q.k lies in [-groups, groups], so exp(scale*q.k) spans e^(2*scale*groups).  fp16's NORMAL range
            is 2^-14 .. 2^15 (e^20); shift = scale*groups - 15 ln 2 puts the largest possible p at 2^15 and, as
            long as scale*groups <= 10, the smallest at 2^15 e^-20 > 2^-14: nothing under- or overflows.
      fp16, scale*groups > 10: more range than fp16 has without a row max.  Same choice as the reference
            (shift = scale): tiny p flush to zero, and once scale*(groups - 1) > ln 65504 the rows whose best
            match is GOOD (q.k near `groups`) have p = exp(scale*(q.k - 1)) above fp16's maximum.  The kernels
            saturate that p at 65504 for P V but add the unsaturated fp32 p to the row sum, so such a row comes
            out finite and wrong (o scaled down by 65504 / p; dq, dk follow).  `_fp16_overflows` tells when that
            can happen and the entry points warn.  Use bf16 (or float32 inputs, which switch to the bf16
            kernels by themselves) for grouped l2norm with a large scale*groups."""
    if not l2norm_qk:
        return float(scale)
    if dtype == torch.bfloat16:
        return float(scale * groups)
    if scale * groups <= _FP16_GROUPED_RANGE:
        return float(scale * groups) - 15.0 * math.log(2.0)
    return float(scale)


def _fp16_overflows(dtype, scale, groups, l2norm_qk):
    """True when fp16 kernels with l2norm can meet p = exp(scale*q.k - shift) above fp16's maximum 65504: q.k reaches
    `groups` (a query aligned with a key in every l2norm group), so the largest p is exp(scale*groups - shift)."""
    if dtype != torch.float16 or not l2norm_qk:
        return False
    return scale * groups - _choose_shift(dtype, scale, groups, True) > math.log(65504.0)


def _warn_fp16_overflow(dtype, scale, groups, l2norm_qk):
    if _fp16_overflows(dtype, scale, groups, l2norm_qk):
        _warn_once("f16-overflow", f"flash_cosine_sim_attention: float16 with l2norm at scale {scale:g} and groups "
                                   f"{groups}: exp(scale*q.k - shift) exceeds fp16's maximum when q.k is near "
                                   "`groups`, so rows whose query matches a key well come out wrong (finite, not "
                                   "inf) and so do their gradients; use bfloat16")


class _FusedCosineSimAttention(Function):
    """One autograd node for l2norm(q), l2norm(k) -> attention, all in CUDA kernels."""

    @staticmethod
    def forward(ctx, q, k, v, mask, scale, causal, groups, l2norm_qk, shift_groups=0, window=0, deterministic=False):
        ext = _ext()
        # shift_groups > 0: q, k arrive already normalised over that many groups (padded head dims)
        shift = (_choose_shift(q.dtype, scale, shift_groups, True) if shift_groups > 0
                 else _choose_shift(q.dtype, scale, groups, l2norm_qk))
        needs_grad = any(ctx.needs_input_grad[:3])
        o, inv_l, qn, kn, rq, rk = ext.forward_ex(q, k, v, mask, None, False, None, scale, shift, causal,
                                                  groups if l2norm_qk else 0, needs_grad, False, window)
        if needs_grad:
            if not l2norm_qk:
                qn, kn = q, k
            ctx.save_for_backward(o, inv_l, qn, kn, v, mask, rq, rk)
            ctx.params = (scale, shift, causal, groups, l2norm_qk, window, deterministic)
        return o

    @staticmethod
    def backward(ctx, do):
        o, inv_l, qn, kn, v, mask, rq, rk = ctx.saved_tensors
        scale, shift, causal, groups, l2norm_qk, window, deterministic = ctx.params
        dq, dk, dv, _ = _ext().backward_ex(do, o, inv_l, qn, kn, v, rq, rk, mask, None, False, None, False, None,
                                           scale, shift, causal, groups if l2norm_qk else 0, False, window,
                                           deterministic)
        return dq, dk, dv, None, None, None, None, None, None, None, None


class _L2Norm(Function):
    """l2norm_tensors on CUDA 16-bit inputs: the fused kernel with its own backward."""

    @staticmethod
    def forward(ctx, x, groups):
        y, rnorm = _ext().l2norm_forward(x, groups)
        ctx.save_for_backward(y, rnorm)
        ctx.groups = groups
        return y

    @staticmethod
    def backward(ctx, dy):
        y, rnorm = ctx.saved_tensors
        return _ext().l2norm_backward(dy, y, rnorm, ctx.groups), None


# --------------------------------------------------------------------------------------------
# public API
# --------------------------------------------------------------------------------------------

def _check_window(window, attn_bias, name):
    """The `window` keyword of the attention entry points: None (no window) or a positive int W; returns W or 0.
    With off = n_k - n_q and d = i + off - j, key j is visible to query i iff 0 <= d < W (causal) or |d| < W (not
    causal).  Rejected before any launch: a bool or non-int, W < 1, and a window together with attn_bias."""
    if window is None:
        return 0
    if isinstance(window, bool) or not isinstance(window, int):
        raise TypeError(f"{name}: window must be a positive int or None, got {window!r}")
    if window < 1:
        raise ValueError(f"{name}: window must be at least 1 (None for no window), got {window}")
    if exists(attn_bias):
        raise NotImplementedError(f"{name}: window with attn_bias is not supported (the bias kernels take no window)")
    return min(window, 2 ** 31 - 1)


def _check_deterministic(deterministic, attn_bias, name):
    """The `deterministic` keyword of the training entry points: a bool.  Rejected before any launch: anything else,
    and True together with attn_bias (its gradient is summed with atomics)."""
    if not isinstance(deterministic, bool):
        raise TypeError(f"{name}: deterministic must be a bool, got {deterministic!r}")
    if deterministic and exists(attn_bias):
        raise NotImplementedError(f"{name}: deterministic=True with attn_bias is not supported (the bias gradient is "
                                  "summed with atomics)")
    return deterministic


def _band(nq, nk, window, causal, device):
    """(nq, nk) bool: the keys a sliding window of `window` lets each query see (see `_check_window`)."""
    d = torch.arange(nq, device=device)[:, None] + (nk - nq) - torch.arange(nk, device=device)[None, :]
    return ((d >= 0) & (d < window)) if causal else (d.abs() < window)


def _l2norm_torch(t, groups):
    shape = t.shape
    g = t.reshape(*shape[:-1], groups, shape[-1] // groups)
    acc = g.float() if g.dtype in (torch.float16, torch.bfloat16) else g
    g = torch.nn.functional.normalize(acc, dim=-1).to(t.dtype)
    return g.reshape(shape)


def l2norm_tensors(*tensors, groups=1):
    """l2-normalise each tensor over `groups` chunks of the last dim; results keep the dtype of
    the first tensor (reference py:57-65)."""
    assert len(tensors) > 0
    dtype = tensors[0].dtype
    out = []
    for t in tensors:
        assert t.shape[-1] % groups == 0, "groups must divide the feature dimension"
        gs = t.shape[-1] // groups
        fused = (t.is_cuda and t.dtype in _KERNEL_DTYPES and t.ndim in (3, 4)
                 and t.shape[-1] in (32, 64, 128, 256) and (gs & (gs - 1)) == 0)
        y = _L2Norm.apply(t, groups) if fused else _l2norm_torch(t, groups)
        out.append(y.type(dtype))
    return tuple(out)


def plain_cosine_sim_attention(q, k, v, mask=None, attn_bias=None, scale=8, groups=1, causal=False,
                               l2norm_qk=True, attn_bias_batch_dim=False, window=None):
    """The naive, un-fused formulation (reference py:75-126): explicit similarity matrix,
    masked softmax, weighted sum.  Public API of the reference package (used by
    transformer.py when the fused kernel is switched off); any device, any float dtype.
    window: sliding-window attention as in flash_cosine_sim_attention, applied as a band mask."""
    assert not (causal and exists(mask)), "mask should not be supplied if causality is needed"
    window = _check_window(window, None, "plain_cosine_sim_attention")
    merged = q.ndim == 3
    single_head_kv = k.ndim == 3
    if merged:
        assert k.ndim == 3 and v.ndim == 3, (
            "if batch and heads are merged for queries, keys and values must also similarly "
            "have only 3 dimensions")
        attn_bias_batch_dim = True
        q = q.unsqueeze(1)
    elif not single_head_kv:
        _check_kv_heads(q, k, v)
    # grouped-query attention: q viewed as (batch, kv_heads, group, seq, dim) against k, v unsqueezed at dim 2
    # (autograd sums each group's gradients into its key/value head)
    grouped = not merged and not single_head_kv and k.shape[1] != q.shape[1]
    if grouped:
        B, H = q.shape[:2]
        Hk = k.shape[1]
        q = q.unflatten(1, (Hk, H // Hk))
        k, v = k.unsqueeze(2), v.unsqueeze(2)
        if exists(attn_bias) and not attn_bias_batch_dim:
            attn_bias = attn_bias.unflatten(0, (Hk, H // Hk))
    if l2norm_qk:
        q, k = (_l2norm_torch(t, groups) for t in (q, k))
    kk = k.unsqueeze(1) if single_head_kv else k
    vv = v.unsqueeze(1) if single_head_kv else v
    sim = torch.matmul(q, kk.transpose(-1, -2)) * scale
    lead = (None,) * (sim.ndim - 3)             # the head dims between batch and (i, j)
    if exists(attn_bias):
        sim = sim + (attn_bias[(slice(None),) + lead] if attn_bias_batch_dim else attn_bias)
    neg = -torch.finfo(sim.dtype).max
    if causal:
        i, j = sim.shape[-2:]
        future = torch.ones((i, j), device=q.device, dtype=torch.bool).triu(j - i + 1)
        sim = sim.masked_fill(future, neg)
    if exists(mask):
        sim = sim.masked_fill(~mask[(slice(None),) + lead + (None, slice(None))], neg)
    if window:
        sim = sim.masked_fill(~_band(sim.shape[-2], sim.shape[-1], window, causal, q.device), neg)
    out = torch.matmul(sim.softmax(dim=-1), vv)
    if grouped:
        out = out.flatten(1, 2)
    return out.squeeze(1) if merged else out


# --------------------------------------------------------------------------------------------
# float32 inputs (reference: Float is dispatched in forward and backward, cu:1702-1703, 1832-1834; half of
# its test grid is f32, tests/test.py:33-35).  The wgmma kernels take 16-bit operands, so float32
# tensors run on the SAME fused fp16 kernels at tf32-class operand precision - fp16 and tf32 share the
# 11-bit significand - with fp32 accumulation throughout:
#   * q, k are l2-normalised in fp32 first (|q_hat|, |k_hat| <= 1 sit comfortably in fp16), then rounded;
#   * v and the incoming gradient are scaled by a power of two computed ON THE DEVICE from their max
#     magnitude (exact, undone afterwards), so fp16's narrower exponent range never clips them;
#   * o, dq, dk, dv come back as float32 (one rounding to 11 bits at the kernels' output).
# Every op around the kernels is an asynchronous elementwise torch op: no host synchronisation.
# --------------------------------------------------------------------------------------------
def _pow2_scale(t, top_exp):
    """Power of two s (1-element fp32 tensor, on t's device) with amax|t| / s in [2^(top_exp-1), 2^top_exp)."""
    amax = torch.linalg.vector_norm(t.detach(), float("inf")).float().clamp_min(1e-30).reshape(1)
    return torch.exp2(torch.floor(torch.log2(amax)) + 1 - top_exp)


_F32_CAST_DIMS = (16, 32, 64, 128)


def _cast16(x, half, groups, mul, reciprocal, Dp):
    """float32 x -> ((l2norm over `groups` +) scaled) 16-bit tensor with Dp >= D zero-padded features, and rnorm.
    One fused CUDA pass (fcsa_f32_cast) for head dims 16 / 32 / 64 / 128; other multiples of 8 (96) take torch ops."""
    D = x.shape[-1]
    if D in _F32_CAST_DIMS and x.ndim in (3, 4):
        return _ext().f32_cast(x, half == torch.bfloat16, groups, mul, reciprocal, Dp)
    assert groups == 0
    y = x if mul is None else (x / mul if reciprocal else x * mul)
    y = y.to(half)
    return (torch.nn.functional.pad(y, (0, Dp - D)) if Dp > D else y), None


def _uncast16(dy, y, rnorm, groups, mul, reciprocal, D):
    """Backward of _cast16: float32 gradient w.r.t. y (possibly padded) -> float32 gradient w.r.t. x."""
    if D in _F32_CAST_DIMS and dy.ndim in (3, 4):
        return _ext().f32_cast_backward(dy, y, rnorm, groups, mul, reciprocal, D)
    assert groups == 0
    g = dy[..., :D]
    return g if mul is None else (g / mul if reciprocal else g * mul)


class _Float32OnHalfKernels(Function):
    """float32 q, k, v (+ bias) -> float32 o, on the 16-bit kernels: operands are rounded to `half` (fp16: 11-bit
    significand, tf32's; bf16 when fp16's exponent range is too small), v and the incoming gradient are brought to
    [1, 2) by an exact power-of-two scale chosen on the device (the kernels form dP = dO V^T and dS = P (dP - delta) in
    the 16-bit range, so operands keep headroom), accumulation is fp32 and the results are written as float32 straight
    from the accumulators (out_f32).  norm_groups > 0: q, k arrive RAW and are l2-normalised by the cast pass itself
    (its backward is the cast pass of the gradients); 0: they are used as given."""

    @staticmethod
    def forward(ctx, q, k, v, mask, attn_bias, scale, causal, attn_bias_batch_dim, shift, half, use_amax, norm_groups,
                window=0, deterministic=False):
        ext = _ext()
        D = q.shape[-1]
        Dp = D if D in _KERNEL_HEAD_DIMS else (64 if D < 64 else 128)        # 16 / 32 / 96: zero-padded features
        sv = _pow2_scale(v, 1)
        qh, rq = _cast16(q, half, norm_groups, None, False, Dp)
        kh, rk = _cast16(k, half, norm_groups, None, False, Dp)
        vh, _ = _cast16(v, half, 0, sv, True, Dp)
        batch_dim = bool(attn_bias_batch_dim) or q.ndim == 3
        bias = amax = None
        if exists(attn_bias):
            bias = ext.prepare_bias(qh, kh, vh, attn_bias.detach().to(half), batch_dim)
            if use_amax:
                amax = attn_bias.detach().amax().float().reshape(1)
        needs_grad = any(ctx.needs_input_grad[:3]) or (exists(attn_bias) and ctx.needs_input_grad[4])
        o, inv_l = ext.forward_ex(qh, kh, vh, mask, bias, batch_dim, amax, scale, shift, causal, 0, needs_grad, True,
                                  window)[:2]
        if needs_grad:
            ctx.save_for_backward(o, inv_l, qh, kh, vh, mask, bias, amax, sv, rq, rk)
            ctx.params = (scale, shift, causal, batch_dim, D, exists(attn_bias) and ctx.needs_input_grad[4], norm_groups,
                          window, deterministic)
        return o[..., :D] * sv

    @staticmethod
    def backward(ctx, g):
        o, inv_l, qh, kh, vh, mask, bias, amax, sv, rq, rk = ctx.saved_tensors
        scale, shift, causal, batch_dim, D, bias_grad, norm_groups, window, deterministic = ctx.params
        # o = o_kernel * sv, so d(o_kernel) = g * sv; it enters the kernels as fp16 scaled into [1, 2):
        # g * sv / sg with sg = pg * sv, pg = pow2 scale of g  ->  the cast pass computes g / pg
        pg = _pow2_scale(g, 1)
        gh, _ = _cast16(g, qh.dtype, 0, pg, True, qh.shape[-1])
        dq, dk, dv, db = _ext().backward_ex(gh, o, inv_l, qh, kh, vh, None, None, mask, bias, batch_dim, amax,
                                            bias_grad, None, scale, shift, causal, 0, True, window, deterministic)
        sg = pg * sv                                          # undo the gradient scale; dv also undoes v / sv
        dq = _uncast16(dq, qh, rq, norm_groups, sg, False, D)
        dk = _uncast16(dk, kh, rk, norm_groups, sg, False, D)
        dv = _uncast16(dv, None, None, 0, pg, False, D)
        return dq, dk, dv, None, (db * sg if bias_grad else None), None, None, None, None, None, None, None, None, None


def _float32_on_half_kernels(q, k, v, mask, attn_bias, scale, groups, causal, l2norm_qk, attn_bias_batch_dim, window=0,
                             deterministic=False):
    D = q.shape[-1]
    assert D % groups == 0, "groups must divide the head dim"
    # fp16 (11-bit significand, like tf32) whenever its exponent range holds exp(scale * q.k); bf16 (8 bits, fp32's
    # range) for grouped l2norm with a large scale*groups and for un-normalised q, k
    h = torch.float16 if (l2norm_qk and scale * groups <= _FP16_GROUPED_RANGE) else torch.bfloat16
    if h == torch.bfloat16:
        _warn_once("f32-bf16", "flash_cosine_sim_attention: float32 inputs with scale*groups > "
                               f"{_FP16_GROUPED_RANGE:g} (or l2norm_qk=False) run on the bfloat16 kernels - fp16's "
                               "exponent range cannot hold exp(scale*q.k) there; operands carry 8 significant bits")
    gs = D // groups
    norm_groups = 0
    if l2norm_qk:
        if D in _F32_CAST_DIMS and (gs & (gs - 1)) == 0 and q.ndim in (3, 4):
            norm_groups = groups                                              # fused into the cast pass
        else:
            q, k = _l2norm_torch(q, groups), _l2norm_torch(k, groups)       # fp32, differentiable
    shift = _choose_shift(h, scale, groups if l2norm_qk else 1, l2norm_qk)
    return _Float32OnHalfKernels.apply(q, k, v, mask, attn_bias, float(scale), bool(causal), bool(attn_bias_batch_dim),
                                       float(shift), h, bool(l2norm_qk and h == torch.float16), int(norm_groups),
                                       int(window), deterministic)


_warned = set()


def _warn_once(key, msg):
    if key not in _warned:
        _warned.add(key)
        warnings.warn(msg, stacklevel=3)


def flash_cosine_sim_attention(q, k, v, mask=None, attn_bias=None, scale=8, groups=1, causal=False,
                               l2norm_qk=True, attn_bias_batch_dim=False, l2norm_groups=None, window=None,
                               deterministic=False):
    """Fused cosine-similarity attention (reference py:308-334, same arguments and meaning;
    `l2norm_groups` is accepted as an alias of `groups`).

    window: sliding-window (local) attention, None or a positive int W.  With off = n_k - n_q (the bottom-right
    alignment of causal masking) and d = i + off - j, key j is visible to query i iff 0 <= d < W with causal=True (the
    query itself and the W - 1 keys before it) and iff |d| < W otherwise, on top of `mask`.  The kernels skip the key
    tiles outside the band, so a causal pass costs O(n * W).  Rows that see no key give 0.  Not with attn_bias.

    deterministic: True runs the backward without atomics (a dK / dV kernel and a dQ kernel that sum in a fixed
    order), so dq, dk and dv are bitwise the same from run to run and a batch element's do not depend on the rest of
    the batch.  Slower than the default backward; the forward is the same.  Not with attn_bias.

    Every supported input runs the hand-written sm_90a kernels: float16 / bfloat16 natively, float32 at
    tf32-class operand precision on the fp16 kernels (see _float32_on_half_kernels), head dims 64 and 128
    natively and 16 / 32 / 96 (any multiple of 8 below 128) on zero-padded features.  Anything else raises:
    there is no un-fused or CPU fallback."""
    if exists(l2norm_groups):
        groups = l2norm_groups
    assert not (causal and exists(mask)), "mask should not be supplied if causality is needed"
    window = _check_window(window, attn_bias, "flash_cosine_sim_attention")
    deterministic = _check_deterministic(deterministic, attn_bias, "flash_cosine_sim_attention")
    if not q.is_cuda:
        raise RuntimeError(
            "flash_cosine_sim_attention: CUDA tensors required - this build has no CPU path "
            "(use plain_cosine_sim_attention on CPU tensors)")
    D = q.shape[-1]
    if not (k.dtype == q.dtype and v.dtype == q.dtype):
        raise TypeError("flash_cosine_sim_attention: q, k, v must share one dtype")
    _check_kv_heads(q, k, v)
    if D > 128 or D % 8 != 0 or D % groups != 0:
        raise NotImplementedError(
            f"flash_cosine_sim_attention: head_dim {D} with groups {groups} has no sm_90a kernel (head dims: multiples "
            "of 8 up to 128; the reference supports 16, 32, 64, 96, 128 - cu:84)")
    if exists(attn_bias) and not attn_bias.is_cuda:
        raise RuntimeError("flash_cosine_sim_attention: attn_bias must be a CUDA tensor")
    if q.dtype == torch.float32:
        return _float32_on_half_kernels(q, k, v, mask, attn_bias, scale, groups, causal, l2norm_qk, attn_bias_batch_dim,
                                        window, deterministic)
    if q.dtype not in _KERNEL_DTYPES:
        raise TypeError(f"flash_cosine_sim_attention: dtype {q.dtype} is not supported (float16, bfloat16, float32)")
    _warn_fp16_overflow(q.dtype, scale, groups, l2norm_qk)
    if D not in _KERNEL_HEAD_DIMS:
        # Head dims the kernels are not instantiated for (the reference's 16, 32 and 96): zero-pad the
        # features to 64 / 128 and run the same wgmma kernels.  Zero features change neither q.k nor
        # the norms (the l2norm runs first, on the real features), the padded output columns are
        # zero and sliced off; autograd takes care of the slices.  Costs two pad copies per tensor.
        Dp = 64 if D < 64 else 128
        if l2norm_qk:
            q, k = _l2norm_torch(q, groups), _l2norm_torch(k, groups)
        pad = lambda t: torch.nn.functional.pad(t, (0, Dp - D))
        if exists(attn_bias):
            shift = _choose_shift(q.dtype, scale, groups if l2norm_qk else 1, l2norm_qk)
            amax = (attn_bias.detach().amax().float().reshape(1)
                    if (q.dtype == torch.float16 and l2norm_qk) else None)
            o = FlashCosineSimAttention.apply(pad(q), pad(k), pad(v), mask, attn_bias, float(scale), bool(causal),
                                              bool(attn_bias_batch_dim), float(shift), amax)
        else:
            o = _FusedCosineSimAttention.apply(pad(q), pad(k), pad(v), mask, float(scale), bool(causal), 1, False,
                                               int(groups) if l2norm_qk else 0, window, deterministic)
        return o[..., :D]
    if exists(attn_bias):
        # additive bias: l2norm kernels (with their own backward), then the BIAS instantiations of the
        # attention kernels; d_bias is reduced in fp32 and returned in the bias's dtype
        if l2norm_qk:
            q, k = l2norm_tensors(q, k, groups=groups)
        shift = _choose_shift(q.dtype, scale, groups if l2norm_qk else 1, l2norm_qk)
        amax = None
        if q.dtype == torch.float16 and l2norm_qk:
            # p = exp(logit - shift) is stored in fp16: keep its top below 2^15 whatever the bias adds.  The
            # bound stays on the device (a 1-element tensor the kernels read) - no host synchronisation.
            amax = attn_bias.detach().amax().float().reshape(1)
        return FlashCosineSimAttention.apply(q, k, v, mask, attn_bias, float(scale), bool(causal),
                                             bool(attn_bias_batch_dim), float(shift), amax)
    gs = q.shape[-1] // groups
    assert (gs & (gs - 1)) == 0, "groups must divide the head dim into power-of-two chunks"
    return _FusedCosineSimAttention.apply(q, k, v, mask, float(scale), bool(causal), int(groups), bool(l2norm_qk), 0,
                                          window, deterministic)


def _check_kv_cache_args(q, k_cache, v_cache, cache_seqlens, k, v, groups, mask, attn_bias, cu_seqlens_q=None,
                         max_seqlen_q=None, window=0, rolling=False):
    """Everything flash_cosine_sim_attention_with_kv_cache rejects before touching a device.  With cu_seqlens_q, q, k
    and v are packed: (total_q, heads, head_dim) and (total_q, kv_heads, head_dim).  window: _check_window's."""
    packed = cu_seqlens_q is not None
    if exists(attn_bias):
        raise NotImplementedError("flash_cosine_sim_attention_with_kv_cache: attn_bias is not supported")
    if exists(mask):
        raise NotImplementedError("flash_cosine_sim_attention_with_kv_cache: no key-padding mask - cache_seqlens "
                                  "gives each batch element's valid cache rows")
    if packed and (q.ndim != 3 or k_cache.ndim != 4 or v_cache.ndim != 4):
        raise ValueError("flash_cosine_sim_attention_with_kv_cache: with cu_seqlens_q, q must be packed as (total_q, "
                         "heads, head_dim) and the caches (batch, kv_heads, capacity, head_dim)")
    if q.ndim != (3 if packed else 4) or k_cache.ndim != 4 or v_cache.ndim != 4:
        raise ValueError("flash_cosine_sim_attention_with_kv_cache: q must be (batch, heads, seq, head_dim) and the "
                         "caches (batch, kv_heads, capacity, head_dim); merged batch-heads are not supported")
    if exists(k) != exists(v):
        raise ValueError("flash_cosine_sim_attention_with_kv_cache: pass both k and v, or neither")
    if torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in (q, k_cache, v_cache, k, v)):
        raise RuntimeError("flash_cosine_sim_attention_with_kv_cache is inference-only (no autograd): call it under "
                           "torch.no_grad() or with tensors that do not require grad")
    if q.dtype == torch.float32:
        raise TypeError("flash_cosine_sim_attention_with_kv_cache: float32 is not supported - use float16 or "
                        "bfloat16 (run the model in 16-bit or under autocast)")
    if q.dtype not in _KERNEL_DTYPES:
        raise TypeError(f"flash_cosine_sim_attention_with_kv_cache: dtype {q.dtype} is not supported")
    if any(t is not None and t.dtype != q.dtype for t in (k_cache, v_cache, k, v)):
        raise TypeError("flash_cosine_sim_attention_with_kv_cache: q, the caches, k and v must share one dtype")
    D = q.shape[-1]
    if D not in _KERNEL_HEAD_DIMS:
        raise NotImplementedError(f"flash_cosine_sim_attention_with_kv_cache: head_dim {D} (64 and 128 only)")
    if k_cache.shape != v_cache.shape or (not packed and k_cache.shape[0] != q.shape[0]) or k_cache.shape[-1] != D:
        raise ValueError(f"flash_cosine_sim_attention_with_kv_cache: caches of shape {tuple(k_cache.shape)} and "
                         f"{tuple(v_cache.shape)} do not match q {tuple(q.shape)}")
    hk = k_cache.shape[1]
    if hk <= 0 or q.shape[1] % hk != 0:
        raise ValueError(f"flash_cosine_sim_attention_with_kv_cache: kv_heads ({hk}) must divide the query heads "
                         f"({q.shape[1]})")
    if packed and exists(k) and (k.shape != v.shape or k.shape != (q.shape[0], hk, D)):
        raise ValueError(f"flash_cosine_sim_attention_with_kv_cache: k and v must be packed like q, (total_q, kv_heads, "
                         f"head_dim) = {(q.shape[0], hk, D)} (got {tuple(k.shape)} and {tuple(v.shape)})")
    if not packed and exists(k) and (k.shape != v.shape or k.ndim != 4 or k.shape[:2] != k_cache.shape[:2]
                                     or k.shape[-1] != D):
        raise ValueError(f"flash_cosine_sim_attention_with_kv_cache: k and v must be (batch, kv_heads, n_new, {D}) "
                         f"like the caches (got {tuple(k.shape)} and {tuple(v.shape)})")
    B = k_cache.shape[0]
    if not torch.is_tensor(cache_seqlens) or cache_seqlens.dtype != torch.int32 or cache_seqlens.shape != (B,):
        raise TypeError("flash_cosine_sim_attention_with_kv_cache: cache_seqlens must be an int32 tensor of shape "
                        f"({B},)")
    if not cache_seqlens.is_contiguous():
        raise ValueError("flash_cosine_sim_attention_with_kv_cache: cache_seqlens must be contiguous (the kernels read "
                         "it as a dense array and a CUDA graph replay reads the caller's buffer; not a strided or "
                         "expanded view)")
    if packed:
        _check_cu_seqlens_q(q, B, cu_seqlens_q, max_seqlen_q)
    elif max_seqlen_q is not None:
        raise ValueError("flash_cosine_sim_attention_with_kv_cache: max_seqlen_q is for packed new tokens - pass "
                         "cu_seqlens_q with it")
    gs = D // groups if groups > 0 and D % groups == 0 else 0
    if gs == 0 or (gs & (gs - 1)) != 0:
        raise ValueError(f"flash_cosine_sim_attention_with_kv_cache: groups {groups} must divide head_dim {D} into "
                         "power-of-two chunks")
    if not isinstance(rolling, bool):
        raise TypeError(f"flash_cosine_sim_attention_with_kv_cache: rolling must be a bool, got {rolling!r}")
    if rolling:
        _check_rolling(q, k_cache, k, window, max(max_seqlen_q, 1) if packed else q.shape[2], packed)
    if not (q.is_cuda and cache_seqlens.is_cuda and (not packed or cu_seqlens_q.is_cuda)):
        raise RuntimeError("flash_cosine_sim_attention_with_kv_cache: CUDA tensors required (cache_seqlens and "
                           "cu_seqlens_q included: the host never reads them) - this build has no CPU path")


def _check_rolling(q, k_cache, k, window, n, packed):
    """A rolling cache of C = k_cache.shape[2] rows for calls of at most n new tokens: it needs a window W, whole
    128-row tiles and C >= W + n - 1 (the keys a call sees, [T_b - n - W + 1, T_b), must survive its own append)."""
    name = "flash_cosine_sim_attention_with_kv_cache"
    C = k_cache.shape[2]
    if window == 0:
        raise ValueError(f"{name}: a rolling cache needs a window (it keeps the window's keys only)")
    if C % 128 != 0:
        raise ValueError(f"{name}: a rolling cache's capacity must be a multiple of 128 rows, got {C}")
    if C < window + n - 1:
        raise ValueError(f"{name}: a rolling cache of {C} rows is too small for window {window} and {n} new tokens "
                         f"per call: it needs at least window + n - 1 = {window + n - 1} rows")
    if not packed and k is not None and k.shape[2] != q.shape[2]:
        raise ValueError(f"{name}: with a rolling cache, k and v bring one row per query ({q.shape[2]}), got "
                         f"{k.shape[2]}")


def _check_cu_seqlens_q(q, B, cu_seqlens_q, max_seqlen_q):
    """The packed new tokens of flash_cosine_sim_attention_with_kv_cache: cu_seqlens_q (B + 1,) and max_seqlen_q."""
    name = "flash_cosine_sim_attention_with_kv_cache"
    if not torch.is_tensor(cu_seqlens_q) or cu_seqlens_q.dtype != torch.int32 or cu_seqlens_q.ndim != 1:
        raise TypeError(f"{name}: cu_seqlens_q must be an int32 tensor of shape (batch + 1,) = ({B + 1},)")
    if cu_seqlens_q.shape[0] != B + 1:
        raise ValueError(f"{name}: cu_seqlens_q has {cu_seqlens_q.shape[0]} entries; the caches' batch {B} needs "
                         f"{B + 1}")
    if not cu_seqlens_q.is_contiguous():
        raise ValueError(f"{name}: cu_seqlens_q must be contiguous (the kernels read it as a dense array and a CUDA "
                         "graph replay reads the caller's buffer; not a strided or expanded view)")
    if cu_seqlens_q.device != q.device:
        raise RuntimeError(f"{name}: cu_seqlens_q must be on q's device ({q.device}, got {cu_seqlens_q.device}); the "
                           "host never reads it")
    if isinstance(max_seqlen_q, bool) or not isinstance(max_seqlen_q, int) or max_seqlen_q < 0:
        raise TypeError(f"{name}: max_seqlen_q must be a non-negative Python int with cu_seqlens_q (got "
                        f"{max_seqlen_q!r})")


def flash_cosine_sim_attention_with_kv_cache(q, k_cache, v_cache, cache_seqlens, k=None, v=None, scale=8, groups=1,
                                             causal=True, l2norm_qk=True, mask=None, attn_bias=None, window=None,
                                             cu_seqlens_q=None, max_seqlen_q=None, rolling=False):
    """Cosine-sim attention of new queries against a key/value cache, for inference (generation).

    q: (batch, heads, n_q, head_dim) new queries.  k_cache, v_cache: (batch, kv_heads, capacity, head_dim), kv_heads
    dividing heads (query head h reads kv head h // (heads // kv_heads)).  cache_seqlens: int32 CUDA tensor (batch,)
    of valid cache rows L_b; it is never read on the host, so a call does not synchronise and can be captured in a
    CUDA graph.  k, v: optional (batch, kv_heads, n_new, head_dim), written into the caches at rows
    [L_b, L_b + n_new) by this call.  cache_seqlens is NOT advanced: the caller adds n_new afterwards.

    The cache holds keys in the form the kernel reads them: with l2norm_qk=True the appended rows are
    l2norm(k, groups) rounded to the cache dtype (so the prefix is never renormalised), with l2norm_qk=False k as
    given.  v is stored as given.  With T_b = L_b + n_new, new query i sees key j iff j < T_b and, with causal=True,
    j <= i + T_b - n_q (the bottom-right rule of flash_cosine_sim_attention with n_k = T_b); rows that see no key
    give 0.  scale, groups and the exponent shift are those of flash_cosine_sim_attention.

    L_b + n_new must not exceed the capacity: rows that do not fit are not written, and T_b is clamped to the
    capacity.  float16 / bfloat16 and head dims 64 and 128 only; no autograd, attn_bias, mask, float32 or merged
    batch-heads.  window: sliding-window attention as in flash_cosine_sim_attention with n_k = T_b; a step then reads
    the tiles of its window, not the whole valid cache (the cache itself stays full-length unless rolling=True).
    Returns o (batch, heads, n_q, head_dim).

    A different number of new tokens per batch element (speculative verification, chunked prefill, ragged prompts):
    cu_seqlens_q, a contiguous int32 CUDA tensor (batch + 1,), non-decreasing, and max_seqlen_q, a Python int at least
    every length (it sizes the grid; longer sequences are clamped to it).  q is then packed as (total_q, heads,
    head_dim) and k, v (optional) as (total_q, kv_heads, head_dim) with the same boundaries: batch element b brings
    n_b = cu_seqlens_q[b + 1] - cu_seqlens_q[b] new tokens at rows [cu_seqlens_q[b], cu_seqlens_q[b + 1]) and appends
    its k, v rows at cache rows [L_b, L_b + n_b).  Without k, v nothing is appended and n_b counts queries only.  The
    rules above hold per element with n_q = n_b and T_b = min(L_b + (n_b if appending, else 0), capacity).  Rows
    outside every sequence ([0, cu_seqlens_q[0]) and [cu_seqlens_q[-1], total_q)) give 0.  cu_seqlens_q is never read
    on the host either, and cache_seqlens is not advanced: add cu_seqlens_q[1:] - cu_seqlens_q[:-1] afterwards.
    Returns o (total_q, heads, head_dim).

    rolling=True: the caches are rolling caches for sliding-window decoding, rings of C = capacity rows that keep the
    window's keys only, so their memory is bounded by the window instead of the sequence (as Mistral-style rolling
    caches).  The rules above then read:
      - absolute position p lives at ring row p mod C;
      - cache_seqlens[b] = L_b counts every token element b has seen, and may be far larger than C; the caller still
        advances it after the call;
      - T_b = L_b + n_b (n_b = n_q dense, or the packed length when appending) with no clamp to C, and the window rule
        holds over absolute positions: query i sees key j iff 0 <= i + T_b - n_b - j < window (causal) or
        |i + T_b - n_b - j| < window;
      - new row n of element b is written to ring row (L_b + n) mod C.
    A window is required, C must be a multiple of 128, and C >= window + n - 1 with n = n_q (dense) or max_seqlen_q
    (packed): below that, a call's append would overwrite a key that one of its own queries still sees.  Dense k, v
    bring one row per query.  L_b + n_b must
    stay below 2^31 - 128; cache_seqlens is never read on the host, so this is not checked.  With the same number of
    key splits, o is bitwise what a full-length cache holding the same keys gives."""
    window = _check_window(window, attn_bias, "flash_cosine_sim_attention_with_kv_cache")
    _check_kv_cache_args(q, k_cache, v_cache, cache_seqlens, k, v, groups, mask, attn_bias, cu_seqlens_q, max_seqlen_q,
                         window, rolling)
    _warn_fp16_overflow(q.dtype, scale, groups, l2norm_qk)
    shift = _choose_shift(q.dtype, scale, groups, l2norm_qk)
    g = int(groups) if l2norm_qk else 0
    if cu_seqlens_q is None:
        return _ext().decode(q, k_cache, v_cache, cache_seqlens, k, v, float(scale), float(shift), bool(causal), g,
                             window, rolling)
    if q.shape[0] == 0:
        return q.new_empty(q.shape)
    return _ext().decode_varlen(q, k_cache, v_cache, cache_seqlens, cu_seqlens_q, max(int(max_seqlen_q), 1), k, v,
                                float(scale), float(shift), bool(causal), g, window, rolling)


class _FusedVarlenAttention(Function):
    """One autograd node for packed sequences: l2norm(q), l2norm(k) -> attention, all in CUDA kernels."""

    @staticmethod
    def forward(ctx, q, k, v, cu_q, cu_k, max_q, max_k, scale, causal, groups, l2norm_qk, window=0, deterministic=False):
        shift = _choose_shift(q.dtype, scale, groups, l2norm_qk)
        g = groups if l2norm_qk else 0
        needs_grad = any(ctx.needs_input_grad[:3])
        o, inv_l, qn, kn, rq, rk = _ext().forward_varlen(q, k, v, cu_q, cu_k, max_q, max_k, scale, shift, causal, g,
                                                         needs_grad, window)
        if needs_grad:
            if not l2norm_qk:
                qn, kn = q, k
            ctx.save_for_backward(o, inv_l, qn, kn, v, rq, rk, cu_q, cu_k)
            ctx.params = (max_q, max_k, scale, shift, causal, g, window, deterministic)
        return o

    @staticmethod
    def backward(ctx, do):
        o, inv_l, qn, kn, v, rq, rk, cu_q, cu_k = ctx.saved_tensors
        max_q, max_k, scale, shift, causal, g, window, deterministic = ctx.params
        dq, dk, dv = _ext().backward_varlen(do, o, inv_l, qn, kn, v, rq, rk, cu_q, cu_k, max_q, max_k, scale, shift,
                                            causal, g, window, deterministic)
        return (dq, dk, dv) + (None,) * 10


class _EmptyVarlenAttention(Function):
    """Packed tensors with no query or no key rows: o = 0 and zero gradients, with no kernel launch."""

    @staticmethod
    def forward(ctx, q, k, v):
        ctx.kv = (k.shape, v.shape, k.dtype, k.device)
        return q.new_zeros(q.shape)

    @staticmethod
    def backward(ctx, do):
        ks, vs, dtype, device = ctx.kv
        return (torch.zeros_like(do), torch.zeros(ks, dtype=dtype, device=device),
                torch.zeros(vs, dtype=dtype, device=device))


def _check_varlen_args(q, k, v, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k, groups, mask, attn_bias):
    """Everything flash_cosine_sim_attention_varlen rejects before touching a device."""
    name = "flash_cosine_sim_attention_varlen"
    if exists(attn_bias):
        raise NotImplementedError(f"{name}: attn_bias is not supported")
    if exists(mask):
        raise NotImplementedError(f"{name}: no key-padding mask - cu_seqlens_k gives each sequence's keys")
    if q.ndim != 3 or k.ndim != 3 or v.ndim != 3:
        raise ValueError(f"{name}: q must be (total_q, heads, head_dim) and k, v (total_k, kv_heads, head_dim)")
    if q.dtype == torch.float32:
        raise TypeError(f"{name}: float32 is not supported - use float16 or bfloat16")
    if q.dtype not in _KERNEL_DTYPES:
        raise TypeError(f"{name}: dtype {q.dtype} is not supported (float16, bfloat16)")
    if k.dtype != q.dtype or v.dtype != q.dtype:
        raise TypeError(f"{name}: q, k, v must share one dtype")
    D = q.shape[-1]
    if D not in _KERNEL_HEAD_DIMS:
        raise NotImplementedError(f"{name}: head_dim {D} (64 and 128 only)")
    if k.shape != v.shape or k.shape[-1] != D:
        raise ValueError(f"{name}: k and v must both be (total_k, kv_heads, {D}) (got {tuple(k.shape)} and "
                         f"{tuple(v.shape)})")
    hk = k.shape[1]
    if hk <= 0 or q.shape[1] % hk != 0:
        raise ValueError(f"{name}: kv_heads ({hk}) must divide the query heads ({q.shape[1]})")
    for t in (cu_seqlens_q, cu_seqlens_k):
        if not torch.is_tensor(t) or t.dtype != torch.int32 or t.ndim != 1 or t.shape[0] < 2:
            raise TypeError(f"{name}: cu_seqlens_q and cu_seqlens_k must be int32 tensors of shape (batch + 1,)")
        if not t.is_contiguous():
            raise ValueError(f"{name}: cu_seqlens must be contiguous (the kernels read them as dense arrays and a CUDA "
                             "graph replay reads the caller's buffer; not a strided or expanded view)")
    if cu_seqlens_q.shape != cu_seqlens_k.shape:
        raise ValueError(f"{name}: cu_seqlens_q and cu_seqlens_k must have the same length")
    for m in (max_seqlen_q, max_seqlen_k):
        if isinstance(m, bool) or not isinstance(m, int) or m < 0:
            raise TypeError(f"{name}: max_seqlen_q and max_seqlen_k must be non-negative Python ints")
    gs = D // groups if groups > 0 and D % groups == 0 else 0
    if gs == 0 or (gs & (gs - 1)) != 0:
        raise ValueError(f"{name}: groups {groups} must divide head_dim {D} into power-of-two chunks")
    if not (q.is_cuda and k.is_cuda and v.is_cuda):
        raise RuntimeError(f"{name}: CUDA tensors required - this build has no CPU path")
    if not (cu_seqlens_q.is_cuda and cu_seqlens_k.is_cuda and cu_seqlens_q.device == q.device
            and cu_seqlens_k.device == q.device):
        raise RuntimeError(f"{name}: cu_seqlens must be on q's CUDA device (the host never reads them)")


def flash_cosine_sim_attention_varlen(q, k, v, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k, scale=8,
                                      groups=1, causal=False, l2norm_qk=True, mask=None, attn_bias=None, window=None,
                                      deterministic=False):
    """Cosine-sim attention over packed variable-length sequences (training: forward and backward).

    q: (total_q, heads, head_dim); k, v: (total_k, kv_heads, head_dim), kv_heads dividing heads (query head h reads kv
    head h // (heads // kv_heads)).  Views with a contiguous head dim (e.g. slices of a packed projection output) are
    read without a copy.  cu_seqlens_q, cu_seqlens_k: contiguous int32 CUDA tensors (batch + 1,), non-decreasing from 0;
    sequence b is query rows [cu_seqlens_q[b], cu_seqlens_q[b + 1]) and key rows [cu_seqlens_k[b], cu_seqlens_k[b + 1]).
    Pass the same tensor twice for self-attention.  They are never read on the host, so a call does not synchronise and
    a training step can be captured in a CUDA graph.  max_seqlen_q, max_seqlen_k: Python ints, at least every length
    (they size the grids; lengths above them are clamped).

    Each sequence gets what flash_cosine_sim_attention gives on it alone: the same scale, groups, l2norm and exponent
    shift; causal masking is bottom-right per sequence (key j visible to query i iff j <= i + len_k - len_q).  Empty
    sequences are allowed, and query rows that see no key give 0.  Rows outside every sequence ([0, cu[0]) and
    [cu[-1], total), e.g. the unused end of a fixed-size packing buffer) give o = 0 and zero gradients.  Packed tensors
    with no query or no key rows give zeros (and zero gradients) without a kernel launch.  float16 / bfloat16 and head dims 64 and 128 only; no float32, mask or
    attn_bias.  window: sliding-window attention as in flash_cosine_sim_attention, with each sequence's own lengths.
    deterministic: the backward of flash_cosine_sim_attention(deterministic=True); a sequence's gradients are then
    also bitwise independent of the other sequences in the pack.
    Returns o (total_q, heads, head_dim)."""
    window = _check_window(window, attn_bias, "flash_cosine_sim_attention_varlen")
    deterministic = _check_deterministic(deterministic, attn_bias, "flash_cosine_sim_attention_varlen")
    _check_varlen_args(q, k, v, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k, groups, mask, attn_bias)
    _warn_fp16_overflow(q.dtype, scale, groups, l2norm_qk)
    if q.shape[0] == 0 or k.shape[0] == 0:
        return _EmptyVarlenAttention.apply(q, k, v)
    return _FusedVarlenAttention.apply(q, k, v, cu_seqlens_q, cu_seqlens_k, max(int(max_seqlen_q), 1),
                                       max(int(max_seqlen_k), 1), float(scale), bool(causal), int(groups),
                                       bool(l2norm_qk), window, deterministic)
