"""Decoder-only transformer around the attention operator - the caller side of the hot path.

Same public classes and constructor arguments as the reference's
flash_cosine_sim_attention/transformer.py (`Attention` tf:59-105, `CosineSimCausalTransformer`
tf:109-202), same parameter names (`to_q/to_k/to_v/to_out`, `token_emb`, `pos_emb`, `layers`,
`to_logits`) so state dicts interchange, and `train.py` runs against it unchanged.  Re-authored,
not copied: this module is glue, the work happens in flash_cosine_sim_attention().

One deliberate fix: the reference forwards `attn_l2norm_groups` as `groups=` into `Attention`,
where it falls into **kwargs and is overridden by the call-time `groups=self.l2norm_groups` (=1)
(tf:66, 80, 95-102, 137) - so its train.py silently trains with one group.  Here `groups` is
accepted as an alias of `l2norm_groups`, i.e. the setting takes effect.
"""
import torch
import torch.nn.functional as F
from torch import nn

from .flash_cosine_sim_attention import (flash_cosine_sim_attention, flash_cosine_sim_attention_varlen,
                                         flash_cosine_sim_attention_with_kv_cache, plain_cosine_sim_attention)


def _softmax_attention(q, k, v, **unused):
    """Ordinary scaled dot-product causal attention (the `non_cosine_sim_attn` ablation, tf:31-38)."""
    d = q.shape[-1]
    sim = torch.matmul(q * d ** -0.5, k.transpose(-1, -2))
    i, j = sim.shape[-2:]
    future = torch.ones((i, j), dtype=torch.bool, device=q.device).triu(j - i + 1)
    sim = sim.masked_fill(future, -torch.finfo(sim.dtype).max)
    return torch.matmul(sim.softmax(dim=-1), v)


def _keep_top_fraction(logits, thres=0.9):
    """Keep the top (1 - thres) fraction of logits per row, -inf elsewhere (tf:42-47)."""
    k = int((1 - thres) * logits.shape[-1])
    val, ind = torch.topk(logits, k)
    out = torch.full_like(logits, float("-inf"))
    return out.scatter_(1, ind, val)


def FeedForward(dim, mult=4, pre_norm=False):
    hidden = int(dim * mult)
    return nn.Sequential(
        nn.LayerNorm(dim) if pre_norm else nn.Identity(),
        nn.Linear(dim, hidden, bias=False),
        nn.GELU(),
        nn.Linear(hidden, dim, bias=False),
    )


class KVCache:
    """Keys and values of one attention layer, for decoding token after token (`forward(x, cache=...)`).

    `k`, `v`: (batch, kv_heads, capacity, dim_head), allocated at the first call in the dtype of the keys.  With the
    CUDA kernel they hold what flash_cosine_sim_attention_with_kv_cache stores (l2-normalised keys); with the plain
    attention the raw keys.  `seqlens`: the valid rows per batch element on the device (int32), `length`: the same
    count on the host (the batch elements advance together here)."""

    def __init__(self, capacity):
        self.capacity = capacity
        self.k = self.v = self.seqlens = None
        self.length = 0


class Attention(nn.Module):
    def __init__(self, dim, dim_head=64, heads=8, scale=8, l2norm_groups=1, pre_norm=False,
                 use_cuda_kernel=False, non_cosine_sim_attn=False, groups=None, kv_heads=None, window=None, **kwargs):
        super().__init__()
        # window: sliding-window attention - each token attends to itself and the window - 1 tokens before it, on
        # every path (dense, packed documents, the key/value cache; the cache itself stays full-length)
        if window is not None and non_cosine_sim_attn:
            raise NotImplementedError("window is implemented for cosine-sim attention only (not non_cosine_sim_attn)")
        self.window = window
        # kv_heads: grouped-query attention - `kv_heads` key/value heads (dividing `heads`), each read by
        # heads // kv_heads consecutive query heads.  None = one per query head (the reference's layout).
        kv_heads = heads if kv_heads is None else kv_heads
        assert heads % kv_heads == 0, f"kv_heads ({kv_heads}) must divide heads ({heads})"
        inner = dim_head * heads
        self.norm = nn.LayerNorm(dim) if pre_norm else nn.Identity()
        self.scale = scale
        self.heads = heads
        self.kv_heads = kv_heads
        self.l2norm_groups = groups if groups is not None else l2norm_groups
        self.use_cuda_kernel = use_cuda_kernel and not non_cosine_sim_attn
        self.non_cosine_sim_attn = non_cosine_sim_attn
        self.kernel_kwargs = kwargs         # extra keywords of flash_cosine_sim_attention (CUDA kernel only)
        if non_cosine_sim_attn:
            g = heads // kv_heads
            self.attn_fn = (_softmax_attention if g == 1 else
                            lambda q, k, v, **kw: _softmax_attention(q, k.repeat_interleave(g, dim=1),
                                                                     v.repeat_interleave(g, dim=1)))
        elif use_cuda_kernel:
            self.attn_fn = (lambda q, k, v, **kw: flash_cosine_sim_attention(q, k, v, **{**kwargs, **kw}))
        else:
            self.attn_fn = plain_cosine_sim_attention
        self.to_q = nn.Linear(dim, inner, bias=False)
        self.to_k = nn.Linear(dim, dim_head * kv_heads, bias=False)
        self.to_v = nn.Linear(dim, dim_head * kv_heads, bias=False)
        self.to_out = nn.Linear(inner, dim, bias=False)

    def forward(self, x, cache=None, cu_seqlens=None, max_seqlen=None):
        """cu_seqlens: x is one packed row of documents, (1, total, dim), and cu_seqlens (documents + 1,) int32 their
        boundaries; every document attends causally to itself only.  max_seqlen: at least every document's length
        (default: total)."""
        if cu_seqlens is not None:
            if cache is not None:
                raise NotImplementedError("packed documents (cu_seqlens) with a key/value cache are not supported")
            return self._forward_packed(x, cu_seqlens, max_seqlen)
        b, n, _ = x.shape
        x = self.norm(x)
        # (b, n, h*d) -> (b, h, n, d) views: strided, feature dim contiguous - the fused op reads
        # them through TMA tensor maps without a copy
        split = lambda t, h: t.view(b, n, h, -1).transpose(1, 2)
        q = split(self.to_q(x), self.heads)
        k, v = split(self.to_k(x), self.kv_heads), split(self.to_v(x), self.kv_heads)
        if cache is None:
            o = self.attn_fn(q, k, v, causal=True, scale=self.scale, groups=self.l2norm_groups, window=self.window)
        else:
            o = self._attend_cached(q, k, v, cache)
        return self.to_out(o.transpose(1, 2).reshape(b, n, -1))

    def _forward_packed(self, x, cu_seqlens, max_seqlen):
        if x.ndim != 3 or x.shape[0] != 1:
            raise ValueError(f"packed documents take x of shape (1, total, dim), got {tuple(x.shape)}")
        n = x.shape[1]
        x = self.norm(x)
        # (1, total, h*d) -> (total, h, d) views of the projections, read by the varlen kernels without a copy
        q = self.to_q(x).view(n, self.heads, -1)
        k, v = self.to_k(x).view(n, self.kv_heads, -1), self.to_v(x).view(n, self.kv_heads, -1)
        if self.use_cuda_kernel:
            unsupported = sorted(set(self.kernel_kwargs) - {"l2norm_qk", "deterministic"})
            if unsupported:
                raise NotImplementedError(f"packed documents do not support the attention keywords {unsupported}")
            m = n if max_seqlen is None else int(max_seqlen)
            o = flash_cosine_sim_attention_varlen(q, k, v, cu_seqlens, cu_seqlens, m, m, scale=self.scale,
                                                  groups=self.l2norm_groups, causal=True,
                                                  l2norm_qk=self.kernel_kwargs.get("l2norm_qk", True), window=self.window,
                                                  deterministic=self.kernel_kwargs.get("deterministic", False))
        else:
            # the reference: one call per document (reads the boundaries on the host)
            bounds = cu_seqlens.tolist()
            # rows outside every document give 0, as with the kernel
            outs = [q.new_zeros(bounds[0], self.heads, q.shape[-1])] if bounds[0] > 0 else []
            for s, e in zip(bounds[:-1], bounds[1:]):
                if e > s:
                    per_doc = lambda t: t[s:e].transpose(0, 1).unsqueeze(0)
                    o_d = self.attn_fn(per_doc(q), per_doc(k), per_doc(v), causal=True, scale=self.scale,
                                       groups=self.l2norm_groups, window=self.window)
                    outs.append(o_d[0].transpose(0, 1))
            if bounds[-1] < n:
                outs.append(q.new_zeros(n - bounds[-1], self.heads, q.shape[-1]))
            o = torch.cat(outs) if outs else q.new_zeros(q.shape)
        return self.to_out(o.reshape(1, n, -1))

    def _attend_cached(self, q, k, v, cache):
        """q, k, v of the next n tokens against the cached prefix; appends k, v to the cache."""
        if self.non_cosine_sim_attn:
            raise NotImplementedError("the key/value cache is implemented for cosine-sim attention only")
        b, _, n, d = k.shape
        L = cache.length
        if L + n > cache.capacity:
            raise ValueError(f"key/value cache full: {L} + {n} tokens exceed its capacity {cache.capacity}")
        # the uncached CUDA path hands these keywords to flash_cosine_sim_attention; with a cache only l2norm_qk has a
        # meaning, and a silently dropped one would make cached and uncached outputs differ.  `deterministic` only
        # concerns the backward, and the cache is inference only: it changes no output here.
        unsupported = sorted(set(self.kernel_kwargs) - {"l2norm_qk", "deterministic"}) if self.use_cuda_kernel else []
        if unsupported:
            raise NotImplementedError(f"the key/value cache does not support the attention keywords {unsupported}")
        if self.use_cuda_kernel and k.dtype == torch.float32:
            raise RuntimeError("the key/value cache with the CUDA kernel needs 16-bit activations: run the model in "
                               "16-bit or under autocast")
        if cache.k is None:
            cache.k = torch.zeros(b, self.kv_heads, cache.capacity, d, dtype=k.dtype, device=k.device)
            cache.v = torch.zeros_like(cache.k)
            cache.seqlens = torch.zeros(b, dtype=torch.int32, device=k.device)
        if self.use_cuda_kernel:
            o = flash_cosine_sim_attention_with_kv_cache(q, cache.k, cache.v, cache.seqlens, k, v, scale=self.scale,
                                                         groups=self.l2norm_groups, causal=True,
                                                         l2norm_qk=self.kernel_kwargs.get("l2norm_qk", True),
                                                         window=self.window)
        else:
            cache.k[:, :, L:L + n] = k
            cache.v[:, :, L:L + n] = v
            o = plain_cosine_sim_attention(q, cache.k[:, :, :L + n], cache.v[:, :, :L + n], causal=True,
                                           scale=self.scale, groups=self.l2norm_groups, window=self.window)
        cache.seqlens += n
        cache.length += n
        return o


class CosineSimCausalTransformer(nn.Module):
    def __init__(self, *, num_tokens, dim, max_seq_len, depth, attn_scale=8, attn_l2norm_groups=1,
                 heads=8, dim_head=64, use_cuda_kernel=False, pre_norm=False, non_cosine_sim_attn=False,
                 kv_heads=None, window=None, **kwargs):
        super().__init__()
        self.max_seq_len = max_seq_len
        self.token_emb = nn.Embedding(num_tokens, dim)
        self.pos_emb = nn.Embedding(max_seq_len, dim)
        # post-norm residual scaling and init follow DeepNet (reference tf:123, 151-165)
        self.residual_scale = 1 if pre_norm else (2 * depth) ** 0.25
        norm = (lambda: nn.Identity()) if pre_norm else (lambda: nn.LayerNorm(dim))
        self.layers = nn.ModuleList([
            nn.ModuleList([
                Attention(dim, dim_head=dim_head, heads=heads, use_cuda_kernel=use_cuda_kernel,
                          scale=attn_scale, groups=attn_l2norm_groups, pre_norm=pre_norm,
                          non_cosine_sim_attn=non_cosine_sim_attn, kv_heads=kv_heads, window=window, **kwargs),
                norm(),
                FeedForward(dim, pre_norm=pre_norm),
                norm(),
            ]) for _ in range(depth)
        ])
        self.to_logits = nn.Sequential(
            nn.LayerNorm(dim) if pre_norm else nn.Identity(),
            nn.Linear(dim, num_tokens, bias=False),
        )
        if not pre_norm:
            self.init_(depth)

    def init_(self, depth):
        nn.init.normal_(self.token_emb.weight, std=1e-5)
        nn.init.normal_(self.pos_emb.weight, std=1e-5)
        gain = (8 * depth) ** -0.25
        for attn, _, ff, _ in self.layers:
            for lin, g in ((attn.to_q, 1.0), (attn.to_k, 1.0), (attn.to_v, gain), (attn.to_out, gain),
                           (ff[1], gain), (ff[3], gain)):
                nn.init.xavier_normal_(lin.weight.data, gain=g)
        nn.init.xavier_normal_(self.to_logits[-1].weight.data, gain=1.0)

    def new_cache(self):
        """One empty KVCache per layer, holding up to max_seq_len tokens, for forward(x, cache=...)."""
        return [KVCache(self.max_seq_len) for _ in self.layers]

    @torch.no_grad()
    def generate(self, start_tokens, seq_len, temperature=1.0, filter_thres=0.9, kv_cache=False, **kwargs):
        """kv_cache=True: one forward over the prompt, then one token per step against the cached keys / values.
        Once the sequence is longer than max_seq_len, the window slides and its positions are re-encoded from 0, so
        from then on each step re-fills a fresh cache with the window - the same computation as without the cache."""
        was_training = self.training
        self.eval()
        n0 = start_tokens.shape[1]
        out = start_tokens
        cache = None
        for _ in range(seq_len):
            if not kv_cache:
                logits = self.forward(out[:, -self.max_seq_len:], **kwargs)[:, -1, :]
            elif cache is None or out.shape[1] > self.max_seq_len:
                cache = self.new_cache()
                logits = self.forward(out[:, -self.max_seq_len:], cache=cache, **kwargs)[:, -1, :]
            else:
                logits = self.forward(out[:, -1:], cache=cache, **kwargs)[:, -1, :]
            probs = F.softmax(_keep_top_fraction(logits, filter_thres) / temperature, dim=-1)
            out = torch.cat((out, torch.multinomial(probs, 1)), dim=-1)
        self.train(was_training)
        return out[:, n0:]

    def forward(self, x, return_loss=False, cache=None, cu_seqlens=None, max_seqlen=None):
        """cache: the list new_cache() returned - x are then the next tokens after the cached ones, and their
        positions start at the cache's length.  cu_seqlens: x is one packed row of documents, (1, total), split at
        the int32 boundaries cu_seqlens (documents + 1,); positions restart at 0 in every document and no document
        sees another.  max_seqlen: at least every document's length (default: min(total, max_seq_len)); documents
        must not be longer than max_seq_len."""
        if cu_seqlens is not None:
            if cache is not None or return_loss:
                raise NotImplementedError("packed documents (cu_seqlens) with a key/value cache or return_loss are not "
                                          "supported")
            return self._forward_packed(x, cu_seqlens, max_seqlen)
        if return_loss:
            x, labels = x[:, :-1], x[:, 1:]
        start = 0 if cache is None else cache[0].length
        if start + x.shape[1] > self.max_seq_len:
            if cache is None:
                raise ValueError(f"{x.shape[1]} tokens exceed max_seq_len {self.max_seq_len}")
            raise ValueError(f"key/value cache full: {start} + {x.shape[1]} tokens exceed its capacity "
                             f"{self.max_seq_len} (max_seq_len)")
        x = self.token_emb(x) + self.pos_emb(torch.arange(start, start + x.shape[1], device=x.device))
        for i, (attn, attn_norm, ff, ff_norm) in enumerate(self.layers):
            x = attn_norm(attn(x, cache=None if cache is None else cache[i]) + x * self.residual_scale)
            x = ff_norm(ff(x) + x * self.residual_scale)
        logits = self.to_logits(x)
        if not return_loss:
            return logits
        return F.cross_entropy(logits.transpose(1, 2), labels)

    def _forward_packed(self, x, cu_seqlens, max_seqlen):
        if x.ndim != 2 or x.shape[0] != 1:
            raise ValueError(f"packed documents take x of shape (1, total), got {tuple(x.shape)}")
        n = x.shape[1]
        if max_seqlen is None:
            max_seqlen = min(n, self.max_seq_len)
        elif max_seqlen > self.max_seq_len:
            raise ValueError(f"max_seqlen {max_seqlen} exceeds max_seq_len {self.max_seq_len}")
        # positions restart at 0 in every document, computed on the device: row t belongs to the last document that
        # starts at or before it (clamped into the embedding table for out-of-contract boundaries)
        t = torch.arange(n, device=x.device, dtype=cu_seqlens.dtype)
        doc = (torch.searchsorted(cu_seqlens, t, right=True) - 1).clamp(0, cu_seqlens.shape[0] - 1)
        pos = (t - cu_seqlens[doc]).clamp(0, self.max_seq_len - 1)
        x = self.token_emb(x) + self.pos_emb(pos)[None]
        for attn, attn_norm, ff, ff_norm in self.layers:
            x = attn_norm(attn(x, cu_seqlens=cu_seqlens, max_seqlen=max_seqlen) + x * self.residual_scale)
            x = ff_norm(ff(x) + x * self.residual_scale)
        return self.to_logits(x)
