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

from .flash_cosine_sim_attention import flash_cosine_sim_attention, plain_cosine_sim_attention


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


class Attention(nn.Module):
    def __init__(self, dim, dim_head=64, heads=8, scale=8, l2norm_groups=1, pre_norm=False,
                 use_cuda_kernel=False, non_cosine_sim_attn=False, groups=None, kv_heads=None, **kwargs):
        super().__init__()
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

    def forward(self, x):
        b, n, _ = x.shape
        x = self.norm(x)
        # (b, n, h*d) -> (b, h, n, d) views: strided, feature dim contiguous - the fused op reads
        # them through TMA tensor maps without a copy
        split = lambda t, h: t.view(b, n, h, -1).transpose(1, 2)
        q = split(self.to_q(x), self.heads)
        k, v = split(self.to_k(x), self.kv_heads), split(self.to_v(x), self.kv_heads)
        o = self.attn_fn(q, k, v, causal=True, scale=self.scale, groups=self.l2norm_groups)
        return self.to_out(o.transpose(1, 2).reshape(b, n, -1))


class CosineSimCausalTransformer(nn.Module):
    def __init__(self, *, num_tokens, dim, max_seq_len, depth, attn_scale=8, attn_l2norm_groups=1,
                 heads=8, dim_head=64, use_cuda_kernel=False, pre_norm=False, non_cosine_sim_attn=False,
                 kv_heads=None, **kwargs):
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
                          non_cosine_sim_attn=non_cosine_sim_attn, kv_heads=kv_heads, **kwargs),
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

    @torch.no_grad()
    def generate(self, start_tokens, seq_len, temperature=1.0, filter_thres=0.9, **kwargs):
        was_training = self.training
        self.eval()
        n0 = start_tokens.shape[1]
        out = start_tokens
        for _ in range(seq_len):
            logits = self.forward(out[:, -self.max_seq_len:], **kwargs)[:, -1, :]
            probs = F.softmax(_keep_top_fraction(logits, filter_thres) / temperature, dim=-1)
            out = torch.cat((out, torch.multinomial(probs, 1)), dim=-1)
        self.train(was_training)
        return out[:, n0:]

    def forward(self, x, return_loss=False):
        if return_loss:
            x, labels = x[:, :-1], x[:, 1:]
        x = self.token_emb(x) + self.pos_emb(torch.arange(x.shape[1], device=x.device))
        for attn, attn_norm, ff, ff_norm in self.layers:
            x = attn_norm(attn(x) + x * self.residual_scale)
            x = ff_norm(ff(x) + x * self.residual_scale)
        logits = self.to_logits(x)
        if not return_loss:
            return logits
        return F.cross_entropy(logits.transpose(1, 2), labels)
