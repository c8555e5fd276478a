"""float64 reference for grouped-query attention, built on the oracle: k, v with kv_heads heads dividing q's heads
mean exactly the attention with k, v repeated to the query heads in the `repeat_interleave` layout (query head h
reads kv head h // (heads // kv_heads)), whose gradients w.r.t. the repeated copies summed over each group are the
gradients w.r.t. k, v.  Test infrastructure only."""
import numpy as np

from oracle import cosine_sim_attention_oracle as oracle


def group_sum(x, kv_heads):
    """(B, H, N, D) gradients of repeated keys/values -> (B, kv_heads, N, D): the sum over each group."""
    B, H = x.shape[:2]
    return x.reshape(B, kv_heads, H // kv_heads, *x.shape[2:]).sum(2)


def gqa_attention(q, k, v, d_out=None, **kw):
    """oracle.attention with 4-D k, v of kv_heads heads dividing q's heads; returns what oracle.attention returns,
    with dk, dv of k's and v's shapes."""
    q, k, v = (np.asarray(t, dtype=np.float64) for t in (q, k, v))
    H, Hk = q.shape[1], k.shape[1]
    assert q.ndim == 4 and k.ndim == 4 and v.shape == k.shape and H % Hk == 0
    G = H // Hk
    r = oracle.attention(q, np.repeat(k, G, axis=1), np.repeat(v, G, axis=1), d_out=d_out, **kw)
    if d_out is None:
        return r
    r = list(r)
    r[2], r[3] = group_sum(r[2], Hk), group_sum(r[3], Hk)
    return tuple(r)
