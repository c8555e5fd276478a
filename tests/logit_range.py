"""Seeded inputs at the ends of the logit range.  Test infrastructure only.

Every kernel computes p = exp(scale * q^.k^ - shift) with a constant shift (`_choose_shift`, no row max), chosen
from where q^.k^ can go: up to +groups (bf16: p <= 1 there; fp16: p <= 2^15) and down to -groups (fp16: p still a
normal number).  Isotropic Gaussian q and k never get near either end - at D = 64 the cosine of two independent
rows is about N(0, 1/64) - so the top of the exponential's range, and the backward's cancellation in
dS = P (dP - delta) when one key takes the whole row (o ~ v_j), go untested with them.  These families control q^.k^
(k is Gaussian unless said otherwise; pi(i) is a key visible to query row i):

  aligned<s>  q_i = k_pi(i) + s * noise, s in {0, 0.05, 0.3}, pi(i) drawn from a pool of Nk / 8 keys, so several rows
              share a key (its dk gathers them all).  q^.k^ -> groups in every l2norm group; s = 0 gives exact
              duplicates after rounding.
  diagonal    q_i = k_(i + Nk - Nq) + 0.05 noise: every token attends to itself (the causal diagonal).
  one_peak    q_i = k_pi(i) exactly, pi injective where the visible keys allow: one aligned key per row among random
              ones, P ~ 1 on it when scale * groups is large.
  dup_run     keys [40, 140) identical (the run crosses the 64-key warpgroup half and the 128-key tile), their values
              distinct; the even rows are aligned to that key (0.05 noise), the odd ones are Gaussian.
  opposed     keys spread around one direction c (k_j = c + 0.3 noise) and q_i = -k_pi(i) + 0.05 noise: every p of a
              row sits near the bottom of its range.
  zero_rows   aligned0.3 with one all-zero query row and one all-zero key row (the l2norm's 1e-12 clamp: the zero row
              normalises to zero, its gradient is multiplied by 1e12 - beyond fp16's range).

`qk` builds one batch element (or one packed sequence, or one cache); `dense`, `packed` and `cache` lay them out as
the three entry points take them.  v and dO are Gaussian."""
import torch

FAMILIES = ("aligned0", "aligned0.05", "aligned0.3", "diagonal", "one_peak", "dup_run", "opposed", "zero_rows")
DUP_RUN = (40, 140)


def _visible_hi(Nq, Nk, causal):
    """Last key visible to each query row (bottom-right causal rule), -1 when the row sees none."""
    hi = torch.full((Nq,), Nk - 1, dtype=torch.long)
    if causal:
        hi = torch.clamp(torch.arange(Nq) + (Nk - Nq), max=Nk - 1)
    return hi.clamp(min=-1)


def _uniform_visible(hi, g):
    return torch.where(hi >= 0, (torch.rand(hi.shape, generator=g) * (hi + 1)).long().clamp(max=hi.clamp(min=0)), -1)


def qk(family, H, Hk, Nq, Nk, D, causal, g):
    """q (H, Nq, D) and k (Hk, Nk, D), float32, of one problem; query head h reads key head h // (H // Hk).  Also
    returns peak (H, Nq): the key each query row was built from, -1 for rows built from none."""
    assert family in FAMILIES, family
    G = H // Hk
    hi = _visible_hi(Nq, Nk, causal)
    k = torch.randn(Hk, Nk, D, generator=g)
    if family == "opposed":
        k = torch.randn(Hk, 1, D, generator=g) + 0.3 * k
    q = torch.randn(H, Nq, D, generator=g)
    peak = torch.full((H, Nq), -1, dtype=torch.long)
    sigma = {"aligned0": 0.0, "aligned0.05": 0.05, "aligned0.3": 0.3, "zero_rows": 0.3}.get(family, 0.05)
    if family == "dup_run":
        r0, r1 = min(DUP_RUN[0], Nk - 1), min(DUP_RUN[1], Nk)
        k[:, r0:r1] = k[:, r0:r0 + 1]
    for h in range(H):
        if family in ("aligned0", "aligned0.05", "aligned0.3", "zero_rows"):
            pool = torch.randperm(Nk, generator=g)[:max(1, Nk // 8)].sort().values
            n_ok = (pool[None, :] <= hi[:, None]).sum(1)              # pool is sorted: its first n_ok keys are visible
            pick = (torch.rand(Nq, generator=g) * n_ok).long().clamp(max=(n_ok - 1).clamp(min=0))
            pi = torch.where(n_ok > 0, pool[pick], _uniform_visible(hi, g))
        elif family == "diagonal":
            pi = torch.where(hi >= 0, torch.clamp(torch.arange(Nq) + (Nk - Nq), 0, Nk - 1), -1)
        elif family == "one_peak":
            pi = torch.randperm(Nk, generator=g)[:Nq] if (not causal and Nq <= Nk) else _uniform_visible(hi, g)
        elif family == "dup_run":
            run = torch.full((Nq,), min(DUP_RUN[0], Nk - 1), dtype=torch.long)
            pi = torch.where((torch.arange(Nq) % 2 == 0) & (hi >= run), run, -1)
        else:                                                          # opposed
            pi = _uniform_visible(hi, g)
        noise = torch.randn(Nq, D, generator=g)
        rows = pi >= 0
        src = k[h // G, pi.clamp(min=0)]
        built = (-src if family == "opposed" else src) + sigma * noise
        q[h] = torch.where(rows[:, None], built, q[h])
        peak[h] = pi
    if family == "zero_rows":
        q[:, Nq // 2] = 0
        k[:, Nk // 3] = 0
    return q, k, peak


def dense(family, B, H, Hk, Nq, Nk, D, dtype, causal=False, seed=0):
    """(B, H, Nq, D) q and dO, (B, Hk, Nk, D) k and v in `dtype`, and peak (B, H, Nq)."""
    g = torch.Generator().manual_seed(seed)
    parts = [qk(family, H, Hk, Nq, Nk, D, causal, g) for _ in range(B)]
    q = torch.stack([p[0] for p in parts])
    k = torch.stack([p[1] for p in parts])
    peak = torch.stack([p[2] for p in parts])
    v = torch.randn(B, Hk, Nk, D, generator=g)
    do = torch.randn(B, H, Nq, D, generator=g)
    return q.to(dtype), k.to(dtype), v.to(dtype), do.to(dtype), peak


def packed(family, lq, lk, H, Hk, D, dtype, causal=False, seed=0):
    """Packed (total_q, H, D) q and dO, (total_k, Hk, D) k and v: sequence b is built by `qk` on its own."""
    g = torch.Generator().manual_seed(seed)
    qs, ks = [], []
    for a, b in zip(lq, lk):
        if a and b:
            q, k, _ = qk(family, H, Hk, a, b, D, causal, g)
        else:
            q, k = torch.randn(H, a, D, generator=g), torch.randn(Hk, b, D, generator=g)
        qs.append(q.transpose(0, 1))
        ks.append(k.transpose(0, 1))
    q, k = torch.cat(qs), torch.cat(ks)
    v = torch.randn(k.shape, generator=g)
    do = torch.randn(q.shape, generator=g)
    return q.to(dtype), k.to(dtype), v.to(dtype), do.to(dtype)


def cache(family, lens, cap, n_new, H, Hk, Nq, D, dtype, causal=True, seed=0):
    """Decoding: batch element b has T_b = lens[b] + n_new keys, the first lens[b] in the cache and the last n_new
    passed as new keys, built by `qk` with the Nq new queries (query i sees key j iff j <= i + T_b - Nq when causal).
    Returns q (B, H, Nq, D), the raw cache contents k_cache, v_cache (B, Hk, cap, D; rows from lens[b] on are
    Gaussian filler) and k, v (B, Hk, n_new, D)."""
    g = torch.Generator().manual_seed(seed)
    B = len(lens)
    q = torch.empty(B, H, Nq, D)
    kc = torch.randn(B, Hk, cap, D, generator=g)
    vc = torch.randn(B, Hk, cap, D, generator=g)
    kn = torch.randn(B, Hk, n_new, D, generator=g)
    vn = torch.randn(B, Hk, n_new, D, generator=g)
    for b, L in enumerate(lens):
        qb, kb, _ = qk(family, H, Hk, Nq, L + n_new, D, causal, g)
        q[b] = qb
        kc[b, :, :L] = kb[:, :L]
        kn[b] = kb[:, L:]
    return tuple(t.to(dtype) for t in (q, kc, vc, kn, vn))
