"""float64 reference and element-wise bound of sliding-window attention.  Test infrastructure only.

`window_attention_bounds` is `elementwise_bounds.attention_bounds` (same model of the kernels' roundings, same
|got - ref| <= C u M contract, same return value) with the band of a sliding window W added to the visibility:
with off = Nk - Nq and d = i + off - j, key j is visible to query i iff 0 <= d < W (causal) or |d| < W (not causal),
on top of the key mask.  A window takes no attn_bias, so there is none here.  Grouped-query, single-head and merged
keys/values, key masks, l2norm groups, l2norm_qk=False and round_qk are supported as there."""
import math

import torch

from elementwise_bounds import ETA, U, _f64, _l2norm, _l2norm_backward, _l2norm_bound, round_to


def window_attention_bounds(q, k, v, d_out=None, mask=None, window=None, scale=8, groups=1, causal=False,
                            l2norm_qk=True, round_qk=None, fmt="bf16", shift=None, device=None, chunk=1024,
                            ds_scale=1.0):
    """(ref, bound) dicts over o (and dq, dk, dv with d_out) of float64 tensors on `device`, shaped like the inputs.
    window=None is no window.  ds_scale: as in attention_bounds."""
    device = device or (q.device if torch.is_tensor(q) else "cpu")
    q, k, v, do = (_f64(t, device) for t in (q, k, v, d_out))
    mask = None if mask is None else torch.as_tensor(mask).to(device=device, dtype=torch.bool)
    assert not (causal and mask is not None)
    u, eta = U[fmt], ETA[fmt]
    merged, single = q.ndim == 3, k.ndim == 3
    if merged:
        q, k, v = q[:, None], k[:, None], v[:, None]
        do = None if do is None else do[:, None]
    elif single:
        k, v = k[:, None], v[:, None]
    B, H, Nq, D = q.shape
    Hk, Nk = k.shape[1], k.shape[2]
    G = H // Hk
    off = Nk - Nq
    if l2norm_qk:
        qn, nq = _l2norm(q, groups)
        kn, nk = _l2norm(k, groups)
        qn, kn = round_to(qn, round_qk), round_to(kn, round_qk)
    else:
        qn, kn = q, k
    grads = do is not None
    z = lambda t: torch.zeros_like(t)
    o, Mo = z(q), z(q)
    if grads:
        dqn, Mdq, dkn, Mdk, dv, Mdv = z(q), z(q), z(k), z(k), z(v), z(v)
    cols = torch.arange(Nk, device=device)
    # (the loop order of attention_bounds, so that without a band both sum dk, dv in the same order)
    for b in range(B):
        for h in range(H):
            hk = h // G
            for r0 in range(0, Nq, chunk):
                r1 = min(Nq, r0 + chunk)
                # keys [k0, ke) hold every key the chunk's rows can see; the others contribute exactly 0 (as in
                # attention_bounds, and the same range when the band hides nothing)
                ke = Nk
                if causal or window is not None:
                    ke = min(Nk, max(1, r1 + off + (0 if causal else window - 1)))
                k0 = 0 if window is None else min(ke - 1, max(0, r0 + off - window + 1))
                kb, vb = kn[b, hk, k0:ke], v[b, hk, k0:ke]
                d = torch.arange(r0, r1, device=device)[:, None] + off - cols[None, k0:ke]
                vis = torch.ones_like(d, dtype=torch.bool)
                if causal:
                    vis &= d >= 0
                if window is not None:
                    vis &= (d < window) if causal else (d.abs() < window)
                if mask is not None:
                    vis &= mask[b][None, k0:ke]
                anyv = vis.any(-1)
                visf = vis.double()
                s = (scale * (qn[b, h, r0:r1] @ kb.T)).masked_fill(~vis, -math.inf)
                m = torch.where(anyv, s.amax(-1), torch.zeros_like(s[:, 0]))
                e = torch.exp(s - m[:, None])
                l = e.sum(-1)
                P = e / l.clamp_min(1e-300)[:, None]
                ob = P @ vb
                o[b, h, r0:r1] = ob
                # the kernels round the UNNORMALISED p = exp(logit - shift): eta / l_kernel after normalising
                sh = m if shift is None else torch.full_like(m, float(shift))
                inv_lk = torch.where(anyv, torch.exp(sh - m) / l.clamp_min(1e-300), torch.zeros_like(m))
                Mo[b, h, r0:r1] = P @ vb.abs() + ob.abs() + (eta / u) * inv_lk[:, None] * (visf @ vb.abs())
                if not grads:
                    continue
                dob = do[b, h, r0:r1]
                dv[b, hk, k0:ke] += P.T @ dob
                Mdv[b, hk, k0:ke] += P.T @ dob.abs() + (eta / u) * (visf.T @ dob.abs())
                ds = P * (dob @ vb.T - (dob * ob).sum(-1, keepdim=True))
                A = ds.abs() + P * (dob.abs() * ob.abs()).sum(-1, keepdim=True) + (eta / u) * ds_scale * visf
                dqn[b, h, r0:r1] = scale * (ds @ kb)
                Mdq[b, h, r0:r1] = scale * (A @ kb.abs())
                qb = qn[b, h, r0:r1]
                dkn[b, hk, k0:ke] += scale * (ds.T @ qb)
                Mdk[b, hk, k0:ke] += scale * (A.T @ qb.abs())
    ref, bound = {"o": o}, {"o": Mo}
    if grads:
        Mdq += dqn.abs()
        Mdk += dkn.abs()
        Mdv += dv.abs()
        if l2norm_qk:
            dq, dk = _l2norm_backward(dqn, q, groups), _l2norm_backward(dkn, k, groups)
            Mdq = _l2norm_bound(Mdq, qn, nq, groups) + dq.abs()
            Mdk = _l2norm_bound(Mdk, kn, nk, groups) + dk.abs()
        else:
            dq, dk = dqn, dkn
        ref.update(dq=dq, dk=dk, dv=dv)
        bound.update(dq=Mdq, dk=Mdk, dv=Mdv)
    for name in bound:
        # the store of each output to T: eta where the result is not structurally zero
        bound[name] = bound[name] + (eta / u) * (bound[name] > 0)
    for name in ("o", "dq"):
        if name in ref and merged:
            ref[name], bound[name] = ref[name][:, 0], bound[name][:, 0]
    for name in ("dk", "dv"):
        if name in ref and (merged or single):
            ref[name], bound[name] = ref[name][:, 0], bound[name][:, 0]
    return ref, bound
