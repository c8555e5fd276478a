"""Element-wise error bounds for the fused kernels, from a float64 reference of the same problem.  Test
infrastructure only.

A relative-to-max metric (`max|got - ref| / max|ref|`) hardly sees the small end of a causal problem: the last
query rows of o and dq and the last keys of dk and dv are tens of times smaller than the first, and they are
exactly the tiles where the kernels branch (the last CTAs, the pipeline drain, one or two query tiles per CTA).
Here every element gets its own bound, from a model of the roundings the kernels do:

    |got - ref| <= C * u * M          everywhere, one constant C for every dtype, quantity and test

u is the unit roundoff of the operand type T (2^-8 bf16, 2^-11 f16).  Each rounding of a value x to T is modelled
as an error of u|x| + eta, eta = half the smallest subnormal of T (2^-25 for f16); every output carries
one more eta for its own store.  The kernels round:
  forward   p = exp(logit - shift) to T before P V (the row sum l stays fp32), o to T;
  backward  P to T before dV = P^T dO, dS = P (dP - delta) to T before dK = dS^T Q and dQ = dS K, delta from the
            STORED o, every output to T.
So, with P the normalised probabilities, A = |dS| + P * (sum_d |dO||O|) and all products taken with |.|:
  M_o      = P|V| + |O|                  (+ eta/u * sum_j |v_j| / l_kernel: the unnormalised p rounded)
  M_dv     = P^T|dO| + |dV|              (+ eta/u * per visible pair)
  M_dq^    = scale * A |K^| + |dq^|      M_dk^ = scale * A^T |Q^| + |dk^|      M_dbias = A summed like d_bias
  (A carries + eta/u per visible pair for the rounding of dS)
and when q, k are normalised inside the op, the l2norm backward carries the bound of dx^ to the raw input:
  M_dx     = (M_dx^ + |x^| <|x^|, M_dx^>_group) / ||x||_group + |dx|.

`attention_bounds` returns the float64 reference (equal to `oracle.attention` with empty_rows="zero") and M for
o, dq, dk, dv and d_bias.  It is torch float64 on any device, chunked over query rows, so (4, 8, 4096, 64) and
(1, 2, 16384, 128) problems fit on one GPU.  Grouped-query keys/values (kv head h // G, dk and dv summed over the
group), single-head keys/values, merged batch-heads, key masks, bottom-right causal masks, per-head and
per-batch bias, l2norm groups, l2norm_qk=False and round_qk are supported."""
import math

import numpy as np
import torch

U = {"bf16": 2.0 ** -8, "f16": 2.0 ** -11}
ETA = {"bf16": 2.0 ** -134, "f16": 2.0 ** -25}
# The one constant of |got - ref| <= C u M.  Chosen from the CPU emulation of the kernels' rounding points
# (tests/test_elementwise_bounds.py): its worst ratio err / (u M) over the pinned shapes is 0.98 (bf16 o: p and o
# each rounded by up to half an ulp, the model's own worst case), so C = 2 leaves a factor of 2 for what the
# emulation does not reproduce (fp32 summation order, ex2.approx) and still rejects a 3 % error in one tile.
C = 2.0
FMT = {torch.bfloat16: "bf16", torch.float16: "f16"}
QUANTITIES = ("o", "dq", "dk", "dv", "d_bias")


def round_to(x, fmt):
    """float64 tensor rounded to bf16 / f16 through float32 (as the oracle and the fp32 kernels do)."""
    if fmt is None or x is None:
        return x
    return x.float().to(torch.bfloat16 if fmt == "bf16" else torch.float16).double()


def _l2norm(x, groups):
    g = x.reshape(*x.shape[:-1], groups, x.shape[-1] // groups)
    n = g.norm(dim=-1, keepdim=True)
    return (g / n.clamp_min(1e-12)).reshape(x.shape), n.clamp_min(1e-12)


def _l2norm_backward(dy, x, groups):
    g = x.reshape(*x.shape[:-1], groups, x.shape[-1] // groups)
    n = g.norm(dim=-1, keepdim=True).clamp_min(1e-12)
    y = g / n
    d = dy.reshape(g.shape)
    return ((d - y * (y * d).sum(-1, keepdim=True)) / n).reshape(x.shape)


def _l2norm_bound(m, xhat, norm, groups):
    """Bound of the l2norm backward's output from the bound m of its input dx^ (same rounded x^ the kernels use)."""
    a = xhat.abs().reshape(*xhat.shape[:-1], groups, xhat.shape[-1] // groups)
    mg = m.reshape(a.shape)
    return ((mg + a * (a * mg).sum(-1, keepdim=True)) / norm).reshape(m.shape)


def kernel_shift(fmt, scale, groups=1, l2norm_qk=True, attn_bias=None):
    """The constant the kernels subtract from the logits (`_choose_shift`, plus the bias maximum for fp16)."""
    from flash_cosine_sim_attention_b200.flash_cosine_sim_attention import _choose_shift
    dt = torch.bfloat16 if fmt == "bf16" else torch.float16
    s = _choose_shift(dt, scale, groups if l2norm_qk else 1, l2norm_qk)
    if attn_bias is not None and fmt == "f16" and l2norm_qk:
        s += float(torch.as_tensor(attn_bias).float().max())
    return float(s)


def _f64(t, device):
    if t is None:
        return None
    if isinstance(t, np.ndarray):
        t = torch.from_numpy(t)
    return t.detach().to(device=device, dtype=torch.float64)


def attention_bounds(q, k, v, d_out=None, mask=None, attn_bias=None, scale=8, groups=1, causal=False,
                     l2norm_qk=True, attn_bias_batch_dim=False, round_qk=None, fmt="bf16", shift=None,
                     device=None, chunk=1024, eta=None, ds_scale=1.0):
    """float64 reference and per-element bound M of cosine-sim attention (module docstring).

    fmt: the kernels' operand type ("bf16" | "f16"), which sets u and eta.  round_qk: the type q^, k^ are stored in
    before the attention (as `oracle.attention`).  shift: the kernels' logit shift (`kernel_shift`); it only enters
    the eta term of o, and None takes each row's maximum.  eta: overrides the format's eta (0 gives the bound without
    the subnormal terms, to measure their share).  ds_scale: how many times smaller the kernels' dS is than the
    caller's (the float32 path runs them on v / sv and dO / pg, so on dS / (sv pg)); the eta of dS's rounding counts
    that many times over in the caller's units.  Returns (ref, bound): dicts over QUANTITIES (o only without d_out,
    d_bias only with a bias) of float64 tensors on `device` shaped like the inputs."""
    device = device or (q.device if torch.is_tensor(q) else "cpu")
    q, k, v, do, bias = (_f64(t, device) for t in (q, k, v, d_out, attn_bias))
    mask = None if mask is None else torch.as_tensor(mask).to(device=device, dtype=torch.bool)
    assert not (causal and mask is not None)
    u, eta = U[fmt], (ETA[fmt] if eta is None else eta)
    merged, single = q.ndim == 3, k.ndim == 3
    if merged:
        q, k, v = q[:, None], k[:, None], v[:, None]
        do = None if do is None else do[:, None]
        attn_bias_batch_dim = True
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
        dbias = None if bias is None else z(bias)
        Mdb = None if bias is None else z(bias)
    cols = torch.arange(Nk, device=device)
    for b in range(B):
        for h in range(H):
            hk = h // G
            for r0 in range(0, Nq, chunk):
                r1 = min(Nq, r0 + chunk)
                # causal: the keys past the chunk's last visible one contribute exactly 0, so they are left out
                ke = min(Nk, max(1, r1 + off)) if causal else Nk
                kb, vb = kn[b, hk, :ke], v[b, hk, :ke]
                rows = torch.arange(r0, r1, device=device)
                vis = torch.ones(r1 - r0, ke, dtype=torch.bool, device=device)
                if causal:
                    vis &= cols[None, :ke] <= rows[:, None] + off
                if mask is not None:
                    vis &= mask[b][None, :ke]
                s = scale * (qn[b, h, r0:r1] @ kb.T)
                if bias is not None:
                    s = s + bias[b if attn_bias_batch_dim else h, r0:r1, :ke]
                s = s.masked_fill(~vis, -math.inf)
                anyv = vis.any(-1)
                m = torch.where(anyv, s.amax(-1), torch.zeros_like(s[:, 0]))
                e = torch.exp(s - m[:, None])
                l = e.sum(-1)
                P = e / l.clamp_min(1e-300)[:, None]
                visf = vis.double()
                ob = P @ vb
                o[b, h, r0:r1] = ob
                mo = P @ vb.abs() + ob.abs()
                # the kernels round the UNNORMALISED p = exp(logit - shift): eta / l_kernel after normalising
                sh = m if shift is None else torch.full_like(m, float(shift))
                inv_lk = torch.where(anyv, torch.exp(sh - m) / l.clamp_min(1e-300), torch.zeros_like(m))
                mo += (eta / u) * inv_lk[:, None] * (visf @ vb.abs())
                Mo[b, h, r0:r1] = mo
                if not grads:
                    continue
                dob = do[b, h, r0:r1]
                dv[b, hk, :ke] += P.T @ dob
                Mdv[b, hk, :ke] += P.T @ dob.abs() + (eta / u) * (visf.T @ dob.abs())
                dp = dob @ vb.T
                delta = (dob * ob).sum(-1, keepdim=True)
                ds = P * (dp - delta)
                A = ds.abs() + P * (dob.abs() * ob.abs()).sum(-1, keepdim=True) + (eta / u) * ds_scale * visf
                dqn[b, h, r0:r1] = scale * (ds @ kb)
                Mdq[b, h, r0:r1] = scale * (A @ kb.abs())
                qb = qn[b, h, r0:r1]
                dkn[b, hk, :ke] += scale * (ds.T @ qb)
                Mdk[b, hk, :ke] += scale * (A.T @ qb.abs())
                if bias is not None:
                    i = b if attn_bias_batch_dim else h
                    dbias[i, r0:r1, :ke] += ds
                    Mdb[i, r0:r1, :ke] += A
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
        if bias is not None:
            ref["d_bias"], bound["d_bias"] = dbias, Mdb
    for name in bound:
        # the store of each output to T: eta where the result is not structurally zero (masked keys stay exact)
        bound[name] = bound[name] + (eta / u) * (bound[name] > 0)
    for name in ("o", "dq"):
        if name in ref and merged:
            ref[name], bound[name] = ref[name][:, 0], bound[name][:, 0]
    for name in ("dk", "dv"):
        if name in ref and (merged or single):
            ref[name], bound[name] = ref[name][:, 0], bound[name][:, 0]
    return ref, bound


def _where(name, idx, shape):
    """(b, h, row or key, feature) of an element and the tiles it belongs to."""
    if name == "d_bias":
        i, r, c = idx
        return f"bias plane {i}, query row {r} (query tile {r // 64} of 64), key {c} (key tile {c // 128} of 128)"
    lead = idx[:-2]
    r, f = idx[-2], idx[-1]
    head = ", ".join(str(x) for x in lead)
    if name in ("o", "dq"):
        return (f"(b, h) ({head}), query row {r}, feature {f} (forward query tile {r // 128} of 128, "
                f"backward query tile {r // 64} of 64)")
    return f"(b, kv head) ({head}), key {r}, feature {f} (key tile {r // 128} of 128, half {(r % 128) // 64})"


def ratio(got, ref, bound, fmt):
    """err / (u M) per element (inf where the bound is 0 and the error is not)."""
    got = got.detach().to(device=ref.device, dtype=torch.float64).reshape(ref.shape)
    err = (got - ref).abs()
    ub = U[fmt] * bound
    r = torch.where(err == 0, torch.zeros_like(err), err / ub)
    return torch.where(torch.isfinite(got), r, torch.full_like(r, math.inf))


def check_bound(name, got, ref, bound, fmt, c=C):
    """Assert |got - ref| <= c u M everywhere; returns the worst err / (c u M).  The message names the worst
    element and its tiles."""
    r = ratio(got, ref[name], bound[name], fmt) / c
    worst = float(r.max()) if r.numel() else 0.0
    if not worst <= 1.0:
        idx = np.unravel_index(int(torch.argmax(torch.nan_to_num(r, posinf=1e300))), tuple(r.shape))
        idx = tuple(int(i) for i in idx)
        g = got.detach().reshape(r.shape)[idx].item()
        raise AssertionError(
            f"{name}: |got - ref| = {c * worst:.3g} u M exceeds the element-wise bound {c:g} u M ({fmt}) at "
            f"{_where(name, idx, r.shape)}: got {g:.6g}, ref {ref[name][idx].item():.6g}, "
            f"M {bound[name][idx].item():.4g}")
    return worst
