"""Packed decode benchmark: one flash_cosine_sim_attention_with_kv_cache call with cu_seqlens_q against what a caller
can do without it, on one GPU.

    python tests/gpu_decode_varlen_bench.py [--rounds 5] [--calls 20]

Workloads (bf16, seeded; each call appends its new tokens and attends them to the cache):
  speculative    B 16, H 32, kv_heads 8, D 128: L_b drawn in [2048, 8192], n_b drawn in [1, 8]
  chunked        B 8, H 16, kv_heads 2, D 128: one sequence with 1024 new tokens on a 4096 prefix, seven with 1 new
                 token on prefixes drawn in [4096, 16384]
Variants:
  packed         one call with cu_seqlens_q / max_seqlen_q
  per_sequence   one dense call per sequence (q[b:b+1], its cache row, its n_b tokens)
  padded         one dense call with every sequence padded to the largest n_b.  It computes something else (the
                 padding rows become visible keys), so it is only a cost bound.
Each call is timed with CUDA events after an L2 flush, the variants alternate over the rounds, and the median and the
p10-p90 range over all calls are reported.  The caches are restored from a copy before every call (outside the timed
window), so every call sees the same lengths.  Before timing, the packed and per-sequence outputs are compared within
the relative tolerance of test_gpu_parity.py.  The card's name and power limit are read in the same run."""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from flash_cosine_sim_attention_b200 import flash_cosine_sim_attention_with_kv_cache as op  # noqa: E402
from flash_cosine_sim_attention_b200 import l2norm_tensors  # noqa: E402

TOL = 1e-2        # bf16: TOL_OUT of test_gpu_parity.py


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        return torch.cuda.get_device_name()


def workloads():
    g = torch.Generator().manual_seed(0)
    spec_L = torch.randint(2048, 8193, (16,), generator=g).tolist()
    spec_n = torch.randint(1, 9, (16,), generator=g).tolist()
    chunk_L = [4096] + torch.randint(4096, 16385, (7,), generator=g).tolist()
    chunk_n = [1024] + [1] * 7
    return [("speculative", 32, 8, 128, spec_L, spec_n), ("chunked", 16, 2, 128, chunk_L, chunk_n)]


def setup(H, Hk, D, lens, ns):
    g = torch.Generator(device="cuda").manual_seed(1)
    dt = torch.bfloat16
    rnd = lambda *s: torch.randn(*s, device="cuda", generator=g).to(dt)
    B, cap, total, nmax = len(lens), max(L + n for L, n in zip(lens, ns)), sum(ns), max(ns)
    kc0 = l2norm_tensors(rnd(B, Hk, cap, D))[0]
    vc0 = rnd(B, Hk, cap, D)
    kc, vc = kc0.clone(), vc0.clone()
    q, k, v = rnd(total, H, D), rnd(total, Hk, D), rnd(total, Hk, D)
    cu_list = [0]
    for n in ns:
        cu_list.append(cu_list[-1] + n)
    cu = torch.tensor(cu_list, dtype=torch.int32, device="cuda")
    seqlens = torch.tensor(lens, dtype=torch.int32, device="cuda")
    seq_one = [seqlens[b:b + 1] for b in range(B)]
    dense = lambda x, b: x[cu_list[b]:cu_list[b + 1]].transpose(0, 1).unsqueeze(0)
    qs = [dense(q, b).contiguous() for b in range(B)]
    ks = [dense(k, b).contiguous() for b in range(B)]
    vs = [dense(v, b).contiguous() for b in range(B)]
    qp, kp, vp = rnd(B, H, nmax, D), rnd(B, Hk, nmax, D), rnd(B, Hk, nmax, D)

    def packed():
        return op(q, kc, vc, seqlens, k, v, cu_seqlens_q=cu, max_seqlen_q=nmax)

    def per_sequence():
        return [op(qs[b], kc[b:b + 1], vc[b:b + 1], seq_one[b], ks[b], vs[b]) for b in range(B)]

    def padded():
        return op(qp, kc, vc, seqlens, kp, vp)

    def reset():
        kc.copy_(kc0)
        vc.copy_(vc0)
    return {"packed": packed, "per_sequence": per_sequence, "padded": padded}, reset, cu_list


def time_calls(fn, reset, calls, flush):
    ts = []
    for _ in range(calls):
        reset()
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b) * 1e3)
    return ts


def pct(xs, p):
    xs = sorted(xs)
    return xs[min(len(xs) - 1, int(round(p / 100 * (len(xs) - 1))))]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gpu_decode_varlen_bench.py needs a CUDA device")
    print(json.dumps({"card": card()}), flush=True)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    for name, H, Hk, D, lens, ns in workloads():
        fns, reset, cu = setup(H, Hk, D, lens, ns)
        with torch.no_grad():
            # the packed call against one call per sequence, at the timed size
            reset()
            o = fns["packed"]().double()
            reset()
            per = fns["per_sequence"]()
            err = max(float((o[cu[b]:cu[b + 1]] - p[0].transpose(0, 1).double()).abs().max() /
                            p.double().abs().max().clamp_min(1e-30)) for b, p in enumerate(per))
            assert err <= TOL, f"{name}: packed vs per-sequence relative error {err:.3e}"
            for fn in fns.values():
                for _ in range(3):
                    reset()
                    fn()
            torch.cuda.synchronize()
            samples = {v: [] for v in fns}
            for _ in range(args.rounds):
                for v, fn in fns.items():
                    samples[v] += time_calls(fn, reset, args.calls, flush)
        meta = {"workload": name, "B": len(lens), "H": H, "kv_heads": Hk, "D": D, "n_b": ns, "L_b": lens}
        print(json.dumps({**meta, "packed_vs_per_sequence_rel_err": round(err, 6)}), flush=True)
        for v, ts in samples.items():
            print(json.dumps({"workload": name, "variant": v, "us_median": round(pct(ts, 50), 2),
                              "us_p10": round(pct(ts, 10), 2), "us_p90": round(pct(ts, 90), 2)}), flush=True)
        med = {v: pct(ts, 50) for v, ts in samples.items()}
        print(json.dumps({"workload": name, "per_sequence_over_packed": round(med["per_sequence"] / med["packed"], 2),
                          "padded_over_packed": round(med["padded"] / med["packed"], 2)}), flush=True)
        del fns
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
