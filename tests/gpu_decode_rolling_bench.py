"""Rolling-cache decode benchmark: one decode step (1 new token per sequence, appended) on a rolling cache of the
window against the same step on a full-length cache, at the same window, on one GPU.

    python tests/gpu_decode_rolling_bench.py [--rounds 5] [--calls 20]

Workloads (bf16, causal, window W = 4096, seeded), (B, H, kv_heads, L, D) with L cached positions:
  (1, 16, 2, 65536, 128), (8, 32, 8, 32768, 128), (8, 16, 4, 32768, 64)
Variants:
  full      a cache of L + 1 rows, position p at row p (rolling=False)
  rolling   a ring of C = round_up(W - 1 + 128, 128) = 4224 rows, position p at row p mod C (rolling=True)
The ring is filled from the full-length cache, so both hold the same keys; before timing, the two outputs are compared
(bitwise when both use the same number of key splits, else within the relative tolerance of test_gpu_parity.py).
cache_seqlens is not advanced, so every call appends the same row and sees the same lengths.  Each call is timed with
CUDA events after an L2 flush, the variants alternate over the rounds, and the median and the p10-p90 range over all
calls are reported with the bytes of each variant's K and V caches.  The card's name and power limit are read in the
same run."""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from flash_cosine_sim_attention_b200 import flash_cosine_sim_attention_with_kv_cache as op  # noqa: E402
from flash_cosine_sim_attention_b200 import l2norm_tensors  # noqa: E402
from flash_cosine_sim_attention_b200.transformer import rolling_capacity  # noqa: E402

TOL = 1e-2        # bf16: TOL_OUT of test_gpu_parity.py
WINDOW = 4096
SHAPES = [(1, 16, 2, 65536, 128), (8, 32, 8, 32768, 128), (8, 16, 4, 32768, 64)]


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        return torch.cuda.get_device_name()


def setup(B, H, Hk, L, D):
    g = torch.Generator(device="cuda").manual_seed(1)
    dt = torch.bfloat16
    rnd = lambda *s: torch.randn(*s, device="cuda", generator=g).to(dt)
    C = rolling_capacity(WINDOW)
    kf, vf = l2norm_tensors(rnd(B, Hk, L + 1, D))[0], rnd(B, Hk, L + 1, D)
    p = torch.arange(L - C, L, device="cuda")
    kr = torch.zeros(B, Hk, C, D, dtype=dt, device="cuda")
    vr = torch.zeros_like(kr)
    kr[:, :, p % C] = kf[:, :, p]
    vr[:, :, p % C] = vf[:, :, p]
    q, k, v = rnd(B, H, 1, D), rnd(B, Hk, 1, D), rnd(B, Hk, 1, D)
    seqlens = torch.full((B,), L, dtype=torch.int32, device="cuda")
    fns = {"full": lambda: op(q, kf, vf, seqlens, k, v, window=WINDOW),
           "rolling": lambda: op(q, kr, vr, seqlens, k, v, window=WINDOW, rolling=True)}
    cache_bytes = {"full": 2 * kf.numel() * kf.element_size(), "rolling": 2 * kr.numel() * kr.element_size()}
    return fns, cache_bytes, C


def time_calls(fn, calls, flush):
    ts = []
    for _ in range(calls):
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
        raise SystemExit("gpu_decode_rolling_bench.py needs a CUDA device")
    print(json.dumps({"card": card()}), flush=True)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    for B, H, Hk, L, D in SHAPES:
        fns, cache_bytes, C = setup(B, H, Hk, L, D)
        with torch.no_grad():
            o_full, o_ring = fns["full"](), fns["rolling"]()
            torch.cuda.synchronize()
            bitwise = torch.equal(o_full.view(torch.int16), o_ring.view(torch.int16))
            err = float((o_ring.double() - o_full.double()).abs().max() / o_full.double().abs().max().clamp_min(1e-30))
            assert err <= TOL, f"{(B, H, Hk, L, D)}: rolling vs full relative error {err:.3e}"
            for fn in fns.values():
                for _ in range(3):
                    fn()
            torch.cuda.synchronize()
            samples = {v: [] for v in fns}
            for _ in range(args.rounds):
                for v, fn in fns.items():
                    samples[v] += time_calls(fn, args.calls, flush)
        meta = {"B": B, "H": H, "kv_heads": Hk, "L": L, "D": D, "window": WINDOW, "ring_rows": C}
        print(json.dumps({**meta, "bitwise_equal": bitwise, "rel_err": round(err, 6)}), flush=True)
        for v, ts in samples.items():
            print(json.dumps({**meta, "variant": v, "cache_bytes": cache_bytes[v], "us_median": round(pct(ts, 50), 2),
                              "us_p10": round(pct(ts, 10), 2), "us_p90": round(pct(ts, 90), 2)}), flush=True)
        del fns
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
