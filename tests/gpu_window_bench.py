"""Time of sliding-window attention against the full causal op on the same tensors.
    python tests/gpu_window_bench.py [--steps K] [--rounds R] [--json PATH]
Training (bf16, causal): one forward and one backward through flash_cosine_sim_attention per step, for window = None,
1024 and 4096, alternated round by round within one process, each step timed with CUDA events after a flush of L2.
TFLOP/s count the visible (query, key) pairs only: 3.5 x 4 D per pair and head (forward 4 D, backward 2.5 x), so the
windowed and the full op are compared at the work each really has to do.
Decode: one new token against a (1, 16 heads, 2 kv heads, 65536, 128) cache that is full, with window 4096 against
none (flash_cosine_sim_attention_with_kv_cache, no append), timed the same way.
The card's name and power limit are read (query only) in the same run.  Measurement helper only."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from flash_cosine_sim_attention_b200 import (flash_cosine_sim_attention,  # noqa: E402
                                             flash_cosine_sim_attention_with_kv_cache)
from gpu_varlen_bench import card  # noqa: E402

TRAIN = {                      # (B, H, kv_heads, N, D)
    "T1": (4, 8, 8, 16384, 64),
    "T2": (1, 16, 16, 32768, 128),
    "T3": (2, 16, 4, 32768, 128),
}
WINDOWS = (None, 1024, 4096)


def pairs(N, w):
    """visible (query, key) pairs of one causal head: sum_i min(i + 1, w)"""
    if w is None or w >= N:
        return N * (N + 1) // 2
    return w * N - w * (w - 1) // 2


def timed(fn, steps, flush):
    evs = []
    for _ in range(steps):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        evs.append((a, b))
    torch.cuda.synchronize()
    return [a.elapsed_time(b) for a, b in evs]


def summary(t):
    t = sorted(t)
    return {"median_ms": t[len(t) // 2], "p10_ms": t[len(t) // 10], "p90_ms": t[(9 * len(t)) // 10]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")      # > the 50 MB L2
    res = {"card": card(), "steps": args.steps, "rounds": args.rounds, "train": {}, "decode": {}}
    g = torch.Generator(device="cuda").manual_seed(0)
    rn = lambda *s: torch.randn(*s, generator=g, device="cuda", dtype=torch.bfloat16)
    for name, (B, H, Hk, N, D) in TRAIN.items():
        q, k, v, do = rn(B, H, N, D), rn(B, Hk, N, D), rn(B, Hk, N, D), rn(B, H, N, D)
        for t in (q, k, v):
            t.requires_grad_()

        def step(w):
            o = flash_cosine_sim_attention(q, k, v, causal=True, window=w)
            torch.autograd.grad(o, (q, k, v), do)

        for w in WINDOWS:
            for _ in range(2):
                step(w)
        times = {w: [] for w in WINDOWS}
        for _ in range(args.rounds):
            for w in WINDOWS:
                times[w] += timed(lambda: step(w), args.steps, flush)
        row = {"B": B, "H": H, "kv_heads": Hk, "N": N, "D": D}
        for w in WINDOWS:
            s = summary(times[w])
            s["visible_tflops"] = 3.5 * 4 * D * H * B * pairs(N, w) / s["median_ms"] / 1e9
            row[str(w)] = s
        res["train"][name] = row
        print(f"{name} ({B}, {H}, kv {Hk}, {N}, {D}): " + "  ".join(
            f"window {w}: {row[str(w)]['median_ms']:.2f} ms ({row[str(w)]['visible_tflops']:.0f} TFLOP/s)"
            for w in WINDOWS), flush=True)
        del q, k, v, do

    B, H, Hk, cap, D = 1, 16, 2, 65536, 128
    q, kc, vc = rn(B, H, 1, D), rn(B, Hk, cap, D), rn(B, Hk, cap, D)
    seq = torch.full((B,), cap, dtype=torch.int32, device="cuda")
    with torch.no_grad():
        for w in (None, 4096):
            for _ in range(3):
                flash_cosine_sim_attention_with_kv_cache(q, kc, vc, seq, window=w)
        times = {w: [] for w in (None, 4096)}
        for _ in range(args.rounds):
            for w in times:
                times[w] += timed(lambda: flash_cosine_sim_attention_with_kv_cache(q, kc, vc, seq, window=w),
                                  args.steps * 5, flush)
    res["decode"] = {"shape": [B, H, Hk, cap, D, 1], **{str(w): summary(t) for w, t in times.items()}}
    print(f"decode ({B}, {H}, kv {Hk}, cache {cap}, {D}, 1 token): " + "  ".join(
        f"window {w}: {res['decode'][str(w)]['median_ms'] * 1e3:.1f} us" for w in times), flush=True)
    print("card:", res["card"])
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
