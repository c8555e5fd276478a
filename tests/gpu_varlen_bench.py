"""fwd+bwd time of packed variable-length attention against the two ways to get the same result without it.
    python tests/gpu_varlen_bench.py [--steps K] [--rounds R] [--json PATH]
Variants, alternated round by round within one process (bf16, causal):
    varlen  the packed (total, heads, dim) tensors and cu_seqlens straight into flash_cosine_sim_attention_varlen
    padded  every sequence padded to the longest: one dense call on (B, heads, max, dim) tensors, padded beforehand
            (padding at the end of q and k is never visible to a valid query under the bottom-right causal rule)
    loop    one dense call per sequence on views of the packed tensors
    view    (equal lengths only) one dense call on the packed tensors viewed as (B, heads, N, dim): the dense op on
            the same memory layout as varlen, which separates the cost of the layout from that of the packing
Each step is one forward and one backward through the public API, timed with CUDA events, after a flush of L2.
Useful TFLOP/s count each sequence's own causal FLOPs only: 3.5 x 2 H D L^2 (forward 2 H D L^2, backward 2.5 x).
The card's name and power limit are read (query only) in the same run.  Measurement helper only."""
import argparse
import json
import os
import random
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from flash_cosine_sim_attention_b200 import flash_cosine_sim_attention, flash_cosine_sim_attention_varlen  # noqa: E402


def skewed(total=32768, lo=64, hi=8192, seed=0):
    """seeded lengths between lo and hi summing to total (log-uniform draws)"""
    rng = random.Random(seed)
    out = []
    while sum(out) < total:
        out.append(int(min(hi, lo * 2 ** rng.uniform(0, 7))))
    out[-1] -= sum(out) - total
    if out[-1] < lo:
        out[-2] += out.pop()
    return out


WORKLOADS = {                  # (lengths, H, kv_heads, D)
    "W1": ([4096] * 4, 8, 8, 64),
    "W2": (skewed(), 8, 8, 64),
    "W3": (skewed(), 16, 4, 128),
}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def make(lengths, H, Hk, D, variant, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g, device="cuda", dtype=torch.bfloat16)
    T, B, M = sum(lengths), len(lengths), max(lengths)
    if variant == "padded":
        q, do = rn(B, H, M, D), rn(B, H, M, D)
        k, v = rn(B, Hk, M, D), rn(B, Hk, M, D)
    else:
        q, do = rn(T, H, D), rn(T, H, D)
        k, v = rn(T, Hk, D), rn(T, Hk, D)
    for t in (q, k, v):
        t.requires_grad_()
    cu = torch.tensor([0] + list(torch.tensor(lengths).cumsum(0).tolist()), dtype=torch.int32, device="cuda")
    starts = cu.tolist()

    def step():
        if variant == "varlen":
            o = flash_cosine_sim_attention_varlen(q, k, v, cu, cu, M, M, causal=True)
            torch.autograd.grad(o, (q, k, v), do)
        elif variant == "view":
            bhnd = lambda t: t.view(B, M, t.shape[1], D).transpose(1, 2)
            o = flash_cosine_sim_attention(bhnd(q), bhnd(k), bhnd(v), causal=True)
            torch.autograd.grad(o, (q, k, v), bhnd(do))
        elif variant == "padded":
            o = flash_cosine_sim_attention(q, k, v, causal=True)
            torch.autograd.grad(o, (q, k, v), do)
        else:
            seq = lambda t, s, n: t[s:s + n].transpose(0, 1).unsqueeze(0)
            outs = [flash_cosine_sim_attention(seq(q, s, n), seq(k, s, n), seq(v, s, n), causal=True)
                    for s, n in zip(starts, lengths)]
            torch.autograd.grad(outs, (q, k, v), [seq(do, s, n) for s, n in zip(starts, lengths)])

    return step


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")      # > the 50 MB L2
    res = {"card": card(), "steps": args.steps, "rounds": args.rounds, "workloads": {}}
    for name, (lengths, H, Hk, D) in WORKLOADS.items():
        flops = sum(3.5 * 2 * H * D * n * n for n in lengths)
        variants = ("varlen", "padded", "loop") + (("view",) if len(set(lengths)) == 1 else ())
        steps = {var: make(lengths, H, Hk, D, var) for var in variants}
        for s in steps.values():                     # warm-up: module loads, workspaces, allocator
            for _ in range(3):
                s()
        torch.cuda.synchronize()
        times = {var: [] for var in steps}
        for _ in range(args.rounds):
            for var, s in steps.items():
                evs = []
                for _ in range(args.steps):
                    flush.zero_()
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record()
                    s()
                    b.record()
                    evs.append((a, b))
                torch.cuda.synchronize()
                times[var] += [a.elapsed_time(b) for a, b in evs]
        row = {"lengths": lengths, "H": H, "kv_heads": Hk, "D": D, "useful_tflop": flops / 1e12}
        for var, t in times.items():
            t = sorted(t)
            med = t[len(t) // 2]
            row[var] = {"median_ms": med, "p10_ms": t[len(t) // 10], "p90_ms": t[(9 * len(t)) // 10],
                        "useful_tflops": flops / med / 1e9}
        res["workloads"][name] = row
        m = {v: row[v]["median_ms"] for v in steps}
        print(f"{name} B={len(lengths)} max={max(lengths)} total={sum(lengths)} H={H} kv={Hk} D={D}: " +
              "  ".join(f"{v} {m[v]:.3f} ms ({row[v]['useful_tflops']:.0f} TFLOP/s)" for v in steps) +
              f"  padded/varlen {m['padded'] / m['varlen']:.2f}x  loop/varlen {m['loop'] / m['varlen']:.2f}x",
              flush=True)
    print("card:", res["card"])
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
