"""fwd+bwd time of grouped-query attention against the two ways to get the same result without it.
    python tests/gpu_gqa_bench.py [--steps K] [--rounds R] [--json PATH]
Variants, alternated round by round within one process:
    gqa     k, v with kv_heads heads straight into the operator
    expand  the workaround: k, v repeat_interleave'd to the query heads (copies in the forward, autograd sums
            dk, dv in the backward), then the multi-head call
    mha     k, v with as many heads as q (same attention FLOPs, no group)
Each step is one forward and one backward through the public API, timed with CUDA events, after a flush of L2.
The card's name and power limit are read (query only) in the same run.  Measurement helper only."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from flash_cosine_sim_attention_b200 import flash_cosine_sim_attention  # noqa: E402

WORKLOADS = {                  # (B, H, kv_heads, N, D), bf16, causal
    "W1": (4, 8, 2, 4096, 64),
    "W2": (1, 16, 2, 4096, 64),
    "W3": (2, 16, 4, 4096, 128),
}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def make(B, H, Hk, N, D, variant, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g, device="cuda", dtype=torch.bfloat16)
    q, do = rn(B, H, N, D), rn(B, H, N, D)
    kh = H if variant == "mha" else Hk
    k, v = rn(B, kh, N, D), rn(B, kh, N, D)
    for t in (q, k, v):
        t.requires_grad_()
    G = H // Hk

    def step():
        kk, vv = (k.repeat_interleave(G, 1), v.repeat_interleave(G, 1)) if variant == "expand" else (k, v)
        o = flash_cosine_sim_attention(q, kk, vv, causal=True)
        torch.autograd.grad(o, (q, k, v), do)

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
    for name, shape in WORKLOADS.items():
        steps = {var: make(*shape, var) for var in ("gqa", "expand", "mha")}
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
        row = {}
        for var, t in times.items():
            t = sorted(t)
            row[var] = {"median_ms": t[len(t) // 2], "p10_ms": t[len(t) // 10], "p90_ms": t[(9 * len(t)) // 10]}
        row["shape"] = dict(zip(("B", "H", "kv_heads", "N", "D"), shape))
        res["workloads"][name] = row
        m = {v: row[v]["median_ms"] for v in ("gqa", "expand", "mha")}
        print(f"{name} {shape}: gqa {m['gqa']:.3f} ms  expand {m['expand']:.3f} ms  mha {m['mha']:.3f} ms  "
              f"(gqa / expand {m['gqa'] / m['expand']:.3f}, gqa / mha {m['gqa'] / m['mha']:.3f})", flush=True)
    print("card:", res["card"])
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
