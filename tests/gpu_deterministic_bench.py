"""fwd+bwd time of the deterministic backward against the default one.
    python tests/gpu_deterministic_bench.py [--steps K] [--rounds R] [--json PATH]
Variants, alternated round by round within one process:
    default        flash_cosine_sim_attention(..., deterministic=False)
    deterministic  the same call with deterministic=True
Each step is one forward and one backward through the public API, timed with CUDA events after a flush of L2; the
medians are reported.  A separate profiled pass (torch.profiler, CUDA activities) gives each kernel's time per step.
The card's name and power limit are read (query only) in the same run.  Measurement helper only."""
import argparse
import json
import os
import sys
from collections import defaultdict

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from flash_cosine_sim_attention_b200 import flash_cosine_sim_attention, flash_cosine_sim_attention_varlen  # noqa: E402
from gpu_gqa_bench import card  # noqa: E402
from gpu_varlen_bench import skewed  # noqa: E402

WORKLOADS = {                  # bf16, causal: (B, H, kv_heads, N, D, window) dense, or (lengths, H, kv_heads, D) packed
    "C3-D64": (4, 8, 8, 4096, 64, None),
    "C3-D128": (4, 8, 8, 4096, 128, None),
    "grouped": (1, 16, 2, 4096, 64, None),
    "mqa": (2, 16, 1, 4096, 64, None),
    "varlen-W2": (skewed(), 8, 8, 64),
    "window4096": (4, 8, 8, 16384, 64, 4096),
}
VARIANTS = {"default": False, "deterministic": True}


def make(spec, deterministic, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g, device="cuda", dtype=torch.bfloat16).requires_grad_()
    if isinstance(spec[0], list):
        lengths, H, Hk, D = spec
        T = sum(lengths)
        q, k, v, do = rn(T, H, D), rn(T, Hk, D), rn(T, Hk, D), rn(T, H, D).detach()
        cu = torch.tensor([0] + list(torch.tensor(lengths).cumsum(0).tolist()), dtype=torch.int32, device="cuda")
        M = max(lengths)
        call = lambda: flash_cosine_sim_attention_varlen(q, k, v, cu, cu, M, M, causal=True, deterministic=deterministic)
    else:
        B, H, Hk, N, D, window = spec
        q, do = rn(B, H, N, D), rn(B, H, N, D).detach()
        k, v = rn(B, Hk, N, D), rn(B, Hk, N, D)
        call = lambda: flash_cosine_sim_attention(q, k, v, causal=True, window=window, deterministic=deterministic)

    def step():
        torch.autograd.grad(call(), (q, k, v), do)

    return step


def kernel_times(step, n=5):
    """Device time per step of each kernel (ms), from a profiled run of n steps."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            step()
        torch.cuda.synchronize()
    acc = defaultdict(float)
    for e in prof.events():
        if e.device_type.name == "CUDA":
            name = e.name.split("<")[0].split("(")[0].replace("void ", "").replace("fcsa::", "")
            acc[name] += e.time_range.elapsed_us() / 1000.0 / n
    return {k: round(v, 4) for k, v in sorted(acc.items(), key=lambda kv: -kv[1]) if v >= 0.001}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")      # > the 50 MB L2
    res = {"card": card(), "steps": args.steps, "rounds": args.rounds, "workloads": {}}
    print("card:", res["card"], flush=True)
    for name, spec in WORKLOADS.items():
        steps = {var: make(spec, det) for var, det in VARIANTS.items()}
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
            row[var] = {"median_ms": t[len(t) // 2], "p10_ms": t[len(t) // 10], "p90_ms": t[(9 * len(t)) // 10],
                        "kernels_ms": kernel_times(steps[var])}
        res["workloads"][name] = row
        m = {v: row[v]["median_ms"] for v in VARIANTS}
        print(f"{name}: default {m['default']:.3f} ms  deterministic {m['deterministic']:.3f} ms  "
              f"(ratio {m['deterministic'] / m['default']:.3f})", flush=True)
        for var in VARIANTS:
            print(f"    {var}: {row[var]['kernels_ms']}", flush=True)
        del steps
        torch.cuda.empty_cache()
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
