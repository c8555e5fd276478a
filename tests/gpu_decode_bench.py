"""Decode benchmark: flash_cosine_sim_attention_with_kv_cache against the path that exists without it, on one GPU.

    python tests/gpu_decode_bench.py [--rounds 5] [--calls 20] [--skip-model]

Operator level, bf16, all batch elements at the same length (so the baseline can run), capacity = T:
  op        flash_cosine_sim_attention_with_kv_cache(q, k_cache, v_cache, seqlens, k_new, v_new): append + attention
  baseline  l2norm_tensors(q, k_new), a copy of k_hat / v_new into the caches, then
            flash_cosine_sim_attention(q_hat, k_cache[:T], v_cache[:T], causal=True, l2norm_qk=False)
Each call is timed with CUDA events after an L2 flush; the variants alternate over the rounds; the median and the
p10-p90 range over all calls are reported, with the bandwidth over the bytes the work needs (K_hat and V of the
prefix, q, o, and the appended rows read and written) and its share of the data sheet's 3.35 TB/s (H100 SXM).
Model level: `generate` tokens/s of train.py's model in fp16 (batch 1, prompt 512, 512 new tokens), with and without
kv_cache.  The card's name and power limit are read in the same run."""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from flash_cosine_sim_attention_b200 import (flash_cosine_sim_attention,  # noqa: E402
                                             flash_cosine_sim_attention_with_kv_cache, l2norm_tensors)

WORKLOADS = [  # (B, H, kv_heads, T, D, Nq): one decode step each (Nq new tokens appended, T = visible length)
    (8, 8, 8, 4096, 64, 1),
    (1, 16, 2, 32768, 128, 1),
    (4, 32, 8, 8192, 128, 4),
    (1, 8, 8, 8192, 64, 1),
]
HBM_BYTES_PER_S = 3.35e12


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        return torch.cuda.get_device_name()


def needed_bytes(B, H, Hk, T, D, Nq):
    e = 2
    return (2 * B * Hk * T * D + 2 * B * H * Nq * D + 4 * B * Hk * Nq * D) * e


def setup(B, H, Hk, T, D, Nq):
    g = torch.Generator(device="cuda").manual_seed(0)
    dt = torch.bfloat16
    rnd = lambda *s: torch.randn(*s, device="cuda", generator=g).to(dt)
    kc = l2norm_tensors(rnd(B, Hk, T, D))[0]
    vc = rnd(B, Hk, T, D)
    q, k, v = rnd(B, H, Nq, D), rnd(B, Hk, Nq, D), rnd(B, Hk, Nq, D)
    seqlens = torch.full((B,), T - Nq, dtype=torch.int32, device="cuda")
    L = T - Nq

    def op():
        return flash_cosine_sim_attention_with_kv_cache(q, kc, vc, seqlens, k, v)

    def baseline():
        qh, kh = l2norm_tensors(q, k)
        kc[:, :, L:T].copy_(kh)
        vc[:, :, L:T].copy_(v)
        return flash_cosine_sim_attention(qh, kc[:, :, :T], vc[:, :, :T], causal=True, l2norm_qk=False)
    return {"op": op, "baseline": baseline}


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


def operator_level(rounds, calls):
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    out = []
    for w in WORKLOADS:
        fns = setup(*w)
        with torch.no_grad():
            for fn in fns.values():
                for _ in range(3):
                    fn()
            torch.cuda.synchronize()
            samples = {name: [] for name in fns}
            for _ in range(rounds):
                for name, fn in fns.items():
                    samples[name] += time_calls(fn, calls, flush)
        nb = needed_bytes(*w)
        for name, ts in samples.items():
            med = pct(ts, 50)
            r = {"workload": dict(zip(("B", "H", "kv_heads", "T", "D", "Nq"), w)), "variant": name,
                 "us_median": round(med, 2), "us_p10": round(pct(ts, 10), 2), "us_p90": round(pct(ts, 90), 2),
                 "bytes": nb, "GB_per_s": round(nb / med / 1e3, 1),
                 "share_of_3.35TB_s": round(nb / med / 1e-6 / HBM_BYTES_PER_S, 3)}
            out.append(r)
            print(json.dumps(r), flush=True)
        sp = pct(samples["baseline"], 50) / pct(samples["op"], 50)
        print(json.dumps({"workload": w, "speedup_op_over_baseline": round(sp, 2)}), flush=True)
        del fns
        torch.cuda.empty_cache()
    return out


def model_level():
    from flash_cosine_sim_attention_b200.transformer import CosineSimCausalTransformer
    torch.manual_seed(0)
    m = CosineSimCausalTransformer(num_tokens=256, dim=512, max_seq_len=1024, depth=8, heads=8, dim_head=64,
                                   attn_scale=1, attn_l2norm_groups=8, use_cuda_kernel=True).cuda().half().eval()
    prompt = torch.randint(0, 256, (1, 512), device="cuda")
    res = {}
    for kv in (True, False):
        m.generate(prompt, 8, kv_cache=kv)                   # warm-up
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        m.generate(prompt, 512, kv_cache=kv)
        torch.cuda.synchronize()
        res["kv_cache" if kv else "no_cache"] = round(512 / (time.perf_counter() - t0), 1)
    r = {"model": "dim 512 depth 8 heads 8 dim_head 64 fp16, batch 1, prompt 512, 512 new tokens",
         "tokens_per_s": res, "speedup": round(res["kv_cache"] / res["no_cache"], 2)}
    print(json.dumps(r), flush=True)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--skip-model", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gpu_decode_bench.py needs a CUDA device")
    print(json.dumps({"card": card()}), flush=True)
    operator_level(args.rounds, args.calls)
    if not args.skip_model:
        model_level()


if __name__ == "__main__":
    main()
