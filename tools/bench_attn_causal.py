#!/usr/bin/env python
"""Causal attention against the unmasked kernel, torch SDPA (is_causal=True) and a decode shape, in one run.

    python tools/bench_attn_causal.py [--reps 5] [--steps 20] [--out FILE]

Prints one JSON object (and writes it to FILE if given).  The card's name, power limit and max SM clock are read in
the same run.  Timing: CUDA events around `steps` back-to-back launches; causal and non-causal are timed alternately,
`reps` times each, and the median with the min .. max spread is reported.  FLOPs are counted as 4 B H D x (visible
(query, key) pairs): N (N + 1) / 2 per head with the causal mask, N^2 without.  The decode shape reports the bytes of K
and V it has to read (2 B H Nk D x 2 bytes) over its time; Nq = 1 gives a grid of only B*H CTAs, so no target applies.
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))


def card():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else f"unknown ({r.stderr.strip()})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    import torch.nn.functional as F
    from leetcuda_b200 import flash_attn

    assert torch.cuda.is_available(), "this benchmark needs a CUDA device"
    torch.manual_seed(0)

    def time_ms(fn, steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / steps

    def summary(ms, flops):
        med = statistics.median(ms)
        return {"ms_median": med, "ms_min": min(ms), "ms_max": max(ms), "tflops_median": flops / (med * 1e-3) / 1e12,
                "tflops_min": flops / (max(ms) * 1e-3) / 1e12, "tflops_max": flops / (min(ms) * 1e-3) / 1e12}

    result = {"card": card(), "reps": args.reps, "steps": args.steps, "rows": []}
    B, H, N = 4, 32, 4096
    for D in (128, 64):
        q, k, v = (torch.randn(B, H, N, D, device="cuda", dtype=torch.half) for _ in range(3))
        o = torch.empty_like(q)
        runs = {
            "causal": lambda: flash_attn.fmha_fwd(q, k, v, o, causal=True),
            "full": lambda: flash_attn.fmha_fwd(q, k, v, o),
            "sdpa_causal": lambda: F.scaled_dot_product_attention(q, k, v, is_causal=True),
        }
        for fn in runs.values():
            for _ in range(3):
                fn()
        ms = {name: [] for name in runs}
        for _ in range(args.reps):
            for name, fn in runs.items():      # alternated: every repetition times each variant once
                ms[name].append(time_ms(fn, args.steps))
        pairs = {"causal": N * (N + 1) / 2, "full": N * N, "sdpa_causal": N * (N + 1) / 2}
        row = {"shape": f"B{B} H{H} N{N} D{D}"}
        for name in runs:
            row[name] = summary(ms[name], 4.0 * B * H * D * pairs[name])
        ratios = [c / f for c, f in zip(ms["causal"], ms["full"])]
        row["causal_over_full_time"] = {"median": statistics.median(ratios), "min": min(ratios), "max": max(ratios)}
        result["rows"].append(row)
        del q, k, v, o
        torch.cuda.empty_cache()

    Bd, Hd, Nk, D = 8, 32, 8192, 128
    q = torch.randn(Bd, Hd, 1, D, device="cuda", dtype=torch.half)
    k, v = (torch.randn(Bd, Hd, Nk, D, device="cuda", dtype=torch.half) for _ in range(2))
    o = torch.empty_like(q)
    fn = lambda: flash_attn.fmha_fwd(q, k, v, o, causal=True)   # noqa: E731  (Nq = 1: the mask hides nothing)
    for _ in range(3):
        fn()
    dms = [time_ms(fn, args.steps) for _ in range(args.reps)]
    kv_bytes = 2 * Bd * Hd * Nk * D * 2
    med = statistics.median(dms)
    result["rows"].append({"shape": f"decode B{Bd} H{Hd} Nq1 Nk{Nk} D{D}", "ms_median": med, "ms_min": min(dms),
                           "ms_max": max(dms), "kv_gbs_median": kv_bytes / (med * 1e-3) / 1e9,
                           "kv_bytes": kv_bytes})
    text = json.dumps(result)
    print(text)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(text + "\n")


if __name__ == "__main__":
    main()
