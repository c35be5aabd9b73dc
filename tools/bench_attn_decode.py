#!/usr/bin/env python
"""Grouped-query attention and split-KV decoding against the unsplit kernel, the expanded-K/V path and torch SDPA.

    python tools/bench_attn_decode.py [--reps 5] [--steps 20] [--out FILE] [--small]

Prints one JSON object (and writes it to FILE if given).  The card's name, power limit and max SM clock are read in
the same run.  Timing: CUDA events around `steps` back-to-back calls; the variants of a shape are timed alternately,
`reps` times each, and the median with the min .. max spread is reported.  Variants:
  auto      fmha_fwd(..., num_splits=0) (`auto_splits`: the library's choice, b200_fmha_fwd_f16_gqa_splits)
  split1    fmha_fwd(..., num_splits=1): GQA packing without a split
  expanded  fmha_fwd on K and V with every head repeated H / Hkv times (repeat_interleave done once, outside the timing)
  sdpa      torch.nn.functional.scaled_dot_product_attention(..., enable_gqa=True); with Nq != Nk and the mask
            an explicit bottom-right boolean mask (SDPA's is_causal would align the diagonal top-left)
and for the first shape a sweep of fixed split counts.  Decode rows report GB/s of the unique K and V bytes,
2 B Hkv Nk D x 2; the prefill rows report TFLOPS of 4 B H D x (visible (query, key) pairs).
--small runs tiny shapes (argument parsing and byte counts, not a measurement).
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

# (name, B, H, Hkv, Nq, Nk, D, causal)
SHAPES = [
    ("decode", 1, 64, 8, 1, 32768, 128, False),
    ("decode", 8, 32, 8, 1, 8192, 128, False),
    ("decode", 8, 32, 32, 1, 8192, 128, False),
    ("decode", 64, 32, 8, 1, 2048, 128, False),
    ("speculative", 8, 32, 8, 4, 8192, 128, True),
    ("causal prefill", 4, 32, 8, 4096, 4096, 128, True),
    ("causal prefill", 2, 32, 8, 1000, 1000, 128, True),
]
SMALL = [("decode", 1, 4, 2, 1, 256, 64, False), ("causal prefill", 1, 4, 2, 128, 128, 64, True)]
SWEEP = [2, 4, 8, 16, 32, 64]


def card():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else f"unknown ({r.stderr.strip()})"


def kv_bytes(B, Hkv, Nk, D):
    return 2 * B * Hkv * Nk * D * 2


def flops(B, H, Nq, Nk, D, causal):
    diag = Nk - Nq
    pairs = sum(min(Nk, max(0, i + diag + 1)) for i in range(Nq)) if causal else Nq * Nk
    return 4.0 * B * H * D * pairs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None)
    ap.add_argument("--small", action="store_true")
    args = ap.parse_args()

    import torch
    import torch.nn.functional as F
    from leetcuda_b200 import _capi, flash_attn

    assert torch.cuda.is_available(), "this benchmark needs a CUDA device"
    torch.manual_seed(0)
    sms = torch.cuda.get_device_properties(0).multi_processor_count

    def time_ms(fn, steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / steps

    result = {"card": card(), "sms": sms, "reps": args.reps, "steps": args.steps, "rows": []}
    for si, (name, B, H, Hkv, Nq, Nk, D, causal) in enumerate(SMALL if args.small else SHAPES):
        G = H // Hkv
        q = torch.randn(B, H, Nq, D, device="cuda", dtype=torch.half)
        k, v = (torch.randn(B, Hkv, Nk, D, device="cuda", dtype=torch.half) for _ in range(2))
        ke, ve = k.repeat_interleave(G, 1).contiguous(), v.repeat_interleave(G, 1).contiguous()
        o = torch.empty_like(q)
        # SDPA's is_causal aligns the diagonal top-left; with Nq != Nk the bottom-right mask of fmha_fwd is explicit
        mask = (torch.ones(Nq, Nk, dtype=torch.bool, device="cuda").tril(Nk - Nq)
                if causal and Nq != Nk else None)
        runs = {
            "auto": lambda: flash_attn.fmha_fwd(q, k, v, o, causal=causal, num_splits=0),
            "split1": lambda: flash_attn.fmha_fwd(q, k, v, o, causal=causal, num_splits=1),
            "expanded": lambda: flash_attn.fmha_fwd(q, ke, ve, o, causal=causal),
            "sdpa": lambda: F.scaled_dot_product_attention(q, k, v, attn_mask=mask, is_causal=causal and mask is None,
                                                           enable_gqa=True),
        }
        if si == 0:
            for s in SWEEP:
                runs[f"splits{s}"] = (lambda s=s: flash_attn.fmha_fwd(q, k, v, o, causal=causal, num_splits=s))
        for fn in runs.values():
            for _ in range(3):
                fn()
        ms = {n: [] for n in runs}
        for _ in range(args.reps):
            for n, fn in runs.items():   # alternated: every repetition times each variant once
                ms[n].append(time_ms(fn, args.steps))
        decode = name != "causal prefill"
        work = kv_bytes(B, Hkv, Nk, D) if decode else flops(B, H, Nq, Nk, D, causal)
        unit = "kv_gbs" if decode else "tflops"
        scale = 1e9 if decode else 1e12
        row = {"shape": f"{name} B{B} H{H} Hkv{Hkv} Nq{Nq} Nk{Nk} D{D}" + (" causal" if causal else ""),
               "auto_splits": _capi.lib().b200_fmha_fwd_f16_gqa_splits(B, H, Hkv, Nq, Nk, D),
               "kv_bytes" if decode else "flops": work}
        for n in runs:
            med = statistics.median(ms[n])
            row[n] = {"ms_median": med, "ms_min": min(ms[n]), "ms_max": max(ms[n]),
                      f"{unit}_median": work / (med * 1e-3) / scale, f"{unit}_min": work / (max(ms[n]) * 1e-3) / scale,
                      f"{unit}_max": work / (min(ms[n]) * 1e-3) / scale}
        result["rows"].append(row)
        del q, k, v, ke, ve, o
        torch.cuda.empty_cache()
    text = json.dumps(result)
    print(text)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(text + "\n")


if __name__ == "__main__":
    main()
