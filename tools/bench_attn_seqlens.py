#!/usr/bin/env python
"""Per-sequence lengths over a padded KV cache: the seqlens call against what a caller can do without it.

    python tools/bench_attn_seqlens.py [--reps 5] [--steps 20] [--out FILE] [--small]

Prints one JSON object (and writes it to FILE if given).  The card's name, power limit and max SM clock are read in
the same run.  Timing: CUDA events around `steps` back-to-back calls; the variants of a shape are timed alternately,
`reps` times each, and the median with the min .. max spread is reported.  Lengths are drawn from a seeded generator.
Variants:
  seqlens   fmha_fwd(..., num_splits=0, seqlens_q=, seqlens_k=)
  padded    fmha_fwd(..., num_splits=0) on the padded buffers without lengths: what padding costs today (its results are
            wrong for the short sequences)
  loop      one fmha_fwd(..., num_splits=0) per sequence on its sliced tensors (slices made once, outside the timing):
            today's only correct way
  sdpa      torch SDPA with an explicit per-sequence bottom-right boolean mask and enable_gqa
Decode rows report GB/s of the visible K and V bytes, 2 Hkv D x 2 x sum Lk_b; prefill rows TFLOPS of 4 H D x (visible
(query, key) pairs).  --small runs tiny shapes (argument parsing and byte counts, not a measurement).
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

# (name, B, H, Hkv, Nq, Nk, D, causal, (lo, hi) of Lk_b; prefill: Lq_b = Lk_b)
SHAPES = [
    ("decode", 32, 32, 8, 1, 8192, 128, False, (256, 8192)),
    ("decode", 4, 64, 8, 1, 32768, 128, False, (1024, 32768)),
    ("causal prefill", 8, 32, 8, 4096, 4096, 128, True, (512, 4096)),
]
SMALL = [("decode", 4, 4, 2, 1, 512, 64, False, (16, 512)), ("causal prefill", 2, 4, 2, 256, 256, 64, True, (32, 256))]


def card():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else f"unknown ({r.stderr.strip()})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None)
    ap.add_argument("--small", action="store_true")
    args = ap.parse_args()

    import numpy as np
    import torch
    import torch.nn.functional as F
    from leetcuda_b200 import flash_attn

    assert torch.cuda.is_available(), "this benchmark needs a CUDA device"
    torch.manual_seed(0)
    rng = np.random.default_rng(0)

    def time_ms(fn, steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / steps

    result = {"card": card(), "reps": args.reps, "steps": args.steps, "rows": []}
    for name, B, H, Hkv, Nq, Nk, D, causal, (lo, hi) in (SMALL if args.small else SHAPES):
        prefill = name == "causal prefill"
        lk = [int(x) for x in rng.integers(lo, hi + 1, size=B)]
        lq = lk if prefill else [Nq] * B
        q = torch.randn(B, H, Nq, D, device="cuda", dtype=torch.half)
        k, v = (torch.randn(B, Hkv, Nk, D, device="cuda", dtype=torch.half) for _ in range(2))
        o = torch.empty_like(q)
        tq = torch.tensor(lq, dtype=torch.int32, device="cuda")
        tk = torch.tensor(lk, dtype=torch.int32, device="cuda")
        sl = [(q[b:b + 1, :, :lq[b]].contiguous(), k[b:b + 1, :, :lk[b]].contiguous(),
               v[b:b + 1, :, :lk[b]].contiguous(), torch.empty(1, H, lq[b], D, device="cuda", dtype=torch.half))
              for b in range(B)]
        i = torch.arange(Nq, device="cuda")[:, None]
        j = torch.arange(Nk, device="cuda")[None, :]
        mask = torch.stack([(i < lq[b]) & (j < lk[b]) & ((j <= i + lk[b] - lq[b]) if causal else True)
                            for b in range(B)])[:, None]

        def loop():
            for qs, ks, vs, os_ in sl:
                flash_attn.fmha_fwd(qs, ks, vs, os_, causal=causal, num_splits=0)

        runs = {
            "seqlens": lambda: flash_attn.fmha_fwd(q, k, v, o, causal=causal, num_splits=0, seqlens_q=tq,
                                                   seqlens_k=tk),
            "padded": lambda: flash_attn.fmha_fwd(q, k, v, o, causal=causal, num_splits=0),
            "loop": loop,
            "sdpa": lambda: F.scaled_dot_product_attention(q, k, v, attn_mask=mask, enable_gqa=True),
        }
        for fn in runs.values():
            for _ in range(3):
                fn()
        ms = {n: [] for n in runs}
        for _ in range(args.reps):
            for n, fn in runs.items():   # alternated: every repetition times each variant once
                ms[n].append(time_ms(fn, args.steps))
        if prefill:
            pairs = sum(sum(min(lk[b], i + lk[b] - lq[b] + 1) for i in range(lq[b])) for b in range(B))
            work, unit, scale = 4.0 * H * D * pairs, "tflops", 1e12
        else:
            work, unit, scale = 2.0 * Hkv * D * 2 * sum(lk), "kv_gbs", 1e9
        row = {"shape": f"{name} B{B} H{H} Hkv{Hkv} Nq{Nq} Nk{Nk} D{D}" + (" causal" if causal else ""),
               "lengths": f"Lk in [{lo}, {hi}]" + (", Lq = Lk" if prefill else ""), "sum_lk": sum(lk),
               "work": work}
        for n in runs:
            med = statistics.median(ms[n])
            row[n] = {"ms_median": med, "ms_min": min(ms[n]), "ms_max": max(ms[n]),
                      f"{unit}_median": work / (med * 1e-3) / scale, f"{unit}_min": work / (max(ms[n]) * 1e-3) / scale,
                      f"{unit}_max": work / (min(ms[n]) * 1e-3) / scale}
        result["rows"].append(row)
        del q, k, v, o, sl, mask
        torch.cuda.empty_cache()
    text = json.dumps(result)
    print(text)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(text + "\n")


if __name__ == "__main__":
    main()
