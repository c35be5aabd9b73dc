#!/usr/bin/env python
"""Paged KV cache: the paged call against a contiguous padded cache and against gathering the pages first.

    python tools/bench_attn_paged.py [--reps 5] [--steps 20] [--out FILE] [--small]

Prints one JSON object (and writes it to FILE if given).  The card's name, power limit and max SM clock are read in
the same run.  Timing: CUDA events around `steps` back-to-back calls; the variants of a shape are timed alternately,
`reps` times each, and the median with the min .. max spread is reported.  Lengths are the seeded draws of
tools/bench_attn_seqlens.py (same generator, same shapes).  Each sequence's pages are assigned through a random
permutation of a pool with 25 % more pages than the batch uses; table entries past a sequence's pages are -1.
Variants:
  paged/16, paged/256   fmha_fwd(..., num_splits=0, seqlens_q=, seqlens_k=, block_table=) on pools of 16- / 256-key
                        pages
  seqlens               fmha_fwd(..., num_splits=0, seqlens_q=, seqlens_k=) on a contiguous padded cache that holds the
                        same keys: the same kernel without the table
  gather+seqlens        what a caller with a page pool does today: gather the 16-key pages into the padded cache
                        (torch indexing), then the seqlens call, both inside the timing
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

# (name, B, H, Hkv, Nq, Nk, D, causal, (lo, hi) of Lk_b; prefill: Lq_b = Lk_b): those of bench_attn_seqlens.py
SHAPES = [
    ("decode", 32, 32, 8, 1, 8192, 128, False, (256, 8192)),
    ("decode", 4, 64, 8, 1, 32768, 128, False, (1024, 32768)),
    ("causal prefill", 8, 32, 8, 4096, 4096, 128, True, (512, 4096)),
]
SMALL = [("decode", 4, 4, 2, 1, 512, 64, False, (16, 512)), ("causal prefill", 2, 4, 2, 256, 256, 64, True, (32, 256))]
PAGE_SIZES = (16, 256)


def card():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else f"unknown ({r.stderr.strip()})"


def paginate(k, v, lk, page_size, gen):
    """Pools [num_pages, page_size, Hkv, D] holding k, v [B,Hkv,Nk,D] (rows < lk[b]) in randomly placed pages, and
    the table [B, Nk / page_size] (-1 past each sequence's pages).  `gen`: a torch.Generator on the CPU."""
    import torch
    B, Hkv, Nk, D = k.shape
    used = [-(-x // page_size) for x in lk]
    num_pages = max(1, (sum(used) * 5 + 3) // 4)
    perm = torch.randperm(num_pages, generator=gen).tolist()
    table = torch.full((B, Nk // page_size), -1, dtype=torch.int32)
    pools = [torch.zeros(num_pages, page_size, Hkv, D, dtype=k.dtype, device=k.device) for _ in range(2)]
    n = 0
    for b in range(B):
        ids = perm[n:n + used[b]]
        n += used[b]
        table[b, :used[b]] = torch.tensor(ids, dtype=torch.int32)
        if ids:
            idx = torch.tensor(ids, device=k.device)
            for pool, x in zip(pools, (k, v)):
                pool[idx] = x[b, :, :used[b] * page_size].reshape(Hkv, used[b], page_size, D).permute(1, 2, 0, 3)
    return pools[0], pools[1], table.to(k.device)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None)
    ap.add_argument("--small", action="store_true")
    args = ap.parse_args()

    import numpy as np
    import torch
    from leetcuda_b200 import flash_attn

    assert torch.cuda.is_available(), "this benchmark needs a CUDA device"
    torch.manual_seed(0)
    rng = np.random.default_rng(0)
    gen = torch.Generator().manual_seed(0)

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
        pools = {ps: paginate(k, v, lk, ps, gen) for ps in PAGE_SIZES}
        kg, vg = torch.empty_like(k), torch.empty_like(v)
        kp16, vp16, t16 = pools[16]
        flat = t16.clamp(min=0).long()   # gathering reads every table slot; -1 entries fall on page 0 (masked)

        def gather_seqlens():
            for pool, out in ((kp16, kg), (vp16, vg)):
                out.copy_(pool[flat].reshape(B, Nk, Hkv, D).transpose(1, 2))
            flash_attn.fmha_fwd(q, kg, vg, o, causal=causal, num_splits=0, seqlens_q=tq, seqlens_k=tk)

        def paged(ps):
            kp, vp, t = pools[ps]
            return lambda: flash_attn.fmha_fwd(q, kp, vp, o, causal=causal, num_splits=0, seqlens_q=tq, seqlens_k=tk,
                                               block_table=t)

        runs = {f"paged/{ps}": paged(ps) for ps in PAGE_SIZES}
        runs["seqlens"] = lambda: flash_attn.fmha_fwd(q, k, v, o, causal=causal, num_splits=0, seqlens_q=tq,
                                                      seqlens_k=tk)
        runs["gather+seqlens"] = gather_seqlens
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
               "work": work, "pool_pages": {ps: pools[ps][0].shape[0] for ps in PAGE_SIZES}}
        for n in runs:
            med = statistics.median(ms[n])
            row[n] = {"ms_median": med, "ms_min": min(ms[n]), "ms_max": max(ms[n]),
                      f"{unit}_median": work / (med * 1e-3) / scale, f"{unit}_min": work / (max(ms[n]) * 1e-3) / scale,
                      f"{unit}_max": work / (min(ms[n]) * 1e-3) / scale}
        result["rows"].append(row)
        del q, k, v, o, pools, kg, vg, kp16, vp16, t16, flat
        torch.cuda.empty_cache()
    text = json.dumps(result)
    print(text)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(text + "\n")


if __name__ == "__main__":
    main()
