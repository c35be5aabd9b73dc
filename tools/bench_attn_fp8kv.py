#!/usr/bin/env python
"""fp8 (e4m3) K/V attention against the same calls with bf16 / fp16 K and V, and against expanding the fp8 cache first.

    python tools/bench_attn_fp8kv.py [--reps 7] [--steps 20] [--out FILE] [--small]

Prints one JSON object (and writes it to FILE if given).  The card's name, power limit and max SM clock are read in
the same run.  Timing: CUDA events around `steps` back-to-back calls; the variants of a shape are timed alternately,
`reps` times each, and the median with the min .. max spread is reported.
Variants (one call each; k_scale = v_scale = 1 costs the same as any other scale):
  fp8 bf16     flash_attn.fmha_fwd with float8_e4m3fn K / V and bf16 Q / O (b200_fmha_fwd_bf16_fp8kv_seqlens / _paged)
  bf16         the same call with bf16 K / V (b200_fmha_fwd_bf16_seqlens / _paged)
  expand bf16  what a caller without fp8 K/V does: K.to(bf16), V.to(bf16) of the whole cache or pool with torch, then
               the bf16 call
  fp8 fp16     fp8 K / V with fp16 Q / O
  fp16         the same call with fp16 K / V (dense rows: the dense fp16 kernel)
Shapes (test_attn_fp8kv_gpu.BENCH_SHAPES, each with a GPU test at full size): decode B8 H32 Hkv8 Nk8192 D128 with
num_splits=0; the decode batch B32 H32 Hkv8 D128 with Lk_b seeded in [256, 8192] as a seqlens call and as paged calls
over 16- and 256-key pages; decode B4 H64 Hkv8 over a 32768-key cache; causal prefill B8 H32 Hkv8 N4096 over 256-key
pages.  Decode rows report GB/s of the K and V bytes the call reads (the visible rows of the cache, 1 byte per element
for fp8, 2 for bf16 / fp16); the prefill row TFLOPS (2 B H N^2 D, causal).  --small runs tiny shapes (not a measurement).
"""
from __future__ import annotations

import argparse
import json
import statistics
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parent))

# (name, B, H, Hkv, Nq, Nk, D, causal, kind, page_size): kind "dense" (num_splits=0 when Nq = 1), "seqlens" or "paged"
SHAPES = [
    ("dense decode", 8, 32, 8, 1, 8192, 128, False, "dense", None),
    ("seqlens decode", 32, 32, 8, 1, 8192, 128, False, "seqlens", None),
    ("paged decode p16", 32, 32, 8, 1, 8192, 128, False, "paged", 16),
    ("paged decode p256", 32, 32, 8, 1, 8192, 128, False, "paged", 256),
    ("long decode", 4, 64, 8, 1, 32768, 128, False, "dense", None),
    ("paged causal prefill", 8, 32, 8, 4096, 4096, 128, True, "paged", 256),
]
SMALL = [("dense decode", 2, 4, 2, 1, 1024, 128, False, "dense", None),
         ("seqlens decode", 4, 4, 2, 1, 512, 128, False, "seqlens", None),
         ("paged decode p16", 4, 4, 2, 1, 512, 128, False, "paged", 16),
         ("paged causal prefill", 1, 4, 2, 256, 256, 128, True, "paged", 64)]
LK_RANGE = (256, 8192)


def lengths(index, shapes=SHAPES, lk_range=LK_RANGE):
    """Lk_b of shape `index`: every key for dense and causal rows, else seeded draws in lk_range."""
    import numpy as np
    _, B, _, _, _, Nk, _, causal, kind, _ = shapes[index]
    if kind == "dense" or causal:
        return [Nk] * B
    rng = np.random.default_rng(index)
    return [int(x) for x in rng.integers(lk_range[0], lk_range[1] + 1, size=B)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None)
    ap.add_argument("--small", action="store_true")
    args = ap.parse_args()

    import torch
    from bench_attn_paged import card, paginate
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

    shapes = SMALL if args.small else SHAPES
    result = {"card": card(), "reps": args.reps, "steps": args.steps, "rows": []}
    for index, (name, B, H, Hkv, Nq, Nk, D, causal, kind, ps) in enumerate(shapes):
        lk = lengths(index, shapes, (16, Nk) if args.small else LK_RANGE)
        q = torch.randn(B, H, Nq, D, device="cuda")
        k8 = torch.randn(B, Hkv, Nk, D, device="cuda").to(torch.float8_e4m3fn)
        v8 = torch.randn(B, Hkv, Nk, D, device="cuda").to(torch.float8_e4m3fn)
        kw = dict(causal=causal, num_splits=0 if Nq == 1 else 1)
        if kind != "dense":
            kw.update(seqlens_q=torch.full((B,), Nq, dtype=torch.int32, device="cuda"),
                      seqlens_k=torch.tensor(lk, dtype=torch.int32, device="cuda"))
        if kind == "paged":
            kp, vp, table = paginate(k8.view(torch.uint8), v8.view(torch.uint8), lk, ps, torch.Generator().manual_seed(1))
            k8, v8 = kp.view(torch.float8_e4m3fn), vp.view(torch.float8_e4m3fn)
            kw["block_table"] = table
        runs = {}
        for dt, label in ((torch.bfloat16, "bf16"), (torch.float16, "fp16")):
            qd, od = q.to(dt), torch.empty(B, H, Nq, D, device="cuda", dtype=dt)
            kd, vd = k8.to(dt), v8.to(dt)
            runs["fp8 " + label] = (lambda qd=qd, od=od: flash_attn.fmha_fwd(qd, k8, v8, od, **kw))
            runs[label] = (lambda qd=qd, kd=kd, vd=vd, od=od: flash_attn.fmha_fwd(qd, kd, vd, od, **kw))
            if dt == torch.bfloat16:
                runs["expand bf16"] = (lambda qd=qd, od=od, dt=dt: flash_attn.fmha_fwd(qd, k8.to(dt), v8.to(dt), od,
                                                                                      **kw))
        for fn in runs.values():
            for _ in range(3):
                fn()
        ms = {n: [] for n in runs}
        for _ in range(args.reps):
            for n, fn in runs.items():   # alternated: every repetition times each variant once
                ms[n].append(time_ms(fn, args.steps))
        kv_elems = 2.0 * Hkv * D * sum(lk)
        row = {"shape": f"{name} B{B} H{H} Hkv{Hkv} Nq{Nq} Nk{Nk} D{D}" + (" causal" if causal else "")
                        + (f" pages{ps}" if ps else ""),
               "lengths": f"Lk in [{min(lk)}, {max(lk)}]"}
        for n in runs:
            med = statistics.median(ms[n])
            row[n] = {"ms_median": med, "ms_min": min(ms[n]), "ms_max": max(ms[n])}
            if Nq == 1:
                row[n]["kv_gbs_median"] = kv_elems * (1 if n.startswith("fp8") else 2) / (med * 1e-3) / 1e9
            else:
                row[n]["tflops_median"] = 4.0 * B * H * Nq * Nk * D / 2 / (med * 1e-3) / 1e12
        row["bf16_over_fp8_bf16"] = row["bf16"]["ms_median"] / row["fp8 bf16"]["ms_median"]
        row["fp16_over_fp8_fp16"] = row["fp16"]["ms_median"] / row["fp8 fp16"]["ms_median"]
        row["expand_over_fp8_bf16"] = row["expand bf16"]["ms_median"] / row["fp8 bf16"]["ms_median"]
        result["rows"].append(row)
        del q, k8, v8, runs, kw
        torch.cuda.empty_cache()
    text = json.dumps(result)
    print(text)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(text + "\n")


if __name__ == "__main__":
    main()
