#!/usr/bin/env python
"""fp8 (e4m3) scaled GEMM: hgemm.scaled_mm against torch._scaled_mm (cuBLAS) and this library's fp16 GEMM on the
same shapes.

    python tools/bench_gemm_fp8.py [--reps 7] [--steps 20] [--out FILE] [--small]

Prints one JSON object (and writes it to FILE if given).  The card's name, power limit and max SM clock are read in
the same run.  Timing: CUDA events around `steps` back-to-back calls; the variants of a row are timed alternately,
`reps` times each, and the median with the min .. max spread is reported, in TFLOP/s of 2 M N K.
Rows (M, N, K; bf16 C unless noted; A [M,K] and the [N,K] weight seeded randn quantised to e4m3):
  8192^3 with tensor, row and block scales; 2600 x 2344 x 4096 (tensor); a 4096-token batch against 28672 x 8192 and
  8192 x 28672 weights (row scales, the Llama-3 70B MLP shapes).
Variants: ours (hgemm.scaled_mm); torch._scaled_mm with use_fast_accum False and True, where torch takes the recipe;
fp16 (hgemm.hgemm, TN, fp16 inputs of the same shape).  --small runs tiny shapes (not a measurement).
"""
from __future__ import annotations

import argparse
import json
import statistics
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parent))

ROWS = [
    ("8192^3 tensor", (8192, 8192, 8192), "tensor"),
    ("8192^3 row", (8192, 8192, 8192), "row"),
    ("8192^3 block", (8192, 8192, 8192), "block"),
    ("2600x2344x4096 tensor", (2600, 2344, 4096), "tensor"),
    ("4096 tok x 28672x8192 row", (4096, 28672, 8192), "row"),
    ("4096 tok x 8192x28672 row", (4096, 8192, 28672), "row"),
]
SMALL = [("small tensor", (256, 256, 256), "tensor"), ("small block", (300, 264, 384), "block")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None)
    ap.add_argument("--small", action="store_true")
    args = ap.parse_args()

    import torch
    from bench_attn_paged import card
    from leetcuda_b200 import hgemm

    assert torch.cuda.is_available(), "this benchmark needs a CUDA device"
    torch.manual_seed(0)
    dev = "cuda"

    def time_ms(fn, steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / steps

    def scales(recipe, M, N, K):
        kbs, nbs = -(-K // 128), -(-N // 128)
        if recipe == "tensor":
            return torch.full((1,), 0.5, device=dev), torch.full((1,), 0.25, device=dev)
        if recipe == "row":
            return torch.rand(M, device=dev) + 0.5, torch.rand(N, device=dev) + 0.5
        return (torch.rand(kbs, M, device=dev) + 0.5).t(), torch.rand(nbs, kbs, device=dev) + 0.5

    def torch_call(a, b, sa, sb, recipe, c, fast):
        M, N = a.shape[0], b.shape[1]
        if recipe == "tensor":
            sa_t, sb_t = sa.reshape(()), sb.reshape(())
        elif recipe == "row":
            sa_t, sb_t = sa.reshape(M, 1), sb.reshape(1, N)
        else:
            sa_t, sb_t = sa, sb.t()
        try:
            torch._scaled_mm(a, b, sa_t, sb_t, out_dtype=c.dtype, use_fast_accum=fast)
        except (RuntimeError, TypeError, NotImplementedError) as e:
            return None, str(e).splitlines()[0][:160]
        return (lambda: torch._scaled_mm(a, b, sa_t, sb_t, out_dtype=c.dtype, use_fast_accum=fast)), None

    out = {"card": card(), "steps": args.steps, "reps": args.reps, "unit": "TFLOP/s (2MNK), median (min .. max)",
           "rows": []}
    for name, (M, N, K), recipe in (SMALL if args.small else ROWS):
        a = torch.randn(M, K, device=dev).to(torch.float8_e4m3fn)
        w = torch.randn(N, K, device=dev).to(torch.float8_e4m3fn)
        b = w.t()
        sa, sb = scales(recipe, M, N, K)
        c = torch.empty(M, N, dtype=torch.bfloat16, device=dev)
        a16, w16 = a.to(torch.float16), w.to(torch.float16)
        c16 = torch.empty(M, N, dtype=torch.float16, device=dev)
        variants = {"ours": lambda: hgemm.scaled_mm(a, b, c, sa, sb, scale_recipe=recipe),
                    "fp16": lambda: hgemm.hgemm(a16, w16.view(K, N), c16, tn=True)}
        notes = {}
        for fast in (False, True):
            fn, why = torch_call(a, b, sa, sb, recipe, c, fast)
            key = f"torch_scaled_mm_fast_accum_{fast}"
            if fn is None:
                notes[key] = why
            else:
                variants[key] = fn
        for fn in variants.values():       # warm-up: modules, cuBLAS heuristics, tensor maps
            fn()
            time_ms(fn, 3)
        times = {k: [] for k in variants}
        for _ in range(args.reps):
            for k, fn in variants.items():
                times[k].append(time_ms(fn, args.steps))
        flop = 2.0 * M * N * K
        row = {"name": name, "M": M, "N": N, "K": K, "recipe": recipe}
        for k, ts in times.items():
            tf = sorted(flop / (t * 1e-3) / 1e12 for t in ts)
            row[k] = f"{statistics.median(tf):.0f} ({tf[0]:.0f} .. {tf[-1]:.0f})"
            row[k + "_median"] = round(statistics.median(tf), 1)
        row.update({k: "not run: " + v for k, v in notes.items()})
        out["rows"].append(row)
        print(json.dumps(row), flush=True)
        del a, w, b, c, a16, w16, c16
        torch.cuda.empty_cache()
    text = json.dumps(out)
    print(text)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(text)


if __name__ == "__main__":
    main()
