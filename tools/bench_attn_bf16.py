#!/usr/bin/env python
"""bf16 attention against the same calls in fp16 and against torch SDPA in bf16.

    python tools/bench_attn_bf16.py [--reps 7] [--steps 20] [--out FILE] [--small]

Prints one JSON object (and writes it to FILE if given).  The card's name, power limit and max SM clock are read in
the same run.  Timing: CUDA events around `steps` back-to-back calls; the variants of a shape are timed alternately,
`reps` times each, and the median with the min .. max spread is reported.
Variants:
  bf16          flash_attn.fmha_fwd on bf16 tensors (b200_fmha_fwd_bf16_seqlens / _paged; a dense call runs the
                per-sequence-length kernel with null length arrays)
  fp16          the same call on fp16 tensors (dense: attn_fwd_kernel; seqlens / paged: their fp16 kernels)
  fp16 seqlens  dense rows only: b200_fmha_fwd_f16_seqlens with null length arrays, i.e. the fp16 kernel the bf16
                call mirrors, which separates the cost of the element type from that of the kernel body
  sdpa bf16     torch.nn.functional.scaled_dot_product_attention in bf16 (enable_gqa for Hkv < H; seqlens / paged rows
                on the padded cache with a boolean mask of the keys below each sequence's length)
Shapes: B4 H32 N4096 at D128 and D64, causal or not; decode B8 H32 Hkv8 Nq1 Nk8192 D128 with num_splits=0; the decode
batch B32 H32 Hkv8 D128 of tools/bench_attn_seqlens.py (Lk_b seeded in [256, 8192]) as a seqlens call and as a paged
call over 256-key pages (tools/bench_attn_paged.py's page placement).  Dense rows report TFLOPS (4 B H Nq Nk D, halved
when causal), decode rows GB/s of the visible K and V bytes.  --small runs tiny shapes (not a measurement).
"""
from __future__ import annotations

import argparse
import json
import statistics
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parent))

# (name, B, H, Hkv, Nq, Nk, D, causal, kind): kind "dense", "decode" (num_splits=0), "seqlens" or "paged"
SHAPES = [
    ("dense", 4, 32, 32, 4096, 4096, 128, False, "dense"),
    ("dense", 4, 32, 32, 4096, 4096, 128, True, "dense"),
    ("dense", 4, 32, 32, 4096, 4096, 64, False, "dense"),
    ("dense", 4, 32, 32, 4096, 4096, 64, True, "dense"),
    ("decode", 8, 32, 8, 1, 8192, 128, False, "decode"),
    ("seqlens decode", 32, 32, 8, 1, 8192, 128, False, "seqlens"),
    ("paged decode", 32, 32, 8, 1, 8192, 128, False, "paged"),
]
SMALL = [("dense", 1, 4, 4, 256, 256, 64, True, "dense"), ("decode", 2, 4, 2, 1, 1024, 128, False, "decode"),
         ("seqlens decode", 4, 4, 2, 1, 512, 128, False, "seqlens"),
         ("paged decode", 4, 4, 2, 1, 512, 128, False, "paged")]
PAGE_SIZE = 256
LK_RANGE = (256, 8192)   # tools/bench_attn_seqlens.py's decode lengths


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None)
    ap.add_argument("--small", action="store_true")
    args = ap.parse_args()

    import numpy as np
    import torch
    import torch.nn.functional as F
    from bench_attn_paged import card, paginate
    from leetcuda_b200 import _capi, flash_attn

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
    for name, B, H, Hkv, Nq, Nk, D, causal, kind in (SMALL if args.small else SHAPES):
        lo, hi = (16, Nk) if args.small else LK_RANGE
        lk = [int(x) for x in rng.integers(lo, hi + 1, size=B)] if kind in ("seqlens", "paged") else [Nk] * B
        q = torch.randn(B, H, Nq, D, device="cuda")
        k, v = (torch.randn(B, Hkv, Nk, D, device="cuda") for _ in range(2))
        data = {}
        for dt in (torch.bfloat16, torch.float16):
            qd, kd, vd = q.to(dt), k.to(dt), v.to(dt)
            data[dt] = (qd, kd, vd, torch.empty_like(qd))
        tq = torch.tensor([Nq] * B, dtype=torch.int32, device="cuda")
        tk = torch.tensor(lk, dtype=torch.int32, device="cuda")
        runs = {}
        splits = 0 if kind != "dense" else 1
        if kind == "paged":
            pages = {dt: paginate(data[dt][1], data[dt][2], lk, PAGE_SIZE, torch.Generator().manual_seed(1))
                     for dt in data}
            for dt, label in ((torch.bfloat16, "bf16"), (torch.float16, "fp16")):
                qd, _, _, od = data[dt]
                kp, vp, t = pages[dt]
                runs[label] = (lambda qd=qd, kp=kp, vp=vp, od=od, t=t: flash_attn.fmha_fwd(
                    qd, kp, vp, od, num_splits=0, seqlens_q=tq, seqlens_k=tk, block_table=t))
        else:
            for dt, label in ((torch.bfloat16, "bf16"), (torch.float16, "fp16")):
                qd, kd, vd, od = data[dt]
                lens = dict(seqlens_q=tq, seqlens_k=tk) if kind == "seqlens" else {}
                runs[label] = (lambda qd=qd, kd=kd, vd=vd, od=od, lens=lens: flash_attn.fmha_fwd(
                    qd, kd, vd, od, causal=causal, num_splits=splits, **lens))
        if kind == "dense":
            qd, kd, vd, od = data[torch.float16]
            fn16 = _capi.lib().b200_fmha_fwd_f16_seqlens
            stream = _capi.raw_stream(qd.device.index)

            def f16_seqlens(qd=qd, kd=kd, vd=vd, od=od):
                _capi.check(fn16(qd.data_ptr(), kd.data_ptr(), vd.data_ptr(), od.data_ptr(), None, None, None, B, H,
                                 Hkv, Nq, Nk, D, int(causal), 1, 0.0, stream), "fmha_fwd_f16_seqlens")
            runs["fp16 seqlens"] = f16_seqlens
        qb, kb, vb, _ = data[torch.bfloat16]
        mask = None
        if kind in ("seqlens", "paged"):
            mask = (torch.arange(Nk, device="cuda")[None, :] < tk[:, None])[:, None, None, :]
        runs["sdpa bf16"] = (lambda: F.scaled_dot_product_attention(qb, kb, vb, attn_mask=mask,
                                                                    is_causal=causal and mask is None,
                                                                    enable_gqa=Hkv != H))
        for fn in runs.values():
            for _ in range(3):
                fn()
        ms = {n: [] for n in runs}
        for _ in range(args.reps):
            for n, fn in runs.items():   # alternated: every repetition times each variant once
                ms[n].append(time_ms(fn, args.steps))
        if kind == "dense":
            work, unit, scale = 4.0 * B * H * Nq * Nk * D / (2 if causal else 1), "tflops", 1e12
        else:
            work, unit, scale = 2.0 * Hkv * D * 2 * sum(lk), "kv_gbs", 1e9
        row = {"shape": f"{name} B{B} H{H} Hkv{Hkv} Nq{Nq} Nk{Nk} D{D}" + (" causal" if causal else "")
                        + (f" pages{PAGE_SIZE}" if kind == "paged" else ""),
               "lengths": f"Lk in [{lo}, {hi}]" if kind in ("seqlens", "paged") else "full", "work": work}
        for n in runs:
            med = statistics.median(ms[n])
            row[n] = {"ms_median": med, "ms_min": min(ms[n]), "ms_max": max(ms[n]),
                      f"{unit}_median": work / (med * 1e-3) / scale}
        b, f = row["bf16"], row["fp16"]
        row["bf16_within_fp16_spread"] = f["ms_min"] <= b["ms_median"] <= f["ms_max"]
        row["bf16_over_fp16"] = b["ms_median"] / f["ms_median"]
        result["rows"].append(row)
        del q, k, v, data, runs, qb, kb, vb, mask
        torch.cuda.empty_cache()
    text = json.dumps(result)
    print(text)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(text + "\n")


if __name__ == "__main__":
    main()
