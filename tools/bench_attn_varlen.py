#!/usr/bin/env python
"""Packed variable-length attention: the varlen call against the seqlens / paged call on padded copies and against
padding, calling and unpadding around it.

    python tools/bench_attn_varlen.py [--reps 7] [--steps 20] [--out FILE] [--small]

Prints one JSON object (and writes it to FILE if given).  The card's name, power limit and max SM clock are read in
the same run.  Timing: CUDA events around `steps` back-to-back calls; the variants of a shape are timed alternately,
`reps` times each, and the median with the min .. max spread is reported.  Lengths are seeded draws (lengths()).
Variants:
  varlen          fmha_varlen_fwd on token-major [total, H, D] tensors (paged K/V: block_table=, seqused_k=)
  padded          fmha_fwd(..., num_splits=1, seqlens_q=, seqlens_k=) (paged: block_table=) on padded [B, H, N, D]
                  copies made outside the timing: the same kernel work without the token-major addressing
  pad+call+unpad  what a caller with packed tokens does today, all inside the timing: scatter Q (and K, V when they
                  are packed) into the padded buffers, the padded call, gather O back into [total_q, H, D]
Every row reports TFLOPS of 4 H D x (visible (query, key) pairs).  --small runs tiny shapes (argument parsing and
FLOP counts, not a measurement).
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

# (name, B, H, Hkv, D, causal, (lo, hi) of Lk_b, Lq_b (None: Lq_b = Lk_b), page_size (None: packed K/V))
SHAPES = [
    ("causal prefill", 8, 32, 8, 128, True, (512, 4096), None, None),
    ("packed training", 16, 32, 32, 128, True, (128, 8192), None, None),
    ("chunked prefill", 4, 32, 8, 128, True, (4096, 32768), 2048, 256),
]
SMALL = [("causal prefill", 3, 4, 2, 64, True, (16, 300), None, None),
         ("chunked prefill", 2, 4, 2, 64, True, (256, 700), 64, 16)]


def lengths(index, shapes=None):
    """(Lq_b, Lk_b) of shape `index`: Lk_b drawn from default_rng(index) in [lo, hi]."""
    import numpy as np
    _, B, _, _, _, _, (lo, hi), nq, _ = (shapes or SHAPES)[index]
    lk = [int(x) for x in np.random.default_rng(index).integers(lo, hi + 1, size=B)]
    return ([nq] * B if nq else list(lk)), lk


def card():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else f"unknown ({r.stderr.strip()})"


def visible_pairs(lq, lk, causal):
    return sum(sum(max(0, min(k, i + k - q + 1)) for i in range(q)) if causal else q * k for q, k in zip(lq, lk))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None)
    ap.add_argument("--small", action="store_true")
    args = ap.parse_args()

    import torch
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

    def cu(lens):
        return torch.tensor([0] + list(torch.tensor(lens).cumsum(0).tolist()), dtype=torch.int32, device="cuda")

    def rows_of(lens, n):
        """Row of every packed token in a padded [B * n] token-major buffer."""
        return torch.cat([b * n + torch.arange(x) for b, x in enumerate(lens)]).cuda()

    shapes = SMALL if args.small else SHAPES
    result = {"card": card(), "reps": args.reps, "steps": args.steps, "rows": []}
    for index, (name, B, H, Hkv, D, causal, (lo, hi), nq, ps) in enumerate(shapes):
        lq, lk = lengths(index, shapes)
        mq, mk = max(lq), max(lk)
        tq, tk = sum(lq), sum(lk)
        q = torch.randn(tq, H, D, device="cuda", dtype=torch.half)
        o = torch.empty_like(q)
        cq, ck = cu(lq), cu(lk)
        sq, sk = (torch.tensor(x, dtype=torch.int32, device="cuda") for x in (lq, lk))
        qrows, krows = rows_of(lq, mq), rows_of(lk, mk)
        qpad = torch.zeros(B * mq, H, D, device="cuda", dtype=torch.half)
        qpad[qrows] = q
        qp = qpad.view(B, mq, H, D).transpose(1, 2).contiguous()
        op = torch.empty_like(qp)
        if ps is None:
            k, v = (torch.randn(tk, Hkv, D, device="cuda", dtype=torch.half) for _ in range(2))
            kpad = [torch.zeros(B * mk, Hkv, D, device="cuda", dtype=torch.half) for _ in range(2)]
            for buf, x in zip(kpad, (k, v)):
                buf[krows] = x
            kp, vp = (buf.view(B, mk, Hkv, D).transpose(1, 2).contiguous() for buf in kpad)

            def varlen():
                flash_attn.fmha_varlen_fwd(q, k, v, o, cq, ck, mq, mk, causal=causal)

            def padded():
                flash_attn.fmha_fwd(qp, kp, vp, op, causal=causal, seqlens_q=sq, seqlens_k=sk)

            def pad_call_unpad():
                for buf, x, pad, n, rows in ((qpad, q, qp, mq, qrows), (kpad[0], k, kp, mk, krows),
                                             (kpad[1], v, vp, mk, krows)):
                    buf[rows] = x
                    pad.copy_(buf.view(B, n, -1, D).transpose(1, 2))
                flash_attn.fmha_fwd(qp, kp, vp, op, causal=causal, seqlens_q=sq, seqlens_k=sk)
                o.copy_(op.transpose(1, 2).reshape(B * mq, H, D)[qrows])
        else:
            pages = [-(-x // ps) for x in lk]
            num_pages = (sum(pages) * 5 + 3) // 4
            perm = torch.randperm(num_pages, generator=torch.Generator().manual_seed(index)).tolist()
            table = torch.full((B, -(-mk // ps)), -1, dtype=torch.int32)
            n = 0
            for b in range(B):
                table[b, :pages[b]] = torch.tensor(perm[n:n + pages[b]], dtype=torch.int32)
                n += pages[b]
            table = table.cuda()
            kc, vc = (torch.randn(num_pages, ps, Hkv, D, device="cuda", dtype=torch.half) for _ in range(2))

            def varlen():
                flash_attn.fmha_varlen_fwd(q, kc, vc, o, cq, None, mq, 0, causal=causal, block_table=table,
                                           seqused_k=sk)

            def padded():
                flash_attn.fmha_fwd(qp, kc, vc, op, causal=causal, seqlens_q=sq, seqlens_k=sk, block_table=table)

            def pad_call_unpad():
                qpad[qrows] = q
                qp.copy_(qpad.view(B, mq, H, D).transpose(1, 2))
                flash_attn.fmha_fwd(qp, kc, vc, op, causal=causal, seqlens_q=sq, seqlens_k=sk, block_table=table)
                o.copy_(op.transpose(1, 2).reshape(B * mq, H, D)[qrows])

        runs = {"varlen": varlen, "padded": padded, "pad+call+unpad": pad_call_unpad}
        for fn in runs.values():
            for _ in range(3):
                fn()
        ms = {n: [] for n in runs}
        for _ in range(args.reps):
            for n, fn in runs.items():   # alternated: every repetition times each variant once
                ms[n].append(time_ms(fn, args.steps))
        work = 4.0 * H * D * visible_pairs(lq, lk, causal)
        row = {"shape": f"{name} B{B} H{H} Hkv{Hkv} D{D}" + (" causal" if causal else "")
               + (f" pages of {ps}" if ps else ""),
               "lengths": f"Lk in [{lo}, {hi}]" + (f", Lq = {nq}" if nq else ", Lq = Lk"),
               "total_q": tq, "total_k": tk, "work": work}
        for n in runs:
            med = statistics.median(ms[n])
            row[n] = {"ms_median": med, "ms_min": min(ms[n]), "ms_max": max(ms[n]),
                      "tflops_median": work / (med * 1e-3) / 1e12, "tflops_min": work / (max(ms[n]) * 1e-3) / 1e12,
                      "tflops_max": work / (min(ms[n]) * 1e-3) / 1e12}
        result["rows"].append(row)
        del q, o, qpad, qp, op, runs
        torch.cuda.empty_cache()
    text = json.dumps(result)
    print(text)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(text + "\n")


if __name__ == "__main__":
    main()
