#!/usr/bin/env python
"""KV-cache append with rotary: the one-call decode step against the torch path it replaces, and the append alone
against HBM bandwidth.

    python tools/bench_kvcache.py [--reps 7] [--steps 20] [--out FILE] [--small]

Prints one JSON object (and writes it to FILE if given).  The card's name, power limit and max SM clock are read in
the same run.  Timing: CUDA events around `steps` back-to-back calls; the variants of a shape are timed alternately,
`reps` times each, and the median with the min .. max spread is reported.
Decode rows (kvcache_ref.BENCH_DECODE: B32 H32 Hkv8 D128, one new token per sequence at Lk_b seeded in [256, 8192],
NeoX rotary over all 128 columns, paged pools of 16- and 256-key pages, fp16 or e4m3 with k_scale = v_scale = 0.5,
num_splits = 0):
  fused      flash_attn.fmha_fwd_kvcache: one append launch, then the paged attention call
  torch      the path it replaces: torch rotary on q and k (fp32, rounded to fp16), torch quantisation to e4m3, an
             index_put of the new rows through the block table, then the same attention call
  attention  the attention call alone on the appended cache: the floor of both
Append rows (kvcache_ref.BENCH_APPEND: B4 Hkv8 D128, 2048 new tokens per sequence into a dense cache at Lk_b seeded in
[256, 8192], NeoX rotary): flash_attn.kvcache_append alone, with GB/s of the bytes it must move (k and v read in fp16,
the cache rows written in fp16 or e4m3, the cos / sin rows of the positions read once) against the H100 SXM's
3.35 TB/s.  --small runs tiny shapes (argument parsing and byte counts, not a measurement).
"""
from __future__ import annotations

import argparse
import json
import statistics
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parents[1] / "tests"))
sys.path.insert(0, str(Path(__file__).resolve().parent))

import kvcache_ref as K  # noqa: E402

SMALL_DECODE = [("decode p16 fp16", 4, 4, 2, 128, 1, 16, "fp16"), ("decode p16 e4m3", 4, 4, 2, 128, 1, 16, "e4m3")]
SMALL_APPEND = [("prefill append fp16", 2, 2, 128, 64, "fp16"), ("prefill append e4m3", 2, 2, 128, 64, "e4m3")]
HBM = 3.35e12
SCALE = 0.5


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None)
    ap.add_argument("--small", action="store_true")
    args = ap.parse_args()

    import torch
    from bench_attn_paged import card
    from leetcuda_b200 import flash_attn

    assert torch.cuda.is_available(), "this benchmark needs a CUDA device"
    torch.manual_seed(0)
    max_len = 512 if args.small else 8192

    def time_ms(fn, steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / steps

    def timed(runs):
        for fn in runs.values():
            for _ in range(3):
                fn()
        ms = {n: [] for n in runs}
        for _ in range(args.reps):
            for n, fn in runs.items():   # alternated: every repetition times each variant once
                ms[n].append(time_ms(fn, args.steps))
        return {n: {"ms_median": statistics.median(v), "ms_min": min(v), "ms_max": max(v)} for n, v in ms.items()}

    result = {"card": card(), "reps": args.reps, "steps": args.steps, "decode": [], "append": []}
    for index, (name, B, H, Hkv, D, n_new, ps, cache) in enumerate(SMALL_DECODE if args.small else K.BENCH_DECODE):
        lk = [min(x, max_len - n_new) for x in K.bench_lengths(B, index)]
        e4m3 = cache == "e4m3"
        dt = torch.float8_e4m3fn if e4m3 else torch.float16
        mp = max_len // ps
        num_pages = B * mp
        table = torch.randperm(num_pages, device="cuda").view(B, mp).int()
        kc = torch.randn(num_pages, ps, Hkv, D, device="cuda").to(dt)
        vc = torch.randn(num_pages, ps, Hkv, D, device="cuda").to(dt)
        cos, sin = (x.cuda() for x in K.tables(mp * ps + n_new, D))
        q = torch.randn(B, H, n_new, D, device="cuda").half()
        k = torch.randn(B, Hkv, n_new, D, device="cuda").half()
        v = torch.randn(B, Hkv, n_new, D, device="cuda").half()
        o = torch.empty_like(q)
        cl = torch.tensor(lk, dtype=torch.int32, device="cuda")
        lens1 = cl + n_new
        sc = dict(k_scale=SCALE, v_scale=SCALE) if e4m3 else {}
        attn = dict(num_splits=0, seqlens_k=lens1, block_table=table, **sc)
        bidx = torch.arange(B, device="cuda")

        def fused():
            flash_attn.fmha_fwd_kvcache(q, kc, vc, o, k, v, cl, block_table=table, rotary_cos=cos, rotary_sin=sin,
                                        num_splits=0, **sc)

        def torch_path():
            pos = cl.long()
            c, s = cos[pos][:, None, None, :], sin[pos][:, None, None, :]

            def rot(x):
                x0, x1 = x.float().chunk(2, dim=-1)
                return torch.cat((x0 * c - x1 * s, x0 * s + x1 * c), dim=-1).half()
            qr, kr, vr = rot(q), rot(k), v
            if e4m3:
                kr = (kr.float() / SCALE).clamp(-448, 448).to(torch.float8_e4m3fn)
                vr = (vr.float() / SCALE).clamp(-448, 448).to(torch.float8_e4m3fn)
            page, row = table[bidx, pos // ps].long(), pos % ps
            bits = (lambda x: x.view(torch.uint8)) if e4m3 else (lambda x: x)
            bits(kc)[page, row] = bits(kr)[:, :, 0]
            bits(vc)[page, row] = bits(vr)[:, :, 0]
            flash_attn.fmha_fwd(qr, kc, vc, o, **attn)

        def attention():
            flash_attn.fmha_fwd(q, kc, vc, o, **attn)

        row = {"shape": f"{name} B{B} H{H} Hkv{Hkv} D{D} n_new{n_new} pages{ps}", "lengths": f"Lk in [{min(lk)}, "
               f"{max(lk)}]", **timed({"fused": fused, "torch": torch_path, "attention": attention})}
        row["torch_over_fused"] = row["torch"]["ms_median"] / row["fused"]["ms_median"]
        row["fused_minus_attention_us"] = 1e3 * (row["fused"]["ms_median"] - row["attention"]["ms_median"])
        result["decode"].append(row)
        del kc, vc, q, k, v, o
        torch.cuda.empty_cache()

    for index, (name, B, Hkv, D, n_new, cache) in enumerate(SMALL_APPEND if args.small else K.BENCH_APPEND):
        lk = [min(x, max_len) for x in K.bench_lengths(B, 10 + index)]
        e4m3 = cache == "e4m3"
        dt = torch.float8_e4m3fn if e4m3 else torch.float16
        Nk = max_len + n_new
        kc = torch.zeros(B, Hkv, Nk, D, device="cuda").to(dt)
        vc = torch.zeros_like(kc)
        k = torch.randn(B, Hkv, n_new, D, device="cuda").half()
        v = torch.randn(B, Hkv, n_new, D, device="cuda").half()
        cos, sin = (x.cuda() for x in K.tables(Nk + n_new, D))
        cl = torch.tensor(lk, dtype=torch.int32, device="cuda")
        sc = dict(k_scale=SCALE, v_scale=SCALE) if e4m3 else {}
        nbytes = K.append_bytes(B, Hkv, D, n_new, cache) + B * n_new * D * 4   # + cos, sin rows (D / 2 fp32 each)
        t = timed({"append": lambda: flash_attn.kvcache_append(k, v, kc, vc, cl, rotary_cos=cos, rotary_sin=sin,
                                                               **sc)})["append"]
        gbs = nbytes / (t["ms_median"] * 1e-3) / 1e9
        result["append"].append({"shape": f"{name} B{B} Hkv{Hkv} D{D} n_new{n_new}", "bytes": nbytes, **t,
                                 "gbs_median": gbs, "gbs_min": nbytes / (t["ms_max"] * 1e-3) / 1e9,
                                 "gbs_max": nbytes / (t["ms_min"] * 1e-3) / 1e9, "of_3350_gbs": gbs * 1e9 / HBM})
        del kc, vc, k, v
        torch.cuda.empty_cache()
    text = json.dumps(result)
    print(text)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(text + "\n")


if __name__ == "__main__":
    main()
