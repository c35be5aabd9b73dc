#!/usr/bin/env python
"""The GEMM kernel at the shapes bench.py runs it, with cuBLAS in the same process.

    python tools/bench_hgemm.py [--steps 20] [--out FILE]

Prints one JSON object (and writes it to FILE if given).  The card's name, power limit and max SM clock are read in
the same run, and each row samples the SM clock while it is timed (bench.py's ClockSampler).  The library is the one
leetcuda_b200 loads, so LEETCUDA_B200_LIB=<path> times another build of it: to compare two builds, run this script
once per build, alternately, in separate processes.
Rows (CUDA events around `steps` back-to-back calls, after 3 untimed ones):
  nn_8192      bench.py's primary call: hgemm_mma_m16n8k16_mma2x4_warp4x4x2_stages_dsmem_swizzle, 8192^3, operands
               rotating over 3 sets (each > 50 MB of L2), and torch.matmul on the same operands
  nn_16384     the same op at 16384^3 (2 sets), bench.py's strong_scaling_n1 row
  tf32_8192    sgemm_tf32(round_inputs=False) at 8192^3 (2 sets): the [K,N] -> [N,K] transpose and the TF32 GEMM,
               bench.py's TF32 kernel_ms
  nn_ragged    2600 x 2344 x 4096 (3 sets): 21 m-tiles, so the last two-CTA cluster has an m-tile past M
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

OP = "hgemm_mma_m16n8k16_mma2x4_warp4x4x2_stages_dsmem_swizzle"


def card():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else f"unknown ({r.stderr.strip()})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    from bench import ClockSampler, cuda_time_ms, settle
    from leetcuda_b200 import _capi, hgemm, sgemm

    assert torch.cuda.is_available(), "this benchmark needs a CUDA device"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    op = getattr(hgemm, OP)
    sync = torch.cuda.synchronize
    result = {"card": card(), "lib": str(_capi.lib()._name), "steps": args.steps, "rows": {}}

    def timed(fn, steps):
        for i in range(3):
            fn(i)
        settle()
        with ClockSampler(0) as clk:
            ms = cuda_time_ms(fn, steps, sync) / steps
        return ms, clk.summary()

    def hgemm_row(name, M, N, K, nsets, steps, vendor=False):
        torch.manual_seed(1234)
        A = [torch.randn(M, K, device=dev, dtype=torch.half) for _ in range(nsets)]
        B = [torch.randn(K, N, device=dev, dtype=torch.half) for _ in range(nsets)]
        C = [torch.empty(M, N, device=dev, dtype=torch.half) for _ in range(nsets)]
        ms, clk = timed(lambda i: op(A[i % nsets], B[i % nsets], C[i % nsets], 2, True, 2048), steps)
        fl = 2.0 * M * N * K
        row = {"shape": [M, N, K], "ms": ms, "tflops": fl / (ms * 1e-3) / 1e12, "clocks": clk}
        if vendor:
            vms, vclk = timed(lambda i: torch.matmul(A[i % nsets], B[i % nsets], out=C[i % nsets]), steps)
            row["cublas"] = {"ms": vms, "tflops": fl / (vms * 1e-3) / 1e12, "clocks": vclk}
        result["rows"][name] = row
        del A, B, C
        torch.cuda.empty_cache()

    hgemm_row("nn_8192", 8192, 8192, 8192, 3, args.steps, vendor=True)
    hgemm_row("nn_16384", 16384, 16384, 16384, 2, max(3, min(args.steps, 10)))
    torch.manual_seed(1234)
    sa = [torch.randn(8192, 8192, device=dev) for _ in range(2)]
    sb = [torch.randn(8192, 8192, device=dev) for _ in range(2)]
    sc = [torch.empty(8192, 8192, device=dev) for _ in range(2)]
    for i in range(2):
        sgemm.tf32_round_(sa[i])
        sgemm.tf32_round_(sb[i])
    ms, clk = timed(lambda i: sgemm.sgemm_tf32(sa[i % 2], sb[i % 2], sc[i % 2], round_inputs=False), args.steps)
    result["rows"]["tf32_8192"] = {"shape": [8192, 8192, 8192], "ms": ms, "tflops": 2.0 * 8192 ** 3 / (ms * 1e-3) / 1e12,
                                   "clocks": clk}
    del sa, sb, sc
    torch.cuda.empty_cache()
    hgemm_row("nn_ragged", 2600, 2344, 4096, 3, 4 * args.steps)

    text = json.dumps(result)
    print(text)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(text + "\n")


if __name__ == "__main__":
    main()
