"""Side-by-side throughput table on one H100: this library vs the reference's own kernels
(recompiled unmodified for sm_90a, oracle/_ref, where built) vs the vendor libraries, at the BASELINE shapes.
Writes side_by_side.{json,md} to $LEETCUDA_SIDE_BY_SIDE_DIR (default: the system temp directory); asserts only the weak claim "not slower than the
reference kernels it replaces".  CUDA-event timing, warm-up 3, 10 iterations each."""
import json
import os
import tempfile
from pathlib import Path

import pytest
import torch
import torch.nn.functional as F

from leetcuda_b200 import ffpa_attn, flash_attn, hgemm
from oracle.build_ref import load_prebuilt

pytestmark = pytest.mark.gpu
OUT = Path(os.environ.get("LEETCUDA_SIDE_BY_SIDE_DIR", Path(tempfile.gettempdir()) / "leetcuda_side_by_side"))
ROWS = []


def timeit(fn, iters=10, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def add(group, name, ms, flops):
    ROWS.append({"workload": group, "impl": name, "ms": ms, "tflops": flops / ms / 1e9})


def _flush():
    OUT.mkdir(parents=True, exist_ok=True)
    (OUT / "side_by_side.json").write_text(json.dumps(ROWS, indent=1))
    lines = ["| workload | implementation | ms | TFLOPS |", "|---|---|---:|---:|"]
    lines += [f"| {r['workload']} | {r['impl']} | {r['ms']:.4f} | {r['tflops']:.1f} |" for r in ROWS]
    (OUT / "side_by_side.md").write_text("\n".join(lines) + "\n")


@pytest.mark.parametrize("S", [512, 8192])
def test_hgemm_side_by_side(S):
    g = torch.Generator(device="cuda").manual_seed(0)
    a = torch.randn(S, S, device="cuda", dtype=torch.half, generator=g)
    b = torch.randn(S, S, device="cuda", dtype=torch.half, generator=g)
    bt = b.t().reshape(S, S).contiguous()
    c = torch.zeros(S, S, device="cuda", dtype=torch.half)
    fl = 2.0 * S ** 3
    grp = f"HGEMM {S}^3 fp16"
    ours_nn = timeit(lambda: hgemm.hgemm_mma_m16n8k16_mma2x4_warp4x4x2_stages_dsmem_swizzle(a, b, c, 2, True, 2048))
    add(grp, "leetcuda_b200 NN (wgmma/TMA)", ours_nn, fl)
    ours_tn = timeit(lambda: hgemm.hgemm_mma_stages_block_swizzle_tn_cute(a, bt, c, 2, True, 2048))
    add(grp, "leetcuda_b200 TN (wgmma/TMA)", ours_tn, fl)
    add(grp, "cuBLAS NN (torch.matmul)", timeit(lambda: torch.matmul(a, b, out=c)), fl)
    ref = load_prebuilt("ref_hgemm")
    best_ref = None
    if ref is not None:
        stride = 2048 if S >= 2048 else 256   # hgemm.py:198-208
        for name, bb in [("hgemm_mma_m16n8k16_mma2x4_warp4x4x2_stages_dsmem_swizzle", b),
                         ("hgemm_mma_m16n8k16_mma2x4_warp4x4x2_stages_dsmem", b),
                         ("hgemm_wmma_m16n16k16_mma4x2_warp2x4_stages_dsmem", b),
                         ("hgemm_mma_m16n8k16_mma2x4_warp4x4_stages_dsmem_tn", bt),
                         ("hgemm_mma_stages_block_swizzle_tn_cute", bt)]:
            for st in (2, 3):
                ms = timeit(lambda: getattr(ref, name)(a, bb, c, st, True, stride))
                add(grp, f"reference {name} stages={st} (sm_90a rebuild)", ms, fl)
                best_ref = ms if best_ref is None else min(best_ref, ms)
        ref.init_cublas_handle()
        add(grp, "reference hgemm_cublas_tensor_op_nn (COMPUTE_16F)", timeit(lambda: ref.hgemm_cublas_tensor_op_nn(a, b, c)), fl)
        ref.destroy_cublas_handle()
    _flush()
    if best_ref is not None and S >= 8192:
        assert ours_nn < best_ref and ours_tn < best_ref


def test_attention_side_by_side():
    B, H, N, D = 4, 32, 4096, 128
    g = torch.Generator(device="cuda").manual_seed(0)
    q, k, v = (torch.randn(B, H, N, D, device="cuda", dtype=torch.half, generator=g) for _ in range(3))
    o = torch.zeros_like(q)
    fl = 4.0 * B * H * N * N * D
    grp = f"FA-2 fwd B{B} H{H} N{N} D{D} fp16"
    ours = timeit(lambda: flash_attn.flash_attn_mma_stages_split_q_shared_qkv(q, k, v, o, 2))
    add(grp, "leetcuda_b200 fused wgmma FMHA", ours, fl)
    from torch.nn.attention import SDPBackend, sdpa_kernel
    for be in (SDPBackend.CUDNN_ATTENTION, SDPBackend.FLASH_ATTENTION, SDPBackend.EFFICIENT_ATTENTION):
        try:
            with sdpa_kernel(be):
                add(grp, f"SDPA {be.name}", timeit(lambda: F.scaled_dot_product_attention(q, k, v)), fl)
        except Exception:
            pass
    try:
        from flash_attn import flash_attn_func
        fq, fk, fv = (x.transpose(1, 2).contiguous() for x in (q, k, v))
        add(grp, "flash_attn_func (FA2 2.8.3)", timeit(lambda: flash_attn_func(fq, fk, fv)), fl)
    except Exception:
        pass
    ref = load_prebuilt("ref_fa")
    best_ref = None
    if ref is not None:
        for name in ["flash_attn_mma_stages_split_q_shared_qkv", "flash_attn_mma_stages_split_q_shared_qkv_acc_f32",
                     "flash_attn_mma_stages_split_q", "flash_attn_mma_stages_split_q_tiling_qkv"]:
            for st in (1, 2):
                try:
                    ms = timeit(lambda: getattr(ref, name)(q, k, v, o, st), iters=5, warmup=2)
                except Exception:
                    continue
                add(grp, f"reference {name} stages={st} (sm_90a rebuild)", ms, fl)
                best_ref = ms if best_ref is None else min(best_ref, ms)
    _flush()
    if best_ref is not None:
        assert ours < best_ref


def test_ffpa_side_by_side():
    B, H, N, D = 2, 16, 2048, 512
    g = torch.Generator(device="cuda").manual_seed(0)
    q, k, v = (torch.randn(B, H, N, D, device="cuda", dtype=torch.half, generator=g) for _ in range(3))
    o = torch.zeros_like(q)
    fl = 4.0 * B * H * N * N * D
    grp = f"FFPA fwd B{B} H{H} N{N} D{D} fp16"
    try:
        ours = timeit(lambda: ffpa_attn.ffpa_mma_acc_f32_L1(q, k, v, o, 2))
        add(grp, "leetcuda_b200 wgmma attention, 256-column slabs", ours, fl)
    except RuntimeError as e:
        ours = None
        add(grp, f"leetcuda_b200: {e}", float("nan"), fl)
    from torch.nn.attention import SDPBackend, sdpa_kernel
    try:
        with sdpa_kernel(SDPBackend.EFFICIENT_ATTENTION):
            add(grp, "SDPA EFFICIENT_ATTENTION", timeit(lambda: F.scaled_dot_product_attention(q, k, v), iters=5), fl)
    except Exception:
        pass
    ref = load_prebuilt("ref_ffpa")
    best_ref = None
    if ref is not None:
        for name in ["ffpa_mma_acc_f32_L1", "ffpa_mma_acc_f16_L1"]:
            for st in (1, 2, 3):
                try:
                    ms = timeit(lambda: getattr(ref, name)(q, k, v, o, st), iters=5, warmup=2)
                except Exception:
                    continue
                add(grp, f"reference {name} stages={st} (sm_90a rebuild)", ms, fl)
                best_ref = ms if best_ref is None else min(best_ref, ms)
    _flush()
    if ours is not None and best_ref is not None:
        assert ours < best_ref


def test_sgemm_tf32_side_by_side():
    """SURVEY §8f-2: the TF32 SGEMM op (rounding passes included, as in the reference) beside the
    reference's wmma TF32 kernels and the vendor TF32 / fp32 GEMMs."""
    from leetcuda_b200 import sgemm
    S = 8192
    g = torch.Generator(device="cuda").manual_seed(0)
    a = torch.randn(S, S, device="cuda", generator=g)
    b = torch.randn(S, S, device="cuda", generator=g)
    c = torch.empty(S, S, device="cuda")
    fl = 2.0 * S ** 3
    grp = f"SGEMM {S}^3 fp32 (TF32 tensor cores)"
    ours = timeit(lambda: sgemm.sgemm_wmma_m16n16k8_mma4x2_warp2x4_stages(a, b, c, 2, False, 1))
    add(grp, "leetcuda_b200 op: TF32 rounding in place + wgmma .tf32 GEMM", ours, fl)
    add(grp, "leetcuda_b200 GEMM kernel alone (operands already TF32)",
        timeit(lambda: sgemm.sgemm_tf32(a, b, c, round_inputs=False)), fl)
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = True
    add(grp, "cuBLAS TF32 (torch.matmul, allow_tf32)", timeit(lambda: torch.matmul(a, b, out=c)), fl)
    torch.backends.cuda.matmul.allow_tf32 = False
    add(grp, "cuBLAS fp32 (torch.matmul)", timeit(lambda: torch.matmul(a, b, out=c), iters=3, warmup=1), fl)
    torch.backends.cuda.matmul.allow_tf32 = prev
    ref = load_prebuilt("ref_sgemm")
    best_ref = None
    if ref is not None:
        for name, swz in [("sgemm_wmma_m16n16k8_mma4x2_warp2x4_stages", False),
                          ("sgemm_wmma_m16n16k8_mma4x2_warp2x4_stages_dsmem", False),
                          ("sgemm_wmma_m16n16k8_mma4x2_warp2x4_stages_dsmem", True)]:
            for st in (2, 3):
                ms = timeit(lambda: getattr(ref, name)(a, b, c, st, swz, 1024 if swz else 1), iters=3, warmup=1)
                add(grp, f"reference {name} stages={st}{' swizzle' if swz else ''} (sm_90a rebuild)", ms, fl)
                best_ref = ms if best_ref is None else min(best_ref, ms)
    _flush()
    if best_ref is not None:
        assert ours < best_ref


@pytest.mark.parametrize("T", [4096, 131072])
def test_merge_attn_states_side_by_side(T):
    """SURVEY §8f-3: HBM-bound combine step; GB/s over the algorithmic bytes (3*D*2 + 12 per token-head).
    T = 4096 is the largest shape of the reference's own test (L2-resident, launch-bound)."""
    from leetcuda_b200 import merge_attn_states as M
    H, D = 16, 128
    g = torch.Generator(device="cuda").manual_seed(0)
    p = torch.randn(T, H, D, device="cuda", dtype=torch.half, generator=g)
    s = torch.randn(T, H, D, device="cuda", dtype=torch.half, generator=g)
    pl = torch.randn(H, T, device="cuda", generator=g)
    sl = torch.randn(H, T, device="cuda", generator=g)
    o = torch.empty_like(p)
    ol = torch.empty_like(pl)
    nbytes = T * H * (3 * D * 2 + 12)
    grp = f"merge_attn_states T{T} H{H} D{D} fp16"

    def add_bw(name, ms):
        ROWS.append({"workload": grp, "impl": name, "ms": ms, "tflops": nbytes / ms / 1e6 / 1e3})  # GB/s in the last column

    ref = load_prebuilt("ref_merge")
    # order-rotated A/B (ours, reference, ours, reference, ...): the best of each, so neither always runs first
    ours, best_ref = float("inf"), None
    for _ in range(3):
        ours = min(ours, timeit(lambda: M.merge_attn_states_cuda(o, p, pl, s, sl, ol), iters=20))
        if ref is not None:
            r_ms = timeit(lambda: ref.merge_attn_states_cuda(o, ol, p, pl, s, sl), iters=20)
            best_ref = r_ms if best_ref is None else min(best_ref, r_ms)
    add_bw("leetcuda_b200 merge_attn_states (last column: GB/s)", ours)

    def eager():
        m = torch.maximum(pl, sl)
        pe, se = torch.exp(pl - m), torch.exp(sl - m)
        su = pe + se
        return p * (pe / su).t().unsqueeze(2) + s * (se / su).t().unsqueeze(2), torch.log(su) + m
    add_bw("torch eager formula (last column: GB/s)", timeit(eager, iters=5))
    if best_ref is not None:
        add_bw("reference merge_attn_states_cuda (sm_90a rebuild; last column: GB/s)", best_ref)
    _flush()
    if best_ref is not None and T >= 65536:
        # the reference kernel is already bandwidth-bound; at T = 4096 both calls are launch-bound (~11 us)
        # and the comparison measures the Python wrappers, so only the streaming size is asserted
        assert ours < 1.10 * best_ref
