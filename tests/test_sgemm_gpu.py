"""GPU parity tests of the TF32 SGEMM path (SURVEY §8f-2): every call goes through the C ABI
(leetcuda_b200.sgemm -> ctypes -> b200_sgemm_tf32).  The checker is the CPU oracle
(oracle/oracle.c: cvt.rna.tf32 rounding + fp32 accumulation in k8 chunks), the committed golden
outputs of the reference's own TF32 kernels, and exact integer products at a BASELINE-sized shape.

Tolerance: operands are exactly the reference's (rounded in place, bit-checked), so the only
freedom is the accumulation order/rounding inside the tensor core: |C - truth| <= K * 2^-23 * max|C|
(one truncated fp32 addition per product, worst case); measured values are ~30x smaller.
"""
import json
from pathlib import Path

import numpy as np
import pytest
import torch

import gemm_ref
from leetcuda_b200 import _capi, sgemm
from oracle import oracle as O
from oracle.gen_golden import SGEMM_CASES, sgemm_inputs

pytestmark = pytest.mark.gpu
GOLD = Path(__file__).parent / "golden"


def _dev(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _bound(K, truth):
    return K * 2.0 ** -23 * max(np.abs(truth).max(), 1.0)


@pytest.mark.parametrize("tn", [False, True])
@pytest.mark.parametrize("shape", [(128, 256, 32), (256, 256, 128), (512, 512, 512), (520, 264, 72),
                                   (8, 8, 8), (128, 24, 512), (128, 32, 512), (1000, 24, 4096)])
def test_vs_oracle_small(shape, tn):
    """Reference semantics (round a, b to TF32 in place, multiply) on aligned, ragged and
    narrow-N shapes the reference itself cannot run (it needs M,N % 128 == 0)."""
    M, N, K = shape
    a_np, b_np = sgemm_inputs(M, N, K, seed=M + N + K)
    a = _dev(a_np)
    b = _dev(b_np)
    bb = b.t().contiguous().view(K, N) if tn else b
    c = torch.full((M, N), float("nan"), device="cuda")
    sgemm.sgemm_tf32(a, bb, c, tn=tn)
    torch.cuda.synchronize()
    # the in-place side effect is exactly cvt.rna.tf32.f32 (sgemm_wmma_tf32_stage.cu:44-60)
    assert np.array_equal(a.cpu().numpy(), O.tf32_round(a_np))
    b_back = bb.view(N, K).t().cpu().numpy() if tn else bb.cpu().numpy()
    assert np.array_equal(b_back, O.tf32_round(b_np))
    truth = O.sgemm_f64(a_np, b_np, mode="rna")
    got = c.cpu().numpy().astype(np.float64)
    assert np.abs(got - truth).max() <= _bound(K, truth)
    assert np.abs(got - O.sgemm_tf32(a_np, b_np, mode="rna")).max() <= _bound(K, truth)
    ref = gemm_ref.reference(a_np, b_np, "tf32")      # element by element within the bound derived in gemm_ref.py
    assert np.all(np.abs(got - ref["c"]) <= gemm_ref.bound(ref))


def test_unrounded_operands_are_truncated_by_the_tensor_core():
    """round_inputs=False leaves a, b untouched; the TF32 wgmma then reads the upper 19 bits."""
    M, N, K = 256, 256, 512
    a_np, b_np = sgemm_inputs(M, N, K, seed=9)
    a, b = _dev(a_np), _dev(b_np)
    c = torch.empty(M, N, device="cuda")
    sgemm.sgemm_tf32(a, b, c, round_inputs=False)
    torch.cuda.synchronize()
    assert np.array_equal(a.cpu().numpy(), a_np) and np.array_equal(b.cpu().numpy(), b_np)
    got = c.cpu().numpy().astype(np.float64)
    t_trunc = O.sgemm_f64(a_np, b_np, mode="trunc")
    t_rna = O.sgemm_f64(a_np, b_np, mode="rna")
    assert np.abs(got - t_trunc).max() <= _bound(K, t_trunc)
    assert np.abs(got - t_rna).max() > 50 * np.abs(got - t_trunc).max()


@pytest.mark.parametrize("case", SGEMM_CASES)
def test_vs_reference_golden(case):
    """Against the recorded outputs of the reference's own wmma TF32 kernels (rebuilt for sm_100a when they were recorded):
    same operands bit for bit, results within the accumulation-order bound, and at least as close
    to the exact product as the reference is."""
    M, N, K, seed = case
    f = GOLD / f"sgemm_{M}x{N}x{K}_s{seed}.npz"
    if not f.exists():
        pytest.skip("golden not generated")
    g = np.load(f)
    sub = json.loads(str(g["meta"]))["subsample"]
    a_np, b_np = sgemm_inputs(M, N, K, seed)
    a, b = _dev(a_np), _dev(b_np)
    c = torch.empty(M, N, device="cuda")
    sgemm.sgemm_wmma_m16n16k8_mma4x2_warp2x4_stages(a, b, c, 2, False, 1)   # reference signature
    torch.cuda.synchronize()
    assert np.array_equal(a[:8].cpu().numpy(), g["a_after"]) and np.array_equal(b[:8].cpu().numpy(), g["b_after"])
    got = c.cpu().numpy()[::sub, ::sub].astype(np.float64)
    truth = O.sgemm_f64(a_np, b_np, mode="rna")[::sub, ::sub]
    e_ours = np.abs(got - truth).max()
    for name in (k for k in g.files if k.startswith("sgemm_wmma")):
        ref = g[name].astype(np.float64)
        np.testing.assert_allclose(got, ref, rtol=1e-2, atol=1e-2)
        assert np.abs(got - ref).max() <= 2 * _bound(K, truth), name
        assert e_ours <= 1.5 * np.abs(ref - truth).max(), (name, e_ours)


def test_every_op_name_computes_the_same_gemm():
    M, N, K = 256, 384, 128
    a_np, b_np = sgemm_inputs(M, N, K, seed=5)
    truth = O.sgemm_f64(a_np, b_np, mode="asis")
    before = _capi.launch_count()
    for name in sgemm.OP_NAMES:
        a, b = _dev(a_np), _dev(b_np)
        c = torch.full((M, N), float("nan"), device="cuda")
        op = getattr(sgemm, name)
        if "stages" in name:
            op(a, b, c, 2, False, 1)
        else:
            op(a, b, c)
        torch.cuda.synchronize()
        tol = 2e-2 if ("tf32" in name or "wmma" in name) else 1e-3   # TF32 operands vs full fp32
        np.testing.assert_allclose(c.cpu().numpy(), truth, rtol=tol, atol=tol * 10, err_msg=name)
    # the two tensor-core ops launched OUR kernels (2 rounding passes + 1 GEMM each); the 13 fp32 names and the two
    # cublas names are vendor rows by default
    assert _capi.launch_count() - before == 2 * 3


@pytest.mark.parametrize("shape", [(256, 384, 128), (1024, 1024, 1024), (512, 640, 4096), (96, 100, 36)])
def test_3xtf32_accuracy_and_fp32_names(shape, monkeypatch):
    """sgemm_3xtf32 (operands split into two exact TF32 numbers, one wgmma GEMM over K' = 3K): a and b stay untouched,
    the error against an fp64 product is far below a plain TF32 product's and bounded by the tensor core's accumulation
    (K * 2^-23 of the largest output, the bound the TF32 tests use) — but not FFMA-grade, which is why the reference's
    fp32 op names stay vendor rows unless LEETCUDA_B200_SGEMM_FP32=3xtf32."""
    M, N, K = shape
    a_np, b_np = sgemm_inputs(M, N, K, seed=M + K)
    truth = a_np.astype(np.float64) @ b_np.astype(np.float64)
    a, b = _dev(a_np), _dev(b_np)
    c = torch.full((M, N), float("nan"), device="cuda")
    before = _capi.launch_count()
    sgemm.sgemm_3xtf32(a, b, c)
    torch.cuda.synchronize()
    assert _capi.launch_count() - before == 3                     # two split passes + one GEMM
    assert torch.equal(a.cpu(), torch.from_numpy(a_np)) and torch.equal(b.cpu(), torch.from_numpy(b_np))
    scale = np.abs(truth).max()
    e_ours = np.abs(c.cpu().numpy() - truth).max() / scale
    cv = torch.empty(M, N, device="cuda")
    sgemm.sgemm_t_8x8_sliced_k16_f32x4_bcf_dbuf_async(a, b, cv)    # default: vendor fp32
    ct = torch.empty(M, N, device="cuda")
    sgemm.sgemm_tf32(a.clone(), b.clone(), ct)
    torch.cuda.synchronize()
    e_vendor = np.abs(cv.cpu().numpy() - truth).max() / scale
    e_tf32 = np.abs(ct.cpu().numpy() - truth).max() / scale
    assert e_vendor < 1e-5, e_vendor
    assert e_ours < e_tf32 / 3, (e_ours, e_tf32)
    assert e_ours < max(K * 2.0 ** -23, 2e-6), (e_ours, K)
    # the opt-in routes the fp32 names through the same kernel
    monkeypatch.setenv("LEETCUDA_B200_SGEMM_FP32", "3xtf32")
    c2 = torch.full((M, N), float("nan"), device="cuda")
    sgemm.sgemm_naive_f32(a, b, c2)
    torch.cuda.synchronize()
    assert torch.equal(c2, c)
