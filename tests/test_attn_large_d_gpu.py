"""GPU parity tests of the large-head-dim attention path (FFPA / QKV-tiling ops, SURVEY §8a rows a10, a13):
the attention kernel with 256-column slabs of O (128 < D <= 1024, csrc/attn_sm90.cuh), through the C ABI.

Checker: the CPU oracle on small shapes / head subsets, an fp32 GPU restatement of the reference's own
`unfused_standard_attn` (flash_attn_mma.py:448-452) at the BASELINE configs[3] shape, and the
LSE output.  Tolerance allclose(atol=1e-2, rtol=1e-2) = the
reference's `--check` (ffpa-attn/tests/test_ffpa_attn.py:583-614).
"""
import math
from pathlib import Path

import numpy as np
import pytest
import torch

from leetcuda_b200 import _capi, ffpa_attn, flash_attn
from oracle import oracle as O
from oracle.gen_golden import attn_inputs

pytestmark = pytest.mark.gpu
RTOL = ATOL = 1e-2
ROOT = Path(__file__).resolve().parent.parent


def _dev(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _truth_f32(q, k, v):
    """softmax(Q K^T / sqrt(D)) V and the row log-sum-exp in fp32 on the GPU, one head at a time."""
    B, H, N, D = q.shape
    out = torch.empty(B, H, N, D, device=q.device, dtype=torch.float32)
    lse = torch.empty(B, H, N, device=q.device, dtype=torch.float32)
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        for b in range(B):
            for h in range(H):
                s = (q[b, h].float() @ k[b, h].float().t()) * (1.0 / math.sqrt(D))
                lse[b, h] = torch.logsumexp(s, dim=-1)
                out[b, h] = torch.softmax(s, dim=-1) @ v[b, h].float()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    return out, lse


@pytest.mark.parametrize("shape", [(1, 1, 128, 512), (1, 1, 256, 512), (1, 2, 512, 512), (2, 3, 768, 512),
                                   (1, 1, 300, 512), (1, 1, 72, 512), (1, 2, 512, 384), (1, 1, 1000, 384)])
def test_pair_kernel_vs_oracle(shape):
    B, H, N, D = shape
    q_np, k_np, v_np = attn_inputs(B, H, N, D, seed=N + D)
    want = O.attn_f32(q_np, k_np, v_np).astype(np.float32)
    q, k, v = _dev(q_np), _dev(k_np), _dev(v_np)
    o = torch.full_like(q, float("nan"))
    before = _capi.launch_count()
    ffpa_attn.ffpa_mma_acc_f32_L1(q, k, v, o, 2)
    torch.cuda.synchronize()
    assert _capi.launch_count() - before == 1
    got = o.cpu().numpy().astype(np.float32)
    np.testing.assert_allclose(got, want, rtol=RTOL, atol=ATOL)
    assert np.abs(got - want).max() < 2e-3


def test_config4_full_shape():
    """BASELINE configs[3]: B2 H16 N2048 D512 — every output element against the fp32 restatement, a head subset
    against the CPU oracle, the LSE output, and both FFPA op names / the ffpa() front end."""
    B, H, N, D = 2, 16, 2048, 512
    g = torch.Generator(device="cuda").manual_seed(512)
    q, k, v = (torch.randn(B, H, N, D, device="cuda", dtype=torch.half, generator=g) for _ in range(3))
    want, want_lse = _truth_f32(q, k, v)
    o = torch.full_like(q, float("nan"))
    lse = torch.full((B, H, N), float("nan"), device="cuda")
    flash_attn.fmha_fwd(q, k, v, o, lse=lse)
    torch.cuda.synchronize()
    assert torch.allclose(o.float(), want, rtol=RTOL, atol=ATOL)
    assert (o.float() - want).abs().max().item() < 2e-3
    assert (lse - want_lse).abs().max().item() < 2e-3
    # CPU oracle on two heads (its fp32 path is the pinned checker)
    for (b, h) in ((0, 0), (1, 15)):
        sl = lambda t: t[b:b + 1, h:h + 1].cpu().numpy()
        ref = O.attn_f32(sl(q), sl(k), sl(v)).astype(np.float32)
        np.testing.assert_allclose(sl(o).astype(np.float32), ref, rtol=RTOL, atol=ATOL)
    # the reference-facing names run the same kernel
    for fn in (ffpa_attn.ffpa_mma_acc_f32_L1, ffpa_attn.ffpa_mma_acc_f16_L1):
        o2 = torch.zeros_like(q)
        fn(q, k, v, o2, 2)
        torch.cuda.synchronize()
        assert torch.equal(o2, o)
    assert torch.equal(ffpa_attn.ffpa(q, k, v, None, 2, level=ffpa_attn.L1, acc=ffpa_attn.FP32), o)


@pytest.mark.parametrize("shape", [(1, 2, 512, 128), (1, 2, 300, 64), (1, 2, 512, 256), (1, 2, 768, 512), (1, 1, 256, 640)])
def test_lse_output(shape):
    """b200_fmha_fwd_f16_lse: lse = ln sum_j exp(scale q.k_j) for every kernel shape (64-, 128-, 256-column slabs)."""
    B, H, N, D = shape
    g = torch.Generator(device="cuda").manual_seed(N + D)
    q, k, v = (torch.randn(B, H, N, D, device="cuda", dtype=torch.half, generator=g) for _ in range(3))
    want, want_lse = _truth_f32(q, k, v)
    o = torch.zeros_like(q)
    lse = torch.full((B, H, N), float("nan"), device="cuda")
    flash_attn.fmha_fwd(q, k, v, o, lse=lse)
    torch.cuda.synchronize()
    assert torch.allclose(o.float(), want, rtol=RTOL, atol=ATOL)
    assert (lse - want_lse).abs().max().item() < 2e-3
    o2 = torch.zeros_like(q)
    flash_attn.fmha_fwd(q, k, v, o2)           # the statistic is a by-product: O does not change
    torch.cuda.synchronize()
    assert torch.equal(o, o2)


@pytest.mark.parametrize("D", [128, 512])
def test_split_kv_merge_with_kernel_lse(D):
    """The property merge_attn_states exists for, end to end inside this library: attention over [K1;K2] ==
    merge(attention over K1, attention over K2), using the LSEs the attention kernels themselves write
    (the reference's test drives the merge with synthetic LSEs, test_merge_attn_states.py:100-152)."""
    from leetcuda_b200 import merge_attn_states as MA
    H, N, NK = 8, 512, 1024
    g = torch.Generator(device="cuda").manual_seed(11 + D)
    q = torch.randn(1, H, N, D, device="cuda", dtype=torch.half, generator=g)
    k = torch.randn(1, H, NK, D, device="cuda", dtype=torch.half, generator=g)
    v = torch.randn(1, H, NK, D, device="cuda", dtype=torch.half, generator=g)
    # the kernels take equal query / key lengths: run the full problem on N = NK queries (q padded with
    # further random rows) and use the first N rows
    qq = torch.cat([q, torch.randn(1, H, NK - N, D, device="cuda", dtype=torch.half, generator=g)], dim=2)
    full = torch.zeros_like(qq)
    flash_attn.fmha_fwd(qq, k, v, full)
    parts = []
    for ks in (slice(0, 512), slice(512, 1024)):
        qh = qq[:, :, :512].contiguous()                      # 512 queries against 512 keys of this part
        o = torch.zeros_like(qh)
        lse = torch.zeros(1, H, 512, device="cuda")
        flash_attn.fmha_fwd(qh, k[:, :, ks].contiguous(), v[:, :, ks].contiguous(), o, lse=lse,
                            scale=1.0 / math.sqrt(D))
        parts.append((o[0].transpose(0, 1).contiguous(), lse[0].contiguous()))   # [T,H,D], [H,T]
    merged = torch.empty_like(parts[0][0])
    merged_lse = torch.empty_like(parts[0][1])
    MA.merge_attn_states_cuda(merged, parts[0][0], parts[0][1], parts[1][0], parts[1][1], merged_lse)
    torch.cuda.synchronize()
    want = full[0, :, :512].transpose(0, 1).float()
    assert torch.allclose(merged.float(), want, rtol=RTOL, atol=ATOL)
    assert (merged.float() - want).abs().max().item() < 3e-3
    _, want_lse = _truth_f32(qq[:, :, :512].contiguous(), k, v) if False else (None, None)
    s = (qq[0, :, :512].float() @ k[0].float().transpose(-2, -1)) / math.sqrt(D)
    assert (merged_lse - torch.logsumexp(s, dim=-1)).abs().max().item() < 2e-3
