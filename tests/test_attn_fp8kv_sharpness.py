"""The fp8-K/V arithmetic restated on the CPU (attn_fp8kv_ref.kernel_o: exact widening, k_scale folded into the softmax
scale, v_scale on the fp32 O before its one rounding) stays inside attn_fp8kv_ref's bound against fp64 on the dequantised
K and V, and wrong designs break it:
  * k_scale applied to K before a rounding to T (the scale not folded): every score moves by a rounding of T;
  * v_scale applied after O's rounding to T: the product is rounded a second time.  Its extra error, up to one rounding
    of T, fits into the bound's P rounding term u sigma unless that budget is used, so the inputs use it up (see the
    test)."""
import numpy as np
import pytest
import torch

import attn_fp8kv_ref as F
import attn_ref as R


def _inputs(T, N, D, seed, amp=2.0):
    g = torch.Generator().manual_seed(seed)
    q = (torch.randn(N, D, generator=g) * amp).to(F.TORCH[T]).float().numpy()
    k8 = F.quantise(torch.randn(N, D, generator=g) * 3, 1.0)
    v8 = F.quantise(torch.randn(N, D, generator=g) * 3, 1.0)
    return q, k8, v8


def _ratio(T, q, k8, v8, scale, ks, vs, kbn, **wrong):
    o, _ = F.kernel_o(q, k8, v8, scale, ks, vs, kbn, T, **wrong)
    kd, vd = F.decode(k8.view(torch.uint8)).numpy(), F.decode(v8.view(torch.uint8)).numpy()
    sc = float(np.float32(np.float32(scale) * np.float32(ks)))
    truth = R.reference(q, kd, vd, scale * ks)
    ref = R.reference(q, kd, vd, sc)
    bound = F.o_bound(ref, False, T, vs, F.score_max(q, kd, sc))
    return float((np.abs(o - vs * truth["o"]) / bound).max())


@pytest.mark.parametrize("T", F.TYPES)
@pytest.mark.parametrize("scales", F.SCALES, ids=lambda s: f"k{s.k}-v{s.v}")
def test_restated_kernel_inside_the_bound(T, scales):
    for seed in range(3):
        q, k8, v8 = _inputs(T, 192, 64, seed)
        r = _ratio(T, q, k8, v8, R.kernel_scale(64), scales.k, scales.v, 64)
        assert r <= 1.0, r


@pytest.mark.parametrize("T", F.TYPES)
def test_k_scale_applied_to_k_breaks_the_bound(T):
    q, k8, v8 = _inputs(T, 192, 64, 5, amp=6.0)
    assert _ratio(T, q, k8, v8, R.kernel_scale(64), 0.37, 1.0, 64) <= 1.0
    assert _ratio(T, q, k8, v8, R.kernel_scale(64), 0.37, 1.0, 64, k_first=True) > 1.0


@pytest.mark.parametrize("T", F.TYPES)
def test_v_scale_applied_after_the_rounding_breaks_the_bound(T):
    """The bound leaves room for a second rounding of O only where the P rounding budget u sigma goes unused, so the
    inputs use it up: key 0 scores 0 (P = 1 exactly), keys 1 .. 63 score -1 with a scale that puts their P just below
    a rounding midpoint of T in [0.5, 1) (rounded down by almost u), and V is positive, so sigma ~ |O| and O comes out
    low by almost u |O|.  The correct design then rounds once, the wrong one twice."""
    N, D = 64, 64
    u = F.U[T]
    x = np.log2(0.5 + 0.9 * u / 2)   # P = 0.5 + 0.9 (half a spacing of T at 0.5)
    scale = float(-x / R.LOG2E)
    q = np.zeros((8, D), np.float32)
    q[:, 0] = 1.0
    k = torch.zeros(N, D)
    k[1:, 0] = -1.0
    k8 = k.to(torch.float8_e4m3fn)
    codes = F.finite_codes()
    pos = codes[(codes < 0x78) & (codes > 0x08)]   # positive normal codes below 256
    g = torch.Generator().manual_seed(9)
    worst_ok, worst_bad = 0.0, 0.0
    for vs in (1.37, 0.61, 3.3, 0.77, 1.9, 2.9, 0.43):
        v8 = pos[torch.randint(len(pos), (N, D), generator=g)].view(torch.float8_e4m3fn)
        worst_ok = max(worst_ok, _ratio(T, q, k8, v8, scale, 1.0, vs, 64))
        worst_bad = max(worst_bad, _ratio(T, q, k8, v8, scale, 1.0, vs, 64, v_after=True))
    assert worst_ok <= 1.0 and worst_bad > 1.0, (worst_ok, worst_bad)
