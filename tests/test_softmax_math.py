"""CPU restatement of the exp2 evaluation that the D <= 128 attention kernels run on the FMA pipe for a fixed
subset of their score pairs (leetcuda_b200/csrc/softmax_math.cuh: exp2_fma_pipe).  The coefficients are read
from the header, the arithmetic is replayed in fp32 exactly as the kernel orders it, and the result is held to
the bound the header states (max relative error 7.6e-5 — a third of the fp16 rounding P receives afterwards)."""
import re
from pathlib import Path

import numpy as np

HDR = Path(__file__).resolve().parents[1] / "leetcuda_b200" / "csrc" / "softmax_math.cuh"
MAGIC = np.float32(12582912.0)   # 1.5 * 2^23


def _coefficients():
    src = HDR.read_text()
    body = src[src.index("B200_DEVICE float exp2_fma_pipe"):]
    ks = []
    for name in ("k0", "k1", "k2", "k3"):
        m = re.search(name + r" = ([0-9.eE+-]+)f;", body)
        assert m, f"coefficient {name} not found in {HDR.name}"
        ks.append(np.float32(float(m.group(1))))
    assert "12582912.f" in body and "-126.f" in body
    return ks


def exp2_fma_pipe(x):
    """max(x, -126); t = x + 1.5*2^23; f = x - (t - 1.5*2^23); Horner degree 3; exponent by integer add."""
    k0, k1, k2, k3 = _coefficients()
    x = np.maximum(np.asarray(x, dtype=np.float32), np.float32(-126.0))
    t = (x + MAGIC).astype(np.float32)
    f = (np.float32(-1.0) * (t - MAGIC).astype(np.float32) + x).astype(np.float32)
    q = (k3 * f + k2).astype(np.float32)
    q = (q * f + k1).astype(np.float32)
    q = (q * f + k0).astype(np.float32)
    bits = q.view(np.uint32) + (t.view(np.uint32) << np.uint32(23))
    return bits.view(np.float32)


def test_relative_error_bound_over_the_kernel_domain():
    # the lazy rescale keeps x = (s - m) * scale * log2e <= 8; below, anything down to 2^-125 (at the clamp itself,
    # x = -126, the scaled polynomial value c0 * 2^-126 is subnormal: tiny, finite, irrelevant — next test)
    rng = np.random.default_rng(7)
    x = np.concatenate([rng.uniform(-125.0, 8.5, 2_000_000), np.linspace(-125.0, 8.5, 200_001),
                        np.arange(-125, 9) + 0.5, np.arange(-124, 9) - 0.5, np.arange(-125, 9)]).astype(np.float32)
    got = exp2_fma_pipe(x).astype(np.float64)
    want = np.exp2(x.astype(np.float64))
    assert np.abs(got / want - 1.0).max() < 8e-5


def test_fraction_stays_in_the_fitted_interval_and_integers_are_exact_to_the_fit():
    x = np.linspace(-126.0, 8.5, 400_001).astype(np.float32)
    t = (x + MAGIC).astype(np.float32)
    f = (x - (t - MAGIC).astype(np.float32)).astype(np.float32)
    assert f.min() >= -0.5 and f.max() <= 0.5
    ints = np.arange(-125, 9).astype(np.float32)
    np.testing.assert_allclose(exp2_fma_pipe(ints), np.exp2(ints.astype(np.float64)), rtol=8e-5)


def test_masked_and_very_negative_scores_vanish_in_fp16():
    # -inf is what the kernel writes over the ragged key tail; P is rounded to fp16 before P.V
    x = np.array([-np.inf, -1e30, -1000.0, -127.0, -126.0], dtype=np.float32)
    got = exp2_fma_pipe(x)
    assert np.all(np.isfinite(got)) and np.all(got > 0) and np.all(got < 2e-38)
    assert np.all(got.astype(np.float16) == 0)


def test_rounded_to_fp16_it_agrees_with_the_exact_exponential_to_one_ulp():
    rng = np.random.default_rng(11)
    x = rng.uniform(-14.0, 8.0, 1_000_000).astype(np.float32)      # normal fp16 range of P
    got = exp2_fma_pipe(x).astype(np.float16).astype(np.float64)
    want = np.exp2(x.astype(np.float64)).astype(np.float16).astype(np.float64)
    ulp = np.exp2(np.floor(np.log2(want)) - 10)
    assert np.abs(got - want).max() <= ulp.max() and np.all(np.abs(got - want) <= ulp)


def _attention_with_p(q, k, v, mask_bits):
    """Online-softmax-free restatement of what the kernel computes per row: P = exp2((S - max) * scale * log2e) in fp32 —
    through exp2_fma_pipe for the score pairs `mask_bits` selects inside every 32-key chunk, exactly otherwise — rounded
    to fp16 before P.V, row sum from the unrounded values."""
    d = q.shape[-1]
    c = np.float32(1.4426950408889634 / np.sqrt(d))
    s = (q.astype(np.float32) @ k.astype(np.float32).T).astype(np.float32)
    x = ((s - s.max(axis=1, keepdims=True)) * c).astype(np.float32)
    e = np.exp2(x.astype(np.float64)).astype(np.float32)
    pair = (np.arange(x.shape[1]) % 32) // 2
    sel = ((mask_bits >> pair) & 1).astype(bool)
    e[:, sel] = exp2_fma_pipe(x[:, sel])
    p16 = e.astype(np.float16).astype(np.float32)
    return (p16 @ v.astype(np.float32)) / e.sum(axis=1, keepdims=True)


def test_attention_through_the_mix_stays_far_inside_the_parity_tolerance():
    src = (HDR.parent / "attn_sm90.cuh").read_text()
    masks = [int(m, 16) for m in re.findall(r"#define B200_ATTN_POLY_MASK(?:_D64)? (0x[0-9a-fA-F]+)u", src)]
    assert len(masks) == 2 and all(0 < m < 0x10000 for m in masks)
    rng = np.random.default_rng(3)
    for d, mask in ((128, masks[0]), (64, masks[1])):
        q, k, v = (rng.standard_normal((384, d)).astype(np.float16) for _ in range(3))
        k[200] *= 6.0                                     # a hot key: scores far below the row maximum elsewhere
        plain = _attention_with_p(q, k, v, 0)
        mixed = _attention_with_p(q, k, v, mask)
        s = (q.astype(np.float64) @ k.astype(np.float64).T) / np.sqrt(d)
        w = np.exp(s - s.max(axis=1, keepdims=True))
        truth = (w / w.sum(axis=1, keepdims=True)) @ v.astype(np.float64)
        assert np.abs(mixed - plain).max() < 2e-4          # the polynomial moves O by less than the fp16 rounding of P does
        np.testing.assert_allclose(mixed, truth, rtol=1e-2, atol=1e-2)
        assert np.abs(mixed - truth).max() < 2e-3
