"""fp64 GEMM reference, per-element error bounds for every GEMM mode, adversarial input generators and a restatement of
the host's tile choice, for the GEMM tests.

Modes (csrc/hgemm_capi.cu, csrc/hgemm_sm90.cuh):
  "f16"      fp16 A, B; fp32 accumulation on the tensor core; C rounded once to fp16      (b200_hgemm_f16)
  "f16acc"   fp16 A, B; fp16 accumulator, rounded after every k16 wgmma instruction       (b200_hgemm_f16_acc16)
  "tf32"     fp32 A, B rounded to TF32 in place (cvt.rna), fp32 accumulation, fp32 C     (b200_sgemm_tf32, round=1)
  "tf32t"    fp32 A, B left as they are: the TF32 tensor core truncates them              (b200_sgemm_tf32, round=0)
  "3xtf32"   fp32 A, B split x = hi + lo, C = hi hi + hi lo + lo hi in one TF32 GEMM over 3K (b200_sgemm_3xtf32)

Reference (`reference`).  C64 = A B in float64 from the operands as the kernel sees them: the fp16 inputs, the
TF32-rounded operands ("tf32"), the truncated operands ("tf32t"), the raw fp32 operands ("3xtf32"); the sensitivity
s = |A| |B| of the same operands; for "f16acc" the weighted sum W = sum_t (1+u)^(T-t) |P_t| of the k16 prefix sums
P_t = sum_{k < 16t} a_k b_k, t = 1..T = ceil(K/16) (P_T = C64).  Pass sampled rows of A for large shapes.  It takes
numpy arrays (CPU self-check) or torch tensors (GPU tests, computed on the device).  float64 summation adds at most
K 2^-53 s, below 2^-40 s for every K used here, which is negligible against every term below (the smallest is
16 2^-23 s).

Bound (`bound`).  Model of the tensor core, the one attn_ref.py uses for the score error rho: each wgmma k-step adds
its `step` exact products with an error of at most step 2^-23 of their magnitude, and each accumulator add rounds once
(at most 2^-23 of the running sum, whose magnitude is at most s).  Over ceil(K/step) steps that gives

    gamma(K, step) = (ceil(K/step) + step) 2^-23,      |C32 - C64| <= gamma s       (first order; the second-order
                                                                                      terms are below K^2 2^-46 s)

step = 16 for fp16 operands, 8 for TF32.  The zero-filled k past K (the ragged last k-block) adds exact zeros.

  f16     C32 as above, then one rounding to fp16: |C16 - C32| <= u |C32| + 2^-25 (u = 2^-11; 2^-25 is half a step of
          the subnormal grid), and |C32| <= |C64| + gamma s:
              |C16 - C64| <= u |C64| + (1 + u) gamma(K, 16) s + 2^-25
  f16acc  acc_t = fl16(acc_{t-1} + step_t + e_t), |e_t| <= 16 2^-23 s_t (s_t: the magnitude of step t's products).
          With E_t = acc_t - P_t the rounding adds at most u |P_t + E_{t-1} + e_t| + 2^-25, so
              |E_t| <= (1 + u) |E_{t-1}| + (1 + u) |e_t| + u |P_t| + 2^-25,
          and unrolled over the T instructions that carry data (a k16 step of zero-filled k leaves acc unchanged):
              |C - C64| <= u W + 2^-25 sum_t (1+u)^(T-t) + (1+u)^T 16 2^-23 s
          The result is the accumulator itself: no further rounding.
  tf32    the products of two 11-bit significands are exact in fp32 and C is not rounded again:
              |C - C64| <= gamma(K, 8) s          (C64, s of the rounded operands; "tf32t": of the truncated ones)
  3xtf32  hi = tf32(x), lo = tf32(x - hi): |x - hi| <= 2^-11 |x|, x - hi is exact in fp32, |lo| <= 2^-11 (1 + 2^-11)|x|
          and the split leaves a residue d = x - hi - lo, |d| <= 2^-22 |x|.  The exact a b differs from what is summed,
          hi_a hi_b + hi_a lo_b + lo_a hi_b, by lo_a lo_b + d_a b + (hi_a + lo_a) d_b: the dropped term (2^-22 s) and
          one residue per operand (2^-22 s each), 3 2^-22 (1 + 2^-9) s with the factors above.  The 3K-term TF32
          product accumulates with gamma(3K, 8) over its own magnitude, at most (1 + 2^-8) s:
              |C - C64| <= (3 2^-22 (1 + 2^-9) + (1 + 2^-8) gamma(3K, 8)) s      (C64, s of the raw operands)
          The operands here are normal floats or zero; a subnormal operand would add an absolute residue.

Nothing here is fitted to measurements.  |C| < 65520 is assumed (larger values become inf, checked separately).
"""
from __future__ import annotations

import math

import numpy as np
import torch

U16 = 2.0 ** -11
U23 = 2.0 ** -23
SUB16 = 2.0 ** -25                # half a step of the fp16 subnormal grid
MODES = ("f16", "f16acc", "tf32", "tf32t", "3xtf32")
STEP = {"f16": 16, "f16acc": 16, "tf32": 8, "tf32t": 8, "3xtf32": 8}
KBLOCK = {"f16": 64, "f16acc": 64, "tf32": 32, "tf32t": 32, "3xtf32": 32}   # elements per 128-byte k-block
STAGES = {128: 6, 256: 4}          # smem ring slots per tile width (hgemm::Cfg<kBN>::STAGES)


def is_fp16(mode):
    return mode in ("f16", "f16acc")


def gamma(K, step):
    return (math.ceil(K / step) + step) * U23


# ------------------------------------------------------------------ operands
def _is_torch(x):
    return isinstance(x, torch.Tensor)


def tf32(x, truncate=False):
    """cvt.rna.tf32.f32 (round to nearest, ties away from zero, to 10 explicit significand bits) or truncation, of a
    float32 numpy array or torch tensor; inf and NaN are truncated.  Bit for bit what oracle.tf32_round computes."""
    if _is_torch(x):
        bits = x.contiguous().view(torch.int32)
    else:
        bits = np.ascontiguousarray(x, dtype=np.float32).view(np.int32)
    finite = (bits & 0x7F800000) != 0x7F800000
    if not truncate:
        bits = (torch.where if _is_torch(x) else np.where)(finite, bits + 0x1000, bits)
    out = bits & -0x2000
    return out.view(torch.float32) if _is_torch(x) else out.astype(np.int32).view(np.float32)


def operands(a, b, mode):
    """A and B in float64 as the tensor core multiplies them (logical layouts [M,K] and [K,N])."""
    if mode == "tf32":
        a, b = tf32(a), tf32(b)
    elif mode == "tf32t":
        a, b = tf32(a, truncate=True), tf32(b, truncate=True)
    if _is_torch(a):
        return a.double(), b.double()
    return np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)


# ------------------------------------------------------------------ reference and bound
def reference(a, b, mode):
    """C64, s (and W, T for "f16acc") of C = A B; a: [M,K] (or sampled rows of it), b: [K,N]."""
    a, b = operands(a, b, mode)
    K = a.shape[1]
    ref = {"c": a @ b, "s": abs(a) @ abs(b), "K": K, "mode": mode}
    if mode == "f16acc":
        T = math.ceil(K / 16)
        P = a[:, :0] @ b[:0]                     # zeros of C's shape and type
        W = abs(P)
        for t in range(T):
            P = P + a[:, 16 * t:16 * t + 16] @ b[16 * t:16 * t + 16]
            W = W * (1 + U16) + abs(P)           # Horner: W = sum_t (1+u)^(T-t) |P_t|
        ref.update(W=W, T=T)
    return ref


def bound(ref, mode=None):
    """Per-element bound on |C - C64| for `mode` (default: the mode the reference was computed for)."""
    mode = mode or ref["mode"]
    K, s, c = ref["K"], ref["s"], ref["c"]
    if mode == "f16":
        return U16 * abs(c) + (1 + U16) * gamma(K, 16) * s + SUB16
    if mode == "f16acc":
        T = ref["T"]
        geo = ((1 + U16) ** T - 1) / U16         # sum_t (1+u)^(T-t)
        return U16 * ref["W"] + SUB16 * geo + (1 + U16) ** T * 16 * U23 * s
    if mode in ("tf32", "tf32t"):
        return gamma(K, 8) * s
    if mode == "3xtf32":
        return (3 * 2.0 ** -22 * (1 + 2.0 ** -9) + (1 + 2.0 ** -8) * gamma(3 * K, 8)) * s
    raise ValueError(mode)


# ------------------------------------------------------------------ generators
GENERATORS = ("randn", "binade", "cancel", "k_probe", "a_probe")
EXACT = ("k_probe", "a_probe")


def _codes(j):
    """Distinct non-zero integers for j in [0, 4096): 1..2048 and -1..-2048, all exact in fp16 and TF32."""
    j = np.asarray(j) % 4096
    return np.where(j < 2048, j + 1, 2047 - j).astype(np.float32)


def make_inputs(gen, M, N, K, dtype, seed=0):
    """Seeded a [M,K], b [K,N] (logical layouts) of dtype np.float16 or np.float32, and probe data (or None).

    randn    the reference's distribution
    binade   randn with row m of A scaled by 2^e_m, e in [-10, 2], and column n of B by 2^f_n, f in [-6, 2]: outputs
             span about 20 binades, down into fp16 subnormals, while |C| stays below 2^14
    cancel   the second half of k repeats A's first half against -B's first half plus a 2^-6 residue: |C64| << s, so
             the accumulation term dominates the bound
    k_probe  B[k, n] = 1 iff k = sigma(n), A holds distinct exact integers along each row: C[m, n] = A[m, sigma(n)]
             exactly.  sigma reaches k = 0 and k = K - 1.  Probe data: {"sigma": sigma}
    a_probe  A[m, k] = 1 iff k = tau(m), B holds distinct exact integers down each column: C[m, :] = B[tau(m), :]
             exactly (the MN-major B descriptor along k).  Probe data: {"tau": tau}
    """
    assert K <= 4096
    rng = np.random.default_rng(seed)
    info = None
    if gen == "k_probe":
        sigma = rng.integers(0, K, N)
        sigma[0], sigma[-1] = K - 1, 0
        a = _codes(np.arange(K)[None, :] + 131 * np.arange(M)[:, None])
        b = np.zeros((K, N), np.float32)
        b[sigma, np.arange(N)] = 1.0
        info = {"sigma": sigma}
    elif gen == "a_probe":
        tau = rng.integers(0, K, M)
        tau[0], tau[-1] = K - 1, 0
        a = np.zeros((M, K), np.float32)
        a[np.arange(M), tau] = 1.0
        b = _codes(np.arange(K)[:, None] + 37 * np.arange(N)[None, :])
        info = {"tau": tau}
    else:
        a = rng.standard_normal((M, K), dtype=np.float32)
        b = rng.standard_normal((K, N), dtype=np.float32)
        if gen == "binade":
            a *= np.exp2(rng.integers(-10, 3, M)).astype(np.float32)[:, None]
            b *= np.exp2(rng.integers(-6, 3, N)).astype(np.float32)[None, :]
        elif gen == "cancel":
            h = K // 2
            a[:, h:2 * h] = a[:, :h]
            b[h:2 * h] = -b[:h].astype(dtype).astype(np.float32) + np.float32(2.0 ** -6) * b[h:2 * h]
        elif gen != "randn":
            raise ValueError(gen)
    return np.ascontiguousarray(a, dtype=dtype), np.ascontiguousarray(b, dtype=dtype), info


def probe_miss(a, b, got, want, info):
    """Describe the first wrong element of a probe: which (m, k) of the operand landed in the wrong (m', n)."""
    bad = np.argwhere(got != want)
    if not len(bad):
        return "no mismatch"
    m, n = (int(x) for x in bad[0])
    v = got[m, n]
    msg = f"{len(bad)} wrong outputs; first C[{m}, {n}] = {v}, want {want[m, n]}"
    if info and "sigma" in info:
        src = np.argwhere(a == v)[:4].tolist()
        return msg + f" (expected A[{m}, {info['sigma'][n]}]); A holds {v} at (m, k) = {src}"
    if info and "tau" in info:
        src = np.argwhere(b == v)[:4].tolist()
        return msg + f" (expected B[{info['tau'][m]}, {n}]); B holds {v} at (k, n) = {src}"
    return msg


# ------------------------------------------------------------------ tile choice (hgemm_capi.cu, hgemm_impl)
BM, GROUP_M = 128, 16


def tile_width(M, N, sms):
    """The host's choice for an M x N output on `sms` SMs, restated: 128 x 256 tiles unless 0.9 x the last-wave
    occupancy of 128 x 128 tiles beats that of 128 x 256.  Returns a dict with the tile width bn, tiles_m, tiles_n,
    tiles, grid, tiles_per_cta (the most any CTA runs) and the raster groups as (first m-tile, m-tiles, backwards)."""
    def score(bn, eff):
        tiles = -(-M // BM) * -(-N // bn)
        waves = -(-tiles // sms)
        return eff * tiles / (waves * sms)
    bn = 128 if score(128, 0.90) > score(256, 1.0) else 256
    tm, tn = -(-M // BM), -(-N // bn)
    tiles = tm * tn
    grid = min(tiles, sms)
    groups = [(g * GROUP_M, min(GROUP_M, tm - g * GROUP_M), g % 2 == 1) for g in range(-(-tm // GROUP_M))]
    return {"bn": bn, "tiles_m": tm, "tiles_n": tn, "tiles": tiles, "grid": grid,
            "tiles_per_cta": -(-tiles // grid), "groups": groups}


def instantiation(mode, tn, bn):
    """The hgemm_wgmma_kernel<kBN, kBMn, kTf32, kAcc16> template arguments a call runs."""
    if is_fp16(mode):
        return (bn, not tn, False, mode == "f16acc")
    return (bn, False, True, False)       # TF32 operands are always K-major (B is transposed first when [K,N])


ALL_INSTANTIATIONS = frozenset([(bn, mn, False, acc) for bn in (128, 256) for mn in (False, True)
                                for acc in (False, True)] + [(bn, False, True, False) for bn in (128, 256)])
