// softmax_math.cuh — exp2 on the FMA pipe, for a fixed subset of the attention scores.
//
// Per score the softmax issues one FFMA (s * scale * log2e - m) and one MUFU.EX2; the MUFU pipe runs at a
// sixteenth of the FMA pipe's rate.  attn_sm90.cuh evaluates a fixed quarter of the scores of the D <= 128
// kernels (B200_ATTN_POLY_MASK) with the polynomial below instead, which uses no MUFU instruction at all.
#pragma once
#include "sm90_ptx.cuh"

namespace b200 {

// 2^x without the MUFU pipe:
//   x' = max(x, -126);  t = x' + 1.5*2^23 (round-to-nearest integer n = round(x') lands in the low mantissa bits);
//   f = x' - (t - 1.5*2^23) in [-0.5, 0.5];  2^f ~ k0 + f (k1 + f (k2 + f k3))  (minimax, max rel. error 7.6e-5 —
//   a third of the fp16 rounding P gets afterwards);  2^x = bits(2^f) + (bits(t) << 23): the shift drops everything of t
//   but n, negative n wraps to the right exponent decrement.  2 FADD, 4 FFMA, 1 FMNMX, 1 shift + add: no MUFU, no
//   conversion instruction (F2I / FRND run on the MUFU pipe as well).  -inf (masked keys) gives < 2e-38, 0 in fp16.
B200_DEVICE float exp2_fma_pipe(float x) {
  const float k0 = 0.9999276399612427f;
  const float k1 = 0.693252682685852f;
  const float k2 = 0.24261489510536194f;
  const float k3 = 0.05521666631102562f;
  const float xc = fmaxf(x, -126.f);
  const float t = __fadd_rn(xc, 12582912.f);
  const float f = __fmaf_rn(__fadd_rn(t, -12582912.f), -1.f, xc);
  float q = __fmaf_rn(k3, f, k2);
  q = __fmaf_rn(q, f, k1);
  q = __fmaf_rn(q, f, k0);
  return __uint_as_float(__float_as_uint(q) + (__float_as_uint(t) << 23));
}

}  // namespace b200
