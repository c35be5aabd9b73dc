/* oracle.c — TEST INFRASTRUCTURE.  CPU restatement of the reference's two hot
 * paths, used only by tests/, __graft_entry__.smoke() and bench.py's cpu_baseline
 * leg as the checker.  The product (leetcuda_b200/) never links or calls this.
 *
 * Parity status: the reference ships no golden vectors (SURVEY.md §4, §8c).  This
 * oracle is pinned instead against outputs of the reference's own kernels
 * (oracle/_ref, built from /root/reference by oracle/build_ref.py and run on a
 * B200 by oracle/gen_golden.py), committed under tests/golden/.
 *
 * Functions (all fp16 tensors are passed as uint16_t bit patterns):
 *
 *   oracle_hgemm_f64      exact products, double accumulation          -> double C ("truth")
 *   oracle_hgemm_f32acc   fp32 accumulation, k ascending, round to fp16 (what the
 *                         sm_90a kernel computes up to summation order)
 *   oracle_hgemm_f16acc   the reference's semantics: one HMMA.16816.F16 per k16
 *                         chunk, accumulator held in fp16 between chunks
 *                         (kernels/hgemm/mma/basic/hgemm_mma.cu:67-73 `mma...f16.f16.f16.f16`,
 *                         k loop kernels/hgemm/mma/basic/hgemm_mma_stage.cu:843-871)
 *   oracle_attn_f32       softmax(Q K^T * scale) V in fp32, output rounded to fp16:
 *                         the reference's own check function unfused_standard_attn
 *                         (kernels/flash-attn/flash_attn_mma.py:448-452) at fp32
 *   oracle_attn_online    the FA-2 online-softmax recurrence exactly as the reference
 *                         kernels run it (kernels/flash-attn/mma/basic/flash_attn_mma_split_q.cu:393-646):
 *                         per KV tile of Bc keys: m_new = max(m_old, rowmax(S*scale));
 *                         P = exp(S*scale - m_new) (fp32), l += rowsum(P) in fp32, P rounded
 *                         to fp16 for P@V, O rescaled by exp(m_old - m_new), final O/l.
 *   oracle_tf32_round     x -> tf32(x): cvt.rna.tf32.f32 = round to nearest, ties away from zero,
 *                         to 10 explicit mantissa bits (what wmma::__float_to_tf32 emits; the
 *                         reference applies it to a and b IN PLACE before its TF32 GEMM,
 *                         kernels/sgemm/sgemm_wmma_tf32_stage.cu:44-60, 586-592); mode 1 = truncation
 *                         (what a tensor core does with an unrounded fp32 operand)
 *   oracle_sgemm_tf32     C = tf32(A) tf32(B), fp32 accumulation in k chunks of 8 (one
 *                         m16n16k8 wmma::mma_sync per chunk, sgemm_wmma_tf32_stage.cu:226-236);
 *                         inside a chunk the products are exact in fp32 (10 x 10 mantissa bits)
 *                         and are summed in double, then rounded once — the tensor core's
 *                         internal order is not architected, the tests bound the difference
 *   oracle_sgemm_f64      exact double product of the (already rounded) operands ("truth")
 *   oracle_merge_attn_states  section 2.2 of arXiv 2501.01005 exactly as the reference kernel runs it
 *                         (kernels/openai-triton/merge-attn-states/cuda_merge_attn_states.cu:49-93):
 *                         +inf lse -> -inf, m = max, scales exp(lse - m) / sum in fp32, one fp32 fma
 *                         per element, output rounded to the tensor dtype (fp32 / fp16 / bf16)
 *   oracle_rope_f32       kernels/rope/rope.cu:20-34 (rope_f32_kernel; :37-71 are re-indexings of the same
 *                         math): pair i of the row at position p is rotated by p * (1 / powf(theta, 2i/hidden)),
 *                         theta = 10000, every step in fp32 with IEEE powf / sinf / cosf (the reference's own
 *                         build uses --use_fast_math, rope.py:21, so its kernels sit within fast-math error of this)
 *   oracle_rms_norm       kernels/rms-norm/rms_norm.cu:55-73 (fp32) and :319-338 (fp16 storage, fp32 statistics):
 *                         s = rsqrt(sum(x^2)/K + 1e-5) in fp32, y = (x * s) * g, rounded to the storage type
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef _Float16 f16;

static inline float h2f(uint16_t h) {
  f16 x;
  memcpy(&x, &h, 2);
  return (float)x;
}
static inline uint16_t f2h(float f) {
  f16 x = (f16)f; /* round-to-nearest-even */
  uint16_t h;
  memcpy(&h, &x, 2);
  return h;
}
static inline float round_h(float f) { return (float)(f16)f; }

/* b_layout: 0 = b is [K,N] row-major, 1 = b is [N,K] row-major */
static inline float bget(const uint16_t* b, int layout, int k, int n, int N, int K) {
  return layout == 0 ? h2f(b[(size_t)k * N + n]) : h2f(b[(size_t)n * K + k]);
}

void oracle_hgemm_f64(const uint16_t* a, const uint16_t* b, double* c, int M, int N, int K,
                      int b_layout) {
#pragma omp parallel for schedule(static)
  for (int m = 0; m < M; ++m) {
    for (int n = 0; n < N; ++n) {
      double acc = 0.0;
      for (int k = 0; k < K; ++k)
        acc += (double)h2f(a[(size_t)m * K + k]) * (double)bget(b, b_layout, k, n, N, K);
      c[(size_t)m * N + n] = acc;
    }
  }
}

void oracle_hgemm_f32acc(const uint16_t* a, const uint16_t* b, uint16_t* c, int M, int N, int K,
                         int b_layout) {
#pragma omp parallel for schedule(static)
  for (int m = 0; m < M; ++m) {
    for (int n = 0; n < N; ++n) {
      float acc = 0.f;
      for (int k = 0; k < K; ++k)
        acc += h2f(a[(size_t)m * K + k]) * bget(b, b_layout, k, n, N, K);
      c[(size_t)m * N + n] = f2h(acc);
    }
  }
}

void oracle_hgemm_f16acc(const uint16_t* a, const uint16_t* b, uint16_t* c, int M, int N, int K,
                         int b_layout, int k_chunk) {
  if (k_chunk <= 0) k_chunk = 16;
#pragma omp parallel for schedule(static)
  for (int m = 0; m < M; ++m) {
    for (int n = 0; n < N; ++n) {
      float acc = 0.f; /* value always representable in fp16 */
      for (int k0 = 0; k0 < K; k0 += k_chunk) {
        float part = 0.f;
        int k1 = k0 + k_chunk < K ? k0 + k_chunk : K;
        for (int k = k0; k < k1; ++k)
          part += h2f(a[(size_t)m * K + k]) * bget(b, b_layout, k, n, N, K);
        acc = round_h(acc + part);
      }
      c[(size_t)m * N + n] = f2h(acc);
    }
  }
}

/* q,k,o: [B,H,N,D]; v: [B,H,N,D] or [B,H,D,N] when v_transposed */
static inline float vget(const uint16_t* v, int vt, int n, int d, int N, int D) {
  return vt ? h2f(v[(size_t)d * N + n]) : h2f(v[(size_t)n * D + d]);
}

void oracle_attn_f32(const uint16_t* q, const uint16_t* k, const uint16_t* v, uint16_t* o, int B,
                     int H, int N, int D, int v_transposed, float scale) {
  if (scale <= 0.f) scale = 1.0f / sqrtf((float)D);
  const size_t hs = (size_t)N * D;
#pragma omp parallel for schedule(dynamic)
  for (int bh = 0; bh < B * H; ++bh) {
    const uint16_t *qh = q + bh * hs, *kh = k + bh * hs, *vh = v + bh * hs;
    uint16_t* oh = o + bh * hs;
    float* s = (float*)malloc(sizeof(float) * N);
    float* acc = (float*)malloc(sizeof(float) * D);
    for (int i = 0; i < N; ++i) {
      float mx = -INFINITY;
      for (int j = 0; j < N; ++j) {
        float d = 0.f;
        for (int x = 0; x < D; ++x) d += h2f(qh[(size_t)i * D + x]) * h2f(kh[(size_t)j * D + x]);
        s[j] = d * scale;
        mx = fmaxf(mx, s[j]);
      }
      float sum = 0.f;
      for (int j = 0; j < N; ++j) {
        s[j] = expf(s[j] - mx);
        sum += s[j];
      }
      for (int x = 0; x < D; ++x) acc[x] = 0.f;
      for (int j = 0; j < N; ++j) {
        const float p = s[j] / sum;
        for (int x = 0; x < D; ++x) acc[x] += p * vget(vh, v_transposed, j, x, N, D);
      }
      for (int x = 0; x < D; ++x) oh[(size_t)i * D + x] = f2h(acc[x]);
    }
    free(s);
    free(acc);
  }
}

void oracle_attn_online(const uint16_t* q, const uint16_t* k, const uint16_t* v, uint16_t* o, int B,
                        int H, int N, int D, int v_transposed, float scale, int Bc, int s_f16) {
  if (scale <= 0.f) scale = 1.0f / sqrtf((float)D);
  if (Bc <= 0) Bc = 64;
  const size_t hs = (size_t)N * D;
#pragma omp parallel for schedule(dynamic)
  for (int bh = 0; bh < B * H; ++bh) {
    const uint16_t *qh = q + bh * hs, *kh = k + bh * hs, *vh = v + bh * hs;
    uint16_t* oh = o + bh * hs;
    float* s = (float*)malloc(sizeof(float) * Bc);
    float* acc = (float*)malloc(sizeof(float) * D);
    for (int i = 0; i < N; ++i) {
      float m_old = -INFINITY, l = 0.f;
      for (int x = 0; x < D; ++x) acc[x] = 0.f;
      for (int j0 = 0; j0 < N; j0 += Bc) {
        const int jn = j0 + Bc < N ? Bc : N - j0;
        float m_new = -INFINITY;
        for (int j = 0; j < jn; ++j) {
          float d = 0.f;
          for (int x = 0; x < D; ++x)
            d += h2f(qh[(size_t)i * D + x]) * h2f(kh[(size_t)(j0 + j) * D + x]);
          if (s_f16) d = round_h(d); /* S kept in fp16 by the f16-acc kernels */
          s[j] = d;
          m_new = fmaxf(m_new, d * scale);
        }
        m_new = fmaxf(m_old, m_new);
        const float resc = expf(m_old - m_new); /* 0 on the first tile */
        float rs = 0.f;
        for (int j = 0; j < jn; ++j) {
          const float p = expf(fmaf(s[j], scale, -m_new));
          rs += p;
          s[j] = round_h(p); /* P is rounded to fp16 before P@V */
        }
        for (int x = 0; x < D; ++x) {
          float pv = 0.f;
          for (int j = 0; j < jn; ++j) pv += s[j] * vget(vh, v_transposed, j0 + j, x, N, D);
          acc[x] = acc[x] * resc + pv;
        }
        l = l * resc + rs;
        m_old = m_new;
      }
      const float inv = 1.0f / l;
      for (int x = 0; x < D; ++x) oh[(size_t)i * D + x] = f2h(acc[x] * inv);
    }
    free(s);
    free(acc);
  }
}

/* ------------------------------------------------------------------ SGEMM (TF32), SURVEY §8f-2 */
static inline float tf32_of(float x, int mode) {
  uint32_t u;
  memcpy(&u, &x, 4);
  /* rna: add half an ulp of the 13 dropped bits.  Inf and NaN are truncated, not rounded, as cvt.rna.tf32.f32 does
   * on sm_90: a NaN loses the low 13 bits of its payload (and becomes inf if its payload lay only there).  Mode 1
   * (truncation) masks NaN payloads the same way. */
  if (mode == 0 && (u & 0x7f800000u) != 0x7f800000u) u += 0x1000u;
  u &= 0xffffe000u;
  memcpy(&x, &u, 4);
  return x;
}

void oracle_tf32_round(const float* x, float* y, size_t n, int mode) {
#pragma omp parallel for schedule(static)
  for (size_t i = 0; i < n; ++i) y[i] = tf32_of(x[i], mode);
}

static inline float bgetf(const float* b, int layout, int k, int n, int N, int K) {
  return layout == 0 ? b[(size_t)k * N + n] : b[(size_t)n * K + k];
}

/* mode: 0 = operands rounded rna (reference), 1 = truncated, 2 = used as they are */
void oracle_sgemm_tf32(const float* a, const float* b, float* c, int M, int N, int K, int b_layout,
                       int mode) {
#pragma omp parallel for schedule(static)
  for (int m = 0; m < M; ++m) {
    for (int n = 0; n < N; ++n) {
      float acc = 0.f;
      for (int k0 = 0; k0 < K; k0 += 8) {
        double part = 0.0;
        const int k1 = k0 + 8 < K ? k0 + 8 : K;
        for (int k = k0; k < k1; ++k) {
          float x = a[(size_t)m * K + k], y = bgetf(b, b_layout, k, n, N, K);
          if (mode < 2) { x = tf32_of(x, mode); y = tf32_of(y, mode); }
          part += (double)x * (double)y;
        }
        acc = (float)((double)acc + part);
      }
      c[(size_t)m * N + n] = acc;
    }
  }
}

void oracle_sgemm_f64(const float* a, const float* b, double* c, int M, int N, int K, int b_layout,
                      int mode) {
#pragma omp parallel for schedule(static)
  for (int m = 0; m < M; ++m) {
    for (int n = 0; n < N; ++n) {
      double acc = 0.0;
      for (int k = 0; k < K; ++k) {
        float x = a[(size_t)m * K + k], y = bgetf(b, b_layout, k, n, N, K);
        if (mode < 2) { x = tf32_of(x, mode); y = tf32_of(y, mode); }
        acc += (double)x * (double)y;
      }
      c[(size_t)m * N + n] = acc;
    }
  }
}

/* ------------------------------------------------------------------ merge_attn_states, SURVEY §8f-3 */
static inline float bf2f(uint16_t h) {
  uint32_t u = (uint32_t)h << 16;
  float f;
  memcpy(&f, &u, 4);
  return f;
}
static inline uint16_t f2bf(float f) { /* round to nearest even, like __float2bfloat16 */
  uint32_t u;
  memcpy(&u, &f, 4);
  if ((u & 0x7fffffffu) > 0x7f800000u) return 0x7fff; /* nan */
  u += 0x7fffu + ((u >> 16) & 1u);
  return (uint16_t)(u >> 16);
}

/* dtype: 0 fp32, 1 fp16, 2 bf16 (element size 4 / 2 / 2).  out_lse may be NULL. */
void oracle_merge_attn_states(void* out, float* out_lse, const void* p_out, const float* p_lse,
                              const void* s_out, const float* s_lse, int T, int H, int D, int dtype) {
#pragma omp parallel for schedule(static)
  for (int t = 0; t < T; ++t) {
    for (int h = 0; h < H; ++h) {
      float pl = p_lse[(size_t)h * T + t], sl = s_lse[(size_t)h * T + t];
      if (isinf(pl)) pl = -INFINITY;
      if (isinf(sl)) sl = -INFINITY;
      const float m = fmaxf(pl, sl);
      const float pe = expf(pl - m), se = expf(sl - m);
      const float sum = pe + se;
      const float ps = pe / sum, ss = se / sum;
      const size_t base = ((size_t)t * H + h) * D;
      for (int d = 0; d < D; ++d) {
        float x, y;
        if (dtype == 0) { x = ((const float*)p_out)[base + d]; y = ((const float*)s_out)[base + d]; }
        else if (dtype == 1) { x = h2f(((const uint16_t*)p_out)[base + d]); y = h2f(((const uint16_t*)s_out)[base + d]); }
        else { x = bf2f(((const uint16_t*)p_out)[base + d]); y = bf2f(((const uint16_t*)s_out)[base + d]); }
        const float o = fmaf(x, ps, y * ss);
        if (dtype == 0) ((float*)out)[base + d] = o;
        else if (dtype == 1) ((uint16_t*)out)[base + d] = f2h(o);
        else ((uint16_t*)out)[base + d] = f2bf(o);
      }
      if (out_lse) out_lse[(size_t)h * T + t] = logf(sum) + m;
    }
  }
}


/* ---------------------------------------------------------------------------------------------
 * rope / rms_norm (SURVEY §8f-4)
 * ------------------------------------------------------------------------------------------- */
void oracle_rope_f32(const float* x, float* out, int seq_len, int hidden) {
  const int n = hidden / 2;
#pragma omp parallel for
  for (int p = 0; p < seq_len; ++p)
    for (int i = 0; i < n; ++i) {
      const float x1 = x[(size_t)p * hidden + 2 * i], x2 = x[(size_t)p * hidden + 2 * i + 1];
      const float exp_v = 1.0f / powf(10000.0f, 2 * i / (n * 2.0f));
      const float sin_v = sinf(p * exp_v), cos_v = cosf(p * exp_v);
      out[(size_t)p * hidden + 2 * i] = x1 * cos_v - x2 * sin_v;
      out[(size_t)p * hidden + 2 * i + 1] = x1 * sin_v + x2 * cos_v;
    }
}

/* dtype 0: float in/out; 1: fp16 bit patterns in/out.  Statistics in fp32, summed in index order. */
void oracle_rms_norm(const void* x, void* y, float g, int rows, int K, int dtype) {
#pragma omp parallel for
  for (int r = 0; r < rows; ++r) {
    float var = 0.f;
    for (int k = 0; k < K; ++k) {
      const float v = dtype == 0 ? ((const float*)x)[(size_t)r * K + k] : h2f(((const uint16_t*)x)[(size_t)r * K + k]);
      var += v * v;
    }
    const float s = 1.0f / sqrtf(var / (float)K + 1e-5f);
    for (int k = 0; k < K; ++k) {
      if (dtype == 0) {
        ((float*)y)[(size_t)r * K + k] = (((const float*)x)[(size_t)r * K + k] * s) * g;
      } else {
        const float v = h2f(((const uint16_t*)x)[(size_t)r * K + k]);
        ((uint16_t*)y)[(size_t)r * K + k] = f2h((v * s) * g);
      }
    }
  }
}
