// elementwise_capi.cu — the two HBM-bound steps that sit either side of attention in the reference's
// catalogue (SURVEY §8f-4): rotary position embedding and RMS normalisation.
//
//   rope      kernels/rope/rope.cu:20-71 (rope_f32, rope_f32_v2, rope_f32x4_pack; host side :88-125)
//             x, out: [seq_len, hidden] fp32; pair i = (x[2i], x[2i+1]) of the row at position p is rotated
//             by the angle p / theta^(2i/hidden), theta = 10000.
//   rms_norm  kernels/rms-norm/rms_norm.cu:55-110 (fp32), :161-415 (fp16 storage, fp16 or fp32 statistics)
//             x, y: [rows, K]; y = x * rsqrt(mean(x^2) + 1e-5) * g with a scalar gain g.
//
// Both are pure streaming work (8 / 2*sizeof(T) bytes per element), so the kernels are persistent
// grid-stride loops over 16-byte packs with L1-bypassing loads/stores; what differs from the
// reference is where the transcendental work goes:
//   * rope: a thread keeps ONE column group for its whole life, so 1/theta^(2i/hidden) (a powf and a
//     division per pair in the reference) is evaluated once per thread and the per-element cost is one
//     sincosf — otherwise the kernel would be issue-bound, not HBM-bound;
//   * rms_norm: a row lives in the registers of one warp (K <= 2048 halfs / 1024 floats) or one CTA
//     (up to 8x that): x is read from HBM exactly once, the statistics are always fp32 (the reference's
//     *_f16 variants accumulate in fp16; fp32 is at least as accurate for every one of its op names).
#include <cuda_fp16.h>

#include <cmath>

#include "capi_common.cuh"

namespace {

using b200::host::fail;

__device__ __forceinline__ uint4 ld_stream(const void* p) {
  uint4 v;
  asm volatile("ld.global.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p));
  return v;
}
__device__ __forceinline__ void st_stream(void* p, const uint4& v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(v.x), "r"(v.y),
               "r"(v.z), "r"(v.w)
               : "memory");
}

// ------------------------------------------------------------------------------------------------
// rope: one float4 (= two pairs) per thread per step; `lanes` threads cover one row of `groups` =
// hidden/4 float4 groups (lanes = groups when 256 % groups == 0, else 256 and the row is strided)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
rope_f32_kernel(const float* __restrict__ x, float* __restrict__ out, unsigned seq_len, unsigned groups,
                unsigned lanes, float hidden_f) {
  const unsigned rows_per_step = 256u / lanes;
  const unsigned sub = threadIdx.x / lanes;
  const unsigned col0 = threadIdx.x - sub * lanes;
  constexpr float kLog2Theta = 13.287712379549449f;      // log2(10000)
  for (unsigned col = col0; col < groups; col += lanes) {
    // angular frequencies of the two pairs of this column group: theta^(-2i/hidden), i = 2*col, 2*col+1
    const float f0 = exp2f(-kLog2Theta * (static_cast<float>(4u * col) / hidden_f));
    const float f1 = exp2f(-kLog2Theta * (static_cast<float>(4u * col + 2u) / hidden_f));
    for (unsigned pos = blockIdx.x * rows_per_step + sub; pos < seq_len; pos += gridDim.x * rows_per_step) {
      const size_t at = static_cast<size_t>(pos) * groups + col;
      const uint4 v = ld_stream(reinterpret_cast<const uint4*>(x) + at);
      float s0, c0, s1, c1;
      sincosf(static_cast<float>(pos) * f0, &s0, &c0);
      sincosf(static_cast<float>(pos) * f1, &s1, &c1);
      const float a0 = __uint_as_float(v.x), b0 = __uint_as_float(v.y);
      const float a1 = __uint_as_float(v.z), b1 = __uint_as_float(v.w);
      uint4 r;
      r.x = __float_as_uint(a0 * c0 - b0 * s0);
      r.y = __float_as_uint(a0 * s0 + b0 * c0);
      r.z = __float_as_uint(a1 * c1 - b1 * s1);
      r.w = __float_as_uint(a1 * s1 + b1 * c1);
      st_stream(reinterpret_cast<uint4*>(out) + at, r);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// rope on fp16 [rows_total = B*H*N, D] tensors of the attention layout: the position of a row is its
// index inside its (batch, head) sequence (row % N); q and k are rotated by ONE launch (blockIdx.y
// selects the tensor).  A thread owns one 16-byte pack = four (even, odd) pairs of a fixed column group.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
rope_qk_f16_kernel(const __half* __restrict__ q, const __half* __restrict__ k, __half* __restrict__ q_out,
                   __half* __restrict__ k_out, unsigned rows_total, unsigned seq_len, unsigned groups,
                   unsigned lanes, float head_dim_f) {
  const __half* x = blockIdx.y == 0 ? q : k;
  __half* out = blockIdx.y == 0 ? q_out : k_out;
  const unsigned rows_per_step = 256u / lanes;
  const unsigned sub = threadIdx.x / lanes;
  const unsigned col0 = threadIdx.x - sub * lanes;
  constexpr float kLog2Theta = 13.287712379549449f;      // log2(10000)
  for (unsigned col = col0; col < groups; col += lanes) {
    float f[4];
#pragma unroll
    for (int i = 0; i < 4; ++i)     // pair index 4*col + i -> theta^(-2*pair/D)
      f[i] = exp2f(-kLog2Theta * (static_cast<float>(2u * (4u * col + i)) / head_dim_f));
    for (unsigned row = blockIdx.x * rows_per_step + sub; row < rows_total; row += gridDim.x * rows_per_step) {
      const float pos = static_cast<float>(row % seq_len);
      const size_t at = static_cast<size_t>(row) * groups + col;
      const uint4 v = ld_stream(reinterpret_cast<const uint4*>(x) + at);
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
      uint32_t r[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 xy = __half22float2(*reinterpret_cast<const __half2*>(&w[i]));
        float sn, cs;
        sincosf(pos * f[i], &sn, &cs);
        const __half2 h = __float22half2_rn(make_float2(xy.x * cs - xy.y * sn, xy.x * sn + xy.y * cs));
        r[i] = *reinterpret_cast<const uint32_t*>(&h);
      }
      st_stream(reinterpret_cast<uint4*>(out) + at, make_uint4(r[0], r[1], r[2], r[3]));
    }
  }
}

// ------------------------------------------------------------------------------------------------
// rms_norm: kGroup threads own one row (32 = a warp, 256 = the CTA), up to kMaxPacks 16-byte packs each
// ------------------------------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ float pack_sumsq(const uint4& v);
template <>
__device__ __forceinline__ float pack_sumsq<float>(const uint4& v) {
  const float a = __uint_as_float(v.x), b = __uint_as_float(v.y), c = __uint_as_float(v.z), d = __uint_as_float(v.w);
  return a * a + b * b + c * c + d * d;
}
template <>
__device__ __forceinline__ float pack_sumsq<__half>(const uint4& v) {
  float s = 0.f;
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&w[i]));
    s += f.x * f.x + f.y * f.y;
  }
  return s;
}
template <typename T>
__device__ __forceinline__ uint4 pack_scale(const uint4& v, float s, float g);
template <>
__device__ __forceinline__ uint4 pack_scale<float>(const uint4& v, float s, float g) {
  return make_uint4(__float_as_uint(__uint_as_float(v.x) * s * g), __float_as_uint(__uint_as_float(v.y) * s * g),
                    __float_as_uint(__uint_as_float(v.z) * s * g), __float_as_uint(__uint_as_float(v.w) * s * g));
}
template <>
__device__ __forceinline__ uint4 pack_scale<__half>(const uint4& v, float s, float g) {
  uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&w[i]));
    const __half2 h = __float22half2_rn(make_float2(f.x * s * g, f.y * s * g));
    w[i] = *reinterpret_cast<const uint32_t*>(&h);
  }
  return make_uint4(w[0], w[1], w[2], w[3]);
}

constexpr int kMaxPacks = 8;

template <typename T, int kGroup>
__global__ void __launch_bounds__(256)
rms_norm_kernel(const T* __restrict__ x, T* __restrict__ y, float g, unsigned rows, unsigned packs_per_row,
                float inv_k) {
  __shared__ float warp_part[8];
  const unsigned lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  const unsigned in_group = kGroup == 32 ? lane : threadIdx.x;
  const size_t group_id = kGroup == 32 ? (static_cast<size_t>(blockIdx.x) * 8 + warp) : blockIdx.x;
  const size_t n_groups = kGroup == 32 ? static_cast<size_t>(gridDim.x) * 8 : gridDim.x;
  for (size_t row = group_id; row < rows; row += n_groups) {
    const uint4* px = reinterpret_cast<const uint4*>(x) + row * packs_per_row;
    uint4* py = reinterpret_cast<uint4*>(y) + row * packs_per_row;
    uint4 v[kMaxPacks];
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < kMaxPacks; ++i) {
      const unsigned c = in_group + i * kGroup;
      if (c < packs_per_row) v[i] = ld_stream(px + c);
    }
#pragma unroll
    for (int i = 0; i < kMaxPacks; ++i) {
      const unsigned c = in_group + i * kGroup;
      if (c < packs_per_row) ss += pack_sumsq<T>(v[i]);
    }
#pragma unroll
    for (int m = 16; m >= 1; m >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, m);
    if constexpr (kGroup == 256) {
      __syncthreads();                         // warp_part of the previous row has been consumed
      if (lane == 0) warp_part[warp] = ss;
      __syncthreads();
      ss = 0.f;
#pragma unroll
      for (int w = 0; w < 8; ++w) ss += warp_part[w];
    }
    const float s = rsqrtf(ss * inv_k + 1e-5f);
#pragma unroll
    for (int i = 0; i < kMaxPacks; ++i) {
      const unsigned c = in_group + i * kGroup;
      if (c < packs_per_row) st_stream(py + c, pack_scale<T>(v[i], s, g));
    }
  }
}

template <typename T>
int launch_rms(const void* x, void* y, float g, int rows, int K, cudaStream_t stream) {
  constexpr int kPack = 16 / sizeof(T);
  if (K % kPack != 0) return fail(B200_EINVAL, "rms_norm: K (%d) must be a multiple of %d", K, kPack);
  const unsigned packs = static_cast<unsigned>(K / kPack);
  const size_t cap = static_cast<size_t>(b200::host::sm_count()) * 8;
  if (packs <= 32u * kMaxPacks) {
    size_t blocks = (static_cast<size_t>(rows) + 7) / 8;
    if (blocks > cap) blocks = cap;
    rms_norm_kernel<T, 32><<<static_cast<unsigned>(blocks), 256, 0, stream>>>(
        static_cast<const T*>(x), static_cast<T*>(y), g, static_cast<unsigned>(rows), packs, 1.0f / static_cast<float>(K));
  } else if (packs <= 256u * kMaxPacks) {
    size_t blocks = static_cast<size_t>(rows);
    if (blocks > cap) blocks = cap;
    rms_norm_kernel<T, 256><<<static_cast<unsigned>(blocks), 256, 0, stream>>>(
        static_cast<const T*>(x), static_cast<T*>(y), g, static_cast<unsigned>(rows), packs, 1.0f / static_cast<float>(K));
  } else {
    return fail(B200_ENOTSUP, "rms_norm: K = %d exceeds %d elements per row", K, 256 * kMaxPacks * kPack);
  }
  B200_CUDA_OK(cudaGetLastError());
  b200::host::count_launch();
  return 0;
}

}  // namespace

extern "C" {

int b200_rope_f32(const float* x, float* out, int seq_len, int hidden, void* stream_) {
  if (!x || !out) return fail(B200_EINVAL, "rope: null pointer");
  if (seq_len <= 0 || hidden <= 0) return fail(B200_EINVAL, "rope: bad shape seq_len=%d hidden=%d", seq_len, hidden);
  if (hidden % 4 != 0) return fail(B200_EINVAL, "rope: hidden (%d) must be a multiple of 4", hidden);
  if (((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(out)) & 15u) != 0)
    return fail(B200_EINVAL, "rope: x and out must be 16-byte aligned");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const unsigned groups = static_cast<unsigned>(hidden / 4);
  const unsigned lanes = (groups <= 256u && 256u % groups == 0u) ? groups : 256u;
  const unsigned rows_per_step = 256u / lanes;
  // one-shot grid (one row step per CTA; the loop in the kernel only wraps beyond 2^31 CTAs): for streaming kernels the
  // block scheduler beat a persistent grid-stride loop (measured on the B200 this was first written for; not re-measured)
  size_t blocks = (static_cast<size_t>(seq_len) + rows_per_step - 1) / rows_per_step;
  const size_t cap = 0x7FFFFFFFull;
  if (blocks > cap) blocks = cap;
  rope_f32_kernel<<<static_cast<unsigned>(blocks), 256, 0, stream>>>(x, out, static_cast<unsigned>(seq_len), groups,
                                                                    lanes, static_cast<float>(hidden));
  B200_CUDA_OK(cudaGetLastError());
  b200::host::count_launch();
  return 0;
}

int b200_rope_qk_f16(const void* q, const void* k, void* q_out, void* k_out, int B, int H, int N, int D,
                     void* stream_) {
  if (!q || !k || !q_out || !k_out) return fail(B200_EINVAL, "rope_qk: null pointer");
  if (B <= 0 || H <= 0 || N <= 0 || D <= 0) return fail(B200_EINVAL, "rope_qk: bad shape B=%d H=%d N=%d D=%d", B, H, N, D);
  if (D % 8 != 0) return fail(B200_EINVAL, "rope_qk: D (%d) must be a multiple of 8", D);
  const size_t rows = static_cast<size_t>(B) * H * N;
  if (rows > 0xFFFFFFFFull) return fail(B200_EINVAL, "rope_qk: B*H*N exceeds 2^32 rows");
  if (((reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(k) | reinterpret_cast<uintptr_t>(q_out) |
        reinterpret_cast<uintptr_t>(k_out)) & 15u) != 0)
    return fail(B200_EINVAL, "rope_qk: tensors must be 16-byte aligned");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const unsigned groups = static_cast<unsigned>(D / 8);
  const unsigned lanes = (groups <= 256u && 256u % groups == 0u) ? groups : 256u;
  const unsigned rows_per_step = 256u / lanes;
  size_t blocks = (rows + rows_per_step - 1) / rows_per_step;
  // persistent grid here (x 2 tensors in grid.y = 8 CTAs per SM): with four pairs per pack this kernel is bound by
  // the sincosf / exp2f work, and a thread that keeps its column group amortises the frequencies over many rows
  // (measured on the B200 this was first written for; not re-measured on H100)
  const size_t cap = static_cast<size_t>(b200::host::sm_count()) * 4;
  if (blocks > cap) blocks = cap;
  rope_qk_f16_kernel<<<dim3(static_cast<unsigned>(blocks), 2, 1), 256, 0, stream>>>(
      static_cast<const __half*>(q), static_cast<const __half*>(k), static_cast<__half*>(q_out),
      static_cast<__half*>(k_out), static_cast<unsigned>(rows), static_cast<unsigned>(N), groups, lanes,
      static_cast<float>(D));
  B200_CUDA_OK(cudaGetLastError());
  b200::host::count_launch();
  return 0;
}

int b200_rms_norm(const void* x, void* y, float g, int rows, int K, int dtype, void* stream_) {
  if (!x || !y) return fail(B200_EINVAL, "rms_norm: null pointer");
  if (rows <= 0 || K <= 0) return fail(B200_EINVAL, "rms_norm: bad shape rows=%d K=%d", rows, K);
  if (((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 15u) != 0)
    return fail(B200_EINVAL, "rms_norm: x and y must be 16-byte aligned");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  switch (dtype) {
    case B200_DTYPE_F32: return launch_rms<float>(x, y, g, rows, K, stream);
    case B200_DTYPE_F16: return launch_rms<__half>(x, y, g, rows, K, stream);
    default: return fail(B200_ENOTSUP, "rms_norm: unsupported dtype %d", dtype);
  }
}

}  // extern "C"
