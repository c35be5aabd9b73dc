// merge_capi.cu — merge_attn_states (SURVEY §8f-3): combine two partial attention results
// (prefix / suffix of a split KV sequence) from their outputs and log-sum-exps, section 2.2 of
// arXiv 2501.01005.  Replaces merge_attn_states_cuda of the reference
// (kernels/openai-triton/merge-attn-states/cuda_merge_attn_states.cu:19-95, launcher :120-146).
//
//   out[t,h,:]   = prefix[t,h,:] * w_prefix + suffix[t,h,:] * w_suffix
//   w_x          = exp(lse_x - m) / (exp(lse_prefix - m) + exp(lse_suffix - m)),  m = max of the two lse
//   out_lse[h,t] = log(exp(lse_prefix - m) + exp(lse_suffix - m)) + m          (+inf lse counts as -inf)
//
// HBM-bound element-wise work: 3 * D * sizeof(T) + 12 bytes per (token, head) row.
//
// Layout: one thread per 16-byte pack of the output, one-shot grid (packs / 256 CTAs of 256 threads, 32-bit index
// arithmetic whenever the pack count fits): both 128-bit L1-bypassing loads of a pack are issued before the two
// lse values are fetched.  Every thread of a row evaluates the row's two weights itself (a warp executes those few
// instructions once for all its lanes either way).
//
// Numerics: libdevice expf / logf, IEEE division, and per element one multiply and one fused
// multiply-add in fp32 — the operations (not the code) of the reference's kernel, so the outputs
// agree with the recorded reference outputs bit for bit (tests/test_merge_gpu.py).
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <cmath>
#include <limits>

#include "capi_common.cuh"
#include "sm90_ptx.cuh"

namespace {

using b200::host::fail;
using b200::ld_stream;
using b200::st_stream;

// one 16-byte pack: out = prefix * wp + suffix * ws, element type T, arithmetic in fp32
template <typename T>
struct Pack;
template <>
struct Pack<float> {
  static __device__ __forceinline__ uint4 blend(const uint4& a, const uint4& b, float wp, float ws) {
    uint4 r;
    r.x = __float_as_uint(fmaf(__uint_as_float(a.x), wp, __fmul_rn(__uint_as_float(b.x), ws)));
    r.y = __float_as_uint(fmaf(__uint_as_float(a.y), wp, __fmul_rn(__uint_as_float(b.y), ws)));
    r.z = __float_as_uint(fmaf(__uint_as_float(a.z), wp, __fmul_rn(__uint_as_float(b.z), ws)));
    r.w = __float_as_uint(fmaf(__uint_as_float(a.w), wp, __fmul_rn(__uint_as_float(b.w), ws)));
    return r;
  }
};
template <>
struct Pack<__half> {
  static __device__ __forceinline__ uint32_t two(uint32_t a, uint32_t b, float wp, float ws) {
    const float2 fa = __half22float2(*reinterpret_cast<const __half2*>(&a));
    const float2 fb = __half22float2(*reinterpret_cast<const __half2*>(&b));
    const __half lo = __float2half(fmaf(fa.x, wp, __fmul_rn(fb.x, ws)));
    const __half hi = __float2half(fmaf(fa.y, wp, __fmul_rn(fb.y, ws)));
    const __half2 h = __halves2half2(lo, hi);
    return *reinterpret_cast<const uint32_t*>(&h);
  }
  static __device__ __forceinline__ uint4 blend(const uint4& a, const uint4& b, float wp, float ws) {
    return make_uint4(two(a.x, b.x, wp, ws), two(a.y, b.y, wp, ws), two(a.z, b.z, wp, ws), two(a.w, b.w, wp, ws));
  }
};
template <>
struct Pack<__nv_bfloat16> {
  static __device__ __forceinline__ uint32_t two(uint32_t a, uint32_t b, float wp, float ws) {
    // a bf16 is the upper half of its fp32
    const float a0 = __uint_as_float(a << 16), a1 = __uint_as_float(a & 0xffff0000u);
    const float b0 = __uint_as_float(b << 16), b1 = __uint_as_float(b & 0xffff0000u);
    const __nv_bfloat16 lo = __float2bfloat16(fmaf(a0, wp, __fmul_rn(b0, ws)));
    const __nv_bfloat16 hi = __float2bfloat16(fmaf(a1, wp, __fmul_rn(b1, ws)));
    return static_cast<uint32_t>(__bfloat16_as_ushort(lo)) | (static_cast<uint32_t>(__bfloat16_as_ushort(hi)) << 16);
  }
  static __device__ __forceinline__ uint4 blend(const uint4& a, const uint4& b, float wp, float ws) {
    return make_uint4(two(a.x, b.x, wp, ws), two(a.y, b.y, wp, ws), two(a.z, b.z, wp, ws), two(a.w, b.w, wp, ws));
  }
};

// Idx: 32-bit pack indices whenever they fit (64-bit division is emulated).  The grid has one thread per pack, so the
// grid-stride loop runs its body at most once per thread.
template <typename T, typename Idx>
__global__ void __launch_bounds__(256)
merge_attn_states_kernel(T* __restrict__ out, float* __restrict__ out_lse, const T* __restrict__ prefix,
                         const float* __restrict__ prefix_lse, const T* __restrict__ suffix,
                         const float* __restrict__ suffix_lse, unsigned num_tokens, unsigned num_heads,
                         unsigned packs_per_row) {
  const Idx n_packs = static_cast<Idx>(num_tokens) * num_heads * packs_per_row;
  const Idx step = static_cast<Idx>(gridDim.x) * blockDim.x;
  for (Idx pk = static_cast<Idx>(blockIdx.x) * blockDim.x + threadIdx.x; pk < n_packs; pk += step) {
    // the two data packs first: they are the long-latency part
    const uint4 a = ld_stream(reinterpret_cast<const uint4*>(prefix) + pk);
    const uint4 b = ld_stream(reinterpret_cast<const uint4*>(suffix) + pk);
    const Idx row = pk / packs_per_row;                              // = token * num_heads + head
    const unsigned token = static_cast<unsigned>(row / num_heads);
    const unsigned head = static_cast<unsigned>(row - static_cast<Idx>(token) * num_heads);
    const size_t at = static_cast<size_t>(head) * num_tokens + token;   // lse tensors are [heads, tokens]
    float lp = __ldg(prefix_lse + at), ls = __ldg(suffix_lse + at);
    if (isinf(lp)) lp = -INFINITY;       // +inf marks a part without keys (reference :51-52)
    if (isinf(ls)) ls = -INFINITY;
    const float top = fmaxf(lp, ls);
    const float ep = expf(lp - top), es = expf(ls - top);
    const float denom = ep + es;
    const uint4 r = Pack<T>::blend(a, b, ep / denom, es / denom);
    st_stream(reinterpret_cast<uint4*>(out) + pk, r);
    if (out_lse != nullptr && pk == row * packs_per_row) out_lse[at] = logf(denom) + top;   // first pack of the row
  }
}

template <typename T>
int launch_merge(void* out, float* out_lse, const void* prefix, const float* prefix_lse, const void* suffix,
                 const float* suffix_lse, int num_tokens, int num_heads, int head_size, cudaStream_t stream) {
  constexpr int kPack = 16 / sizeof(T);
  if (head_size % kPack != 0)
    return fail(B200_EINVAL, "headsize must be multiple of pack_size:%d", kPack);   // reference :131-132
  const unsigned packs = static_cast<unsigned>(head_size / kPack);
  const size_t total = static_cast<size_t>(num_tokens) * num_heads * packs;
  const size_t blocks = (total + 255) / 256;
  if (blocks > 0x7FFFFFFFull) return fail(B200_EINVAL, "merge_attn_states: too many packs");
  const unsigned g = static_cast<unsigned>(blocks);
  T* o = static_cast<T*>(out);
  const T* pa = static_cast<const T*>(prefix);
  const T* pb = static_cast<const T*>(suffix);
  const unsigned nt = static_cast<unsigned>(num_tokens), nh = static_cast<unsigned>(num_heads);
  // the grid-stride loop adds up to one stride past `total`: keep that inside 32 bits too
  const bool idx32 = total + blocks * 256 < 0xFFFFFFFFull;
  if (idx32) merge_attn_states_kernel<T, unsigned><<<g, 256, 0, stream>>>(o, out_lse, pa, prefix_lse, pb, suffix_lse, nt, nh, packs);
  else merge_attn_states_kernel<T, size_t><<<g, 256, 0, stream>>>(o, out_lse, pa, prefix_lse, pb, suffix_lse, nt, nh, packs);
  B200_CUDA_OK(cudaGetLastError());
  b200::host::count_launch();
  return 0;
}

}  // namespace

extern "C" int b200_merge_attn_states(void* output, float* output_lse, const void* prefix_output,
                                      const float* prefix_lse, const void* suffix_output,
                                      const float* suffix_lse, int num_tokens, int num_heads, int head_size,
                                      int dtype, void* stream_) {
  if (!output || !prefix_output || !prefix_lse || !suffix_output || !suffix_lse)
    return fail(B200_EINVAL, "merge_attn_states: null pointer");
  if (num_tokens < 0 || num_heads <= 0 || head_size <= 0)
    return fail(B200_EINVAL, "merge_attn_states: bad shape tokens=%d heads=%d head_size=%d", num_tokens, num_heads,
                head_size);
  if (((reinterpret_cast<uintptr_t>(output) | reinterpret_cast<uintptr_t>(prefix_output) |
        reinterpret_cast<uintptr_t>(suffix_output)) & 15u) != 0)
    return fail(B200_EINVAL, "merge_attn_states: tensors must be 16-byte aligned");
  if (num_tokens == 0) return 0;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  switch (dtype) {
    case B200_DTYPE_F32:
      return launch_merge<float>(output, output_lse, prefix_output, prefix_lse, suffix_output, suffix_lse,
                                 num_tokens, num_heads, head_size, stream);
    case B200_DTYPE_F16:
      return launch_merge<__half>(output, output_lse, prefix_output, prefix_lse, suffix_output, suffix_lse,
                                  num_tokens, num_heads, head_size, stream);
    case B200_DTYPE_BF16:
      return launch_merge<__nv_bfloat16>(output, output_lse, prefix_output, prefix_lse, suffix_output, suffix_lse,
                                         num_tokens, num_heads, head_size, stream);
    default:
      return fail(B200_ENOTSUP, "Unsupported data type of O: %d", dtype);   // reference :107
  }
}
