// attn_launch.cuh — the host launch of one attention kernel, shared by attn_capi.cu (the C entries and the fp16
// kernels) and the translation units of the other kernels (attn_bf16.cu, attn_fp8kv_*.cu, attn_varlen.cu), which
// compile in parallel.
#pragma once
#include <string.h>

#include "capi_common.cuh"
#include "attn_sm90.cuh"

namespace b200 {
namespace attn {

// One attention kernel on a grid of (query tiles x slabs, K/V heads, splits); attr_smem[dev] remembers the dynamic
// shared memory the kernel was allowed on each device.
template <typename... KParams, typename... Args>
int launch_kernel(void (*kern)(KParams...), int* attr_smem, const Params& p, int qtiles, int BH, int splits,
                  int threads, int smem, cudaStream_t stream, const Args&... args) {
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev >= 0 && dev < 64 && attr_smem[dev] < smem) {
    B200_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    attr_smem[dev] = smem;
  }
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(static_cast<unsigned>(qtiles * p.slabs), static_cast<unsigned>(BH), static_cast<unsigned>(splits));
  cfg.blockDim = dim3(threads, 1, 1);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attrs[1];
  attrs[0].id = cudaLaunchAttributeClusterDimension;   // the slabs of one query tile (fused RMS norm)
  attrs[0].val.clusterDim.x = (p.rms_g > 0.f) ? static_cast<unsigned>(p.slabs) : 1u;
  attrs[0].val.clusterDim.y = 1;
  attrs[0].val.clusterDim.z = 1;
  cfg.attrs = attrs;
  cfg.numAttrs = 1;
  B200_CUDA_OK(cudaLaunchKernelEx(&cfg, kern, args...));
  host::count_launch();
  return 0;
}

// The bf16 kernel of the family (kDS, kBN, kWG) (attn_bf16.cu): attn_fwd_paged_bf16_kernel with pages, else
// attn_fwd_seqlens_bf16_kernel (null length arrays in lens for a dense call).
template <int kDS, int kBN, int kWG>
int launch_attn_bf16(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, const Params& p, int qtiles,
                     int BH, int smem, bool causal, int splits, const Lens& lens, const Pages* pages,
                     cudaStream_t stream);

// The fp8-K/V kernel of the family (kDS, kBN, kWG) with T = __half or __nv_bfloat16 Q and O (attn_fp8kv_f16.cu,
// attn_fp8kv_bf16.cu): attn_fwd_fp8kv_paged_kernel with pages, else attn_fwd_fp8kv_seqlens_kernel.
template <typename T, int kDS, int kBN, int kWG>
int launch_attn_fp8kv(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, const Params& p, int qtiles,
                      int BH, int smem, bool causal, int splits, const Lens& lens, const Pages* pages, float v_scale,
                      cudaStream_t stream);

// The packed variable-length kernel of the family (kDS, kBN, kWG) with T = __half or __nv_bfloat16 (attn_varlen.cu):
// attn_varlen_kernel with paged K/V when pages is given, else with packed K/V.
template <typename T, int kDS, int kBN, int kWG>
int launch_attn_varlen(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, const Params& p, int qtiles,
                       int BH, int smem, bool causal, const Varlen& vl, const Pages* pages, cudaStream_t stream);

}  // namespace attn
}  // namespace b200
