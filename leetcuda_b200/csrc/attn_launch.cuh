// attn_launch.cuh — the host launch of the attention kernels, shared by attn_capi.cu (the C entries and the fp16
// kernels) and the translation units of the other kernels (attn_bf16.cu, attn_fp8kv_*.cu, attn_varlen.cu), which
// compile in parallel.
#pragma once
#include <string.h>

#include <type_traits>

#include "capi_common.cuh"
#include "attn_sm90.cuh"

namespace b200 {
namespace attn {

// Kernel shape per head dim (attn_sm90.cuh):
//   D <= 64        one 64-column slab, 128-key blocks, two consumer warpgroups (128 query rows)
//   64 < D <= 128  one 128-column slab, 64-key blocks, two consumer warpgroups
//   128 < D        256-column slabs (S recomputed per slab), 64-key blocks, one consumer warpgroup (64 query rows)
// The S, P and O fragments of a consumer thread have to fit its registers: ptxas gives a 384-thread CTA
// 168 per thread, a 256-thread CTA 255 (O of a 256-column slab alone takes 128).
template <int DS, int BN, int WG>
struct Fam {
  static constexpr int kDS = DS, kBN = BN, kWG = WG;
};

// f(Fam<kDS, kBN, kWG>{}) for the family of head dim D
template <typename F>
auto with_family(int D, F&& f) {
  if (D <= 64) return f(Fam<64, 128, 2>{});
  if (D <= 128) return f(Fam<128, 64, 2>{});
  return f(Fam<256, 64, 1>{});
}

// f(causal, flag) with both runtime flags as std::bool_constant, to become kernel template arguments
template <typename F>
auto with_flags(bool causal, bool flag, F&& f) {
  using Y = std::true_type;
  using N = std::false_type;
  if (flag) return causal ? f(Y{}, Y{}) : f(N{}, Y{});
  return causal ? f(Y{}, N{}) : f(N{}, N{});
}

// What every attention launch shares: the kernels' leading arguments (the Q, K and V tensor maps and p), the grid
// (query tiles x slabs, K/V heads, splits), the dynamic shared memory and the stream.
struct Launch {
  const CUtensorMap& tq;
  const CUtensorMap& tk;
  const CUtensorMap& tv;
  const Params& p;
  int qtiles, BH, splits, smem;
  cudaStream_t stream;
};

// Kern(tq, tk, tv, p, args...) with threads<kWG>() threads per CTA.  attr_smem remembers, per device, the dynamic
// shared memory Kern was allowed.
template <auto Kern, int kWG, typename... Args>
int launch(const Launch& l, const Args&... args) {
  static int attr_smem[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev >= 0 && dev < 64 && attr_smem[dev] < l.smem) {
    B200_CUDA_OK(cudaFuncSetAttribute(Kern, cudaFuncAttributeMaxDynamicSharedMemorySize, l.smem));
    attr_smem[dev] = l.smem;
  }
  const Params& p = l.p;
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(static_cast<unsigned>(l.qtiles * p.slabs), static_cast<unsigned>(l.BH),
                     static_cast<unsigned>(l.splits));
  cfg.blockDim = dim3(threads<kWG>(), 1, 1);
  cfg.dynamicSmemBytes = l.smem;
  cfg.stream = l.stream;
  cudaLaunchAttribute attrs[1];
  attrs[0].id = cudaLaunchAttributeClusterDimension;   // the slabs of one query tile (fused RMS norm)
  attrs[0].val.clusterDim.x = (p.rms_g > 0.f) ? static_cast<unsigned>(p.slabs) : 1u;
  attrs[0].val.clusterDim.y = 1;
  attrs[0].val.clusterDim.z = 1;
  cfg.attrs = attrs;
  cfg.numAttrs = 1;
  B200_CUDA_OK(cudaLaunchKernelEx(&cfg, Kern, l.tq, l.tk, l.tv, p, args...));
  host::count_launch();
  return 0;
}

// The bf16 kernel of the family of p.D (attn_bf16.cu): attn_fwd_paged_bf16_kernel with pages, else
// attn_fwd_seqlens_bf16_kernel (null length arrays in lens for a dense call).
int launch_attn_bf16(const Launch& l, bool causal, const Lens& lens, const Pages* pages);

// The fp8-K/V kernel of the family of p.D with T = __half or __nv_bfloat16 Q and O (attn_fp8kv_f16.cu,
// attn_fp8kv_bf16.cu): attn_fwd_fp8kv_paged_kernel with pages, else attn_fwd_fp8kv_seqlens_kernel.
template <typename T>
int launch_attn_fp8kv(const Launch& l, bool causal, const Lens& lens, const Pages* pages, float v_scale);

// The packed variable-length kernel of the family of p.D with T = __half or __nv_bfloat16 (attn_varlen.cu):
// attn_varlen_kernel with paged K/V when pages is given, else with packed K/V.
template <typename T>
int launch_attn_varlen(const Launch& l, bool causal, const Varlen& vl, const Pages* pages);

}  // namespace attn
}  // namespace b200
