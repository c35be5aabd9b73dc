// attn_fp8kv.cuh — the launch of the fp8-K/V attention kernels (attn_fwd_fp8kv_seqlens_kernel,
// attn_fwd_fp8kv_paged_kernel), instantiated for one Q/O element type by attn_fp8kv_f16.cu and attn_fp8kv_bf16.cu.
#pragma once
#include "attn_launch.cuh"

namespace b200 {
namespace attn {

template <typename T, int kDS, int kBN, int kWG>
int launch_attn_fp8kv(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, const Params& p, int qtiles,
                      int BH, int smem, bool causal, int splits, const Lens& lens, const Pages* pages, float v_scale,
                      cudaStream_t stream) {
  if (pages != nullptr) {
    auto kern = splits > 1 ? (causal ? attn_fwd_fp8kv_paged_kernel<kDS, kBN, kWG, true, true, T>
                                     : attn_fwd_fp8kv_paged_kernel<kDS, kBN, kWG, false, true, T>)
                           : (causal ? attn_fwd_fp8kv_paged_kernel<kDS, kBN, kWG, true, false, T>
                                     : attn_fwd_fp8kv_paged_kernel<kDS, kBN, kWG, false, false, T>);
    static int attr_smem[4][64] = {};
    return launch_kernel(kern, attr_smem[2 * (splits > 1) + causal], p, qtiles, BH, splits, threads<kWG>(), smem,
                         stream, tq, tk, tv, p, lens, *pages, v_scale);
  }
  auto kern = splits > 1 ? (causal ? attn_fwd_fp8kv_seqlens_kernel<kDS, kBN, kWG, true, true, T>
                                   : attn_fwd_fp8kv_seqlens_kernel<kDS, kBN, kWG, false, true, T>)
                         : (causal ? attn_fwd_fp8kv_seqlens_kernel<kDS, kBN, kWG, true, false, T>
                                   : attn_fwd_fp8kv_seqlens_kernel<kDS, kBN, kWG, false, false, T>);
  static int attr_smem[4][64] = {};
  return launch_kernel(kern, attr_smem[2 * (splits > 1) + causal], p, qtiles, BH, splits, threads<kWG>(), smem, stream,
                       tq, tk, tv, p, lens, v_scale);
}

// the families of attn_capi.cu's family(D): D <= 64, 64 < D <= 128, D > 128
#define B200_ATTN_FP8KV_INSTANTIATE(T)                                                                                 \
  template int launch_attn_fp8kv<T, 64, 128, 2>(const CUtensorMap&, const CUtensorMap&, const CUtensorMap&,           \
                                                const Params&, int, int, int, bool, int, const Lens&, const Pages*,    \
                                                float, cudaStream_t);                                                  \
  template int launch_attn_fp8kv<T, 128, 64, 2>(const CUtensorMap&, const CUtensorMap&, const CUtensorMap&,           \
                                                const Params&, int, int, int, bool, int, const Lens&, const Pages*,    \
                                                float, cudaStream_t);                                                  \
  template int launch_attn_fp8kv<T, 256, 64, 1>(const CUtensorMap&, const CUtensorMap&, const CUtensorMap&,           \
                                                const Params&, int, int, int, bool, int, const Lens&, const Pages*,    \
                                                float, cudaStream_t);

}  // namespace attn
}  // namespace b200
