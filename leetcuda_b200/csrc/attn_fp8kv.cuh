// attn_fp8kv.cuh — the launch of the fp8-K/V attention kernels (attn_fwd_fp8kv_seqlens_kernel,
// attn_fwd_fp8kv_paged_kernel), instantiated for one Q/O element type by attn_fp8kv_f16.cu and attn_fp8kv_bf16.cu.
#pragma once
#include "attn_launch.cuh"

namespace b200 {
namespace attn {

template <typename T>
int launch_attn_fp8kv(const Launch& l, bool causal, const Lens& lens, const Pages* pages, float v_scale) {
  return with_family(l.p.D, [&](auto f) {
    using F = decltype(f);
    return with_flags(causal, l.splits > 1, [&](auto c, auto s) {
      if (pages != nullptr)
        return launch<attn_fwd_fp8kv_paged_kernel<F::kDS, F::kBN, F::kWG, c, s, T>, F::kWG>(l, lens, *pages, v_scale);
      return launch<attn_fwd_fp8kv_seqlens_kernel<F::kDS, F::kBN, F::kWG, c, s, T>, F::kWG>(l, lens, v_scale);
    });
  });
}

}  // namespace attn
}  // namespace b200
