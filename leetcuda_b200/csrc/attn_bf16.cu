// attn_bf16.cu — the bf16 attention kernels (attn_fwd_seqlens_bf16_kernel, attn_fwd_paged_bf16_kernel) of the three
// head-dim families, launched by the bf16 C entries of attn_capi.cu.
#include "attn_launch.cuh"

namespace b200 {
namespace attn {

int launch_attn_bf16(const Launch& l, bool causal, const Lens& lens, const Pages* pages) {
  return with_family(l.p.D, [&](auto f) {
    using F = decltype(f);
    return with_flags(causal, l.splits > 1, [&](auto c, auto s) {
      if (pages != nullptr)
        return launch<attn_fwd_paged_bf16_kernel<F::kDS, F::kBN, F::kWG, c, s>, F::kWG>(l, lens, *pages);
      return launch<attn_fwd_seqlens_bf16_kernel<F::kDS, F::kBN, F::kWG, c, s>, F::kWG>(l, lens);
    });
  });
}

}  // namespace attn
}  // namespace b200
