// attn_varlen.cu — the packed variable-length attention kernels (attn_varlen_kernel) of the three head-dim families,
// fp16 and bf16, packed or paged K/V, launched by the varlen C entries of attn_capi.cu.
#include "attn_launch.cuh"

namespace b200 {
namespace attn {

template <typename T>
int launch_attn_varlen(const Launch& l, bool causal, const Varlen& vl, const Pages* pages) {
  return with_family(l.p.D, [&](auto f) {
    using F = decltype(f);
    return with_flags(causal, pages != nullptr, [&](auto c, auto paged) {
      return launch<attn_varlen_kernel<F::kDS, F::kBN, F::kWG, c, paged, T>, F::kWG>(l, vl, paged ? *pages : Pages{});
    });
  });
}

template int launch_attn_varlen<__half>(const Launch&, bool, const Varlen&, const Pages*);
template int launch_attn_varlen<__nv_bfloat16>(const Launch&, bool, const Varlen&, const Pages*);

}  // namespace attn
}  // namespace b200
