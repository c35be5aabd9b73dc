// attn_bf16.cu — the bf16 attention kernels (attn_fwd_seqlens_bf16_kernel, attn_fwd_paged_bf16_kernel) of the three
// head-dim families, launched by the bf16 C entries of attn_capi.cu.
#include "attn_launch.cuh"

namespace b200 {
namespace attn {

template <int kDS, int kBN, int kWG>
int launch_attn_bf16(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, const Params& p, int qtiles,
                     int BH, int smem, bool causal, int splits, const Lens& lens, const Pages* pages,
                     cudaStream_t stream) {
  if (pages != nullptr) {
    auto kern = splits > 1 ? (causal ? attn_fwd_paged_bf16_kernel<kDS, kBN, kWG, true, true>
                                     : attn_fwd_paged_bf16_kernel<kDS, kBN, kWG, false, true>)
                           : (causal ? attn_fwd_paged_bf16_kernel<kDS, kBN, kWG, true, false>
                                     : attn_fwd_paged_bf16_kernel<kDS, kBN, kWG, false, false>);
    static int attr_smem[4][64] = {};
    return launch_kernel(kern, attr_smem[2 * (splits > 1) + causal], p, qtiles, BH, splits, threads<kWG>(), smem,
                         stream, tq, tk, tv, p, lens, *pages);
  }
  auto kern = splits > 1 ? (causal ? attn_fwd_seqlens_bf16_kernel<kDS, kBN, kWG, true, true>
                                   : attn_fwd_seqlens_bf16_kernel<kDS, kBN, kWG, false, true>)
                         : (causal ? attn_fwd_seqlens_bf16_kernel<kDS, kBN, kWG, true, false>
                                   : attn_fwd_seqlens_bf16_kernel<kDS, kBN, kWG, false, false>);
  static int attr_smem[4][64] = {};
  return launch_kernel(kern, attr_smem[2 * (splits > 1) + causal], p, qtiles, BH, splits, threads<kWG>(), smem, stream,
                       tq, tk, tv, p, lens);
}

// the families of attn_capi.cu's family(D): D <= 64, 64 < D <= 128, D > 128
template int launch_attn_bf16<64, 128, 2>(const CUtensorMap&, const CUtensorMap&, const CUtensorMap&, const Params&, int,
                                          int, int, bool, int, const Lens&, const Pages*, cudaStream_t);
template int launch_attn_bf16<128, 64, 2>(const CUtensorMap&, const CUtensorMap&, const CUtensorMap&, const Params&, int,
                                          int, int, bool, int, const Lens&, const Pages*, cudaStream_t);
template int launch_attn_bf16<256, 64, 1>(const CUtensorMap&, const CUtensorMap&, const CUtensorMap&, const Params&, int,
                                          int, int, bool, int, const Lens&, const Pages*, cudaStream_t);

}  // namespace attn
}  // namespace b200
