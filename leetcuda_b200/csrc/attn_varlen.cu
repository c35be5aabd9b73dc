// attn_varlen.cu — the packed variable-length attention kernels (attn_varlen_kernel) of the three head-dim families,
// fp16 and bf16, packed or paged K/V, launched by the varlen C entries of attn_capi.cu.
#include "attn_launch.cuh"

namespace b200 {
namespace attn {

template <typename T, int kDS, int kBN, int kWG>
int launch_attn_varlen(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, const Params& p, int qtiles,
                       int BH, int smem, bool causal, const Varlen& vl, const Pages* pages, cudaStream_t stream) {
  auto kern = pages != nullptr ? (causal ? attn_varlen_kernel<kDS, kBN, kWG, true, true, T>
                                         : attn_varlen_kernel<kDS, kBN, kWG, false, true, T>)
                               : (causal ? attn_varlen_kernel<kDS, kBN, kWG, true, false, T>
                                         : attn_varlen_kernel<kDS, kBN, kWG, false, false, T>);
  static int attr_smem[4][64] = {};
  return launch_kernel(kern, attr_smem[2 * (pages != nullptr) + causal], p, qtiles, BH, 1, threads<kWG>(), smem, stream,
                       tq, tk, tv, p, vl, pages != nullptr ? *pages : Pages{});
}

// the families of attn_capi.cu's family(D): D <= 64, 64 < D <= 128, D > 128
#define B200_VARLEN_FAMILY(T, DS, BN, WG)                                                                             \
  template int launch_attn_varlen<T, DS, BN, WG>(const CUtensorMap&, const CUtensorMap&, const CUtensorMap&,          \
                                                 const Params&, int, int, int, bool, const Varlen&, const Pages*,     \
                                                 cudaStream_t);
B200_VARLEN_FAMILY(__half, 64, 128, 2)
B200_VARLEN_FAMILY(__half, 128, 64, 2)
B200_VARLEN_FAMILY(__half, 256, 64, 1)
B200_VARLEN_FAMILY(__nv_bfloat16, 64, 128, 2)
B200_VARLEN_FAMILY(__nv_bfloat16, 128, 64, 2)
B200_VARLEN_FAMILY(__nv_bfloat16, 256, 64, 1)
#undef B200_VARLEN_FAMILY

}  // namespace attn
}  // namespace b200
