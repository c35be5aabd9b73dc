// attn_fp8kv_bf16.cu — the fp8-K/V attention kernels with bf16 Q and O, launched by b200_fmha_fwd_bf16_fp8kv_seqlens
// and b200_fmha_fwd_bf16_fp8kv_paged (attn_capi.cu).  A translation unit of their own so that they compile in parallel.
#include "attn_fp8kv.cuh"

namespace b200 {
namespace attn {

template int launch_attn_fp8kv<__nv_bfloat16>(const Launch&, bool, const Lens&, const Pages*, float);

}  // namespace attn
}  // namespace b200
