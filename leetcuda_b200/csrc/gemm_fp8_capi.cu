// gemm_fp8_capi.cu — C-ABI entry point of the fp8 (e4m3) scaled GEMM (include/leetcuda_b200.h, b200_gemm_e4m3).
#include "capi_common.cuh"

#include "gemm_fp8_sm90.cuh"

namespace {

using namespace b200;
using b200::host::fail;
using b200::host::overlaps;

// Persistent launch in clusters of `cs` CTAs, as launch_hgemm (hgemm_capi.cu)
template <typename OutT, bool kBlockScale>
int launch_gemm_e4m3(const CUtensorMap& ta, const CUtensorMap& tb, const gemm_fp8::Params& p, int cs,
                     cudaStream_t stream) {
  return host::launch_persistent<gemm_fp8::gemm_e4m3_kernel<OutT, kBlockScale>>(
      "gemm_e4m3", gemm_fp8::kThreads, gemm_fp8::C_::SMEM_BYTES, p.g.num_tiles, cs, stream, ta, tb, p);
}

}  // namespace

extern "C" {

int b200_gemm_e4m3(const void* a, const void* b_nk, void* c, const float* scale_a, const float* scale_b, int M, int N,
                   int K, int scale_recipe, int c_dtype, void* stream_) {
  const char* who = "gemm_e4m3";
  struct Ptr { const void* p; const char* name; unsigned align; };
  const Ptr ptrs[] = {{a, "a", 16}, {b_nk, "b_nk", 16}, {c, "c", 16}, {scale_a, "scale_a", 4}, {scale_b, "scale_b", 4}};
  for (const Ptr& x : ptrs)
    if (x.p == nullptr) return fail(B200_EINVAL, "%s: %s is NULL", who, x.name);
  for (const Ptr& x : ptrs)
    if ((reinterpret_cast<uintptr_t>(x.p) & (x.align - 1)) != 0)
      return fail(B200_EINVAL, "%s: %s must be %u-byte aligned", who, x.name, x.align);
  if (M < 1) return fail(B200_EINVAL, "%s: M=%d must be >= 1", who, M);
  if (N < 1) return fail(B200_EINVAL, "%s: N=%d must be >= 1", who, N);
  if (K < 1) return fail(B200_EINVAL, "%s: K=%d must be >= 1", who, K);
  if (K % 16 != 0) return fail(B200_EINVAL, "%s: K=%d must be a multiple of 16 (the TMA row stride)", who, K);
  if (N % 8 != 0) return fail(B200_EINVAL, "%s: N=%d must be a multiple of 8 (16-byte C stores)", who, N);
  if (scale_recipe != B200_SCALE_TENSOR && scale_recipe != B200_SCALE_ROW && scale_recipe != B200_SCALE_BLOCK)
    return fail(B200_EINVAL, "%s: scale_recipe=%d must be B200_SCALE_TENSOR (%d), B200_SCALE_ROW (%d) or "
                "B200_SCALE_BLOCK (%d)", who, scale_recipe, B200_SCALE_TENSOR, B200_SCALE_ROW, B200_SCALE_BLOCK);
  if (c_dtype != B200_DTYPE_F16 && c_dtype != B200_DTYPE_BF16)
    return fail(B200_EINVAL, "%s: c_dtype=%d must be B200_DTYPE_F16 (%d) or B200_DTYPE_BF16 (%d)", who, c_dtype,
                B200_DTYPE_F16, B200_DTYPE_BF16);
  // c must not share a byte with anything the kernel reads
  const size_t m = static_cast<size_t>(M), n = static_cast<size_t>(N), k = static_cast<size_t>(K);
  const size_t kbs = (k + 127) / 128, nbs = (n + 127) / 128;
  const size_t sa_n = scale_recipe == B200_SCALE_TENSOR ? 1 : scale_recipe == B200_SCALE_ROW ? m : m * kbs;
  const size_t sb_n = scale_recipe == B200_SCALE_TENSOR ? 1 : scale_recipe == B200_SCALE_ROW ? n : nbs * kbs;
  const size_t c_bytes = m * n * 2;
  const Ptr* in[] = {&ptrs[0], &ptrs[1], &ptrs[3], &ptrs[4]};
  const size_t in_bytes[] = {m * k, n * k, sa_n * 4, sb_n * 4};
  for (int i = 0; i < 4; ++i)
    if (overlaps(c, c_bytes, in[i]->p, in_bytes[i])) return fail(B200_EINVAL, "%s: c overlaps %s", who, in[i]->name);

  gemm_fp8::Params p;
  memset(&p, 0, sizeof(p));
  const int tiles_m = (M + gemm_fp8::BM - 1) / gemm_fp8::BM;
  const int cs = tiles_m >= 2 ? 2 : 1;   // clusters of two share each B tile whenever there are two m-tiles to pair
  p.g.C = c;
  p.g.M = M; p.g.N = N; p.g.K = K; p.g.ldc = N;
  p.g.tiles_m = tiles_m;
  p.g.tiles_n = (N + gemm_fp8::BN - 1) / gemm_fp8::BN;
  p.g.num_tiles = (tiles_m + cs - 1) / cs * p.g.tiles_n;
  p.sa = scale_a;
  p.sb = scale_b;
  p.sa_stride = scale_recipe == B200_SCALE_ROW ? 1 : 0;
  p.sb_stride = scale_recipe == B200_SCALE_ROW ? 1 : 0;

  CUtensorMap ta, tb;
  {
    uint64_t dims[2] = {static_cast<uint64_t>(K), static_cast<uint64_t>(M)};
    uint64_t str[1] = {static_cast<uint64_t>(K)};
    uint32_t box[2] = {gemm_fp8::BK, gemm_fp8::BM};
    int rc = host::get_tmap(&ta, a, 2, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_DATA_TYPE_UINT8);
    if (rc) return rc;
  }
  {
    uint64_t dims[2] = {static_cast<uint64_t>(K), static_cast<uint64_t>(N)};
    uint64_t str[1] = {static_cast<uint64_t>(K)};
    uint32_t box[2] = {gemm_fp8::BK, static_cast<uint32_t>(gemm_fp8::BN / cs)};   // each CTA loads 1/cs of B
    int rc = host::get_tmap(&tb, b_nk, 2, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_DATA_TYPE_UINT8);
    if (rc) return rc;
  }
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const bool block = scale_recipe == B200_SCALE_BLOCK;
  if (c_dtype == B200_DTYPE_F16)
    return block ? launch_gemm_e4m3<__half, true>(ta, tb, p, cs, stream)
                 : launch_gemm_e4m3<__half, false>(ta, tb, p, cs, stream);
  return block ? launch_gemm_e4m3<__nv_bfloat16, true>(ta, tb, p, cs, stream)
               : launch_gemm_e4m3<__nv_bfloat16, false>(ta, tb, p, cs, stream);
}

}  // extern "C"
