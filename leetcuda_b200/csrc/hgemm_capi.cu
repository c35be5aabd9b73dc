// hgemm_capi.cu — C-ABI entry points of the HGEMM path (include/leetcuda_b200.h).
#include "capi_common.cuh"
#include <vector>

#include "hgemm_sm90.cuh"
#include <stdlib.h>

namespace {

using namespace b200;
using b200::host::fail;

template <int kBN, bool kBMn, bool kTf32, bool kAcc16>
int launch_hgemm(const CUtensorMap& ta, const CUtensorMap& tb, const hgemm::Params& p, int grid, cudaStream_t stream) {
  using C_ = hgemm::Cfg<kBN>;
  auto kern = hgemm::hgemm_wgmma_kernel<kBN, kBMn, kTf32, kAcc16>;
  static bool attr_set[64] = {false};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev >= 0 && dev < 64 && !attr_set[dev]) {
    B200_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C_::SMEM_BYTES));
    attr_set[dev] = true;
  }
  kern<<<grid, hgemm::kThreads, C_::SMEM_BYTES, stream>>>(ta, tb, p);
  B200_CUDA_OK(cudaGetLastError());
  host::count_launch();
  return 0;
}

// x <- tf32(x), round-to-nearest (ties away), in place: what the reference's tf32 ops do to their
// inputs before the MMAs (sgemm_wmma_tf32_stage.cu:44-60, 586-592).  HBM-bound, grid-stride, float4.
__global__ void __launch_bounds__(256) tf32_round_inplace_kernel(float* __restrict__ x, size_t n) {
  auto rna = [](float v) -> float {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(v));
    return __uint_as_float(r);
  };
  const size_t n4 = n / 4;
  float4* x4 = reinterpret_cast<float4*>(x);
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n4; i += stride) {
    float4 v = x4[i];
    v.x = rna(v.x); v.y = rna(v.y); v.z = rna(v.z); v.w = rna(v.w);
    x4[i] = v;
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) x[n4 * 4 + threadIdx.x] = rna(x[n4 * 4 + threadIdx.x]);
}

// 3xTF32 split (b200_sgemm_3xtf32): x = hi + lo + O(2^-22 |x|) with hi = tf32(x), lo = tf32(x - hi), both exactly
// representable in TF32.  Each input element is written three times, at out[r * ld + c + off_j], carrying hi or lo
// as `sel` bit j says (0 = hi, 1 = lo): A' = [hi | hi | lo] (column blocks), B' = [hi ; lo ; hi] (row blocks), so
// that A' B' = hi_a hi_b + hi_a lo_b + lo_a hi_b in ONE tf32 GEMM with K' = 3K.
__global__ void __launch_bounds__(256) tf32_split3_kernel(const float* __restrict__ x, float* __restrict__ out, size_t rows,
                                                          size_t cols, size_t ld_out, size_t off0, size_t off1, size_t off2,
                                                          unsigned sel) {
  auto rna = [](float v) -> float {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(v));
    return __uint_as_float(r);
  };
  const size_t c4 = cols / 4;
  const size_t total = rows * c4;
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
    const size_t r = i / c4, c = (i - r * c4) * 4;
    const float4 v = *reinterpret_cast<const float4*>(x + r * cols + c);
    float4 hi, lo;
    hi.x = rna(v.x); hi.y = rna(v.y); hi.z = rna(v.z); hi.w = rna(v.w);
    lo.x = rna(v.x - hi.x); lo.y = rna(v.y - hi.y); lo.z = rna(v.z - hi.z); lo.w = rna(v.w - hi.w);
    float* o = out + r * ld_out + c;
    *reinterpret_cast<float4*>(o + off0) = (sel & 1u) ? lo : hi;
    *reinterpret_cast<float4*>(o + off1) = (sel & 2u) ? lo : hi;
    *reinterpret_cast<float4*>(o + off2) = (sel & 4u) ? lo : hi;
  }
}

// b[K,N] (fp32) -> bt[N, ld]: the TF32 wgmma reads both operands K-major, so the [K,N] layout of the reference's
// SGEMM is restored to [N,K] first (HBM-bound, one pass).  mode 0: copy (ld = K); 1: also round b to TF32 in place
// and copy the rounded value (ld = K); 2: the 3xTF32 split of b, bt[n, k] = hi, bt[n, K + k] = lo, bt[n, 2K + k] = hi
// (ld = 3K; b is not written).
__global__ void __launch_bounds__(256) tf32_transpose_kernel(float* __restrict__ b, float* __restrict__ bt, int K, int N,
                                                             int mode) {
  auto rna = [](float v) -> float {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(v));
    return __uint_as_float(r);
  };
  __shared__ float tile[32][33];
  const int n0 = blockIdx.x * 32, k0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int k = k0 + i, n = n0 + threadIdx.x;
    if (k < K && n < N) {
      float v = b[static_cast<size_t>(k) * N + n];
      if (mode == 1) {
        v = rna(v);
        b[static_cast<size_t>(k) * N + n] = v;
      }
      tile[i][threadIdx.x] = v;
    }
  }
  __syncthreads();
  const size_t ld = mode == 2 ? 3 * static_cast<size_t>(K) : K;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int n = n0 + i, k = k0 + threadIdx.x;
    if (k >= K || n >= N) continue;
    const float v = tile[threadIdx.x][i];
    float* o = bt + static_cast<size_t>(n) * ld + k;
    if (mode == 2) {
      const float hi = rna(v), lo = rna(v - hi);
      o[0] = hi;
      o[K] = lo;
      o[2 * static_cast<size_t>(K)] = hi;
    } else {
      o[0] = v;
    }
  }
}

int launch_tf32_transpose(const float* b, float* bt, int K, int N, int mode, cudaStream_t stream) {
  dim3 grid((N + 31) / 32, (K + 31) / 32, 1), block(32, 8, 1);
  tf32_transpose_kernel<<<grid, block, 0, stream>>>(const_cast<float*>(b), bt, K, N, mode);
  B200_CUDA_OK(cudaGetLastError());
  host::count_launch();
  return 0;
}

struct Fanout {           // fused all-gather targets (see hgemm::Params)
  void* mc = nullptr;
  void* const* peers = nullptr;
  int n_peers = 0;
  size_t elem_offset = 0;  // offset (in elements) of this shard inside the full C buffers
};

int hgemm_impl(const void* a, const void* b, void* c, int M, int N, int K, int b_layout,
               int tile_sel, int group_m, int max_ctas, uint32_t b_lbo, uint32_t b_sbo,
               uint32_t b_kstep, void* stream_, const Fanout* fan = nullptr, int acc_f16 = 0,
               bool tf32 = false) {
  // tf32: a, b, c are fp32 and b is [N,K] (the callers transpose a [K,N] operand first)
  const int esize = tf32 ? 4 : 2;
  const int bke = 128 / esize;   // elements per 128-byte swizzle row = k-block
  const CUtensorMapDataType dt = tf32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  if (!a || !b || !c) return fail(B200_EINVAL, "gemm: null pointer");
  if (M <= 0 || N <= 0 || K <= 0) return fail(B200_EINVAL, "gemm: bad shape M=%d N=%d K=%d", M, N, K);
  if ((K % (16 / esize)) != 0 || (N % (16 / esize)) != 0)
    return fail(B200_EINVAL, "gemm: K (%d) and N (%d) must be multiples of %d", K, N, 16 / esize);
  if (b_layout != B200_B_ROW_MAJOR_KN && b_layout != B200_B_ROW_MAJOR_NK)
    return fail(B200_EINVAL, "hgemm: unknown b_layout %d", b_layout);
  if (tf32 && b_layout != B200_B_ROW_MAJOR_NK) return fail(B200_EINVAL, "gemm: internal error (tf32 B must be [N,K])");
  if ((reinterpret_cast<uintptr_t>(c) & 15u) != 0)
    return fail(B200_EINVAL, "hgemm: c is not 16-byte aligned");
  if (tile_sel < 0 || tile_sel > 2) return fail(B200_EINVAL, "hgemm: tile selector %d (0 auto, 1: 128x128, 2: 128x256)", tile_sel);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const int sms = host::sm_count();

  // Tile: 128x256 (least operand traffic per flop) unless a 128x128 tiling fills the last wave of the
  // SMs markedly better (mid-size problems would otherwise leave many of the SMs idle).
  int bn = 256;
  if (tile_sel == 1) bn = 128;
  if (tile_sel == 0) {
    auto score = [&](int bnc, double eff) {
      const long tiles = static_cast<long>((M + 127) / 128) * ((N + bnc - 1) / bnc);
      const long waves = (tiles + sms - 1) / sms;
      return eff * static_cast<double>(tiles) / static_cast<double>(waves * sms);
    };
    if (score(128, 0.90) > score(256, 1.0)) bn = 128;
  }

  hgemm::Params p;
  memset(&p, 0, sizeof(p));
  p.C = c;
  p.M = M; p.N = N; p.K = K; p.ldc = N;
  p.tiles_m = (M + hgemm::BM - 1) / hgemm::BM;
  p.tiles_n = (N + bn - 1) / bn;
  p.num_tiles = p.tiles_m * p.tiles_n;
  p.group_m = group_m > 0 ? group_m : 16;
  {
    static int serp = -1;   // B200_HGEMM_SERPENTINE=0|1 (A/B knob), default on
    if (serp < 0) { const char* e = getenv("B200_HGEMM_SERPENTINE"); serp = (e && e[0] == '0') ? 0 : 1; }
    p.serpentine = serp;
  }
  // MN-major B (the [K,N] layout, fp16): boxes {64 n x 64 k}, 8-k-row swizzle atoms (SBO 1024), the
  // 64-column boxes of one stage 8 KiB apart (LBO), +16 k-rows per k16 step.
  p.b_lbo = b_lbo ? b_lbo : 8192u;
  p.b_sbo = b_sbo ? b_sbo : 1024u;
  p.b_kstep = b_kstep ? b_kstep : 2048u;
  {
    // L2 eviction priority of the A / B operand loads: A panels (re-used by the other column tiles of
    // the same row group) evict-last, B panels normal.  B200_HGEMM_HINTS=<a><b>, each n|f|l, overrides.
    static unsigned long long ha = 0, hb = 0;
    if (ha == 0) {
      auto dec = [](char ch) { return ch == 'f' ? b200::kEvictFirst : (ch == 'l' ? b200::kEvictLast : b200::kEvictNormal); };
      const char* e = getenv("B200_HGEMM_HINTS");
      ha = dec(e && e[0] ? e[0] : 'l');
      hb = dec(e && e[0] && e[1] ? e[1] : 'n');
    }
    p.hint_a = ha;
    p.hint_b = hb;
  }
  if (fan) {
    if (fan->n_peers < 0 || fan->n_peers > 7) return fail(B200_EINVAL, "hgemm: %d peers", fan->n_peers);
    if (fan->mc) p.C_mc = static_cast<char*>(fan->mc) + fan->elem_offset * esize;
    for (int i = 0; i < fan->n_peers; ++i) {
      if (!fan->peers[i]) return fail(B200_EINVAL, "hgemm: null peer pointer %d", i);
      p.C_peer[i] = static_cast<char*>(fan->peers[i]) + fan->elem_offset * esize;
    }
    p.n_peers = fan->n_peers;
  }

  CUtensorMap ta, tb;
  {
    uint64_t dims[2] = {static_cast<uint64_t>(K), static_cast<uint64_t>(M)};
    uint64_t str[1] = {static_cast<uint64_t>(K) * esize};
    uint32_t box[2] = {static_cast<uint32_t>(bke), hgemm::BM};
    int rc = host::get_tmap(&ta, a, 2, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B, dt);
    if (rc) return rc;
  }
  if (b_layout == B200_B_ROW_MAJOR_NK) {
    uint64_t dims[2] = {static_cast<uint64_t>(K), static_cast<uint64_t>(N)};
    uint64_t str[1] = {static_cast<uint64_t>(K) * esize};
    uint32_t box[2] = {static_cast<uint32_t>(bke), static_cast<uint32_t>(bn)};
    int rc = host::get_tmap(&tb, b, 2, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B, dt);
    if (rc) return rc;
  } else {
    uint64_t dims[2] = {static_cast<uint64_t>(N), static_cast<uint64_t>(K)};
    uint64_t str[1] = {static_cast<uint64_t>(N) * esize};
    uint32_t box[2] = {64, 64};
    int rc = host::get_tmap(&tb, b, 2, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B, dt);
    if (rc) return rc;
  }

  int grid = p.num_tiles;
  const int cap = (max_ctas > 0 && max_ctas < sms) ? max_ctas : sms;
  if (grid > cap) grid = cap;

  const bool mn = (b_layout == B200_B_ROW_MAJOR_KN);
  if (tf32)
    return bn == 128 ? launch_hgemm<128, false, true, false>(ta, tb, p, grid, stream)
                     : launch_hgemm<256, false, true, false>(ta, tb, p, grid, stream);
  if (acc_f16) {
    if (bn == 128)
      return mn ? launch_hgemm<128, true, false, true>(ta, tb, p, grid, stream)
                : launch_hgemm<128, false, false, true>(ta, tb, p, grid, stream);
    return mn ? launch_hgemm<256, true, false, true>(ta, tb, p, grid, stream)
              : launch_hgemm<256, false, false, true>(ta, tb, p, grid, stream);
  }
  if (bn == 128)
    return mn ? launch_hgemm<128, true, false, false>(ta, tb, p, grid, stream)
              : launch_hgemm<128, false, false, false>(ta, tb, p, grid, stream);
  return mn ? launch_hgemm<256, true, false, false>(ta, tb, p, grid, stream)
            : launch_hgemm<256, false, false, false>(ta, tb, p, grid, stream);
}

// cached device workspace for the *_host wrappers (per thread and device).  Those entry points return only after their
// stream has drained, so two calls of one thread never overlap on it; growing it frees the old block (a device-wide
// synchronisation) — acceptable for a convenience path whose cost is the PCIe copy.  Kernels that need scratch on the
// caller's stream (transposed V, 3xTF32) use cudaMallocAsync / cudaFreeAsync instead.
struct Workspace {
  void* ptr = nullptr;
  size_t bytes = 0;
  int dev = -1;
};
thread_local Workspace g_ws;

}  // namespace

namespace b200 { namespace host {
int workspace(void** out, size_t bytes) {
  int dev = 0;
  cudaGetDevice(&dev);
  if (g_ws.ptr && (g_ws.bytes < bytes || g_ws.dev != dev)) {
    cudaFree(g_ws.ptr);
    g_ws.ptr = nullptr;
    g_ws.bytes = 0;
  }
  if (!g_ws.ptr) {
    B200_CUDA_OK(cudaMalloc(&g_ws.ptr, bytes));
    g_ws.bytes = bytes;
    g_ws.dev = dev;
  }
  *out = g_ws.ptr;
  return 0;
}
}}  // namespace b200::host

extern "C" {

int b200_hgemm_f16(const void* a, const void* b, void* c, int M, int N, int K, int b_layout,
                   void* stream) {
  return hgemm_impl(a, b, c, M, N, K, b_layout, 0, 0, 0, 0, 0, 0, stream);
}

int b200_hgemm_f16_ex(const void* a, const void* b, void* c, int M, int N, int K, int b_layout,
                      int cta_group, int group_m, int max_ctas, uint32_t b_lbo, uint32_t b_sbo,
                      uint32_t b_kstep, void* stream) {
  return hgemm_impl(a, b, c, M, N, K, b_layout, cta_group, group_m, max_ctas, b_lbo, b_sbo,
                    b_kstep, stream);
}

int b200_hgemm_f16_acc16(const void* a, const void* b, void* c, int M, int N, int K, int b_layout,
                         void* stream) {
  return hgemm_impl(a, b, c, M, N, K, b_layout, 0, 0, 0, 0, 0, 0, stream, nullptr, 1);
}

int b200_hgemm_f16_rows(const void* a_shard, const void* b, void* c_full, int rows, int N, int K,
                        int b_layout, int row0, void* stream) {
  if (row0 < 0) return fail(B200_EINVAL, "hgemm_rows: row0 %d", row0);
  __half* c = static_cast<__half*>(c_full) + static_cast<size_t>(row0) * N;
  return hgemm_impl(a_shard, b, c, rows, N, K, b_layout, 0, 0, 0, 0, 0, 0, stream);
}

int b200_hgemm_f16_rows_fused(const void* a_shard, const void* b, void* c_full, void* c_full_multicast,
                              void* const* c_full_peers, int n_peers, int rows, int N, int K,
                              int b_layout, int row0, void* stream) {
  if (row0 < 0) return fail(B200_EINVAL, "hgemm_rows_fused: row0 %d", row0);
  if (n_peers < 0 || n_peers > 7) return fail(B200_EINVAL, "hgemm_rows_fused: n_peers %d (0..7)", n_peers);
  if (n_peers > 0 && !c_full_peers) return fail(B200_EINVAL, "hgemm_rows_fused: n_peers %d but c_full_peers is NULL", n_peers);
  if (!c_full_multicast && n_peers == 0)
    return fail(B200_EINVAL, "hgemm_rows_fused: neither a multicast mapping nor peer mappings were given");
  Fanout fan;
  fan.elem_offset = static_cast<size_t>(row0) * N;
  // Transport (see the header): peer mappings given -> the epilogue stores to C and to every peer (NVLink
  // P2P); only a multicast mapping given -> one multimem.st through it reaches every GPU.
  // B200_FUSED_EPILOGUE=direct (or mc) prefers the multicast mapping when both are given.
  const char* e = getenv("B200_FUSED_EPILOGUE");
  if (c_full_multicast && (n_peers == 0 || (e && (e[0] == 'd' || e[0] == 'm')))) {
    fan.mc = c_full_multicast;
  } else {
    fan.peers = c_full_peers;
    fan.n_peers = n_peers;
  }
  __half* c = static_cast<__half*>(c_full) + fan.elem_offset;
  return hgemm_impl(a_shard, b, c, rows, N, K, b_layout, 0, 0, 0, 0, 0, 0, stream, &fan);
}

// ---------------------------------------------------------------------------------------------
// SGEMM through TF32 tensor cores (SURVEY §8f-2: kernels/sgemm/sgemm_wmma_tf32_stage.cu)
// ---------------------------------------------------------------------------------------------
int b200_tf32_round_inplace(float* x, size_t n, void* stream_) {
  if (!x && n) return fail(B200_EINVAL, "tf32_round: null pointer");
  if ((reinterpret_cast<uintptr_t>(x) & 15u) != 0) return fail(B200_EINVAL, "tf32_round: x is not 16-byte aligned");
  if (n == 0) return 0;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const size_t n4 = n / 4;
  size_t blocks = (n4 + 256 * 4 - 1) / (256 * 4);          // 4 float4 per thread
  const size_t cap = static_cast<size_t>(host::sm_count()) * 16;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  tf32_round_inplace_kernel<<<static_cast<unsigned>(blocks), 256, 0, stream>>>(x, n);
  B200_CUDA_OK(cudaGetLastError());
  host::count_launch();
  return 0;
}

}  // extern "C"

namespace {
int sgemm_tf32_impl(float* a, float* b, float* c, int M, int N, int K, int b_layout, int round, int tile_sel,
                    int group_m, int max_ctas, void* stream_) {
  // validate everything the GEMM would reject BEFORE touching the caller's a and b
  if (!a || !b || !c || M <= 0 || N <= 0 || K <= 0) return fail(B200_EINVAL, "sgemm: bad args");
  if ((K % 4) != 0 || (N % 4) != 0)
    return fail(B200_EINVAL, "gemm: K (%d) and N (%d) must be multiples of 4", K, N);
  if (b_layout != B200_B_ROW_MAJOR_KN && b_layout != B200_B_ROW_MAJOR_NK)
    return fail(B200_EINVAL, "hgemm: unknown b_layout %d", b_layout);
  if (((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) | reinterpret_cast<uintptr_t>(c)) & 15u) != 0)
    return fail(B200_EINVAL, "sgemm: a, b, c must be 16-byte aligned");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int rc;
  if (round && (rc = b200_tf32_round_inplace(a, static_cast<size_t>(M) * K, stream))) return rc;
  if (b_layout == B200_B_ROW_MAJOR_NK) {
    if (round && (rc = b200_tf32_round_inplace(b, static_cast<size_t>(K) * N, stream))) return rc;
    return hgemm_impl(a, b, c, M, N, K, B200_B_ROW_MAJOR_NK, tile_sel, group_m, max_ctas, 0, 0, 0, stream, nullptr, 0, true);
  }
  // [K,N]: round b in place (if asked) and transpose it into stream-ordered scratch in one pass
  float* bt = nullptr;
  B200_CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&bt), static_cast<size_t>(K) * N * sizeof(float), stream));
  rc = launch_tf32_transpose(b, bt, K, N, round ? 1 : 0, stream);
  if (!rc)
    rc = hgemm_impl(a, bt, c, M, N, K, B200_B_ROW_MAJOR_NK, tile_sel, group_m, max_ctas, 0, 0, 0, stream, nullptr, 0, true);
  cudaFreeAsync(bt, stream);
  return rc;
}
}  // namespace

extern "C" {

int b200_sgemm_tf32(float* a, float* b, float* c, int M, int N, int K, int b_layout,
                    int round_inputs_in_place, void* stream) {
  return sgemm_tf32_impl(a, b, c, M, N, K, b_layout, round_inputs_in_place, 0, 0, 0, stream);
}

int b200_sgemm_3xtf32(const float* a, const float* b, float* c, int M, int N, int K, void* stream_) {
  if (!a || !b || !c || M <= 0 || N <= 0 || K <= 0) return fail(B200_EINVAL, "sgemm_3xtf32: bad args");
  if ((K % 4) != 0 || (N % 4) != 0)
    return fail(B200_EINVAL, "gemm: K (%d) and N (%d) must be multiples of 4", K, N);
  if (((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) | reinterpret_cast<uintptr_t>(c)) & 15u) != 0)
    return fail(B200_EINVAL, "sgemm: a, b, c must be 16-byte aligned");
  if (static_cast<long long>(K) * 3 > 0x7FFFFFFFll) return fail(B200_EINVAL, "sgemm_3xtf32: K too large");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const size_t m = static_cast<size_t>(M), n = static_cast<size_t>(N), k = static_cast<size_t>(K);
  float* ws = nullptr;                               // [A' : M x 3K][B'^T : N x 3K], stream-ordered scratch
  B200_CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&ws), (m * 3 * k + 3 * k * n) * sizeof(float), stream));
  float* a3 = ws;
  float* b3 = ws + m * 3 * k;
  const unsigned cap = static_cast<unsigned>(host::sm_count()) * 8;
  auto blocks = [&](size_t elems) { size_t g = (elems / 4 + 255) / 256; return static_cast<unsigned>(g < 1 ? 1 : (g > cap ? cap : g)); };
  tf32_split3_kernel<<<blocks(m * k), 256, 0, stream>>>(a, a3, m, k, 3 * k, 0, k, 2 * k, 0x4u);          // hi | hi | lo
  cudaError_t le = cudaGetLastError();
  int rc = 0;
  if (le != cudaSuccess) rc = fail(B200_ECUDA, "tf32 split launch failed: %s", cudaGetErrorString(le));
  else {
    host::count_launch();
    rc = launch_tf32_transpose(b, b3, K, N, 2, stream);                                                   // hi ; lo ; hi
    if (!rc) rc = hgemm_impl(a3, b3, c, M, N, 3 * K, B200_B_ROW_MAJOR_NK, 0, 0, 0, 0, 0, 0, stream, nullptr, 0, true);
  }
  cudaFreeAsync(ws, stream);
  return rc;
}

int b200_sgemm_tf32_ex(const float* a, const float* b, float* c, int M, int N, int K, int b_layout,
                       int cta_group, int group_m, int max_ctas, uint32_t b_lbo, uint32_t b_sbo,
                       uint32_t b_kstep, void* stream) {
  (void)b_lbo; (void)b_sbo; (void)b_kstep;   // descriptor knobs of the fp16 MN-major B operand only
  return sgemm_tf32_impl(const_cast<float*>(a), const_cast<float*>(b), c, M, N, K, b_layout, 0, cta_group, group_m,
                         max_ctas, stream);
}

int b200_hgemm_f16_host(const void* a, const void* b, void* c, int M, int N, int K, int b_layout,
                        void* stream_) {
  if (!a || !b || !c || M <= 0 || N <= 0 || K <= 0) return fail(B200_EINVAL, "hgemm_host: bad args");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  auto up = [](size_t x) { return (x + 255) & ~static_cast<size_t>(255); };
  const size_t ab = up(static_cast<size_t>(M) * K * 2), bb = up(static_cast<size_t>(K) * N * 2),
               cb = up(static_cast<size_t>(M) * N * 2);
  void* ws = nullptr;
  int rc = b200::host::workspace(&ws, ab + bb + cb);
  if (rc) return rc;
  char* da = static_cast<char*>(ws);
  char* db = da + ab;
  char* dc = db + bb;

  // Pipeline over row panels of A / C: the H2D copy engine streams B, then A panel by panel;
  // the GEMM of panel i runs as soon as its rows have landed, the D2H engine drains C panel
  // i while panel i+1 is being copied in and multiplied.  With pinned host memory the call
  // costs ~ (bytes in) / PCIe instead of copy-in + compute + copy-out back to back.
  constexpr int kMaxPanels = 16;
  host::HostPipe* pp = nullptr;
  rc = host::host_pipe(&pp);
  if (rc) return rc;
  host::HostPipe& pipe = *pp;
  int panels = (M + 1023) / 1024;
  if (panels > kMaxPanels) panels = kMaxPanels;
  if (panels < 1) panels = 1;
  const int rows_per = ((M + panels - 1) / panels + 255) / 256 * 256;
  cudaEvent_t ev_start = pipe.ev[2 * kMaxPanels], ev_b = pipe.ev[2 * kMaxPanels + 1];
  B200_CUDA_OK(cudaEventRecord(ev_start, stream));           // order after prior work on `stream`
  B200_CUDA_OK(cudaStreamWaitEvent(pipe.in, ev_start, 0));
  B200_CUDA_OK(cudaStreamWaitEvent(pipe.out, ev_start, 0));
  B200_CUDA_OK(cudaMemcpyAsync(db, b, static_cast<size_t>(K) * N * 2, cudaMemcpyHostToDevice, pipe.in));
  B200_CUDA_OK(cudaEventRecord(ev_b, pipe.in));
  B200_CUDA_OK(cudaStreamWaitEvent(stream, ev_b, 0));
  int np = 0;
  for (int r0 = 0; r0 < M; r0 += rows_per, ++np) {
    const int rows = (M - r0 < rows_per) ? (M - r0) : rows_per;
    const char* ha = static_cast<const char*>(a) + static_cast<size_t>(r0) * K * 2;
    B200_CUDA_OK(cudaMemcpyAsync(da + static_cast<size_t>(r0) * K * 2, ha, static_cast<size_t>(rows) * K * 2,
                                 cudaMemcpyHostToDevice, pipe.in));
    B200_CUDA_OK(cudaEventRecord(pipe.ev[2 * np], pipe.in));
    B200_CUDA_OK(cudaStreamWaitEvent(stream, pipe.ev[2 * np], 0));
    rc = hgemm_impl(da + static_cast<size_t>(r0) * K * 2, db, dc + static_cast<size_t>(r0) * N * 2, rows, N, K,
                    b_layout, 0, 0, 0, 0, 0, 0, stream);
    if (rc) return rc;
    B200_CUDA_OK(cudaEventRecord(pipe.ev[2 * np + 1], stream));
    B200_CUDA_OK(cudaStreamWaitEvent(pipe.out, pipe.ev[2 * np + 1], 0));
    B200_CUDA_OK(cudaMemcpyAsync(static_cast<char*>(c) + static_cast<size_t>(r0) * N * 2,
                                 dc + static_cast<size_t>(r0) * N * 2, static_cast<size_t>(rows) * N * 2,
                                 cudaMemcpyDeviceToHost, pipe.out));
  }
  B200_CUDA_OK(cudaStreamSynchronize(pipe.out));
  B200_CUDA_OK(cudaStreamSynchronize(stream));
  return 0;
}

}  // extern "C"
