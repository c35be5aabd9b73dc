// attn_capi.cu — C-ABI entry points of the attention path (include/leetcuda_b200.h).
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "capi_common.cuh"
#include "attn_sm90.cuh"

namespace {

using namespace b200;
using b200::host::fail;

template <int kDS, int kBN, int kWG, bool kVT>
int launch_attn(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, const attn::Params& p, int qtiles,
                int BH, int smem, bool causal, cudaStream_t stream) {
  auto kern = causal ? attn::attn_fwd_kernel<kDS, kBN, kWG, kVT, true> : attn::attn_fwd_kernel<kDS, kBN, kWG, kVT, false>;
  static int attr_smem[2][64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev >= 0 && dev < 64 && attr_smem[causal][dev] < smem) {
    B200_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    attr_smem[causal][dev] = smem;
  }
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(static_cast<unsigned>(qtiles * p.slabs), static_cast<unsigned>(BH), 1);
  cfg.blockDim = dim3(attn::threads<kWG>(), 1, 1);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attrs[1];
  attrs[0].id = cudaLaunchAttributeClusterDimension;   // the slabs of one query tile (fused RMS norm)
  attrs[0].val.clusterDim.x = (p.rms_g > 0.f) ? static_cast<unsigned>(p.slabs) : 1u;
  attrs[0].val.clusterDim.y = 1;
  attrs[0].val.clusterDim.z = 1;
  cfg.attrs = attrs;
  cfg.numAttrs = 1;
  B200_CUDA_OK(cudaLaunchKernelEx(&cfg, kern, tq, tk, tv, p));
  host::count_launch();
  return 0;
}

// [BH, D, N] -> [BH, N, D] (fp16): the three reference ops that take V pre-transposed
// (flash_attn_mma.py:441-442) are served for D > 128 by restoring the natural layout first —
// an HBM-bound pre-pass (4*N*D bytes per head) in front of a tensor-bound kernel.
__global__ void transpose_dn_to_nd_kernel(const __half* __restrict__ in, __half* __restrict__ out, int D, int N) {
  __shared__ __half tile[32][33];
  const size_t head = static_cast<size_t>(blockIdx.z) * D * N;
  const int n0 = blockIdx.x * 32, d0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int d = d0 + i, n = n0 + threadIdx.x;
    if (d < D && n < N) tile[i][threadIdx.x] = in[head + static_cast<size_t>(d) * N + n];
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int n = n0 + i, d = d0 + threadIdx.x;
    if (d < D && n < N) out[head + static_cast<size_t>(n) * D + d] = tile[threadIdx.x][i];
  }
}

// Kernel shape per head dim (attn_sm90.cuh):
//   D <= 64        one 64-column slab, 128-key blocks, two consumer warpgroups (128 query rows)
//   64 < D <= 128  one 128-column slab, 64-key blocks, two consumer warpgroups
//   128 < D        256-column slabs (S recomputed per slab), 64-key blocks, one consumer warpgroup (64 query rows)
// The S, P and O fragments of a consumer thread have to fit its registers: ptxas gives a 384-thread CTA
// 168 per thread, a 256-thread CTA 255 (O of a 256-column slab alone takes 128).
int fmha_dispatch(const void* q, const void* k, const void* v, void* o, float* lse, float rms_g, int B, int H, int Nq,
                  int Nk, int D, bool vt, bool causal, float scale, cudaStream_t stream) {
  const uint64_t BH = static_cast<uint64_t>(B) * H;
  const int ds = D <= 64 ? 64 : (D <= 128 ? 128 : 256);
  const int bn = ds == 64 ? 128 : 64;
  const int wgs = ds == 256 ? 1 : 2;
  attn::Params p;
  p.Nq = Nq;
  p.Nk = Nk;
  p.D = D;
  p.nq = (D + 63) / 64;
  p.num_kv = (Nk + bn - 1) / bn;
  p.diag = Nk - Nq;
  p.slabs = (D + ds - 1) / ds;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.lse = lse;
  p.rms_g = rms_g;
  p.o_ptr = static_cast<__half*>(o);
  if (rms_g > 0.f && D > 256 && !(D <= 512 && D % 128 == 0))
    return fail(B200_ENOTSUP, "fused rms_norm: D=%d (supported: D <= 256, 384, 512)", D);
  // ring: every slot that fits next to Q, at most 16 (two key blocks of K and V chunks at D = 512)
  const int kMaxSmem = 227 * 1024;
  const int slot = attn::slot_bytes(bn, ds, vt);
  const int fixed = attn::smem_bytes(wgs, slot, p.nq, 0);
  p.ring = (kMaxSmem - fixed) / (slot + 16);
  if (p.ring > 16) p.ring = 16;
  if (p.ring < 2) return fail(B200_ENOTSUP, "headdim not support! (D=%d)", D);
  const int smem = attn::smem_bytes(wgs, slot, p.nq, p.ring);
  const int qtiles = (Nq + 64 * wgs - 1) / (64 * wgs);

  CUtensorMap tq, tk, tv;
  uint64_t qdims[3] = {static_cast<uint64_t>(D), static_cast<uint64_t>(Nq), BH};
  uint64_t qstr[2] = {static_cast<uint64_t>(D) * 2, static_cast<uint64_t>(Nq) * D * 2};
  uint64_t kdims[3] = {static_cast<uint64_t>(D), static_cast<uint64_t>(Nk), BH};
  uint64_t kstr[2] = {static_cast<uint64_t>(D) * 2, static_cast<uint64_t>(Nk) * D * 2};
  uint32_t qbox[3] = {64, 64, 1};
  uint32_t kbox[3] = {64, static_cast<uint32_t>(bn), 1};
  int rc;
  if ((rc = host::get_tmap(&tq, q, 3, qdims, qstr, qbox, CU_TENSOR_MAP_SWIZZLE_128B))) return rc;
  if ((rc = host::get_tmap(&tk, k, 3, kdims, kstr, kbox, CU_TENSOR_MAP_SWIZZLE_128B))) return rc;
  if (vt) {
    uint64_t vd[3] = {static_cast<uint64_t>(Nk), static_cast<uint64_t>(D), BH};
    uint64_t vs[2] = {static_cast<uint64_t>(Nk) * 2, static_cast<uint64_t>(Nk) * D * 2};
    uint32_t vb[3] = {64, static_cast<uint32_t>(ds), 1};
    if ((rc = host::get_tmap(&tv, v, 3, vd, vs, vb, CU_TENSOR_MAP_SWIZZLE_128B))) return rc;
  } else {
    if ((rc = host::get_tmap(&tv, v, 3, kdims, kstr, kbox, CU_TENSOR_MAP_SWIZZLE_128B))) return rc;
  }
  const int bh = static_cast<int>(BH);
  if (ds == 64) return vt ? launch_attn<64, 128, 2, true>(tq, tk, tv, p, qtiles, bh, smem, causal, stream)
                          : launch_attn<64, 128, 2, false>(tq, tk, tv, p, qtiles, bh, smem, causal, stream);
  if (ds == 128) return vt ? launch_attn<128, 64, 2, true>(tq, tk, tv, p, qtiles, bh, smem, causal, stream)
                           : launch_attn<128, 64, 2, false>(tq, tk, tv, p, qtiles, bh, smem, causal, stream);
  if (vt) return fail(B200_EINVAL, "fmha: internal dispatch error (transposed V with D=%d)", D);
  return launch_attn<256, 64, 1, false>(tq, tk, tv, p, qtiles, bh, smem, causal, stream);
}

// The checks common to every attention entry and the transpose pre-pass.  The entries with one sequence length pass
// Nq = Nk = N; b200_fmha_fwd_f16_kv checks its own lengths, causal flag and Nk % 8 first, with messages naming them.
int fmha_impl(const void* q, const void* k, const void* v, void* o, float* lse, int B, int H, int Nq, int Nk, int D,
              int v_transposed, bool causal, float scale, void* stream_, float rms_g = 0.f) {
  if (!q || !k || !v || !o) return fail(B200_EINVAL, "fmha: null pointer");
  if (B <= 0 || H <= 0 || Nq <= 0 || Nk <= 0 || D <= 0)
    return fail(B200_EINVAL, "fmha: bad shape B=%d H=%d N=%d D=%d", B, H, Nq, D);
  if (static_cast<long long>(B) * H > 65535)
    return fail(B200_EINVAL, "fmha: B*H = %lld exceeds the grid limit 65535", static_cast<long long>(B) * H);
  if (D % 8 != 0) return fail(B200_ENOTSUP, "headdim not support! (D=%d must be a multiple of 8)", D);
  if (D > 1024) return fail(B200_ENOTSUP, "headdim not support! (D=%d > 1024)", D);
  if (v_transposed && (Nk % 8) != 0)
    return fail(B200_EINVAL, "fmha: N (%d) must be a multiple of 8 for transposed V", Nk);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!(scale > 0.f)) scale = 1.0f / sqrtf(static_cast<float>(D));
  if (D > 128) {
    if (v_transposed) {
      // the restored V lives in a stream-ordered allocation: calls on different streams never share
      // scratch, nothing stays pinned between calls, and neither the allocation nor the free
      // synchronises the device (the memory returns to the pool once this stream passes the free)
      void* ws = nullptr;
      const size_t bytes = static_cast<size_t>(B) * H * Nk * D * 2;
      B200_CUDA_OK(cudaMallocAsync(&ws, bytes, stream));
      dim3 grid((Nk + 31) / 32, (D + 31) / 32, B * H), block(32, 8, 1);
      transpose_dn_to_nd_kernel<<<grid, block, 0, stream>>>(static_cast<const __half*>(v),
                                                            static_cast<__half*>(ws), D, Nk);
      cudaError_t le = cudaGetLastError();
      int rc = 0;
      if (le != cudaSuccess) rc = fail(B200_ECUDA, "transpose launch failed: %s", cudaGetErrorString(le));
      else {
        host::count_launch();
        rc = fmha_dispatch(q, k, ws, o, lse, rms_g, B, H, Nq, Nk, D, false, causal, scale, stream);
      }
      cudaFreeAsync(ws, stream);
      return rc;
    }
  }
  return fmha_dispatch(q, k, v, o, lse, rms_g, B, H, Nq, Nk, D, v_transposed != 0, causal, scale, stream);
}

}  // namespace

extern "C" {

int b200_fmha_fwd_f16(const void* q, const void* k, const void* v, void* o, int B, int H, int N,
                      int D, int v_transposed, float scale, void* stream) {
  return fmha_impl(q, k, v, o, nullptr, B, H, N, N, D, v_transposed, false, scale, stream);
}

int b200_fmha_fwd_f16_lse(const void* q, const void* k, const void* v, void* o, float* lse, int B, int H,
                          int N, int D, int v_transposed, float scale, void* stream) {
  if (!lse) return fail(B200_EINVAL, "fmha_lse: null lse pointer");
  return fmha_impl(q, k, v, o, lse, B, H, N, N, D, v_transposed, false, scale, stream);
}

int b200_fmha_fwd_f16_kv(const void* q, const void* k, const void* v, void* o, float* lse, int B, int H, int Nq,
                         int Nk, int D, int v_transposed, int causal, float scale, void* stream) {
  if (Nq <= 0 || Nk <= 0) return fail(B200_EINVAL, "fmha_kv: bad lengths Nq=%d Nk=%d (both must be >= 1)", Nq, Nk);
  if (causal != 0 && causal != 1) return fail(B200_EINVAL, "fmha_kv: causal must be 0 or 1, got %d", causal);
  if (v_transposed && (Nk % 8) != 0)
    return fail(B200_EINVAL, "fmha_kv: Nk (%d) must be a multiple of 8 for transposed V", Nk);
  return fmha_impl(q, k, v, o, lse, B, H, Nq, Nk, D, v_transposed, causal == 1, scale, stream);
}

int b200_fmha_fwd_f16_rmsnorm(const void* q, const void* k, const void* v, void* o, float* lse, int B, int H,
                              int N, int D, int v_transposed, float scale, float rms_g, void* stream) {
  return fmha_impl(q, k, v, o, lse, B, H, N, N, D, v_transposed, false, scale, stream, rms_g > 0.f ? rms_g : 0.f);
}

int b200_fmha_fwd_f16_host(const void* q, const void* k, const void* v, void* o, int B, int H,
                           int N, int D, int v_transposed, float scale, void* stream_) {
  if (!q || !k || !v || !o || B <= 0 || H <= 0 || N <= 0 || D <= 0)
    return fail(B200_EINVAL, "fmha_host: bad args");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const int BH = B * H;
  const size_t head = static_cast<size_t>(N) * D * 2;            // bytes of one (b,h) slice
  const size_t bytes = head * BH;
  const size_t slot = (bytes + 255) & ~static_cast<size_t>(255);
  void* ws = nullptr;
  int rc = b200::host::workspace(&ws, 4 * slot);
  if (rc) return rc;
  char* dq = static_cast<char*>(ws);
  char* dk = dq + slot;
  char* dv = dk + slot;
  char* dout = dv + slot;
  // (batch x head) units are independent: pipeline chunks of heads through the copy engines
  // (H2D of chunk i+1 and D2H of chunk i-1 overlap the kernel of chunk i)
  host::HostPipe* pp = nullptr;
  if ((rc = host::host_pipe(&pp))) return rc;
  host::HostPipe& pipe = *pp;
  int chunks = BH < 16 ? BH : 16;
  const int per = (BH + chunks - 1) / chunks;
  cudaEvent_t ev_start = pipe.ev[host::kPipeEvents - 1];
  B200_CUDA_OK(cudaEventRecord(ev_start, stream));
  B200_CUDA_OK(cudaStreamWaitEvent(pipe.in, ev_start, 0));
  B200_CUDA_OK(cudaStreamWaitEvent(pipe.out, ev_start, 0));
  int ci = 0;
  for (int h0 = 0; h0 < BH; h0 += per, ++ci) {
    const int nh = (BH - h0 < per) ? (BH - h0) : per;
    const size_t off = head * h0, len = head * nh;
    B200_CUDA_OK(cudaMemcpyAsync(dq + off, static_cast<const char*>(q) + off, len, cudaMemcpyHostToDevice, pipe.in));
    B200_CUDA_OK(cudaMemcpyAsync(dk + off, static_cast<const char*>(k) + off, len, cudaMemcpyHostToDevice, pipe.in));
    B200_CUDA_OK(cudaMemcpyAsync(dv + off, static_cast<const char*>(v) + off, len, cudaMemcpyHostToDevice, pipe.in));
    B200_CUDA_OK(cudaEventRecord(pipe.ev[2 * ci], pipe.in));
    B200_CUDA_OK(cudaStreamWaitEvent(stream, pipe.ev[2 * ci], 0));
    rc = fmha_impl(dq + off, dk + off, dv + off, dout + off, nullptr, 1, nh, N, N, D, v_transposed, false, scale,
                   stream);
    if (rc) return rc;
    B200_CUDA_OK(cudaEventRecord(pipe.ev[2 * ci + 1], stream));
    B200_CUDA_OK(cudaStreamWaitEvent(pipe.out, pipe.ev[2 * ci + 1], 0));
    B200_CUDA_OK(cudaMemcpyAsync(static_cast<char*>(o) + off, dout + off, len, cudaMemcpyDeviceToHost, pipe.out));
  }
  B200_CUDA_OK(cudaStreamSynchronize(pipe.out));
  B200_CUDA_OK(cudaStreamSynchronize(stream));
  return 0;
}

}  // extern "C"
