// hgemm_sm90.cuh — persistent, warp-specialised GEMM for sm_90a (H100).
//
//   C[M,N] = A[M,K] (row-major) x B      fp16 in / fp16 out (fp32 or fp16 accumulation)
//                                         or fp32 in / fp32 out through TF32 wgmma
//   B is either [K,N] row-major ("NN", MN-major wgmma operand, fp16 only) or
//                [N,K] row-major ("TN", K-major wgmma operand).
//
// Replaces the whole family of reference kernels behind the hgemm op surface
// (reference: kernels/hgemm/mma/swizzle/hgemm_mma_stage_swizzle.cu:174-596 and
// siblings, SURVEY.md §8a rows a1-a7), which tile 128x128x32 per 256-thread CTA
// with mma.sync + cp.async.  Here instead:
//
//   * one 128 x kBN output tile (kBN = 256 or 128) per step of a persistent CTA walking a
//     rasterised tile list (grid = min(#tiles, #SMs));
//   * warpgroup 0 = TMA producer (one thread; 128B-swizzled boxes, one k-block = 128 bytes of k),
//     warpgroups 1-2 = wgmma consumers, 64 rows each, accumulators in registers;
//   * smem ring (4 stages at kBN = 256, 6 at 128) guarded by full/empty mbarriers; one wgmma
//     group stays in flight while the stage before it is released to the producer;
//   * epilogue straight from the accumulator registers to global memory (and, for the fused
//     all-gather, to the peer GPUs' C buffers or through an NVLS multicast mapping), while the
//     producer already streams the next tile's operands.
#pragma once
#include <cuda.h>

#include <type_traits>

#include "sm90_ptx.cuh"

namespace b200 {
namespace hgemm {

constexpr int BM = 128;        // rows per tile: two consumer warpgroups x 64
constexpr int kThreads = 384;  // three warpgroups

template <int kBN>
struct Cfg {
  static constexpr int A_BYTES = BM * 128;     // 16 KiB: 128 rows x 128 bytes of k
  static constexpr int B_BYTES = kBN * 128;    // 32 / 16 KiB
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STAGES = (kBN == 256) ? 4 : 6;
  static constexpr int BAR_BYTES = 256;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + BAR_BYTES + 1024;  // + align slack
};

struct Params {
  void* C;                 // fp16 (or fp32 for tf32) [M, ldc]
  int M, N, K;
  int ldc;
  int tiles_m, tiles_n;    // in units of BM x kBN
  int group_m;             // rasterisation: m-tiles per L2 group
  int serpentine;          // odd groups walk the n-tiles backwards (reuses the last B panels in L2)
  int num_tiles;
  unsigned long long hint_a, hint_b;   // L2 cache-policy descriptors of the A / B TMA loads
  // wgmma descriptor fields of the MN-major B operand (bytes)
  uint32_t b_lbo, b_sbo, b_kstep;
  // Fused all-gather of C (multi-GPU row sharding, SURVEY §8e): the epilogue stores every value
  // either through an NVLS multicast mapping (one multimem.st reaches the C buffer of every GPU,
  // this one included) or to C and to each peer-mapped C buffer.  All null/0 = C only.
  void* C_mc;
  void* C_peer[7];
  int n_peers;
};

__device__ __forceinline__ void tile_coords(const Params& p, int t, int& tm, int& tn) {
  const int per_group = p.group_m * p.tiles_n;
  const int g = t / per_group;
  const int r = t - g * per_group;
  const int first_m = g * p.group_m;
  const int gm = min(p.group_m, p.tiles_m - first_m);
  tn = r / gm;
  tm = first_m + (r - tn * gm);
  if (p.serpentine && (g & 1)) tn = p.tiles_n - 1 - tn;
}

template <typename T>
__device__ __forceinline__ void store_pair(const Params& p, size_t off, T v) {
  if (p.C_mc) {
    static_assert(sizeof(T) == 4 || sizeof(T) == 8, "pair of fp16 or fp32");
    char* dst = static_cast<char*>(p.C_mc) + off * (sizeof(T) / 2);
    if constexpr (sizeof(T) == 4) {
      asm volatile("multimem.st.relaxed.sys.global.f32 [%0], %1;" ::"l"(dst),
                   "f"(*reinterpret_cast<const float*>(&v)) : "memory");
    } else {
      const float2 f = *reinterpret_cast<const float2*>(&v);
      asm volatile("multimem.st.relaxed.sys.global.v2.f32 [%0], {%1, %2};" ::"l"(dst), "f"(f.x), "f"(f.y)
                   : "memory");
    }
    return;
  }
  *reinterpret_cast<T*>(static_cast<char*>(p.C) + off * (sizeof(T) / 2)) = v;
  for (int i = 0; i < p.n_peers; ++i)
    *reinterpret_cast<T*>(static_cast<char*>(p.C_peer[i]) + off * (sizeof(T) / 2)) = v;
}

// kBMn: B is [K,N] (MN-major operand; fp16 only).  kTf32: fp32 operands through wgmma .tf32 (K-major
// A and B; a 128-byte row holds 32 elements: k-block 32, k-step 8).  kAcc16: fp16 accumulation
// (the reference's HMMA.F16 numerics, see b200_hgemm_f16_acc16).
template <int kBN, bool kBMn, bool kTf32, bool kAcc16>
__global__ void __launch_bounds__(kThreads, 1)
hgemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                   const Params p) {
  static_assert(!(kTf32 && (kBMn || kAcc16)), "tf32 operands are K-major with fp32 accumulation");
  using C_ = Cfg<kBN>;
  constexpr int STAGES = C_::STAGES;
  constexpr int BKE = kTf32 ? 32 : 64;   // elements per k-block = per 128-byte swizzle row
  constexpr int NACC = kAcc16 ? kBN / 4 : kBN / 2;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const uint32_t sbase = smem_u32(smem);
  const uint32_t bars = sbase + STAGES * C_::STAGE_BYTES;
  auto full = [&](int s) { return bars + 8u * s; };
  auto empty = [&](int s) { return bars + 8u * (STAGES + s); };

  const int wg = threadIdx.x / 128;
  const int tid = threadIdx.x % 128;
  const int kblocks = (p.K + BKE - 1) / BKE;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full(s), 1);
      mbar_init(empty(s), 8);   // lane 0 of every consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    reg_dealloc<40>();
    if (tid == 0) {
      prefetch_tmap(&tmap_a);
      prefetch_tmap(&tmap_b);
      int it = 0;
      for (int t = blockIdx.x; t < p.num_tiles; t += gridDim.x) {
        int tm, tn;
        tile_coords(p, t, tm, tn);
        const int m0 = tm * BM, n0 = tn * kBN;
        for (int kb = 0; kb < kblocks; ++kb, ++it) {
          const int s = it % STAGES;
          if (it >= STAGES) mbar_wait(empty(s), ((it / STAGES) - 1) & 1, 1);
          const uint32_t sa = sbase + s * C_::STAGE_BYTES, sb = sa + C_::A_BYTES;
          mbar_expect_tx(full(s), C_::STAGE_BYTES);
          tma_load_2d(sa, &tmap_a, full(s), kb * BKE, m0, p.hint_a);
          if constexpr (kBMn) {
#pragma unroll
            for (int c = 0; c < kBN / 64; ++c)
              tma_load_2d(sb + c * 8192, &tmap_b, full(s), n0 + 64 * c, kb * 64, p.hint_b);
          } else {
            tma_load_2d(sb, &tmap_b, full(s), kb * BKE, n0, p.hint_b);
          }
        }
      }
    }
    return;
  }

  reg_alloc<232>();
  using AccT = typename std::conditional<kAcc16, uint32_t, float>::type;
  AccT acc[NACC];
  const int warp = tid / 32, lane = tid % 32;
  int it = 0;
  for (int t = blockIdx.x; t < p.num_tiles; t += gridDim.x) {
    int tm, tn;
    tile_coords(p, t, tm, tn);
    const int m0 = tm * BM, n0 = tn * kBN;
#pragma unroll
    for (int i = 0; i < NACC; ++i) acc[i] = 0;
    for (int kb = 0; kb < kblocks; ++kb, ++it) {
      const int s = it % STAGES;
      mbar_wait(full(s), (it / STAGES) & 1, 2);
      const uint32_t sa = sbase + s * C_::STAGE_BYTES + (wg - 1) * 64 * 128, sb = sbase + s * C_::STAGE_BYTES + C_::A_BYTES;
      wg_fence();
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        const uint64_t da = wg_desc(sa + ks * 32, 16);
        const uint32_t go = (kb > 0 || ks > 0) ? 1u : 0u;
        if constexpr (kTf32) {
          const uint64_t db = wg_desc(sb + ks * 32, 16);
          if constexpr (kBN == 256) wgmma_ss_m64n256k8_f32_tf32(acc, da, db, go);
          else wgmma_ss_m64n128k8_f32_tf32(acc, da, db, go);
        } else {
          const uint64_t db = kBMn ? wg_desc(sb + ks * p.b_kstep, p.b_lbo, p.b_sbo) : wg_desc(sb + ks * 32, 16);
          constexpr int kTB = kBMn ? 1 : 0;
          if constexpr (kAcc16 && kBN == 256) wgmma_ss_m64n256k16_f16_f16<0, kTB>(acc, da, db, go);
          else if constexpr (kAcc16) wgmma_ss_m64n128k16_f16_f16<0, kTB>(acc, da, db, go);
          else if constexpr (kBN == 256) wgmma_ss_m64n256k16_f32_f16<0, kTB>(acc, da, db, go);
          else wgmma_ss_m64n128k16_f32_f16<0, kTB>(acc, da, db, go);
        }
      }
      wg_commit();
      // keep one group in flight: the previous k-block's stage is free once its group retired
      wg_wait<1>();
      if (kb > 0 && lane == 0) mbar_arrive(empty((it - 1) % STAGES));
    }
    wg_wait<0>();
    wg_fence_regs(acc);
    if (kblocks > 0 && lane == 0) mbar_arrive(empty((it - 1) % STAGES));

    // epilogue: thread owns rows r0, r0 + 8 and column pairs 8j + 2 (lane % 4) of its warpgroup's 64 x kBN block
    const int r0 = m0 + (wg - 1) * 64 + warp * 16 + lane / 4;
#pragma unroll
    for (int j = 0; j < kBN / 8; ++j) {
      const int col = n0 + 8 * j + 2 * (lane % 4);
      if (col >= p.N) continue;
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int row = r0 + 8 * i;
        if (row >= p.M) continue;
        const size_t off = static_cast<size_t>(row) * p.ldc + col;
        if constexpr (kAcc16) {
          store_pair(p, off, acc[2 * j + i]);
        } else if constexpr (kTf32) {
          store_pair(p, off, make_float2(acc[4 * j + 2 * i], acc[4 * j + 2 * i + 1]));
        } else {
          store_pair(p, off, pack_half2(acc[4 * j + 2 * i], acc[4 * j + 2 * i + 1]));
        }
      }
    }
  }
}

}  // namespace hgemm
}  // namespace b200
