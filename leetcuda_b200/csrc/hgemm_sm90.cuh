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
//     rasterised tile list;
//   * CTAs in clusters of two (one CTA when there is a single m-tile): the two CTAs of a cluster
//     take the two m-tiles of one 256 x kBN pair tile, and each loads half of the shared B tile
//     with a TMA multicast into both CTAs' shared memory, so each B byte leaves L2 once per pair;
//   * warpgroup 0 = TMA producer (one thread; 128B-swizzled boxes, one k-block = 128 bytes of k),
//     warpgroups 1-2 = wgmma consumers, 64 rows each, accumulators in registers;
//   * smem ring (4 stages at kBN = 256, 6 at 128) guarded by full/empty mbarriers; one wgmma
//     group stays in flight while the stage before it is released to the producers of both
//     CTAs of the cluster;
//   * epilogue straight from the accumulator registers to global memory, fp16 C in 16-byte stores
//     after a transpose across each quad of lanes (and, for the fused
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

// Rasterisation: tiles are walked in groups of kGroupM m-tiles, and odd groups walk the n-tiles backwards,
// so a group starts on the B panels the previous group loaded last (still in L2).  With clusters of two the
// walk is over pair tiles (two m-tiles), kGroupM / 2 pairs per group.
constexpr int kGroupM = 16;
// L2 eviction priority of the operand loads: A panels (re-used by the other column tiles of the same row
// group) evict-last, B panels normal.
constexpr uint64_t kHintA = kEvictLast;
constexpr uint64_t kHintB = kEvictNormal;
// wgmma descriptor of the MN-major B operand (the fp16 [K,N] layout), which follows from its TMA boxes
// {64 n x 64 k} with 128B swizzle: the kBN / 64 boxes of one stage lie 8 KiB apart (LBO), a swizzle atom
// spans 8 k-rows (SBO 1 KiB), and a k16 step advances 16 k-rows (2 KiB).
constexpr uint32_t kBLbo = 8192;
constexpr uint32_t kBSbo = 1024;
constexpr uint32_t kBKStep = 2048;

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
  int num_tiles;           // cluster tiles: ceil(tiles_m / cluster size) x tiles_n
  // Fused all-gather of C (multi-GPU row sharding, SURVEY §8e): the epilogue stores every value
  // either through an NVLS multicast mapping (one multimem.st reaches the C buffer of every GPU,
  // this one included) or to C and to each peer-mapped C buffer.  All null/0 = C only.
  void* C_mc;
  void* C_peer[7];
  int n_peers;
};

// Cluster tile t of a cluster of `cs` CTAs -> this CTA's tile (tm, tn); the CTA of rank r takes m-tile cs * pm + r of
// cluster row pm.  With an odd tiles_m the last row's rank-1 m-tile lies past M.
__device__ __forceinline__ void tile_coords(const Params& p, int t, int cs, int rank, int& tm, int& tn) {
  const int rows = (p.tiles_m + cs - 1) / cs;
  const int group = kGroupM / cs;
  const int per_group = group * p.tiles_n;
  const int g = t / per_group;
  const int r = t - g * per_group;
  const int first = g * group;
  const int gm = min(group, rows - first);
  tn = r / gm;
  tm = (first + (r - tn * gm)) * cs + rank;
  if (g & 1) tn = p.tiles_n - 1 - tn;
}

// 2 fp32 values of C at element offset off
__device__ __forceinline__ void store_f32x2(const Params& p, size_t off, float2 v) {
  if (p.C_mc) {
    asm volatile("multimem.st.relaxed.sys.global.v2.f32 [%0], {%1, %2};" ::"l"(static_cast<char*>(p.C_mc) + off * 4),
                 "f"(v.x), "f"(v.y)
                 : "memory");
    return;
  }
  *reinterpret_cast<float2*>(static_cast<char*>(p.C) + off * 4) = v;
  for (int i = 0; i < p.n_peers; ++i) *reinterpret_cast<float2*>(static_cast<char*>(p.C_peer[i]) + off * 4) = v;
}

// 8 fp16 values of C at element offset off (16-byte aligned)
__device__ __forceinline__ void store_fp16x8(const Params& p, size_t off, uint4 v) {
  if (p.C_mc) {
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(
                     static_cast<char*>(p.C_mc) + off * 2),
                 "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w)
                 : "memory");
    return;
  }
  *reinterpret_cast<uint4*>(static_cast<char*>(p.C) + off * 2) = v;
  for (int i = 0; i < p.n_peers; ++i) *reinterpret_cast<uint4*>(static_cast<char*>(p.C_peer[i]) + off * 2) = v;
}

// 4 x 4 transpose of 32-bit words across the 4 lanes of a quad (q = lane % 4): on return x[k] of lane q holds what
// x[q] of lane k held.  Two butterfly stages, each swapping the two words whose index differs from q in that bit.
__device__ __forceinline__ void quad_transpose(uint32_t (&x)[4], int q) {
#pragma unroll
  for (int b = 1; b <= 2; b <<= 1) {
    const bool up = (q & b) != 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (k & b) continue;                     // pairs (k, k | b)
      const uint32_t send = up ? x[k] : x[k | b];
      const uint32_t got = __shfl_xor_sync(0xffffffffu, send, b);
      if (up) x[k] = got;
      else x[k | b] = got;
    }
  }
}

// kBMn: B is [K,N] (MN-major operand; fp16 only).  kTf32: fp32 operands through wgmma .tf32 (K-major
// A and B; a 128-byte row holds 32 elements: k-block 32, k-step 8).  kAcc16: fp16 accumulation
// (the reference's HMMA.F16 numerics, see b200_hgemm_f16_acc16).
// p is __grid_constant__ because the epilogue indexes p.C_peer at run time: a plain by-value struct of up to
// 128 bytes is then copied to local memory, a __grid_constant__ one is read in place from the parameter bank.
template <int kBN, bool kBMn, bool kTf32, bool kAcc16>
__global__ void __launch_bounds__(kThreads, 1)
hgemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                   const __grid_constant__ Params p) {
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
  // Cluster of cs = 1 or 2 CTAs (the host picks it).  Both CTAs walk the same cluster tiles in step.  A stage is
  // refilled only when the consumers of both CTAs have released it (empty counts the 8 consumer warps of each CTA),
  // because each producer writes half of B into its peer's stage too; that also means the peer's full barrier of the
  // stage has finished the phase the multicast refills.
  const int cs = static_cast<int>(cluster_nctarank());
  const int rank = static_cast<int>(cluster_ctarank());
  const int cluster = blockIdx.x / cs, clusters = gridDim.x / cs;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full(s), 1);
      mbar_init(empty(s), 8 * cs);   // lane 0 of every consumer warp of every CTA of the cluster
    }
    fence_mbar_init();
  }
  cluster_sync_all();   // the peer's barriers are initialised before any multicast or remote arrive

  if (wg == 0) {
    reg_dealloc<40>();
    if (tid == 0) {
      prefetch_tmap(&tmap_a);
      prefetch_tmap(&tmap_b);
      int it = 0;
      for (int t = cluster; t < p.num_tiles; t += clusters) {
        int tm, tn;
        tile_coords(p, t, cs, rank, tm, tn);
        const int m0 = tm * BM, n0 = tn * kBN;
        for (int kb = 0; kb < kblocks; ++kb, ++it) {
          const int s = it % STAGES;
          if (it >= STAGES) mbar_wait(empty(s), ((it / STAGES) - 1) & 1);
          const uint32_t sa = sbase + s * C_::STAGE_BYTES, sb = sa + C_::A_BYTES;
          // the whole stage, the half of B the peer multicasts included; an m-tile past M loads zeros (full count)
          mbar_expect_tx(full(s), C_::STAGE_BYTES);
          tma_load_2d(sa, &tmap_a, full(s), kb * BKE, m0, kHintA);
          if (cs == 1) {
            if constexpr (kBMn) {
#pragma unroll
              for (int c = 0; c < kBN / 64; ++c)
                tma_load_2d(sb + c * kBLbo, &tmap_b, full(s), n0 + 64 * c, kb * 64, kHintB);
            } else {
              tma_load_2d(sb, &tmap_b, full(s), kb * BKE, n0, kHintB);
            }
          } else if constexpr (kBMn) {   // the 64 x 64 boxes c = rank (mod 2)
#pragma unroll
            for (int c = 0; c < kBN / 64; c += 2)
              tma_load_2d_multicast(sb + (c + rank) * kBLbo, &tmap_b, full(s), n0 + 64 * (c + rank), kb * 64, 0x3,
                                    kHintB);
          } else {   // rows [rank kBN/2, (rank + 1) kBN/2) of the K-major tile: half-height boxes side by side
            tma_load_2d_multicast(sb + rank * (kBN / 2) * 128, &tmap_b, full(s), kb * BKE, n0 + rank * (kBN / 2), 0x3,
                                  kHintB);
          }
        }
      }
    }
  } else {
    reg_alloc<232>();
    using AccT = typename std::conditional<kAcc16, uint32_t, float>::type;
    AccT acc[NACC];
    const int warp = tid / 32, lane = tid % 32;
    // releases stage s in this CTA and, in a cluster of two, in the peer
    const uint32_t peer_bars = cs > 1 ? mapa(bars, static_cast<uint32_t>(rank ^ 1)) : 0u;
    auto release = [&](int s) {
      mbar_arrive(empty(s));
      if (cs > 1) mbar_arrive_cluster(peer_bars + 8u * (STAGES + s));
    };
    int it = 0;
    for (int t = cluster; t < p.num_tiles; t += clusters) {
      int tm, tn;
      tile_coords(p, t, cs, rank, tm, tn);
      const int m0 = tm * BM, n0 = tn * kBN;
#pragma unroll
      for (int i = 0; i < NACC; ++i) acc[i] = 0;
      for (int kb = 0; kb < kblocks; ++kb, ++it) {
        const int s = it % STAGES;
        mbar_wait(full(s), (it / STAGES) & 1);
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
            const uint64_t db = kBMn ? wg_desc(sb + ks * kBKStep, kBLbo, kBSbo) : wg_desc(sb + ks * 32, 16);
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
        if (kb > 0 && lane == 0) release((it - 1) % STAGES);
      }
      wg_wait<0>();
      wg_fence_regs(acc);
      if (kblocks > 0 && lane == 0) release((it - 1) % STAGES);

      // epilogue: thread owns rows r0, r0 + 8 and column pairs 8j + 2 (lane % 4) of its warpgroup's 64 x kBN block
      const int r0 = m0 + (wg - 1) * 64 + warp * 16 + lane / 4;
      if constexpr (!kTf32) {
        // fp16 C: the 4 lanes of a quad hold 8 consecutive columns of a row for each j; transposing the half2 words
        // of 4 consecutive j across the quad gives each lane 8 columns (16 bytes) of its own j, and a warp stores 64
        // contiguous bytes per row instead of 16
        const int q = lane % 4;
#pragma unroll
        for (int j0 = 0; j0 < kBN / 8; j0 += 4) {
          const int col = n0 + 8 * (j0 + q);
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            uint32_t x[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              if constexpr (kAcc16) x[k] = acc[2 * (j0 + k) + i];
              else x[k] = pack_half2(acc[4 * (j0 + k) + 2 * i], acc[4 * (j0 + k) + 2 * i + 1]);
            }
            quad_transpose(x, q);
            const int row = r0 + 8 * i;
            if (row < p.M && col < p.N)
              store_fp16x8(p, static_cast<size_t>(row) * p.ldc + col, make_uint4(x[0], x[1], x[2], x[3]));
          }
        }
      } else {
#pragma unroll
        for (int j = 0; j < kBN / 8; ++j) {
          const int col = n0 + 8 * j + 2 * (lane % 4);
          if (col >= p.N) continue;
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            const int row = r0 + 8 * i;
            if (row >= p.M) continue;
            store_f32x2(p, static_cast<size_t>(row) * p.ldc + col, make_float2(acc[4 * j + 2 * i], acc[4 * j + 2 * i + 1]));
          }
        }
      }
    }
  }
  cluster_sync_all();   // no CTA exits while its peer can still arrive on its barriers
}

}  // namespace hgemm
}  // namespace b200
