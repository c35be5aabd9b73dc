// gemm_fp8_sm90.cuh — persistent, warp-specialised fp8 (e4m3) scaled GEMM for sm_90a (H100).
//
//   C[M,N] = OutT( scaled( A[M,K] . B[N,K]^T ) )      A, B e4m3, both K-major; OutT fp16 or bf16
//
// The skeleton is hgemm_wgmma_kernel's TN path (hgemm_sm90.cuh): the same persistent raster walk (tile_coords), two-CTA
// clusters that multicast the B tile, a TMA producer warpgroup feeding a ring of 128B-swizzled stages through full /
// empty mbarriers, and the quad-transposed 16-byte epilogue stores.  What differs:
//
//   * the tile is 128 x 128 (Cfg<128>: 6 stages of 16 KiB A + 16 KiB B); a 128-byte k-block holds 128 e4m3 values and
//     takes four m64n128k32 e4m3 wgmmas at +32 B on the descriptors;
//   * fp32 promotion per k-block: the first k32 wgmma of a k-block runs with scale-d = 0, so the tensor-core
//     accumulator holds that k-block's partial sum only; once its group has retired the consumer adds it into a second
//     set of fp32 registers (FADD, or FFMA with the k-block's scale for block scaling).  The wait per k-block leaves
//     this warpgroup's tensor-core slot to the other consumer warpgroup, whose wgmmas run during the adds;
//   * scales: kBlockScale = false applies (acc * sa[m]) * sb[n] in the epilogue (tensor-wise scaling is the row-wise
//     path with stride 0); kBlockScale = true folds fp32(sa[m, kb] * sb[n / 128, kb]) into every promotion
//     (DeepSeek-V3's 1 x 128 activation and 128 x 128 weight blocks).  Scales are read on the GPU only.
#pragma once
#include <cuda.h>

#include <type_traits>

#include "hgemm_sm90.cuh"
#include "sm90_ptx.cuh"

namespace b200 {
namespace gemm_fp8 {

constexpr int BM = hgemm::BM;    // 128 rows: two consumer warpgroups x 64
constexpr int BN = 128;          // columns per tile (= the 128 x 128 weight block of the block recipe)
constexpr int BK = 128;          // e4m3 values per k-block = one 128-byte swizzle row
constexpr int kThreads = hgemm::kThreads;
using C_ = hgemm::Cfg<BN>;

struct Params {
  hgemm::Params g;               // C, M, N, K, ldc, tiles and cluster tiles (the peer / multicast fields stay null)
  const float* sa;               // tensor / row: sa[m * sa_stride]; block: sa[m + kb * M] ([M, ceil(K/128)], M-major)
  const float* sb;               // tensor / row: sb[n * sb_stride]; block: sb[(n / 128) * kblocks + kb] (row-major)
  int sa_stride, sb_stride;      // 0 (tensor) or 1 (row); unused for block
};

// D (+)= A * B, m64n128k32, e4m3 x e4m3 -> fp32, both operands K-major from shared memory; acc = 0 overwrites D
B200_DEVICE void wgmma_ss_m64n128k32_f32_e4m3(float (&d)[64], uint64_t da, uint64_t db, uint32_t acc) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k32.f32.e4m3.e4m3 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(acc));
}

template <typename OutT>
B200_DEVICE uint32_t pack2(float lo, float hi) {
  if constexpr (std::is_same_v<OutT, __nv_bfloat16>) return pack_bf162(lo, hi);
  else return pack_half2(lo, hi);
}

template <typename OutT, bool kBlockScale>
__global__ void __launch_bounds__(kThreads, 1)
gemm_e4m3_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                 const __grid_constant__ Params p) {
  constexpr int STAGES = C_::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const uint32_t sbase = smem_u32(smem);
  const uint32_t bars = sbase + STAGES * C_::STAGE_BYTES;
  auto full = [&](int s) { return bars + 8u * s; };
  auto empty = [&](int s) { return bars + 8u * (STAGES + s); };

  const int wg = threadIdx.x / 128;
  const int tid = threadIdx.x % 128;
  const int M = p.g.M, N = p.g.N;
  const int kblocks = (p.g.K + BK - 1) / BK;
  // the cluster protocol of hgemm_wgmma_kernel: a stage is refilled once the consumers of both CTAs released it
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
  cluster_sync_all();

  if (wg == 0) {
    reg_dealloc<40>();
    if (tid == 0) {
      prefetch_tmap(&tmap_a);
      prefetch_tmap(&tmap_b);
      int it = 0;
      for (int t = cluster; t < p.g.num_tiles; t += clusters) {
        int tm, tn;
        hgemm::tile_coords(p.g, t, cs, rank, tm, tn);
        const int m0 = tm * BM, n0 = tn * BN;
        for (int kb = 0; kb < kblocks; ++kb, ++it) {
          const int s = it % STAGES;
          if (it >= STAGES) mbar_wait(empty(s), ((it / STAGES) - 1) & 1);
          const uint32_t sa = sbase + s * C_::STAGE_BYTES, sb = sa + C_::A_BYTES;
          mbar_expect_tx(full(s), C_::STAGE_BYTES);
          tma_load_2d(sa, &tmap_a, full(s), kb * BK, m0, hgemm::kHintA);
          if (cs == 1) tma_load_2d(sb, &tmap_b, full(s), kb * BK, n0, hgemm::kHintB);
          else   // rows [rank 64, rank 64 + 64) of the K-major B tile, into both CTAs
            tma_load_2d_multicast(sb + rank * (BN / 2) * 128, &tmap_b, full(s), kb * BK, n0 + rank * (BN / 2), 0x3,
                                  hgemm::kHintB);
        }
      }
    }
  } else {
    reg_alloc<232>();
    float acc[64];   // the tensor core's partial sum of the current k-block
    float sum[64];   // fp32 promoted sum
    const int warp = tid / 32, lane = tid % 32, q = lane % 4;
    const uint32_t peer_bars = cs > 1 ? mapa(bars, static_cast<uint32_t>(rank ^ 1)) : 0u;
    auto release = [&](int s) {
      mbar_arrive(empty(s));
      if (cs > 1) mbar_arrive_cluster(peer_bars + 8u * (STAGES + s));
    };
    int it = 0;
    for (int t = cluster; t < p.g.num_tiles; t += clusters) {
      int tm, tn;
      hgemm::tile_coords(p.g, t, cs, rank, tm, tn);
      const int m0 = tm * BM, n0 = tn * BN;
      // thread owns rows r0, r0 + 8 and column pairs 8j + 2q of its warpgroup's 64 x 128 block:
      // acc[4j + 2i + e] is C[r0 + 8i, n0 + 8j + 2q + e]
      const int r0 = m0 + (wg - 1) * 64 + warp * 16 + lane / 4;
#pragma unroll
      for (int i = 0; i < 64; ++i) sum[i] = 0.f;
      for (int kb = 0; kb < kblocks; ++kb, ++it) {
        // block scales of this k-block, loaded before the wait so their latency hides under the wgmmas
        float g0 = 0.f, g1 = 0.f;
        if constexpr (kBlockScale) {
          const size_t col = static_cast<size_t>(kb) * M;
          const float b_s = p.sb[static_cast<size_t>(tn) * kblocks + kb];
          const float a0 = r0 < M ? p.sa[col + r0] : 0.f;
          const float a1 = r0 + 8 < M ? p.sa[col + r0 + 8] : 0.f;
          g0 = a0 * b_s;
          g1 = a1 * b_s;
        }
        const int s = it % STAGES;
        mbar_wait(full(s), (it / STAGES) & 1);
        const uint32_t sa = sbase + s * C_::STAGE_BYTES + (wg - 1) * 64 * 128, sb = sbase + s * C_::STAGE_BYTES + C_::A_BYTES;
        wg_fence();
#pragma unroll
        for (int ks = 0; ks < 4; ++ks)
          wgmma_ss_m64n128k32_f32_e4m3(acc, wg_desc(sa + ks * 32, 16), wg_desc(sb + ks * 32, 16), ks > 0 ? 1u : 0u);
        wg_commit();
        wg_wait<0>();
        wg_fence_regs(acc);
        if (lane == 0) release(s);
        // promotion: one fp32 add (FFMA with the block scale) per accumulator
#pragma unroll
        for (int j = 0; j < 16; ++j) {
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int i = 4 * j + e;
            if constexpr (kBlockScale) sum[i] = fmaf(acc[i], e < 2 ? g0 : g1, sum[i]);
            else sum[i] += acc[i];
          }
        }
      }

      // epilogue: (sum * sa[m]) * sb[n], one rounding to OutT, quad-transposed 16-byte stores masked to M x N
      float ra[2] = {1.f, 1.f};
      if constexpr (!kBlockScale) {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int row = r0 + 8 * i;
          ra[i] = row < M ? p.sa[static_cast<size_t>(row) * p.sa_stride] : 0.f;
        }
      }
#pragma unroll
      for (int j0 = 0; j0 < BN / 8; j0 += 4) {
        const int col = n0 + 8 * (j0 + q);
        float cb[4][2];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int c = n0 + 8 * (j0 + k) + 2 * q + e;
            cb[k][e] = 1.f;
            if constexpr (!kBlockScale) cb[k][e] = c < N ? p.sb[static_cast<size_t>(c) * p.sb_stride] : 0.f;
          }
        }
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          uint32_t x[4];
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            float v0 = sum[4 * (j0 + k) + 2 * i], v1 = sum[4 * (j0 + k) + 2 * i + 1];
            if constexpr (!kBlockScale) {
              v0 = (v0 * ra[i]) * cb[k][0];
              v1 = (v1 * ra[i]) * cb[k][1];
            }
            x[k] = pack2<OutT>(v0, v1);
          }
          hgemm::quad_transpose(x, q);
          const int row = r0 + 8 * i;
          if (row < M && col < N)
            *reinterpret_cast<uint4*>(static_cast<char*>(p.g.C) + (static_cast<size_t>(row) * p.g.ldc + col) * 2) =
                make_uint4(x[0], x[1], x[2], x[3]);
        }
      }
    }
  }
  cluster_sync_all();   // no CTA exits while its peer can still arrive on its barriers
}

}  // namespace gemm_fp8
}  // namespace b200
