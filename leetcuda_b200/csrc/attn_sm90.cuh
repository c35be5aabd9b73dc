// attn_sm90.cuh — FlashAttention-2 forward for sm_90a (H100): TMA + mbarrier + wgmma.
//
//   O = softmax(Q K^T * scale) V per (batch, head), fp16 in / out, fp32 scores, statistics and O.
//
// One CTA = kWG consumer warpgroups (64 query rows each) + one producer warpgroup (one thread
// issuing TMA).  Every CTA owns one query tile and one column slab of O (kDS columns); for
// D > kDS several CTAs share a query tile and each recomputes S for its slab.
//
//   * Q (all of D) stays in shared memory, 64-column chunks of 64 rows, 128B-swizzled;
//   * K and V stream through one ring of 128B-swizzled chunks guarded by full / empty
//     mbarriers: per key block of kBN keys, ceil(D/64) K chunks {64 d, kBN keys}, then the
//     slab's V chunks ({64 d, kBN keys}, or {64 keys, kDS d} for V given as [B,H,D,N]);
//   * S = Q K^T: wgmma m64 n=kBN k16 from shared memory, one commit group per K chunk so that a
//     chunk returns to the producer as soon as its group retired;
//   * online softmax in registers (ex2.approx; for D <= 128 a fixed quarter of the keys through the FMA-pipe
//     polynomial of softmax_math.cuh), P rounded to fp16 and fed
//     to P V as the register A operand (the accumulator layout of S is the A-fragment layout);
//   * O = P V: wgmma m64n64k16 per 64-column chunk of the slab.
#pragma once
#include <cuda.h>

#include "softmax_math.cuh"

namespace b200 {
namespace attn {

struct Params {
  int N, D;
  int num_kv;          // key blocks of kBN keys
  int nq;              // 64-column chunks of D (Q and K)
  int ring;            // K/V ring slots
  int slabs;           // column slabs of O per query tile
  float scale_log2;    // softmax scale * log2(e)
  float* lse;          // [B*H, N] natural-log LSE, or nullptr
  float rms_g;         // > 0: RMS-normalise every output row; with several slabs the CTAs of a query tile form
                       // a cluster and add up the row statistics through distributed shared memory
  __half* o_ptr;
};

// Keys whose exponential the D <= 128 kernels evaluate on the FMA pipe (exp2_fma_pipe) instead of MUFU.EX2: bit i
// selects the key pair (2i, 2i + 1) of every 32 keys.  A thread holds the pairs 8 jj + 2 (lane % 4), i.e. pair
// 4 (jj % 4) + lane % 4, so a selection that is uniform over a warp takes whole nibbles.
// Kept although this kernel is not MUFU-bound (it costs 0.3 % at D = 128 and 1.5 % at D = 64, DESIGN.md §5): the
// MUFU pipe executes 16 exponentials per clock per SM, i.e. >= 0.5 ms of B4 H32 N4096 D128 whatever the MMAs do, and
// it becomes the bound once the softmax overlaps the MMAs of the next block — the next step for this kernel.  The
// quarter moves O by < 2e-4 (tests/test_softmax_math.py).  -DB200_ATTN_POLY_MASK=0x0u -DB200_ATTN_POLY_MASK_D64=0x0u
// compiles every exponential onto MUFU.EX2.
#ifndef B200_ATTN_POLY_MASK
#define B200_ATTN_POLY_MASK 0x000Fu       // head dims 65 .. 128
#endif
#ifndef B200_ATTN_POLY_MASK_D64
#define B200_ATTN_POLY_MASK_D64 0x000Fu   // head dims <= 64
#endif

template <int kWG>
constexpr int threads() { return 128 * (kWG + 1); }

// one ring slot: a {64 columns, bn keys} chunk of K or V, or a {64 keys, ds columns} chunk of V^T
__host__ __device__ constexpr int slot_bytes(int bn, int ds, bool vt) { return 128 * (vt && ds > bn ? ds : bn); }
inline int smem_bytes(int kWG, int slot, int nq, int ring) {
  return kWG * nq * 8192 + ring * slot + 8 * (1 + 2 * ring) + kWG * 64 * 4 + 1024;
}

// kDS: columns of O per CTA (64, 128 or 256); kBN: keys per block; kVT: V is [B,H,D,N].
template <int kDS, int kBN, int kWG, bool kVT>
__global__ void __launch_bounds__(threads<kWG>(), 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                const __grid_constant__ CUtensorMap tmap_v, const Params p) {
  static_assert(!kVT || kDS <= 128, "transposed V: one slab of <= 128 columns");
  constexpr int SLOT = slot_bytes(kBN, kDS, kVT);
  constexpr int KV_BYTES = 64 * kBN * 2;   // one {64 columns, kBN keys} chunk of K or V
  constexpr int NS = kBN / 2;     // S accumulator registers per thread
  constexpr int NDC = kDS / 64;   // 64-column chunks of the slab
  constexpr uint32_t kPolyMask = kDS <= 64 ? B200_ATTN_POLY_MASK_D64 : (kDS <= 128 ? B200_ATTN_POLY_MASK : 0u);
  static_assert((kPolyMask & 0x1111u) * 0xF == kPolyMask, "the FMA-pipe selection must take whole nibbles");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const uint32_t sq = smem_u32(smem);
  const uint32_t sring = sq + kWG * p.nq * 8192;
  const uint32_t bars = sring + p.ring * SLOT;
  const uint32_t qbar = bars;
  const uint32_t rowss = bars + 8u * (1 + 2 * p.ring);   // per-row sum of squares (fused RMS norm over slabs)
  const bool rms_cluster = p.rms_g > 0.f && p.slabs > 1;
  auto full = [&](int s) { return bars + 8u * (1 + s); };
  auto empty = [&](int s) { return bars + 8u * (1 + p.ring + s); };

  const int wg = threadIdx.x / 128, tid = threadIdx.x % 128;
  const int qtile = blockIdx.x / p.slabs, slab = blockIdx.x % p.slabs;
  const int bh = blockIdx.y;
  const int q0 = qtile * 64 * kWG;
  const int d0 = slab * kDS;
  // V chunks of this slab per key block
  const int nvc = kVT ? kBN / 64 : min(NDC, (p.D - d0 + 63) / 64);

  if (threadIdx.x == 0) {
    mbar_init(qbar, 1);
    for (int s = 0; s < p.ring; ++s) {
      mbar_init(full(s), 1);
      mbar_init(empty(s), 4 * kWG);   // lane 0 of every consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    if constexpr (kWG > 1) reg_dealloc<40>();
    if (tid == 0) {
      prefetch_tmap(&tmap_q);
      prefetch_tmap(&tmap_k);
      prefetch_tmap(&tmap_v);
      mbar_expect_tx(qbar, kWG * p.nq * 8192);
      for (int w = 0; w < kWG; ++w)
        for (int c = 0; c < p.nq; ++c)
          tma_load_3d(sq + (w * p.nq + c) * 8192, &tmap_q, qbar, 64 * c, q0 + 64 * w, bh, kEvictFirst);
      int it = 0;
      auto next = [&](uint32_t bytes) {
        const int s = it % p.ring;
        if (it >= p.ring) mbar_wait(empty(s), ((it / p.ring) - 1) & 1, 11);
        mbar_expect_tx(full(s), bytes);
        ++it;
        return s;
      };
      for (int j = 0; j < p.num_kv; ++j) {
        for (int c = 0; c < p.nq; ++c) {
          const int s = next(KV_BYTES);
          tma_load_3d(sring + s * SLOT, &tmap_k, full(s), 64 * c, j * kBN, bh, kEvictLast);
        }
        for (int c = 0; c < nvc; ++c) {
          if constexpr (kVT) {
            const int s = next(64 * kDS * 2);
            tma_load_3d(sring + s * SLOT, &tmap_v, full(s), j * kBN + 64 * c, d0, bh, kEvictLast);
          } else {
            const int s = next(KV_BYTES);
            tma_load_3d(sring + s * SLOT, &tmap_v, full(s), d0 + 64 * c, j * kBN, bh, kEvictLast);
          }
        }
      }
    }
    if (rms_cluster) {   // the consumers' two cluster barriers (epilogue)
      cluster_sync_all();
      cluster_sync_all();
    }
    return;
  }

  if constexpr (kWG > 1) reg_alloc<232>();
  const int w = wg - 1, warp = tid / 32, lane = tid % 32;
  float o[NDC][32];
#pragma unroll
  for (int c = 0; c < NDC; ++c)
#pragma unroll
    for (int i = 0; i < 32; ++i) o[c][i] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  mbar_wait(qbar, 0, 12);

  int it = 0;
  auto release = [&](int i) {
    if (lane == 0) mbar_arrive(empty(i % p.ring));
  };
  for (int j = 0; j < p.num_kv; ++j) {
    // ---- S = Q K^T over the d-chunks
    float s[NS];
    wg_fence();
    for (int c = 0; c < p.nq; ++c, ++it) {
      mbar_wait(full(it % p.ring), (it / p.ring) & 1, 13);
      const uint32_t qa = sq + (w * p.nq + c) * 8192, ka = sring + (it % p.ring) * SLOT;
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        const uint64_t da = wg_desc(qa + ks * 32, 16), db = wg_desc(ka + ks * 32, 16);
        const uint32_t go = (c > 0 || ks > 0) ? 1u : 0u;
        if constexpr (kBN == 128) wgmma_ss_m64n128k16_f32_f16<0, 0>(s, da, db, go);
        else wgmma_ss_m64n64k16_f32_f16<0, 0>(s, da, db, go);
      }
      wg_commit();
      wg_wait<1>();
      if (c > 0) release(it - 1);
    }
    wg_wait<0>();
    wg_fence_regs(s);
    release(it - 1);

    // ---- online softmax: this thread holds rows (lane/4) and (lane/4 + 8) of its warp's 16 rows,
    // columns 8 jj + 2 (lane % 4) + {0, 1}: s[4 jj + 2 i + e]
    const int kbase = j * kBN + 2 * (lane % 4);
    if (j * kBN + kBN > p.N) {
#pragma unroll
      for (int jj = 0; jj < kBN / 8; ++jj)
#pragma unroll
        for (int e = 0; e < 2; ++e)
          if (kbase + 8 * jj + e >= p.N) {
            s[4 * jj + e] = -INFINITY;
            s[4 * jj + 2 + e] = -INFINITY;
          }
    }
    float alpha[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      float mx = -INFINITY;
#pragma unroll
      for (int jj = 0; jj < kBN / 8; ++jj) mx = fmaxf(mx, fmaxf(s[4 * jj + 2 * i], s[4 * jj + 2 * i + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float mn = fmaxf(m[i], mx * p.scale_log2);
      alpha[i] = fast_exp2(m[i] - mn);
      m[i] = mn;
      float sum = 0.f;
#pragma unroll
      for (int jj = 0; jj < kBN / 8; ++jj)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float x = fmaf(s[4 * jj + 2 * i + e], p.scale_log2, -mn);
          const float pe = ((kPolyMask >> (4 * (jj % 4))) & 1u) ? exp2_fma_pipe(x) : fast_exp2(x);
          s[4 * jj + 2 * i + e] = pe;
          sum += pe;
        }
      l[i] = l[i] * alpha[i] + sum;
    }
#pragma unroll
    for (int c = 0; c < NDC; ++c)
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        o[c][4 * jj + 0] *= alpha[0];
        o[c][4 * jj + 1] *= alpha[0];
        o[c][4 * jj + 2] *= alpha[1];
        o[c][4 * jj + 3] *= alpha[1];
      }
    // P (fp16) as the A fragments of the k16 steps over the keys of this block
    uint32_t pa[kBN / 16][4];
#pragma unroll
    for (int kk = 0; kk < kBN / 16; ++kk) {
      pa[kk][0] = pack_half2(s[8 * kk + 0], s[8 * kk + 1]);
      pa[kk][1] = pack_half2(s[8 * kk + 2], s[8 * kk + 3]);
      pa[kk][2] = pack_half2(s[8 * kk + 4], s[8 * kk + 5]);
      pa[kk][3] = pack_half2(s[8 * kk + 6], s[8 * kk + 7]);
    }

    // ---- O += P V over the slab's V chunks
    wg_fence();
#pragma unroll
    for (int c = 0; c < (kVT ? kBN / 64 : NDC); ++c) {
      if (c >= nvc) break;
      mbar_wait(full(it % p.ring), (it / p.ring) & 1, 14);
      const uint32_t va = sring + (it % p.ring) * SLOT;
      if constexpr (kVT) {
        // chunk c = keys 64c .. 64c+63 (K-major rows of V^T), all kDS columns
#pragma unroll
        for (int kq = 0; kq < 4; ++kq)
#pragma unroll
          for (int dc = 0; dc < NDC; ++dc)
            wgmma_rs_m64n64k16_f32_f16<0>(o[dc], pa[4 * c + kq], wg_desc(va + dc * 8192 + kq * 32, 16), 1u);
      } else {
        // chunk c = columns d0 + 64c .. +63 for all kBN keys (MN-major)
#pragma unroll
        for (int kk = 0; kk < kBN / 16; ++kk)
          wgmma_rs_m64n64k16_f32_f16<1>(o[c], pa[kk], wg_desc(va + kk * 2048, 8192), 1u);
      }
      wg_commit();
      wg_wait<1>();
      if (c > 0) release(it - 1);
      ++it;
    }
    wg_wait<0>();
#pragma unroll
    for (int c = 0; c < NDC; ++c) wg_fence_regs(o[c]);
    if (nvc > 0) release(it - 1);
  }

  // ---- epilogue
  const size_t head = static_cast<size_t>(bh) * p.N;
  float inv[2], lsum[2], ss[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    float lt = l[i];
    lt += __shfl_xor_sync(0xffffffffu, lt, 1);
    lt += __shfl_xor_sync(0xffffffffu, lt, 2);
    lsum[i] = lt;
    inv[i] = 1.f / lt;
    ss[i] = 0.f;
    if (p.rms_g > 0.f) {
#pragma unroll
      for (int c = 0; c < NDC; ++c)
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          const float a = o[c][4 * jj + 2 * i] * inv[i], b = o[c][4 * jj + 2 * i + 1] * inv[i];
          ss[i] += a * a + b * b;
        }
      ss[i] += __shfl_xor_sync(0xffffffffu, ss[i], 1);
      ss[i] += __shfl_xor_sync(0xffffffffu, ss[i], 2);
    }
  }
  if (rms_cluster) {
    // the slabs of this query tile are the CTAs of the cluster: publish, barrier, add up the peers' values
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const uint32_t slot = rowss + 4u * (64 * w + 16 * warp + lane / 4 + 8 * i);
      if (lane % 4 == 0) asm volatile("st.shared.f32 [%0], %1;" ::"r"(slot), "f"(ss[i]) : "memory");
    }
    cluster_sync_all();
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const uint32_t slot = rowss + 4u * (64 * w + 16 * warp + lane / 4 + 8 * i);
      float tot = 0.f;
      for (int r = 0; r < p.slabs; ++r) {
        float v;
        asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(v) : "r"(mapa(slot, r)) : "memory");
        tot += v;
      }
      ss[i] = tot;
    }
    cluster_sync_all();   // no CTA leaves while a peer may still read its statistics
  }
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    if (p.rms_g > 0.f) inv[i] *= rsqrtf(ss[i] / static_cast<float>(p.D) + 1e-5f) * p.rms_g;
    const int row = q0 + 64 * w + 16 * warp + lane / 4 + 8 * i;
    if (row >= p.N) continue;
    if (p.lse && slab == 0 && (lane % 4) == 0) p.lse[head + row] = (m[i] + __log2f(lsum[i])) * 0.6931471805599453f;
    __half* orow = p.o_ptr + (head + row) * p.D;
#pragma unroll
    for (int c = 0; c < NDC; ++c)
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        const int col = d0 + 64 * c + 8 * jj + 2 * (lane % 4);
        if (col < p.D)
          *reinterpret_cast<uint32_t*>(orow + col) =
              pack_half2(o[c][4 * jj + 2 * i] * inv[i], o[c][4 * jj + 2 * i + 1] * inv[i]);
      }
  }
}

}  // namespace attn
}  // namespace b200
