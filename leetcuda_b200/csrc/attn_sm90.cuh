// attn_sm90.cuh — FlashAttention-2 forward for sm_90a (H100): TMA + mbarrier + wgmma.
//
//   O = softmax(Q K^T * scale) V per (batch, head), fp16 in / out, fp32 scores, statistics and O.
//
// One CTA = kWG consumer warpgroups (64 query rows each) + one producer warpgroup (one thread
// issuing TMA; a whole warp for paged K/V).  Every CTA owns one query tile and one column slab of O (kDS columns); for
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
//
// Queries and keys have their own lengths Nq and Nk.  kCausal masks key j for query i when j > i + (Nk - Nq):
// the diagonal is aligned bottom-right as in FlashAttention-2, so the last Nq positions of a sequence attend to the
// Nk - Nq keys before them and to themselves.  This is NOT torch SDPA's is_causal when Nq != Nk (SDPA aligns the
// diagonal top-left).  With Nq > Nk the query rows i < Nq - Nk see no key: O = 0 and lse = -inf there.
//   * a CTA visits only the key blocks left of the diagonal of its last query row; both consumer warpgroups run all of
//     them (they share the K/V ring), so warpgroup 0 may see its last block fully masked;
//   * the per-element mask runs only in the blocks that cross the diagonal of the warpgroup's rows;
//   * query tiles are issued in reverse within a head, the longest ones first.
//
// Grouped-query attention and split-KV (b200_fmha_fwd_f16_gqa):
//   * Packing: query head h reads K/V head h / G.  The G query heads of one KV group are contiguous in Q [B,H,Nq,D],
//     so they form one [G*Nq, D] "head" of packed rows and grid.y walks the B*Hkv KV heads.  Without the mask that
//     is the plain kernel with G*Nq rows; with it (kGQA) packed row r has the query position r % Nq, which the
//     causal mask, the diagonal test and the block count use.  With Nq >= the tile rows, each query head gets tiles of
//     its own (tph per head, longest first across the G heads): the tiles and the work are those of the expanded
//     kernel and positions are row - g * Nq.  Shorter heads (decoding) are packed across head boundaries, so a tile
//     holds the rows of several heads.
//   * kSplit: grid.z cuts the key blocks [0, nkv) a CTA visits into contiguous ranges; the epilogue writes the
//     split's normalised O in fp32 and its lse to a workspace that a combine kernel reduces.
//
// Per-sequence lengths (attn_fwd_seqlens_kernel, b200_fmha_fwd_f16_seqlens): Q and K/V are padded to Nq and Nk, and
// sequence b has Lq_b <= Nq queries and Lk_b <= Nk keys, read from device arrays by every CTA before it starts.
//   * a CTA runs with Nk = Lk_b, diag = Lk_b - Lq_b and the key blocks of Lk_b; packed row r has position r % Nq (for
//     every G, causal or not) and is a padded row when that position is >= Lq_b; a causal tile visits the blocks left
//     of the diagonal of its greatest valid position, a tile of padded rows none;
//   * keys >= Lk_b are masked like the tail past Nk; V rows >= Lk_b of the one partial key block are zeroed in shared
//     memory (producer warp 1) before the consumers read them, since P = 0 times a NaN or Inf of V is NaN;
//   * padded rows and rows without a visible key store O = 0 and lse = -inf as literal values.
//
// Paged K/V (attn_fwd_paged_kernel, b200_fmha_fwd_f16_paged): K and V are pools [num_pages, page_size, Hkv, D] and
// sequence b's key t is row t % page_size of page table[b][t / page_size]; everything else is the per-sequence-length
// kernel with the padded Nk = max_pages * page_size.
//   * the K / V tensor maps are {D, Hkv, num_pages * page_size} with a box {64, 1, R}, R = min(page_size, kBN): a
//     {64 d, kBN keys} chunk is kBN / R sub-loads into one ring slot, sub-load i at slot + i * R * 128 bytes (a multiple
//     of 1024, so the 128B swizzle is that of one kBN-row box), all onto the slot's full barrier with the usual tx count;
//   * the producer is a whole warp: lane i holds the pool row of sub-load i of the next key block, read one block ahead
//     (the table load's latency hides behind the current block's issues) and broadcast to lane 0 with __shfl_sync;
//   * sub-loads past the sequence's last page, ceil(Lk_b / page_size) - 1, read that page again instead of the table:
//     their keys are masked and their V rows zeroed, since the partial key block's V rows past Lk_b come from real pages
//     (zeroed whenever Lk_b % kBN != 0, not only below the padded Nk);
//   * a page id is only a TMA coordinate: one outside [0, num_pages) reads zeros (wrong values, no out-of-bounds access).
//
// Packed variable-length sequences (attn_varlen_kernel, b200_fmha_fwd_{f16,bf16}_varlen[_paged]): token-major Q, O
// [total_q, H, D] and lse [H, total_q], sequence b at rows cu_q[b] ..; K/V [total_k, Hkv, D] at rows cu_k[b] .., or
// paged.  The per-sequence-length kernel with per-head tiles and token-major addresses (the end of this file); a tile
// past Lq_b exits before its first load, and only rows t < Lq_b inside [0, total_q) are stored.
#pragma once
#include <cuda.h>

#include <type_traits>

#include "softmax_math.cuh"

namespace b200 {
namespace attn {

struct Params {
  int Nq, Nk, D;       // Nq: rows of a head (kGQA: G * Nq packed rows of one KV group)
  int num_kv;          // key blocks of kBN keys over Nk
  int diag;            // Nk - Nq: with kCausal, key j is masked for query i when j > i + diag
  int nq;              // 64-column chunks of D (Q and K)
  int ring;            // K/V ring slots
  int slabs;           // column slabs of O per query tile
  float scale_log2;    // softmax scale * log2(e)
  float* lse;          // [B*H, Nq] natural-log LSE, or nullptr
  float rms_g;         // > 0: RMS-normalise every output row; with several slabs the CTAs of a query tile form
                       // a cluster and add up the row statistics through distributed shared memory
  __half* o_ptr;       // the output, of the kernel's element type (__half or __nv_bfloat16)
  float* ws_o;         // kSplit: [splits, B*H*Nq', D] fp32 normalised O of every split
  float* ws_lse;       //                          [splits, B*H*Nq'] natural-log LSE of every split
  int qpos;            // kGQA: query positions per head (the call's Nq); packed row r has position r % qpos
  int tph;             // kGQA: > 0: every query head has its own tph tiles (no tile straddles two heads), 0: the
                       // tiles cut the packed rows of the group
};

// attn_fwd_seqlens_kernel: the per-sequence lengths (int32 [B] on the device, or nullptr for Nq / Nk) and the K/V heads
// per sequence (grid.y = b * hkv + K/V head)
struct Lens {
  const int* q;
  const int* k;
  int hkv;
};

// attn_fwd_paged_kernel: the block table (int32 [B, max_pages] on the device) and the page size (a power of two >= 16)
struct Pages {
  const int* table;
  int page_size;
  int max_pages;
};

// attn_varlen_kernel: token-major Q / O [total_q, h, D] and lse [h, total_q]; sequence b is rows cu_q[b] .. cu_q[b+1]-1
// of them, and (packed K/V) rows cu_k[b] .. cu_k[b+1]-1 of K and V [total_k, hkv, D].  Paged K/V: k_used[b] keys.
struct Varlen {
  const int* cu_q;     // int32 [B + 1]
  const int* cu_k;     // packed K/V: int32 [B + 1]; paged K/V: seqused_k, int32 [B]
  int total_q;         // rows of Q and O
  int h;               // query heads
  int hkv;             // K/V heads (grid.y = b * hkv + K/V head)
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

// kVarlen: TMA row coordinate `first + t` of a sequence that starts at row `first` (device data): wraps instead of
// overflowing, and TMA reads zeros for any row outside the tensor
__device__ __forceinline__ int vrow(int first, int t) {
  return static_cast<int>(static_cast<unsigned>(first) + static_cast<unsigned>(t));
}

// one ring slot: a {64 columns, bn keys} chunk of K or V, or a {64 keys, ds columns} chunk of V^T
__host__ __device__ constexpr int slot_bytes(int bn, int ds, bool vt) { return 128 * (vt && ds > bn ? ds : bn); }
inline int smem_bytes(int kWG, int slot, int nq, int ring) {
  return kWG * nq * 8192 + ring * slot + 8 * (1 + 2 * ring) + kWG * 64 * 4 + 1024;
}

// Key blocks of kbn keys that a causal CTA whose query rows end before `rows_end` visits.  The producer and the
// consumers must agree on this count: every block the producer loads is released by every consumer warp.
__device__ __forceinline__ int causal_kv_blocks(const Params& p, int rows_end, int kbn) {
  const int keys = rows_end + p.diag;   // keys 0 .. keys - 1 are visible to the CTA's last row
  return keys <= 0 ? 0 : min(p.num_kv, (keys + kbn - 1) / kbn);
}

// The key blocks [x, y) of a CTA whose rows start at q0: with kCausal the blocks left of the diagonal of its greatest
// query position (kGQA: of a packed row), with kSplit the grid.z-th of gridDim.z contiguous ranges of them (possibly
// empty).  The producer and the consumers both take their loop bounds from here.
// kGQA: the CTA's rows [q0, row_end) are query positions from q0 - off on (per-head tiles), or packed rows (p.tph = 0).
// kSeqlens: p holds the sequence's Lk and diag, and only the positions below lq count; a tile without one visits no
// block.  A packed tile that crosses into the next query head holds position 0 and is taken to reach lq - 1.
template <int kBN, int kRows, bool kCausal, bool kGQA, bool kSplit, bool kSeqlens = false>
__device__ __forceinline__ int2 kv_blocks(const Params& p, int q0, int row_end, int off, int lq = 0) {
  int nkv = p.num_kv;
  if constexpr (kSeqlens) {
    int first, end;   // the tile's query positions [first, end)
    if (p.tph > 0) {
      first = q0 - off;
      end = min(q0 + kRows, row_end) - off;
    } else {
      const int last = min(q0 + kRows, p.Nq) - 1;
      const bool cross = last / p.qpos != q0 / p.qpos;
      first = cross ? 0 : q0 % p.qpos;
      end = cross ? p.qpos : last % p.qpos + 1;
    }
    end = min(end, lq);
    if (end <= first) nkv = 0;
    else if (kCausal) nkv = causal_kv_blocks(p, end, kBN);
  } else if constexpr (kCausal) {
    int rows_end = q0 + kRows;
    if constexpr (kGQA) {
      if (p.tph > 0) {
        rows_end = min(rows_end, row_end) - off;
      } else {
        // packed rows: a tile that crosses into the next query head (or ends the group) holds position Nq - 1
        const int last = min(rows_end, p.Nq) - 1;
        rows_end = last / p.qpos != q0 / p.qpos ? p.qpos : last % p.qpos + 1;
      }
    }
    nkv = causal_kv_blocks(p, rows_end, kBN);
  }
  if constexpr (kSplit) {
    const long long z = blockIdx.z, splits = gridDim.z;
    return make_int2(static_cast<int>(nkv * z / splits), static_cast<int>(nkv * (z + 1) / splits));
  }
  return make_int2(0, nkv);
}

// kDS: columns of O per CTA (64, 128 or 256); kBN: keys per block; kVT: V is [B,H,D,N]; kCausal: the causal mask;
// kGQA: the causal mask on packed query heads; kSplit: split-KV; kSeqlens: per-sequence lengths from `lens` (see the top
// of this file); kPaged: K and V in pages of a pool through `pages` (implies kSeqlens).  kCausal, kGQA, kSplit, kSeqlens
// and kPaged are template parameters so that the other kernels compile to the code they had without them.  T: the
// element type of Q, K, V and O, __half or __nv_bfloat16 (the top of this file; natural V only for bf16).
// kFP8: K and V are e4m3 bytes, staged by TMA and widened to T in shared memory by producer warps 1-3 (the end of
// this file); v_scale multiplies the normalised fp32 O before its rounding to T.
// kVarlen: token-major Q, O and lse through `vl`, K/V packed by cu_k or paged (the end of this file); implies kSeqlens
// and kGQA, per-head tiles (p.tph > 0) and no split.
template <int kDS, int kBN, int kWG, bool kVT, bool kCausal, bool kGQA, bool kSplit, bool kSeqlens, bool kPaged = false,
          typename T = __half, bool kFP8 = false, bool kVarlen = false>
__device__ __forceinline__ void attn_fwd_body(const CUtensorMap& tmap_q, const CUtensorMap& tmap_k,
                                              const CUtensorMap& tmap_v, Params p, const Lens& lens,
                                              const Pages& pages = Pages{}, float v_scale = 1.f,
                                              const Varlen& vl = Varlen{}) {
  static_assert(!kVT || kDS <= 128, "transposed V: one slab of <= 128 columns");
  static_assert(!kSeqlens || (!kVT && kGQA), "per-sequence lengths: natural V, query positions of packed rows");
  static_assert(!kPaged || kSeqlens, "paged K/V: per-sequence lengths");
  static_assert(!kFP8 || kSeqlens, "fp8 K/V: the per-sequence-length and paged kernels");
  static_assert(!kVarlen || (kSeqlens && !kSplit && !kFP8), "varlen: per-sequence lengths, no split, fp16 / bf16 K/V");
  constexpr bool kBF16 = std::is_same_v<T, __nv_bfloat16>;
  static_assert(kBF16 || std::is_same_v<T, __half>, "elements: fp16 or bf16");
  static_assert(!kBF16 || !kVT, "bf16: natural V");
  auto pack = [](float lo, float hi) {   // two fp32 values rounded to T (P, O)
    if constexpr (kBF16) return pack_bf162(lo, hi);
    else return pack_half2(lo, hi);
  };
  constexpr int SLOT = slot_bytes(kBN, kDS, kVT);
  constexpr int KV_BYTES = 64 * kBN * 2;   // one {64 columns, kBN keys} chunk of K or V
  constexpr int STG = kFP8 ? 64 * kBN : 0;   // kFP8: one staged e4m3 chunk {64 d, kBN keys}, 64-byte rows
  constexpr int NS = kBN / 2;     // S accumulator registers per thread
  constexpr int NDC = kDS / 64;   // 64-column chunks of the slab
  constexpr uint32_t kPolyMask = kDS <= 64 ? B200_ATTN_POLY_MASK_D64 : (kDS <= 128 ? B200_ATTN_POLY_MASK : 0u);
  static_assert((kPolyMask & 0x1111u) * 0xF == kPolyMask, "the FMA-pipe selection must take whole nibbles");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const uint32_t sq = smem_u32(smem);
  const uint32_t sring = sq + kWG * p.nq * 8192;
  const uint32_t sstg = sring + p.ring * SLOT;   // kFP8: the staging ring, one chunk per ring slot
  const uint32_t bars = sstg + p.ring * STG;
  const uint32_t qbar = bars;
  // per-row sum of squares (fused RMS norm over slabs)
  const uint32_t rowss = bars + 8u * (1 + (kFP8 ? 3 : 2) * p.ring);
  const bool rms_cluster = p.rms_g > 0.f && p.slabs > 1;
  auto full = [&](int s) { return bars + 8u * (1 + s); };
  auto empty = [&](int s) { return bars + 8u * (1 + p.ring + s); };
  [[maybe_unused]] auto staged = [&](int s) { return bars + 8u * (1 + 2 * p.ring + s); };   // kFP8: TMA landed

  const int wg = threadIdx.x / 128, tid = threadIdx.x % 128;
  // causal: the last query tile of a head has the most key blocks and starts first.  The head stays on grid.y, so the
  // resident CTAs still cover few heads and their K / V stays in L2.
  const int qtile = kCausal ? gridDim.x / p.slabs - 1 - blockIdx.x / p.slabs : blockIdx.x / p.slabs;
  int q0 = qtile * 64 * kWG;
  int row_end = p.Nq, off = 0;   // kGQA: the rows this CTA stores end before row_end; query position = row - off
  // kSeqlens: the CTA's sequence b and K/V head hk; kVarlen: its query head qh
  [[maybe_unused]] int b = 0, hk = 0, qh = 0;
  if constexpr (kSeqlens) {
    b = blockIdx.y / lens.hkv;
    hk = blockIdx.y % lens.hkv;
  }
  if constexpr (kVarlen) {
    // per-head tiles with or without the mask; causal: the longest first across the G heads, as below
    const int x = blockIdx.x / p.slabs, G = gridDim.x / p.slabs / p.tph;
    off = (x % G) * p.qpos;
    q0 = off + (kCausal ? p.tph - 1 - x / G : x / G) * 64 * kWG;
    row_end = off + p.qpos;
    qh = hk * G + x % G;
  } else if constexpr (kCausal && kGQA) {
    if (p.tph > 0) {
      // per-head tiles, the longest first across the G heads of the group, not only within one
      const int x = blockIdx.x / p.slabs, G = gridDim.x / p.slabs / p.tph;
      off = (x % G) * p.qpos;
      q0 = off + (p.tph - 1 - x / G) * 64 * kWG;
      row_end = off + p.qpos;
    }
  }
  const int slab = blockIdx.x % p.slabs;
  const int bh = blockIdx.y;
  const int d0 = slab * kDS;
  // kSeqlens: this sequence's valid query positions lq and keys p.Nk (nk_pad: the padded Nk of the K/V buffers)
  int lq = 0;
  [[maybe_unused]] const int nk_pad = p.Nk;
  // kVarlen: the sequence's first row of Q / O and (packed K/V) of K / V
  [[maybe_unused]] int qs = 0, ks = 0;
  if constexpr (kVarlen) {
    qs = __ldg(vl.cu_q + b);
    lq = static_cast<int>(min(max(static_cast<long long>(__ldg(vl.cu_q + b + 1)) - qs, 0ll),
                              static_cast<long long>(p.qpos)));
    long long lk;
    if constexpr (kPaged) {
      lk = __ldg(vl.cu_k + b);
    } else {
      ks = __ldg(vl.cu_k + b);
      lk = static_cast<long long>(__ldg(vl.cu_k + b + 1)) - ks;
    }
    p.Nk = static_cast<int>(min(max(lk, 0ll), static_cast<long long>(nk_pad)));
    p.diag = p.Nk - lq;
    p.num_kv = (p.Nk + kBN - 1) / kBN;
    // a tile of positions past the sequence: nothing to load, nothing to store (uniform over the CTA, no cluster)
    if (q0 - off >= lq) return;
  } else if constexpr (kSeqlens) {
    lq = lens.q ? min(max(__ldg(lens.q + b), 0), p.qpos) : p.qpos;
    const int lk = lens.k ? min(max(__ldg(lens.k + b), 0), nk_pad) : nk_pad;
    p.Nk = lk;
    p.diag = lk - lq;
    p.num_kv = (lk + kBN - 1) / kBN;
  }
  const int2 kv = kv_blocks<kBN, 64 * kWG, kCausal, kGQA, kSplit, kSeqlens>(p, q0, row_end, off, lq);
  // V chunks of this slab per key block
  const int nvc = kVT ? kBN / 64 : min(NDC, (p.D - d0 + 63) / 64);
  // kSeqlens: the visited key block that ends past Lk_b inside the K/V buffers (-1: none).  TMA zero-fills only past
  // nk_pad, so its V rows of keys >= Lk_b are zeroed in shared memory before the consumers read them.  kPaged: every
  // row of a sub-load comes from a page, so any partial key block is one.
  [[maybe_unused]] int vz = -1;
  [[maybe_unused]] const uint32_t vbar = rowss;   // its V chunks land here (no fused RMS norm with kSeqlens)
  // kFP8: the converters write those rows as zeros instead (vz stays -1)
  if constexpr (kSeqlens && !kFP8) {
    if (p.Nk % kBN != 0 && (kPaged || kVarlen || p.Nk < nk_pad) && p.num_kv - 1 >= kv.x && p.num_kv - 1 < kv.y)
      vz = p.num_kv - 1;
  }

  if (threadIdx.x == 0) {
    mbar_init(qbar, 1);
    for (int s = 0; s < p.ring; ++s) {
      mbar_init(full(s), kFP8 ? 3 : 1);   // kFP8: lane 0 of each converter warp
      mbar_init(empty(s), 4 * kWG);   // lane 0 of every consumer warp
      if constexpr (kFP8) mbar_init(staged(s), 1);
    }
    if constexpr (kSeqlens && !kFP8) mbar_init(vbar, 1);
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    if constexpr (kWG > 1) reg_dealloc<40>();
    if (kPaged ? tid < 32 : tid == 0) {
      // lane 0 issues every load.  kPaged: a chunk is nsub sub-loads of R rows, and lane i < nsub holds the pool row of
      // sub-load i of a key block (the top of this file)
      const int lane = tid, ps = kPaged ? pages.page_size : kBN, shift = __ffs(ps) - 1;
      const int R = min(ps, kBN), nsub = kBN / R;
      const int* table = pages.table + static_cast<size_t>(b) * pages.max_pages;
      const int last = ((p.Nk + ps - 1) >> shift) - 1;   // the sequence's last page (p.Nk >= 1 if a block is visited)
      auto pool_row = [&](int j) {
        const int t = j * kBN + min(lane, nsub - 1) * R;
        const unsigned page = static_cast<unsigned>(__ldg(table + min(t >> shift, last)));
        return static_cast<int>((page << shift) + static_cast<unsigned>(t & (ps - 1)));
      };
      if (lane == 0) {
        prefetch_tmap(&tmap_q);
        prefetch_tmap(&tmap_k);
        prefetch_tmap(&tmap_v);
        mbar_expect_tx(qbar, kWG * p.nq * 8192);
        for (int w = 0; w < kWG; ++w)
          for (int c = 0; c < p.nq; ++c) {
            if constexpr (kVarlen)
              tma_load_3d(sq + (w * p.nq + c) * 8192, &tmap_q, qbar, 64 * c, qh, vrow(qs, q0 - off + 64 * w),
                          kEvictFirst);
            else
              tma_load_3d(sq + (w * p.nq + c) * 8192, &tmap_q, qbar, 64 * c, q0 + 64 * w, bh, kEvictFirst);
          }
      }
      int it = 0;
      int row = kPaged && kv.x < kv.y ? pool_row(kv.x) : 0;
      for (int j = kv.x; j < kv.y; ++j) {
        const int cur = row;
        if (kPaged && j + 1 < kv.y) row = pool_row(j + 1);   // one block ahead
        // the block's K chunks, then its V chunks, one ring slot each.  The partial block's V (j == vz) lands on vbar,
        // not on the slots' full barriers: warp 1 arrives there once the rows past Lk_b are zero.
        for (int c = 0; c < p.nq + nvc; ++c, ++it) {
          const bool isv = c >= p.nq, zeroed = isv && j == vz;
          const int s = it % p.ring;
          // kFP8: into the staging slot s, onto staged(s) (rows of R * 64 bytes)
          const uint32_t bar = kFP8 ? staged(s) : (zeroed ? vbar : full(s));
          if (lane == 0) {
            if (it >= p.ring) mbar_wait(empty(s), ((it / p.ring) - 1) & 1);
            if (!zeroed) mbar_expect_tx(bar, kFP8 ? STG : (kVT && isv ? 64 * kDS * 2 : KV_BYTES));
            else if (c == p.nq) mbar_expect_tx(vbar, nvc * KV_BYTES);
          }
          const CUtensorMap* map = isv ? &tmap_v : &tmap_k;
          const int x = isv ? d0 + 64 * (c - p.nq) : 64 * c;
          for (int i = 0; i < nsub; ++i) {
            const int r = kPaged ? __shfl_sync(0xffffffffu, cur, i) : 0;
            if (lane != 0) continue;
            const uint32_t dst = kFP8 ? sstg + s * STG + i * R * 64 : sring + s * SLOT + i * R * 128;
            if constexpr (kPaged) tma_load_3d(dst, map, bar, x, hk, r, kEvictLast);
            else if constexpr (kVarlen) tma_load_3d(dst, map, bar, x, hk, vrow(ks, j * kBN), kEvictLast);
            else if (kVT && isv) tma_load_3d(dst, map, bar, j * kBN + 64 * (c - p.nq), d0, bh, kEvictLast);
            else tma_load_3d(dst, map, bar, x, j * kBN, bh, kEvictLast);
          }
        }
      }
    }
    if constexpr (kFP8) {
      if (tid >= 32) {
        // warps 1-3 widen every staged chunk of the producer's order into its ring slot: 16 e4m3 bytes of staged row r
        // (64 bytes per row) per thread and step, written as two 16-byte units of ring row r (128 bytes, 128B swizzle:
        // unit u of row r at u ^ (r % 8)).  V rows of keys >= Lk_b are written as zeros (NaN bytes there must not
        // reach P V); K rows past Lk_b are masked in the scores.
        const int ct = tid - 32;
        int it = 0;
        for (int j = kv.x; j < kv.y; ++j) {
          for (int c = 0; c < p.nq + nvc; ++c, ++it) {
            const int s = it % p.ring;
            const int rows = c >= p.nq ? min(kBN, p.Nk - j * kBN) : kBN;
            mbar_wait(staged(s), (it / p.ring) & 1);
            if (it >= p.ring) mbar_wait(empty(s), ((it / p.ring) - 1) & 1);
            const uint8_t* src = smem + (sstg - sq) + s * STG;
            uint8_t* out = smem + (sring - sq) + s * SLOT;
            for (int x = ct; x < kBN * 4; x += 96) {
              const int r = x >> 2, q = x & 3;
              uint4 lo = make_uint4(0u, 0u, 0u, 0u), hi = lo;
              if (r < rows) {
                const uint4 in = *reinterpret_cast<const uint4*>(src + 16 * x);
                const uint2 a = e4m3x4_to<T>(in.x), b = e4m3x4_to<T>(in.y), d = e4m3x4_to<T>(in.z),
                            e = e4m3x4_to<T>(in.w);
                lo = make_uint4(a.x, a.y, b.x, b.y);
                hi = make_uint4(d.x, d.y, e.x, e.y);
              }
              *reinterpret_cast<uint4*>(out + 128 * r + 16 * ((2 * q) ^ (r & 7))) = lo;
              *reinterpret_cast<uint4*>(out + 128 * r + 16 * ((2 * q + 1) ^ (r & 7))) = hi;
            }
            fence_proxy_async_smem();   // the consumers' wgmma reads the slot through the async proxy
            __syncwarp();
            if (tid % 32 == 0) mbar_arrive(full(s));
          }
        }
      }
    }
    if constexpr (kSeqlens && !kFP8) {
      if (tid / 32 == 1 && vz >= 0) {
        // a natural-V chunk {64 d, kBN keys} holds key r in the 128-byte row r (the 128B swizzle permutes 16-byte units
        // within a row only): zero rows Lk_b - vz * kBN .. kBN - 1 of the block's V chunks, then publish them
        const int it0 = (vz - kv.x) * (p.nq + nvc) + p.nq;   // the producer's slot count at the block's first V chunk
        const int zb = (p.Nk - vz * kBN) * 128;
        mbar_wait(vbar, 0);
        for (int c = 0; c < nvc; ++c) {
          uint8_t* chunk = smem + (sring - sq) + ((it0 + c) % p.ring) * SLOT;
          for (int x = zb + 16 * (tid % 32); x < kBN * 128; x += 512)
            *reinterpret_cast<uint4*>(chunk + x) = make_uint4(0u, 0u, 0u, 0u);
        }
        fence_proxy_async_smem();   // the consumers' wgmma reads V through the async proxy
        __syncwarp();
        if (tid % 32 == 0)
          for (int c = 0; c < nvc; ++c) mbar_arrive(full((it0 + c) % p.ring));
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
  mbar_wait(qbar, 0);

  int it = 0;
  auto release = [&](int i) {
    if (lane == 0) mbar_arrive(empty(i % p.ring));
  };
  const int r0 = q0 + 64 * w;   // first query row of this warpgroup
  // kGQA: query positions of packed rows for the mask: the least one of the warpgroup's rows, and those of this
  // thread's two rows (without kGQA a row's position is the row)
  int pos0 = 0, pos[2] = {0, 0};
  if constexpr (kCausal && kGQA) {
    if (p.tph > 0) {
      pos0 = r0 - off;
      pos[0] = r0 + 16 * warp + lane / 4 - off;
      pos[1] = pos[0] + 8;
    } else {
      pos0 = min(r0 + 63, p.Nq - 1) / p.qpos != r0 / p.qpos ? 0 : r0 % p.qpos;
      pos[0] = (r0 + 16 * warp + lane / 4) % p.qpos;
      pos[1] = (r0 + 16 * warp + lane / 4 + 8) % p.qpos;
    }
  }
  for (int j = kv.x; j < kv.y; ++j) {
    // ---- S = Q K^T over the d-chunks
    float s[NS];
    wg_fence();
    for (int c = 0; c < p.nq; ++c, ++it) {
      mbar_wait(full(it % p.ring), (it / p.ring) & 1);
      const uint32_t qa = sq + (w * p.nq + c) * 8192, ka = sring + (it % p.ring) * SLOT;
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        const uint64_t da = wg_desc(qa + ks * 32, 16), db = wg_desc(ka + ks * 32, 16);
        const uint32_t go = (c > 0 || ks > 0) ? 1u : 0u;
        if constexpr (kBF16 && kBN == 128) wgmma_ss_m64n128k16_f32_bf16<0, 0>(s, da, db, go);
        else if constexpr (kBF16) wgmma_ss_m64n64k16_f32_bf16<0, 0>(s, da, db, go);
        else if constexpr (kBN == 128) wgmma_ss_m64n128k16_f32_f16<0, 0>(s, da, db, go);
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
    if (j * kBN + kBN > p.Nk) {
#pragma unroll
      for (int jj = 0; jj < kBN / 8; ++jj)
#pragma unroll
        for (int e = 0; e < 2; ++e)
          if (kbase + 8 * jj + e >= p.Nk) {
            s[4 * jj + e] = -INFINITY;
            s[4 * jj + 2 + e] = -INFINITY;
          }
    }
    if (kCausal && j * kBN + kBN - 1 > (kGQA ? pos0 : r0) + p.diag) {   // the block crosses the diagonal of this
#pragma unroll                                                          // warpgroup's rows
      for (int i = 0; i < 2; ++i) {
        // last visible key, from kbase
        const int last = (kGQA ? pos[i] : r0 + 16 * warp + lane / 4 + 8 * i) + p.diag - kbase;
#pragma unroll
        for (int jj = 0; jj < kBN / 8; ++jj)
#pragma unroll
          for (int e = 0; e < 2; ++e)
            if (8 * jj + e > last) s[4 * jj + 2 * i + e] = -INFINITY;
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
      // a row without a visible key so far (causal or per-sequence lengths only): subtract 0, so that alpha and x are
      // exp2(-inf), not NaN
      const float mb = (kCausal || kSeqlens) && mn == -INFINITY ? 0.f : mn;
      alpha[i] = fast_exp2(m[i] - mb);
      m[i] = mn;
      float sum = 0.f;
#pragma unroll
      for (int jj = 0; jj < kBN / 8; ++jj)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float x = fmaf(s[4 * jj + 2 * i + e], p.scale_log2, -mb);
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
    // P (rounded to T) as the A fragments of the k16 steps over the keys of this block
    uint32_t pa[kBN / 16][4];
#pragma unroll
    for (int kk = 0; kk < kBN / 16; ++kk) {
      pa[kk][0] = pack(s[8 * kk + 0], s[8 * kk + 1]);
      pa[kk][1] = pack(s[8 * kk + 2], s[8 * kk + 3]);
      pa[kk][2] = pack(s[8 * kk + 4], s[8 * kk + 5]);
      pa[kk][3] = pack(s[8 * kk + 6], s[8 * kk + 7]);
    }

    // ---- O += P V over the slab's V chunks
    wg_fence();
#pragma unroll
    for (int c = 0; c < (kVT ? kBN / 64 : NDC); ++c) {
      if (c >= nvc) break;
      mbar_wait(full(it % p.ring), (it / p.ring) & 1);
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
        for (int kk = 0; kk < kBN / 16; ++kk) {
          if constexpr (kBF16) wgmma_rs_m64n64k16_f32_bf16<1>(o[c], pa[kk], wg_desc(va + kk * 2048, 8192), 1u);
          else wgmma_rs_m64n64k16_f32_f16<1>(o[c], pa[kk], wg_desc(va + kk * 2048, 8192), 1u);
        }
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
  // kFP8: the normalised fp32 O times v_scale, then rounded once (kSplit: written to the workspace)
  auto vs = [&](float x) {
    if constexpr (kFP8) return x * v_scale;
    else return x;
  };
  const size_t head = static_cast<size_t>(bh) * p.Nq;
  float inv[2], lsum[2], ss[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    float lt = l[i];
    lt += __shfl_xor_sync(0xffffffffu, lt, 1);
    lt += __shfl_xor_sync(0xffffffffu, lt, 2);
    lsum[i] = lt;
    // an empty row (or a split that visited no block) is told by m, not by l: exp2_fma_pipe(-inf) = 2^-126 leaves l
    // slightly above 0
    inv[i] = (kCausal || kSplit || kSeqlens) && m[i] == -INFINITY ? 0.f : 1.f / lt;
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
  // One store per row of this thread.  kSplit: the split's normalised O in fp32 and its lse go to the workspace that
  // attn_combine_kernel reduces.  kVarlen: token-major O row cu_q[b] + t of head qh and lse [h, total_q]; only
  // positions t < Lq_b of rows inside [0, total_q) are stored (the rows past them belong to the next sequence or to
  // none).  A padded row (kSeqlens) stores O = 0 and lse = -inf, and so does a row without a visible key except in a
  // split's part; the zeros are selected, not computed, since o * inv may be NaN in a padded row.
  const size_t part = kSplit ? static_cast<size_t>(blockIdx.z) * gridDim.y * p.Nq : 0;
  float* const lse = kSplit ? p.ws_lse : p.lse;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    if (!kSplit && !kVarlen && p.rms_g > 0.f) inv[i] *= rsqrtf(ss[i] / static_cast<float>(p.D) + 1e-5f) * p.rms_g;
    const int row = q0 + 64 * w + 16 * warp + lane / 4 + 8 * i;
    const long long grow = static_cast<long long>(qs) + (row - off);   // kVarlen: the row of Q and O
    const bool pad = kSeqlens && (kVarlen || p.tph > 0 ? row - off : row % p.qpos) >= lq;
    if (kVarlen ? pad || grow < 0 || grow >= vl.total_q : row >= row_end) continue;
    const bool none = (kCausal || kSplit || kSeqlens) && m[i] == -INFINITY;
    const bool zero = pad || (kSeqlens && !kSplit && none);
    const size_t at = kVarlen ? static_cast<size_t>(grow) * vl.h + qh : part + head + row;   // the row of O
    if ((kSplit || lse) && slab == 0 && (lane % 4) == 0)
      lse[kVarlen ? static_cast<size_t>(qh) * vl.total_q + grow : at] =
          pad || none ? -INFINITY : (m[i] + __log2f(lsum[i])) * 0.6931471805599453f;
#pragma unroll
    for (int c = 0; c < NDC; ++c)
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        const int col = d0 + 64 * c + 8 * jj + 2 * (lane % 4);
        if (col >= p.D) continue;
        const float x = zero ? 0.f : vs(o[c][4 * jj + 2 * i] * inv[i]);
        const float y = zero ? 0.f : vs(o[c][4 * jj + 2 * i + 1] * inv[i]);
        if constexpr (kSplit) *reinterpret_cast<float2*>(p.ws_o + at * p.D + col) = make_float2(x, y);
        else *reinterpret_cast<uint32_t*>(reinterpret_cast<T*>(p.o_ptr) + at * p.D + col) = pack(x, y);
      }
  }
}

template <int kDS, int kBN, int kWG, bool kVT, bool kCausal, bool kGQA = false, bool kSplit = false>
__global__ void __launch_bounds__(threads<kWG>(), 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                const __grid_constant__ CUtensorMap tmap_v, const Params p) {
  attn_fwd_body<kDS, kBN, kWG, kVT, kCausal, kGQA, kSplit, false>(tmap_q, tmap_k, tmap_v, p, Lens{});
}

// Per-sequence lengths (b200_fmha_fwd_f16_seqlens): natural V, query positions of packed rows for every G.
template <int kDS, int kBN, int kWG, bool kCausal, bool kSplit>
__global__ void __launch_bounds__(threads<kWG>(), 1)
attn_fwd_seqlens_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                        const __grid_constant__ CUtensorMap tmap_v, const Params p, const Lens lens) {
  attn_fwd_body<kDS, kBN, kWG, false, kCausal, true, kSplit, true>(tmap_q, tmap_k, tmap_v, p, lens);
}

// Paged K/V (b200_fmha_fwd_f16_paged): the per-sequence-length kernel reading K and V through a block table.
template <int kDS, int kBN, int kWG, bool kCausal, bool kSplit>
__global__ void __launch_bounds__(threads<kWG>(), 1)
attn_fwd_paged_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                      const __grid_constant__ CUtensorMap tmap_v, const Params p, const Lens lens, const Pages pages) {
  attn_fwd_body<kDS, kBN, kWG, false, kCausal, true, kSplit, true, true>(tmap_q, tmap_k, tmap_v, p, lens, pages);
}

// bf16 Q, K, V and O (b200_fmha_fwd_bf16_seqlens, b200_fmha_fwd_bf16_paged): the two kernels above with bf16 elements.
// A dense bf16 call runs attn_fwd_seqlens_bf16_kernel with null length arrays.  Instantiated in attn_bf16.cu.
template <int kDS, int kBN, int kWG, bool kCausal, bool kSplit>
__global__ void __launch_bounds__(threads<kWG>(), 1)
attn_fwd_seqlens_bf16_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                             const __grid_constant__ CUtensorMap tmap_v, const Params p, const Lens lens) {
  attn_fwd_body<kDS, kBN, kWG, false, kCausal, true, kSplit, true, false, __nv_bfloat16>(tmap_q, tmap_k, tmap_v, p,
                                                                                         lens);
}

template <int kDS, int kBN, int kWG, bool kCausal, bool kSplit>
__global__ void __launch_bounds__(threads<kWG>(), 1)
attn_fwd_paged_bf16_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                           const __grid_constant__ CUtensorMap tmap_v, const Params p, const Lens lens,
                           const Pages pages) {
  attn_fwd_body<kDS, kBN, kWG, false, kCausal, true, kSplit, true, true, __nv_bfloat16>(tmap_q, tmap_k, tmap_v, p, lens,
                                                                                        pages);
}

// fp8 (e4m3) K and V with T = __half or __nv_bfloat16 Q and O (b200_fmha_fwd_{f16,bf16}_fp8kv_{seqlens,paged}): the two
// kernels above, with K and V staged as e4m3 and widened exactly to T in shared memory.  The softmax scale arrives
// with k_scale folded in; v_scale multiplies the normalised O.  Instantiated in attn_fp8kv_f16.cu / attn_fp8kv_bf16.cu.
//   * the producer's lane 0 issues TMA loads of e4m3 chunks {64 d, kBN keys} (64-byte rows, no swizzle; paged: kBN / R
//     sub-loads of R rows) into a staging ring of one chunk per ring slot, onto that chunk's `staged` barrier;
//   * warps 1-3 of the producer warpgroup wait for the staged chunk and for the ring slot's `empty` barrier, widen
//     the chunk with cvt.rn.f16x2.e4m3x2 (bf16: through fp32, also exact) into the 128B-swizzled layout the consumers
//     read, fence the async proxy and arrive on the slot's `full` barrier (three arrivals);
//   * the staging slot is free again once the ring slot is (its converters read it before publishing the slot), so
//     the producer's wait on `empty` covers both;
//   * V rows of keys >= Lk_b in the partial key block are written as zeros by the converters, which replaces warp 1's
//     zeroing of the fp16 / bf16 kernels.
template <int kDS, int kBN, int kWG, bool kCausal, bool kSplit, typename T>
__global__ void __launch_bounds__(threads<kWG>(), 1)
attn_fwd_fp8kv_seqlens_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                              const __grid_constant__ CUtensorMap tmap_v, const Params p, const Lens lens,
                              const float v_scale) {
  attn_fwd_body<kDS, kBN, kWG, false, kCausal, true, kSplit, true, false, T, true>(tmap_q, tmap_k, tmap_v, p, lens,
                                                                                  Pages{}, v_scale);
}

template <int kDS, int kBN, int kWG, bool kCausal, bool kSplit, typename T>
__global__ void __launch_bounds__(threads<kWG>(), 1)
attn_fwd_fp8kv_paged_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                            const __grid_constant__ CUtensorMap tmap_v, const Params p, const Lens lens,
                            const Pages pages, const float v_scale) {
  attn_fwd_body<kDS, kBN, kWG, false, kCausal, true, kSplit, true, true, T, true>(tmap_q, tmap_k, tmap_v, p, lens,
                                                                                 pages, v_scale);
}

// Packed variable-length sequences (b200_fmha_fwd_{f16,bf16}_varlen, _varlen_paged): token-major Q and O
// [total_q, H, D], lse [H, total_q], sequence b at rows cu_q[b] ..; K/V [total_k, Hkv, D] at rows cu_k[b] .. (kPagedKV
// false) or paged pools read through the block table (kPagedKV true, lengths seqused_k).  The per-sequence-length
// kernel in every other respect, with p.qpos = max_seqlen_q and p.Nk = max_seqlen_k (paged: max_pages * page_size).
//   * grid (G * tph * slabs, B * Hkv): per-head tiles whatever the mask (tph = ceil(max_seqlen_q / (64 kWG))), causal
//     the longest first; a tile whose first position is >= Lq_b returns before it initialises a barrier;
//   * Q: a {D, H, total_q} tensor map, box {64, 1, 64}: chunk c of warpgroup w at (64 c, head, cu_q[b] + t0 + 64 w);
//     packed K/V: {D, Hkv, total_k}, box {64, 1, kBN}: key block j at row cu_k[b] + j kBN (rows of the next sequence
//     in the partial block are masked in S and zeroed in V, as under kPaged);
//   * the epilogue stores only positions t < Lq_b of rows cu_q[b] + t inside [0, total_q), indexed in size_t.
// T in the template arguments carries the element type (the kernel's name has no "bf16" in it).  Instantiated in
// attn_varlen.cu.
template <int kDS, int kBN, int kWG, bool kCausal, bool kPagedKV, typename T>
__global__ void __launch_bounds__(threads<kWG>(), 1)
attn_varlen_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                   const __grid_constant__ CUtensorMap tmap_v, const Params p, const Varlen vl, const Pages pages) {
  attn_fwd_body<kDS, kBN, kWG, false, kCausal, true, false, true, kPagedKV, T, false, true>(
      tmap_q, tmap_k, tmap_v, p, Lens{nullptr, nullptr, vl.hkv}, pages, 1.f, vl);
}

}  // namespace attn
}  // namespace b200
