// attn_capi.cu — C-ABI entry points of the attention path (include/leetcuda_b200.h).
#include <math.h>
#include <float.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>

#include <type_traits>

#include <cuda_fp8.h>

#include "attn_launch.cuh"

namespace {

using namespace b200;
using b200::host::fail;

// Split-KV: the most splits b200_fmha_fwd_f16_gqa accepts (B200_FMHA_MAX_SPLITS); for num_splits = 0 the fewest key
// blocks a split keeps, and the fewest key blocks of a CTA worth splitting at all.  Measured on an H100 80GB HBM3
// (400 W, 1980 MHz), D = 128, one CTA (B1 H8 Hkv1 and B1 H32 Hkv4, Nq = 1), fixed split counts timed alternately:
// at 8 key blocks (Nk = 512) every split was slower than none (0.024 ms unsplit, >= 0.029 ms split: the combine launch
// and the workspace cost more than they save); from 16 blocks on, splits of about 4 blocks were as fast as the best
// count or within its spread (Nk = 2048: 8 splits 0.039 .. 0.046 ms, 4 splits 0.046, unsplit 0.072 ms).
constexpr int kMaxSplits = 64;
constexpr int kMinBlocksPerSplit = 4;
constexpr int kMinBlocksToSplit = 16;

// The fp16 kernel of family F.  lens != nullptr: per-sequence lengths, attn_fwd_seqlens_kernel (natural V only); with
// pages also: paged K/V, attn_fwd_paged_kernel
template <typename F, bool kVT>
int launch_attn(const attn::Launch& l, bool causal, bool packed, const attn::Lens* lens, const attn::Pages* pages) {
  constexpr int kDS = F::kDS, kBN = F::kBN, kWG = F::kWG;
  return attn::with_flags(causal, l.splits > 1, [&](auto c, auto s) {
    if constexpr (!kVT) {
      if (lens != nullptr && pages != nullptr)
        return attn::launch<attn::attn_fwd_paged_kernel<kDS, kBN, kWG, c, s>, kWG>(l, *lens, *pages);
      if (lens != nullptr) return attn::launch<attn::attn_fwd_seqlens_kernel<kDS, kBN, kWG, c, s>, kWG>(l, *lens);
    }
    // packed query heads need the kGQA kernels only for the mask; a split always runs a kSplit kernel
    if constexpr (c && !s) {
      if (packed) return attn::launch<attn::attn_fwd_kernel<kDS, kBN, kWG, kVT, true, true>, kWG>(l);
    }
    return attn::launch<attn::attn_fwd_kernel<kDS, kBN, kWG, kVT, c, c && s, s>, kWG>(l);
  });
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

// out[r, :] = sum_s w_s o_s[r, :] / sum_s w_s,  w_s = exp(lse_s[r] - max_s lse_s[r]),  out_lse[r] = ln sum_s w_s + max
// over the fp32 parts the split kernel wrote (ws_o [splits, rows, D], ws_lse [splits, rows]), rounded once to T.  A
// row whose parts are all empty (lse -inf) gets 0 and -inf: the max is clamped to -FLT_MAX, every weight is 0, and the
// divisor is clamped to 1 (otherwise one weight is expf(0) = 1, so the clamp changes nothing).
// HBM-bound: one thread per 16-byte pack of the output (8 elements), 32 bytes and one lse read per split.  T: __half or
// __nv_bfloat16.
template <typename Idx, typename T = __half>
__global__ void __launch_bounds__(256)
attn_combine_kernel(T* __restrict__ out, float* __restrict__ out_lse, const float* __restrict__ ws_o,
                    const float* __restrict__ ws_lse, unsigned rows, unsigned packs_per_row, int splits) {
  auto pack = [](float lo, float hi) {
    if constexpr (std::is_same_v<T, __nv_bfloat16>) return pack_bf162(lo, hi);
    else return pack_half2(lo, hi);
  };
  const Idx n_packs = static_cast<Idx>(rows) * packs_per_row;
  const Idx pk = static_cast<Idx>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (pk >= n_packs) return;
  const Idx row = pk / packs_per_row;
  const size_t part = static_cast<size_t>(n_packs) * 8;   // floats of one split's O
  const float* src = ws_o + static_cast<size_t>(pk) * 8;
  float top = -FLT_MAX;
  for (int s = 0; s < splits; ++s) top = fmaxf(top, __ldg(ws_lse + static_cast<size_t>(s) * rows + row));
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  float denom = 0.f;
  for (int s = 0; s < splits; ++s) {
    const uint4 a = ld_stream(src + s * part), b = ld_stream(src + s * part + 4);
    const float w = expf(__ldg(ws_lse + static_cast<size_t>(s) * rows + row) - top);
    const float x[8] = {__uint_as_float(a.x), __uint_as_float(a.y), __uint_as_float(a.z), __uint_as_float(a.w),
                        __uint_as_float(b.x), __uint_as_float(b.y), __uint_as_float(b.z), __uint_as_float(b.w)};
    denom += w;
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] = fmaf(w, x[e], acc[e]);
  }
  const float inv = 1.f / fmaxf(denom, 1.f);
  uint4 r;
  r.x = pack(acc[0] * inv, acc[1] * inv);
  r.y = pack(acc[2] * inv, acc[3] * inv);
  r.z = pack(acc[4] * inv, acc[5] * inv);
  r.w = pack(acc[6] * inv, acc[7] * inv);
  st_stream(reinterpret_cast<uint4*>(out) + pk, r);
  if (out_lse != nullptr && pk == row * packs_per_row) out_lse[row] = logf(denom) + top;   // first pack of the row
}

template <typename T>
int launch_combine(T* out, float* out_lse, const float* ws_o, const float* ws_lse, size_t rows, int D, int splits,
                   cudaStream_t stream) {
  const unsigned ppr = static_cast<unsigned>(D / 8);
  const size_t total = rows * ppr;
  const size_t blocks = (total + 255) / 256;
  if (rows > 0xFFFFFFFFull || blocks > 0x7FFFFFFFull) return fail(B200_EINVAL, "fmha_gqa: too many output rows");
  const unsigned g = static_cast<unsigned>(blocks), nr = static_cast<unsigned>(rows);
  if (total + 256 < 0xFFFFFFFFull)
    attn_combine_kernel<unsigned, T><<<g, 256, 0, stream>>>(out, out_lse, ws_o, ws_lse, nr, ppr, splits);
  else
    attn_combine_kernel<size_t, T><<<g, 256, 0, stream>>>(out, out_lse, ws_o, ws_lse, nr, ppr, splits);
  B200_CUDA_OK(cudaGetLastError());
  host::count_launch();
  return 0;
}

// The family of head dim D (attn::with_family) at run time
struct Family {
  int ds, bn, wgs;
};
Family family(int D) {
  return attn::with_family(D, [](auto f) {
    using F = decltype(f);
    return Family{F::kDS, F::kBN, F::kWG};
  });
}

// The K/V ring of family f next to Q (nq 64-column chunks per tile row): every slot that fits, at most 16 (two key
// blocks of K and V chunks at D = 512).  stage: the bytes each slot adds beside it (fp8: its staging chunk and
// barrier).  Returns the dynamic shared memory with *ring slots, or 0 when fewer than two fit.
int ring_smem(const Family& f, int nq, bool vt, int stage, int* ring) {
  const int kMaxSmem = 227 * 1024;
  const int slot = attn::slot_bytes(f.bn, f.ds, vt);
  const int fixed = attn::smem_bytes(f.wgs, slot, nq, 0);
  *ring = (kMaxSmem - fixed) / (slot + 16 + stage);
  if (*ring > 16) *ring = 16;
  if (*ring < 2) return 0;
  return attn::smem_bytes(f.wgs, slot, nq, *ring) + *ring * stage;
}

// *p for G * Nq packed rows per K/V head (Nq query positions per head) against Nk keys on the family of D, without a
// split workspace and with p->tph = 0, and its K/V ring (ring_smem).  Returns the dynamic shared memory, or 0 when
// the ring does not fit.
int attn_params(attn::Params* p, int G, int Nq, int Nk, int D, float scale, float* lse, float rms_g, void* o, bool vt,
                int stage) {
  const Family f = family(D);
  p->Nq = G * Nq;
  p->qpos = Nq;
  p->Nk = Nk;
  p->D = D;
  p->nq = (D + 63) / 64;
  p->num_kv = (Nk + f.bn - 1) / f.bn;
  p->diag = Nk - Nq;
  p->slabs = (D + f.ds - 1) / f.ds;
  p->scale_log2 = scale * 1.4426950408889634f;
  p->lse = lse;
  p->rms_g = rms_g;
  p->o_ptr = static_cast<__half*>(o);
  p->ws_o = nullptr;
  p->ws_lse = nullptr;
  p->tph = 0;
  return ring_smem(f, p->nq, vt, stage, &p->ring);
}

// A tensor map over `rows` rows of `heads` heads of D elements (row-major [rows, heads, D]): dims {D, heads, rows},
// boxes of {64, 1, box_rows}, 128B-swizzled unless given.  The paged pools [num_pages * page_size, Hkv, D] and the
// token-major varlen Q [total_q, H, D] and K / V [total_k, Hkv, D].
int rows_map(CUtensorMap* m, const void* base, int D, int heads, uint64_t rows, int box_rows, uint64_t elem_bytes,
             CUtensorMapDataType dt, CUtensorMapSwizzle sw = CU_TENSOR_MAP_SWIZZLE_128B) {
  uint64_t dims[3] = {static_cast<uint64_t>(D), static_cast<uint64_t>(heads), rows};
  uint64_t str[2] = {static_cast<uint64_t>(D) * elem_bytes, static_cast<uint64_t>(heads) * D * elem_bytes};
  uint32_t box[3] = {64, 1, static_cast<uint32_t>(box_rows)};
  return host::get_tmap(m, base, 3, dims, str, box, sw, dt);
}

// G: query heads per K/V head (H = G * Hkv; the kernel sees B * Hkv heads of G * Nq packed rows).  splits > 1: grid.z
// splits whose fp32 parts go to ws_o / ws_lse instead of o / lse (kSplit kernels).  Causal with G > 1 runs kGQA.
// pages: k and v are pools of num_pages pages [page_size, Hkv, D], and Nk is the padded max_pages * page_size.
// T: the element type of q and o, KV that of k and v: T (__nv_bfloat16 runs the bf16 kernels, attn_bf16.cu) or
// __nv_fp8_e4m3 (the fp8-K/V kernels, attn_fp8kv_*.cu, with v_scale); both take lens always.
template <typename T, typename KV = T>
int fmha_dispatch(const void* q, const void* k, const void* v, void* o, float* lse, float rms_g, int B, int Hkv, int G,
                  int Nq, int Nk, int D, bool vt, bool causal, float scale, int splits, float* ws_o, float* ws_lse,
                  cudaStream_t stream, const attn::Lens* lens = nullptr, const attn::Pages* pages = nullptr,
                  int num_pages = 0, float v_scale = 1.f) {
  constexpr bool fp8 = std::is_same_v<KV, __nv_fp8_e4m3>;
  static_assert(fp8 || std::is_same_v<KV, T>, "K/V: the element type of Q and O, or e4m3");
  const uint64_t BH = static_cast<uint64_t>(B) * Hkv;
  const Family f = family(D);
  const int ds = f.ds, bn = f.bn, wgs = f.wgs;
  const int rows = G * Nq;   // packed rows per K/V head
  if (rms_g > 0.f && D > 256 && !(D <= 512 && D % 128 == 0))
    return fail(B200_ENOTSUP, "fused rms_norm: D=%d (supported: D <= 256, 384, 512)", D);
  attn::Params p;
  // fp8: every ring slot has a staging chunk of e4m3 bytes and its barrier beside it (attn_sm90.cuh)
  const int smem = attn_params(&p, G, Nq, Nk, D, scale, lse, rms_g, o, vt, fp8 ? 64 * bn + 8 : 0);
  if (smem == 0) return fail(B200_ENOTSUP, "headdim not support! (D=%d)", D);
  p.ws_o = splits > 1 ? ws_o : nullptr;
  p.ws_lse = splits > 1 ? ws_lse : nullptr;
  // causal packed heads of at least one tile of rows: tiles of their own per head (attn_sm90.cuh), else packed tiles
  p.tph = causal && Nq >= 64 * wgs ? (Nq + 64 * wgs - 1) / (64 * wgs) : 0;
  const int qtiles = p.tph > 0 ? G * p.tph : (rows + 64 * wgs - 1) / (64 * wgs);

  constexpr bool bf16 = std::is_same_v<T, __nv_bfloat16>;
  const CUtensorMapDataType dt = bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  // fp8: K and V rows of D bytes, staged unswizzled (the converters write the 128B-swizzled T rows)
  const CUtensorMapDataType kvdt = fp8 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : dt;
  const CUtensorMapSwizzle kvsw = fp8 ? CU_TENSOR_MAP_SWIZZLE_NONE : CU_TENSOR_MAP_SWIZZLE_128B;
  const uint64_t kveb = sizeof(KV);
  CUtensorMap tq, tk, tv;
  uint64_t qdims[3] = {static_cast<uint64_t>(D), static_cast<uint64_t>(rows), BH};
  uint64_t qstr[2] = {static_cast<uint64_t>(D) * 2, static_cast<uint64_t>(rows) * D * 2};
  uint64_t kdims[3] = {static_cast<uint64_t>(D), static_cast<uint64_t>(Nk), BH};
  uint64_t kstr[2] = {static_cast<uint64_t>(D) * kveb, static_cast<uint64_t>(Nk) * D * kveb};
  uint32_t qbox[3] = {64, 64, 1};
  uint32_t kbox[3] = {64, static_cast<uint32_t>(bn), 1};
  int rc;
  if ((rc = host::get_tmap(&tq, q, 3, qdims, qstr, qbox, CU_TENSOR_MAP_SWIZZLE_128B, dt))) return rc;
  if (pages) {
    // pool rows {D, Hkv, num_pages * page_size}; a key block is kBN / R boxes of R = min(page_size, kBN) rows
    const uint64_t prows = static_cast<uint64_t>(num_pages) * static_cast<uint64_t>(pages->page_size);
    const int R = std::min(pages->page_size, bn);
    if ((rc = rows_map(&tk, k, D, Hkv, prows, R, kveb, kvdt, kvsw))) return rc;
    if ((rc = rows_map(&tv, v, D, Hkv, prows, R, kveb, kvdt, kvsw))) return rc;
  } else {
    if ((rc = host::get_tmap(&tk, k, 3, kdims, kstr, kbox, kvsw, kvdt))) return rc;
    if (vt) {
      uint64_t vd[3] = {static_cast<uint64_t>(Nk), static_cast<uint64_t>(D), BH};
      uint64_t vs[2] = {static_cast<uint64_t>(Nk) * 2, static_cast<uint64_t>(Nk) * D * 2};
      uint32_t vb[3] = {64, static_cast<uint32_t>(ds), 1};
      if ((rc = host::get_tmap(&tv, v, 3, vd, vs, vb, CU_TENSOR_MAP_SWIZZLE_128B, dt))) return rc;
    } else {
      if ((rc = host::get_tmap(&tv, v, 3, kdims, kstr, kbox, kvsw, kvdt))) return rc;
    }
  }
  if (vt && lens) return fail(B200_EINVAL, "fmha: internal dispatch error (transposed V with lengths)");
  const attn::Launch l{tq, tk, tv, p, qtiles, static_cast<int>(BH), splits, smem, stream};
  if constexpr (fp8) {
    if (vt || !lens) return fail(B200_EINVAL, "fmha: internal dispatch error (fp8 K/V without lengths or with V^T)");
    return attn::launch_attn_fp8kv<T>(l, causal, *lens, pages, v_scale);
  } else if constexpr (bf16) {
    if (vt || !lens) return fail(B200_EINVAL, "fmha: internal dispatch error (bf16 without lengths or with V^T)");
    return attn::launch_attn_bf16(l, causal, *lens, pages);
  } else {
    return attn::with_family(D, [&](auto fam) {
      using F = decltype(fam);
      if (!vt) return launch_attn<F, false>(l, causal, G > 1, lens, pages);
      if constexpr (F::kDS == 256)
        return fail(B200_EINVAL, "fmha: internal dispatch error (transposed V with D=%d)", D);
      else
        return launch_attn<F, true>(l, causal, G > 1, lens, pages);
    });
  }
}

// The attention kernel, and with splits > 1 its fp32 parts in a stream-ordered workspace and the combine kernel.
template <typename T, typename KV = T>
int fmha_run(const void* q, const void* k, const void* v, void* o, float* lse, float rms_g, int B, int Hkv, int G,
             int Nq, int Nk, int D, bool vt, bool causal, float scale, int splits, cudaStream_t stream,
             const attn::Lens* lens = nullptr, const attn::Pages* pages = nullptr, int num_pages = 0,
             float v_scale = 1.f) {
  if (splits <= 1)
    return fmha_dispatch<T, KV>(q, k, v, o, lse, rms_g, B, Hkv, G, Nq, Nk, D, vt, causal, scale, 1, nullptr, nullptr,
                                stream, lens, pages, num_pages, v_scale);
  const size_t rows = static_cast<size_t>(B) * Hkv * G * Nq;
  const size_t lse_bytes = (static_cast<size_t>(splits) * rows * 4 + 255) & ~static_cast<size_t>(255);
  void* ws = nullptr;
  B200_CUDA_OK(cudaMallocAsync(&ws, lse_bytes + static_cast<size_t>(splits) * rows * D * 4, stream));
  float* ws_lse = static_cast<float*>(ws);
  float* ws_o = reinterpret_cast<float*>(static_cast<char*>(ws) + lse_bytes);
  int rc = fmha_dispatch<T, KV>(q, k, v, o, lse, rms_g, B, Hkv, G, Nq, Nk, D, vt, causal, scale, splits, ws_o, ws_lse,
                                stream, lens, pages, num_pages, v_scale);
  if (rc == 0) rc = launch_combine(static_cast<T*>(o), lse, ws_o, ws_lse, rows, D, splits, stream);
  cudaFreeAsync(ws, stream);
  return rc;
}

// num_splits = 0: split until the grid covers the SMs once (a CTA takes a whole SM, so a second wave of shorter CTAs
// would not finish sooner), keeping at least kMinBlocksPerSplit key blocks per split; 1 when the grid already fills
// the machine or the keys span fewer than kMinBlocksToSplit blocks.
int auto_splits(int B, int Hkv, int G, int Nq, int Nk, int D) {
  const int n = host::sm_count();
  const Family f = family(D);
  const long long rows = static_cast<long long>(G) * Nq;
  const long long ctas = (rows + 64 * f.wgs - 1) / (64 * f.wgs) * ((D + f.ds - 1) / f.ds) * B * Hkv;
  const long long num_kv = (Nk + f.bn - 1) / f.bn;
  if (ctas >= n || num_kv < kMinBlocksToSplit) return 1;
  long long s = n / ctas;
  s = std::min<long long>(s, num_kv / kMinBlocksPerSplit);
  s = std::min<long long>(s, kMaxSplits);
  return s < 1 ? 1 : static_cast<int>(s);
}

// The argument checks the attention entries share: each returns 0 or fails with a message that starts with the
// entry's name (who).

// b200_fmha_fwd_f16_kv and _gqa: both lengths, the causal flag, and Nk % 8 for transposed V
int check_kv(const char* who, int Nq, int Nk, int v_transposed, int causal) {
  if (Nq <= 0 || Nk <= 0) return fail(B200_EINVAL, "%s: bad lengths Nq=%d Nk=%d (both must be >= 1)", who, Nq, Nk);
  if (causal != 0 && causal != 1) return fail(B200_EINVAL, "%s: causal must be 0 or 1, got %d", who, causal);
  if (v_transposed && (Nk % 8) != 0)
    return fail(B200_EINVAL, "%s: Nk (%d) must be a multiple of 8 for transposed V", who, Nk);
  return 0;
}

int check_hkv(const char* who, int H, int Hkv) {
  if (Hkv <= 0 || H % Hkv != 0) return fail(B200_EINVAL, "%s: Hkv=%d must be >= 1 and divide H=%d", who, Hkv, H);
  return 0;
}

// grid.y: B * Hkv K/V heads (heads names the product: "B*Hkv", or "B*H" where every head has its own K/V head)
int check_grid_heads(const char* who, const char* heads, int B, int Hkv) {
  if (static_cast<long long>(B) * Hkv > 65535)
    return fail(B200_EINVAL, "%s: %s = %lld exceeds the grid limit 65535", who, heads, static_cast<long long>(B) * Hkv);
  return 0;
}

int check_splits(const char* who, int num_splits) {
  if (num_splits < 0 || num_splits > kMaxSplits)
    return fail(B200_EINVAL, "%s: num_splits=%d must be in 0 .. %d", who, num_splits, kMaxSplits);
  return 0;
}

int check_split_out(const char* who, int num_splits, const void* o) {
  if (num_splits != 1 && (reinterpret_cast<uintptr_t>(o) & 15u) != 0)
    return fail(B200_EINVAL, "%s: o must be 16-byte aligned when num_splits != 1 (the combine stores 16 bytes)", who);
  return 0;
}

// G * nq packed query rows per K/V head; nq_name: "Nq" or "max_seqlen_q"
int check_rows(const char* who, int G, int nq, const char* nq_name) {
  if (static_cast<long long>(G) * nq > 0x7FFFFFFFll)
    return fail(B200_EINVAL, "%s: (H/Hkv)*%s = %lld query rows per K/V head exceed 2^31 - 1", who, nq_name,
                static_cast<long long>(G) * nq);
  return 0;
}

int check_int32(const char* who, const int* a, const char* name) {
  if ((reinterpret_cast<uintptr_t>(a) & 3u) != 0)
    return fail(B200_EINVAL, "%s: %s must be 4-byte aligned (int32)", who, name);
  return 0;
}

// a paged K/V pool of num_pages pages of page_size rows, and block tables of max_pages entries
int check_pool(const char* who, int num_pages, int page_size, int max_pages) {
  if (num_pages < 1) return fail(B200_EINVAL, "%s: num_pages=%d must be >= 1", who, num_pages);
  if (max_pages < 1) return fail(B200_EINVAL, "%s: max_pages_per_seq=%d must be >= 1", who, max_pages);
  if (page_size < 16 || (page_size & (page_size - 1)) != 0)
    return fail(B200_EINVAL, "%s: page_size=%d must be a power of two >= 16", who, page_size);
  if (static_cast<long long>(num_pages) * page_size > 0x7FFFFFFFll)
    return fail(B200_EINVAL, "%s: num_pages*page_size = %lld pool rows exceed 2^31 - 1", who,
                static_cast<long long>(num_pages) * page_size);
  if (static_cast<long long>(max_pages) * page_size > 0x7FFFFFFFll)
    return fail(B200_EINVAL, "%s: max_pages_per_seq*page_size = %lld keys per sequence exceed 2^31 - 1", who,
                static_cast<long long>(max_pages) * page_size);
  return 0;
}

// who = "": the message is the reference's, without a prefix
int check_head_dim(const char* who, int D) {
  const char* sep = *who ? ": " : "";
  if (D % 8 != 0) return fail(B200_ENOTSUP, "%s%sheaddim not support! (D=%d must be a multiple of 8)", who, sep, D);
  if (D > 1024) return fail(B200_ENOTSUP, "%s%sheaddim not support! (D=%d > 1024)", who, sep, D);
  return 0;
}

// The checks common to every attention entry and the transpose pre-pass.  The entries with one sequence length pass
// Nq = Nk = N; b200_fmha_fwd_f16_kv checks its own lengths, causal flag and Nk % 8 first, with messages naming them;
// b200_fmha_fwd_f16_gqa also its head counts and splits.  G: query heads per K/V head (K and V have H / G heads);
// splits = 0 picks the split count (auto_splits).
int fmha_impl(const void* q, const void* k, const void* v, void* o, float* lse, int B, int H, int Nq, int Nk, int D,
              int v_transposed, bool causal, float scale, void* stream_, float rms_g = 0.f, int G = 1,
              int splits = 1) {
  if (!q || !k || !v || !o) return fail(B200_EINVAL, "fmha: null pointer");
  if (B <= 0 || H <= 0 || Nq <= 0 || Nk <= 0 || D <= 0)
    return fail(B200_EINVAL, "fmha: bad shape B=%d H=%d N=%d D=%d", B, H, Nq, D);
  const int Hkv = H / G;
  if (int rc = check_grid_heads("fmha", "B*H", B, Hkv)) return rc;
  if (int rc = check_head_dim("", D)) return rc;
  if (v_transposed && (Nk % 8) != 0)
    return fail(B200_EINVAL, "fmha: N (%d) must be a multiple of 8 for transposed V", Nk);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!(scale > 0.f)) scale = 1.0f / sqrtf(static_cast<float>(D));
  if (splits == 0) splits = auto_splits(B, Hkv, G, Nq, Nk, D);
  if (D > 128) {
    if (v_transposed) {
      // the restored V lives in a stream-ordered allocation: calls on different streams never share
      // scratch, nothing stays pinned between calls, and neither the allocation nor the free
      // synchronises the device (the memory returns to the pool once this stream passes the free)
      void* ws = nullptr;
      const size_t bytes = static_cast<size_t>(B) * Hkv * Nk * D * 2;
      B200_CUDA_OK(cudaMallocAsync(&ws, bytes, stream));
      dim3 grid((Nk + 31) / 32, (D + 31) / 32, B * Hkv), block(32, 8, 1);
      transpose_dn_to_nd_kernel<<<grid, block, 0, stream>>>(static_cast<const __half*>(v),
                                                            static_cast<__half*>(ws), D, Nk);
      cudaError_t le = cudaGetLastError();
      int rc = 0;
      if (le != cudaSuccess) rc = fail(B200_ECUDA, "transpose launch failed: %s", cudaGetErrorString(le));
      else {
        host::count_launch();
        rc = fmha_run<__half>(q, k, ws, o, lse, rms_g, B, Hkv, G, Nq, Nk, D, false, causal, scale, splits, stream);
      }
      cudaFreeAsync(ws, stream);
      return rc;
    }
  }
  return fmha_run<__half>(q, k, v, o, lse, rms_g, B, Hkv, G, Nq, Nk, D, v_transposed != 0, causal, scale, splits, stream);
}

// The fp8-K/V entries' own checks, after those of their counterparts (who: "fmha_seqlens" or "fmha_paged"), and the
// softmax scale (defaulted as by the counterparts) with k_scale folded in: fp32(scale * k_scale), so that K elements
// are never multiplied.
int fp8kv_scales(const char* who, int D, float k_scale, float v_scale, float* scale) {
  if (D % 16 != 0)
    return fail(B200_EINVAL, "%s: fp8 K/V need D %% 16 == 0 (an e4m3 row of D bytes is the TMA row stride), got D=%d",
                who, D);
  if (!(isfinite(k_scale) && k_scale > 0.f))
    return fail(B200_EINVAL, "%s: k_scale=%g must be finite and > 0", who, static_cast<double>(k_scale));
  if (!(isfinite(v_scale) && v_scale > 0.f))
    return fail(B200_EINVAL, "%s: v_scale=%g must be finite and > 0", who, static_cast<double>(v_scale));
  if (!(*scale > 0.f)) *scale = 1.0f / sqrtf(static_cast<float>(D));
  const float folded = *scale * k_scale;
  if (!(isfinite(folded) && folded > 0.f))
    return fail(B200_EINVAL, "%s: scale*k_scale = %g must be finite and > 0 in fp32", who,
                static_cast<double>(folded));
  *scale = folded;
  return 0;
}

// b200_fmha_fwd_{f16,bf16}_seqlens (pages == nullptr, who "fmha_seqlens") and _paged (who "fmha_paged": k and v are
// pools of num_pages pages [page_size, Hkv, D] read through pages->table, and Nk is the padded max_pages * page_size):
// the same checks and messages for both element types T, and for the fp8-K/V entries (KV = __nv_fp8_e4m3) with their
// own checks after these.
template <typename T, typename KV = T>
int fmha_lens(const void* q, const void* k, const void* v, void* o, float* lse, const int* seqlens_q,
              const int* seqlens_k, const attn::Pages* pages, int num_pages, int B, int H, int Hkv, int Nq, int Nk,
              int D, int causal, int num_splits, float scale, void* stream, float k_scale = 1.f, float v_scale = 1.f) {
  const char* who = pages ? "fmha_paged" : "fmha_seqlens";
  if (pages && (!q || !k || !v || !o || !pages->table))
    return fail(B200_EINVAL, "fmha_paged: null pointer (q, k_cache, v_cache, o and block_table are required)");
  if (!q || !k || !v || !o) return fail(B200_EINVAL, "fmha_seqlens: null pointer (q, k, v and o are required)");
  if (B <= 0 || H <= 0 || D <= 0) return fail(B200_EINVAL, "%s: bad shape B=%d H=%d D=%d", who, B, H, D);
  if (pages && Nq <= 0) return fail(B200_EINVAL, "fmha_paged: bad length Nq=%d (must be >= 1)", Nq);
  if (!pages && (Nq <= 0 || Nk <= 0))
    return fail(B200_EINVAL, "fmha_seqlens: bad lengths Nq=%d Nk=%d (both must be >= 1)", Nq, Nk);
  if (causal != 0 && causal != 1) return fail(B200_EINVAL, "%s: causal must be 0 or 1, got %d", who, causal);
  if (int rc = check_hkv(who, H, Hkv)) return rc;
  if (int rc = check_splits(who, num_splits)) return rc;
  if (int rc = check_grid_heads(who, "B*Hkv", B, Hkv)) return rc;
  if (int rc = check_split_out(who, num_splits, o)) return rc;
  if (int rc = check_rows(who, H / Hkv, Nq, "Nq")) return rc;
  if (int rc = check_int32(who, seqlens_q, "seqlens_q")) return rc;
  if (int rc = check_int32(who, seqlens_k, "seqlens_k")) return rc;
  if (pages) {
    if (int rc = check_int32(who, pages->table, "block_table")) return rc;
    if (int rc = check_pool(who, num_pages, pages->page_size, pages->max_pages)) return rc;
    Nk = pages->max_pages * pages->page_size;
  }
  if (int rc = check_head_dim(who, D)) return rc;
  if constexpr (!std::is_same_v<KV, T>) {
    if (int rc = fp8kv_scales(who, D, k_scale, v_scale, &scale)) return rc;
  }
  if (!(scale > 0.f)) scale = 1.0f / sqrtf(static_cast<float>(D));
  const int G = H / Hkv;
  // the split count follows the padded shape, as for b200_fmha_fwd_f16_gqa: the lengths stay on the device (and
  // b200_fmha_fwd_f16_gqa_splits gives it for either element type); a paged call is the seqlens call on the padded Nk
  const int splits = num_splits == 0 ? auto_splits(B, Hkv, G, Nq, Nk, D) : num_splits;
  const attn::Lens lens{seqlens_q, seqlens_k, Hkv};
  return fmha_run<T, KV>(q, k, v, o, lse, 0.f, B, Hkv, G, Nq, Nk, D, false, causal == 1, scale, splits,
                         static_cast<cudaStream_t>(stream), &lens, pages, num_pages, v_scale);
}

// b200_fmha_fwd_{f16,bf16}_varlen (table == nullptr: cu_k is cu_seqlens_k, K / V [total_k, Hkv, D]) and _varlen_paged
// (cu_k is seqused_k, K / V pools of num_pages pages [page_size, Hkv, D], total_k unused).  Every check comes before
// the first CUDA call.  One launch of attn_varlen_kernel with the ring and shared memory of the seqlens kernels.
template <typename T>
int fmha_varlen(const char* who, const void* q, const void* k, const void* v, void* o, float* lse, const int* cu_q,
                const int* cu_k, const int* table, int B, int H, int Hkv, int total_q, int total_k, int max_q, int max_k,
                int num_pages, int page_size, int max_pages, int D, int causal, float scale, void* stream) {
  const bool paged = table != nullptr;
  if (!q || !k || !v || !o || !cu_q || !cu_k)
    return fail(B200_EINVAL, paged ? "%s: null pointer (q, k_cache, v_cache, o, cu_seqlens_q, seqused_k and "
                                     "block_table are required)"
                                   : "%s: null pointer (q, k, v, o, cu_seqlens_q and cu_seqlens_k are required)",
                who);
  if (B <= 0 || H <= 0 || D <= 0) return fail(B200_EINVAL, "%s: bad shape B=%d H=%d D=%d", who, B, H, D);
  if (total_q <= 0) return fail(B200_EINVAL, "%s: total_q=%d must be >= 1", who, total_q);
  if (!paged && total_k <= 0) return fail(B200_EINVAL, "%s: total_k=%d must be >= 1", who, total_k);
  if (max_q <= 0) return fail(B200_EINVAL, "%s: max_seqlen_q=%d must be >= 1", who, max_q);
  if (!paged && max_k <= 0) return fail(B200_EINVAL, "%s: max_seqlen_k=%d must be >= 1", who, max_k);
  if (causal != 0 && causal != 1) return fail(B200_EINVAL, "%s: causal must be 0 or 1, got %d", who, causal);
  if (int rc = check_hkv(who, H, Hkv)) return rc;
  if (int rc = check_grid_heads(who, "B*Hkv", B, Hkv)) return rc;
  if (int rc = check_int32(who, cu_q, "cu_seqlens_q")) return rc;
  if (int rc = check_int32(who, cu_k, paged ? "seqused_k" : "cu_seqlens_k")) return rc;
  if (paged) {
    if (int rc = check_int32(who, table, "block_table")) return rc;
    if (int rc = check_pool(who, num_pages, page_size, max_pages)) return rc;
  }
  if (int rc = check_head_dim(who, D)) return rc;
  // the bytes of q / o must be addressable in int64 (k / v: rows < 2^31 times Hkv <= 65535 times D <= 1024 are)
  if (static_cast<long long>(total_q) * H > 0x3FFFFFFFFFFFFFFFll / D)
    return fail(B200_EINVAL, "%s: total_q*H*D = %d*%d*%d elements overflow", who, total_q, H, D);
  const long long kv_rows = paged ? static_cast<long long>(num_pages) * page_size : total_k;
  const int G = H / Hkv;
  if (int rc = check_rows(who, G, max_q, "max_seqlen_q")) return rc;
  const Family f = family(D);
  const int tph = (max_q + 64 * f.wgs - 1) / (64 * f.wgs), slabs = (D + f.ds - 1) / f.ds;
  if (static_cast<long long>(G) * tph * slabs > 0x7FFFFFFFll)
    return fail(B200_EINVAL, "%s: (H/Hkv)*ceil(max_seqlen_q/%d)*%d = %lld CTAs exceed the grid limit 2^31 - 1", who,
                64 * f.wgs, slabs, static_cast<long long>(G) * tph * slabs);
  if (!(scale > 0.f)) scale = 1.0f / sqrtf(static_cast<float>(D));

  const int nk_pad = paged ? max_pages * page_size : max_k;   // the clamp of every sequence's keys
  attn::Params p;
  const int smem = attn_params(&p, G, max_q, nk_pad, D, scale, lse, 0.f, o, false, 0);
  if (smem == 0) return fail(B200_ENOTSUP, "%s: headdim not support! (D=%d)", who, D);
  p.tph = tph;

  constexpr bool bf16 = std::is_same_v<T, __nv_bfloat16>;
  const CUtensorMapDataType dt = bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  CUtensorMap tq, tk, tv;
  int rc;
  if ((rc = rows_map(&tq, q, D, H, static_cast<uint64_t>(total_q), 64, 2, dt))) return rc;
  const int box = paged ? std::min(page_size, f.bn) : f.bn;
  if ((rc = rows_map(&tk, k, D, Hkv, static_cast<uint64_t>(kv_rows), box, 2, dt))) return rc;
  if ((rc = rows_map(&tv, v, D, Hkv, static_cast<uint64_t>(kv_rows), box, 2, dt))) return rc;
  const attn::Varlen vl{cu_q, cu_k, total_q, H, Hkv};
  const attn::Pages pages{table, page_size, max_pages};
  const attn::Launch l{tq, tk, tv, p, G * tph, B * Hkv, 1, smem, static_cast<cudaStream_t>(stream)};
  return attn::launch_attn_varlen<T>(l, causal == 1, vl, paged ? &pages : nullptr);
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
  if (int rc = check_kv("fmha_kv", Nq, Nk, v_transposed, causal)) return rc;
  return fmha_impl(q, k, v, o, lse, B, H, Nq, Nk, D, v_transposed, causal == 1, scale, stream);
}

int b200_fmha_fwd_f16_gqa(const void* q, const void* k, const void* v, void* o, float* lse, int B, int H, int Hkv,
                          int Nq, int Nk, int D, int v_transposed, int causal, int num_splits, float scale,
                          void* stream) {
  const char* who = "fmha_gqa";
  if (int rc = check_kv(who, Nq, Nk, v_transposed, causal)) return rc;
  if (int rc = check_hkv(who, H, Hkv)) return rc;
  if (int rc = check_splits(who, num_splits)) return rc;
  if (int rc = check_grid_heads(who, "B*Hkv", B, Hkv)) return rc;
  if (int rc = check_split_out(who, num_splits, o)) return rc;
  if (int rc = check_rows(who, H / Hkv, Nq, "Nq")) return rc;
  return fmha_impl(q, k, v, o, lse, B, H, Nq, Nk, D, v_transposed, causal == 1, scale, stream, 0.f, H / Hkv,
                   num_splits);
}

int b200_fmha_fwd_f16_gqa_splits(int B, int H, int Hkv, int Nq, int Nk, int D) {
  if (B <= 0 || H <= 0 || Nq <= 0 || Nk <= 0 || D <= 0)
    return fail(B200_EINVAL, "fmha_gqa_splits: bad shape B=%d H=%d Nq=%d Nk=%d D=%d", B, H, Nq, Nk, D);
  if (Hkv <= 0 || H % Hkv != 0)
    return fail(B200_EINVAL, "fmha_gqa_splits: Hkv=%d must be >= 1 and divide H=%d", Hkv, H);
  return auto_splits(B, Hkv, H / Hkv, Nq, Nk, D);
}

int b200_fmha_fwd_f16_seqlens(const void* q, const void* k, const void* v, void* o, float* lse, const int* seqlens_q,
                              const int* seqlens_k, int B, int H, int Hkv, int Nq, int Nk, int D, int causal,
                              int num_splits, float scale, void* stream) {
  return fmha_lens<__half>(q, k, v, o, lse, seqlens_q, seqlens_k, nullptr, 0, B, H, Hkv, Nq, Nk, D, causal, num_splits,
                           scale, stream);
}

int b200_fmha_fwd_f16_paged(const void* q, const void* k_cache, const void* v_cache, void* o, float* lse,
                            const int* block_table, const int* seqlens_q, const int* seqlens_k, int B, int H, int Hkv,
                            int Nq, int num_pages, int page_size, int max_pages_per_seq, int D, int causal,
                            int num_splits, float scale, void* stream) {
  const attn::Pages pages{block_table, page_size, max_pages_per_seq};
  return fmha_lens<__half>(q, k_cache, v_cache, o, lse, seqlens_q, seqlens_k, &pages, num_pages, B, H, Hkv, Nq, 0, D,
                           causal, num_splits, scale, stream);
}

int b200_fmha_fwd_bf16_seqlens(const void* q, const void* k, const void* v, void* o, float* lse, const int* seqlens_q,
                               const int* seqlens_k, int B, int H, int Hkv, int Nq, int Nk, int D, int causal,
                               int num_splits, float scale, void* stream) {
  return fmha_lens<__nv_bfloat16>(q, k, v, o, lse, seqlens_q, seqlens_k, nullptr, 0, B, H, Hkv, Nq, Nk, D, causal,
                                  num_splits, scale, stream);
}

int b200_fmha_fwd_bf16_paged(const void* q, const void* k_cache, const void* v_cache, void* o, float* lse,
                             const int* block_table, const int* seqlens_q, const int* seqlens_k, int B, int H, int Hkv,
                             int Nq, int num_pages, int page_size, int max_pages_per_seq, int D, int causal,
                             int num_splits, float scale, void* stream) {
  const attn::Pages pages{block_table, page_size, max_pages_per_seq};
  return fmha_lens<__nv_bfloat16>(q, k_cache, v_cache, o, lse, seqlens_q, seqlens_k, &pages, num_pages, B, H, Hkv, Nq,
                                  0, D, causal, num_splits, scale, stream);
}

int b200_fmha_fwd_f16_fp8kv_seqlens(const void* q, const void* k, const void* v, void* o, float* lse,
                                    const int* seqlens_q, const int* seqlens_k, int B, int H, int Hkv, int Nq, int Nk,
                                    int D, int causal, int num_splits, float scale, float k_scale, float v_scale,
                                    void* stream) {
  return fmha_lens<__half, __nv_fp8_e4m3>(q, k, v, o, lse, seqlens_q, seqlens_k, nullptr, 0, B, H, Hkv, Nq, Nk, D,
                                          causal, num_splits, scale, stream, k_scale, v_scale);
}

int b200_fmha_fwd_bf16_fp8kv_seqlens(const void* q, const void* k, const void* v, void* o, float* lse,
                                     const int* seqlens_q, const int* seqlens_k, int B, int H, int Hkv, int Nq, int Nk,
                                     int D, int causal, int num_splits, float scale, float k_scale, float v_scale,
                                     void* stream) {
  return fmha_lens<__nv_bfloat16, __nv_fp8_e4m3>(q, k, v, o, lse, seqlens_q, seqlens_k, nullptr, 0, B, H, Hkv, Nq, Nk,
                                                 D, causal, num_splits, scale, stream, k_scale, v_scale);
}

int b200_fmha_fwd_f16_fp8kv_paged(const void* q, const void* k_cache, const void* v_cache, void* o, float* lse,
                                  const int* block_table, const int* seqlens_q, const int* seqlens_k, int B, int H,
                                  int Hkv, int Nq, int num_pages, int page_size, int max_pages_per_seq, int D,
                                  int causal, int num_splits, float scale, float k_scale, float v_scale, void* stream) {
  const attn::Pages pages{block_table, page_size, max_pages_per_seq};
  return fmha_lens<__half, __nv_fp8_e4m3>(q, k_cache, v_cache, o, lse, seqlens_q, seqlens_k, &pages, num_pages, B, H,
                                          Hkv, Nq, 0, D, causal, num_splits, scale, stream, k_scale, v_scale);
}

int b200_fmha_fwd_bf16_fp8kv_paged(const void* q, const void* k_cache, const void* v_cache, void* o, float* lse,
                                   const int* block_table, const int* seqlens_q, const int* seqlens_k, int B, int H,
                                   int Hkv, int Nq, int num_pages, int page_size, int max_pages_per_seq, int D,
                                   int causal, int num_splits, float scale, float k_scale, float v_scale,
                                   void* stream) {
  const attn::Pages pages{block_table, page_size, max_pages_per_seq};
  return fmha_lens<__nv_bfloat16, __nv_fp8_e4m3>(q, k_cache, v_cache, o, lse, seqlens_q, seqlens_k, &pages, num_pages,
                                                 B, H, Hkv, Nq, 0, D, causal, num_splits, scale, stream, k_scale,
                                                 v_scale);
}

int b200_fmha_fwd_f16_varlen(const void* q, const void* k, const void* v, void* o, float* lse, const int* cu_seqlens_q,
                             const int* cu_seqlens_k, int B, int H, int Hkv, int total_q, int total_k, int max_seqlen_q,
                             int max_seqlen_k, int D, int causal, float scale, void* stream) {
  return fmha_varlen<__half>("fmha_varlen", q, k, v, o, lse, cu_seqlens_q, cu_seqlens_k, nullptr, B, H, Hkv, total_q,
                             total_k, max_seqlen_q, max_seqlen_k, 0, 0, 0, D, causal, scale, stream);
}

int b200_fmha_fwd_bf16_varlen(const void* q, const void* k, const void* v, void* o, float* lse, const int* cu_seqlens_q,
                              const int* cu_seqlens_k, int B, int H, int Hkv, int total_q, int total_k,
                              int max_seqlen_q, int max_seqlen_k, int D, int causal, float scale, void* stream) {
  return fmha_varlen<__nv_bfloat16>("fmha_varlen", q, k, v, o, lse, cu_seqlens_q, cu_seqlens_k, nullptr, B, H, Hkv,
                                    total_q, total_k, max_seqlen_q, max_seqlen_k, 0, 0, 0, D, causal, scale, stream);
}

// block_table is checked here: a null one would turn the call into the packed one
int b200_fmha_fwd_f16_varlen_paged(const void* q, const void* k_cache, const void* v_cache, void* o, float* lse,
                                   const int* cu_seqlens_q, const int* seqused_k, const int* block_table, int B, int H,
                                   int Hkv, int total_q, int max_seqlen_q, int num_pages, int page_size,
                                   int max_pages_per_seq, int D, int causal, float scale, void* stream) {
  if (!block_table) return fail(B200_EINVAL, "fmha_varlen_paged: null pointer (block_table is required)");
  return fmha_varlen<__half>("fmha_varlen_paged", q, k_cache, v_cache, o, lse, cu_seqlens_q, seqused_k, block_table, B,
                             H, Hkv, total_q, 0, max_seqlen_q, 0, num_pages, page_size, max_pages_per_seq, D, causal,
                             scale, stream);
}

int b200_fmha_fwd_bf16_varlen_paged(const void* q, const void* k_cache, const void* v_cache, void* o, float* lse,
                                    const int* cu_seqlens_q, const int* seqused_k, const int* block_table, int B, int H,
                                    int Hkv, int total_q, int max_seqlen_q, int num_pages, int page_size,
                                    int max_pages_per_seq, int D, int causal, float scale, void* stream) {
  if (!block_table) return fail(B200_EINVAL, "fmha_varlen_paged: null pointer (block_table is required)");
  return fmha_varlen<__nv_bfloat16>("fmha_varlen_paged", q, k_cache, v_cache, o, lse, cu_seqlens_q, seqused_k,
                                    block_table, B, H, Hkv, total_q, 0, max_seqlen_q, 0, num_pages, page_size,
                                    max_pages_per_seq, D, causal, scale, stream);
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
