// kvcache_capi.cu — KV-cache append with rotary embedding: the write half of a decode or chunked-prefill step, in one
// launch.  For every sequence b, new token t < n_new and head:
//
//   L_b = clamp(cache_seqlens[b], 0, capacity)      (read on the GPU; capacity = Nk, or max_pages_per_seq * page_size)
//   p   = L_b + t                                    (the token's position)
//   k_new[b,h,t,:] (rotated at p) and v_new[b,h,t,:] go to position p of the cache when p < capacity:
//     dense  [B, Hkv, Nk, D]                  row p of (b, h)
//     paged  [num_pages, page_size, Hkv, D]   row p % page_size of page block_table[b][p / page_size]; an entry outside
//                                             [0, num_pages) means the token is not written
//   q[b,h,t,:] (rotated at p) goes to q_out[b,h,t,:] for every token, written or dropped
//   seqlens_out[b] = min(L_b + n_new, capacity)
//
// Rotary (k and q, never v): fp32 tables cos, sin [rotary_len, rotary_dim / 2] indexed [p, i]; pair i is (2i, 2i+1)
// when interleaved (GPT-J), else (i, i + rotary_dim / 2) (NeoX / Llama); x0' = x0 c - x1 s, x1' = x0 s + x1 c in fp32
// (one product rounded, the other fused), rounded once to T.  Columns >= rotary_dim are copied.
// e4m3 caches: code = cvt.rn.satfinite.e4m3x2.f32(float(x_T) / scale), an IEEE division of the value already rounded to
// T, k with k_scale and v with v_scale: bit for bit (x_T.float() / scale).clamp(-448, 448).to(float8_e4m3fn).
//
// Layout: one thread per unit of 8 columns (one 16-byte pack of T) of one row of k, v or q; under NeoX rotary a unit of
// the rotated columns is the pack pair (j, j + rotary_dim / 16), both halves of its pairs.  Units run over the rows of
// k_new, then v_new, then q, each [B, heads, n_new] in memory order, so consecutive threads read consecutive bytes.  A
// grid-stride loop with 64-bit unit indices and 64-bit element offsets: pools past 2^31 elements are normal.  A unit
// whose token is not written loads nothing.  HBM-bound: every input byte is read once and every output byte written
// once (e4m3: 8-byte stores of 8 codes).
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_fp8.h>

#include <cmath>

#include "capi_common.cuh"
#include "sm90_ptx.cuh"

namespace {

using b200::host::fail;
using b200::host::overlaps;

struct AppendParams {
  const void* k_new;
  const void* v_new;
  void* k_cache;
  void* v_cache;
  const int* cache_seqlens;
  int* seqlens_out;          // may be null
  const int* block_table;    // null: dense cache
  const void* q;             // null: no q
  void* q_out;
  const float* cos;          // null: no rotary
  const float* sin;
  int B, H, Hkv, n_new, D;
  int capacity;              // positions a sequence can hold
  int page_shift, num_pages, max_pages;
  int rotary_dim, interleaved;
  float k_scale, v_scale;
  unsigned upr;              // units per row
  unsigned kv_rows;          // B * Hkv * n_new
  unsigned long long units;  // all units of k, v and q
};

template <typename T>
struct Elt;
template <>
struct Elt<__half> {
  static __device__ __forceinline__ float2 unpack(uint32_t w) {
    return __half22float2(*reinterpret_cast<const __half2*>(&w));
  }
  static __device__ __forceinline__ uint32_t pack(float lo, float hi) { return b200::pack_half2(lo, hi); }
};
template <>
struct Elt<__nv_bfloat16> {
  // a bf16 is the upper half of its fp32
  static __device__ __forceinline__ float2 unpack(uint32_t w) {
    return make_float2(__uint_as_float(w << 16), __uint_as_float(w & 0xffff0000u));
  }
  static __device__ __forceinline__ uint32_t pack(float lo, float hi) { return b200::pack_bf162(lo, hi); }
};

// (x0 c - x1 s, x0 s + x1 c) in fp32 with the products' roundings fixed, so every build computes the same bits
__device__ __forceinline__ float2 rotate(float x0, float x1, float c, float s) {
  return make_float2(fmaf(x0, c, -__fmul_rn(x1, s)), fmaf(x0, s, __fmul_rn(x1, c)));
}

// one word (2 elements) of T: rotate the pair (lo, hi) of the word (interleaved)
template <typename T>
__device__ __forceinline__ uint32_t rotate_word(uint32_t w, float c, float s) {
  const float2 x = Elt<T>::unpack(w);
  const float2 y = rotate(x.x, x.y, c, s);
  return Elt<T>::pack(y.x, y.y);
}

// eight T elements to eight e4m3 codes of x / scale
template <typename T>
__device__ __forceinline__ uint2 quantise(const uint4& v, float scale) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
  uint32_t c[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 x = Elt<T>::unpack(w[i]);
    c[i] = b200::float2_to_e4m3x2(__fdiv_rn(x.x, scale), __fdiv_rn(x.y, scale));
  }
  return make_uint2(c[0] | (c[1] << 16), c[2] | (c[3] << 16));
}

// one 16-byte pack of T to element offset `at` of the cache (or of q_out)
template <typename T, typename CacheT>
__device__ __forceinline__ void store(CacheT* base, size_t at, const uint4& v, float scale) {
  if constexpr (std::is_same_v<CacheT, __nv_fp8_e4m3>)
    *reinterpret_cast<uint2*>(base + at) = quantise<T>(v, scale);
  else
    b200::st_stream(base + at, v);
}

template <typename T, typename CacheT>
__global__ void __launch_bounds__(256) kvcache_append_kernel(const AppendParams p) {
  const unsigned long long stride = static_cast<unsigned long long>(gridDim.x) * blockDim.x;
  const unsigned long long first = static_cast<unsigned long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (p.seqlens_out != nullptr) {
    for (unsigned long long b = first; b < static_cast<unsigned long long>(p.B); b += stride) {
      const int L = min(max(__ldg(p.cache_seqlens + b), 0), p.capacity);
      p.seqlens_out[b] = static_cast<int>(min(static_cast<long long>(L) + p.n_new, static_cast<long long>(p.capacity)));
    }
  }
  const unsigned half = static_cast<unsigned>(p.rotary_dim) / 16;   // packs in one half of the rotated columns
  const bool neox = p.cos != nullptr && !p.interleaved;
  for (unsigned long long u = first; u < p.units; u += stride) {
    unsigned row, unit;
    if (u <= 0xFFFFFFFFull) {   // 64-bit division is emulated: only for indices that need it
      row = static_cast<unsigned>(u) / p.upr;
      unit = static_cast<unsigned>(u) - row * p.upr;
    } else {
      row = static_cast<unsigned>(u / p.upr);
      unit = static_cast<unsigned>(u - static_cast<unsigned long long>(row) * p.upr);
    }
    int which = 0;              // 0: k, 1: v, 2: q
    unsigned r = row, heads = p.Hkv;
    if (r >= p.kv_rows) {
      r -= p.kv_rows;
      which = 1;
      if (r >= p.kv_rows) {
        r -= p.kv_rows;
        which = 2;
        heads = p.H;
      }
    }
    const unsigned t = r % p.n_new, bh = r / p.n_new;
    const unsigned h = bh % heads, b = bh / heads;
    const int L = min(max(__ldg(p.cache_seqlens + b), 0), p.capacity);
    const unsigned pos = static_cast<unsigned>(L) + t;

    size_t dst;                 // element offset of the destination row
    if (which == 2) {
      dst = static_cast<size_t>(r) * p.D;
    } else {
      if (pos >= static_cast<unsigned>(p.capacity)) continue;   // past capacity: dropped
      if (p.block_table == nullptr) {
        dst = (static_cast<size_t>(b * p.Hkv + h) * p.capacity + pos) * p.D;
      } else {
        const int page = __ldg(p.block_table + static_cast<size_t>(b) * p.max_pages + (pos >> p.page_shift));
        if (page < 0 || page >= p.num_pages) continue;           // no page: not written
        const size_t prow = (static_cast<size_t>(page) << p.page_shift) + (pos & ((1u << p.page_shift) - 1));
        dst = (prow * p.Hkv + h) * p.D;
      }
    }

    unsigned pk0 = unit, pk1 = 0xFFFFFFFFu;   // pk1: the NeoX partner pack, if any
    if (neox) {
      if (unit < half) pk1 = unit + half;
      else pk0 = unit + half;
    }
    const T* src = static_cast<const T*>(which == 0 ? p.k_new : which == 1 ? p.v_new : p.q) +
                   static_cast<size_t>(r) * p.D;
    uint4 a = b200::ld_stream(src + pk0 * 8);
    uint4 c2 = make_uint4(0, 0, 0, 0);
    if (pk1 != 0xFFFFFFFFu) c2 = b200::ld_stream(src + pk1 * 8);

    if (which != 1 && p.cos != nullptr && pk0 * 8 < static_cast<unsigned>(p.rotary_dim)) {
      const size_t trow = static_cast<size_t>(pos) * (p.rotary_dim / 2);
      if (p.interleaved) {      // pairs (2i, 2i+1), i = 4 pk0 .. 4 pk0 + 3: one word each
        const float4 c = __ldg(reinterpret_cast<const float4*>(p.cos + trow + pk0 * 4));
        const float4 s = __ldg(reinterpret_cast<const float4*>(p.sin + trow + pk0 * 4));
        a = make_uint4(rotate_word<T>(a.x, c.x, s.x), rotate_word<T>(a.y, c.y, s.y), rotate_word<T>(a.z, c.z, s.z),
                       rotate_word<T>(a.w, c.w, s.w));
      } else {                  // pairs (i, i + rotary_dim / 2), i = 8 pk0 .. 8 pk0 + 7: element m of a and of c2
        const float4* cp = reinterpret_cast<const float4*>(p.cos + trow + pk0 * 8);
        const float4* sp = reinterpret_cast<const float4*>(p.sin + trow + pk0 * 8);
        const float4 c0 = __ldg(cp), c1 = __ldg(cp + 1), s0 = __ldg(sp), s1 = __ldg(sp + 1);
        const float cs[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
        const float sn[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
        uint32_t wa[4] = {a.x, a.y, a.z, a.w}, wb[4] = {c2.x, c2.y, c2.z, c2.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float2 x0 = Elt<T>::unpack(wa[i]), x1 = Elt<T>::unpack(wb[i]);
          const float2 lo = rotate(x0.x, x1.x, cs[2 * i], sn[2 * i]);
          const float2 hi = rotate(x0.y, x1.y, cs[2 * i + 1], sn[2 * i + 1]);
          wa[i] = Elt<T>::pack(lo.x, hi.x);
          wb[i] = Elt<T>::pack(lo.y, hi.y);
        }
        a = make_uint4(wa[0], wa[1], wa[2], wa[3]);
        c2 = make_uint4(wb[0], wb[1], wb[2], wb[3]);
      }
    }

    if (which == 2) {
      T* out = static_cast<T*>(p.q_out) + dst;
      b200::st_stream(out + pk0 * 8, a);
      if (pk1 != 0xFFFFFFFFu) b200::st_stream(out + pk1 * 8, c2);
    } else {
      CacheT* cache = static_cast<CacheT*>(which == 0 ? p.k_cache : p.v_cache);
      const float scale = which == 0 ? p.k_scale : p.v_scale;
      store<T, CacheT>(cache, dst + pk0 * 8, a, scale);
      if (pk1 != 0xFFFFFFFFu) store<T, CacheT>(cache, dst + pk1 * 8, c2, scale);
    }
  }
}

// The arguments of both entries; dense calls have block_table = null, num_pages = page_size = max_pages = 0.
struct AppendArgs {
  const void* k_new;
  const void* v_new;
  void* k_cache;
  void* v_cache;
  const int* block_table;
  const int* cache_seqlens;
  int* seqlens_out;
  const void* q;
  void* q_out;
  const float* cos;
  const float* sin;
  int B, H, Hkv, n_new, Nk, num_pages, page_size, max_pages_per_seq, D, rotary_dim, rotary_len, interleaved;
  int cache_dtype;
  float k_scale, v_scale;
};

constexpr long long kIntMax = 0x7FFFFFFFll;
constexpr unsigned long long kMaxElems = 1ull << 56;

// a * b * c * d, or kMaxElems when that is reached (every factor >= 1)
unsigned long long elems(long long a, long long b, long long c, long long d) {
  unsigned long long r = 1;
  for (long long x : {a, b, c, d}) {
    if (r > kMaxElems / static_cast<unsigned long long>(x)) return kMaxElems;
    r *= static_cast<unsigned long long>(x);
  }
  return r;
}

template <typename T>
int kvcache_append(const AppendArgs& a, int t_dtype, bool paged, cudaStream_t stream) {
  const char* who = "kvcache_append";
  const struct { const void* p; const char* name; } required[] = {
      {a.k_new, "k_new"}, {a.v_new, "v_new"}, {a.k_cache, "k_cache"}, {a.v_cache, "v_cache"},
      {a.cache_seqlens, "cache_seqlens"}, {paged ? a.block_table : a.k_new, "block_table"}};
  for (const auto& r : required)
    if (r.p == nullptr) return fail(B200_EINVAL, "%s: %s is NULL", who, r.name);
  if ((a.q == nullptr) != (a.q_out == nullptr))
    return fail(B200_EINVAL, "%s: q and q_out must both be NULL or both be set", who);
  if ((a.cos == nullptr) != (a.sin == nullptr))
    return fail(B200_EINVAL, "%s: rotary_cos and rotary_sin must both be NULL or both be set", who);
  const struct { int v; const char* name; } dims[] = {
      {a.B, "B"}, {a.H, "H"}, {a.Hkv, "Hkv"}, {a.n_new, "n_new"}, {a.D, "D"},
      {paged ? a.num_pages : a.Nk, paged ? "num_pages" : "Nk"}, {paged ? a.page_size : 1, "page_size"},
      {paged ? a.max_pages_per_seq : 1, "max_pages_per_seq"}};
  for (const auto& d : dims)
    if (d.v < 1) return fail(B200_EINVAL, "%s: %s=%d must be >= 1", who, d.name, d.v);
  if (a.H % a.Hkv != 0) return fail(B200_EINVAL, "%s: Hkv=%d must divide H=%d", who, a.Hkv, a.H);
  if (a.cache_dtype != t_dtype && a.cache_dtype != B200_DTYPE_E4M3)
    return fail(B200_EINVAL, "%s: cache_dtype=%d must be %d (the type of k_new) or B200_DTYPE_E4M3 (%d)", who,
                a.cache_dtype, t_dtype, B200_DTYPE_E4M3);
  const bool e4m3 = a.cache_dtype == B200_DTYPE_E4M3;
  if (a.D % (e4m3 ? 16 : 8) != 0)
    return fail(B200_EINVAL, "%s: D=%d must be a multiple of %d%s", who, a.D, e4m3 ? 16 : 8,
                e4m3 ? " with an e4m3 cache" : "");
  if (paged && (a.page_size < 16 || (a.page_size & (a.page_size - 1)) != 0))
    return fail(B200_EINVAL, "%s: page_size=%d must be a power of two >= 16", who, a.page_size);
  const long long capacity = paged ? static_cast<long long>(a.max_pages_per_seq) * a.page_size : a.Nk;
  if (capacity + a.n_new > kIntMax)
    return fail(B200_EINVAL, "%s: capacity %lld + n_new %d positions exceed 2^31 - 1", who, capacity, a.n_new);
  const unsigned long long knew_elems = elems(a.B, a.Hkv, a.n_new, a.D), q_elems = elems(a.B, a.H, a.n_new, a.D);
  const unsigned long long cache_elems =
      paged ? elems(a.num_pages, a.page_size, a.Hkv, a.D) : elems(a.B, a.Hkv, a.Nk, a.D);
  const unsigned long long rows = static_cast<unsigned long long>(a.B) * a.n_new * (2ull * a.Hkv + a.H);
  if (knew_elems >= kMaxElems || q_elems >= kMaxElems || cache_elems >= kMaxElems || rows > kIntMax)
    return fail(B200_EINVAL, "%s: element counts out of range (B*n_new*(2*Hkv+H) = %llu rows, at most 2^31 - 1)", who,
                rows);
  if (a.cos != nullptr) {
    if (a.interleaved != 0 && a.interleaved != 1)
      return fail(B200_EINVAL, "%s: rotary_interleaved must be 0 or 1, got %d", who, a.interleaved);
    if (a.rotary_dim <= 0 || a.rotary_dim > a.D || a.rotary_dim % 16 != 0)
      return fail(B200_EINVAL, "%s: rotary_dim=%d must be a multiple of 16 in 16 .. D=%d", who, a.rotary_dim, a.D);
    if (a.rotary_len < capacity + a.n_new)
      return fail(B200_EINVAL, "%s: rotary_len=%d must be >= capacity + n_new = %lld (the largest position + 1)", who,
                  a.rotary_len, capacity + a.n_new);
  } else if (a.rotary_dim != 0 || a.rotary_len != 0 || a.interleaved != 0) {
    return fail(B200_EINVAL, "%s: rotary_dim, rotary_len and rotary_interleaved must be 0 without rotary tables", who);
  }
  const struct { float v; const char* name; } scales[] = {{a.k_scale, "k_scale"}, {a.v_scale, "v_scale"}};
  for (const auto& s : scales) {
    if (!(std::isfinite(s.v) && s.v > 0.f))
      return fail(B200_EINVAL, "%s: %s=%g must be finite and > 0", who, s.name, static_cast<double>(s.v));
    if (!e4m3 && s.v != 1.f)
      return fail(B200_EINVAL, "%s: %s=%g must be 1 unless the cache is e4m3", who, s.name, static_cast<double>(s.v));
  }
  const size_t tb = sizeof(T), cb = e4m3 ? 1 : sizeof(T);
  const size_t table_bytes = a.cos ? static_cast<size_t>(a.rotary_len) * (a.rotary_dim / 2) * sizeof(float) : 0;
  const struct Buf { const void* p; size_t bytes; const char* name; bool written; unsigned align; } bufs[] = {
      {a.k_new, knew_elems * tb, "k_new", false, 16},
      {a.v_new, knew_elems * tb, "v_new", false, 16},
      {a.k_cache, cache_elems * cb, "k_cache", true, 16},
      {a.v_cache, cache_elems * cb, "v_cache", true, 16},
      {a.q, a.q ? q_elems * tb : 0, "q", false, 16},
      {a.q_out == a.q ? nullptr : a.q_out, a.q_out == a.q ? 0 : q_elems * tb, "q_out", true, 16},
      {a.cos, table_bytes, "rotary_cos", false, 16},
      {a.sin, table_bytes, "rotary_sin", false, 16},
      {a.cache_seqlens, a.B * sizeof(int), "cache_seqlens", false, 4},
      {a.seqlens_out, a.seqlens_out ? a.B * sizeof(int) : 0, "seqlens_out", true, 4},
      {a.block_table, paged ? static_cast<size_t>(a.B) * a.max_pages_per_seq * sizeof(int) : 0, "block_table", false, 4}};
  for (const Buf& x : bufs) {
    if ((reinterpret_cast<uintptr_t>(x.p) & (x.align - 1)) != 0)
      return fail(B200_EINVAL, "%s: %s must be %u-byte aligned", who, x.name, x.align);
  }
  // Every buffer the kernel writes is disjoint from every other buffer (q_out may be q itself: each thread reads its
  // packs before it writes them).
  for (const Buf& w : bufs) {
    if (!w.written) continue;
    for (const Buf& x : bufs)
      if (&x != &w && overlaps(w.p, w.bytes, x.p, x.bytes))
        return fail(B200_EINVAL, "%s: %s overlaps %s", who, w.name, x.name);
  }

  AppendParams p;
  p.k_new = a.k_new;
  p.v_new = a.v_new;
  p.k_cache = a.k_cache;
  p.v_cache = a.v_cache;
  p.cache_seqlens = a.cache_seqlens;
  p.seqlens_out = a.seqlens_out;
  p.block_table = paged ? a.block_table : nullptr;
  p.q = a.q;
  p.q_out = a.q_out;
  p.cos = a.cos;
  p.sin = a.sin;
  p.B = a.B;
  p.H = a.H;
  p.Hkv = a.Hkv;
  p.n_new = a.n_new;
  p.D = a.D;
  p.capacity = static_cast<int>(capacity);
  p.page_shift = paged ? __builtin_ctz(static_cast<unsigned>(a.page_size)) : 0;
  p.num_pages = paged ? a.num_pages : 0;
  p.max_pages = paged ? a.max_pages_per_seq : 0;
  p.rotary_dim = a.cos ? a.rotary_dim : 0;
  p.interleaved = a.interleaved;
  p.k_scale = a.k_scale;
  p.v_scale = a.v_scale;
  const bool neox = a.cos != nullptr && !a.interleaved;
  p.upr = static_cast<unsigned>(a.D / 8 - (neox ? a.rotary_dim / 16 : 0));
  p.kv_rows = static_cast<unsigned>(static_cast<unsigned long long>(a.B) * a.Hkv * a.n_new);
  const unsigned long long all_rows = 2ull * p.kv_rows + (a.q ? static_cast<unsigned long long>(a.B) * a.H * a.n_new : 0);
  p.units = all_rows * p.upr;
  const unsigned long long want = (p.units + 255) / 256;
  const unsigned long long cap = static_cast<unsigned long long>(b200::host::sm_count()) * 16;
  const unsigned grid = static_cast<unsigned>(want < cap ? want : cap);
  if (e4m3) kvcache_append_kernel<T, __nv_fp8_e4m3><<<grid, 256, 0, stream>>>(p);
  else kvcache_append_kernel<T, T><<<grid, 256, 0, stream>>>(p);
  B200_CUDA_OK(cudaGetLastError());
  b200::host::count_launch();
  return 0;
}

}  // namespace

#define B200_APPEND_ARGS_DENSE                                                                                       \
  const void *k_new, const void *v_new, void *k_cache, void *v_cache, const int *cache_seqlens, int *seqlens_out,   \
      const void *q, void *q_out, const float *rotary_cos, const float *rotary_sin, int B, int H, int Hkv,          \
      int n_new, int Nk, int D, int rotary_dim, int rotary_len, int rotary_interleaved, int cache_dtype,            \
      float k_scale, float v_scale, void *stream
#define B200_APPEND_ARGS_PAGED                                                                                       \
  const void *k_new, const void *v_new, void *k_cache, void *v_cache, const int *block_table,                       \
      const int *cache_seqlens, int *seqlens_out, const void *q, void *q_out, const float *rotary_cos,              \
      const float *rotary_sin, int B, int H, int Hkv, int n_new, int num_pages, int page_size, int max_pages_per_seq, \
      int D, int rotary_dim, int rotary_len, int rotary_interleaved, int cache_dtype, float k_scale, float v_scale,  \
      void *stream

extern "C" int b200_kvcache_append_f16(B200_APPEND_ARGS_DENSE) {
  const AppendArgs a{k_new, v_new, k_cache, v_cache, nullptr, cache_seqlens, seqlens_out, q, q_out, rotary_cos,
                     rotary_sin, B, H, Hkv, n_new, Nk, 0, 0, 0, D, rotary_dim, rotary_len, rotary_interleaved,
                     cache_dtype, k_scale, v_scale};
  return kvcache_append<__half>(a, B200_DTYPE_F16, false, static_cast<cudaStream_t>(stream));
}
extern "C" int b200_kvcache_append_bf16(B200_APPEND_ARGS_DENSE) {
  const AppendArgs a{k_new, v_new, k_cache, v_cache, nullptr, cache_seqlens, seqlens_out, q, q_out, rotary_cos,
                     rotary_sin, B, H, Hkv, n_new, Nk, 0, 0, 0, D, rotary_dim, rotary_len, rotary_interleaved,
                     cache_dtype, k_scale, v_scale};
  return kvcache_append<__nv_bfloat16>(a, B200_DTYPE_BF16, false, static_cast<cudaStream_t>(stream));
}
extern "C" int b200_kvcache_append_f16_paged(B200_APPEND_ARGS_PAGED) {
  const AppendArgs a{k_new, v_new, k_cache, v_cache, block_table, cache_seqlens, seqlens_out, q, q_out, rotary_cos,
                     rotary_sin, B, H, Hkv, n_new, 0, num_pages, page_size, max_pages_per_seq, D, rotary_dim,
                     rotary_len, rotary_interleaved, cache_dtype, k_scale, v_scale};
  return kvcache_append<__half>(a, B200_DTYPE_F16, true, static_cast<cudaStream_t>(stream));
}
extern "C" int b200_kvcache_append_bf16_paged(B200_APPEND_ARGS_PAGED) {
  const AppendArgs a{k_new, v_new, k_cache, v_cache, block_table, cache_seqlens, seqlens_out, q, q_out, rotary_cos,
                     rotary_sin, B, H, Hkv, n_new, 0, num_pages, page_size, max_pages_per_seq, D, rotary_dim,
                     rotary_len, rotary_interleaved, cache_dtype, k_scale, v_scale};
  return kvcache_append<__nv_bfloat16>(a, B200_DTYPE_BF16, true, static_cast<cudaStream_t>(stream));
}
