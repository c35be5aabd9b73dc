// capi_common.cu — see capi_common.cuh
#include "capi_common.cuh"

namespace b200 {
namespace host {

static thread_local char g_err[512] = {0};
static std::atomic<uint64_t> g_launches{0};

char* last_error_buf() { return g_err; }

int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

void count_launch(uint64_t n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

int sm_count() {
  static int cached[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;   // H100 SXM
  if (cached[dev] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
      n = 132;
    cached[dev] = n;
  }
  return cached[dev];
}

int host_pipe(HostPipe** out) {
  static thread_local HostPipe pipe;
  int dev = 0;
  cudaGetDevice(&dev);
  if (!pipe.ok || pipe.dev != dev) {
    B200_CUDA_OK(cudaStreamCreateWithFlags(&pipe.in, cudaStreamNonBlocking));
    B200_CUDA_OK(cudaStreamCreateWithFlags(&pipe.out, cudaStreamNonBlocking));
    for (auto& e : pipe.ev) B200_CUDA_OK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    pipe.ok = true;
    pipe.dev = dev;
  }
  *out = &pipe;
  return 0;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPointByVersion("cuTensorMapEncodeTiled", &p, 12000, cudaEnableDefault,
                                         &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

struct TmapKey {
  uint64_t w[12];
  bool operator==(const TmapKey& o) const { return memcmp(w, o.w, sizeof(w)) == 0; }
};
struct TmapKeyHash {
  size_t operator()(const TmapKey& k) const {
    uint64_t h = 1469598103934665603ull;
    for (uint64_t v : k.w) { h ^= v; h *= 1099511628211ull; }
    return static_cast<size_t>(h);
  }
};

int get_tmap(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
             const uint64_t* strides_bytes, const uint32_t* box, CUtensorMapSwizzle swizzle,
             CUtensorMapDataType dtype) {
  static std::mutex mu;
  static std::unordered_map<TmapKey, CUtensorMap, TmapKeyHash> cache;
  if (rank < 2 || rank > 3) return fail(B200_EINVAL, "get_tmap: rank %d unsupported", rank);
  int dev = 0;
  cudaGetDevice(&dev);
  TmapKey key;
  memset(&key, 0, sizeof(key));
  key.w[0] = reinterpret_cast<uint64_t>(base);
  key.w[1] = (static_cast<uint64_t>(rank) << 32) | (static_cast<uint64_t>(dtype) << 16) |
             (static_cast<uint64_t>(swizzle) << 8) | static_cast<uint64_t>(dev);
  for (int i = 0; i < rank; ++i) { key.w[2 + i] = dims[i]; key.w[8 + i] = box[i]; }
  for (int i = 0; i < rank - 1; ++i) key.w[5 + i] = strides_bytes[i];
  {
    std::lock_guard<std::mutex> g(mu);
    auto it = cache.find(key);
    if (it != cache.end()) { *out = it->second; return 0; }
  }
  EncodeTiledFn fn = encode_fn();
  if (!fn) return fail(B200_ECUDA, "cuTensorMapEncodeTiled entry point not available (no driver?)");
  if ((reinterpret_cast<uint64_t>(base) & 15u) != 0)
    return fail(B200_EINVAL, "tensor base address %p is not 16-byte aligned", base);
  cuuint64_t gdim[3];
  cuuint64_t gstr[2];
  cuuint32_t bdim[3];
  cuuint32_t estr[3] = {1, 1, 1};
  for (int i = 0; i < rank; ++i) { gdim[i] = dims[i]; bdim[i] = box[i]; }
  for (int i = 0; i < rank - 1; ++i) {
    gstr[i] = strides_bytes[i];
    if (gstr[i] % 16 != 0)
      return fail(B200_EINVAL, "tensor stride %llu B is not a multiple of 16",
                  static_cast<unsigned long long>(gstr[i]));
  }
  CUresult r = fn(out, dtype, static_cast<cuuint32_t>(rank),
                  const_cast<void*>(base), gdim, gstr, bdim, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return fail(B200_ECUDA,
                "cuTensorMapEncodeTiled failed with CUresult %d (rank %d dims %llu,%llu,%llu box "
                "%u,%u,%u)",
                static_cast<int>(r), rank, static_cast<unsigned long long>(dims[0]),
                static_cast<unsigned long long>(dims[1]),
                static_cast<unsigned long long>(rank > 2 ? dims[2] : 0), box[0], box[1],
                rank > 2 ? box[2] : 0);
  {
    std::lock_guard<std::mutex> g(mu);
    if (cache.size() > 4096) cache.clear();
    cache.emplace(key, *out);
  }
  return 0;
}

}  // namespace host
}  // namespace b200

extern "C" {
int b200_version(void) { return 2000; }
const char* b200_last_error(void) { return b200::host::last_error_buf(); }
uint64_t b200_launch_count(void);
}

// defined here so the atomic stays file-local
namespace b200 { namespace host { uint64_t launches_now() { return g_launches.load(); } } }
extern "C" uint64_t b200_launch_count(void) { return b200::host::launches_now(); }
