// capi_common.cuh — host-side helpers shared by the C-ABI translation units:
// error text, launch counter, driver entry point for cuTensorMapEncodeTiled
// (resolved at run time so the library loads on a machine without libcuda),
// a small cache of encoded tensor maps, and the persistent cluster launch of the GEMMs.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <atomic>
#include <mutex>
#include <unordered_map>

#include "../../include/leetcuda_b200.h"

namespace b200 {
namespace host {

char* last_error_buf();  // thread-local, 512 bytes
int fail(int code, const char* fmt, ...);
void count_launch(uint64_t n = 1);

#define B200_CUDA_OK(expr)                                                              \
  do {                                                                                  \
    cudaError_t _e = (expr);                                                            \
    if (_e != cudaSuccess)                                                              \
      return ::b200::host::fail(B200_ECUDA, "%s failed: %s (%s:%d)", #expr,             \
                                cudaGetErrorString(_e), __FILE__, __LINE__);            \
  } while (0)

int sm_count();  // SMs of the current device (cached per device)

// Persistent launch of Kern(args...) in clusters of `cs` CTAs (1 or 2) over num_tiles cluster tiles, with `threads`
// threads and `smem` bytes of dynamic shared memory per CTA.  A cluster of two occupies two SMs of one GPC, so with
// cs = 2 the grid is as many clusters as fit the GPU at once (cached per device), not #SMs / 2: a GPC with an odd
// number of SMs then leaves one SM idle instead of running a cluster in a second wave.  who prefixes the error.
template <auto Kern, typename... Args>
int launch_persistent(const char* who, int threads, int smem, int num_tiles, int cs, cudaStream_t stream,
                      const Args&... args) {
  static bool attr_set[64] = {false};
  static int max_clusters[64] = {0};
  int dev = 0;
  cudaGetDevice(&dev);
  const bool cached = dev >= 0 && dev < 64;
  if (!cached || !attr_set[dev]) {
    B200_CUDA_OK(cudaFuncSetAttribute(Kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    if (cached) attr_set[dev] = true;
  }
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.blockDim = dim3(threads, 1, 1);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attrs[1];
  attrs[0].id = cudaLaunchAttributeClusterDimension;
  attrs[0].val.clusterDim.x = static_cast<unsigned>(cs);
  attrs[0].val.clusterDim.y = 1;
  attrs[0].val.clusterDim.z = 1;
  cfg.attrs = attrs;
  cfg.numAttrs = 1;
  int slots = sm_count();
  if (cs > 1) {
    slots = cached ? max_clusters[dev] : 0;
    if (slots == 0) {
      cfg.gridDim = dim3(static_cast<unsigned>(cs), 1, 1);
      B200_CUDA_OK(cudaOccupancyMaxActiveClusters(&slots, Kern, &cfg));
      if (slots <= 0) return fail(B200_ECUDA, "%s: no cluster of %d CTAs fits the device", who, cs);
      if (cached) max_clusters[dev] = slots;
    }
  }
  const int grid = cs * (num_tiles < slots ? num_tiles : slots);
  cfg.gridDim = dim3(static_cast<unsigned>(grid), 1, 1);
  B200_CUDA_OK(cudaLaunchKernelEx(&cfg, Kern, args...));
  count_launch();
  return 0;
}

// Do the byte ranges [a, a + na) and [b, b + nb) share a byte?
inline bool overlaps(const void* a, size_t na, const void* b, size_t nb) {
  const uintptr_t x = reinterpret_cast<uintptr_t>(a), y = reinterpret_cast<uintptr_t>(b);
  return na != 0 && nb != 0 && x < y + nb && y < x + na;
}

// Copy-engine pipeline of the *_host entry points: one H2D stream, one D2H stream and a pool of
// events per thread and device (created on first use).
constexpr int kPipeEvents = 66;
struct HostPipe {
  cudaStream_t in = nullptr, out = nullptr;
  cudaEvent_t ev[kPipeEvents];
  bool ok = false;
  int dev = -1;
};
int host_pipe(HostPipe** out);

// Cached device workspace of the *_host entry points (per thread and device) of at least `bytes`.
// Growing it frees the old block, so a caller must have drained its previous use.
int workspace(void** out, size_t bytes);

// Encode (or fetch from cache) a tiled tensor map over fp16 (default) or fp32 data.
//   rank 2: dims {d0 (contiguous), d1}, strides_bytes {s1}
//   rank 3: dims {d0, d1, d2},          strides_bytes {s1, s2}
// Returns 0 or a negative error code.
int get_tmap(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
             const uint64_t* strides_bytes, const uint32_t* box, CUtensorMapSwizzle swizzle,
             CUtensorMapDataType dtype = CU_TENSOR_MAP_DATA_TYPE_FLOAT16);

}  // namespace host
}  // namespace b200
