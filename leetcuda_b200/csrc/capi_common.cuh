// capi_common.cuh — host-side helpers shared by the C-ABI translation units:
// error text, launch counter, driver entry point for cuTensorMapEncodeTiled
// (resolved at run time so the library loads on a machine without libcuda),
// and a small cache of encoded tensor maps.
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
