// Host-side plumbing shared by every translation unit of libao_b200.so:
// error reporting, tensor-map encoding (driver entry point fetched at run time so the
// library does not link libcuda), launch helper with the PDL attribute, launch counter.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>

#include <atomic>

#include "../../include/ao_b200.h"

namespace ao {

char* error_buffer();  // thread-local, 512 bytes
inline int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(error_buffer(), 512, fmt, ap);
  va_end(ap);
  return code;
}

#define AO_CUDA_CHECK(expr)                                                              \
  do {                                                                                   \
    cudaError_t _e = (expr);                                                             \
    if (_e != cudaSuccess)                                                               \
      return ::ao::fail(AO_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), \
                        __FILE__, __LINE__);                                             \
  } while (0)

#define AO_REQUIRE(cond, ...)                                       \
  do {                                                              \
    if (!(cond)) return ::ao::fail(AO_ERR_INVALID_ARG, __VA_ARGS__); \
  } while (0)

extern std::atomic<uint64_t> g_launch_count;

// Encode a tiled tensor map.  dims/box innermost-first; strides in bytes for dims 1..rank-1.
int make_tmap(CUtensorMap* out, CUtensorMapDataType dtype, int rank, const void* gaddr,
              const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box,
              CUtensorMapSwizzle swizzle);

// Launch with optional programmatic-dependent-launch attribute.
template <typename... KArgs, typename... Args>
inline cudaError_t launch(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem,
                          cudaStream_t stream, bool pdl, Args... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  g_launch_count.fetch_add(1, std::memory_order_relaxed);
  return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

inline int ceil_div(int a, int b) { return (a + b - 1) / b; }

// cudaFuncAttributeMaxDynamicSharedMemorySize is a per-device property of a kernel: set it once per (kernel, device).
cudaError_t ensure_dynamic_smem(const void* kernel, size_t bytes);

// PDL can be disabled globally (AO_B200_NO_PDL=1) for debugging.
bool pdl_enabled();
int ts_min_units();    // AO_B200_TS_MIN_UNITS: minimum chunks per CTA of ts_gemm.cuh grids, 0 = by problem size
int sm_count();

}  // namespace ao
