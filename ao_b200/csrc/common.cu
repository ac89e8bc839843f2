#include "common.h"

#include <stdlib.h>
#include <string.h>

#include <mutex>
#include <set>
#include <utility>

namespace ao {

char* error_buffer() {
  static thread_local char buf[512] = {0};
  return buf;
}

std::atomic<uint64_t> g_launch_count{0};

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) ==
            cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

int make_tmap(CUtensorMap* out, CUtensorMapDataType dtype, int rank, const void* gaddr,
              const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box,
              CUtensorMapSwizzle swizzle) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return fail(AO_ERR_CUDA, "cuTensorMapEncodeTiled driver entry point unavailable");
  cuuint64_t gdims[5];
  cuuint64_t gstr[4];
  cuuint32_t gbox[5];
  cuuint32_t estr[5];
  for (int i = 0; i < rank; ++i) {
    gdims[i] = dims[i];
    gbox[i] = box[i];
    estr[i] = 1;
  }
  for (int i = 0; i + 1 < rank; ++i) gstr[i] = strides_bytes[i];
  CUresult r = fn(out, dtype, (cuuint32_t)rank, const_cast<void*>(gaddr), gdims, gstr, gbox, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return fail(AO_ERR_CUDA,
                "cuTensorMapEncodeTiled failed (CUresult %d) rank=%d dims=[%llu,%llu,%llu] "
                "box=[%u,%u,%u]",
                (int)r, rank, (unsigned long long)dims[0],
                (unsigned long long)(rank > 1 ? dims[1] : 0),
                (unsigned long long)(rank > 2 ? dims[2] : 0), box[0], rank > 1 ? box[1] : 0,
                rank > 2 ? box[2] : 0);
  return AO_OK;
}

cudaError_t ensure_dynamic_smem(const void* kernel, size_t bytes) {
  static std::mutex mu;
  static std::set<std::pair<const void*, int>> done;
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  std::lock_guard<std::mutex> lock(mu);
  if (done.count({kernel, dev})) return cudaSuccess;
  e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  // the whole unified memory as shared memory: a CTA of the next kernel (PDL) can only join an SM whose current
  // shared-memory carve-out has room for it, so every such kernel asks for the same (largest) one
  if (e == cudaSuccess)
    e = cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
  if (e == cudaSuccess) done.insert({kernel, dev});
  return e;
}

bool pdl_enabled() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("AO_B200_NO_PDL");
    v = (e && e[0] == '1') ? 0 : 1;
  }
  return v == 1;
}

// test-only override of the stream-K grid (ao_b200_debug_set_streamk_ctas); 0 = the heuristic of launch_gemm
static std::atomic<int> g_streamk_ctas{0};
int streamk_ctas_override() { return g_streamk_ctas.load(std::memory_order_relaxed); }

int sm_count() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    cudaDeviceProp p;
    if (cudaGetDeviceProperties(&p, dev) != cudaSuccess) return 132;
    n = p.multiProcessorCount;
  }
  return n;
}

}  // namespace ao

extern "C" {

int ao_b200_version(void) { return 100; }

const char* ao_b200_last_error(void) { return ao::error_buffer(); }

int ao_b200_device_ok(void) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 0;
  cudaDeviceProp p;
  if (cudaGetDeviceProperties(&p, dev) != cudaSuccess) return 0;
  return (p.major == 9 && p.minor == 0) ? 1 : 0;
}

size_t ao_b200_workspace_bytes(int M, int N) {
  (void)M;
  (void)N;
  // the split-tile flags (64 KiB), then at most (SM count) x 128 x 128 32-bit words of stream-K partials, then (the
  // block-scaled linears, from the next MiB on) the bf16 activation slab: as many rows as fit in what is left.
  return (size_t)64 * 1024 + (size_t)24 * 1024 * 1024;
}

uint64_t ao_b200_launch_count(void) { return ao::g_launch_count.load(); }

int ao_b200_debug_set_streamk_ctas(int n) { return ao::g_streamk_ctas.exchange(n > 0 ? n : 0); }

}  // extern "C"
