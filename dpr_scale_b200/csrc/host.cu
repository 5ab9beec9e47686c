// Host plumbing shared by the kernel files: the thread-local error string, the launch counter, the SM count and the one
// TMA tensor-map encoder, plus the C entry points that report them.
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include "common.cuh"
#include "dprb_internal.h"

namespace dprb {

static thread_local char g_err[1024] = "";

void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

static std::atomic<long long> g_launches{0};
void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

int num_sms() {
  static std::atomic<int> cached{0};
  int n = cached.load(std::memory_order_relaxed);
  if (n > 0) return n;
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
  if (e != cudaSuccess || n <= 0) {
    set_last_error("SM count query failed: CUDA error %d (%s)", (int)e, cudaGetErrorString(e));
    return -1;
  }
  cached.store(n, std::memory_order_relaxed);
  return n;
}

namespace {
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
}  // namespace

int encode_tmap(CUtensorMap* out, const char* what, CUtensorMapDataType dtype, int rank, const void* base,
                const cuuint64_t* dims, const cuuint64_t* strides, const cuuint32_t* box,
                CUtensorMapL2promotion l2) {
  // cuTensorMapEncodeTiled is a DRIVER call: it needs a current context on the calling thread.  Entry points may be
  // called from any host thread (autograd runs backward on its own), where this may be the first CUDA call of any
  // kind - bind the primary context first.
  static thread_local bool ctx_bound = false;
  if (!ctx_bound) {
    DPRB_CHECK_CUDA(cudaFree(nullptr));
    ctx_bound = true;
  }
  static const EncodeTiledFn fn = []() -> EncodeTiledFn {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) != cudaSuccess ||
        qres != cudaDriverEntryPointSuccess)
      return nullptr;
    return reinterpret_cast<EncodeTiledFn>(ptr);
  }();
  DPRB_REQUIRE(fn != nullptr, "cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
  const cuuint32_t estr[3] = {1u, 1u, 1u};
  const CUresult r = fn(out, dtype, (cuuint32_t)rank, const_cast<void*>(base), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, l2,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  DPRB_REQUIRE(r == CUDA_SUCCESS, "%s: cuTensorMapEncodeTiled failed with CUresult %d (dims %llu x %llu x %llu)",
               what, (int)r, (unsigned long long)dims[0], (unsigned long long)dims[1],
               (unsigned long long)(rank == 3 ? dims[2] : 1));
  return 0;
}

}  // namespace dprb

extern "C" int dprb_version(void) { return DPRB_VERSION; }
extern "C" const char* dprb_last_error(void) { return dprb::g_err; }
extern "C" int dprb_num_sms(void) { return dprb::num_sms(); }
extern "C" int64_t dprb_launch_count(void) { return dprb::g_launches.load(std::memory_order_relaxed); }
