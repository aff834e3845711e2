#include <cstdlib>
// seedx-b200: host-side runtime glue of libseedx.so (error string, SM count, tensor-map encoder, launch counter).
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <mutex>

#include "common.cuh"
#include "../../include/seedx.h"

namespace seedx {

static thread_local char g_err[512] = "";
static std::atomic<long long> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int check_cuda(cudaError_t e, const char* what) {
  if (e == cudaSuccess) return 0;
  set_error("CUDA error %d (%s) at %s", (int)e, cudaGetErrorString(e), what);
  return 1;
}

static std::atomic<int> g_pdl{-1};
int pdl_enabled() {
  int v = g_pdl.load(std::memory_order_relaxed);
  if (v < 0) {
    const char* e = getenv("SEEDX_PDL");
    v = (e && e[0] == '0') ? 0 : 1;
    g_pdl.store(v);
  }
  return v;
}
void set_pdl(int on) { g_pdl.store(on ? 1 : 0); }
void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaDeviceProp prop;
    if (cudaGetDevice(&dev) == cudaSuccess && cudaGetDeviceProperties(&prop, dev) == cudaSuccess)
      n = prop.multiProcessorCount;
    else
      n = 132;
  }
  return n;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
  });
  return fn;
}

int encode_tmap(CUtensorMap* map, CUtensorMapDataType dt, uint32_t rank, const void* gptr, const uint64_t* dims,
                const uint64_t* strides_bytes, const uint32_t* box, CUtensorMapSwizzle swz) {
  EncodeTiledFn fn = get_encode();
  if (!fn) {
    set_error("cuTensorMapEncodeTiled is unavailable (no CUDA driver?)");
    return 3;
  }
  cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  CUresult r = fn(map, dt, rank, const_cast<void*>(gptr), (const cuuint64_t*)dims, (const cuuint64_t*)strides_bytes,
                  (const cuuint32_t*)box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (%d): rank=%u dims=[%llu,%llu,%llu] stride0=%llu box=[%u,%u,%u] ptr=%p",
              (int)r, rank, (unsigned long long)dims[0], (unsigned long long)dims[1],
              (unsigned long long)(rank > 2 ? dims[2] : 0), (unsigned long long)strides_bytes[0], box[0], box[1],
              rank > 2 ? box[2] : 0, gptr);
    return 4;
  }
  return 0;
}

}  // namespace seedx

extern "C" const char* seedx_last_error(void) { return seedx::g_err; }
extern "C" int seedx_abi_version(void) { return SEEDX_ABI_VERSION; }
extern "C" int seedx_set_pdl(int on) {
  seedx::set_pdl(on);
  return 0;
}
extern "C" int64_t seedx_launch_count(void) { return (int64_t)seedx::g_launches.load(); }
