// seedx-b200: shared device helpers (sm_90a).
// Raw PTX wrappers for mbarrier / TMA / clusters + small math utilities (warpgroup MMA: wgmma.cuh).
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#define SEEDX_DEVINL __device__ __forceinline__

namespace seedx {

// ----------------------------------------------------------------------------------------------
// error plumbing (host)
// ----------------------------------------------------------------------------------------------
void set_error(const char* fmt, ...);
int check_cuda(cudaError_t e, const char* what);

// ---- programmatic dependent launch (PDL).  Every kernel of this library is launched through launch_k() with the
// programmatic-stream-serialization attribute and begins its data-dependent part with pdl_wait(): a kernel's launch latency and
// prologue (barrier init, descriptor prefetch, weight prefetch) then overlap the tail of its predecessor, in
// eager streams and inside captured CUDA graphs alike.  seedx_set_pdl(0) (or SEEDX_PDL=0) turns the attribute off.
int pdl_enabled();
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;\n" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;\n" ::: "memory"); }
template <typename... KA, typename... A>
static inline cudaError_t launch_k(void (*kernel)(KA...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, A&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid, cfg.blockDim = block, cfg.dynamicSmemBytes = smem, cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KA>(args)...);
}

#define SEEDX_CUDA(x)                                          \
  do {                                                         \
    int _e = ::seedx::check_cuda((x), #x);                     \
    if (_e) return _e;                                         \
  } while (0)
#define SEEDX_REQUIRE(cond, ...)                               \
  do {                                                         \
    if (!(cond)) {                                             \
      ::seedx::set_error(__VA_ARGS__);                         \
      return 2;                                                \
    }                                                          \
  } while (0)

int num_sms();
// cuTensorMapEncodeTiled through cudaGetDriverEntryPoint (no link-time libcuda dependency)
int encode_tmap(CUtensorMap* map, CUtensorMapDataType dt, uint32_t rank, const void* gptr,
                const uint64_t* dims, const uint64_t* strides_bytes /*rank-1*/, const uint32_t* box,
                CUtensorMapSwizzle swz);

// ----------------------------------------------------------------------------------------------
// device: misc
// ----------------------------------------------------------------------------------------------
SEEDX_DEVINL uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
SEEDX_DEVINL uint32_t lane_id() { return threadIdx.x & 31; }
SEEDX_DEVINL bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}

// ----------------------------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------------------------
SEEDX_DEVINL void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(bar), "r"(count));
}
SEEDX_DEVINL void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory"); }
SEEDX_DEVINL void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(bar), "r"(bytes) : "memory");
}
SEEDX_DEVINL void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(bar) : "memory");
}
SEEDX_DEVINL bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}\n"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
SEEDX_DEVINL void mbar_wait(uint32_t bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}
// for waiters that are NOT on the critical path (epilogue warps parked during a main loop): back off so the polling does not
// steal issue slots / barrier-unit bandwidth from the TMA and MMA issuing threads that share the SM sub-partitions
SEEDX_DEVINL void mbar_wait_relaxed(uint32_t bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) __nanosleep(128);
}

// ----------------------------------------------------------------------------------------------
// TMA (cp.async.bulk.tensor) loads, mbarrier completion
// ----------------------------------------------------------------------------------------------
SEEDX_DEVINL void tma_prefetch_desc(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];\n" ::"l"(tmap) : "memory");
}
SEEDX_DEVINL void tma_load_3d(uint32_t dst, const void* tmap, uint32_t bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];\n" ::
          "r"(dst),
      "l"(tmap), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
SEEDX_DEVINL void tma_load_4d(uint32_t dst, const void* tmap, uint32_t bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], "
      "[%2];\n" ::"r"(dst),
      "l"(tmap), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}


// ---- TMA stores (shared -> global), bulk async groups, proxy fence ---------------------------------
SEEDX_DEVINL void tma_store_3d(const void* tmap, uint32_t src, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];\n" ::"l"(tmap), "r"(src), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
SEEDX_DEVINL void bulk_commit() { asm volatile("cp.async.bulk.commit_group;\n" ::: "memory"); }
template <int N>
SEEDX_DEVINL void bulk_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;\n" ::"n"(N) : "memory");
}
SEEDX_DEVINL void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory"); }
SEEDX_DEVINL uint4 lds128(uint32_t a) {
  uint4 v;
  asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];\n" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a));
  return v;
}
SEEDX_DEVINL void sts128(uint32_t a, uint4 v) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};\n" ::"r"(a), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// ---- thread-block clusters -----------------------------------------------------------------------
SEEDX_DEVINL uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;\n" : "=r"(r));
  return r;
}
SEEDX_DEVINL void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;\n" ::: "memory");
}
// address of the same shared-memory offset in CTA `rank` of this cluster (shared::cluster window)
SEEDX_DEVINL uint32_t mapa_cluster(uint32_t saddr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;\n" : "=r"(r) : "r"(saddr), "r"(rank));
  return r;
}
SEEDX_DEVINL void mbar_arrive_cluster(uint32_t cluster_addr) {
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];\n" ::"r"(cluster_addr) : "memory");
}
// TMA load delivered to the same shared-memory offset of every CTA in `mask`; each destination's mbarrier at `bar` receives its bytes
SEEDX_DEVINL void tma_load_3d_mc(uint32_t dst, const void* tmap, uint32_t bar, int c0, int c1, int c2, uint16_t mask) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4, %5}], [%2], %6;\n" ::"r"(dst),
      "l"(tmap), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "h"(mask)
      : "memory");
}

// ---- register budget of warp-specialised kernels (warpgroup-wide)
template <int N>
SEEDX_DEVINL void setmaxnreg_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;\n" ::"n"(N));
}
template <int N>
SEEDX_DEVINL void setmaxnreg_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;\n" ::"n"(N));
}
// named barrier over `threads` threads (warp multiples)
SEEDX_DEVINL void named_bar_sync(int id, int threads) { asm volatile("bar.sync %0, %1;\n" ::"r"(id), "r"(threads) : "memory"); }
SEEDX_DEVINL float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;\n" : "=f"(y) : "f"(x));
  return y;
}


// ----------------------------------------------------------------------------------------------
// math
// ----------------------------------------------------------------------------------------------
SEEDX_DEVINL float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }
// exact-GELU with erf from Abramowitz-Stegun 7.1.26 (|abs err| <= 1.5e-7, far below the fp16 output rounding); ~3x cheaper than erff
SEEDX_DEVINL float rcp_approx(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;\n" : "=f"(y) : "f"(x));
  return y;
}
// exact (erf) GELU in 9 FP32 issue slots + 1 MUFU per value — the GEGLU epilogue of the UNet feed-forward GEMMs is issue-bound on this function
// (round 1 used Abramowitz-Stegun 7.1.26: 15 FP32 + 2 MUFU).  erf(t) = 1 - 2^(-q(t)) for t >= 0 with q a degree-5 polynomial without constant
// term, fitted to -log2(erfc(t)) on [0, 4.3] (max |error| of erf 8.6e-7, monotone beyond: 2^-q underflows to 0 = erf saturates at 1), so
//   gelu(x) = 0.5 x (1 + erf(x / sqrt 2)) = max(x, 0) - 0.5 |x| 2^(-q(|x| / sqrt 2)).
SEEDX_DEVINL float gelu_erf_fast(float x) {
  const float t = fabsf(x) * 0.70710678118654752440f;
  float q = fmaf(t, 0.0030152f, -0.02984835f);
  q = fmaf(q, t, 0.14897545f);
  q = fmaf(q, t, 0.9183691f);
  q = fmaf(q, t, 1.627908f);
  q *= t;
  const float e = fast_exp2(-q);
  return fmaf(-0.5f * fabsf(x), e, fmaxf(x, 0.f));
}
SEEDX_DEVINL float silu(float x) { return x * rcp_approx(1.0f + fast_exp2(-1.4426950408889634f * x)); }

SEEDX_DEVINL float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
SEEDX_DEVINL float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

}  // namespace seedx
