// seedx-b200: wgmma flash attention (forward) for sm_90a.
//
//   O[b,h,i,:] = softmax_j( scale * Q[b,h,i,:] . K[b,h,j,:]  (+ causal mask) ) V[b,h,j,:]
//
// One CTA = 128 query rows of one (batch, head): warpgroups 0 and 1 own 64 rows each, warp 8 is the TMA producer.  Q, K and V arrive by TMA
// as 128B-swizzled tiles of 64 head-dim columns (a head dim below 64 / 128 is zero-filled by the tensor map); K/V tiles of BN keys go
// through a two-stage mbarrier ring.  Per key tile a warpgroup computes S = Q K^T with wgmma (operands in shared memory, S in registers),
// the online softmax in registers, and O += P V with P as the register A operand and V read MN-major from shared memory.
//
// Replaces the same call sites as attention.cu (its mma.sync kernel takes what this kernel does not: head dim > 128, fewer than 64 queries).
#include <math.h>

#include "common.cuh"
#include "wgmma.cuh"
#include "../../include/seedx.h"

namespace seedx {

struct WgParams {
  __half* o;
  long long o_sb, o_sh, o_ss;
  int sq, sk, d;
  float scale_log2;
  int causal, q_batched;
};

SEEDX_DEVINL uint32_t pack_half2_u32(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *(uint32_t*)&h;
}

constexpr int WG_BM = 128;
constexpr int WG_KS = 2;           // K/V pipeline stages
constexpr int WG_THREADS = 288;    // 2 consumer warpgroups + 1 producer warp

template <int DP, int BN>
struct WgCfg {
  static constexpr int DC = DP / 64;                   // 64-column chunks of the head dim
  static constexpr int Q_CHUNK = WG_BM * 128;          // bytes of one Q column chunk
  static constexpr int KV_CHUNK = BN * 128;            // bytes of one K (or V) column chunk
  static constexpr int Q_BYTES = DC * Q_CHUNK;
  static constexpr int KV_BYTES = DC * KV_CHUNK;
  static constexpr int SMEM_BYTES = Q_BYTES + WG_KS * 2 * KV_BYTES + 1024;   // + barriers
};

template <int DP, int BN>
__global__ void __launch_bounds__(WG_THREADS, 1)
flash_attn_wg_kernel(const __grid_constant__ CUtensorMap tq, const __grid_constant__ CUtensorMap tk, const __grid_constant__ CUtensorMap tv,
                     const WgParams p) {
  using Cfg = WgCfg<DP, BN>;
  extern __shared__ __align__(1024) uint8_t smem[];
  const uint32_t base = smem_u32(smem);
  if ((base & 1023u) != 0u) __trap();
  const uint32_t sQ = base;
  auto sK = [&](int s) { return base + Cfg::Q_BYTES + (uint32_t)(2 * s) * Cfg::KV_BYTES; };
  auto sV = [&](int s) { return base + Cfg::Q_BYTES + (uint32_t)(2 * s + 1) * Cfg::KV_BYTES; };
  const uint32_t bar = base + Cfg::Q_BYTES + 2 * WG_KS * Cfg::KV_BYTES;
  const uint32_t q_full = bar;
  auto kv_full = [&](int s) { return bar + 8u * (1 + s); };
  auto kv_empty = [&](int s) { return bar + 8u * (1 + WG_KS + s); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m0 = blockIdx.x * WG_BM;
  const int h = blockIdx.y, b = blockIdx.z;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tq);
    tma_prefetch_desc(&tk);
    tma_prefetch_desc(&tv);
    mbar_init(q_full, 1);
    for (int s = 0; s < WG_KS; ++s) {
      mbar_init(kv_full(s), 1);
      mbar_init(kv_empty(s), 2);   // one arrival per consumer warpgroup
    }
    mbar_fence_init();
  }
  __syncthreads();
  pdl_wait();
  pdl_trigger();

  int n_tiles = (p.sk + BN - 1) / BN;
  const int causal_off = p.sk - p.sq;  // key j visible to query i iff j <= i + causal_off
  if (p.causal) {
    const int last = m0 + WG_BM - 1 + causal_off;  // last visible key of this row block
    const int lim = last < 0 ? 1 : last / BN + 1;
    if (lim < n_tiles) n_tiles = lim;
  }

  if (warp == 8) {
    // ------------------------------------------------ TMA producer
    if (lane == 0) {
      const int qb = p.q_batched ? b : 0;
      mbar_expect_tx(q_full, Cfg::Q_BYTES);
      for (int c = 0; c < Cfg::DC; ++c) tma_load_4d(sQ + c * Cfg::Q_CHUNK, &tq, q_full, 64 * c, m0, h, qb);
      for (int j = 0; j < n_tiles; ++j) {
        const int s = j % WG_KS;
        mbar_wait(kv_empty(s), ((j / WG_KS) & 1) ^ 1u);
        mbar_expect_tx(kv_full(s), 2 * Cfg::KV_BYTES);
        for (int c = 0; c < Cfg::DC; ++c) {
          tma_load_4d(sK(s) + c * Cfg::KV_CHUNK, &tk, kv_full(s), 64 * c, j * BN, h, b);
          tma_load_4d(sV(s) + c * Cfg::KV_CHUNK, &tv, kv_full(s), 64 * c, j * BN, h, b);
        }
      }
    }
    return;
  }

  // ------------------------------------------------ consumer warpgroups
  const int wg = warp >> 2, q = warp & 3;
  const int qrow0 = m0 + 64 * wg + 16 * q + (lane >> 2);  // this thread's rows: qrow0 and qrow0 + 8
  float o_acc[DP / 2];
#pragma unroll
  for (int i = 0; i < DP / 2; ++i) o_acc[i] = 0.f;
  float s_acc[BN / 2];
  float row_max[2] = {-INFINITY, -INFINITY};
  float row_sum[2] = {0.f, 0.f};
  mbar_wait(q_full, 0);

  for (int j = 0; j < n_tiles; ++j) {
    const int s = j % WG_KS;
    mbar_wait(kv_full(s), (j / WG_KS) & 1);
    // ---- S = Q K^T (64 x BN per warpgroup)
    wgmma_fence_regs<BN / 2>(s_acc);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < DP / 16; ++ks) {
      const uint32_t koff = (uint32_t)((ks & 3) * 32);   // 16 fp16 = 32 B inside the 128B swizzle atom
      const uint64_t ad = wgmma_desc_k_sw128(sQ + (ks >> 2) * Cfg::Q_CHUNK + wg * 64 * 128 + koff);
      const uint64_t bd = wgmma_desc_k_sw128(sK(s) + (ks >> 2) * Cfg::KV_CHUNK + koff);
      wgmma_ss_n<BN>(s_acc, ad, bd, ks != 0);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs<BN / 2>(s_acc);

    // ---- mask + online softmax (base 2); a row's values are spread over the 4 lanes of a quad
    const int col_base = j * BN + (lane & 3) * 2;
    const bool need_mask = (j * BN + BN > p.sk) || (p.causal && (j * BN + BN - 1 > m0 + 64 * wg + causal_off));
    float tmax[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int g = 0; g < BN / 8; ++g) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float v = s_acc[4 * g + e] * p.scale_log2;
        if (need_mask) {
          const int col = col_base + g * 8 + (e & 1);
          const int row = qrow0 + (e >> 1) * 8;
          if (col >= p.sk || (p.causal && col > row + causal_off)) v = -INFINITY;
        }
        s_acc[4 * g + e] = v;
        tmax[e >> 1] = fmaxf(tmax[e >> 1], v);
      }
    }
    float corr[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      tmax[r] = fmaxf(tmax[r], __shfl_xor_sync(0xffffffffu, tmax[r], 1));
      tmax[r] = fmaxf(tmax[r], __shfl_xor_sync(0xffffffffu, tmax[r], 2));
      const float nm = fmaxf(row_max[r], tmax[r]);
      const float bse = (nm == -INFINITY) ? 0.f : nm;  // fully masked row so far
      corr[r] = exp2f(row_max[r] - bse);               // row_max = -inf -> 0
      row_max[r] = nm;
      tmax[r] = bse;
      row_sum[r] *= corr[r];
    }
    float psum[2] = {0.f, 0.f};
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) {
      const float pv = exp2f(s_acc[i] - tmax[(i >> 1) & 1]);
      s_acc[i] = pv;
      psum[(i >> 1) & 1] += pv;
    }
    row_sum[0] += psum[0];
    row_sum[1] += psum[1];
#pragma unroll
    for (int i = 0; i < DP / 2; ++i) o_acc[i] *= corr[(i >> 1) & 1];

    // ---- O += P V: P (fp16) is the A operand straight from registers, 16 keys per instruction.  Every fragment is packed BEFORE the
    // wgmma.fence (a register an in-flight wgmma reads must not be written after the fence) and stays live until the wait below, so that
    // no fragment register is reused while an asynchronous wgmma may still be reading it.
    uint32_t pa[BN / 16][4];
#pragma unroll
    for (int kk = 0; kk < BN / 16; ++kk) {
      pa[kk][0] = pack_half2_u32(s_acc[8 * kk + 0], s_acc[8 * kk + 1]);
      pa[kk][1] = pack_half2_u32(s_acc[8 * kk + 2], s_acc[8 * kk + 3]);
      pa[kk][2] = pack_half2_u32(s_acc[8 * kk + 4], s_acc[8 * kk + 5]);
      pa[kk][3] = pack_half2_u32(s_acc[8 * kk + 6], s_acc[8 * kk + 7]);
    }
    wgmma_fence_regs<DP / 2>(o_acc);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < BN / 16; ++kk) wgmma_rs_tb<DP>(o_acc, pa[kk], wgmma_desc_mn_sw128(sV(s) + kk * 16 * 128, Cfg::KV_CHUNK), 1);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs<DP / 2>(o_acc);
#pragma unroll
    for (int kk = 0; kk < BN / 16; ++kk)
#pragma unroll
      for (int i = 0; i < 4; ++i) asm volatile("" : "+r"(pa[kk][i])::"memory");
    if ((threadIdx.x & 127) == 0) mbar_arrive(kv_empty(s));
  }

  // ---- finalise: O /= row_sum, write fp16
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    row_sum[r] += __shfl_xor_sync(0xffffffffu, row_sum[r], 1);
    row_sum[r] += __shfl_xor_sync(0xffffffffu, row_sum[r], 2);
  }
  const float inv0 = row_sum[0] > 0.f ? 1.f / row_sum[0] : 0.f;
  const float inv1 = row_sum[1] > 0.f ? 1.f / row_sum[1] : 0.f;
  __half* og = p.o + b * p.o_sb + h * p.o_sh;
#pragma unroll
  for (int g = 0; g < DP / 8; ++g) {
    const int col = g * 8 + (lane & 3) * 2;
    if (col < p.d) {
      if (qrow0 < p.sq) *(__half2*)(og + (long long)qrow0 * p.o_ss + col) = __floats2half2_rn(o_acc[4 * g] * inv0, o_acc[4 * g + 1] * inv0);
      if (qrow0 + 8 < p.sq)
        *(__half2*)(og + (long long)(qrow0 + 8) * p.o_ss + col) = __floats2half2_rn(o_acc[4 * g + 2] * inv1, o_acc[4 * g + 3] * inv1);
    }
  }
}

void count_launch();

template <int DP, int BN>
static int launch_wg(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, const WgParams& p, int B, int H, cudaStream_t st) {
  using Cfg = WgCfg<DP, BN>;
  static bool attr = false;
  if (!attr) {
    SEEDX_CUDA(cudaFuncSetAttribute(flash_attn_wg_kernel<DP, BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    attr = true;
  }
  dim3 grid((p.sq + WG_BM - 1) / WG_BM, H, B);
  const cudaError_t e = launch_k(flash_attn_wg_kernel<DP, BN>, grid, WG_THREADS, Cfg::SMEM_BYTES, st, tq, tk, tv, p);
  count_launch();
  return check_cuda(e != cudaSuccess ? e : cudaGetLastError(), "flash_attn_wg_kernel launch");
}

static int make_map_wg(CUtensorMap* m, const void* ptr, int d, int s, int H, int B, long long ss, long long sh, long long sb, int rows) {
  uint64_t dims[4] = {(uint64_t)d, (uint64_t)s, (uint64_t)H, (uint64_t)B};
  uint64_t strides[3] = {(uint64_t)ss * 2, (uint64_t)(H > 1 ? sh : ss * s) * 2, (uint64_t)(B > 1 ? sb : ss * s) * 2};
  uint32_t box[4] = {64, (uint32_t)rows, 1, 1};
  return encode_tmap(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, ptr, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
}

// returns -1 when the problem is not eligible (the caller then runs the mma.sync kernel)
int attention_wg_try(const seedx_attn_args* a, cudaStream_t st) {
  if (a->d > 128 || a->d % 8 != 0 || a->sq < 64 || a->sk < 16 || !(a->scale > 0.f)) return -1;
  const long long str[] = {a->q_stride_s, a->q_stride_h, a->q_stride_b, a->k_stride_s, a->k_stride_h, a->k_stride_b,
                           a->v_stride_s, a->v_stride_h, a->v_stride_b};
  for (long long s : str)
    if (s % 8 != 0 || s < 0) return -1;
  if (a->q_stride_s == 0 || a->k_stride_s == 0 || a->v_stride_s == 0) return -1;
  if ((a->heads > 1 && (a->q_stride_h == 0 || a->k_stride_h == 0 || a->v_stride_h == 0)) ||
      (a->batch > 1 && (a->k_stride_b == 0 || a->v_stride_b == 0)))
    return -1;
  const bool qb = !(a->batch > 1 && a->q_stride_b == 0);
  const int bn = a->sk <= 64 ? 64 : 128;
  CUtensorMap tq, tk, tv;
  if (make_map_wg(&tq, a->q, a->d, a->sq, a->heads, qb ? a->batch : 1, a->q_stride_s, a->q_stride_h, a->q_stride_b, WG_BM)) return -1;
  if (make_map_wg(&tk, a->k, a->d, a->sk, a->heads, a->batch, a->k_stride_s, a->k_stride_h, a->k_stride_b, bn)) return -1;
  if (make_map_wg(&tv, a->v, a->d, a->sk, a->heads, a->batch, a->v_stride_s, a->v_stride_h, a->v_stride_b, bn)) return -1;
  WgParams p;
  p.o = (__half*)a->o;
  p.o_sb = a->o_stride_b, p.o_sh = a->o_stride_h, p.o_ss = a->o_stride_s;
  p.sq = a->sq, p.sk = a->sk, p.d = a->d;
  p.scale_log2 = a->scale * 1.4426950408889634f;
  p.causal = a->causal;
  p.q_batched = qb ? 1 : 0;
  if (a->d <= 64) return bn == 64 ? launch_wg<64, 64>(tq, tk, tv, p, a->batch, a->heads, st) : launch_wg<64, 128>(tq, tk, tv, p, a->batch, a->heads, st);
  return bn == 64 ? launch_wg<128, 64>(tq, tk, tv, p, a->batch, a->heads, st) : launch_wg<128, 128>(tq, tk, tv, p, a->batch, a->heads, st);
}

}  // namespace seedx
