// seedx-b200: fused softmax attention (flash-style, online softmax, no S x S materialisation).
//
//   O[b,h,i,:] = softmax_j( scale * Q[b,h,i,:] . K[b,h,j,:]  (+ causal mask) ) V[b,h,j,:]
//
// fp16 operands, fp32 scores / statistics / accumulation.  One CTA = 64 query rows x one (batch, head); 4 warps,
// 16 rows each; K/V tiles of 64 keys double-buffered through cp.async, mma.sync.m16n8k16.  The wgmma kernel
// (attention_wg.cu) takes every problem it is built for; this one covers the rest (head dim > 128, fewer than 64 queries).
//
// Replaces: src/models/tokenizer/qwen_visual.py:204-215 (ViT MHSA, d=104), :136-146 (nn.MultiheadAttention of the
// Resampler, d=128/160), src/models/mllm/modeling_llama_xformer.py:225-237 (xformers memory_efficient_attention,
// causal prefill, d=128), src/models/detokenizer/resampler.py:62-73, 104-116 (perceiver / pool attention, d=64),
// diffusers AttnProcessor2_0 (UNet self/cross attention, d=64).
#include "common.cuh"
#include "../../include/seedx.h"

namespace seedx {

struct AttnParams {
  const __half* q;
  const __half* k;
  const __half* v;
  __half* o;
  long long q_sb, q_sh, q_ss;  // element strides: batch, head, sequence
  long long k_sb, k_sh, k_ss;
  long long v_sb, v_sh, v_ss;
  long long o_sb, o_sh, o_ss;
  int sq, sk, d;
  float scale_log2;  // scale * log2(e)
  int causal;
};

SEEDX_DEVINL void cp_async16(uint32_t dst, const void* src, bool valid) {
  const int bytes = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(dst), "l"(src), "r"(bytes) : "memory");
}
SEEDX_DEVINL void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N>
SEEDX_DEVINL void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory");
}
SEEDX_DEVINL void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
SEEDX_DEVINL void ldsm_x4_t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];\n"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
SEEDX_DEVINL void mma16816(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
SEEDX_DEVINL uint32_t pack_half2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *(uint32_t*)&h;
}

constexpr int ATT_BM = 64;
constexpr int ATT_BN = 64;

template <int DPAD>
struct AttnSmem {
  static constexpr int LD = DPAD + 8;                                 // padded row (halves): conflict-free ldmatrix
  static constexpr int BYTES = (ATT_BM + 4 * ATT_BN) * LD * 2;        // Q + 2 x (K, V)
};

// copy `rows` x d (valid rows < rows_valid) from global (row stride gs) into smem tile (row stride LD)
template <int DPAD>
SEEDX_DEVINL void load_tile(uint32_t sdst, const __half* g, long long gs, int row0, int rows_valid, int d) {
  constexpr int LD = AttnSmem<DPAD>::LD;
  const int chunks = d >> 3;  // 16-byte chunks per row
  for (int idx = threadIdx.x; idx < 64 * chunks; idx += 128) {
    const int r = idx / chunks;
    const int c = idx - r * chunks;
    const bool ok = (row0 + r) < rows_valid;
    const __half* src = g + (long long)(ok ? (row0 + r) : 0) * gs + c * 8;
    cp_async16(sdst + (uint32_t)(r * LD + c * 8) * 2u, src, ok);
  }
}

template <int DPAD>
__global__ void __launch_bounds__(128) flash_attn_kernel(const AttnParams p) {
  pdl_wait();
  pdl_trigger();
  constexpr int LD = AttnSmem<DPAD>::LD;
  constexpr int KSTEPS = DPAD / 16;  // k16 steps over the head dim
  constexpr int DTILES = DPAD / 8;   // n8 tiles of the output
  extern __shared__ __align__(16) uint8_t smem[];
  const uint32_t sQ = smem_u32(smem);
  const uint32_t sK0 = sQ + ATT_BM * LD * 2;
  const uint32_t sV0 = sK0 + 2 * ATT_BN * LD * 2;
  auto sK = [&](int s) { return sK0 + (uint32_t)s * ATT_BN * LD * 2; };
  auto sV = [&](int s) { return sV0 + (uint32_t)s * ATT_BN * LD * 2; };

  const int m0 = blockIdx.x * ATT_BM;
  const int h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const __half* qg = p.q + b * p.q_sb + h * p.q_sh;
  const __half* kg = p.k + b * p.k_sb + h * p.k_sh;
  const __half* vg = p.v + b * p.v_sb + h * p.v_sh;

  // zero the padding columns [d, DPAD) (+ the 8 pad halves) of every tile once; cp.async never touches them
  if (p.d < DPAD) {
    const int padc = DPAD - p.d;
    __half* s = (__half*)smem;
    for (int idx = threadIdx.x; idx < (ATT_BM + 4 * ATT_BN) * padc; idx += 128) {
      const int r = idx / padc, c = idx - r * padc;
      s[r * LD + p.d + c] = __float2half(0.f);
    }
  }

  int n_tiles = (p.sk + ATT_BN - 1) / ATT_BN;
  const int causal_off = p.sk - p.sq;  // key j visible to query i iff j <= i + causal_off
  if (p.causal) {
    const int last = m0 + ATT_BM - 1 + causal_off;  // last visible key of this row block
    const int lim = last / ATT_BN + 1;
    if (lim < n_tiles) n_tiles = lim < 1 ? 1 : lim;
  }

  load_tile<DPAD>(sQ, qg, p.q_ss, m0, p.sq, p.d);
  load_tile<DPAD>(sK(0), kg, p.k_ss, 0, p.sk, p.d);
  load_tile<DPAD>(sV(0), vg, p.v_ss, 0, p.sk, p.d);
  cp_async_commit();

  float o_acc[DTILES][4];
#pragma unroll
  for (int i = 0; i < DTILES; ++i) o_acc[i][0] = o_acc[i][1] = o_acc[i][2] = o_acc[i][3] = 0.f;
  float row_max[2] = {-INFINITY, -INFINITY};
  float row_sum[2] = {0.f, 0.f};
  const int qrow0 = m0 + warp * 16 + (lane >> 2);  // rows qrow0 and qrow0 + 8

  for (int t = 0; t < n_tiles; ++t) {
    const int st = t & 1;
    if (t + 1 < n_tiles) {
      load_tile<DPAD>(sK(st ^ 1), kg, p.k_ss, (t + 1) * ATT_BN, p.sk, p.d);
      load_tile<DPAD>(sV(st ^ 1), vg, p.v_ss, (t + 1) * ATT_BN, p.sk, p.d);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();

    // ---- S = Q K^T  (16 x 64 per warp)
    float s_acc[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) s_acc[j][0] = s_acc[j][1] = s_acc[j][2] = s_acc[j][3] = 0.f;
#pragma unroll
    for (int ks = 0; ks < KSTEPS; ++ks) {
      uint32_t a0, a1, a2, a3;
      {
        const int r = warp * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
        const int c = ks * 16 + (lane >> 4) * 8;
        ldsm_x4(sQ + (uint32_t)(r * LD + c) * 2u, a0, a1, a2, a3);
      }
#pragma unroll
      for (int jp = 0; jp < 4; ++jp) {  // pairs of n8 tiles
        uint32_t b0, b1, b2, b3;
        const int r = jp * 16 + (lane & 7) + (lane >> 4) * 8;
        const int c = ks * 16 + ((lane >> 3) & 1) * 8;
        ldsm_x4(sK(st) + (uint32_t)(r * LD + c) * 2u, b0, b1, b2, b3);
        mma16816(s_acc[2 * jp], a0, a1, a2, a3, b0, b1);
        mma16816(s_acc[2 * jp + 1], a0, a1, a2, a3, b2, b3);
      }
    }

    // ---- mask + online softmax (base-2)
    const int col_base = t * ATT_BN + (lane & 3) * 2;
    const bool need_mask = (t * ATT_BN + ATT_BN > p.sk) || (p.causal && (t * ATT_BN + ATT_BN - 1 > m0 + causal_off));
    float tmax[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float v = s_acc[j][e] * p.scale_log2;
        if (need_mask) {
          const int col = col_base + j * 8 + (e & 1);
          const int row = qrow0 + (e >> 1) * 8;
          if (col >= p.sk || (p.causal && col > row + causal_off)) v = -INFINITY;
        }
        s_acc[j][e] = v;
        tmax[e >> 1] = fmaxf(tmax[e >> 1], v);
      }
    }
    float corr[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      tmax[r] = fmaxf(tmax[r], __shfl_xor_sync(0xffffffffu, tmax[r], 1));
      tmax[r] = fmaxf(tmax[r], __shfl_xor_sync(0xffffffffu, tmax[r], 2));
      const float nm = fmaxf(row_max[r], tmax[r]);
      const float base = (nm == -INFINITY) ? 0.f : nm;  // fully masked row so far
      corr[r] = exp2f(row_max[r] - base);               // row_max = -inf -> 0
      row_max[r] = nm;
      tmax[r] = base;
      row_sum[r] *= corr[r];
    }
    float psum[2] = {0.f, 0.f};
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float pv = exp2f(s_acc[j][e] - tmax[e >> 1]);
        s_acc[j][e] = pv;
        psum[e >> 1] += pv;
      }
    }
    row_sum[0] += psum[0];
    row_sum[1] += psum[1];
#pragma unroll
    for (int i = 0; i < DTILES; ++i) {
      o_acc[i][0] *= corr[0], o_acc[i][1] *= corr[0];
      o_acc[i][2] *= corr[1], o_acc[i][3] *= corr[1];
    }

    // ---- O += P V
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {  // k16 steps over the 64 keys
      const uint32_t a0 = pack_half2(s_acc[2 * kk][0], s_acc[2 * kk][1]);
      const uint32_t a1 = pack_half2(s_acc[2 * kk][2], s_acc[2 * kk][3]);
      const uint32_t a2 = pack_half2(s_acc[2 * kk + 1][0], s_acc[2 * kk + 1][1]);
      const uint32_t a3 = pack_half2(s_acc[2 * kk + 1][2], s_acc[2 * kk + 1][3]);
#pragma unroll
      for (int dp = 0; dp < DTILES / 2; ++dp) {
        uint32_t b0, b1, b2, b3;
        const int r = kk * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
        const int c = dp * 16 + (lane >> 4) * 8;
        ldsm_x4_t(sV(st) + (uint32_t)(r * LD + c) * 2u, b0, b1, b2, b3);
        mma16816(o_acc[2 * dp], a0, a1, a2, a3, b0, b1);
        mma16816(o_acc[2 * dp + 1], a0, a1, a2, a3, b2, b3);
      }
    }
    __syncthreads();  // everyone done with stage st before it is refilled
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
  for (int i = 0; i < DTILES; ++i) {
    const int col = i * 8 + (lane & 3) * 2;
    if (col < p.d) {
      if (qrow0 < p.sq) *(__half2*)(og + (long long)qrow0 * p.o_ss + col) = __floats2half2_rn(o_acc[i][0] * inv0, o_acc[i][1] * inv0);
      if (qrow0 + 8 < p.sq)
        *(__half2*)(og + (long long)(qrow0 + 8) * p.o_ss + col) = __floats2half2_rn(o_acc[i][2] * inv1, o_acc[i][3] * inv1);
    }
  }
}

void count_launch();

template <int DPAD>
static int launch_attn(const AttnParams& p, int B, int H, cudaStream_t st) {
  static bool attr_done = false;
  if (!attr_done) {
    SEEDX_CUDA(cudaFuncSetAttribute(flash_attn_kernel<DPAD>, cudaFuncAttributeMaxDynamicSharedMemorySize, AttnSmem<DPAD>::BYTES));
    attr_done = true;
  }
  dim3 grid((p.sq + ATT_BM - 1) / ATT_BM, H, B);
  launch_k(flash_attn_kernel<DPAD>, grid, 128, AttnSmem<DPAD>::BYTES, st, p);
  count_launch();
  return check_cuda(cudaGetLastError(), "flash_attn_kernel launch");
}

}  // namespace seedx

namespace seedx {
int attention_wg_try(const seedx_attn_args* a, cudaStream_t st);
static int g_attn_impl = 0;  // 0 = auto (wgmma kernel when eligible, else mma.sync), 1 = force mma.sync
static int g_attn_last = 0;  // implementation used by the most recent call: 2 = wgmma, 1 = mma.sync
}
using namespace seedx;

extern "C" void seedx_attention_set_impl(int impl) { seedx::g_attn_impl = impl; }
extern "C" int seedx_attention_last_impl(void) { return seedx::g_attn_last; }

extern "C" int seedx_attention_f16(const seedx_attn_args* a, void* stream) {
  SEEDX_REQUIRE(a && a->q && a->k && a->v && a->o, "seedx_attention_f16: null pointer");
  SEEDX_REQUIRE(a->batch > 0 && a->heads > 0 && a->sq > 0 && a->sk > 0, "seedx_attention_f16: empty problem");
  SEEDX_REQUIRE(a->d % 8 == 0 && a->d >= 8 && a->d <= 160, "seedx_attention_f16: head dim %d unsupported (multiple of 8, <= 160)", a->d);
  const long long strides[] = {a->q_stride_b, a->q_stride_h, a->q_stride_s, a->k_stride_b, a->k_stride_h, a->k_stride_s,
                               a->v_stride_b, a->v_stride_h, a->v_stride_s};
  for (long long s : strides) SEEDX_REQUIRE(s % 8 == 0, "seedx_attention_f16: q/k/v strides must be multiples of 8 elements (16 B)");
  SEEDX_REQUIRE(a->o_stride_b % 2 == 0 && a->o_stride_h % 2 == 0 && a->o_stride_s % 2 == 0, "seedx_attention_f16: o strides must be even");
  SEEDX_REQUIRE(((uintptr_t)a->q % 16 == 0) && ((uintptr_t)a->k % 16 == 0) && ((uintptr_t)a->v % 16 == 0) && ((uintptr_t)a->o % 4 == 0),
                "seedx_attention_f16: q/k/v must be 16B aligned");
  SEEDX_REQUIRE(a->heads <= 65535 && a->batch <= 65535, "seedx_attention_f16: grid too large");
  AttnParams p;
  p.q = (const __half*)a->q, p.k = (const __half*)a->k, p.v = (const __half*)a->v, p.o = (__half*)a->o;
  p.q_sb = a->q_stride_b, p.q_sh = a->q_stride_h, p.q_ss = a->q_stride_s;
  p.k_sb = a->k_stride_b, p.k_sh = a->k_stride_h, p.k_ss = a->k_stride_s;
  p.v_sb = a->v_stride_b, p.v_sh = a->v_stride_h, p.v_ss = a->v_stride_s;
  p.o_sb = a->o_stride_b, p.o_sh = a->o_stride_h, p.o_ss = a->o_stride_s;
  p.sq = a->sq, p.sk = a->sk, p.d = a->d;
  p.scale_log2 = a->scale * 1.4426950408889634f;
  p.causal = a->causal;
  cudaStream_t st = (cudaStream_t)stream;
  if (g_attn_impl != 1) {
    const int rc = attention_wg_try(a, st);
    if (rc >= 0) {
      g_attn_last = 2;
      return rc;
    }
  }
  g_attn_last = 1;
  if (a->d <= 64) return launch_attn<64>(p, a->batch, a->heads, st);
  if (a->d <= 112) return launch_attn<112>(p, a->batch, a->heads, st);
  if (a->d <= 128) return launch_attn<128>(p, a->batch, a->heads, st);
  return launch_attn<160>(p, a->batch, a->heads, st);
}
