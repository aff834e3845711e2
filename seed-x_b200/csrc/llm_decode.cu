// seedx-b200: HBM-bound kernels of the LLaMA token loop (batch-1 greedy decode) and the prefill glue.
//
// Decode reads every weight once per token (26 GB at 13 B parameters) -> the roofline is HBM bandwidth, not the tensor
// cores: the projections are GEMVs streaming fp16 rows with 128-bit loads (RMSNorm fused in the prologue, SwiGLU /
// residual in the epilogue), attention walks the fp16 KV cache with 16-byte loads, and the sampler state (sequence,
// length, done flag) lives on the device so a whole step is one CUDA-graph replay with no host synchronisation.
//
// Replaces: src/models/mllm/modeling_llama_xformer.py:141-149 (RoPE), 204-239 (q/k/v/o at M=1, KV torch.cat append,
// xformers attention over the cache), 166-167 (SwiGLU MLP), 707 (lm_head); transformers LlamaRMSNorm; the python
// logits processor src/models/mllm/generation.py:19-31 and the argmax of HF greedy_search (SURVEY.md B.1).
#include "common.cuh"
#include "../../include/seedx.h"

namespace seedx {
void count_launch();

// ------------------------------------------------------------------------------------------------
// Batched GEMV: out[b][n] = epi( W[n,:] . norm(x[b,:]) ) for up to 8 sequences.  The fp16 weight matrix is streamed from HBM exactly
// once (one 128-bit ld.global.cs per lane per 8x32 weight block) and multiplied on the tensor cores: mma.sync.m16n8k16 with the
// weight block as the A operand (8 rows used), the activations of the 8 sequence slots as the B operand (from shared memory, fp16)
// and fp32 accumulators — so the instruction stream per byte is ~10x shorter than scalar FMAs and decode stays HBM-bound for 8
// sequences as well as for 1.  The dot product is order-independent in k, so a lane's 16 contiguous bytes of a weight row serve
// as the k-slots {2q,2q+1,2q+8,2q+9} of two consecutive MMAs and the activations are read with the same permutation.
// One CTA per SM (16 warps split K); a CTA owns a balanced contiguous range of 8-row tiles.
// ------------------------------------------------------------------------------------------------
constexpr int GEMV_THREADS = 512;
constexpr int GEMV_WARPS = GEMV_THREADS / 32;
constexpr int GEMV_ROWS = 8;    // weight rows per tile
constexpr int GEMV_MAXKB = 14;  // 32-wide k blocks a warp keeps in registers (16 B per lane each)

SEEDX_DEVINL void mma16816_f32(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

template <int NB>  // sequence slots held in shared memory: 1, 2, 4 or 8
__global__ void __launch_bounds__(GEMV_THREADS, 1)
gemv_mma_kernel(const __half* __restrict__ W, const float* __restrict__ x, long long ldx, const float* __restrict__ rms_w, float eps,
                const float* __restrict__ residual, long long ldr, float* __restrict__ out, long long ldo, int N, int K, int gated) {
  extern __shared__ __align__(16) uint8_t gsm[];
  __half* xs = (__half*)gsm;                                   // [NB][K + 8]: rows 16 B apart in bank space (conflict-free LDS.128)
  const int KP = K + 8;
  __shared__ float part_sm[2][GEMV_WARPS][GEMV_ROWS * 8];
  __shared__ float red[GEMV_WARPS][NB];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  const int g = lane >> 2, q = lane & 3;   // g: weight row inside the tile AND sequence slot of the B fragment; q: 16-byte k-chunk
  const int tiles = (N + GEMV_ROWS - 1) / GEMV_ROWS;
  const int t_begin = (int)((long long)blockIdx.x * tiles / gridDim.x);
  const int t_end = (int)((long long)(blockIdx.x + 1) * tiles / gridDim.x);
  const int kblocks = K >> 5;              // 32-wide k blocks (K % 32 == 0 checked on the host)
  const int kb_begin = (int)((long long)warp * kblocks / GEMV_WARPS), kb_end = (int)((long long)(warp + 1) * kblocks / GEMV_WARPS);
  const int kparts = (((kblocks + GEMV_WARPS - 1) / GEMV_WARPS) + GEMV_MAXKB - 1) / GEMV_MAXKB;   // block-uniform
  const bool has_x = g < NB;

  // The weight stream is software-pipelined across tiles: the registers of unit u+1 (a tile's k-part) are requested right after
  // unit u has been fed to the tensor cores, i.e. BEFORE the cross-warp reduction and its barrier, so HBM requests never drain.
  uint4 wreg[GEMV_MAXKB];
  auto load_unit = [&](int t, int part) {
    const int row = min(t * GEMV_ROWS + g, N - 1);
    const uint4* wrow = (const uint4*)(W + (long long)row * K) + q;
    const int kb0 = kb_begin + part * GEMV_MAXKB;
#pragma unroll
    for (int i = 0; i < GEMV_MAXKB; ++i)
      if (kb0 + i < kb_end) wreg[i] = __ldcs(wrow + (kb0 + i) * 4);   // 8 consecutive halves of weight row g: k = kb*32 + q*8 ..
  };
  // Weights never depend on the previous kernel: the first unit is requested before the programmatic-dependent-launch wait, so
  // the HBM stream is already running while the producer of `x` drains.
  if (t_begin < t_end) load_unit(t_begin, 0);
  pdl_wait();
  pdl_trigger();
  // ---- prologue: activations -> (RMSNorm) -> fp16 in shared memory
  float ss[NB];
#pragma unroll
  for (int b = 0; b < NB; ++b) ss[b] = 0.f;
  if (rms_w != nullptr) {
    for (int k = threadIdx.x; k < K; k += GEMV_THREADS) {
#pragma unroll
      for (int b = 0; b < NB; ++b) {
        const float v = x[b * ldx + k];
        ss[b] += v * v;
      }
    }
#pragma unroll
    for (int b = 0; b < NB; ++b) {
      ss[b] = warp_sum(ss[b]);
      if (lane == 0) red[warp][b] = ss[b];
    }
    __syncthreads();
#pragma unroll
    for (int b = 0; b < NB; ++b) {
      float t = 0.f;
#pragma unroll
      for (int w = 0; w < GEMV_WARPS; ++w) t += red[w][b];
      ss[b] = rsqrtf(t / (float)K + eps);
    }
  }
  for (int k = threadIdx.x; k < K; k += GEMV_THREADS) {
    const float g = rms_w ? rms_w[k] : 1.f;
#pragma unroll
    for (int b = 0; b < NB; ++b) {
      const float v = x[b * ldx + k];
      xs[b * KP + k] = __float2half_rn(rms_w ? v * ss[b] * g : v);
    }
  }
  __syncthreads();

  const __half* xrow = xs + (has_x ? g : 0) * KP + q * 8;
  int buf = 0;
  for (int t = t_begin; t < t_end; ++t, buf ^= 1) {
    float c[4] = {0.f, 0.f, 0.f, 0.f};
    for (int part = 0; part < kparts; ++part) {
      const int kb0 = kb_begin + part * GEMV_MAXKB;
#pragma unroll
      for (int i = 0; i < GEMV_MAXKB; ++i) {
        if (kb0 + i < kb_end) {
          uint4 xq = make_uint4(0, 0, 0, 0);
          if (has_x) xq = *(const uint4*)(xrow + (kb0 + i) * 32);       // the same k positions of sequence g
          mma16816_f32(c, wreg[i].x, 0u, wreg[i].y, 0u, xq.x, xq.y);
          mma16816_f32(c, wreg[i].z, 0u, wreg[i].w, 0u, xq.z, xq.w);
        }
      }
      if (part + 1 < kparts) load_unit(t, part + 1);
      else if (t + 1 < t_end) load_unit(t + 1, 0);
    }
    // c[0], c[1] = partial dot products of weight row g with sequences 2q, 2q+1
    part_sm[buf][warp][g * 8 + 2 * q] = c[0];
    part_sm[buf][warp][g * 8 + 2 * q + 1] = c[1];
    __syncthreads();
    if (threadIdx.x < GEMV_ROWS * NB) {
      const int r = threadIdx.x / NB, b = threadIdx.x % NB;
      float v = 0.f;
#pragma unroll
      for (int w = 0; w < GEMV_WARPS; ++w) v += part_sm[buf][w][r * 8 + b];
      const int orow = t * GEMV_ROWS + r;
      if (!gated) {
        if (orow < N) out[b * ldo + orow] = v + (residual ? residual[b * ldr + orow] : 0.f);
      } else if ((r & 1) == 0 && orow + 1 < N) {
        float gate = 0.f;
#pragma unroll
        for (int w = 0; w < GEMV_WARPS; ++w) gate += part_sm[buf][w][(r + 1) * 8 + b];
        out[b * ldo + (orow >> 1)] = v * silu(gate);  // rows interleaved [up_j, gate_j]: silu(gate(x)) * up(x), :166-167
      }
    }
    // the next tile writes the other partial buffer; its __syncthreads orders these reads before the buffer is reused
  }
}

// ------------------------------------------------------------------------------------------------
// FP8 (e4m3) weights: the same GEMV with half the bytes per row.  W8 holds q[n,k] and row_scale s[n] (fp32) such that the weight is
// s[n] * q[n,k]; the scale is applied to the fp32 dot product in the epilogue.  A lane's 16-byte load now carries 16 consecutive e4m3
// weights of its row, k = kb*64 + q*16 .. +15; cvt.rn.f16x2.e4m3x2 turns them into 8 f16x2 registers (exactly: every e4m3 value is an
// fp16 value) that feed four m16n8k16 MMAs.  As in gemv_mma_kernel, lane (g, q) supplies k-slots {2q,2q+1,2q+8,2q+9} for the weights of
// row g AND for the activations of sequence g, so reading the activations at the same 16 k positions keeps the pairing right.
// Same register budget as the fp16 kernel: GEMV8_MAXKB x 16 B of weights per lane, which covers K = 13824 in one unit.
// ------------------------------------------------------------------------------------------------
constexpr int GEMV8_MAXKB = 14;  // 64-wide k blocks a warp keeps in registers (16 B per lane each)

SEEDX_DEVINL uint32_t e4m3x2_to_f16x2(uint16_t v) {   // low byte -> low half (the lower k), high byte -> high half
  uint32_t r;
  asm("cvt.rn.f16x2.e4m3x2 %0, %1;\n" : "=r"(r) : "h"(v));
  return r;
}

template <int NB>  // sequence slots held in shared memory: 1, 2, 4 or 8
__global__ void __launch_bounds__(GEMV_THREADS, 1)
gemv_fp8_kernel(const uint8_t* __restrict__ W8, const float* __restrict__ row_scale, const float* __restrict__ x, long long ldx,
                const float* __restrict__ rms_w, float eps, const float* __restrict__ residual, long long ldr, float* __restrict__ out,
                long long ldo, int N, int K, int gated) {
  extern __shared__ __align__(16) uint8_t gsm[];
  __half* xs = (__half*)gsm;                                   // [NB][K + 8]: rows 16 B apart in bank space (conflict-free LDS.128)
  const int KP = K + 8;
  __shared__ float part_sm[2][GEMV_WARPS][GEMV_ROWS * 8];
  __shared__ float red[GEMV_WARPS][NB];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  const int g = lane >> 2, q = lane & 3;   // g: weight row inside the tile AND sequence slot of the B fragment; q: 16-byte k-chunk
  const int tiles = (N + GEMV_ROWS - 1) / GEMV_ROWS;
  const int t_begin = (int)((long long)blockIdx.x * tiles / gridDim.x);
  const int t_end = (int)((long long)(blockIdx.x + 1) * tiles / gridDim.x);
  const int kblocks = K >> 6;              // 64-wide k blocks (K % 64 == 0 checked on the host)
  const int kb_begin = (int)((long long)warp * kblocks / GEMV_WARPS), kb_end = (int)((long long)(warp + 1) * kblocks / GEMV_WARPS);
  const int kparts = (((kblocks + GEMV_WARPS - 1) / GEMV_WARPS) + GEMV8_MAXKB - 1) / GEMV8_MAXKB;   // block-uniform
  const bool has_x = g < NB;

  // software pipeline across tiles, as in gemv_mma_kernel: unit u+1 is requested before the cross-warp reduction of unit u
  uint4 wreg[GEMV8_MAXKB];
  auto load_unit = [&](int t, int part) {
    const int row = min(t * GEMV_ROWS + g, N - 1);
    const uint4* wrow = (const uint4*)(W8 + (long long)row * K) + q;
    const int kb0 = kb_begin + part * GEMV8_MAXKB;
#pragma unroll
    for (int i = 0; i < GEMV8_MAXKB; ++i)
      if (kb0 + i < kb_end) wreg[i] = __ldcs(wrow + (kb0 + i) * 4);   // 16 consecutive e4m3 of weight row g: k = kb*64 + q*16 ..
  };
  if (t_begin < t_end) load_unit(t_begin, 0);   // weights never depend on the previous kernel: requested before the PDL wait
  pdl_wait();
  pdl_trigger();
  // ---- prologue: activations -> (RMSNorm) -> fp16 in shared memory
  float ss[NB];
#pragma unroll
  for (int b = 0; b < NB; ++b) ss[b] = 0.f;
  if (rms_w != nullptr) {
    for (int k = threadIdx.x; k < K; k += GEMV_THREADS) {
#pragma unroll
      for (int b = 0; b < NB; ++b) {
        const float v = x[b * ldx + k];
        ss[b] += v * v;
      }
    }
#pragma unroll
    for (int b = 0; b < NB; ++b) {
      ss[b] = warp_sum(ss[b]);
      if (lane == 0) red[warp][b] = ss[b];
    }
    __syncthreads();
#pragma unroll
    for (int b = 0; b < NB; ++b) {
      float t = 0.f;
#pragma unroll
      for (int w = 0; w < GEMV_WARPS; ++w) t += red[w][b];
      ss[b] = rsqrtf(t / (float)K + eps);
    }
  }
  for (int k = threadIdx.x; k < K; k += GEMV_THREADS) {
    const float g = rms_w ? rms_w[k] : 1.f;
#pragma unroll
    for (int b = 0; b < NB; ++b) {
      const float v = x[b * ldx + k];
      xs[b * KP + k] = __float2half_rn(rms_w ? v * ss[b] * g : v);
    }
  }
  __syncthreads();

  const __half* xrow = xs + (has_x ? g : 0) * KP + q * 16;
  int buf = 0;
  for (int t = t_begin; t < t_end; ++t, buf ^= 1) {
    float c[4] = {0.f, 0.f, 0.f, 0.f};
    for (int part = 0; part < kparts; ++part) {
      const int kb0 = kb_begin + part * GEMV8_MAXKB;
#pragma unroll
      for (int i = 0; i < GEMV8_MAXKB; ++i) {
        if (kb0 + i < kb_end) {
          uint4 x0 = make_uint4(0, 0, 0, 0), x1 = make_uint4(0, 0, 0, 0);
          if (has_x) {                                                   // the same 16 k positions of sequence g
            x0 = *(const uint4*)(xrow + (kb0 + i) * 64);
            x1 = *(const uint4*)(xrow + (kb0 + i) * 64 + 8);
          }
          const uint4 w = wreg[i];
          mma16816_f32(c, e4m3x2_to_f16x2((uint16_t)w.x), 0u, e4m3x2_to_f16x2((uint16_t)(w.x >> 16)), 0u, x0.x, x0.y);
          mma16816_f32(c, e4m3x2_to_f16x2((uint16_t)w.y), 0u, e4m3x2_to_f16x2((uint16_t)(w.y >> 16)), 0u, x0.z, x0.w);
          mma16816_f32(c, e4m3x2_to_f16x2((uint16_t)w.z), 0u, e4m3x2_to_f16x2((uint16_t)(w.z >> 16)), 0u, x1.x, x1.y);
          mma16816_f32(c, e4m3x2_to_f16x2((uint16_t)w.w), 0u, e4m3x2_to_f16x2((uint16_t)(w.w >> 16)), 0u, x1.z, x1.w);
        }
      }
      if (part + 1 < kparts) load_unit(t, part + 1);
      else if (t + 1 < t_end) load_unit(t + 1, 0);
    }
    part_sm[buf][warp][g * 8 + 2 * q] = c[0];
    part_sm[buf][warp][g * 8 + 2 * q + 1] = c[1];
    __syncthreads();
    if (threadIdx.x < GEMV_ROWS * NB) {
      const int r = threadIdx.x / NB, b = threadIdx.x % NB;
      float v = 0.f;
#pragma unroll
      for (int w = 0; w < GEMV_WARPS; ++w) v += part_sm[buf][w][r * 8 + b];
      const int orow = t * GEMV_ROWS + r;
      if (!gated) {
        if (orow < N) out[b * ldo + orow] = row_scale[orow] * v + (residual ? residual[b * ldr + orow] : 0.f);
      } else if ((r & 1) == 0 && orow + 1 < N) {
        float gate = 0.f;
#pragma unroll
        for (int w = 0; w < GEMV_WARPS; ++w) gate += part_sm[buf][w][(r + 1) * 8 + b];
        out[b * ldo + (orow >> 1)] = (row_scale[orow] * v) * silu(row_scale[orow + 1] * gate);   // rows [up_j, gate_j], each with its scale
      }
    }
  }
}

// out[n, k] = (half)(float(q[n, k]) * s[n]): one 16-byte load of 16 e4m3 values, two 16-byte stores of fp16.  The output is a scratch
// buffer that the kernels before this one may still read, so every store waits for the PDL dependency; the loads do not.
__global__ void __launch_bounds__(256)
dequant_fp8_kernel(const uint4* __restrict__ q, const float* __restrict__ row_scale, uint4* __restrict__ out, long long chunks, int row_chunks) {
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  uint4 w = make_uint4(0, 0, 0, 0);
  if (i < chunks) w = __ldcs(q + i);
  pdl_wait();
  pdl_trigger();
  for (; i < chunks; i += (long long)gridDim.x * blockDim.x) {
    const float s = __ldg(row_scale + i / row_chunks);
    const uint32_t wv[4] = {w.x, w.y, w.z, w.w};
    uint32_t o[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const uint32_t h2 = e4m3x2_to_f16x2((uint16_t)(wv[j >> 1] >> ((j & 1) * 16)));
      const float2 f = __half22float2(*(const __half2*)&h2);
      const __half2 r = __floats2half2_rn(f.x * s, f.y * s);
      o[j] = *(const uint32_t*)&r;
    }
    out[2 * i] = make_uint4(o[0], o[1], o[2], o[3]);
    out[2 * i + 1] = make_uint4(o[4], o[5], o[6], o[7]);
    const long long nx = i + (long long)gridDim.x * blockDim.x;
    if (nx < chunks) w = __ldcs(q + nx);
  }
}

// ------------------------------------------------------------------------------------------------
// decode attention for one new token: RoPE(q,k) -> append k,v to the cache -> softmax(q K^T) V over positions 0..pos
// one CTA per head, head_dim 128, 8 warps, each half-warp walks keys with 16-byte loads.
// state[0] = current sequence length (the token being consumed sits at position state[0] - 1)
// ------------------------------------------------------------------------------------------------
constexpr int DA_THREADS = 256;
constexpr int DA_GROUPS = DA_THREADS / 16;  // half-warps

// KV-cache row of logical position t of one sequence.  Paged mode (pt != NULL): the cache is a pool of pages of 2^shift tokens and
// pt[] is the sequence's page table (physical page of logical page t >> shift); contiguous mode: the sequence owns one slab.
__device__ __forceinline__ long long kv_row(const int* __restrict__ pt, int shift, int t) {
  return pt ? ((((long long)__ldg(pt + (t >> shift))) << shift) | (long long)(t & ((1 << shift) - 1))) : (long long)t;
}

__global__ void __launch_bounds__(DA_THREADS)
decode_attn_kernel(const float* __restrict__ qkv_all, const int* __restrict__ state_all, const float* __restrict__ inv_freq,
                   __half* __restrict__ kcache_all, __half* __restrict__ vcache_all, long long cache_stride, float* __restrict__ out_all, int H,
                   float scale, const int* __restrict__ page_table, int table_stride, int page_shift) {
  pdl_wait();
  pdl_trigger();
  constexpr int HD = 128;
  __shared__ float qs[HD];
  __shared__ float gm[DA_GROUPS], gl[DA_GROUPS];
  __shared__ float gacc[DA_GROUPS][HD];
  const int h = blockIdx.x;
  const int D = H * HD;
  const int bidx = blockIdx.y;                    // sequence slot
  const float* qkv = qkv_all + (long long)bidx * 3 * D;
  const int* state = state_all + bidx * 4;
  __half* kcache = kcache_all + (page_table ? 0ll : (long long)bidx * cache_stride);
  __half* vcache = vcache_all + (page_table ? 0ll : (long long)bidx * cache_stride);
  const int* pt = page_table ? page_table + (long long)bidx * table_stride : nullptr;
  float* out = out_all + (long long)bidx * D;
  const int pos = state[0] - 1;
  const int tid = threadIdx.x;
  const long long prow = kv_row(pt, page_shift, pos) * D;      // cache row that receives this step's k, v
  if (tid < HD / 2) {
    const float ang = (float)pos * inv_freq[tid];
    const float c = cosf(ang), s = sinf(ang);
    const float q0 = qkv[h * HD + tid], q1 = qkv[h * HD + tid + HD / 2];
    const float k0 = qkv[D + h * HD + tid], k1 = qkv[D + h * HD + tid + HD / 2];
    qs[tid] = (q0 * c - q1 * s) * scale;
    qs[tid + HD / 2] = (q1 * c + q0 * s) * scale;
    kcache[prow + h * HD + tid] = __float2half_rn(k0 * c - k1 * s);
    kcache[prow + h * HD + tid + HD / 2] = __float2half_rn(k1 * c + k0 * s);
  } else if (tid < HD / 2 + HD) {
    const int i = tid - HD / 2;
    vcache[prow + h * HD + i] = __float2half_rn(qkv[2 * D + h * HD + i]);
  }
  __syncthreads();

  const int grp = tid >> 4, gl_lane = tid & 15;
  float q[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) q[i] = qs[gl_lane * 8 + i];
  float m = -INFINITY, l = 0.f, acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;
  // Each half-warp owns tokens grp, grp + 16, ...; DA_UNROLL of them are requested before the first is consumed, so a CTA keeps
  // 16 x DA_UNROLL x 512 B of K/V reads in flight instead of one dependent 32-byte pair per half-warp (the walk over ~300 cached tokens was
  // load-latency bound: 11 % of the token step for < 4 % of its bytes).
  constexpr int DA_UNROLL = 4;
  for (int t0 = 0; t0 <= pos; t0 += DA_GROUPS * DA_UNROLL) {  // warp-uniform trip count: the half-warp shuffles need all 32 lanes
    uint4 kq[DA_UNROLL], vq[DA_UNROLL];
#pragma unroll
    for (int u = 0; u < DA_UNROLL; ++u) {
      const int t = t0 + u * DA_GROUPS + grp;
      kq[u] = make_uint4(0, 0, 0, 0), vq[u] = make_uint4(0, 0, 0, 0);
      if (t <= pos) {   // one half-warp = one token: 16 lanes x 16 bytes = the head's 256 contiguous bytes of the row (two full 128 B lines)
        const long long r = kv_row(pt, page_shift, t) * D + h * HD + gl_lane * 8;
        kq[u] = *(const uint4*)(kcache + r);
        vq[u] = *(const uint4*)(vcache + r);
      }
    }
    float sc[DA_UNROLL];
#pragma unroll
    for (int u = 0; u < DA_UNROLL; ++u) {
      const __half2* kh = (const __half2*)&kq[u];
      float s = 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = __half22float2(kh[j]);
        s += f.x * q[2 * j] + f.y * q[2 * j + 1];
      }
#pragma unroll
      for (int o = 8; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);  // within the 16-lane group
      sc[u] = (t0 + u * DA_GROUPS + grp <= pos) ? s : -INFINITY;
    }
    // one rescale for the DA_UNROLL tokens (same arithmetic as token-by-token up to the order of the exponentials' reference maximum)
    float nm = m;
#pragma unroll
    for (int u = 0; u < DA_UNROLL; ++u) nm = fmaxf(nm, sc[u]);
    if (nm > -INFINITY) {
      const float corr = __expf(m - nm);
      l *= corr;
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] *= corr;
#pragma unroll
      for (int u = 0; u < DA_UNROLL; ++u) {
        const float p = __expf(sc[u] - nm);      // exp(-inf) = 0 for the slots past the end
        l += p;
        const __half2* vh = (const __half2*)&vq[u];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 f = __half22float2(vh[j]);
          acc[2 * j] = fmaf(p, f.x, acc[2 * j]);
          acc[2 * j + 1] = fmaf(p, f.y, acc[2 * j + 1]);
        }
      }
      m = nm;
    }
  }
  if (gl_lane == 0) gm[grp] = m, gl[grp] = l;
#pragma unroll
  for (int i = 0; i < 8; ++i) gacc[grp][gl_lane * 8 + i] = acc[i];
  __syncthreads();
  if (tid < HD) {
    float M = -INFINITY;
#pragma unroll
    for (int g = 0; g < DA_GROUPS; ++g) M = fmaxf(M, gm[g]);
    float L = 0.f, o = 0.f;
#pragma unroll
    for (int g = 0; g < DA_GROUPS; ++g) {
      const float w = (gm[g] == -INFINITY) ? 0.f : __expf(gm[g] - M);
      L += w * gl[g];
      o += w * gacc[g][tid];
    }
    out[h * HD + tid] = o / L;
  }
}

// RoPE on the prefill q/k (in place, fp16 [T, 3D] = [q | k | v]) + copy of k, v into the cache rows pos0..pos0+T-1
__global__ void rope_kv_prefill_kernel(__half* __restrict__ qkv, int T, int pos0, int H, const float* __restrict__ inv_freq,
                                       __half* __restrict__ kcache, __half* __restrict__ vcache, const int* __restrict__ pt, int page_shift) {
  pdl_wait();
  pdl_trigger();
  constexpr int HD = 128;
  const int D = H * HD;
  const long long total = (long long)T * H * (HD / 2);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int j = (int)(i % (HD / 2));
    const long long r = i / (HD / 2);
    const int h = (int)(r % H);
    const int t = (int)(r / H);
    const float ang = (float)(pos0 + t) * inv_freq[j];
    const float c = cosf(ang), s = sinf(ang);
    __half* row = qkv + (long long)t * 3 * D;
    const int o = h * HD + j;
    const float q0 = __half2float(row[o]), q1 = __half2float(row[o + HD / 2]);
    const float k0 = __half2float(row[D + o]), k1 = __half2float(row[D + o + HD / 2]);
    row[o] = __float2half_rn(q0 * c - q1 * s);
    row[o + HD / 2] = __float2half_rn(q1 * c + q0 * s);
    const __half kr0 = __float2half_rn(k0 * c - k1 * s), kr1 = __float2half_rn(k1 * c + k0 * s);
    row[D + o] = kr0;
    row[D + o + HD / 2] = kr1;
    const long long cr = kv_row(pt, page_shift, pos0 + t) * D;
    kcache[cr + o] = kr0;
    kcache[cr + o + HD / 2] = kr1;
    vcache[cr + o] = row[2 * D + o];
    vcache[cr + o + HD / 2] = row[2 * D + o + HD / 2];
  }
}

// rows of the embedding table -> fp32.  ids == NULL: single row for the last token of the device-resident sequence
__global__ void embed_rows_kernel(const __half* __restrict__ table, const int* __restrict__ ids, const int* __restrict__ state,
                                  const int* __restrict__ seq, int seq_stride, int n, int D, float* __restrict__ out) {
  pdl_wait();
  pdl_trigger();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < (long long)n * D; i += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(i / D), c = (int)(i - (long long)r * D);
    const int id = ids ? ids[r] : seq[(long long)r * seq_stride + state[r * 4] - 1];
    out[i] = __half2float(table[(long long)id * D + c]);
  }
}

template <typename TS>
__global__ void scatter_rows_kernel(const TS* __restrict__ src, const int* __restrict__ src_idx, const int* __restrict__ idx, int n, int D,
                                    float* __restrict__ dst) {
  pdl_wait();
  pdl_trigger();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < (long long)n * D; i += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(i / D), c = (int)(i - (long long)r * D);
    const long long sr = src_idx ? src_idx[r] : r;
    dst[(long long)idx[r] * D + c] = (float)src[sr * D + c];
  }
}

// hidden[(state[0] - prompt_len - 1) * D + i] = x[i]   (post-norm last hidden state of the position consuming generated token j)
__global__ void store_hidden_kernel(const float* __restrict__ x, const int* __restrict__ state, int max_rows, int D,
                                    float* __restrict__ hidden) {
  pdl_wait();
  pdl_trigger();
  const int b = blockIdx.y;                       // state[b][3] = prompt length of sequence b
  const int row = state[b * 4] - state[b * 4 + 3] - 1;
  if (row < 0 || row >= max_rows) return;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < D; i += gridDim.x * blockDim.x)
    hidden[((long long)b * max_rows + row) * D + i] = x[(long long)b * D + i];
}

// torch.argmax order: a NaN ranks above every number, then the larger value, then the lower index wins.  So a row with NaN logits gives
// the id HF greedy search gives, and an all-NaN row gives id 0 instead of no id at all.
SEEDX_DEVINL bool argmax_before(float v, int i, float best, int bi) {
  const bool vn = isnan(v), bn = isnan(best);
  if (vn != bn) return vn;
  return v > best || ((v == best || vn) && i < bi);
}

// logits processor (generation.py:19-31) + greedy argmax + sequence append, all on the device.
// state[0] = sequence length, state[1] = done flag (EOS seen), state[2] = number of generated tokens
__global__ void __launch_bounds__(1024)
logits_argmax_kernel(float* __restrict__ logits_all, int V, const int* __restrict__ img_ids, int n_img_ids, int* __restrict__ seq_all,
                     int* __restrict__ state_all, int eos_id, int suppress_eos, int max_len) {
  pdl_wait();
  pdl_trigger();
  float* logits = logits_all + (long long)blockIdx.x * V;      // one CTA per sequence
  int* seq = seq_all + (long long)blockIdx.x * max_len;
  int* state = state_all + blockIdx.x * 4;
  __shared__ float smax[32];
  __shared__ int sidx[32];
  __shared__ int forced;
  const int len = state[0];
  const int last = seq[len - 1];
  if (threadIdx.x == 0) forced = -1;
  __syncthreads();
  if ((int)threadIdx.x < n_img_ids - 1 && img_ids[threadIdx.x] == last) forced = img_ids[threadIdx.x + 1];
  __syncthreads();
  int next;
  if (forced >= 0) {
    next = forced;  // scores[next] = max + 10 -> argmax is `next`
  } else {
    if (threadIdx.x >= 1 && (int)threadIdx.x < n_img_ids) logits[img_ids[threadIdx.x]] = 0.0f;  // img_ids[1:] <- 0.0 (not -inf!)
    if (suppress_eos && threadIdx.x == 0 && eos_id >= 0 && eos_id < V) logits[eos_id] = -INFINITY;
    __syncthreads();
    float best = -INFINITY;
    int bi = 0x7fffffff;
    for (int i = threadIdx.x; i < V; i += blockDim.x) {
      const float v = logits[i];
      if (argmax_before(v, i, best, bi)) best = v, bi = i;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (argmax_before(ov, oi, best, bi)) best = ov, bi = oi;
    }
    if ((threadIdx.x & 31) == 0) smax[threadIdx.x >> 5] = best, sidx[threadIdx.x >> 5] = bi;
    __syncthreads();
    if (threadIdx.x < 32) {
      best = threadIdx.x < (blockDim.x >> 5) ? smax[threadIdx.x] : -INFINITY;
      bi = threadIdx.x < (blockDim.x >> 5) ? sidx[threadIdx.x] : 0x7fffffff;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (argmax_before(ov, oi, best, bi)) best = ov, bi = oi;
      }
      if (threadIdx.x == 0) sidx[0] = bi;
    }
    __syncthreads();
    next = sidx[0];
  }
  // a slot whose state[1] is non-zero is parked: it has produced its EOS (the host truncates there anyway) or the host has retired the request
  // (continuous batching: a free slot waits for the next admission) — its sequence, KV length and harvest row stop moving
  if (threadIdx.x == 0 && len < max_len && state[1] == 0) {
    seq[len] = next;
    state[0] = len + 1;
    state[2] += 1;
    if (next == eos_id && !suppress_eos && state[1] == 0) state[1] = state[2];  // index (1-based) of the EOS token
  }
}

}  // namespace seedx
using namespace seedx;

static inline int ew_grid(long long work, int threads) {
  long long b = (work + threads - 1) / threads;
  const long long cap = (long long)num_sms() * 16;
  return (int)(b > cap ? cap : (b < 1 ? 1 : b));
}

extern "C" int seedx_gemv_f16(const void* W, const float* x, int64_t ldx, const float* rms_w, float eps, const float* residual, int64_t ldr,
                              float* out, int64_t ldo, int64_t N, int64_t K, int batch, int gated, void* stream) {
  SEEDX_REQUIRE(W && x && out, "seedx_gemv_f16: null pointer");
  SEEDX_REQUIRE(batch >= 1 && batch <= 8, "seedx_gemv_f16: batch %d out of range (1..8)", batch);
  SEEDX_REQUIRE(K % 32 == 0 && K > 0 && N > 0, "seedx_gemv_f16: K=%lld must be a positive multiple of 32", (long long)K);
  SEEDX_REQUIRE((uintptr_t)W % 16 == 0, "seedx_gemv_f16: W must be 16B aligned");
  if (gated) SEEDX_REQUIRE(N % 2 == 0 && residual == nullptr, "seedx_gemv_f16: gated needs even N and no residual");
  const int nb = batch <= 1 ? 1 : batch <= 2 ? 2 : batch <= 4 ? 4 : 8;
  SEEDX_REQUIRE(nb == batch, "seedx_gemv_f16: batch must be 1, 2, 4 or 8 (pad the sequence slots)");
  const size_t smem = (size_t)nb * (K + 8) * 2;
  SEEDX_REQUIRE(smem <= 216 * 1024, "seedx_gemv_f16: batch*K = %d*%lld does not fit in shared memory", nb, (long long)K);
  const long long tiles = (N + GEMV_ROWS - 1) / GEMV_ROWS;
  long long blocks = num_sms();
  if (blocks > tiles) blocks = tiles;
  cudaStream_t st = (cudaStream_t)stream;
#define GEMV_LAUNCH(NBV)                                                                                                               \
  do {                                                                                                                                 \
    static bool attr = false;                                                                                                          \
    if (!attr) {                                                                                                                       \
      SEEDX_CUDA(cudaFuncSetAttribute(gemv_mma_kernel<NBV>, cudaFuncAttributeMaxDynamicSharedMemorySize, 216 * 1024));                 \
      attr = true;                                                                                                                     \
    }                                                                                                                                  \
    launch_k(gemv_mma_kernel<NBV>, (unsigned)blocks, GEMV_THREADS, smem, st, (const __half*)W, x, ldx, rms_w, eps, residual, ldr, out, ldo, \
                                                                       (int)N, (int)K, gated);                                          \
  } while (0)
  if (nb == 1) GEMV_LAUNCH(1);
  else if (nb == 2) GEMV_LAUNCH(2);
  else if (nb == 4) GEMV_LAUNCH(4);
  else GEMV_LAUNCH(8);
#undef GEMV_LAUNCH
  count_launch();
  return check_cuda(cudaGetLastError(), "gemv launch");
}

extern "C" int seedx_gemv_fp8(const void* W8, const float* row_scale, const float* x, int64_t ldx, const float* rms_w, float eps,
                              const float* residual, int64_t ldr, float* out, int64_t ldo, int64_t N, int64_t K, int batch, int gated, void* stream) {
  SEEDX_REQUIRE(W8 && row_scale && x && out, "seedx_gemv_fp8: null pointer");
  SEEDX_REQUIRE(batch >= 1 && batch <= 8, "seedx_gemv_fp8: batch %d out of range (1..8)", batch);
  SEEDX_REQUIRE(K % 64 == 0 && K > 0 && N > 0, "seedx_gemv_fp8: K=%lld must be a positive multiple of 64", (long long)K);
  SEEDX_REQUIRE((uintptr_t)W8 % 16 == 0, "seedx_gemv_fp8: W8 must be 16B aligned");
  if (gated) SEEDX_REQUIRE(N % 2 == 0 && residual == nullptr, "seedx_gemv_fp8: gated needs even N and no residual");
  const int nb = batch <= 1 ? 1 : batch <= 2 ? 2 : batch <= 4 ? 4 : 8;
  SEEDX_REQUIRE(nb == batch, "seedx_gemv_fp8: batch must be 1, 2, 4 or 8 (pad the sequence slots)");
  const size_t smem = (size_t)nb * (K + 8) * 2;
  SEEDX_REQUIRE(smem <= 216 * 1024, "seedx_gemv_fp8: batch*K = %d*%lld does not fit in shared memory", nb, (long long)K);
  const long long tiles = (N + GEMV_ROWS - 1) / GEMV_ROWS;
  long long blocks = num_sms();
  if (blocks > tiles) blocks = tiles;
  cudaStream_t st = (cudaStream_t)stream;
#define GEMV8_LAUNCH(NBV)                                                                                                              \
  do {                                                                                                                                 \
    static bool attr = false;                                                                                                          \
    if (!attr) {                                                                                                                       \
      SEEDX_CUDA(cudaFuncSetAttribute(gemv_fp8_kernel<NBV>, cudaFuncAttributeMaxDynamicSharedMemorySize, 216 * 1024));                 \
      attr = true;                                                                                                                     \
    }                                                                                                                                  \
    launch_k(gemv_fp8_kernel<NBV>, (unsigned)blocks, GEMV_THREADS, smem, st, (const uint8_t*)W8, row_scale, x, ldx, rms_w, eps, residual, \
             ldr, out, ldo, (int)N, (int)K, gated);                                                                                    \
  } while (0)
  if (nb == 1) GEMV8_LAUNCH(1);
  else if (nb == 2) GEMV8_LAUNCH(2);
  else if (nb == 4) GEMV8_LAUNCH(4);
  else GEMV8_LAUNCH(8);
#undef GEMV8_LAUNCH
  count_launch();
  return check_cuda(cudaGetLastError(), "gemv_fp8 launch");
}

extern "C" int seedx_dequant_fp8(const void* W8, const float* row_scale, void* out, int64_t N, int64_t K, void* stream) {
  SEEDX_REQUIRE(W8 && row_scale && out, "seedx_dequant_fp8: null pointer");
  SEEDX_REQUIRE(N > 0 && K > 0 && K % 16 == 0, "seedx_dequant_fp8: K=%lld must be a positive multiple of 16", (long long)K);
  SEEDX_REQUIRE((uintptr_t)W8 % 16 == 0 && (uintptr_t)out % 16 == 0, "seedx_dequant_fp8: W8 and out must be 16B aligned");
  const long long chunks = N * (K / 16);
  launch_k(dequant_fp8_kernel, ew_grid(chunks, 256), 256, 0, (cudaStream_t)stream, (const uint4*)W8, row_scale, (uint4*)out, chunks, (int)(K / 16));
  count_launch();
  return check_cuda(cudaGetLastError(), "dequant_fp8 launch");
}

extern "C" int seedx_decode_attention(const float* qkv, const int32_t* state, const float* inv_freq, void* kcache, void* vcache,
                                      int64_t cache_stride, float* out, int batch, int heads, int head_dim, float scale, void* stream) {
  SEEDX_REQUIRE(qkv && state && inv_freq && kcache && vcache && out && batch >= 1, "seedx_decode_attention: bad arguments");
  SEEDX_REQUIRE(head_dim == 128, "seedx_decode_attention: head_dim must be 128 (LLaMA)");
  launch_k(decode_attn_kernel, dim3(heads, batch), DA_THREADS, 0, (cudaStream_t)stream, qkv, state, inv_freq, (__half*)kcache, (__half*)vcache,
                                                                                  (long long)cache_stride, out, heads, scale, (const int*)nullptr, 0, 0);
  count_launch();
  return check_cuda(cudaGetLastError(), "decode_attention launch");
}

static int log2_exact(int64_t v) {
  int s = 0;
  while ((1ll << s) < v) ++s;
  return (1ll << s) == v ? s : -1;
}

extern "C" int seedx_decode_attention_paged(const float* qkv, const int32_t* state, const float* inv_freq, void* kpool, void* vpool,
                                            const int32_t* page_table, int64_t table_stride, int64_t page_size, float* out, int batch, int heads,
                                            int head_dim, float scale, void* stream) {
  SEEDX_REQUIRE(qkv && state && inv_freq && kpool && vpool && page_table && out && batch >= 1, "seedx_decode_attention_paged: bad arguments");
  SEEDX_REQUIRE(head_dim == 128, "seedx_decode_attention_paged: head_dim must be 128 (LLaMA)");
  const int shift = log2_exact(page_size);
  SEEDX_REQUIRE(shift >= 0 && table_stride >= 1, "seedx_decode_attention_paged: page_size=%lld must be a power of two", (long long)page_size);
  launch_k(decode_attn_kernel, dim3(heads, batch), DA_THREADS, 0, (cudaStream_t)stream, qkv, state, inv_freq, (__half*)kpool, (__half*)vpool, 0ll, out,
                                                                                  heads, scale, (const int*)page_table, (int)table_stride, shift);
  count_launch();
  return check_cuda(cudaGetLastError(), "decode_attention_paged launch");
}

extern "C" int seedx_rope_kv_prefill(void* qkv, int64_t tokens, int64_t pos0, int heads, int head_dim, const float* inv_freq, void* kcache,
                                     void* vcache, void* stream) {
  SEEDX_REQUIRE(qkv && inv_freq && kcache && vcache && tokens > 0, "seedx_rope_kv_prefill: bad arguments");
  SEEDX_REQUIRE(head_dim == 128, "seedx_rope_kv_prefill: head_dim must be 128 (LLaMA)");
  launch_k(rope_kv_prefill_kernel, ew_grid(tokens * heads * 64, 256), 256, 0, (cudaStream_t)stream, (__half*)qkv, (int)tokens, (int)pos0, heads, inv_freq,
                                                                                             (__half*)kcache, (__half*)vcache, (const int*)nullptr, 0);
  count_launch();
  return check_cuda(cudaGetLastError(), "rope_kv_prefill launch");
}

extern "C" int seedx_rope_kv_prefill_paged(void* qkv, int64_t tokens, int64_t pos0, int heads, int head_dim, const float* inv_freq, void* kpool,
                                           void* vpool, const int32_t* page_table_row, int64_t page_size, void* stream) {
  SEEDX_REQUIRE(qkv && inv_freq && kpool && vpool && page_table_row && tokens > 0, "seedx_rope_kv_prefill_paged: bad arguments");
  SEEDX_REQUIRE(head_dim == 128, "seedx_rope_kv_prefill_paged: head_dim must be 128 (LLaMA)");
  const int shift = log2_exact(page_size);
  SEEDX_REQUIRE(shift >= 0, "seedx_rope_kv_prefill_paged: page_size=%lld must be a power of two", (long long)page_size);
  launch_k(rope_kv_prefill_kernel, ew_grid(tokens * heads * 64, 256), 256, 0, (cudaStream_t)stream, (__half*)qkv, (int)tokens, (int)pos0, heads, inv_freq,
                                                                                             (__half*)kpool, (__half*)vpool, (const int*)page_table_row, shift);
  count_launch();
  return check_cuda(cudaGetLastError(), "rope_kv_prefill_paged launch");
}

extern "C" int seedx_embed_rows(const void* table, const int32_t* ids, const int32_t* state, const int32_t* seq, int64_t seq_stride, int64_t n,
                                int64_t dim, float* out, void* stream) {
  SEEDX_REQUIRE(table && out && n > 0 && (ids || (state && seq)), "seedx_embed_rows: bad arguments");
  launch_k(embed_rows_kernel, ew_grid(n * dim, 256), 256, 0, (cudaStream_t)stream, (const __half*)table, ids, state, seq, (int)seq_stride, (int)n,
                                                                             (int)dim, out);
  count_launch();
  return check_cuda(cudaGetLastError(), "embed_rows launch");
}

extern "C" int seedx_scatter_rows(const void* src, int src_dtype, const int32_t* src_idx, const int32_t* idx, int64_t n, int64_t dim, float* dst,
                                  void* stream) {
  SEEDX_REQUIRE(src && idx && dst && n > 0, "seedx_scatter_rows: bad arguments");
  const int g = ew_grid(n * dim, 256);
  if (src_dtype == SEEDX_F32) launch_k(scatter_rows_kernel<float>, g, 256, 0, (cudaStream_t)stream, (const float*)src, src_idx, idx, (int)n, (int)dim, dst);
  else if (src_dtype == SEEDX_F16) launch_k(scatter_rows_kernel<__half>, g, 256, 0, (cudaStream_t)stream, (const __half*)src, src_idx, idx, (int)n, (int)dim, dst);
  else SEEDX_REQUIRE(false, "seedx_scatter_rows: bad dtype");
  count_launch();
  return check_cuda(cudaGetLastError(), "scatter_rows launch");
}

extern "C" int seedx_store_hidden(const float* x, const int32_t* state, int batch, int64_t max_rows, int64_t dim, float* hidden, void* stream) {
  SEEDX_REQUIRE(x && state && hidden && batch >= 1, "seedx_store_hidden: bad arguments");
  launch_k(store_hidden_kernel, dim3(ew_grid(dim, 256), batch), 256, 0, (cudaStream_t)stream, x, state, (int)max_rows, (int)dim, hidden);
  count_launch();
  return check_cuda(cudaGetLastError(), "store_hidden launch");
}

extern "C" int seedx_logits_argmax(float* logits, int64_t vocab, const int32_t* img_ids, int n_img_ids, int32_t* seq, int32_t* state, int batch,
                                   int eos_id, int suppress_eos, int64_t max_len, void* stream) {
  SEEDX_REQUIRE(logits && seq && state && vocab > 0 && batch >= 1, "seedx_logits_argmax: bad arguments");
  SEEDX_REQUIRE(n_img_ids >= 0 && n_img_ids <= 1024, "seedx_logits_argmax: too many image token ids");
  launch_k(logits_argmax_kernel, batch, 1024, 0, (cudaStream_t)stream, logits, (int)vocab, img_ids, n_img_ids, seq, state, eos_id, suppress_eos, (int)max_len);
  count_launch();
  return check_cuda(cudaGetLastError(), "logits_argmax launch");
}
