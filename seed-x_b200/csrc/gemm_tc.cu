// seedx-b200: wgmma tensor-core GEMM / implicit-GEMM convolution for sm_90a.
//
//   D[b][m][n] = epi( alpha * sum_k A[b][m][k] * B[b][n][k] )      fp16 operands, fp32 accumulate in registers
//   D[m][n]    = epi( alpha * acc[m][n] * a_scale[m] * b_scale[n] )  FP8 variant (seedx_gemm_fp8): e4m3 operands, per-row scales
//
// Persistent, warp-specialised: warpgroup 0 = TMA producer, warpgroups 1 and 2 = wgmma on 64 rows each of the 128-row tile, then the epilogue.
// Operands are staged by TMA into 128B-swizzled K-major tiles (BM=128 x BK=64, BN x BK=64) through a
// STAGES-deep mbarrier ring; the producer keeps filling it with the next tile's k-blocks while the consumers run
// the epilogue of the current one.  In conv mode the A tile of k-step (tap, channel-chunk) is a
// shifted [th x tw] pixel window of the NHWC image fetched by a 4-D tensor map, out-of-bounds = zero padding
// (im2col-free implicit GEMM).
//
// Reference call sites replaced: see include/seedx.h (seedx_gemm_f16).
#include <cuda_fp8.h>
#include <math.h>
#include <cstdlib>
#include <type_traits>

#include "common.cuh"
#include "wgmma.cuh"
#include "../../include/seedx.h"

namespace seedx {

struct GemmParams {
  void* D;
  const float* bias_n;
  const float* bias_m;
  const float* bias_g;
  const void* residual;
  int M, N, K;
  int batch;
  int m_blocks, n_blocks, k_blocks;
  long long ldd, strideD, ldr, strideR;
  int res_row_mod, bias_g_rows;
  float alpha;
  int act, gated, out_f32, res_f32, vec_ok, b_batched, bias_vec;
  int tma_epi, epi_row_bytes, r_batched;  // TMA epilogue: output (and residual) tiles of 32 rows x epi_row_bytes staged in shared memory
  unsigned long long* dbg;                // optional per-CTA phase timestamps (%globaltimer ns), 8 slots per CTA; NULL in production
  int epi_out_bytes, epi_res_bytes;       // per-warp staging split: output buffers | residual buffers (host policy, see seedx_gemm_f16)
  int stages, epi_warp_bytes;             // pipeline depth and per-epilogue-warp staging bytes, sized on the host to fill shared memory
  // LayerNorm folded into the epilogue (A = the un-normalised rows, B = gamma-scaled weights): x = rstd[m] * (acc - mean[m] * colsum[n])
  const float2* ln_stats;                 // [M] (mean, rstd) or NULL
  const float* ln_colsum;                 // [N] sum_k B[n][k]
  int b_static;                           // B does not depend on the preceding kernel (weights): its first tiles are requested before the PDL wait
  int ln_parts;                           // > 0: ln_stats holds ln_parts x [M] (sum, sum of squares) partials written by the producer of A (row_part)
  float ln_eps, ln_inv_cols;
  // statistics of the STORED output, emitted by the epilogue for the normalisation that reads it next (fp16 output, TMA epilogue only):
  // stream-K schedule (host: seedx_gemm_set_workspace): every cluster takes an equal share of the linearised (tile, k-block) iterations; a
  // cluster that starts inside a tile writes its raw fp32 partial accumulator to sk_scratch[cluster], the cluster that holds the tile's first
  // k-block adds those partials in cluster order before its normal epilogue (fixed order: bit-reproducible)
  int stream_k;
  float* sk_scratch;                      // [clusters][CL][128][BN] fp32
  unsigned* sk_flags;                     // [clusters][CL][EPI_WARPS], 0 between launches
  float2* row_part;                       // [N/32][M]  per row:    (sum, sumsq) over the 32 columns of a chunk      -> LayerNorm of the next GEMM
  float2* col_part;                       // [M/32][N]  per column: (sum, sumsq) over the 32 rows of a warp's slab   -> GroupNorm (fixed-order finalize)
  // optional: the warp that delivers the LAST partial of a 32-row slab (ticket per slab, self-resetting) turns the slab's row partials into
  // (mean, rstd) right here, in chunk order (deterministic whoever comes last): no separate finalize launch for the consumer's folded LayerNorm
  float2* row_stats_out;                  // [M] (mean, rstd)
  unsigned* row_tickets;                  // [M/32], zero before the launch, zero again after it
  float row_eps;
  // conv
  int conv, taps_w, c_chunks, conv_w, conv_h, tile_w, tile_h, tiles_per_img, tiles_w, pad, imgs_per_tile;
  // FP8 (e4m3) operands only: the accumulator is scaled by a_scale[m] * b_scale[n] before the rest of the epilogue
  const float* a_scale;                   // [M]
  const float* b_scale;                   // [N]
};

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int A_STAGE_BYTES = BM * BK * 2;

constexpr int EPI_WARPS = 8;                       // the two consumer warpgroups: 64 accumulator rows each, then the epilogue of those rows
constexpr int GEMM_THREADS = 128 + EPI_WARPS * 32; // warpgroup 0 = TMA producer (one thread), warpgroups 1, 2 = MMA + epilogue
constexpr int SMEM_LIMIT = 227 * 1024;
constexpr int EPI_OUT_BYTES = 4096;                      // per epilogue warp: output tiles (2 x <=2 KB, or 1 x 4 KB)
constexpr int EPI_RES_BYTES = 8192;                      // per epilogue warp: residual tiles, ideally every chunk of a 256-wide tile in flight
constexpr int MAX_STAGES = 8;
constexpr int VEC_BYTES = 1024;                          // one per-tile column vector of the epilogue (bias_n | LayerNorm column sums | FP8 b_scale), 256 fp32
constexpr int BK_FP8 = 128;                              // e4m3 K elements per stage: 128 bytes per row, the same tile bytes and swizzle as 64 fp16
// The epilogue works on rows of 32 accumulator columns (lane = row).  The accumulators live in the wgmma fragment layout (a thread holds 2 rows x
// 2 columns of every 8-column group), so each warpgroup passes 64 columns at a time through shared memory: 64 rows x ACC_LD fp32.
// ACC_LD = 72: the fragment's 8-byte stores hit 32 distinct banks per half warp.
constexpr int ACC_LD = 72;
constexpr int ACC_WG_BYTES = 64 * ACC_LD * 4;
constexpr int ACC_STAGE_BYTES = 2 * ACC_WG_BYTES;

template <int BN, int CL = 1>
struct TileCfg {
  static_assert(BN % 16 == 0 && BN >= 32 && BN <= 256, "wgmma N: multiple of 16, <= 256");
  static constexpr int B_STAGE_BYTES = BN * BK * 2;   // in a cluster pair each CTA loads half of it and multicasts that half to both
  static constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
  // pipeline depth for a given amount of epilogue staging (runtime: depends on whether a residual is streamed through shared memory)
  // `tail_bytes` = barriers (512) + the per-tile epilogue vectors (1 KB per vector in use).  The dynamic shared memory is declared 1024-byte
  // aligned (the 128-byte-swizzled tiles need it), so no alignment slack is budgeted.
  static int stages_for(int epi_bytes, int tail_bytes) {
    const int fit = (SMEM_LIMIT - tail_bytes - epi_bytes - ACC_STAGE_BYTES) / STAGE_BYTES;
    return fit > MAX_STAGES ? MAX_STAGES : fit;
  }
  static int smem_for(int stages, int epi_bytes, int tail_bytes) { return stages * STAGE_BYTES + ACC_STAGE_BYTES + epi_bytes + tail_bytes; }
};

SEEDX_DEVINL unsigned long long gtime_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;\n" : "=l"(t));
  return t;
}
#define GEMM_STAMP(slot) do { if (p.dbg != nullptr) p.dbg[(size_t)blockIdx.x * 8 + (slot)] = gtime_ns(); } while (0)

SEEDX_DEVINL float apply_act(float x, int act) {
  if (act == SEEDX_ACT_GELU_ERF) return gelu_erf_fast(x);
  if (act == SEEDX_ACT_SILU) return silu(x);
  return x;
}

// Work list of one cluster: segments (tile, k-blocks [kb0, kb1)).  Data-parallel: whole tiles first, first + step, ...  Stream-K: the
// iterations [it, it1) of the linearised (tile, k-block) space, cut at tile boundaries.
// SK is a compile-time property of the kernel, so that the data-parallel launches (the large majority) carry none of the stream-K code.
struct SegState {
  long long it, it1;
  int t_next;
};
template <bool SK>
SEEDX_DEVINL SegState seg_init(const GemmParams& p, int cluster, int n_clusters, int num_tiles) {
  SegState s;
  s.t_next = cluster;
  const long long total = (long long)num_tiles * p.k_blocks;
  s.it = SK ? (long long)cluster * total / n_clusters : 0;
  s.it1 = SK ? (long long)(cluster + 1) * total / n_clusters : 0;
  return s;
}
template <bool SK>
SEEDX_DEVINL bool seg_next(const GemmParams& p, SegState& s, int n_clusters, int num_tiles, int& t, int& kb0, int& kb1) {
  if (SK) {
    if (s.it >= s.it1) return false;
    t = (int)(s.it / p.k_blocks);
    kb0 = (int)(s.it - (long long)t * p.k_blocks);
    const long long left = s.it1 - s.it;
    kb1 = (left < (long long)(p.k_blocks - kb0)) ? kb0 + (int)left : p.k_blocks;
    s.it += kb1 - kb0;
    return true;
  }
  if (s.t_next >= num_tiles) return false;
  t = s.t_next, s.t_next += n_clusters, kb0 = 0, kb1 = p.k_blocks;
  return true;
}

// CL = CTAs per cluster (1, or 2 = two CTAs on vertically adjacent 128 x BN tiles of the same column block).  In a pair each CTA loads its own
// 128 rows of A and HALF of the B tile, which TMA multicasts into both CTAs' shared memory: each SM fetches a quarter fewer operand bytes from L2.
// A stage of a CTA is refilled only when the consumers of BOTH CTAs have released it (the peer writes into it), so every consumer warpgroup
// arrives on the `empty` barriers of both CTAs.
// TE = operand element type: __half, or __nv_fp8_e4m3 (single CTA, data-parallel, batch 1 only: the host never instantiates FP8 with CL = 2 or
// stream-K).  Every FP8 difference is under `if constexpr`, so the fp16 kernels are the same code with or without it.
// CONV8 = the FP8 implicit-GEMM conv (seedx_conv_fp8; TE = e4m3, conv mode): the A window advances 128 channels per stage, every 128-element
// k-block is accumulated by its own MMAs from zero and then added into the fp32 accumulator (promotion: the FP8 wgmma does not keep full fp32
// over long K), and row m takes the scale of its image, a_scale[m / (H*W)].  Only the FP8 conv instantiations set it.
template <int BN, int CL, bool SK, typename TE = __half, bool CONV8 = false>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmD,
               const __grid_constant__ CUtensorMap tmR, const GemmParams p) {
  using Cfg = TileCfg<BN, CL>;
  constexpr bool FP8 = std::is_same<TE, __nv_fp8_e4m3>::value;
  static_assert(!CONV8 || (FP8 && CL == 1 && !SK), "the FP8 conv is single-CTA, data-parallel");
  constexpr int KB = FP8 ? BK_FP8 : BK;   // K elements per stage (TMA box coordinate step)
  const int STAGES = p.stages;
  if (threadIdx.x == 0) GEMM_STAMP(0);
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t smem_base = smem_u32(smem_raw);
  if ((smem_base & 1023u) != 0u) __trap();                          // the launch budgets no alignment slack (TileCfg::smem_for)
  const uint32_t acc_base = smem_base + STAGES * Cfg::STAGE_BYTES;  // accumulator hand-over, ACC_WG_BYTES per consumer warpgroup
  const uint32_t epi_base = acc_base + ACC_STAGE_BYTES;             // 1024-aligned
  const uint32_t bar_base = epi_base + (uint32_t)(EPI_WARPS * p.epi_warp_bytes);
  // barrier layout (8 B each): full[STAGES], empty[STAGES], residual[EPI_WARPS][4]
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (STAGES + s); };
  auto res_bar = [&](int w, int i) { return bar_base + 8u * (2 * STAGES + 4 * w + i); };  // residual tile landed (per epilogue warp, <= 4 buffers)
  const uint32_t vec_base = bar_base + 512u;       // [bias_n tile | colsum tile | FP8: b_scale tile], 256 fp32 each: staged once per tile, read as broadcast 128-bit loads

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int crank = (CL > 1) ? (int)cluster_ctarank() : 0;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 2 * CL);  // one arrival per consumer warpgroup of every CTA that reads this CTA's B half
    }
    for (int w = 0; w < EPI_WARPS; ++w)
      for (int i = 0; i < 4; ++i) mbar_init(res_bar(w, i), 1);
    mbar_fence_init();
  }
  __syncthreads();
  if (CL > 1) cluster_sync_all();  // peer barriers are initialised before any remote arrive / multicast transaction can reach them
  if (threadIdx.x == 0) GEMM_STAMP(1);
  // tile space: (batch, n block, m group) with CL consecutive m blocks per group; a cluster walks groups, CTA `crank` takes m = group*CL + crank
  const int m_groups = (p.m_blocks + CL - 1) / CL;
  const int tiles_per_batch = m_groups * p.n_blocks;
  const int num_tiles = tiles_per_batch * p.batch;
  const int tile0 = (int)blockIdx.x / CL, tile_step = (int)gridDim.x / CL;
  // B half of a stage: rows [n_blk*BN + crank*BN/CL, +BN/CL), at the same offset in every CTA of the cluster
  auto load_b = [&](uint32_t sb, uint32_t bar, int kb, int n_blk, int b) {
    if (CL == 1) tma_load_3d(sb, &tmB, bar, kb * KB, n_blk * BN, p.b_batched ? b : 0);
    else tma_load_3d_mc(sb + (uint32_t)(crank * (BN / CL) * BK * 2), &tmB, bar, kb * KB, n_blk * BN + crank * (BN / CL), p.b_batched ? b : 0,
                        (uint16_t)((1u << CL) - 1u));
  };
  // Weights never depend on the kernel before this one: the B tiles of the first stages of this CTA's first tile are requested BEFORE the
  // dependency wait (their bytes are already counted on the `full` barriers; the A tiles follow after the wait).
  int b_pre = 0;
  {
    SegState s0 = seg_init<SK>(p, tile0, tile_step, num_tiles);
    int t, kb0, kb1;
    if (p.b_static && seg_next<SK>(p, s0, tile_step, num_tiles, t, kb0, kb1)) {
      b_pre = (kb1 - kb0) < STAGES ? (kb1 - kb0) : STAGES;
      if (warp == 0 && lane == 0) {
        const int b = t / tiles_per_batch;
        const int n_blk = (t - b * tiles_per_batch) / m_groups;
        for (int i = 0; i < b_pre; ++i) {
          mbar_expect_tx(full_bar(i), Cfg::STAGE_BYTES);
          load_b(smem_base + i * Cfg::STAGE_BYTES + A_STAGE_BYTES, full_bar(i), kb0 + i, n_blk, b);
        }
      }
    }
  }
  // everything above touched only this CTA's shared memory (and weights): under programmatic dependent launch it ran while the previous
  // kernel was still draining.  Operands, residual and output may be that kernel's data: wait for it here.
  pdl_wait();
  pdl_trigger();
  if (threadIdx.x == 0) GEMM_STAMP(2);

  if (warp < 4) {
    // ------------------------------------------------ TMA producer
    setmaxnreg_dec<40>();
    if (warp == 0 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      SegState ss = seg_init<SK>(p, tile0, tile_step, num_tiles);
      int t, kb0, kb1;
      bool first_seg = true;
      while (seg_next<SK>(p, ss, tile_step, num_tiles, t, kb0, kb1)) {
        const int b = t / tiles_per_batch;
        const int r = t - b * tiles_per_batch;
        const int n_blk = r / m_groups;
        const int m_blk = (r - n_blk * m_groups) * CL + crank;
        int img = 0, h0 = 0, w0 = 0;
        if (p.conv) {
          if (p.imgs_per_tile > 1) {
            img = m_blk * p.imgs_per_tile;  // whole images per tile; images past the end are TMA zero fill
          } else {
            img = m_blk / p.tiles_per_img;
            const int rem = m_blk - img * p.tiles_per_img;
            const int th_i = rem / p.tiles_w;
            h0 = th_i * p.tile_h;
            w0 = (rem - th_i * p.tiles_w) * p.tile_w;
          }
        }
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(empty_bar(stage), phase ^ 1u);
          const uint32_t sa = smem_base + stage * Cfg::STAGE_BYTES;
          const uint32_t sb = sa + A_STAGE_BYTES;
          const bool b_done = first_seg && (kb - kb0 < b_pre);   // this stage's barrier is armed and its B tile is in flight already
          if (!b_done) mbar_expect_tx(full_bar(stage), Cfg::STAGE_BYTES);
          if (p.conv) {
            const int tap = kb / p.c_chunks;
            const int cc = kb - tap * p.c_chunks;
            const int kh = tap / p.taps_w;
            const int kw = tap - kh * p.taps_w;
            tma_load_4d(sa, &tmA, full_bar(stage), cc * (CONV8 ? BK_FP8 : BK), w0 + kw - p.pad, h0 + kh - p.pad, img);
          } else {
            tma_load_3d(sa, &tmA, full_bar(stage), kb * KB, m_blk * BM, b);
          }
          if (!b_done) load_b(sb, full_bar(stage), kb, n_blk, b);
          if (++stage == STAGES) {
            stage = 0;
            phase ^= 1u;
          }
        }
        first_seg = false;
      }
    }
  } else {
    // ------------------------------------------------ consumer warpgroups: wgmma main loop (accumulator in registers), then the epilogue
    setmaxnreg_inc<232>();
    const int ew = warp - 4;                  // epilogue warp 0..7
    const int wg = ew >> 2;                   // accumulator rows [64*wg, +64) of the tile
    const int q = ew & 3;                     // warp of the warpgroup
    const int lane_grp = 2 * wg + (q & 1);    // epilogue rows [32*lane_grp, +32): lane = row
    const int chunk0 = (q >> 1) * 32;         // warps 0, 1 of a warpgroup take the even 32-column chunks, warps 2, 3 the odd ones
    const uint32_t acc_wg = acc_base + (uint32_t)(wg * ACC_WG_BYTES);
    const int tq = (threadIdx.x & 127);       // thread of the warpgroup
    const int frag_row = 16 * q + (lane >> 2);
    float acc[BN / 2];
    int stage = 0;
    uint32_t phase = 0;
    uint32_t epi_res_phase = 0;   // parity bits of this warp's residual barriers
    int vec_nblk = -1;            // column block whose bias / column-sum vectors sit in shared memory
    SegState ss = seg_init<SK>(p, tile0, tile_step, num_tiles);
    int t, kb0, kb1;
    bool first_seg = true;
    // release a stage: this warpgroup is done reading it (in a pair, the peer's producer writes its B half into it too)
    auto release = [&](int s) {
      if (tq == 0) {
        if (CL == 1) mbar_arrive(empty_bar(s));
        else
          for (int c = 0; c < CL; ++c) mbar_arrive_cluster(mapa_cluster(empty_bar(s), (uint32_t)c));
      }
    };
    while (seg_next<SK>(p, ss, tile_step, num_tiles, t, kb0, kb1)) {
      const int b = t / tiles_per_batch;
      const int r = t - b * tiles_per_batch;
      const int n_blk = r / m_groups;
      const int m_blk = (r - n_blk * m_groups) * CL + crank;
      const int row = m_blk * BM + lane_grp * 32 + lane;
      const bool row_ok = row < p.M;
      const int n0 = n_blk * BN;

      // ---- main loop: the MMAs of k-block kb are in flight while the stage of kb-1 is released
      {
        int prev = -1;
        if constexpr (CONV8) {
#pragma unroll
          for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
        }
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(full_bar(stage), phase);
          if (first_seg && kb == kb0 && ew == 0 && lane == 0) GEMM_STAMP(3);
          const uint32_t sa = smem_base + stage * Cfg::STAGE_BYTES + (uint32_t)(wg * 64 * BK * 2);
          const uint64_t adesc = wgmma_desc_k_sw128(sa);
          const uint64_t bdesc = wgmma_desc_k_sw128(smem_base + stage * Cfg::STAGE_BYTES + A_STAGE_BYTES);
          if constexpr (CONV8) {
            // promotion: the four QGMMAs of this 128-element k-block sum into `blk` from zero (scale-d = 0 on the first), their result is
            // waited for, the stage goes back to the producer and the block sum is added into the fp32 accumulator by the CUDA cores.
            // The other consumer warpgroup's MMAs keep the tensor core busy meanwhile.
            float blk[BN / 2];
            wgmma_fence_regs<BN / 2>(blk);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < BK / 16; ++k) wgmma_ss_e4m3<BN>(blk, adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), k != 0);
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_fence_regs<BN / 2>(blk);
            release(stage);
#pragma unroll
            for (int i = 0; i < BN / 2; ++i) acc[i] += blk[i];
            if (++stage == STAGES) {
              stage = 0;
              phase ^= 1u;
            }
            continue;
          }
          wgmma_fence_regs<BN / 2>(acc);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < BK / 16; ++k) {  // advance 16 fp16 (or 32 e4m3) = 32 B inside the 128B swizzle atom: +2 in the (addr >> 4) field
            if constexpr (FP8) wgmma_ss_e4m3<BN>(acc, adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), ((kb - kb0) | k) != 0);
            else wgmma_ss_n<BN>(acc, adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), ((kb - kb0) | k) != 0);
          }
          wgmma_commit();
          wgmma_wait<1>();
          wgmma_fence_regs<BN / 2>(acc);
          if (prev >= 0) release(prev);
          prev = stage;
          if (++stage == STAGES) {
            stage = 0;
            phase ^= 1u;
          }
        }
        wgmma_wait<0>();
        wgmma_fence_regs<BN / 2>(acc);
        if (prev >= 0) release(prev);
      }
      if (ew == 0 && lane == 0) {
        if (first_seg) GEMM_STAMP(4);
        GEMM_STAMP(5);                                 // overwritten every tile: the last tile's value survives
      }
      // columns [cp, cp + 64) of this warpgroup's accumulator -> shared memory (64 rows x ACC_LD), then every warp reads back its row x 32 columns
      auto stage_acc = [&](int cp) {
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          if (8 * j >= cp && 8 * j < cp + 64) {
            const uint32_t a = acc_wg + 4u * (uint32_t)(frag_row * ACC_LD + 8 * j - cp + 2 * (lane & 3));
            asm volatile("st.shared.v2.f32 [%0], {%1, %2};\n" ::"r"(a), "f"(acc[4 * j]), "f"(acc[4 * j + 1]) : "memory");
            asm volatile("st.shared.v2.f32 [%0], {%1, %2};\n" ::"r"(a + 8u * ACC_LD * 4u), "f"(acc[4 * j + 2]), "f"(acc[4 * j + 3]) : "memory");
          }
        }
      };
      auto load_acc = [&](uint32_t (&v)[32]) {
        const uint32_t a = acc_wg + 4u * (uint32_t)(((q & 1) * 32 + lane) * ACC_LD + chunk0);
#pragma unroll
        for (int i = 0; i < 32; i += 4) {
          const uint4 u = lds128(a + 4u * (uint32_t)i);
          v[i] = u.x, v[i + 1] = u.y, v[i + 2] = u.z, v[i + 3] = u.w;
        }
      };
      const int col_end = min(p.N, n0 + BN);   // columns of this tile that exist
      // walk the 64-column slices of the accumulator (warpgroup-uniform); fn(c) handles this warp's 32-column chunk c when it exists
      auto for_each_chunk = [&](auto&& fn) {
        for (int cp = 0; cp < BN && n0 + cp < col_end; cp += 64) {
          stage_acc(cp);
          named_bar_sync(2 + wg, 128);
          const int c = cp + chunk0;
          if (c < BN && n0 + c < col_end) fn(c);
          named_bar_sync(2 + wg, 128);           // the slice is consumed before the next one overwrites it
        }
      };

      const float bm = (p.bias_m != nullptr && row_ok) ? p.bias_m[row] : 0.f;
      float a_s = 1.f;                         // FP8: the scale of this lane's row of A
      if constexpr (CONV8) a_s = row_ok ? __ldg(p.a_scale + row / (p.conv_h * p.conv_w)) : 0.f;   // one scale per image (rows = pixels)
      else if constexpr (FP8) a_s = row_ok ? __ldg(p.a_scale + row) : 0.f;
      float ln_rstd = 1.f, ln_nmr = 0.f;       // folded LayerNorm: x = rstd * acc + (-mean * rstd) * colsum[n]
      if (p.ln_stats != nullptr && row_ok) {
        float2 mr;
        if (p.ln_parts > 0) {      // partial sums of the row, one per 32-column chunk of the producing GEMM, added in chunk order
          float s1 = 0.f, s2 = 0.f;
          for (int k = 0; k < p.ln_parts; ++k) {
            const float2 qq = __ldcg(p.ln_stats + (long long)k * p.M + row);
            s1 += qq.x, s2 += qq.y;
          }
          const float mean = s1 * p.ln_inv_cols;
          mr = make_float2(mean, rsqrtf(fmaxf(s2 * p.ln_inv_cols - mean * mean, 0.f) + p.ln_eps));
        } else {
          mr = __ldg(p.ln_stats + row);
        }
        ln_rstd = mr.y, ln_nmr = -mr.x * mr.y;
      }
      // per-row-group bias (time embedding of a ResnetBlock2D): when the 128 rows of this CTA's tile lie in one group (bias_g_rows % 128 == 0) it is
      // folded into the staged bias vector; otherwise every value fetches its own element
      const bool bg_vec = p.bias_g != nullptr && (p.bias_g_rows % BM) == 0;
      const int bg_grp = p.bias_g != nullptr ? (m_blk * BM) / p.bias_g_rows : 0;
      const float* bg = (p.bias_g != nullptr && row_ok && !bg_vec) ? p.bias_g + (long long)(row / p.bias_g_rows) * p.N : nullptr;
      const int rrow = p.res_row_mod ? (row % p.res_row_mod) : row;

      // ---- TMA epilogue state: tiles of 32 rows x RB bytes in this warp's staging area, XOR-swizzled like the tensor maps
      const uint32_t stg_out = epi_base + (uint32_t)(ew * p.epi_warp_bytes), stg_res = stg_out + (uint32_t)p.epi_out_bytes;
      const int RB = p.epi_row_bytes;
      const uint32_t tile_bytes = 32u * (uint32_t)RB;
      const int nbuf = (uint32_t)p.epi_out_bytes >= 4u * tile_bytes ? 4 : ((uint32_t)p.epi_out_bytes >= 2u * tile_bytes ? 2 : 1);   // output buffers
      int nres = (int)((uint32_t)p.epi_res_bytes / tile_bytes);     // residual buffers, at most 4 (barriers)
      nres = nres > 4 ? 4 : nres;
      const int row_base = m_blk * BM + lane_grp * 32;
      const bool tma_res = p.tma_epi && p.residual != nullptr;
      int n_chunks = 0;
      for (int c = chunk0; c < BN && n0 + c < col_end; c += 64) ++n_chunks;
      auto out_col = [&](int k) { const int col0 = n0 + chunk0 + 64 * k; return p.gated ? (col0 >> 1) : col0; };
      auto issue_res = [&](int k) {  // lane 0: fetch the residual tile of chunk k into residual buffer k % nres
        const int rb = k % nres;
        mbar_expect_tx(res_bar(ew, rb), tile_bytes);
        tma_load_3d(stg_res + (uint32_t)rb * tile_bytes, &tmR, res_bar(ew, rb), out_col(k), p.res_row_mod ? (row_base % p.res_row_mod) : row_base,
                    p.r_batched ? b : 0);
      };
      // ---- stream-K roles of this segment
      const bool sk_partial = SK && kb0 > 0;                          // the tile's first k-blocks belong to an earlier cluster: hand my raw sums over
      const bool sk_owner = SK && (kb0 == 0) && (kb1 < p.k_blocks);   // later clusters hold the rest of this tile: add their partials, then finish
      const int my_cluster = tile0;
      constexpr int BNP = (BN + 31) & ~31;                      // scratch row stride: the last 32-column chunk of a tile may reach past BN
      const size_t sk_tile_elems = (size_t)BM * BNP;
      if (sk_partial) {
        // layout of a slot: [BNP / 4 column quads][128 rows][4 floats]: the 32 lanes (= rows) of a store cover 512 contiguous bytes
        float* dst = p.sk_scratch + ((size_t)my_cluster * CL + crank) * sk_tile_elems + (size_t)(lane_grp * 32 + lane) * 4;
        for_each_chunk([&](int c) {
          uint32_t v[32];
          load_acc(v);
#pragma unroll
          for (int i = 0; i < 32; i += 4) *(uint4*)(dst + (size_t)((c + i) >> 2) * (BM * 4)) = make_uint4(v[i], v[i + 1], v[i + 2], v[i + 3]);
        });
        __threadfence();                                        // my stores are visible device-wide before the flag
        __syncwarp();
        if (lane == 0)
          asm volatile("st.release.gpu.global.u32 [%0], %1;\n" ::"l"(p.sk_flags + ((size_t)my_cluster * CL + crank) * EPI_WARPS + ew), "r"(1u) : "memory");
        first_seg = false;
        continue;
      }
      int sk_last = my_cluster;                                 // contributors = clusters my_cluster+1 .. sk_last
      if (sk_owner) {
        const long long total = (long long)num_tiles * p.k_blocks;
        const long long tile_end = (long long)(t + 1) * p.k_blocks;
        while (sk_last + 1 < tile_step && (long long)(sk_last + 1) * total / tile_step < tile_end) ++sk_last;
      }
      if (tma_res && lane == 0)
        for (int k = 0; k < nres && k < n_chunks; ++k) issue_res(k);
      // column vectors of this tile -> shared memory: the chunk loop then reads them with broadcast 128-bit shared loads instead of dependent
      // L1/L2 round trips per chunk
      const int vec_key = n_blk + (bg_vec ? (bg_grp + 1) * 65536 : 0);
      const bool use_vec = (p.bias_n != nullptr || p.ln_stats != nullptr || bg_vec || FP8) && vec_key != vec_nblk;   // consecutive tiles of a CTA mostly differ in m only
      if (use_vec) {
        vec_nblk = vec_key;
        named_bar_sync(1, EPI_WARPS * 32);      // every epilogue warp has finished reading the previous tile's vectors
        for (int i = ew * 32 + lane; i < BN; i += EPI_WARPS * 32) {
          const bool in = n0 + i < col_end;
          float bv = (p.bias_n != nullptr && in) ? __ldg(p.bias_n + n0 + i) : 0.f;
          if (bg_vec && in && m_blk * BM < p.M) bv += __ldg(p.bias_g + (long long)bg_grp * p.N + n0 + i);
          const float cv = (p.ln_stats != nullptr && in) ? __ldg(p.ln_colsum + n0 + i) : 0.f;
          asm volatile("st.shared.f32 [%0], %1;\n" ::"r"(vec_base + 4u * (uint32_t)i), "f"(bv) : "memory");
          if (p.ln_stats != nullptr) asm volatile("st.shared.f32 [%0], %1;\n" ::"r"(vec_base + 1024u + 4u * (uint32_t)i), "f"(cv) : "memory");
          if constexpr (FP8) {
            const float sv = in ? __ldg(p.b_scale + n0 + i) : 0.f;
            asm volatile("st.shared.f32 [%0], %1;\n" ::"r"(vec_base + 2048u + 4u * (uint32_t)i), "f"(sv) : "memory");
          }
        }
        named_bar_sync(1, EPI_WARPS * 32);
      }
      int kchunk = 0;
      if (sk_owner) {                                  // the contributors wrote their partials at the START of their work: normally long done
        for (int cc = my_cluster + 1; cc <= sk_last; ++cc) {
          const unsigned* f = p.sk_flags + ((size_t)cc * CL + crank) * EPI_WARPS + ew;
          unsigned ready = 0;
          do {
            asm volatile("ld.acquire.gpu.global.u32 %0, [%1];\n" : "=r"(ready) : "l"(f) : "memory");
            if (!ready) __nanosleep(64);
          } while (!ready);
        }
        __syncwarp();
      }
      for_each_chunk([&](int c) {
        uint32_t v[32];
        load_acc(v);
        if (sk_owner) {            // partial sums of the later k-blocks, added in cluster order (fixed order: reproducible)
          for (int cc = my_cluster + 1; cc <= sk_last; ++cc) {
            const float* src = p.sk_scratch + ((size_t)cc * CL + crank) * sk_tile_elems + (size_t)(lane_grp * 32 + lane) * 4;
#pragma unroll
            for (int i = 0; i < 32; i += 4) {
              const float4 qv = __ldcg((const float4*)(src + (size_t)((c + i) >> 2) * (BM * 4)));
              v[i] = __float_as_uint(__uint_as_float(v[i]) + qv.x), v[i + 1] = __float_as_uint(__uint_as_float(v[i + 1]) + qv.y);
              v[i + 2] = __float_as_uint(__uint_as_float(v[i + 2]) + qv.z), v[i + 3] = __float_as_uint(__uint_as_float(v[i + 3]) + qv.w);
            }
          }
        }
        if constexpr (FP8) {       // acc <- (acc * a_scale[m]) * b_scale[n], then the fp16 epilogue below, unchanged
#pragma unroll
          for (int i = 0; i < 32; i += 4) {
            const uint4 qs = lds128(vec_base + 2048u + 4u * (uint32_t)(c + i));
            v[i] = __float_as_uint(__uint_as_float(v[i]) * a_s * __uint_as_float(qs.x));
            v[i + 1] = __float_as_uint(__uint_as_float(v[i + 1]) * a_s * __uint_as_float(qs.y));
            v[i + 2] = __float_as_uint(__uint_as_float(v[i + 2]) * a_s * __uint_as_float(qs.z));
            v[i + 3] = __float_as_uint(__uint_as_float(v[i + 3]) * a_s * __uint_as_float(qs.w));
          }
        }
        float x[32];
        const int col0 = n0 + c;
        if (p.ln_stats != nullptr) {
          // folded LayerNorm (alpha = 1, no bias_m: host check): x = rstd * acc + (bias - rstd * mean * colsum) -> two FFMAs per value
#pragma unroll
          for (int i = 0; i < 32; i += 4) {
            const uint4 qb = lds128(vec_base + 4u * (uint32_t)(c + i)), qc = lds128(vec_base + 1024u + 4u * (uint32_t)(c + i));
            x[i] = fmaf(__uint_as_float(v[i]), ln_rstd, fmaf(ln_nmr, __uint_as_float(qc.x), __uint_as_float(qb.x)));
            x[i + 1] = fmaf(__uint_as_float(v[i + 1]), ln_rstd, fmaf(ln_nmr, __uint_as_float(qc.y), __uint_as_float(qb.y)));
            x[i + 2] = fmaf(__uint_as_float(v[i + 2]), ln_rstd, fmaf(ln_nmr, __uint_as_float(qc.z), __uint_as_float(qb.z)));
            x[i + 3] = fmaf(__uint_as_float(v[i + 3]), ln_rstd, fmaf(ln_nmr, __uint_as_float(qc.w), __uint_as_float(qb.w)));
          }
        } else if (p.bias_n != nullptr || bg_vec) {
#pragma unroll
          for (int i = 0; i < 32; i += 4) {
            const uint4 qb = lds128(vec_base + 4u * (uint32_t)(c + i));
            x[i] = fmaf(__uint_as_float(v[i]), p.alpha, __uint_as_float(qb.x) + bm), x[i + 1] = fmaf(__uint_as_float(v[i + 1]), p.alpha, __uint_as_float(qb.y) + bm);
            x[i + 2] = fmaf(__uint_as_float(v[i + 2]), p.alpha, __uint_as_float(qb.z) + bm), x[i + 3] = fmaf(__uint_as_float(v[i + 3]), p.alpha, __uint_as_float(qb.w) + bm);
          }
        } else {
#pragma unroll
          for (int i = 0; i < 32; ++i) x[i] = fmaf(__uint_as_float(v[i]), p.alpha, bm);
        }
        if (bg != nullptr) {
#pragma unroll
          for (int i = 0; i < 32; ++i)
            if (col0 + i < col_end) x[i] += __ldg(bg + col0 + i);
        }
        int nvals = 32;
        int ocol0 = col0;
        // activation chosen once per chunk (warp-uniform), not once per value
        if (p.gated) {
          if (p.act == SEEDX_ACT_GELU_ERF) {
#pragma unroll
            for (int i = 0; i < 16; ++i) x[i] = x[2 * i] * gelu_erf_fast(x[2 * i + 1]);
          } else if (p.act == SEEDX_ACT_SILU) {
#pragma unroll
            for (int i = 0; i < 16; ++i) x[i] = x[2 * i] * silu(x[2 * i + 1]);
          } else {
#pragma unroll
            for (int i = 0; i < 16; ++i) x[i] = x[2 * i] * x[2 * i + 1];
          }
          nvals = 16;
          ocol0 = col0 >> 1;
        } else if (p.act == SEEDX_ACT_GELU_ERF) {
#pragma unroll
          for (int i = 0; i < 32; ++i) x[i] = gelu_erf_fast(x[i]);
        } else if (p.act == SEEDX_ACT_SILU) {
#pragma unroll
          for (int i = 0; i < 32; ++i) x[i] = silu(x[i]);
        }
        if (p.tma_epi) {
          // ---- shared-memory staged epilogue: residual tile arrives by TMA, output tile leaves by TMA (whole 32-row x RB-byte
          // boxes; rows / columns outside the matrix are clipped by the tensor map).  Lane = row; the 16-byte chunk index is
          // XOR-swizzled exactly like the tensor map's swizzle mode, which also makes the 128-bit accesses bank-conflict free.
          const int k = kchunk++;
          const uint32_t sw = RB == 128 ? (uint32_t)(lane & 7) : (RB == 64 ? (uint32_t)((lane >> 1) & 3) : (uint32_t)((lane >> 2) & 1));
          if (tma_res) {
            const int rb = k % nres;
            mbar_wait(res_bar(ew, rb), (epi_res_phase >> rb) & 1u);
            epi_res_phase ^= 1u << rb;
            const uint32_t rrow_addr = stg_res + (uint32_t)rb * tile_bytes + (uint32_t)(lane * RB);
            if (p.out_f32) {
#pragma unroll
              for (int j = 0; j < 8; ++j) {
                if (4 * j < nvals) {
                  const uint4 qv = lds128(rrow_addr + (((uint32_t)j ^ sw) << 4));
                  x[4 * j] += __uint_as_float(qv.x), x[4 * j + 1] += __uint_as_float(qv.y);
                  x[4 * j + 2] += __uint_as_float(qv.z), x[4 * j + 3] += __uint_as_float(qv.w);
                }
              }
            } else {
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                if (8 * j < nvals) {
                  const uint4 qv = lds128(rrow_addr + (((uint32_t)j ^ sw) << 4));
                  const __half2* h = (const __half2*)&qv;
#pragma unroll
                  for (int e = 0; e < 4; ++e) {
                    const float2 f = __half22float2(h[e]);
                    x[8 * j + 2 * e] += f.x, x[8 * j + 2 * e + 1] += f.y;
                  }
                }
              }
            }
            __syncwarp();                                             // every lane has consumed buffer rb
            if (lane == 0 && k + nres < n_chunks) issue_res(k + nres);
          }
          const int ob = k % nbuf;
          if (lane == 0) {                                            // the store that last read this output buffer has drained it
            if (nbuf == 4) bulk_wait_read<3>();
            else if (nbuf == 2) bulk_wait_read<1>();
            else bulk_wait_read<0>();
          }
          __syncwarp();
          const uint32_t orow_addr = stg_out + (uint32_t)ob * tile_bytes + (uint32_t)(lane * RB);
          if (p.out_f32) {
#pragma unroll
            for (int j = 0; j < 8; ++j)
              if (4 * j < nvals)
                sts128(orow_addr + (((uint32_t)j ^ sw) << 4), make_uint4(__float_as_uint(x[4 * j]), __float_as_uint(x[4 * j + 1]),
                                                                         __float_as_uint(x[4 * j + 2]), __float_as_uint(x[4 * j + 3])));
          } else {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              if (8 * j < nvals) {
                uint4 qv;
                __half2* h = (__half2*)&qv;
#pragma unroll
                for (int e = 0; e < 4; ++e) h[e] = __floats2half2_rn(x[8 * j + 2 * e], x[8 * j + 2 * e + 1]);
                sts128(orow_addr + (((uint32_t)j ^ sw) << 4), qv);
              }
            }
          }
          fence_proxy_async();                                        // generic-proxy writes -> visible to the TMA engine
          __syncwarp();
          if (lane == 0) {
            tma_store_3d(&tmD, stg_out + (uint32_t)ob * tile_bytes, ocol0, row_base, b);
            bulk_commit();
          }
          if (p.row_part != nullptr && row_ok) {                      // this thread's row over the 32 columns of the chunk
            float s1 = 0.f, s2 = 0.f;
#pragma unroll
            for (int i = 0; i < 32; ++i) s1 += x[i], s2 = fmaf(x[i], x[i], s2);
            p.row_part[(long long)(col0 >> 5) * p.M + row] = make_float2(s1, s2);
          }
          if (p.col_part != nullptr && row_base < p.M) {    // (M % 32 == 0: a slab is either wholly inside the matrix or wholly outside)
            // lane = column: walk the 32 staged rows (the fp16 values the consumer will read) in row order.  RB = 64 here (fp16, not gated).
            const uint32_t tb = stg_out + (uint32_t)ob * tile_bytes + (uint32_t)((lane & 7) * 2);
            float s1 = 0.f, s2 = 0.f;
#pragma unroll
            for (int rr = 0; rr < 32; ++rr) {
              const uint32_t a = tb + (uint32_t)(rr * 64) + ((((uint32_t)lane >> 3) ^ (((uint32_t)rr >> 1) & 3u)) << 4);
              unsigned short hv;
              asm volatile("ld.shared.u16 %0, [%1];\n" : "=h"(hv) : "r"(a));
              const float fv = __half2float(__ushort_as_half(hv));
              s1 += fv, s2 = fmaf(fv, fv, s2);
            }
            if (col0 + lane < col_end) p.col_part[(long long)(row_base >> 5) * p.N + col0 + lane] = make_float2(s1, s2);
          }
          return;
        }
        const int n_out = p.gated ? (col_end >> 1) : col_end;  // output columns of this tile end here
        if (!row_ok) return;
        const bool full = (ocol0 + nvals <= n_out) && p.vec_ok;
        if (p.residual != nullptr) {
          if (p.res_f32) {
            const float* rp = (const float*)p.residual + (long long)b * p.strideR + (long long)rrow * p.ldr + ocol0;
            if (full) {
#pragma unroll
              for (int i = 0; i < 32; i += 4) {
                if (i < nvals) {
                  const float4 qv = *(const float4*)(rp + i);
                  x[i] += qv.x, x[i + 1] += qv.y, x[i + 2] += qv.z, x[i + 3] += qv.w;
                }
              }
            } else {
#pragma unroll
              for (int i = 0; i < 32; ++i)
                if (i < nvals && ocol0 + i < n_out) x[i] += rp[i];
            }
          } else {
            const __half* rp = (const __half*)p.residual + (long long)b * p.strideR + (long long)rrow * p.ldr + ocol0;
            if (full) {
#pragma unroll
              for (int i = 0; i < 32; i += 8) {
                if (i < nvals) {
                  const uint4 qv = *(const uint4*)(rp + i);
                  const __half2* h = (const __half2*)&qv;
#pragma unroll
                  for (int j = 0; j < 4; ++j) {
                    const float2 f = __half22float2(h[j]);
                    x[i + 2 * j] += f.x, x[i + 2 * j + 1] += f.y;
                  }
                }
              }
            } else {
#pragma unroll
              for (int i = 0; i < 32; ++i)
                if (i < nvals && ocol0 + i < n_out) x[i] += __half2float(rp[i]);
            }
          }
        }
        if (p.out_f32) {
          float* dp = (float*)p.D + (long long)b * p.strideD + (long long)row * p.ldd + ocol0;
          if (full) {
#pragma unroll
            for (int i = 0; i < 32; i += 4)
              if (i < nvals) *(float4*)(dp + i) = make_float4(x[i], x[i + 1], x[i + 2], x[i + 3]);
          } else {
#pragma unroll
            for (int i = 0; i < 32; ++i)
              if (i < nvals && ocol0 + i < n_out) dp[i] = x[i];
          }
        } else {
          __half* dp = (__half*)p.D + (long long)b * p.strideD + (long long)row * p.ldd + ocol0;
          if (full) {
#pragma unroll
            for (int i = 0; i < 32; i += 8) {
              if (i < nvals) {
                uint4 qv;
                __half2* h = (__half2*)&qv;
#pragma unroll
                for (int j = 0; j < 4; ++j) h[j] = __floats2half2_rn(x[i + 2 * j], x[i + 2 * j + 1]);
                *(uint4*)(dp + i) = qv;
              }
            }
          } else {
#pragma unroll
            for (int i = 0; i < 32; ++i)
              if (i < nvals && ocol0 + i < n_out) dp[i] = __float2half_rn(x[i]);
          }
        }
      });
      __syncwarp();
      if (p.row_stats_out != nullptr && row_base < p.M) {
        // my partials of this slab are written: take a ticket.  A slab receives 2 * n_blocks deliveries (the even- and the odd-chunk warp of its
        // rows, once per column block); the last one reduces the slab.
        __threadfence();
        __syncwarp();
        unsigned last = 0;
        if (lane == 0) last = (atomicAdd(p.row_tickets + (row_base >> 5), 1u) == (unsigned)(2 * p.n_blocks - 1)) ? 1u : 0u;
        last = __shfl_sync(0xffffffffu, last, 0);
        if (last) {
          __threadfence();
          if (row_ok) {
            const int parts = p.N >> 5;
            float s1 = 0.f, s2 = 0.f;
#pragma unroll 4
            for (int k = 0; k < parts; ++k) {
              const float2 qq = __ldcg(p.row_part + (long long)k * p.M + row);
              s1 += qq.x, s2 += qq.y;
            }
            const float inv = 1.0f / (float)p.N;
            const float mean = s1 * inv;
            p.row_stats_out[row] = make_float2(mean, rsqrtf(fmaxf(s2 * inv - mean * mean, 0.f) + p.row_eps));
          }
          if (lane == 0) p.row_tickets[row_base >> 5] = 0u;
        }
      }
      if (lane == 0 && sk_owner)                       // flags back to 0: one writer and one reader each, nobody else looks at them
        for (int cc = my_cluster + 1; cc <= sk_last; ++cc) p.sk_flags[((size_t)cc * CL + crank) * EPI_WARPS + ew] = 0u;
      first_seg = false;
    }
    if (p.tma_epi && lane == 0) bulk_wait_read<0>();  // shared memory stays alive until the last TMA store has read it
    if (ew == 0 && lane == 0) GEMM_STAMP(6);
  }

  __syncthreads();
  if (CL > 1) cluster_sync_all();  // no CTA leaves while its peer may still write into its shared memory / arrive on its barriers
  if (threadIdx.x == 0) GEMM_STAMP(7);
}

// ------------------------------------------------------------------------------------------------
// host
// ------------------------------------------------------------------------------------------------
void count_launch();

// stream-K fix-up workspace (seedx_gemm_set_workspace): flags first (zeroed by the caller), partial tiles behind them
static int g_gemm_stream_k = 1;       // 0 = off, 1 = auto, 2 = whenever legal (tests)
static int g_sk_min_kblocks = 90;     // auto mode: shortest K (in 64-element blocks) that is split: the 3x3 convs from 640 channels (K >= 5760).  Shorter K
                                      // gains little from balancing, and the stream-K order defeats the L2 reuse of A
static float* g_sk_scratch = nullptr;
static size_t g_sk_scratch_bytes = 0;
static unsigned* g_sk_flags = nullptr;
constexpr size_t SK_FLAG_BYTES = 16384;
// what the most recent launch ran (seedx_gemm_last_config): tile width, cluster size, stream-K, TMA epilogue, vec_ok, pipeline stages
static int g_gemm_last[6] = {0, 0, 0, 0, 0, 0};

template <int BN, int CL, typename TE = __half, bool CONV8 = false>
static int launch_gemm_cl(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& td, const CUtensorMap& tr, const GemmParams& p_in,
                          cudaStream_t st) {
  using Cfg = TileCfg<BN, CL>;
  constexpr bool kFP8 = std::is_same<TE, __nv_fp8_e4m3>::value;
  // stream-K kernels exist for cluster pairs with 32-column-multiple tiles of at least 128 columns (where the schedule is ever chosen)
  constexpr bool kHasSK = (CL == 2) && (BN % 32 == 0) && (BN >= 128) && !kFP8;
  static bool attr_done = false;
  if (!attr_done) {
    SEEDX_CUDA(cudaFuncSetAttribute(gemm_tc_kernel<BN, CL, false, TE, CONV8>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LIMIT));
    if (kHasSK) SEEDX_CUDA(cudaFuncSetAttribute(gemm_tc_kernel<BN, CL, kHasSK, TE, CONV8>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LIMIT));
    attr_done = true;
  }
  GemmParams p = p_in;
  int epi_bytes = EPI_WARPS * p.epi_warp_bytes;
  // FP8 stages the b_scale vector behind the bias and column-sum slots, so it budgets all three
  const int tail_bytes = kFP8 ? 512 + 3 * VEC_BYTES
                              : 512 + (p.bias_n != nullptr || p.ln_stats != nullptr || p.bias_g != nullptr ? VEC_BYTES : 0) + (p.ln_stats != nullptr ? VEC_BYTES : 0);
  p.stages = Cfg::stages_for(epi_bytes, tail_bytes);
  if (p.stages < 3 && p.tma_epi && p.epi_warp_bytes > 32 * p.epi_row_bytes * (p.epi_res_bytes ? 2 : 1)) {
    // the short-K staging (several boxes in flight per warp) would leave a wide tile fewer than three pipeline stages: one box each
    p.epi_out_bytes = 32 * p.epi_row_bytes;
    p.epi_res_bytes = p.epi_res_bytes ? 32 * p.epi_row_bytes : 0;
    p.epi_warp_bytes = p.epi_out_bytes + p.epi_res_bytes;
    epi_bytes = EPI_WARPS * p.epi_warp_bytes;
    p.stages = Cfg::stages_for(epi_bytes, tail_bytes);
  }
  if (p.stages < 2) {
    set_error("%s: tile %dx%d does not fit in shared memory with %d B of epilogue staging", CONV8 ? "seedx_conv_fp8" : (kFP8 ? "seedx_gemm_fp8" : "seedx_gemm_f16"),
              BM * CL, BN, epi_bytes);
    return 5;
  }
  const int smem_bytes = Cfg::smem_for(p.stages, epi_bytes, tail_bytes);
  const int groups = ((p.m_blocks + CL - 1) / CL) * p.n_blocks * p.batch;
  int max_clusters = num_sms() / CL;
  if (CL > 1) {
    // a cluster must fit in one GPC: fewer pairs than num_sms / 2 may be co-resident, and a persistent grid larger than that runs a second wave
    static int occ_smem = -1, occ_clusters = 0;
    if (occ_smem != smem_bytes) {
      cudaLaunchConfig_t q{};
      q.gridDim = dim3(max_clusters * CL), q.blockDim = dim3(GEMM_THREADS), q.dynamicSmemBytes = smem_bytes;
      cudaLaunchAttribute qa[1];
      qa[0].id = cudaLaunchAttributeClusterDimension;
      qa[0].val.clusterDim.x = CL, qa[0].val.clusterDim.y = 1, qa[0].val.clusterDim.z = 1;
      q.attrs = qa, q.numAttrs = 1;
      SEEDX_CUDA(cudaOccupancyMaxActiveClusters(&occ_clusters, gemm_tc_kernel<BN, CL, false, TE, CONV8>, &q));
      occ_smem = smem_bytes;
    }
    if (occ_clusters > 0 && occ_clusters < max_clusters) max_clusters = occ_clusters;
  }
  const int grid = (groups < max_clusters ? groups : max_clusters) * CL;
  // Stream-K when the last wave of whole tiles would leave SMs idle: every cluster gets total/clusters k-iterations instead of whole tiles.
  // Needs the fix-up workspace, at least 4 iterations per cluster (no empty cluster, a partial is worth its round trip) and a tile that
  // fits a scratch slot.
  p.stream_k = 0;
  {
    const int clusters = grid / CL;
    const long long total = (long long)groups * p.k_blocks;
    const int rem = groups % clusters;
    const bool idle_tail = rem != 0 && (double)(clusters - rem) / clusters / ((groups + clusters - 1) / clusters) > 0.04;   // > 4 % of the launch idle
    const size_t need = (size_t)clusters * CL * BM * ((BN + 31) & ~31) * sizeof(float);
    // the fix-up round trip of a partial tile (2 x 128 x BN fp32 through L2) is only worth it for long K (g_sk_min_kblocks)
    const bool long_k = p.k_blocks >= g_sk_min_kblocks;
    if (kHasSK && g_gemm_stream_k != 0 && g_sk_scratch != nullptr && need <= g_sk_scratch_bytes && total >= 4LL * clusters && groups > clusters &&
        ((idle_tail && long_k) || g_gemm_stream_k == 2)) {
      p.stream_k = 1;
      p.sk_scratch = g_sk_scratch, p.sk_flags = g_sk_flags;
    }
  }
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(GEMM_THREADS);
  cfg.dynamicSmemBytes = smem_bytes;
  cfg.stream = st;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = CL, attr[0].val.clusterDim.y = 1, attr[0].val.clusterDim.z = 1;
  attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[1].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 2 : 1;
  g_gemm_last[0] = BN, g_gemm_last[1] = CL, g_gemm_last[2] = p.stream_k, g_gemm_last[3] = p.tma_epi, g_gemm_last[4] = p.vec_ok, g_gemm_last[5] = p.stages;
  const cudaError_t e = (kHasSK && p.stream_k) ? cudaLaunchKernelEx(&cfg, gemm_tc_kernel<BN, CL, kHasSK, TE, CONV8>, ta, tb, td, tr, p)
                                               : cudaLaunchKernelEx(&cfg, gemm_tc_kernel<BN, CL, false, TE, CONV8>, ta, tb, td, tr, p);
  count_launch();
  return check_cuda(e != cudaSuccess ? e : cudaGetLastError(), "gemm_tc_kernel launch");
}

template <int BN>
static int launch_gemm(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& td, const CUtensorMap& tr, const GemmParams& p, int cl,
                       cudaStream_t st) {
  if (cl == 2) return launch_gemm_cl<BN, 2>(ta, tb, td, tr, p, st);
  return launch_gemm_cl<BN, 1>(ta, tb, td, tr, p, st);
}

static unsigned long long* g_gemm_dbg = nullptr;
static int g_gemm_cluster = 1;  // 0 = never cluster, 1 = auto (single-CTA tiles), 2 = always when legal
static int g_gemm_tma_epi = 1;  // 0 = row-per-thread direct stores, 1 = TMA-store epilogue when eligible

static const int kTileN[] = {64, 96, 128, 144, 160, 192, 208, 224, 240, 256};

static bool valid_tile_n(int bn) {
  for (int t : kTileN)
    if (t == bn) return true;
  return false;
}

// Pick the N tile that minimises a simple cycle model of the persistent kernel:
//   waves = ceil(tiles / SMs); per tile MMA cycles + epilogue cycles (the consumer warpgroups run both in turn).
// MMA: a 128 x BN x 16 step is BN cycles at the dense fp16 rate of an H100 SM (2048 FMA/clk), divided by the rate a tile width reaches
// relative to the 256-wide tile.  Measured on an H100 SXM at 700 W, 8192^3 single-CTA launches (256 wide: 616 TFLOP/s): narrower tiles
// re-read A more often per FLOP and leave more stages' worth of latency exposed, widths that are not one wgmma instruction issue several.
// The FP8 GEMM reuses this table with k_blocks counted in its 128-element stages (one stage = the MMA time of a 64-element fp16 stage at twice
// the rate).  The rates were measured for fp16, not for FP8.
struct TileRate {
  int bn;
  double rate;
};
static const TileRate kAutoTiles[] = {{128, 0.82}, {160, 0.78}, {192, 0.94}, {224, 0.73}, {256, 1.0}};

// max_bn: the widest tile the caller has kernels for (the FP8 conv: 160, see kConv8Tiles)
static int choose_tile_n(int m_tiles, int N, int k_blocks, bool heavy_epilogue, bool only32, int max_bn = 256) {
  const int sms = num_sms();
  double best = 1e30;
  int best_bn = 256;
  for (const TileRate& tr : kAutoTiles) {
    const int bn = tr.bn;
    if (only32 && bn % 32 != 0) continue;  // the TMA epilogue stores whole 32-column chunks
    if (bn > max_bn) continue;
    const int n_blocks = (N + bn - 1) / bn;
    const long long tiles = (long long)m_tiles * n_blocks;
    // stream-K (cluster pairs forced, workspace present): a launch of more than one wave costs its fractional number of waves plus the partial-tile round trip
    const bool sk = (bn % 32 == 0 && bn >= 128) && g_gemm_cluster == 2 && g_gemm_stream_k != 0 && g_sk_scratch != nullptr && tiles > sms &&
                    (long long)tiles * k_blocks >= 4LL * sms &&
                    (k_blocks >= g_sk_min_kblocks || g_gemm_stream_k == 2);
    const double waves = sk ? (double)tiles / sms + 0.12 : (double)((tiles + sms - 1) / sms);
    const double mma_k16 = bn / tr.rate;
    const double mma = k_blocks * 4.0 * mma_k16;
    const double epi = bn * (heavy_epilogue ? 14.0 : 8.0) + 300.0;
    const double cost = waves * (mma + epi + 150.0);
    if (cost < best - 1e-9 || (fabs(cost - best) <= 1e-9 && bn > best_bn)) best = cost, best_bn = bn;
  }
  return best_bn;
}

}  // namespace seedx

using namespace seedx;

extern "C" void seedx_gemm_set_debug(void* device_buffer) { seedx::g_gemm_dbg = (unsigned long long*)device_buffer; }
extern "C" void seedx_gemm_set_cluster(int mode) { seedx::g_gemm_cluster = mode; }
extern "C" void seedx_gemm_set_tma_epilogue(int on) { seedx::g_gemm_tma_epi = on; }
extern "C" void seedx_gemm_last_config(int32_t out[6]) {
  for (int i = 0; i < 6; ++i) out[i] = seedx::g_gemm_last[i];
}
extern "C" void seedx_gemm_set_stream_k(int mode) {
  seedx::g_gemm_stream_k = mode;
  if (const char* e = getenv("SEEDX_SK_MIN_KBLOCKS")) seedx::g_sk_min_kblocks = atoi(e);
}
extern "C" int seedx_gemm_set_workspace(void* ptr, int64_t bytes) {
  if (ptr == nullptr) {
    seedx::g_sk_scratch = nullptr, seedx::g_sk_flags = nullptr, seedx::g_sk_scratch_bytes = 0;
    return 0;
  }
  SEEDX_REQUIRE(((uintptr_t)ptr % 256 == 0) && bytes > (int64_t)seedx::SK_FLAG_BYTES, "seedx_gemm_set_workspace: need a 256-byte aligned buffer larger than %d bytes",
                (int)seedx::SK_FLAG_BYTES);
  seedx::g_sk_flags = (unsigned*)ptr;
  seedx::g_sk_scratch = (float*)((char*)ptr + seedx::SK_FLAG_BYTES);
  seedx::g_sk_scratch_bytes = (size_t)bytes - seedx::SK_FLAG_BYTES;
  return 0;
}

// FP8 conv tile widths: the promoted accumulation holds a second BN/2-register accumulator per consumer thread, and wider tiles spill under
// the 232-register consumer budget
static const int kConv8Tiles[] = {64, 128, 160};

// seedx_gemm_f16, seedx_gemm_fp8 and seedx_conv_fp8: one host path.  FP8 differs in the element size (1 byte), the K per stage (128), the
// tensor-map type and the scales; it runs single-CTA, data-parallel, batch 1, at the widths the auto chooser returns (and 64).  conv8: the FP8
// implicit-GEMM conv (per-image a_scale, promoted accumulation), at the widths of kConv8Tiles.
static int gemm_entry(const seedx_gemm_args* a, bool fp8, bool conv8, const float* a_scale, const float* b_scale, void* stream) {
  const char* fn = conv8 ? "seedx_conv_fp8" : (fp8 ? "seedx_gemm_fp8" : "seedx_gemm_f16");
  SEEDX_REQUIRE(a != nullptr, "%s: null args", fn);
  SEEDX_REQUIRE(a->A && a->B && a->D, "%s: null operand pointer", fn);
  SEEDX_REQUIRE(a->M > 0 && a->N > 0 && a->K > 0 && a->batch > 0, "%s: empty problem M=%lld N=%lld K=%lld", fn,
                (long long)a->M, (long long)a->N, (long long)a->K);
  const int es = fp8 ? 1 : 2;                 // operand element bytes
  const int kb_elems = fp8 ? BK_FP8 : BK;     // K elements per pipeline stage
  const int row_align = 16 / es;              // elements per 16 bytes: TMA rows start and end on 16-byte boundaries
  if (conv8) {
    SEEDX_REQUIRE(a->conv_taps_h > 0 && a->conv_taps_w > 0, "seedx_conv_fp8: not a conv call (conv_taps_h / conv_taps_w are 0)");
    SEEDX_REQUIRE(a->batch == 1, "seedx_conv_fp8: batch=%lld, only batch 1 is supported", (long long)a->batch);
    SEEDX_REQUIRE(a_scale != nullptr && b_scale != nullptr, "seedx_conv_fp8: a_scale and b_scale are required");
    bool tile_ok = a->tile_n == 0;
    for (int t : kConv8Tiles) tile_ok = tile_ok || a->tile_n == t;
    SEEDX_REQUIRE(tile_ok, "seedx_conv_fp8: tile_n must be 0 (auto) or one of 64/128/160");
  } else if (fp8) {
    SEEDX_REQUIRE(a->conv_taps_h == 0 && a->conv_taps_w == 0, "seedx_gemm_fp8: conv mode is not supported");
    SEEDX_REQUIRE(a->batch == 1, "seedx_gemm_fp8: batch=%lld, only batch 1 is supported", (long long)a->batch);
    SEEDX_REQUIRE(a_scale != nullptr && b_scale != nullptr, "seedx_gemm_fp8: a_scale and b_scale are required");
    SEEDX_REQUIRE(a->tile_n == 0 || a->tile_n == 64 || a->tile_n == 128 || a->tile_n == 160 || a->tile_n == 192 || a->tile_n == 224 || a->tile_n == 256,
                  "seedx_gemm_fp8: tile_n must be 0 (auto) or one of 64/128/160/192/224/256");
  }
  SEEDX_REQUIRE(a->K % row_align == 0, "%s: K=%lld must be a multiple of %d (16-byte TMA rows)", fn, (long long)a->K, row_align);
  SEEDX_REQUIRE(((uintptr_t)a->A % 16 == 0) && ((uintptr_t)a->B % 16 == 0), "%s: operands must be 16B aligned", fn);
  SEEDX_REQUIRE(a->out_dtype == SEEDX_F16 || a->out_dtype == SEEDX_F32, "%s: bad out_dtype", fn);
  const bool conv = a->conv_taps_h > 0;
  GemmParams p{};
  int bn = a->tile_n;
  SEEDX_REQUIRE(bn == 0 || valid_tile_n(bn), "%s: tile_n must be 0 (auto) or one of 64/96/128/144/160/192/208/224/240/256", fn);
  if (a->gated) SEEDX_REQUIRE(a->N % 2 == 0, "%s: gated epilogue needs even N", fn);

  // ---- TMA epilogue eligibility (output / residual tiles go through shared memory and cp.async.bulk.tensor stores)
  const int out_es = a->out_dtype == SEEDX_F32 ? 4 : 2;
  const long long n_out_ll = a->gated ? a->N / 2 : a->N;
  // The output rows must also END on a 16-byte boundary: on an H100 a TMA store box that straddles the end of a row writes the whole 16-byte
  // granule, i.e. up to 14 bytes past n_out into the ldd gap of an output view (measured: 4 fp16 columns per row for n_out = 196).
  bool tma_epi = g_gemm_tma_epi && ((uintptr_t)a->D % 16 == 0) && ((a->ldd * out_es) % 16 == 0) && (a->batch == 1 || (a->strideD * out_es) % 16 == 0) &&
                 (a->N % 2 == 0) && ((n_out_ll * out_es) % 16 == 0);
  if (a->residual) {
    tma_epi = tma_epi && !a->gated && a->residual_dtype == a->out_dtype && ((uintptr_t)a->residual % 16 == 0) && ((a->ldr * out_es) % 16 == 0) &&
              (a->res_row_mod % 32 == 0) && (a->batch == 1 || a->strideR == 0 || (a->strideR * out_es) % 16 == 0);
  }
  if (bn != 0 && bn % 32 != 0) tma_epi = false;
  CUtensorMap ta, tb, td, tr;
  int cl = 1;
  if (!conv) {
    SEEDX_REQUIRE(a->lda % row_align == 0 && a->lda >= a->K, "%s: lda must be >= K and a multiple of %d", fn, row_align);
    uint64_t dims[3] = {(uint64_t)a->K, (uint64_t)a->M, (uint64_t)a->batch};
    uint64_t bstride = a->batch > 1 ? (uint64_t)a->strideA * es : (uint64_t)a->lda * es * (uint64_t)a->M;
    SEEDX_REQUIRE(bstride % 16 == 0, "%s: strideA must be a multiple of 8 elements", fn);
    uint64_t strides[2] = {(uint64_t)a->lda * es, bstride};
    uint32_t box[3] = {(uint32_t)kb_elems, BM, 1};
    if (int e = encode_tmap(&ta, fp8 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, a->A, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B))
      return e;
    p.k_blocks = (int)((a->K + kb_elems - 1) / kb_elems);   // the K tail of the last stage is TMA zero fill
    p.m_blocks = (int)((a->M + BM - 1) / BM);
    if (bn == 0) bn = choose_tile_n(p.m_blocks * (int)a->batch, (int)a->N, p.k_blocks, a->act != SEEDX_ACT_NONE, tma_epi);
  } else {
    const int64_t C = a->conv_c, W = a->conv_w, H = a->conv_h, NI = a->conv_n;
    if (conv8) SEEDX_REQUIRE(C % 16 == 0 && C > 0, "seedx_conv_fp8: channels must be a multiple of 16 (16-byte e4m3 pixels)");
    SEEDX_REQUIRE(C % 8 == 0 && C > 0, "seedx_gemm_f16(conv): channels must be a multiple of 8");
    SEEDX_REQUIRE(a->conv_taps_h == a->conv_taps_w && (a->conv_taps_h == 1 || a->conv_taps_h == 3),
                  "seedx_gemm_f16(conv): only 1x1 and 3x3 kernels");
    int tw, th, tn = 1;
    if (W <= 128) {
      SEEDX_REQUIRE(128 % W == 0, "seedx_gemm_f16(conv): width %lld must divide 128", (long long)W);
      tw = (int)W, th = (int)(128 / W);
      if (th > H) {  // small images: one 128-row tile spans several whole images
        SEEDX_REQUIRE(th % H == 0, "seedx_gemm_f16(conv): %lldx%lld image does not tile 128 rows", (long long)H, (long long)W);
        tn = (int)(th / H), th = (int)H;
      }
      SEEDX_REQUIRE(H % th == 0, "seedx_gemm_f16(conv): height %lld not a multiple of tile height %d", (long long)H, th);
    } else {
      SEEDX_REQUIRE(W % 128 == 0, "seedx_gemm_f16(conv): width %lld must be a multiple of 128", (long long)W);
      tw = 128, th = 1;
    }
    SEEDX_REQUIRE(a->M == NI * H * W, "seedx_gemm_f16(conv): M != n*h*w");
    const int cchunks = (int)((C + kb_elems - 1) / kb_elems);   // channel chunks of one stage: 64 fp16 or 128 e4m3 (128 bytes per pixel)
    SEEDX_REQUIRE(a->K == (int64_t)a->conv_taps_h * a->conv_taps_w * cchunks * kb_elems,
                  "%s: K=%lld must equal taps*roundup(C,%d)=%lld", conv8 ? fn : "seedx_gemm_f16(conv)", (long long)a->K, kb_elems,
                  (long long)a->conv_taps_h * a->conv_taps_w * cchunks * kb_elems);
    uint64_t dims[4] = {(uint64_t)C, (uint64_t)W, (uint64_t)H, (uint64_t)NI};
    uint64_t strides[3] = {(uint64_t)C * es, (uint64_t)W * C * es, (uint64_t)H * W * C * es};
    if (bn == 0)
      bn = choose_tile_n((int)((a->M + BM - 1) / BM), (int)a->N, a->conv_taps_h * a->conv_taps_w * cchunks, a->act != SEEDX_ACT_NONE, tma_epi,
                         conv8 ? 160 : 256);
    uint32_t box[4] = {(uint32_t)kb_elems, (uint32_t)tw, (uint32_t)th, (uint32_t)tn};
    if (int e = encode_tmap(&ta, conv8 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, a->A, dims, strides, box,
                            CU_TENSOR_MAP_SWIZZLE_128B))
      return e;
    p.conv = 1;
    p.taps_w = a->conv_taps_w;
    p.c_chunks = cchunks;
    p.conv_w = (int)W, p.conv_h = (int)H;
    p.tile_w = tw, p.tile_h = th;
    p.tiles_w = (int)(W / tw);
    p.tiles_per_img = (int)((H / th) * (W / tw));
    p.imgs_per_tile = tn;
    p.pad = a->conv_taps_h / 2;
    p.k_blocks = a->conv_taps_h * a->conv_taps_w * cchunks;
    p.m_blocks = (int)((a->M + BM - 1) / BM);
  }
  {
    SEEDX_REQUIRE(a->ldb % row_align == 0 && a->ldb >= a->K, "%s: ldb must be >= K and a multiple of %d", fn, row_align);
    const bool bb = a->batch > 1 && a->strideB != 0;
    uint64_t dims[3] = {(uint64_t)a->K, (uint64_t)a->N, (uint64_t)(bb ? a->batch : 1)};
    uint64_t bstride = bb ? (uint64_t)a->strideB * es : (uint64_t)a->ldb * es * (uint64_t)a->N;
    SEEDX_REQUIRE(bstride % 16 == 0, "%s: strideB must be a multiple of 8 elements", fn);
    uint64_t strides[2] = {(uint64_t)a->ldb * es, bstride};
    // cluster pairs (B tile multicast in two halves, 16-row aligned) only when forced: on an H100 SXM (700 W) they measured about half the
    // single-CTA rate on every shape tried (8192 x {10240, 1280, 8192} x {1280, 5120, 8192}), so auto mode keeps single-CTA tiles
    if (g_gemm_cluster == 2 && p.m_blocks >= 2 && bn % 32 == 0 && !fp8) cl = 2;
    // a single CTA with residual staging (96 KB) keeps only 2 stages of a 256-wide tile: use a narrower tile there
    if (cl == 1 && tma_epi && a->residual && bn > 160 && a->tile_n == 0) bn = 160;
    uint32_t box[3] = {(uint32_t)kb_elems, (uint32_t)(bn / cl), 1};
    if (int e = encode_tmap(&tb, fp8 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, a->B, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B))
      return e;
    p.b_batched = bb ? 1 : 0;
  }
  p.D = a->D;
  p.dbg = g_gemm_dbg;
  p.a_scale = a_scale, p.b_scale = b_scale;
  if (a->ln_stats || a->ln_colsum) {
    SEEDX_REQUIRE(a->ln_stats && a->ln_colsum, "%s: ln_stats and ln_colsum go together", fn);
    SEEDX_REQUIRE(a->batch == 1 && !conv && ((uintptr_t)a->ln_colsum % 16 == 0) && ((uintptr_t)a->ln_stats % 8 == 0) && a->N % 4 == 0,
                  "%s: folded LayerNorm needs a plain un-batched GEMM, N %% 4 == 0 and aligned statistics", fn);
    SEEDX_REQUIRE(a->alpha == 1.0f && a->bias_m == nullptr, "%s: folded LayerNorm takes alpha = 1 and no per-row bias", fn);
  }
  p.ln_stats = (const float2*)a->ln_stats, p.ln_colsum = a->ln_colsum;
  p.ln_parts = a->ln_parts, p.ln_eps = a->ln_eps, p.ln_inv_cols = a->ln_parts > 0 ? 1.0f / (32.0f * (float)a->ln_parts) : 0.f;
  SEEDX_REQUIRE(a->ln_parts >= 0 && (a->ln_parts == 0 || (a->ln_stats && 32LL * a->ln_parts == a->K)),
                "%s: ln_parts=%d must cover K=%lld columns in 32-column chunks", fn, a->ln_parts, (long long)a->K);
  if (a->row_part || a->col_part) {
    SEEDX_REQUIRE(tma_epi && !a->gated && a->out_dtype == SEEDX_F16 && a->batch == 1 && a->N % 32 == 0 && a->M % 32 == 0,
                  "%s: output statistics need the TMA epilogue (16-byte aligned fp16 output), no gating, batch 1, M and N multiples of 32", fn);
    SEEDX_REQUIRE(((uintptr_t)a->row_part % 8 == 0) && ((uintptr_t)a->col_part % 8 == 0), "%s: statistics buffers must be 8-byte aligned", fn);
  }
  p.row_part = (float2*)a->row_part, p.col_part = (float2*)a->col_part;
  if (a->row_stats_out || a->row_tickets) {
    SEEDX_REQUIRE(a->row_part && a->row_stats_out && a->row_tickets && ((uintptr_t)a->row_stats_out % 8 == 0),
                  "%s: row_stats_out needs row_part and row_tickets (M/32 zeroed counters)", fn);
  }
  p.row_stats_out = (float2*)a->row_stats_out, p.row_tickets = a->row_tickets, p.row_eps = a->row_eps;
  p.b_static = a->b_dynamic ? 0 : 1;
  p.bias_n = a->bias_n, p.bias_m = a->bias_m, p.bias_g = a->bias_g;
  p.bias_g_rows = a->bias_g ? (int)a->bias_g_rows : 1;
  SEEDX_REQUIRE(p.bias_g_rows > 0, "%s: bias_g_rows must be > 0", fn);
  p.residual = a->residual;
  p.M = (int)a->M, p.N = (int)a->N, p.K = (int)a->K, p.batch = (int)a->batch;
  p.n_blocks = (int)((a->N + bn - 1) / bn);
  p.ldd = a->ldd, p.strideD = a->strideD, p.ldr = a->ldr, p.strideR = a->strideR;
  p.res_row_mod = (int)a->res_row_mod;
  p.alpha = a->alpha;
  p.act = a->act, p.gated = a->gated;
  p.out_f32 = a->out_dtype == SEEDX_F32;
  p.res_f32 = a->residual_dtype == SEEDX_F32;
  if (a->residual) SEEDX_REQUIRE(a->residual_dtype == SEEDX_F16 || a->residual_dtype == SEEDX_F32, "%s: bad residual_dtype", fn);
  // vector epilogue needs 16-byte aligned rows on D (and residual)
  const int oe = p.out_f32 ? 4 : 8;
  bool vec = ((uintptr_t)a->D % 16 == 0) && (a->ldd % oe == 0) && (a->strideD % oe == 0);
  if (a->residual) {
    const int re = p.res_f32 ? 4 : 8;
    vec = vec && ((uintptr_t)a->residual % 16 == 0) && (a->ldr % re == 0) && (a->strideR % re == 0);
  }
  p.vec_ok = vec ? 1 : 0;
  p.bias_vec = (a->bias_n && (uintptr_t)a->bias_n % 16 == 0) ? 1 : 0;
  p.tma_epi = tma_epi ? 1 : 0;
  {
    // Staging policy.  Short-K tiles are epilogue-bound: double-buffer the output box and keep up to four residual boxes in flight.
    // Long-K tiles hide the epilogue behind the main loop anyway and want the shared memory for pipeline stages instead: one box each.
    const int box_bytes = 32 * (a->gated ? 16 : 32) * out_es;
    const bool short_k = p.k_blocks < 32;
    const int out_short = a->residual ? EPI_OUT_BYTES : 2 * EPI_OUT_BYTES;   // no residual staging: four output boxes in flight
    p.epi_out_bytes = tma_epi ? (short_k ? (box_bytes > out_short / 2 ? box_bytes : out_short) : box_bytes) : 0;
    p.epi_res_bytes = (tma_epi && a->residual) ? (short_k ? EPI_RES_BYTES : box_bytes) : 0;
    p.epi_warp_bytes = p.epi_out_bytes + p.epi_res_bytes;
  }
  td = ta, tr = ta;  // placeholders when the TMA epilogue is off (never dereferenced)
  if (tma_epi) {
    const int cols = a->gated ? 16 : 32;                    // output columns per 32-column accumulator chunk
    const int rb = cols * out_es;                           // staged row bytes: 32, 64 or 128
    const CUtensorMapSwizzle sw = rb == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : (rb == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
    const CUtensorMapDataType dt = out_es == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
    p.epi_row_bytes = rb;
    uint32_t box[3] = {(uint32_t)cols, 32, 1};
    {
      uint64_t dims[3] = {(uint64_t)n_out_ll, (uint64_t)a->M, (uint64_t)a->batch};
      uint64_t strides[2] = {(uint64_t)a->ldd * out_es, (uint64_t)(a->batch > 1 ? a->strideD : a->ldd * a->M) * out_es};
      if (int e = encode_tmap(&td, dt, 3, a->D, dims, strides, box, sw)) return e;
    }
    if (a->residual) {
      const bool rbat = a->batch > 1 && a->strideR != 0;
      const uint64_t rrows = (uint64_t)(a->res_row_mod ? a->res_row_mod : a->M);
      uint64_t dims[3] = {(uint64_t)n_out_ll, rrows, (uint64_t)(rbat ? a->batch : 1)};
      uint64_t strides[2] = {(uint64_t)a->ldr * out_es, (uint64_t)(rbat ? a->strideR : a->ldr * (long long)rrows) * out_es};
      if (int e = encode_tmap(&tr, dt, 3, a->residual, dims, strides, box, sw)) return e;
      p.r_batched = rbat ? 1 : 0;
    }
  }
  cudaStream_t st = (cudaStream_t)stream;
  if (conv8) {
    switch (bn) {
      case 64: return launch_gemm_cl<64, 1, __nv_fp8_e4m3, true>(ta, tb, td, tr, p, st);
      case 128: return launch_gemm_cl<128, 1, __nv_fp8_e4m3, true>(ta, tb, td, tr, p, st);
      default: return launch_gemm_cl<160, 1, __nv_fp8_e4m3, true>(ta, tb, td, tr, p, st);
    }
  }
  if (fp8) {
    switch (bn) {
      case 64: return launch_gemm_cl<64, 1, __nv_fp8_e4m3>(ta, tb, td, tr, p, st);
      case 128: return launch_gemm_cl<128, 1, __nv_fp8_e4m3>(ta, tb, td, tr, p, st);
      case 160: return launch_gemm_cl<160, 1, __nv_fp8_e4m3>(ta, tb, td, tr, p, st);
      case 192: return launch_gemm_cl<192, 1, __nv_fp8_e4m3>(ta, tb, td, tr, p, st);
      case 224: return launch_gemm_cl<224, 1, __nv_fp8_e4m3>(ta, tb, td, tr, p, st);
      default: return launch_gemm_cl<256, 1, __nv_fp8_e4m3>(ta, tb, td, tr, p, st);
    }
  }
  switch (bn) {
    case 64: return launch_gemm<64>(ta, tb, td, tr, p, cl, st);
    case 96: return launch_gemm<96>(ta, tb, td, tr, p, cl, st);
    case 128: return launch_gemm<128>(ta, tb, td, tr, p, cl, st);
    case 144: return launch_gemm<144>(ta, tb, td, tr, p, cl, st);
    case 160: return launch_gemm<160>(ta, tb, td, tr, p, cl, st);
    case 192: return launch_gemm<192>(ta, tb, td, tr, p, cl, st);
    case 208: return launch_gemm<208>(ta, tb, td, tr, p, cl, st);
    case 224: return launch_gemm<224>(ta, tb, td, tr, p, cl, st);
    case 240: return launch_gemm<240>(ta, tb, td, tr, p, cl, st);
    default: return launch_gemm<256>(ta, tb, td, tr, p, cl, st);
  }
}

extern "C" int seedx_gemm_f16(const seedx_gemm_args* a, void* stream) { return gemm_entry(a, false, false, nullptr, nullptr, stream); }

extern "C" int seedx_gemm_fp8(const seedx_gemm_args* a, const float* a_scale, const float* b_scale, void* stream) {
  return gemm_entry(a, true, false, a_scale, b_scale, stream);
}

extern "C" int seedx_conv_fp8(const seedx_gemm_args* a, const float* a_scale, const float* b_scale, void* stream) {
  return gemm_entry(a, true, true, a_scale, b_scale, stream);
}
