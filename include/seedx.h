/*
 * seedx.h — C ABI of libseedx.so, the H100 (sm_90a) kernel library behind the SEED-X inference hot path.
 *
 * The reference (AILab-CVC/SEED-X) has no FFI/plugin layer: every FLOP is reached through
 * torch.nn.functional / xformers / diffusers library calls made from its nn.Module.forward methods.
 * Each entry point below therefore names the reference call site(s) (file:line under /root/reference)
 * whose arithmetic it replaces.  The Python host (seed-x_b200/*.py) mirrors the reference modules and
 * calls these functions through ctypes with raw device pointers; see INTEGRATION.md for the binding.
 *
 * Conventions
 *  - the caller owns every buffer; pointers are raw CUDA device pointers unless noted otherwise
 *  - `stream` is a cudaStream_t passed as void* (0 = legacy default stream)
 *  - every function returns 0 on success, non-zero on failure; seedx_last_error() describes the failure
 *  - nothing here allocates device memory, spawns threads or synchronises the device
 *  - fp16 = IEEE binary16 (the reference runs `torch.float16`, src/inference/eval_*.py `dtype`)
 */
#ifndef SEEDX_H_
#define SEEDX_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SEEDX_ABI_VERSION 2

/* dtype tags */
enum { SEEDX_F16 = 1, SEEDX_F32 = 2 };
/* activations */
enum { SEEDX_ACT_NONE = 0, SEEDX_ACT_GELU_ERF = 1, SEEDX_ACT_SILU = 2 };

const char* seedx_last_error(void);
int seedx_abi_version(void);
/* number of kernels launched by this process through the library since load (bench.py's gpu_launches) */
int64_t seedx_launch_count(void);
/* Programmatic dependent launch for every kernel of the library (default on; env SEEDX_PDL=0 turns it off): each kernel is launched
 * with the programmatic-stream-serialization attribute and issues griddepcontrol.wait before its first dependent memory access, so
 * its launch and prologue overlap the tail of the kernel before it.  No reference counterpart (the reference runs eager PyTorch). */
int seedx_set_pdl(int on);

/* ------------------------------------------------------------------------------------------------
 * Tensor-core GEMM / implicit-GEMM convolution (wgmma, register accumulators, TMA operand staging)
 *
 *   D[b][m][n] = epilogue( alpha * sum_k A[b][m][k] * B[b][n][k] )         A, B fp16, fp32 accumulate
 *
 * replaces F.linear / nn.Linear / nn.Conv2d / torch.bmm at:
 *   src/models/tokenizer/qwen_visual.py:186,228,253-255,136-146,393,415      (ViT linears, patch-embed conv, proj)
 *   src/models/mllm/modeling_llama_xformer.py:166-167,204-206,239,707        (LLaMA q/k/v/o, SwiGLU MLP, lm_head; prefill)
 *   src/models/detokenizer/resampler.py:9-16,46-75,89-116,266-286            (perceiver resampler linears)
 *   diffusers==0.25.0 UNet2DConditionModel / AutoencoderKL convs + linears, called from
 *   src/models/detokenizer/pipeline_stable_diffusion_xl_t2i_edit.py:915-922,973 and adapter_modules.py:156-167
 *
 * epilogue order: x = alpha*acc; x += bias_n[n]; x += bias_m[m]; x += bias_g[(m / bias_g_rows)*N + n];
 *                 if gated:  y[n/2] = x[2j] * act(x[2j+1])   (N_out = N/2)   else  y = act(x);
 *                 y += residual[(res_row_mod ? m % res_row_mod : m)][n];  store as out_dtype.
 * conv mode (conv_taps_h > 0): A is an NHWC image [conv_n, conv_h, conv_w, conv_c]; M = conv_n*conv_h*conv_w;
 *   stride-1 "same" convolution; B is [N, taps*roundup(conv_c,64)] with k = (kh*KW + kw)*Cpad + c.
 * ---------------------------------------------------------------------------------------------- */
typedef struct seedx_gemm_args {
  const void* A;       /* fp16 [batch][M][K] (row stride lda) — or NHWC image in conv mode            */
  const void* B;       /* fp16 [batch or 1][N][K] (row stride ldb), nn.Linear weight layout            */
  void* D;             /* fp16/fp32 [batch][M][N_out] (row stride ldd)                                 */
  int64_t M, N, K;
  int64_t batch;
  int64_t lda, ldb, ldd;             /* elements */
  int64_t strideA, strideB, strideD; /* batch strides, elements; strideB == 0 → B shared by all batches */
  float alpha;
  const float* bias_n; /* fp32 [N] or NULL */
  const float* bias_m; /* fp32 [M] or NULL */
  const float* bias_g; /* fp32 [M / bias_g_rows][N] or NULL (e.g. time-embedding add of a ResnetBlock2D) */
  int64_t bias_g_rows;
  const void* residual; /* [batch][M or res_row_mod][N_out] or NULL */
  int32_t residual_dtype; /* SEEDX_F16 / SEEDX_F32 */
  int64_t ldr, strideR, res_row_mod;
  int32_t act;       /* SEEDX_ACT_* */
  int32_t gated;     /* 0/1 */
  int32_t out_dtype; /* SEEDX_F16 / SEEDX_F32 */
  /* conv mode */
  int32_t conv_taps_h, conv_taps_w; /* 0,0 = plain GEMM; 3,3 or 1,1 */
  int64_t conv_n, conv_h, conv_w, conv_c;
  int32_t tile_n;    /* 0 = auto (wave/cycle model); else one of 64/96/128/144/160/192/208/224/240/256 accumulator columns */
  /* ABI 2 --------------------------------------------------------------------------------------------------------------------------
   * LayerNorm folded into the GEMM (diffusers BasicTransformerBlock.norm{1,2,3} -> to_q/to_k/to_v / ff.net.0.proj, reached from
   * pipeline_stable_diffusion_xl_t2i_edit.py:915-922): with A = the UN-normalised rows x, B = W * gamma (per input column, folded at load
   * time) and bias_n = W . beta (+ the layer's bias),  LN(x) . W^T = rstd[m] * (x . B^T - mean[m] * colsum[n]) + bias_n,  colsum[n] = sum_k B[n][k].
   * ln_stats = fp32 [M][2] (mean, rstd) from seedx_row_stats; applied right after alpha*acc, before the biases.  NULL = off. */
  const float* ln_stats;
  const float* ln_colsum; /* fp32 [N] */
  /* B is produced by the kernel launched just before this one on the same stream (activation x activation products).  Default 0: B holds
   * weights, whose first tiles are requested before the programmatic-dependent-launch wait. */
  int32_t b_dynamic;
  /* ln_parts > 0: ln_stats is NOT (mean, rstd) but ln_parts x [M] fp32 pairs (sum, sum of squares) as written through row_part by the GEMM
   * that produced A (K = 32 * ln_parts columns); mean / rstd are then formed in this epilogue with ln_eps. */
  int32_t ln_parts;
  float ln_eps;
  /* Statistics of the stored fp16 output for the normalisation that reads it next, emitted by the epilogue (no extra pass over the tensor):
   *   row_part fp32 [N/32][M][2]: per row, (sum, sum of squares) over each 32-column chunk  -> LayerNorm folded into the next GEMM (ln_parts)
   *   col_part fp32 [M/32][N][2]: per column, (sum, sum of squares) over each 32-row slab   -> seedx_groupnorm_nhwc_from_partials
   * Requirements: fp16 output, 16-byte aligned rows, no gating, batch 1, M % 32 == 0, N % 32 == 0.  NULL = off. */
  float* row_part;
  float* col_part;
  /* With row_part: the epilogue warp that delivers the last partial of a 32-row slab reduces the slab's partials (chunk order) to (mean, rstd) and
   * stores them in row_stats_out fp32 [M][2] with eps row_eps — what seedx_row_stats_from_partials computes, without the extra launch.
   * row_tickets: uint32 [M/32], zero before the launch; the kernel leaves them zero. */
  float* row_stats_out;
  uint32_t* row_tickets;
  float row_eps;
} seedx_gemm_args;

int seedx_gemm_f16(const seedx_gemm_args* args, void* stream);
/* A/B switch for the cluster-pair variant (two CTAs on vertically adjacent 128 x tile_n tiles, each CTA loading its own 128 rows of A and
 * half of the B tile, which TMA multicasts to both): 0 = off, 1 = auto (default; single-CTA tiles, the faster choice measured on H100),
 * 2 = whenever legal */
void seedx_gemm_set_cluster(int mode);
/* developer aid: device buffer of 8 uint64 per CTA that receives %globaltimer phase stamps of the following GEMM launches (NULL = off) */
void seedx_gemm_set_debug(void* device_buffer);
/* Stream-K schedule of the cluster-pair kernels (seedx_gemm_set_cluster(2)) for launches whose last wave of whole tiles would leave SMs idle (e.g. M = 8192, N = 1280: 192 pair-tiles on 66 cluster pairs =
 * 2.9 waves): every cluster takes an equal share of the (tile, k-block) iterations; partial accumulators of split tiles go through a workspace.
 * seedx_gemm_set_workspace hands the library that workspace (>= 32 MB recommended, 256-byte aligned, first 16 KB zero-filled by the caller, owned
 * by the caller, used by one stream at a time); without it, or with mode 0, every launch is data-parallel.  mode: 0 off, 1 auto (default), 2 always. */
int seedx_gemm_set_workspace(void* device_buffer, int64_t bytes);
void seedx_gemm_set_stream_k(int mode);
/* A/B switch for the epilogue: 1 (default) = output/residual tiles staged in shared memory and moved by TMA, 0 = direct row-per-thread stores */
void seedx_gemm_set_tma_epilogue(int on);
/* what the most recent seedx_gemm_f16 launch ran, as decided on the host: out = {tile width, CTAs per cluster (1/2), stream-K (0/1),
 * TMA epilogue (0/1), 16-byte vector stores allowed for the direct epilogue (0/1), pipeline stages}; all zero before the first launch */
void seedx_gemm_last_config(int32_t out[6]);
/* The same GEMM on FP8 operands: A and B are e4m3 (OCP "fn" variant, float8_e4m3fn) with one fp32 scale per row of each, so that row m of the
 * true A is a_scale[m] * A[m, :] and row n of the true B is b_scale[n] * B[n, :].  lda / ldb are in elements (= bytes); rows start 16-byte
 * aligned (K % 16 == 0, lda % 16 == 0, ldb % 16 == 0).  The wgmma MMAs take 32 e4m3 values of K per step (QGMMA) at twice the fp16 rate.
 * epilogue order: x = (acc * a_scale[m]) * b_scale[n]   (fp32, each product rounded), then exactly the seedx_gemm_f16 epilogue on x in place of
 *                 the accumulator: x = alpha*x (or the folded-LayerNorm form rstd*x + bias - rstd*mean*colsum); biases; activation or gating;
 *                 residual; store; row / column statistics.
 * Every other field of args means what it means for seedx_gemm_f16.  Rejected (error, nothing launched): conv mode, batch != 1, a NULL scale,
 * tile_n other than 0 (auto) / 64 / 128 / 160 / 192 / 224 / 256.  Runs single-CTA tiles with the data-parallel schedule only (no cluster pairs,
 * no stream-K); seedx_gemm_last_config reports it like any other launch. */
int seedx_gemm_fp8(const seedx_gemm_args* args, const float* a_scale, const float* b_scale, void* stream);
/* Per-row FP8 quantisation of fp16 activations [rows, cols] (row stride ldx): scale[r] = amax_c |x[r, c]| / 448 (1 for an all-zero row) and
 * q[r, c] = e4m3_rn(clamp(x[r, c] / scale[r], -448, 448)) with IEEE division, written to q (e4m3, row stride ldq bytes).  One read of the row,
 * 16-byte loads and stores.  Requires ldx % 8 == 0, ldq % 16 == 0, 16-byte aligned x and q, cols <= 8192.  Feeds the A operand of seedx_gemm_fp8. */
int seedx_quant_rows_fp8(const void* x, int64_t ldx, int64_t rows, int64_t cols, void* q, int64_t ldq, float* scale, void* stream);
/* The implicit-GEMM conv of seedx_gemm_f16 on FP8 operands: A is the NHWC e4m3 image [conv_n, conv_h, conv_w, conv_c] with one fp32 scale per
 * IMAGE (a_scale[conv_n]: a scale constant over K is the only one the conv sum can carry, and no image's quantisation depends on the rest of the
 * batch); B is e4m3 [N, taps*taps*roundup(C,128)] (k = (kh*taps + kw)*Cpad + c, zero channel padding) with one fp32 scale per output channel.
 * Each 128-element k-block is summed by the MMAs from zero and then added into an fp32 accumulator, so long K (up to 23 040 for the UNet's
 * 3x3 convs) keeps fp32 accuracy.  epilogue: x = (acc * a_scale[m / (H*W)]) * b_scale[n], then exactly the seedx_gemm_f16 conv epilogue
 * (alpha, bias_n, per-image bias_g, activation, residual, store, col_part).  Rejected (error, nothing launched): a non-conv call, batch != 1,
 * a NULL scale, C % 16 != 0, K != taps^2 * roundup(C,128), tile_n other than 0 (auto) / 64 / 128 / 160, and every image geometry the fp16 conv
 * rejects.  Single-CTA tiles, data-parallel schedule; seedx_gemm_last_config reports it like any other launch. */
int seedx_conv_fp8(const seedx_gemm_args* args, const float* a_scale, const float* b_scale, void* stream);
/* Per-image FP8 quantisation of a contiguous fp16 tensor seen as [n, per_image] (an NHWC map, one row per image): scale[i] = amax |x[i, :]| / 448
 * (1 for an all-zero image) and q[i, :] = e4m3_rn(clamp(x[i, :] / scale[i], -448, 448)) with IEEE division, q contiguous e4m3.  Two launches
 * (per-chunk maxima into ws, then the per-image maximum and the conversion), deterministic.  ws: seedx_quant_images_fp8_ws_bytes(n, per_image)
 * bytes, no initial contents.  Requires per_image % 16 == 0, 16-byte aligned x and q, n <= 65535.  Feeds the A operand of seedx_conv_fp8. */
int seedx_quant_images_fp8(const void* x, int64_t n, int64_t per_image, void* q, float* scale, void* ws, void* stream);
int64_t seedx_quant_images_fp8_ws_bytes(int64_t n, int64_t per_image);


/* ------------------------------------------------------------------------------------------------
 * Fused softmax attention (flash-style; scores never reach HBM).  fp16 q/k/v/o, fp32 softmax.
 *   O[b,h,i,:] = softmax_j(scale * Q[b,h,i,:].K[b,h,j,:] (+causal: j <= i + sk - sq)) V[b,h,j,:]
 * Strides are in elements; a batch stride of 0 shares the tensor across the batch (learned queries).
 * replaces: src/models/tokenizer/qwen_visual.py:204-215 (ViT MHSA d=104) and :146 (nn.MultiheadAttention in Resampler,
 *   d=128/160); src/models/mllm/modeling_llama_xformer.py:225-237 (xformers memory_efficient_attention, causal prefill);
 *   src/models/detokenizer/resampler.py:62-73,104-116; diffusers AttnProcessor2_0 (F.scaled_dot_product_attention).
 * ---------------------------------------------------------------------------------------------- */
typedef struct seedx_attn_args {
  const void* q; const void* k; const void* v; void* o;
  int64_t q_stride_b, q_stride_h, q_stride_s;
  int64_t k_stride_b, k_stride_h, k_stride_s;
  int64_t v_stride_b, v_stride_h, v_stride_s;
  int64_t o_stride_b, o_stride_h, o_stride_s;
  int32_t batch, heads, sq, sk, d;
  float scale;
  int32_t causal;
} seedx_attn_args;

int seedx_attention_f16(const seedx_attn_args* args, void* stream);
/* implementation switch for A/B tests: 0 = auto (wgmma kernel when d <= 128, sq >= 64 and sk >= 16, else mma.sync), 1 = always mma.sync */
void seedx_attention_set_impl(int impl);
int seedx_attention_last_impl(void); /* most recent call: 2 = wgmma, 1 = mma.sync */

/* ------------------------------------------------------------------------------------------------
 * LayerNorm (rms=0) / RMSNorm (rms=1) over the last dimension, fp32 statistics.
 *   y = (x - mean) * rsqrt(var + eps) * gamma + beta ;  out2 (optional) = y + add[row % add_rows][:]
 * replaces nn.LayerNorm at qwen_visual.py:400,280-281,139-141,414; resampler.py:55-56,279; diffusers
 *   BasicTransformerBlock.norm{1,2,3}; transformers LlamaRMSNorm used at modeling_llama_xformer.py:95,258-259,443.
 * ---------------------------------------------------------------------------------------------- */
int seedx_layernorm(const void* x, int x_dtype, int64_t ldx, const float* gamma, const float* beta, void* out, int out_dtype,
                    int64_t ldo, void* out2, const float* add, int64_t add_rows, int64_t rows, int64_t cols, float eps,
                    int rms, void* stream);

/* per-row LayerNorm statistics of an fp16 matrix: stats[r] = (mean, 1/sqrt(var + eps)) over cols columns, fp32, two-pass on the cached row.
 * Feeds the folded-LayerNorm epilogue of seedx_gemm_f16 (ln_stats): the normalised activations are never written to memory. */
int seedx_row_stats(const void* x, int x_dtype, int64_t ldx, int64_t rows, int64_t cols, float eps, float* stats, void* stream);
/* the same statistics from the row partials a producing GEMM emitted through seedx_gemm_args.row_part (fp32 [nparts][rows][2], cols = 32 * nparts):
 * nparts * 8 bytes are read per row instead of the row */
int seedx_row_stats_from_partials(const float* parts, int nparts, int64_t rows, int64_t cols, float eps, float* stats, void* stream);

/* ------------------------------------------------------------------------------------------------
 * GroupNorm (+ optional SiLU) on NHWC fp16 images; the input may be the channel-concatenation [x1 | x2] (UNet skip
 * connections); raw_out (optional) receives the un-normalised concatenation.  stats_ws: seedx_groupnorm_ws_bytes(n, groups) bytes of
 * scratch, 8-byte aligned (contents need not be initialised).  The statistics are reduced in a fixed order: results are
 * bit-reproducible run to run, like torch's GroupNorm.
 * replaces diffusers ResnetBlock2D.norm1/norm2 + nonlinearity, Transformer2DModel.norm, UNet conv_norm_out, VAE norms
 *   (SURVEY.md Appendix B.2), reached from pipeline_stable_diffusion_xl_t2i_edit.py:915-922,973.
 * ---------------------------------------------------------------------------------------------- */
int seedx_groupnorm_nhwc(const void* x1, int64_t c1, const void* x2, int64_t c2, int64_t n, int64_t hw, int groups,
                         const float* gamma, const float* beta, float eps, int silu_act, void* out, void* raw_out,
                         void* stats_ws, void* stream);
int64_t seedx_groupnorm_ws_bytes(int64_t n, int groups);
/* Same normalisation, with the statistics taken from the column partials the producing GEMM / conv epilogues wrote (col_part of
 * seedx_gemm_args: fp32 [n*hw/32][c][2], hw % 32 == 0) instead of a pass over the tensor: a finalize kernel adds the partials of each
 * (image, group) in a fixed order (bit-reproducible), then the same apply pass runs.  part2 belongs to x2 (NULL when x2 is NULL). */
int seedx_groupnorm_nhwc_from_partials(const void* x1, int64_t c1, const float* part1, const void* x2, int64_t c2, const float* part2, int64_t n,
                                       int64_t hw, int groups, const float* gamma, const float* beta, float eps, int silu_act, void* out,
                                       void* raw_out, void* stats_ws, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Small HBM-bound data-movement kernels
 * ---------------------------------------------------------------------------------------------- */
/* NCHW image -> patch rows [n*gh*gw, kpad] fp16, k = c*p*p + i*p + j, zero padded to kpad
 * (im2col of the stride-14 patch-embed conv, qwen_visual.py:352,393-396) */
int seedx_patchify(const void* x, int x_dtype, int64_t n, int64_t c, int64_t h, int64_t w, int64_t patch, void* out,
                   int64_t kpad, void* stream);
/* elementwise dtype conversion (fp16 <-> fp32), count elements */
int seedx_cast(const void* src, int src_dtype, void* dst, int dst_dtype, int64_t count, void* stream);
/* mean over groups of `k` consecutive tokens: [n, t, c] -> [n, t/k, c]  (F.avg_pool1d at adapter_modules.py:112-115) */
int seedx_avgpool_tokens(const void* x, int dtype, int64_t n, int64_t t, int64_t c, int64_t k, void* out, void* stream);

/* k x k / stride-s patch gather on NHWC fp16 -> [n*ho*wo, k*k*c] (feeds seedx_gemm_f16 for the stride-2 downsample convs of
 * the UNet (pad 1) and of the VAE encoder (asymmetric pad (0,1): pad_before = 0); c % 8 == 0) */
int seedx_im2col_nhwc(const void* x, int64_t n, int64_t h, int64_t w, int64_t c, int k, int stride, int pad_before, int64_t ho,
                      int64_t wo, void* out, void* stream);
/* nearest-neighbour 2x upsample on NHWC fp16 (diffusers Upsample2D before its 3x3 conv) */
int seedx_upsample2x_nhwc(const void* x, int64_t n, int64_t h, int64_t w, int64_t c, void* out, void* stream);
/* diffusers Timesteps(dim, flip_sin_to_cos=True, shift=0): out[i, 0:dim] = [cos | sin](t[i] * 10000^(-j/(dim/2))), fp16, row stride ldo */
int seedx_timestep_embedding(const float* t, int64_t count, int dim, void* out, int64_t ldo, void* stream);
/* out[r, c] = act(x[r, c]) as fp16 (strided rows; act = SEEDX_ACT_*; NONE = plain cast/copy) */
int seedx_unary_f16(const void* x, int x_dtype, int64_t rows, int64_t cols, int64_t ldx, void* out, int64_t ldo, int act, void* stream);
/* out = softmax(scale * x) along rows, fp32 math, fp16 out (VAE mid-block single-head attention, d=512) */
int seedx_softmax_rows(const void* x, int x_dtype, int64_t ldx, int64_t rows, int64_t cols, float scale, void* out, int64_t ldo, void* stream);
/* layout converters at the pipeline boundary (latents / images are NCHW fp32 in the reference API) */
int seedx_nchw_to_nhwc_f16(const float* x, int64_t n, int64_t c, int64_t hw, int64_t cpad, float scale, void* out, void* stream);
int seedx_nhwc_to_nchw_f32(const void* x, int x_dtype, int64_t n, int64_t c, int64_t hw, int64_t ldc, float scale, float* out, void* stream);
/* VaeImageProcessor.postprocess: (x/2+0.5).clamp(0,1)*255 -> uint8 HWC (first 3 channels of an NHWC tensor with row stride ldc) */
int seedx_image_to_u8(const void* x, int x_dtype, int64_t pixels, int64_t ldc, uint8_t* out, void* stream);
/* one denoising step on the fp32 sampler state: CFG combine + EulerDiscreteScheduler.step + scale_model_input for the next step.
 * branches = 2: t2i, eps batch order [uncond, text] (diffusers StableDiffusionXLPipeline via adapter_modules.py:156-167)
 * branches = 3: edit, order [text, image, uncond], sigma-space combine (pipeline_stable_diffusion_xl_t2i_edit.py:905-953)
 * eps == NULL: initialisation, x *= init_sigma (prepare_latents, pipeline...edit.py:474-488) */
int seedx_cfg_euler_step(const float* eps, float* x, void* unet_in, int64_t batch, int64_t hw, int branches, float guidance,
                         float image_guidance, float sigma, float sigma_next, float init_sigma, void* stream);
/* the same step for `slots` independent requests (continuous batching of the denoising loop), each at its own point of its own schedule:
 *   state     int32 [slots][2]              (step index i, step count n) of each slot; a slot is live while i < n
 *   sigmas    fp32  [slots][max_steps + 1]  its EulerDiscreteScheduler sigmas (entry n = 0), timesteps fp32 [slots][max_steps]
 *   scalars   fp32  [slots][3]              guidance, image guidance, init_noise_sigma of its step count
 *   t_dev     fp32  [branches * slots]      per-row UNet timestep, row br * slots + s; x / unet_in / eps as above with batch = slots
 * eps != NULL: every live slot s combines with its own g, ig, sigma = sigmas[s][i], sigma_next = sigmas[s][i+1] (bit-identical to
 * seedx_cfg_euler_step given the same fp32 values), writes x[s] and channels 0..3 of its unet_in rows, then i += 1 and, while i < n,
 * t_dev rows = timesteps[s][i] (two launches: combine, then a one-CTA advance).  fresh_mask must be 0.
 * eps == NULL: initialises exactly the slots whose bit is set in fresh_mask (!= 0): x = x * init_noise_sigma, unet_in scaled by sigmas[s][0],
 * t_dev rows = timesteps[s][0]; state is not touched (one launch).
 * Slots not live / not fresh keep x, unet_in and t_dev bytes.  1 <= slots <= 64, max_steps >= 1, branches 2 or 3; eps / unet_in 16-byte aligned. */
int seedx_cfg_euler_slots(const float* eps, float* x, void* unet_in, float* t_dev, int32_t* state, const float* sigmas, const float* timesteps,
                          const float* scalars, int64_t slots, int64_t hw, int branches, int64_t max_steps, uint64_t fresh_mask, void* stream);

/* ------------------------------------------------------------------------------------------------
 * LLaMA token loop (greedy decode of up to 8 sequences in lock-step; HBM-bound) and prefill glue.  Device-resident state:
 *   seq   int32 [batch][max_len]  prompt ids followed by generated ids
 *   state int32 [batch][4]        [0] current length, [1] 1-based index of the generated EOS (0 = none), [2] #generated, [3] prompt length
 * ---------------------------------------------------------------------------------------------- */
/* out[b][N or N/2] = epi(W[N,K] . (rms_w ? rmsnorm(x[b])*rms_w : x[b])), b < batch (1, 2, 4 or 8); the fp16 weight matrix is
 * streamed once for all sequences.  gated: out[j] = r[2j] * silu(r[2j+1]); else += residual[b].  Row strides ldx/ldr/ldo in elements.
 * replaces the M=1 projections of modeling_llama_xformer.py:204-206,239,166-167,707 (+ LlamaRMSNorm :258-259,443) */
int seedx_gemv_f16(const void* W, const float* x, int64_t ldx, const float* rms_w, float eps, const float* residual, int64_t ldr, float* out,
                   int64_t ldo, int64_t N, int64_t K, int batch, int gated, void* stream);
/* the same GEMV over FP8 weights: W8 = e4m3 (OCP "fn" variant) [N, K] row-major, 16B aligned, K % 64 == 0; row_scale fp32 [N], weight
 * row n = row_scale[n] * W8[n, :].  The scale multiplies the fp32 dot product: out[b][n] = s[n] * dot(n, b) (+ residual[b][n]); gated (rows
 * interleaved [up_j, gate_j]): out[b][j] = s[2j] * up * silu(s[2j+1] * gate).  Half the weight bytes of seedx_gemv_f16 per token. */
int seedx_gemv_fp8(const void* W8, const float* row_scale, const float* x, int64_t ldx, const float* rms_w, float eps, const float* residual,
                   int64_t ldr, float* out, int64_t ldo, int64_t N, int64_t K, int batch, int gated, void* stream);
/* fp16 out[n, k] = (half)(float(W8[n, k]) * row_scale[n]) for an FP8 weight [N, K] (K % 16 == 0, W8 and out 16B aligned): feeds the prefill
 * GEMM of an FP8 model.  Its stores wait for the preceding kernel (PDL), so out may be a scratch buffer that kernel still reads; the GEMM that
 * reads out must treat it as a dynamic operand (seedx_gemm_args.b_dynamic = 1). */
int seedx_dequant_fp8(const void* W8, const float* row_scale, void* out, int64_t N, int64_t K, void* stream);
/* one new token per sequence: RoPE(q,k) (:141-149), append k,v at position state[b][0]-1 (replaces torch.cat :215-218), attention
 * over the cache (:225-237).  qkv fp32 [batch][3*H*d]; caches fp16 [batch][max_len, H*d] (cache_stride elements apart); out fp32 [batch][H*d] */
int seedx_decode_attention(const float* qkv, const int32_t* state, const float* inv_freq, void* kcache, void* vcache, int64_t cache_stride,
                           float* out, int batch, int heads, int head_dim, float scale, void* stream);
/* prefill: RoPE q,k in place on fp16 [tokens, 3*H*d] for positions pos0.., and copy k,v rows into the caches */
int seedx_rope_kv_prefill(void* qkv, int64_t tokens, int64_t pos0, int heads, int head_dim, const float* inv_freq, void* kcache, void* vcache,
                          void* stream);
/* Paged KV cache (vLLM-style): the cache of a layer is a pool of pages, fp16 [n_pages][page_size tokens][H*d]; sequence b reads / appends through
 * its row of the page table (int32 [batch][table_stride]: physical page of logical page t / page_size; page_size a power of two).  Same arithmetic
 * as the two calls above; replaces the per-step torch.cat growth of past_key_value (modeling_llama_xformer.py:215-218) without tying a sequence to
 * one contiguous slab. */
int seedx_decode_attention_paged(const float* qkv, const int32_t* state, const float* inv_freq, void* kpool, void* vpool, const int32_t* page_table,
                                 int64_t table_stride, int64_t page_size, float* out, int batch, int heads, int head_dim, float scale, void* stream);
int seedx_rope_kv_prefill_paged(void* qkv, int64_t tokens, int64_t pos0, int heads, int head_dim, const float* inv_freq, void* kpool, void* vpool,
                                const int32_t* page_table_row, int64_t page_size, void* stream);
/* embedding rows -> fp32 [n, dim]; ids == NULL: row b = last token of device sequence b (seq[b*seq_stride + state[b][0]-1]) */
int seedx_embed_rows(const void* table, const int32_t* ids, const int32_t* state, const int32_t* seq, int64_t seq_stride, int64_t n, int64_t dim,
                     float* out, void* stream);
/* dst[idx[r], :] = src[src_idx ? src_idx[r] : r, :]  (input_embeds[ids_cmp_mask] = image_embeds_lm[embeds_cmp_mask], seed_x.py:173) */
int seedx_scatter_rows(const void* src, int src_dtype, const int32_t* src_idx, const int32_t* idx, int64_t n, int64_t dim, float* dst,
                       void* stream);
/* hidden[b][state[b][0] - state[b][3] - 1, :] = x[b]  (last_hidden_states harvest, seed_x.py:196-197) */
int seedx_store_hidden(const float* x, const int32_t* state, int batch, int64_t max_rows, int64_t dim, float* hidden, void* stream);
/* AutoImageTokenGenerationProcessor (generation.py:19-31) + argmax + append to seq/state per sequence, no host sync.  A sequence whose state[b][1]
 * is non-zero (EOS produced, or retired by the host in continuous batching) is parked: nothing is appended and its length stops growing. */
int seedx_logits_argmax(float* logits, int64_t vocab, const int32_t* img_ids, int n_img_ids, int32_t* seq, int32_t* state, int batch, int eos_id,
                        int suppress_eos, int64_t max_len, void* stream);

/* out[r,:] = fp16(a[r,:] + b[r % b_rows,:]), b fp32 (AttentionPool2d positional add, src/models/detokenizer/resampler.py:93) */
int seedx_add_bcast_f16(const void* a, int a_dtype, const float* b, int64_t rows, int64_t cols, int64_t b_rows, void* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SEEDX_H_ */
