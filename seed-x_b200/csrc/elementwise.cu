// seedx-b200: small HBM-bound data-movement kernels (patchify / cast / token pooling ...).
// Each is a grid-stride loop with 16-byte accesses where the layout allows; reference call sites in include/seedx.h.
#include "common.cuh"
#include "../../include/seedx.h"

namespace seedx {
void count_launch();

static inline int grid_for(long long work, int threads) {
  long long b = (work + threads - 1) / threads;
  const long long cap = (long long)num_sms() * 16;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (int)b;
}

template <typename TI>
__global__ void patchify_kernel(const TI* __restrict__ x, int n, int c, int h, int w, int patch, __half* __restrict__ out, int kpad) {
  pdl_wait();
  pdl_trigger();
  const int gh = h / patch, gw = w / patch;
  const long long total = (long long)n * gh * gw * kpad;
  const int kreal = c * patch * patch;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int k = (int)(i % kpad);
    const long long row = i / kpad;
    float v = 0.f;
    if (k < kreal) {
      const int ci = k / (patch * patch);
      const int rem = k - ci * patch * patch;
      const int pi = rem / patch, pj = rem - pi * patch;
      const int gx = (int)(row % gw);
      const long long t = row / gw;
      const int gy = (int)(t % gh);
      const int img = (int)(t / gh);
      v = (float)x[(((long long)img * c + ci) * h + gy * patch + pi) * w + gx * patch + pj];
    }
    out[i] = __float2half_rn(v);
  }
}

template <typename TI, typename TO>
__global__ void cast_kernel(const TI* __restrict__ s, TO* __restrict__ d, long long n) {
  pdl_wait();
  pdl_trigger();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    d[i] = (TO)(float)s[i];
}

template <typename T>
__global__ void avgpool_tokens_kernel(const T* __restrict__ x, long long n_out_rows, int c, int k, T* __restrict__ out) {
  pdl_wait();
  pdl_trigger();
  const long long total = n_out_rows * c;
  const float inv = 1.f / (float)k;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / c;
    const int ch = (int)(i - r * c);
    float s = 0.f;
    for (int j = 0; j < k; ++j) s += (float)x[(r * k + j) * c + ch];
    out[i] = (T)(s * inv);
  }
}


// Per-row FP8 (e4m3) quantisation of fp16 activations, the A operand of seedx_gemm_fp8: s = amax / 448 (1 for an all-zero row),
// q = e4m3_rn(clamp(x / s, +-448)) with IEEE division.  One warp per row; a lane holds NV units of 16 columns (two 16-byte loads, one 16-byte
// store) in registers between the row maximum and the conversion, so the row is read once.  Columns past the last whole unit (< 16) take one
// lane each.
SEEDX_DEVINL uint16_t f32x2_to_e4m3x2(float lo, float hi) {   // lo -> low byte (the lower column)
  uint16_t r;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;\n" : "=h"(r) : "f"(hi), "f"(lo));
  return r;
}
SEEDX_DEVINL float fp8_quant_val(float x, float s) { return fminf(fmaxf(__fdiv_rn(x, s), -448.f), 448.f); }

template <int NV>
__global__ void __launch_bounds__(128)
quant_rows_fp8_kernel(const __half* __restrict__ x, long long ldx, long long rows, int cols, uint8_t* __restrict__ q, long long ldq,
                      float* __restrict__ scale) {
  pdl_wait();
  pdl_trigger();
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const __half* xr = x + row * ldx;
  uint8_t* qr = q + row * ldq;
  const int units = cols >> 4;
  uint4 v[NV][2];
  __half2 mx = __float2half2_rn(0.f);
#pragma unroll
  for (int j = 0; j < NV; ++j) {
    const int u = lane + 32 * j;
    if (u < units) {
      v[j][0] = __ldg((const uint4*)(xr + 16 * u));
      v[j][1] = __ldg((const uint4*)(xr + 16 * u + 8));
      const __half2* h0 = (const __half2*)&v[j][0];
      const __half2* h1 = (const __half2*)&v[j][1];
#pragma unroll
      for (int e = 0; e < 4; ++e) mx = __hmax2(mx, __hmax2(__habs2(h0[e]), __habs2(h1[e])));
    }
  }
  const int tcol = 16 * units + lane;
  const float tv = tcol < cols ? __half2float(xr[tcol]) : 0.f;
  const float amax = warp_max(fmaxf(fmaxf(__low2float(mx), __high2float(mx)), fabsf(tv)));
  float s = __fdiv_rn(amax, 448.f);
  s = s > 0.f ? s : 1.f;
  if (lane == 0) scale[row] = s;
#pragma unroll
  for (int j = 0; j < NV; ++j) {
    const int u = lane + 32 * j;
    if (u < units) {
      uint32_t o[4];
#pragma unroll
      for (int w = 0; w < 4; ++w) {   // 4 output words of 4 values: halves 2w, 2w+1 of the 16
        const uint4& src = v[j][w >> 1];
        const uint32_t a0 = (w & 1) ? src.z : src.x, a1 = (w & 1) ? src.w : src.y;
        const float2 f0 = __half22float2(*(const __half2*)&a0), f1 = __half22float2(*(const __half2*)&a1);
        const uint32_t lo = f32x2_to_e4m3x2(fp8_quant_val(f0.x, s), fp8_quant_val(f0.y, s));
        const uint32_t hi = f32x2_to_e4m3x2(fp8_quant_val(f1.x, s), fp8_quant_val(f1.y, s));
        o[w] = lo | (hi << 16);
      }
      *(uint4*)(qr + 16 * u) = make_uint4(o[0], o[1], o[2], o[3]);
    }
  }
  if (tcol < cols) qr[tcol] = (uint8_t)f32x2_to_e4m3x2(fp8_quant_val(tv, s), 0.f);
}

// Per-image FP8 (e4m3) quantisation of a contiguous fp16 tensor seen as [n, per_image] (an NHWC activation, one row per image): the A operand
// of seedx_conv_fp8.  An image (up to 128 x 128 x 960 values) is far more than a warp's registers hold, so it takes two launches over
// (chunk, image), QI_CHUNK values per CTA:
//   1. quant_images_amax_kernel: the |x| maximum of every chunk -> ws[image][chunk];
//   2. quant_images_fp8_kernel: every CTA reduces its image's chunk maxima (a maximum is order-free: deterministic, with no atomics and no
//      zero fill), s = amax / 448 (1 for an all-zero image), and converts its chunk, q = e4m3_rn(clamp(x / s, +-448)) with IEEE division.
// A thread holds QI_UNITS units of 16 values: two 16-byte loads and one 16-byte store each.
constexpr int QI_THREADS = 256;
constexpr int QI_UNITS = 2;
constexpr int QI_CHUNK_UNITS = QI_THREADS * QI_UNITS;
constexpr int QI_CHUNK = 16 * QI_CHUNK_UNITS;   // 8192 values

SEEDX_DEVINL float block_max_qi(float v, float* sm) {   // every thread gets the CTA's maximum
  v = warp_max(v);
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = v;
  __syncthreads();
  return warp_max((threadIdx.x & 31) < QI_THREADS / 32 ? sm[threadIdx.x & 31] : 0.f);
}

__global__ void __launch_bounds__(QI_THREADS)
quant_images_amax_kernel(const __half* __restrict__ x, long long per_image, float* __restrict__ ws) {
  __shared__ float sm[QI_THREADS / 32];
  pdl_wait();
  pdl_trigger();
  const long long units = per_image >> 4;
  const __half* xi = x + (long long)blockIdx.y * per_image;
  __half2 mx = __float2half2_rn(0.f);
#pragma unroll
  for (int j = 0; j < QI_UNITS; ++j) {
    const long long u = (long long)blockIdx.x * QI_CHUNK_UNITS + j * QI_THREADS + threadIdx.x;
    if (u < units) {
      const uint4 a = __ldg((const uint4*)(xi + 16 * u)), b = __ldg((const uint4*)(xi + 16 * u + 8));
      const __half2* h0 = (const __half2*)&a;
      const __half2* h1 = (const __half2*)&b;
#pragma unroll
      for (int e = 0; e < 4; ++e) mx = __hmax2(mx, __hmax2(__habs2(h0[e]), __habs2(h1[e])));
    }
  }
  const float amax = block_max_qi(fmaxf(__low2float(mx), __high2float(mx)), sm);
  if (threadIdx.x == 0) ws[(long long)blockIdx.y * gridDim.x + blockIdx.x] = amax;
}

__global__ void __launch_bounds__(QI_THREADS)
quant_images_fp8_kernel(const __half* __restrict__ x, long long per_image, const float* __restrict__ ws, uint8_t* __restrict__ q,
                        float* __restrict__ scale) {
  __shared__ float sm[QI_THREADS / 32];
  pdl_wait();                               // the chunk maxima of launch 1
  pdl_trigger();
  const long long units = per_image >> 4;
  const long long base = (long long)blockIdx.y * per_image;
  uint4 v[QI_UNITS][2];
#pragma unroll
  for (int j = 0; j < QI_UNITS; ++j) {
    const long long u = (long long)blockIdx.x * QI_CHUNK_UNITS + j * QI_THREADS + threadIdx.x;
    if (u < units) {
      v[j][0] = __ldg((const uint4*)(x + base + 16 * u));
      v[j][1] = __ldg((const uint4*)(x + base + 16 * u + 8));
    }
  }
  const int chunks = (int)gridDim.x;
  float m = 0.f;
  for (int i = threadIdx.x; i < chunks; i += QI_THREADS) m = fmaxf(m, __ldcg(ws + (long long)blockIdx.y * chunks + i));
  const float amax = block_max_qi(m, sm);
  float s = __fdiv_rn(amax, 448.f);
  s = s > 0.f ? s : 1.f;
  if (blockIdx.x == 0 && threadIdx.x == 0) scale[blockIdx.y] = s;
#pragma unroll
  for (int j = 0; j < QI_UNITS; ++j) {
    const long long u = (long long)blockIdx.x * QI_CHUNK_UNITS + j * QI_THREADS + threadIdx.x;
    if (u < units) {
      uint32_t o[4];
#pragma unroll
      for (int w = 0; w < 4; ++w) {   // 4 output words of 4 values: halves 2w, 2w+1 of the 16
        const uint4& src = v[j][w >> 1];
        const uint32_t a0 = (w & 1) ? src.z : src.x, a1 = (w & 1) ? src.w : src.y;
        const float2 f0 = __half22float2(*(const __half2*)&a0), f1 = __half22float2(*(const __half2*)&a1);
        const uint32_t lo = f32x2_to_e4m3x2(fp8_quant_val(f0.x, s), fp8_quant_val(f0.y, s));
        const uint32_t hi = f32x2_to_e4m3x2(fp8_quant_val(f1.x, s), fp8_quant_val(f1.y, s));
        o[w] = lo | (hi << 16);
      }
      *(uint4*)(q + base + 16 * u) = make_uint4(o[0], o[1], o[2], o[3]);
    }
  }
}

static int64_t quant_images_chunks(int64_t per_image) { return (per_image + QI_CHUNK - 1) / QI_CHUNK; }

// im2col for strided convs on NHWC fp16 (k x k taps, stride s, pad_before on top/left, zero fill), 8 channels / thread
__global__ void im2col_nhwc_kernel(const __half* __restrict__ x, int n, int h, int w, int c, int k, int stride, int pad, int ho, int wo,
                                   __half* __restrict__ out) {
  pdl_wait();
  pdl_trigger();
  const int cv = c >> 3;
  const long long total = (long long)n * ho * wo * k * k * cv;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % cv);
    long long r = i / cv;
    const int tap = (int)(r % (k * k));
    r /= (k * k);
    const int ox = (int)(r % wo);
    r /= wo;
    const int oy = (int)(r % ho);
    const int img = (int)(r / ho);
    const int iy = oy * stride + tap / k - pad, ix = ox * stride + tap % k - pad;
    uint4 q = make_uint4(0, 0, 0, 0);
    if (iy >= 0 && iy < h && ix >= 0 && ix < w) q = *(const uint4*)(x + (((long long)img * h + iy) * w + ix) * c + v * 8);
    *(uint4*)(out + i * 8) = q;
  }
}

__global__ void upsample2x_nhwc_kernel(const __half* __restrict__ x, int n, int h, int w, int c, __half* __restrict__ out) {
  pdl_wait();
  pdl_trigger();
  const int cv = c >> 3;
  const long long total = (long long)n * (2 * h) * (2 * w) * cv;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % cv);
    long long r = i / cv;
    const int ox = (int)(r % (2 * w));
    r /= (2 * w);
    const int oy = (int)(r % (2 * h));
    const int img = (int)(r / (2 * h));
    *(uint4*)(out + i * 8) = *(const uint4*)(x + (((long long)img * h + (oy >> 1)) * w + (ox >> 1)) * c + v * 8);
  }
}

// diffusers Timesteps(dim, flip_sin_to_cos=True, downscale_freq_shift=0): out[i, :] = [cos(t_i f_j) | sin(t_i f_j)]
__global__ void timestep_embedding_kernel(const float* __restrict__ t, int count, int dim, __half* __restrict__ out, long long ldo) {
  pdl_wait();
  pdl_trigger();
  const int half_dim = dim >> 1;
  const int total = count * half_dim;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int r = i / half_dim, j = i - r * half_dim;
    const float f = expf(-9.210340371976184f * (float)j / (float)half_dim);  // ln(10000)
    const float a = t[r] * f;
    out[(long long)r * ldo + j] = __float2half_rn(cosf(a));
    out[(long long)r * ldo + half_dim + j] = __float2half_rn(sinf(a));
  }
}

template <typename TI>
__global__ void unary_kernel(const TI* __restrict__ x, long long rows, int cols, long long ldx, __half* __restrict__ out, long long ldo, int act) {
  pdl_wait();
  pdl_trigger();
  const long long total = rows * cols;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / cols;
    const int c = (int)(i - r * cols);
    float v = (float)x[r * ldx + c];
    if (act == SEEDX_ACT_SILU) v = silu(v);
    else if (act == SEEDX_ACT_GELU_ERF) v = gelu_erf(v);
    out[r * ldo + c] = __float2half_rn(v);
  }
}

// row softmax: out = softmax(scale * x) ; one CTA per row, fp32 math
template <typename TI>
__global__ void __launch_bounds__(256) softmax_rows_kernel(const TI* __restrict__ x, long long ldx, int cols, float scale, __half* __restrict__ out,
                                                           long long ldo) {
  pdl_wait();
  pdl_trigger();
  __shared__ float sh[8];
  const TI* xr = x + (long long)blockIdx.x * ldx;
  __half* orow = out + (long long)blockIdx.x * ldo;
  float m = -INFINITY;
  for (int c = threadIdx.x; c < cols; c += 256) m = fmaxf(m, (float)xr[c] * scale);
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = m;
  __syncthreads();
  m = sh[0];
#pragma unroll
  for (int i = 1; i < 8; ++i) m = fmaxf(m, sh[i]);
  __syncthreads();
  float s = 0.f;
  for (int c = threadIdx.x; c < cols; c += 256) s += __expf((float)xr[c] * scale - m);
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = s;
  __syncthreads();
  s = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) s += sh[i];
  const float inv = 1.f / s;
  for (int c = threadIdx.x; c < cols; c += 256) orow[c] = __float2half_rn(__expf((float)xr[c] * scale - m) * inv);
}

// NCHW fp32 -> NHWC fp16 with channel padding and scale
__global__ void nchw_to_nhwc_kernel(const float* __restrict__ x, int n, int c, int hw, int cpad, float scale, __half* __restrict__ out) {
  pdl_wait();
  pdl_trigger();
  const long long total = (long long)n * hw * cpad;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int ch = (int)(i % cpad);
    const long long r = i / cpad;
    const int p = (int)(r % hw);
    const int img = (int)(r / hw);
    out[i] = __float2half_rn(ch < c ? x[((long long)img * c + ch) * hw + p] * scale : 0.f);
  }
}

template <typename TI>
__global__ void nhwc_to_nchw_kernel(const TI* __restrict__ x, int n, int c, int hw, int ldc, float scale, float* __restrict__ out) {
  pdl_wait();
  pdl_trigger();
  const long long total = (long long)n * c * hw;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int p = (int)(i % hw);
    const long long r = i / hw;
    const int ch = (int)(r % c);
    const int img = (int)(r / c);
    out[i] = (float)x[((long long)img * hw + p) * ldc + ch] * scale;
  }
}

// VaeImageProcessor.postprocess: (x/2 + 0.5).clamp(0,1) -> uint8 (round half to even like torch .round())
template <typename TI>
__global__ void image_to_u8_kernel(const TI* __restrict__ x, long long pixels, int ldc, uint8_t* __restrict__ out) {
  pdl_wait();
  pdl_trigger();
  const long long total = pixels * 3;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long p = i / 3;
    const int ch = (int)(i - p * 3);
    float v = (float)x[p * ldc + ch] * 0.5f + 0.5f;
    v = fminf(fmaxf(v, 0.f), 1.f);
    out[i] = (uint8_t)__float2int_rn(v * 255.f);
  }
}

// One sampler step (fp32 state): classifier-free guidance combine + Euler update + next-step UNet input.
//   eps   : fp32 NHWC [nb*B, HW, 4] UNet output (NULL -> initialisation: x = noise * init_sigma)
//   x     : fp32 NCHW [B, 4, HW] sampler state (in/out)
//   unet_in: fp16 NHWC [nb*B, HW, 8]; channels 0..3 <- x_new / sqrt(sigma_next^2 + 1) for every branch
//   mode 2 (t2i, branches [uncond, text])   : e = e_u + g (e_t - e_u)                       (adapter_modules.py:156-167 -> diffusers SDXL pipeline)
//   mode 3 (edit, branches [text, image, uncond]): sigma-space combine, pipeline_stable_diffusion_xl_t2i_edit.py:928-950
// The per-element arithmetic lives in cfg_euler_update / cfg_euler_input, shared with cfg_euler_slots_kernel: a slot of the continuous batcher
// gets the bits of this kernel given the same fp32 sigmas and guidance.  eps_at(br) returns the branch-br eps value of the element.
template <typename EpsAt>
SEEDX_DEVINL float cfg_euler_update(const EpsAt& eps_at, float xv, int mode, float g, float ig, float sigma, float sigma_next) {
  float e;
  if (mode == 2) {
    const float eu = eps_at(0);
    const float et = eps_at(1);
    e = eu + g * (et - eu);
  } else {
    const float et = xv - sigma * eps_at(0);
    const float ei = xv - sigma * eps_at(1);
    const float eu = xv - sigma * eps_at(2);
    const float c = eu + g * (et - ei) + ig * (ei - eu);
    e = (c - xv) / (-sigma);
  }
  const float x0 = xv - sigma * e;
  const float d = (xv - x0) / sigma;
  return xv + d * (sigma_next - sigma);
}

SEEDX_DEVINL __half cfg_euler_input(float xn, float sigma_next) { return __float2half_rn(xn * rsqrtf(sigma_next * sigma_next + 1.f)); }

__global__ void cfg_euler_kernel(const float* __restrict__ eps, float* __restrict__ x, __half* __restrict__ unet_in, int B, int hw, int mode,
                                 float g, float ig, float sigma, float sigma_next, float init_sigma) {
  pdl_wait();
  pdl_trigger();
  const long long total = (long long)B * hw * 4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int ch = (int)(i & 3);
    const long long r = i >> 2;
    const int p = (int)(r % hw);
    const int b = (int)(r / hw);
    const long long xi = ((long long)b * 4 + ch) * hw + p;
    float xv = x[xi];
    float xn;
    if (eps == nullptr) {
      xn = xv * init_sigma;
    } else {
      xn = cfg_euler_update([&](int br) { return eps[(((long long)(br * B + b)) * hw + p) * 4 + ch]; }, xv, mode, g, ig, sigma, sigma_next);
    }
    x[xi] = xn;
    const __half s = cfg_euler_input(xn, sigma_next);
    for (int br = 0; br < mode; ++br) unet_in[(((long long)(br * B + b)) * hw + p) * 8 + ch] = s;
  }
}

// The same step for S independent request slots (seedx_b200.serving.DenoiseBatcher), every slot at its own point of its own schedule:
//   state   int32 [S][2]         (step index i, step count n); slot s is live while i < n
//   sig     fp32  [S][max_steps+1] its sigmas (trailing 0), ts fp32 [S][max_steps] its timesteps, scal fp32 [S][3] (g, ig, init_noise_sigma)
// One thread per latent pixel: the 4 channels of a branch's eps are one 16-byte load, the 4 fp16 inputs one 8-byte store.  Slots that are
// not live (eps != NULL) / not in fresh_mask (eps == NULL) are skipped: their x, unet_in and t_dev rows keep their bytes.
// eps == NULL: initialisation of the fresh slots, x = noise * init_sigma[s], inputs scaled by sig[s][0], t_dev rows = ts[s][0].
// This kernel only reads state; the step index is advanced by cfg_euler_slots_advance_kernel, a separate launch that starts its work after
// every CTA here has finished (griddepcontrol.wait returns once the prerequisite grid has completed and its writes are visible), so no CTA
// can see a slot's index move in the middle of its step.
constexpr int SLOT_SCALARS = 3;

__global__ void cfg_euler_slots_kernel(const float* __restrict__ eps, float* __restrict__ x, __half* __restrict__ unet_in, float* __restrict__ t_dev,
                                       const int* __restrict__ state, const float* __restrict__ sig, const float* __restrict__ ts,
                                       const float* __restrict__ scal, int S, int hw, int mode, int max_steps, unsigned long long fresh_mask) {
  pdl_wait();
  pdl_trigger();
  const long long total = (long long)S * hw;
  for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r < total; r += (long long)gridDim.x * blockDim.x) {
    const int p = (int)(r % hw);
    const int s = (int)(r / hw);
    const float* sg = sig + (long long)s * (max_steps + 1);
    float sigma = 0.f, sigma_next, g = 0.f, ig = 0.f, init_sigma = 0.f;
    if (eps == nullptr) {
      if (!((fresh_mask >> s) & 1ull)) continue;
      sigma_next = sg[0];
      init_sigma = scal[s * SLOT_SCALARS + 2];
      if (p == 0)
        for (int br = 0; br < mode; ++br) t_dev[br * S + s] = ts[(long long)s * max_steps];
    } else {
      const int2 st = *(const int2*)(state + 2 * s);
      if (st.x >= st.y) continue;
      sigma = sg[st.x];
      sigma_next = sg[st.x + 1];
      g = scal[s * SLOT_SCALARS + 0];
      ig = scal[s * SLOT_SCALARS + 1];
    }
    float4 e4[3] = {};
    if (eps != nullptr) {
#pragma unroll
      for (int br = 0; br < 3; ++br)
        if (br < mode) e4[br] = __ldg((const float4*)(eps + (((long long)(br * S + s)) * hw + p) * 4));
    }
    uint32_t o[4];
#pragma unroll
    for (int ch = 0; ch < 4; ++ch) {
      const long long xi = ((long long)s * 4 + ch) * hw + p;
      const float xv = x[xi];
      const float xn = eps == nullptr ? xv * init_sigma
                                      : cfg_euler_update([&](int br) { return (&e4[br].x)[ch]; }, xv, mode, g, ig, sigma, sigma_next);
      x[xi] = xn;
      o[ch] = __half_as_ushort(cfg_euler_input(xn, sigma_next));
    }
    const uint2 ov = make_uint2(o[0] | (o[1] << 16), o[2] | (o[3] << 16));
    for (int br = 0; br < mode; ++br) *(uint2*)(unet_in + (((long long)(br * S + s)) * hw + p) * 8) = ov;
  }
}

// one thread per slot: a live slot moves to its next step and, while one remains, its t_dev rows take that step's timestep
__global__ void cfg_euler_slots_advance_kernel(float* __restrict__ t_dev, int* __restrict__ state, const float* __restrict__ ts, int S, int mode,
                                               int max_steps) {
  pdl_wait();                               // the combine launch has completed: nothing reads state[s][0] any more in this step
  pdl_trigger();
  const int s = threadIdx.x;
  if (s >= S) return;
  const int i = state[2 * s], n = state[2 * s + 1];
  if (i >= n) return;
  state[2 * s] = i + 1;
  if (i + 1 < n)
    for (int br = 0; br < mode; ++br) t_dev[br * S + s] = ts[(long long)s * max_steps + i + 1];
}


// out[r, :] = fp16( a[r, :] + b[r % b_rows, :] )   (positional-embedding add of AttentionPool2d, resampler.py:93)
template <typename TA>
__global__ void add_bcast_kernel(const TA* __restrict__ a, const float* __restrict__ b, long long rows, int cols, int b_rows,
                                 __half* __restrict__ out) {
  pdl_wait();
  pdl_trigger();
  const long long total = rows * cols;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / cols;
    const int c = (int)(i - r * cols);
    out[i] = __float2half_rn((float)a[i] + b[(r % b_rows) * cols + c]);
  }
}

}  // namespace seedx
using namespace seedx;

extern "C" int seedx_patchify(const void* x, int x_dtype, int64_t n, int64_t c, int64_t h, int64_t w, int64_t patch, void* out,
                              int64_t kpad, void* stream) {
  SEEDX_REQUIRE(x && out, "seedx_patchify: null pointer");
  SEEDX_REQUIRE(patch > 0 && h % patch == 0 && w % patch == 0, "seedx_patchify: image %lldx%lld not a multiple of patch %lld", (long long)h,
                (long long)w, (long long)patch);
  SEEDX_REQUIRE(kpad >= c * patch * patch, "seedx_patchify: kpad too small");
  const long long total = n * (h / patch) * (w / patch) * kpad;
  const int g = grid_for(total, 256);
  cudaStream_t st = (cudaStream_t)stream;
  if (x_dtype == SEEDX_F32)
    launch_k(patchify_kernel<float>, g, 256, 0, st, (const float*)x, (int)n, (int)c, (int)h, (int)w, (int)patch, (__half*)out, (int)kpad);
  else if (x_dtype == SEEDX_F16)
    launch_k(patchify_kernel<__half>, g, 256, 0, st, (const __half*)x, (int)n, (int)c, (int)h, (int)w, (int)patch, (__half*)out, (int)kpad);
  else
    SEEDX_REQUIRE(false, "seedx_patchify: bad dtype");
  count_launch();
  return check_cuda(cudaGetLastError(), "patchify launch");
}

extern "C" int seedx_cast(const void* src, int sd, void* dst, int dd, int64_t count, void* stream) {
  SEEDX_REQUIRE(src && dst && count > 0, "seedx_cast: bad arguments");
  const int g = grid_for(count, 256);
  cudaStream_t st = (cudaStream_t)stream;
  if (sd == SEEDX_F32 && dd == SEEDX_F16) launch_k(cast_kernel<float, __half>, g, 256, 0, st, (const float*)src, (__half*)dst, count);
  else if (sd == SEEDX_F16 && dd == SEEDX_F32) launch_k(cast_kernel<__half, float>, g, 256, 0, st, (const __half*)src, (float*)dst, count);
  else SEEDX_REQUIRE(false, "seedx_cast: unsupported conversion %d -> %d", sd, dd);
  count_launch();
  return check_cuda(cudaGetLastError(), "cast launch");
}

extern "C" int seedx_quant_rows_fp8(const void* x, int64_t ldx, int64_t rows, int64_t cols, void* q, int64_t ldq, float* scale, void* stream) {
  SEEDX_REQUIRE(x && q && scale, "seedx_quant_rows_fp8: null pointer");
  SEEDX_REQUIRE(rows > 0 && cols > 0 && cols <= 8192, "seedx_quant_rows_fp8: rows=%lld cols=%lld (1 <= cols <= 8192)", (long long)rows, (long long)cols);
  SEEDX_REQUIRE(ldx >= cols && ldq >= cols && ldx % 8 == 0 && ldq % 16 == 0 && (uintptr_t)x % 16 == 0 && (uintptr_t)q % 16 == 0,
                "seedx_quant_rows_fp8: rows must start 16-byte aligned (ldx %% 8 == 0, ldq %% 16 == 0, aligned pointers) and ldx, ldq >= cols");
  const int per_lane = (int)((cols / 16 + 31) / 32);
  const dim3 grid((unsigned)((rows + 3) / 4));
  cudaStream_t st = (cudaStream_t)stream;
  const __half* xp = (const __half*)x;
  uint8_t* qp = (uint8_t*)q;
  if (per_lane <= 1) launch_k(quant_rows_fp8_kernel<1>, grid, 128, 0, st, xp, (long long)ldx, (long long)rows, (int)cols, qp, (long long)ldq, scale);
  else if (per_lane <= 2) launch_k(quant_rows_fp8_kernel<2>, grid, 128, 0, st, xp, (long long)ldx, (long long)rows, (int)cols, qp, (long long)ldq, scale);
  else if (per_lane <= 4) launch_k(quant_rows_fp8_kernel<4>, grid, 128, 0, st, xp, (long long)ldx, (long long)rows, (int)cols, qp, (long long)ldq, scale);
  else if (per_lane <= 8) launch_k(quant_rows_fp8_kernel<8>, grid, 128, 0, st, xp, (long long)ldx, (long long)rows, (int)cols, qp, (long long)ldq, scale);
  else launch_k(quant_rows_fp8_kernel<16>, grid, 128, 0, st, xp, (long long)ldx, (long long)rows, (int)cols, qp, (long long)ldq, scale);
  count_launch();
  return check_cuda(cudaGetLastError(), "quant_rows_fp8 launch");
}

extern "C" int64_t seedx_quant_images_fp8_ws_bytes(int64_t n, int64_t per_image) {
  if (n <= 0 || per_image <= 0) return 0;
  return n * quant_images_chunks(per_image) * (int64_t)sizeof(float);
}

extern "C" int seedx_quant_images_fp8(const void* x, int64_t n, int64_t per_image, void* q, float* scale, void* ws, void* stream) {
  SEEDX_REQUIRE(x && q && scale && ws, "seedx_quant_images_fp8: null pointer");
  SEEDX_REQUIRE(n > 0 && n <= 65535 && per_image > 0 && per_image % 16 == 0, "seedx_quant_images_fp8: n=%lld per_image=%lld (1 <= n <= 65535, per_image %% 16 == 0)",
                (long long)n, (long long)per_image);
  SEEDX_REQUIRE((uintptr_t)x % 16 == 0 && (uintptr_t)q % 16 == 0 && (uintptr_t)ws % 4 == 0, "seedx_quant_images_fp8: x and q must be 16-byte aligned");
  const dim3 grid((unsigned)quant_images_chunks(per_image), (unsigned)n);
  cudaStream_t st = (cudaStream_t)stream;
  launch_k(quant_images_amax_kernel, grid, QI_THREADS, 0, st, (const __half*)x, (long long)per_image, (float*)ws);
  count_launch();
  if (int e = check_cuda(cudaGetLastError(), "quant_images_amax launch")) return e;
  launch_k(quant_images_fp8_kernel, grid, QI_THREADS, 0, st, (const __half*)x, (long long)per_image, (const float*)ws, (uint8_t*)q, scale);
  count_launch();
  return check_cuda(cudaGetLastError(), "quant_images_fp8 launch");
}

extern "C" int seedx_avgpool_tokens(const void* x, int dtype, int64_t n, int64_t t, int64_t c, int64_t k, void* out, void* stream) {
  SEEDX_REQUIRE(x && out && k > 0 && t % k == 0, "seedx_avgpool_tokens: bad arguments");
  const long long rows = n * (t / k);
  const int g = grid_for(rows * c, 256);
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == SEEDX_F16) launch_k(avgpool_tokens_kernel<__half>, g, 256, 0, st, (const __half*)x, rows, (int)c, (int)k, (__half*)out);
  else if (dtype == SEEDX_F32) launch_k(avgpool_tokens_kernel<float>, g, 256, 0, st, (const float*)x, rows, (int)c, (int)k, (float*)out);
  else SEEDX_REQUIRE(false, "seedx_avgpool_tokens: bad dtype");
  count_launch();
  return check_cuda(cudaGetLastError(), "avgpool launch");
}

extern "C" int seedx_im2col_nhwc(const void* x, int64_t n, int64_t h, int64_t w, int64_t c, int k, int stride, int pad_before, int64_t ho,
                                 int64_t wo, void* out, void* stream) {
  SEEDX_REQUIRE(x && out && c % 8 == 0 && k > 0 && stride > 0, "seedx_im2col_nhwc: bad arguments");
  const long long total = n * ho * wo * k * k * (c / 8);
  launch_k(im2col_nhwc_kernel, grid_for(total, 256), 256, 0, (cudaStream_t)stream, (const __half*)x, (int)n, (int)h, (int)w, (int)c, k, stride,
                                                                            pad_before, (int)ho, (int)wo, (__half*)out);
  count_launch();
  return check_cuda(cudaGetLastError(), "im2col launch");
}

extern "C" int seedx_upsample2x_nhwc(const void* x, int64_t n, int64_t h, int64_t w, int64_t c, void* out, void* stream) {
  SEEDX_REQUIRE(x && out && c % 8 == 0, "seedx_upsample2x_nhwc: bad arguments");
  const long long total = n * 4 * h * w * (c / 8);
  launch_k(upsample2x_nhwc_kernel, grid_for(total, 256), 256, 0, (cudaStream_t)stream, (const __half*)x, (int)n, (int)h, (int)w, (int)c, (__half*)out);
  count_launch();
  return check_cuda(cudaGetLastError(), "upsample launch");
}

extern "C" int seedx_timestep_embedding(const float* t, int64_t count, int dim, void* out, int64_t ldo, void* stream) {
  SEEDX_REQUIRE(t && out && count > 0 && dim > 0 && dim % 2 == 0, "seedx_timestep_embedding: bad arguments");
  launch_k(timestep_embedding_kernel, grid_for(count * dim / 2, 128), 128, 0, (cudaStream_t)stream, t, (int)count, dim, (__half*)out, ldo);
  count_launch();
  return check_cuda(cudaGetLastError(), "timestep_embedding launch");
}

extern "C" int seedx_unary_f16(const void* x, int x_dtype, int64_t rows, int64_t cols, int64_t ldx, void* out, int64_t ldo, int act, void* stream) {
  SEEDX_REQUIRE(x && out && rows > 0 && cols > 0, "seedx_unary_f16: bad arguments");
  const int g = grid_for(rows * cols, 256);
  cudaStream_t st = (cudaStream_t)stream;
  if (x_dtype == SEEDX_F32) launch_k(unary_kernel<float>, g, 256, 0, st, (const float*)x, rows, (int)cols, ldx, (__half*)out, ldo, act);
  else if (x_dtype == SEEDX_F16) launch_k(unary_kernel<__half>, g, 256, 0, st, (const __half*)x, rows, (int)cols, ldx, (__half*)out, ldo, act);
  else SEEDX_REQUIRE(false, "seedx_unary_f16: bad dtype");
  count_launch();
  return check_cuda(cudaGetLastError(), "unary launch");
}

extern "C" int seedx_softmax_rows(const void* x, int x_dtype, int64_t ldx, int64_t rows, int64_t cols, float scale, void* out, int64_t ldo,
                                  void* stream) {
  SEEDX_REQUIRE(x && out && rows > 0 && cols > 0, "seedx_softmax_rows: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  if (x_dtype == SEEDX_F32) launch_k(softmax_rows_kernel<float>, (unsigned)rows, 256, 0, st, (const float*)x, ldx, (int)cols, scale, (__half*)out, ldo);
  else if (x_dtype == SEEDX_F16) launch_k(softmax_rows_kernel<__half>, (unsigned)rows, 256, 0, st, (const __half*)x, ldx, (int)cols, scale, (__half*)out, ldo);
  else SEEDX_REQUIRE(false, "seedx_softmax_rows: bad dtype");
  count_launch();
  return check_cuda(cudaGetLastError(), "softmax launch");
}

extern "C" int seedx_nchw_to_nhwc_f16(const float* x, int64_t n, int64_t c, int64_t hw, int64_t cpad, float scale, void* out, void* stream) {
  SEEDX_REQUIRE(x && out && cpad >= c, "seedx_nchw_to_nhwc_f16: bad arguments");
  launch_k(nchw_to_nhwc_kernel, grid_for(n * hw * cpad, 256), 256, 0, (cudaStream_t)stream, x, (int)n, (int)c, (int)hw, (int)cpad, scale, (__half*)out);
  count_launch();
  return check_cuda(cudaGetLastError(), "nchw_to_nhwc launch");
}

extern "C" int seedx_nhwc_to_nchw_f32(const void* x, int x_dtype, int64_t n, int64_t c, int64_t hw, int64_t ldc, float scale, float* out,
                                      void* stream) {
  SEEDX_REQUIRE(x && out && ldc >= c, "seedx_nhwc_to_nchw_f32: bad arguments");
  const int g = grid_for(n * c * hw, 256);
  cudaStream_t st = (cudaStream_t)stream;
  if (x_dtype == SEEDX_F32) launch_k(nhwc_to_nchw_kernel<float>, g, 256, 0, st, (const float*)x, (int)n, (int)c, (int)hw, (int)ldc, scale, out);
  else if (x_dtype == SEEDX_F16) launch_k(nhwc_to_nchw_kernel<__half>, g, 256, 0, st, (const __half*)x, (int)n, (int)c, (int)hw, (int)ldc, scale, out);
  else SEEDX_REQUIRE(false, "seedx_nhwc_to_nchw_f32: bad dtype");
  count_launch();
  return check_cuda(cudaGetLastError(), "nhwc_to_nchw launch");
}

extern "C" int seedx_image_to_u8(const void* x, int x_dtype, int64_t pixels, int64_t ldc, uint8_t* out, void* stream) {
  SEEDX_REQUIRE(x && out && pixels > 0 && ldc >= 3, "seedx_image_to_u8: bad arguments");
  const int g = grid_for(pixels * 3, 256);
  cudaStream_t st = (cudaStream_t)stream;
  if (x_dtype == SEEDX_F32) launch_k(image_to_u8_kernel<float>, g, 256, 0, st, (const float*)x, pixels, (int)ldc, out);
  else if (x_dtype == SEEDX_F16) launch_k(image_to_u8_kernel<__half>, g, 256, 0, st, (const __half*)x, pixels, (int)ldc, out);
  else SEEDX_REQUIRE(false, "seedx_image_to_u8: bad dtype");
  count_launch();
  return check_cuda(cudaGetLastError(), "image_to_u8 launch");
}

extern "C" int seedx_cfg_euler_step(const float* eps, float* x, void* unet_in, int64_t batch, int64_t hw, int branches, float guidance,
                                    float image_guidance, float sigma, float sigma_next, float init_sigma, void* stream) {
  SEEDX_REQUIRE(x && unet_in && (branches == 2 || branches == 3), "seedx_cfg_euler_step: bad arguments");
  if (eps) SEEDX_REQUIRE(sigma > 0.f, "seedx_cfg_euler_step: sigma must be > 0");
  launch_k(cfg_euler_kernel, grid_for(batch * hw * 4, 256), 256, 0, (cudaStream_t)stream, eps, x, (__half*)unet_in, (int)batch, (int)hw, branches,
                                                                                   guidance, image_guidance, sigma, sigma_next, init_sigma);
  count_launch();
  return check_cuda(cudaGetLastError(), "cfg_euler launch");
}

extern "C" int seedx_cfg_euler_slots(const float* eps, float* x, void* unet_in, float* t_dev, int32_t* state, const float* sigmas,
                                     const float* timesteps, const float* scalars, int64_t slots, int64_t hw, int branches, int64_t max_steps,
                                     uint64_t fresh_mask, void* stream) {
  SEEDX_REQUIRE(branches == 2 || branches == 3, "seedx_cfg_euler_slots: branches must be 2 or 3 (got %d)", branches);
  SEEDX_REQUIRE(x && unet_in && t_dev, "seedx_cfg_euler_slots: null x, unet_in or t_dev");
  SEEDX_REQUIRE(state && sigmas && timesteps && scalars, "seedx_cfg_euler_slots: null slot state or table pointer");
  SEEDX_REQUIRE(max_steps >= 1, "seedx_cfg_euler_slots: max_steps must be >= 1 (got %lld)", (long long)max_steps);
  SEEDX_REQUIRE(slots >= 1 && slots <= 64 && hw >= 1, "seedx_cfg_euler_slots: slots=%lld hw=%lld (1 <= slots <= 64, hw >= 1)", (long long)slots,
                (long long)hw);
  SEEDX_REQUIRE((uintptr_t)unet_in % 16 == 0 && (uintptr_t)state % 8 == 0 && (!eps || (uintptr_t)eps % 16 == 0),
                "seedx_cfg_euler_slots: eps and unet_in must be 16-byte aligned, state 8-byte aligned");
  const uint64_t all = slots == 64 ? ~0ull : ((1ull << slots) - 1);
  if (eps) SEEDX_REQUIRE(fresh_mask == 0, "seedx_cfg_euler_slots: fresh_mask only applies to the initialisation (eps == NULL)");
  else SEEDX_REQUIRE(fresh_mask != 0 && (fresh_mask & ~all) == 0, "seedx_cfg_euler_slots: fresh_mask must name at least one of the %lld slots",
                     (long long)slots);
  cudaStream_t st = (cudaStream_t)stream;
  launch_k(cfg_euler_slots_kernel, grid_for(slots * hw, 256), 256, 0, st, eps, x, (__half*)unet_in, t_dev, (const int*)state, sigmas, timesteps,
           scalars, (int)slots, (int)hw, branches, (int)max_steps, (unsigned long long)fresh_mask);
  count_launch();
  if (int e = check_cuda(cudaGetLastError(), "cfg_euler_slots launch")) return e;
  if (!eps) return 0;
  launch_k(cfg_euler_slots_advance_kernel, 1, 64, 0, st, t_dev, (int*)state, timesteps, (int)slots, branches, (int)max_steps);
  count_launch();
  return check_cuda(cudaGetLastError(), "cfg_euler_slots_advance launch");
}

extern "C" int seedx_add_bcast_f16(const void* a, int a_dtype, const float* b, int64_t rows, int64_t cols, int64_t b_rows, void* out,
                                   void* stream) {
  SEEDX_REQUIRE(a && b && out && rows > 0 && cols > 0 && b_rows > 0, "seedx_add_bcast_f16: bad arguments");
  const int g = grid_for(rows * cols, 256);
  cudaStream_t st = (cudaStream_t)stream;
  if (a_dtype == SEEDX_F16) launch_k(add_bcast_kernel<__half>, g, 256, 0, st, (const __half*)a, b, rows, (int)cols, (int)b_rows, (__half*)out);
  else if (a_dtype == SEEDX_F32) launch_k(add_bcast_kernel<float>, g, 256, 0, st, (const float*)a, b, rows, (int)cols, (int)b_rows, (__half*)out);
  else SEEDX_REQUIRE(false, "seedx_add_bcast_f16: bad dtype");
  count_launch();
  return check_cuda(cudaGetLastError(), "add_bcast launch");
}
