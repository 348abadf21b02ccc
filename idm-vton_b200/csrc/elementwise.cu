// HBM-/latency-bound glue kernels of the denoise step (sm_90a): layout seams, samplers' data movement,
// timestep embeddings, skinny (M <= 16) linears, and the fused CFG + DDPM update.
// Reference call sites are cited per kernel; rounding points follow the fp16-autocast path (SURVEY.md App. D.1).
#include "common.cuh"
#include "host.h"

namespace vton {

// ------------------------------------------------------------------------------------------------
// NCHW <-> NHWC seams. The reference's UNet API is NCHW (src/unet_hacked_tryon.py:1006); the engine is NHWC.
// scatter: dst[s, y, x, c_off + c] = src[s % Bs, c, y, x]   (CFG duplication `torch.cat([latents]*2)`,
//          src/tryon_pipeline.py:1769, and the 13-channel concat, :1777, become channel offsets)
// ------------------------------------------------------------------------------------------------
// scale (device scalar, may be null): dst = fp16(src * scale[0]) instead of a copy. This is the
// `scheduler.scale_model_input` of EulerDiscreteScheduler (src/tryon_pipeline.py:1772): the caller passes the fp32
// reciprocal 1 / sqrt(sigma^2 + 1), because torch divides a CUDA tensor by a CPU scalar as a product with its reciprocal.
// ROWS (the `_rows` entry point): scale holds one fp32 per source sample and dst row s is scaled by scale[s % Bs], so the
// CFG duplicate rows b and b + Bs share sample b's scale (per-slot step indices of the continuous-batching denoiser).
template <bool ROWS>
__global__ void nchw_to_nhwc_kernel(const __half* src, int Bs, int Cs, int HW, __half* dst, int Bd, int ldc, int c_off,
                                    const float* scale) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long total = static_cast<long long>(Bd) * HW;
  if (i >= total) return;
  const int s = static_cast<int>(i / HW);
  const int px = static_cast<int>(i % HW);
  const int sb = s % Bs;
  if (scale) {
    const float f = ROWS ? scale[sb] : *scale;
    for (int c = 0; c < Cs; ++c)
      dst[i * ldc + c_off + c] = f2h(h2f(src[(static_cast<long long>(sb) * Cs + c) * HW + px]) * f);
  } else {
    for (int c = 0; c < Cs; ++c) dst[i * ldc + c_off + c] = src[(static_cast<long long>(sb) * Cs + c) * HW + px];
  }
}

__global__ void nhwc_to_nchw_kernel(const __half* src, int B, int C, int HW, int ldc, __half* dst) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long total = static_cast<long long>(B) * C * HW;
  if (i >= total) return;
  const int px = static_cast<int>(i % HW);
  const int c = static_cast<int>((i / HW) % C);
  const int b = static_cast<int>(i / (static_cast<long long>(HW) * C));
  dst[i] = src[(static_cast<long long>(b) * HW + px) * ldc + c];
}

int nchw_to_nhwc_impl(const void* src, int Bs, int Cs, int H, int W, void* dst, int Bd, int ldc, int c_off,
                      const void* scale, cudaStream_t stream, bool scale_rows) {
  VTON_CHECK_ARG(Bs > 0 && Cs > 0 && H > 0 && W > 0 && Bd > 0 && c_off + Cs <= ldc, "nchw_to_nhwc: bad shape");
  VTON_CHECK_ARG(aligned_to(scale, 4), "nchw_to_nhwc: scale must be 4-byte aligned");
  const long long total = static_cast<long long>(Bd) * H * W;
  auto kern = scale_rows ? nchw_to_nhwc_kernel<true> : nchw_to_nhwc_kernel<false>;
  kern<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(
      static_cast<const __half*>(src), Bs, Cs, H * W, static_cast<__half*>(dst), Bd, ldc, c_off,
      static_cast<const float*>(scale));
  count_launch();
  VTON_CUDA(cudaGetLastError());
  return kOk;
}

int nhwc_to_nchw_impl(const void* src, int B, int C, int H, int W, int ldc, void* dst, cudaStream_t stream) {
  VTON_CHECK_ARG(B > 0 && C > 0 && H > 0 && W > 0 && C <= ldc, "nhwc_to_nchw: bad shape");
  const long long total = static_cast<long long>(B) * C * H * W;
  nhwc_to_nchw_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(
      static_cast<const __half*>(src), B, C, H * W, ldc, static_cast<__half*>(dst));
  count_launch();
  VTON_CUDA(cudaGetLastError());
  return kOk;
}

// ------------------------------------------------------------------------------------------------
// Upsample2D data movement: nearest resize to (Hout, Wout) (diffusers Upsample2D = F.interpolate(nearest) then conv3x3;
// built at src/unet_block_hacked_tryon.py:2301,2443). Scale 2 by default; F.interpolate(size=...) when the UNet forwards
// an `upsample_size` (latent size not a multiple of 4: src/unet_hacked_tryon.py:1081-1091,1357-1379). NHWC, 16-byte
// vectors. Source index per axis = ATen's nearest rule (UpSample.h nearest_idx): identity when out == in, dst >> 1 when
// out == 2 in, else min((int)floorf(dst * scale), in - 1) with scale = (float)in / out.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ int nearest_src(int d, int in, int out, float scale) {
  if (out == in) return d;
  if (out == 2 * in) return d >> 1;
  return min(static_cast<int>(floorf(static_cast<float>(d) * scale)), in - 1);
}

__global__ void upsample_nearest_kernel(const uint4* src, int B, int H, int W, int V, int Hout, int Wout, float sh,
                                        float sw, uint4* dst) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long total = static_cast<long long>(B) * Hout * Wout * V;
  if (i >= total) return;
  const int v = static_cast<int>(i % V);
  long long t = i / V;
  const int x = static_cast<int>(t % Wout);
  t /= Wout;
  const int y = static_cast<int>(t % Hout);
  const int b = static_cast<int>(t / Hout);
  const int sy = nearest_src(y, H, Hout, sh), sx = nearest_src(x, W, Wout, sw);
  dst[i] = src[((static_cast<long long>(b) * H + sy) * W + sx) * V + v];
}

int upsample_nearest_impl(const void* src, int B, int H, int W, int C, int Hout, int Wout, void* dst,
                          cudaStream_t stream) {
  VTON_CHECK_ARG(B > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0 && Hout > 0 && Wout > 0,
                 "upsample_nearest: bad shape");
  VTON_CHECK_ARG(aligned_to(src, 16) && aligned_to(dst, 16), "upsample_nearest: src / dst must be 16-byte aligned");
  const long long total = static_cast<long long>(B) * Hout * Wout * (C / 8);
  // scale exactly as ATen computes it for a given output size (compute_scales_value: (float)in / out)
  const float sh = static_cast<float>(H) / static_cast<float>(Hout), sw = static_cast<float>(W) / static_cast<float>(Wout);
  upsample_nearest_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(
      static_cast<const uint4*>(src), B, H, W, C / 8, Hout, Wout, sh, sw, static_cast<uint4*>(dst));
  count_launch();
  VTON_CUDA(cudaGetLastError());
  return kOk;
}

// ------------------------------------------------------------------------------------------------
// Downsample2D (conv3x3 stride 2 pad 1; src/unet_block_hacked_tryon.py:1113,1246): gather the strided patches into
// A[b*Ho*Wo, 9*C] (tap-major K) and run the plain GEMM against W[Cout, 9*C].
// ------------------------------------------------------------------------------------------------
__global__ void im2col_s2_kernel(const uint4* src, int B, int H, int W, int V, int Ho, int Wo, uint4* dst) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long total = static_cast<long long>(B) * Ho * Wo * 9 * V;
  if (i >= total) return;
  const int v = static_cast<int>(i % V);
  long long t = i / V;
  const int tap = static_cast<int>(t % 9);
  t /= 9;
  const int ox = static_cast<int>(t % Wo);
  t /= Wo;
  const int oy = static_cast<int>(t % Ho);
  const int b = static_cast<int>(t / Ho);
  const int iy = 2 * oy + tap / 3 - 1;
  const int ix = 2 * ox + tap % 3 - 1;
  uint4 val = make_uint4(0, 0, 0, 0);
  if (iy >= 0 && iy < H && ix >= 0 && ix < W) val = src[((static_cast<long long>(b) * H + iy) * W + ix) * V + v];
  dst[i] = val;
}

int im2col_s2_impl(const void* src, int B, int H, int W, int C, void* dst, cudaStream_t stream) {
  VTON_CHECK_ARG(B > 0 && H > 0 && W > 0 && C % 8 == 0, "im2col_s2: bad shape");
  const int Ho = (H + 2 - 3) / 2 + 1, Wo = (W + 2 - 3) / 2 + 1;
  const long long total = static_cast<long long>(B) * Ho * Wo * 9 * (C / 8);
  im2col_s2_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(
      static_cast<const uint4*>(src), B, H, W, C / 8, Ho, Wo, static_cast<uint4*>(dst));
  count_launch();
  VTON_CUDA(cudaGetLastError());
  return kOk;
}

// ------------------------------------------------------------------------------------------------
// Sinusoidal timestep embedding (diffusers Timesteps, flip_sin_to_cos=True, freq_shift=0): out = [cos | sin],
// fp32 math, fp16 store (`t_emb.to(dtype=sample.dtype)`, src/unet_hacked_tryon.py:1134-1139).
// values: [n] floats on device; out: [n, dim]
// ------------------------------------------------------------------------------------------------
__global__ void timestep_embed_kernel(const float* values, int n, int dim, __half* out, int rows_repeat) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int half_dim = dim / 2;
  if (i >= n * rows_repeat * half_dim) return;
  const int k = i % half_dim;
  const int r = i / half_dim;
  const float t = values[r % n];
  const float freq = expf(-logf(10000.0f) * static_cast<float>(k) / static_cast<float>(half_dim));
  const float arg = t * freq;
  out[static_cast<long long>(r) * dim + k] = f2h(cosf(arg));
  out[static_cast<long long>(r) * dim + half_dim + k] = f2h(sinf(arg));
}

int timestep_embed_impl(const void* values, int n, int dim, int rows_repeat, void* out, cudaStream_t stream) {
  VTON_CHECK_ARG(n > 0 && dim > 0 && dim % 2 == 0 && rows_repeat > 0, "timestep_embed: bad shape");
  const int total = n * rows_repeat * (dim / 2);
  timestep_embed_kernel<<<(total + 127) / 128, 128, 0, stream>>>(static_cast<const float*>(values), n, dim,
                                                                  static_cast<__half*>(out), rows_repeat);
  count_launch();
  VTON_CUDA(cudaGetLastError());
  return kOk;
}

// ------------------------------------------------------------------------------------------------
// Skinny linear for the embedding MLPs (M <= 16 rows): TimestepEmbedding linear_1/linear_2, add_embedding, and all
// per-resnet time_emb_proj batched into one call (SURVEY.md K12). One warp per output column; weights are read once.
//   x' = in_silu ? fp16(silu(x)) : x ; y = fp16(W x' + b) ; y = out_silu ? fp16(silu(y)) : y ; y = addend ? fp16(y + addend) : y
// ------------------------------------------------------------------------------------------------
constexpr int SK_MAXM = 16;

__global__ void __launch_bounds__(256)
skinny_linear_kernel(const __half* x, int ldx, int M, int K, const __half* W, long long ldw, int N, const __half* bias,
                     int in_silu, int out_silu, const __half* addend, int ld_add, __half* out, int ldo) {
  extern __shared__ __half xs[];  // [M][K] activated input
  for (int i = threadIdx.x; i < M * K; i += blockDim.x) {
    const int m = i / K, k = i % K;
    __half v = x[static_cast<long long>(m) * ldx + k];
    if (in_silu) v = f2h(silu_f(h2f(v)));
    xs[i] = v;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n = blockIdx.x * 8 + warp;
  if (n >= N) return;
  float acc[SK_MAXM];
#pragma unroll
  for (int m = 0; m < SK_MAXM; ++m) acc[m] = 0.f;
  const __half* wrow = W + static_cast<long long>(n) * ldw;
  for (int k = lane * 8; k < K; k += 256) {
    const uint4 wu = *reinterpret_cast<const uint4*>(wrow + k);
    const uint32_t ww[4] = {wu.x, wu.y, wu.z, wu.w};
    float wf[8];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = unpack_h2(ww[j]);
      wf[2 * j] = f.x;
      wf[2 * j + 1] = f.y;
    }
#pragma unroll
    for (int m = 0; m < SK_MAXM; ++m) {
      if (m < M) {
        const uint4 xu = *reinterpret_cast<const uint4*>(xs + m * K + k);
        const uint32_t xw[4] = {xu.x, xu.y, xu.z, xu.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 f = unpack_h2(xw[j]);
          acc[m] += f.x * wf[2 * j] + f.y * wf[2 * j + 1];
        }
      }
    }
  }
#pragma unroll
  for (int m = 0; m < SK_MAXM; ++m) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc[m] += __shfl_xor_sync(0xffffffffu, acc[m], o);
  }
  if (lane == 0) {
    const float b = bias ? h2f(bias[n]) : 0.f;
    for (int m = 0; m < M; ++m) {
      float y = round_h(acc[m] + b);
      if (out_silu) y = round_h(silu_f(y));
      if (addend) y = round_h(y + h2f(addend[static_cast<long long>(m) * ld_add + n]));
      out[static_cast<long long>(m) * ldo + n] = f2h(y);
    }
  }
}

int skinny_linear_impl(const void* x, int ldx, int M, int K, const void* W, long long ldw, int N, const void* bias,
                       int in_silu, int out_silu, const void* addend, int ld_add, void* out, int ldo,
                       cudaStream_t stream) {
  VTON_CHECK_ARG(M > 0 && M <= SK_MAXM, "skinny_linear: M=%d out of range (1..%d)", M, SK_MAXM);
  VTON_CHECK_ARG(K % 8 == 0 && ldw % 8 == 0 && N > 0, "skinny_linear: K/ldw must be multiples of 8");
  const size_t smem = static_cast<size_t>(M) * K * sizeof(__half);
  VTON_CHECK_ARG(smem <= 96 * 1024, "skinny_linear: M*K too large");
  static bool configured = false;
  if (!configured) {
    VTON_CUDA(cudaFuncSetAttribute(skinny_linear_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
    configured = true;
  }
  skinny_linear_kernel<<<cdiv(N, 8), 256, smem, stream>>>(
      static_cast<const __half*>(x), ldx, M, K, static_cast<const __half*>(W), ldw, N, static_cast<const __half*>(bias),
      in_silu, out_silu, static_cast<const __half*>(addend), ld_add, static_cast<__half*>(out), ldo);
  count_launch();
  VTON_CUDA(cudaGetLastError());
  return kOk;
}

// ------------------------------------------------------------------------------------------------
// Fused classifier-free guidance + DDPM ancestral step (src/tryon_pipeline.py:1814-1823; diffusers DDPMScheduler.step,
// epsilon prediction, fixed_small variance). Every op rounds to fp16 like the reference's fp16 tensor arithmetic:
//   g = u + fp16(gs * fp16(c - u));  x0 = fp16(fp16(x - fp16(sb * g)) * inv_sa);
//   prev = fp16(fp16(c0 * x0) + fp16(c1 * x));  out = prev + fp16(sigma * noise)   (noise == null at t == 0)
// eps: NHWC [2B, HW, ldc] (uncond rows first, then cond); latents/noise/out: NCHW [B, 4, HW]. Coefficients live on the
// device ([6] floats: gs, sb, inv_sa, c0, c1, sigma) so a captured CUDA graph can be replayed for every step.
// ROWS (b200vton_cfg_ddpm_step_rows): coef is [B, coef_stride] and sample b reads row b, so every sample of the batch
// can be at its own denoise step (continuous batching); coef_stride 0 is the single-row kernel.
// ------------------------------------------------------------------------------------------------
// The per-value pieces of the step kernels below, shared so that every kernel rounds at the same points.
__device__ __forceinline__ float cfg_guided(float u, float t, float gs) { return round_h(u + round_h(gs * round_h(t - u))); }

// DDPM update without its noise term: x0 = fp16(fp16(x - fp16(sb * g)) * inv_sa); prev = fp16(fp16(c0 x0) + fp16(c1 x)).
__device__ __forceinline__ float ddpm_update(float x, float g, float sb, float inv_sa, float c0, float c1) {
  const float x0 = round_h(round_h(x - round_h(sb * g)) * inv_sa);
  return round_h(round_h(c0 * x0) + round_h(c1 * x));
}

template <bool ROWS>
__global__ void cfg_ddpm_kernel(const __half* eps, int ldc, int B, int C, int HW, const __half* latents,
                                const __half* noise, const float* coef, int coef_stride, int do_cfg, __half* out) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long total = static_cast<long long>(B) * C * HW;
  if (i >= total) return;
  const int px = static_cast<int>(i % HW);
  const int c = static_cast<int>((i / HW) % C);
  const int b = static_cast<int>(i / (static_cast<long long>(HW) * C));
  if (ROWS) coef += static_cast<long long>(b) * coef_stride;
  const float gs = coef[0], sb = coef[1], inv_sa = coef[2], c0 = coef[3], c1 = coef[4], sigma = coef[5];
  float g;
  if (do_cfg) {
    const float u = h2f(eps[(static_cast<long long>(b) * HW + px) * ldc + c]);
    const float t = h2f(eps[(static_cast<long long>(b + B) * HW + px) * ldc + c]);
    g = cfg_guided(u, t, gs);
  } else {
    g = h2f(eps[(static_cast<long long>(b) * HW + px) * ldc + c]);
  }
  const float x = h2f(latents[i]);
  float prev = ddpm_update(x, g, sb, inv_sa, c0, c1);
  if (noise) prev = round_h(prev + round_h(sigma * h2f(noise[i])));
  out[i] = f2h(prev);
}

template <bool ROWS>
static int launch_cfg_ddpm(const void* eps, int ldc, int B, int C, int H, int W, const void* latents, const void* noise,
                           const void* coef, int coef_stride, int do_cfg, void* out, cudaStream_t stream) {
  const long long total = static_cast<long long>(B) * C * H * W;
  cfg_ddpm_kernel<ROWS><<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(
      static_cast<const __half*>(eps), ldc, B, C, H * W, static_cast<const __half*>(latents),
      static_cast<const __half*>(noise), static_cast<const float*>(coef), coef_stride, do_cfg,
      static_cast<__half*>(out));
  count_launch();
  VTON_CUDA(cudaGetLastError());
  return kOk;
}

int cfg_ddpm_impl(const void* eps, int ldc, int B, int C, int H, int W, const void* latents, const void* noise,
                  const void* coef, int do_cfg, void* out, cudaStream_t stream) {
  VTON_CHECK_ARG(B > 0 && C > 0 && C <= ldc && H > 0 && W > 0 && coef, "cfg_ddpm: bad arguments");
  return launch_cfg_ddpm<false>(eps, ldc, B, C, H, W, latents, noise, coef, 0, do_cfg, out, stream);
}

constexpr int kDdpmCoefs = 6;      // {gs, sb, inv_sa, c0, c1, sigma}
constexpr int kSolverCoefs = 8;    // {gs, s, inv_a, p, q, r, sigma_n, k}

int cfg_ddpm_rows_impl(const void* eps, int ldc, int B, int C, int H, int W, const void* latents, const void* noise,
                       const void* coef, int coef_stride, int do_cfg, void* out, cudaStream_t stream) {
  VTON_CHECK_ARG(B > 0 && C > 0 && C <= ldc && H > 0 && W > 0 && coef && eps && latents && out,
                 "cfg_ddpm_rows: bad arguments");
  VTON_CHECK_ARG(coef_stride == 0 || coef_stride >= kDdpmCoefs,
                 "cfg_ddpm_rows: coef_stride %d is neither 0 nor >= %d", coef_stride, kDdpmCoefs);
  VTON_CHECK_ARG(aligned_to(eps, 2) && aligned_to(latents, 2) && aligned_to(noise, 2) && aligned_to(out, 2) &&
                     aligned_to(coef, 4),
                 "cfg_ddpm_rows: fp16 operands must be 2-byte aligned and coef 4-byte aligned");
  return launch_cfg_ddpm<true>(eps, ldc, B, C, H, W, latents, noise, coef, coef_stride, do_cfg, out, stream);
}

// ------------------------------------------------------------------------------------------------
// CFG + guidance rescale + DDPM step (src/tryon_pipeline.py:101-113 rescale_noise_cfg, applied at :1818-1820; the
// "Common Diffusion Noise Schedules and Sample Steps are Flawed" correction). One CTA per sample b:
//   g   = u + fp16(gs * fp16(t - u))                                  (the CFG result of cfg_ddpm_kernel)
//   s_t = fp16(std(t)), s_g = fp16(std(g))   unbiased (torch.std's default), over the C*H*W values of sample b
//   r   = fp16(s_t / s_g)
//   g'  = fp16(fp16(phi * fp16(g * r)) + fp16((1 - phi) * g))
// then cfg_ddpm_kernel's DDPM update on g'. These are the rounding points of the reference's fp16 tensor arithmetic on the
// fp16 noise_pred inside torch.autocast(float16): std of an fp16 tensor returns fp16 there (statistics accumulated in
// fp32 by torch, the result rounded). The statistics here are two-pass (mean, then squared deviations) in double, each
// thread over a fixed strided subset and a fixed-shape tree across the CTA: the result does not depend on timing, and
// there are no atomics. coef: 7 floats {gs, sb, inv_sa, c0, c1, sigma, phi} on the device (graph-replayable).
// ------------------------------------------------------------------------------------------------
constexpr int kRescaleThreads = 1024;

// Sum of v over the CTA in a fixed order; every thread gets the result. red: kRescaleThreads / 32 doubles of shared.
__device__ __forceinline__ double cta_sum(double v, double* red) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();                     // red may still be read by the previous call
  if (lane == 0) red[warp] = v;
  __syncthreads();
  v = lane < (kRescaleThreads >> 5) ? red[lane] : 0.0;
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// The rescaled step of sample b by one CTA of kRescaleThreads threads (cfg_rescale_ddpm_kernel; the DDPM rows with
// phi > 0 of cfg_mixed_kernel). coef: the sample's row.
__device__ __forceinline__ void rescale_ddpm_sample(const __half* eps, int ldc, int B, int C, int HW, int b,
                                                    const __half* latents, const __half* noise, const float* coef,
                                                    __half* out, double* red) {
  const float gs = coef[0], sb = coef[1], inv_sa = coef[2], c0 = coef[3], c1 = coef[4], sigma = coef[5], phi = coef[6];
  const __half* eu = eps + static_cast<long long>(b) * HW * ldc;         // uncond rows of sample b
  const __half* et = eps + static_cast<long long>(b + B) * HW * ldc;     // cond rows of sample b
  const int n = C * HW;
  // the CFG result, from the same fp16 values the apply pass reads
  auto cfg = [&](long long off, float& t) {
    const float u = h2f(eu[off]);
    t = h2f(et[off]);
    return cfg_guided(u, t, gs);
  };
  // pass 1: means (NHWC order: consecutive threads read consecutive channels / pixels)
  double st = 0.0, sg = 0.0;
  for (int k = threadIdx.x; k < n; k += kRescaleThreads) {
    const long long off = static_cast<long long>(k / C) * ldc + k % C;
    float t;
    const float g = cfg(off, t);
    st += t;
    sg += g;
  }
  const double mt = cta_sum(st, red) / n;
  const double mg = cta_sum(sg, red) / n;
  // pass 2: sums of squared deviations
  double qt = 0.0, qg = 0.0;
  for (int k = threadIdx.x; k < n; k += kRescaleThreads) {
    const long long off = static_cast<long long>(k / C) * ldc + k % C;
    float t;
    const float g = cfg(off, t);
    qt += (t - mt) * (t - mt);
    qg += (g - mg) * (g - mg);
  }
  qt = cta_sum(qt, red);
  qg = cta_sum(qg, red);
  // n == 1 gives 0/0 = NaN like torch.std of one value
  const float s_t = round_h(static_cast<float>(sqrt(qt / (n - 1))));
  const float s_g = round_h(static_cast<float>(sqrt(qg / (n - 1))));
  const float r = round_h(s_t / s_g);
  // pass 3: rescale + DDPM update, NCHW order over the latents / noise / out
  const long long base = static_cast<long long>(b) * n;
  for (int k = threadIdx.x; k < n; k += kRescaleThreads) {
    const int c = k / HW, px = k % HW;
    float t;
    const float g = cfg(static_cast<long long>(px) * ldc + c, t);
    const float gr = round_h(round_h(phi * round_h(g * r)) + round_h((1.0f - phi) * g));
    const float x = h2f(latents[base + k]);
    float prev = ddpm_update(x, gr, sb, inv_sa, c0, c1);
    if (noise) prev = round_h(prev + round_h(sigma * h2f(noise[base + k])));
    out[base + k] = f2h(prev);
  }
}

__global__ void __launch_bounds__(kRescaleThreads) cfg_rescale_ddpm_kernel(
    const __half* eps, int ldc, int B, int C, int HW, const __half* latents, const __half* noise, const float* coef,
    __half* out) {
  __shared__ double red[kRescaleThreads / 32];
  rescale_ddpm_sample(eps, ldc, B, C, HW, blockIdx.x, latents, noise, coef, out, red);
}

int cfg_rescale_ddpm_impl(const void* eps, int ldc, int B, int C, int H, int W, const void* latents, const void* noise,
                          const void* coef, int do_cfg, void* out, cudaStream_t stream) {
  // without CFG there is no rescale (the reference applies it only under CFG): the plain step, phi unused
  if (!do_cfg) return cfg_ddpm_impl(eps, ldc, B, C, H, W, latents, noise, coef, 0, out, stream);
  VTON_CHECK_ARG(B > 0 && C > 0 && C <= ldc && H > 0 && W > 0 && coef, "cfg_rescale_ddpm: bad arguments");
  VTON_CHECK_ARG(static_cast<long long>(C) * H * W < (1LL << 31), "cfg_rescale_ddpm: sample too large");
  cfg_rescale_ddpm_kernel<<<B, kRescaleThreads, 0, stream>>>(
      static_cast<const __half*>(eps), ldc, B, C, H * W, static_cast<const __half*>(latents),
      static_cast<const __half*>(noise), static_cast<const float*>(coef), static_cast<__half*>(out));
  count_launch();
  VTON_CUDA(cudaGetLastError());
  return kOk;
}

// ------------------------------------------------------------------------------------------------
// Fused CFG + one step of DDIM, Euler or DPM-Solver++ (src/tryon_pipeline.py:1814-1823 with a DDIMScheduler,
// EulerDiscreteScheduler or DPMSolverMultistepScheduler, epsilon prediction). Same layout as cfg_ddpm_kernel, plus
// x0_prev: the previous step's data prediction [B,C,H,W] fp16 (DPM-Solver++ only; read, then overwritten with this
// step's). coef: 8 fp32 on the device {gs, s, inv_a, p, q, r, sigma_n, k}. In exact arithmetic every kind is
//   g = CFG(eps);  x0 = (x - s g) / a;  D = (1 + k/2) x0 - (k/2) x0_prev;  out = p x + q D + r g + sigma_n noise
// and the kinds differ in their rounding points, which are those of the scheduler's own `step` on fp16 tensors
// (g = u + fp16(gs * fp16(t - u)) under CFG for all three; a CPU-scalar divisor is a product with its fp32 reciprocal):
//   DDIM   (kind 0, fp16 tensor arithmetic; p and k unused):
//          x0 = fp16(fp16(x - fp16(s g)) * inv_a);  out = fp16(fp16(q x0) + fp16(r g));
//          out = fp16(out + fp16(sigma_n noise))                      (eta > 0 only)
//   Euler  (kind 1, sample upcast to fp32; s = sigma, inv_a = 1 / sigma, r = sigma_next - sigma; p, q, k unused):
//          x0 = x - fp16(s g);  d = (x - x0) * inv_a;  out = fp16(x + d r)           (fp32 ops, no FMA contraction)
//   DPM++  (kind 2, data prediction in fp16, update with the sample in fp32; s = sigma_t, inv_a = 1 / alpha_t of the
//          solver at this step, p = sigma_next / sigma_t, q = alpha_next (1 - e^-h), k = 1 / r0 at second order and 0
//          at first order; r unused):
//          x0 = fp16(fp16(x - fp16(s g)) * inv_a);
//          out = fp16((p x + fp16(q x0)) + fp16(fp32(q / 2) * fp16(k * fp16(x0 - x0_prev))));  x0_prev = x0
// sigma_n * noise is added the same way by every kind when noise is not null (only DDIM with eta > 0 draws it).
// ------------------------------------------------------------------------------------------------
// The update of one value of kind KIND without its noise term; x0_prev: this value's DPM-Solver++ state (KIND 2 only).
template <int KIND>
__device__ __forceinline__ float solver_update(float x, float g, float s, float inv_a, float p, float q, float r, float k,
                                               __half* x0_prev) {
  if constexpr (KIND == 0) {
    const float x0 = round_h(round_h(x - round_h(s * g)) * inv_a);
    return round_h(round_h(q * x0) + round_h(r * g));
  } else if constexpr (KIND == 1) {
    const float x0 = __fsub_rn(x, round_h(s * g));
    const float d = __fmul_rn(__fsub_rn(x, x0), inv_a);
    return round_h(__fadd_rn(x, __fmul_rn(d, r)));
  } else {
    const float x0 = round_h(round_h(x - round_h(s * g)) * inv_a);
    const float d1 = round_h(k * round_h(x0 - h2f(*x0_prev)));
    const float prev = round_h(__fadd_rn(__fadd_rn(__fmul_rn(p, x), round_h(q * x0)), round_h(0.5f * q * d1)));
    *x0_prev = f2h(x0);
    return prev;
  }
}

// ROWS (b200vton_cfg_solver_step_rows): coef is [B, coef_stride], sample b reads row b (coef_stride 0: one row for all).
template <int KIND, bool ROWS>
__global__ void cfg_solver_kernel(const __half* eps, int ldc, int B, int C, int HW, const __half* latents,
                                  const __half* noise, __half* x0_prev, const float* coef, int coef_stride, int do_cfg,
                                  __half* out) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long total = static_cast<long long>(B) * C * HW;
  if (i >= total) return;
  const int px = static_cast<int>(i % HW);
  const int c = static_cast<int>((i / HW) % C);
  const int b = static_cast<int>(i / (static_cast<long long>(HW) * C));
  if (ROWS) coef += static_cast<long long>(b) * coef_stride;
  const float gs = coef[0], s = coef[1], inv_a = coef[2], p = coef[3], q = coef[4], r = coef[5], sigma_n = coef[6],
              k = coef[7];
  float g;
  if (do_cfg) {
    const float u = h2f(eps[(static_cast<long long>(b) * HW + px) * ldc + c]);
    const float t = h2f(eps[(static_cast<long long>(b + B) * HW + px) * ldc + c]);
    g = cfg_guided(u, t, gs);
  } else {
    g = h2f(eps[(static_cast<long long>(b) * HW + px) * ldc + c]);
  }
  const float x = h2f(latents[i]);
  float prev = solver_update<KIND>(x, g, s, inv_a, p, q, r, k, KIND == 2 ? x0_prev + i : nullptr);
  if (noise) prev = round_h(prev + round_h(sigma_n * h2f(noise[i])));
  out[i] = f2h(prev);
}

template <bool ROWS>
static int launch_cfg_solver(const void* eps, int ldc, int B, int C, int H, int W, const void* latents,
                             const void* noise, void* x0_prev, const void* coef, int coef_stride, int kind, int do_cfg,
                             void* out, cudaStream_t stream) {
  VTON_CHECK_ARG(B > 0 && C > 0 && C <= ldc && H > 0 && W > 0 && coef && eps && latents && out,
                 "cfg_solver: bad arguments");
  VTON_CHECK_ARG(kind >= 0 && kind <= 2, "cfg_solver: kind %d is not 0 (DDIM), 1 (Euler) or 2 (DPM-Solver++)", kind);
  VTON_CHECK_ARG(kind != 2 || x0_prev, "cfg_solver: DPM-Solver++ needs the x0_prev state buffer");
  VTON_CHECK_ARG(coef_stride == 0 || coef_stride >= kSolverCoefs,
                 "cfg_solver: coef_stride %d is neither 0 nor >= %d", coef_stride, kSolverCoefs);
  VTON_CHECK_ARG(aligned_to(eps, 2) && aligned_to(latents, 2) && aligned_to(noise, 2) && aligned_to(x0_prev, 2) &&
                     aligned_to(out, 2) && aligned_to(coef, 4),
                 "cfg_solver: fp16 operands must be 2-byte aligned and coef 4-byte aligned");
  const long long total = static_cast<long long>(B) * C * H * W;
  const unsigned grid = static_cast<unsigned>((total + 255) / 256);
  auto e = static_cast<const __half*>(eps);
  auto l = static_cast<const __half*>(latents);
  auto n = static_cast<const __half*>(noise);
  auto x0p = static_cast<__half*>(x0_prev);
  auto cf = static_cast<const float*>(coef);
  auto o = static_cast<__half*>(out);
  if (kind == 0)
    cfg_solver_kernel<0, ROWS><<<grid, 256, 0, stream>>>(e, ldc, B, C, H * W, l, n, nullptr, cf, coef_stride, do_cfg, o);
  else if (kind == 1)
    cfg_solver_kernel<1, ROWS><<<grid, 256, 0, stream>>>(e, ldc, B, C, H * W, l, n, nullptr, cf, coef_stride, do_cfg, o);
  else
    cfg_solver_kernel<2, ROWS><<<grid, 256, 0, stream>>>(e, ldc, B, C, H * W, l, n, x0p, cf, coef_stride, do_cfg, o);
  count_launch();
  VTON_CUDA(cudaGetLastError());
  return kOk;
}

int cfg_solver_impl(const void* eps, int ldc, int B, int C, int H, int W, const void* latents, const void* noise,
                    void* x0_prev, const void* coef, int kind, int do_cfg, void* out, cudaStream_t stream) {
  return launch_cfg_solver<false>(eps, ldc, B, C, H, W, latents, noise, x0_prev, coef, 0, kind, do_cfg, out, stream);
}

int cfg_solver_rows_impl(const void* eps, int ldc, int B, int C, int H, int W, const void* latents, const void* noise,
                         void* x0_prev, const void* coef, int coef_stride, int kind, int do_cfg, void* out,
                         cudaStream_t stream) {
  return launch_cfg_solver<true>(eps, ldc, B, C, H, W, latents, noise, x0_prev, coef, coef_stride, kind, do_cfg, out,
                                 stream);
}

// ------------------------------------------------------------------------------------------------
// Mixed-kind step (b200vton_cfg_step_mixed_rows): sample b takes the update of kinds[b] with coefficient row b, so one
// launch steps a batch whose samples follow different schedulers (the sampling presets of continuous batching).
//   0 DDIM, 1 Euler, 2 DPM-Solver++: cfg_solver_kernel<kind, true>, row {gs, s, inv_a, p, q, r, sigma_n, k};
//   3 DDPM: cfg_ddpm_kernel<true>, row {gs, sb, inv_sa, c0, c1, sigma, phi, 0}; under CFG with phi > 0 the guidance
//     rescale of cfg_rescale_ddpm_kernel, by the same CTA-wide reduction (so the same bits as that kernel on the sample).
// noise is added on DDPM and DDIM rows only (Euler draws a noise it does not apply; DPM-Solver++ draws none); x0_prev is
// read and written by DPM-Solver++ rows only. Grid (B, G): CTA (b, y) takes the values y * 1024 + k * G * 1024 of
// sample b in NCHW order; a rescaled sample needs its whole CTA for the statistics, so it runs on y = 0 alone. Every
// value is computed from its own inputs only, so the bits do not depend on G.
// ------------------------------------------------------------------------------------------------
constexpr int kMixedKindDdpm = 3;

__global__ void __launch_bounds__(kRescaleThreads)
cfg_mixed_kernel(const __half* eps, int ldc, int B, int C, int HW, const __half* latents, const __half* noise,
                 __half* x0_prev, const float* coef, int coef_stride, const int* kinds, int do_cfg, __half* out) {
  __shared__ double red[kRescaleThreads / 32];
  pdl_wait();
  pdl_launch_dependents();
  const int b = blockIdx.x;
  const int kind = kinds[b];
  coef += static_cast<long long>(b) * coef_stride;
  if (kind == kMixedKindDdpm && do_cfg && coef[6] > 0.f) {
    if (blockIdx.y == 0) rescale_ddpm_sample(eps, ldc, B, C, HW, b, latents, noise, coef, out, red);
    return;
  }
  const float gs = coef[0], c1 = coef[1], c2 = coef[2], c3 = coef[3], c4 = coef[4], c5 = coef[5], c6 = coef[6],
              c7 = coef[7];
  const __half* eu = eps + static_cast<long long>(b) * HW * ldc;
  const __half* et = eps + static_cast<long long>(b + B) * HW * ldc;
  const int n = C * HW;
  const long long base = static_cast<long long>(b) * n;
  const bool noisy = noise && (kind == 0 || kind == kMixedKindDdpm);
  const float sigma = kind == 0 ? c6 : c5;
  for (int k = blockIdx.y * kRescaleThreads + threadIdx.x; k < n; k += gridDim.y * kRescaleThreads) {
    const long long off = static_cast<long long>(k % HW) * ldc + k / HW;
    const float g = do_cfg ? cfg_guided(h2f(eu[off]), h2f(et[off]), gs) : h2f(eu[off]);
    const float x = h2f(latents[base + k]);
    float prev;
    if (kind == 0) prev = solver_update<0>(x, g, c1, c2, c3, c4, c5, c7, nullptr);
    else if (kind == 1) prev = solver_update<1>(x, g, c1, c2, c3, c4, c5, c7, nullptr);
    else if (kind == 2) prev = solver_update<2>(x, g, c1, c2, c3, c4, c5, c7, x0_prev + base + k);
    else prev = ddpm_update(x, g, c1, c2, c3, c4);
    if (noisy) prev = round_h(prev + round_h(sigma * h2f(noise[base + k])));
    out[base + k] = f2h(prev);
  }
}

int cfg_mixed_rows_impl(const void* eps, int ldc, int B, int C, int H, int W, const void* latents, const void* noise,
                        void* x0_prev, const void* coef, int coef_stride, const void* kinds, int do_cfg, void* out,
                        cudaStream_t stream) {
  VTON_CHECK_ARG(B > 0 && C > 0 && C <= ldc && H > 0 && W > 0 && eps && latents && x0_prev && coef && kinds && out,
                 "cfg_step_mixed_rows: bad arguments (eps, latents, x0_prev, coef, kinds and out are required)");
  VTON_CHECK_ARG(coef_stride == 0 || coef_stride >= kSolverCoefs,
                 "cfg_step_mixed_rows: coef_stride %d is neither 0 nor >= %d", coef_stride, kSolverCoefs);
  VTON_CHECK_ARG(static_cast<long long>(C) * H * W < (1LL << 31), "cfg_step_mixed_rows: sample too large");
  VTON_CHECK_ARG(aligned_to(eps, 2) && aligned_to(latents, 2) && aligned_to(noise, 2) && aligned_to(x0_prev, 2) &&
                     aligned_to(out, 2) && aligned_to(coef, 4) && aligned_to(kinds, 4),
                 "cfg_step_mixed_rows: fp16 operands must be 2-byte aligned, coef and kinds 4-byte aligned");
  // enough CTAs to cover the SMs twice (two 1024-thread CTAs fit one SM), at most one per 1024 values of a sample
  const int n = C * H * W;
  const int G = std::max(1, std::min(cdiv(n, kRescaleThreads), cdiv(2 * num_sms(), B)));
  VTON_CUDA(launch_kernel(cfg_mixed_kernel, dim3(B, G), dim3(kRescaleThreads), 0, stream,
                          static_cast<const __half*>(eps), ldc, B, C, H * W, static_cast<const __half*>(latents),
                          static_cast<const __half*>(noise), static_cast<__half*>(x0_prev),
                          static_cast<const float*>(coef), coef_stride, static_cast<const int*>(kinds), do_cfg,
                          static_cast<__half*>(out)));
  count_launch();
  return kOk;
}

// ------------------------------------------------------------------------------------------------
// Pre / post-processing around the VAE (SURVEY.md 8f item 3; diffusers VaeImageProcessor as the pipeline uses it,
// src/tryon_pipeline.py:418-421, 1588-1602, 940-955, 1885). One launch each instead of ~10 small ATen kernels.
//   preprocess: image [B,3,H,W] fp32 -> init_image = 2x-1 (skipped when the batch already has negative values: diffusers
//               checks `image.min() < 0`; the minimum arrives as a device scalar, so there is no host sync);
//               mask [B,Cm,H,W] (Cm = 1 | 3: grayscale 0.299/0.587/0.114) -> binarised at 0.5;
//               masked_image = init_image * (mask < 0.5);  mask_latent = nearest resize to [B,1,H/s,W/s]
//               (F.interpolate default: source index = floor(dst * s)).
//   postprocess: decoder output [B,3,H,W] fp32 (NCHW, or NHWC memory with `nhwc` set) -> (x/2 + 0.5).clamp(0,1) as
//               fp32 NCHW ("pt") and/or uint8 NHWC (round(x*255): what "np" -> "pil" produces).
// ------------------------------------------------------------------------------------------------
__global__ void preprocess_kernel(const float* image, const float* mask_in, int Cm, const float* img_min, int B, int H,
                                  int W, int s, float* init_image, float* mask_bin, float* masked_image,
                                  __half* mask_latent) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long HW = static_cast<long long>(H) * W;
  if (i >= B * HW) return;
  const int b = static_cast<int>(i / HW);
  const long long px = i % HW;
  const bool normalize = !(*img_min < 0.f);
  float m;
  if (Cm == 3) {
    const float* mp = mask_in + static_cast<long long>(b) * 3 * HW + px;
    // separately rounded products and sums, like the three ATen kernels of the torch expression (no FMA contraction)
    m = __fadd_rn(__fadd_rn(__fmul_rn(0.299f, mp[0]), __fmul_rn(0.587f, mp[HW])), __fmul_rn(0.114f, mp[2 * HW]));
  } else {
    m = mask_in[static_cast<long long>(b) * HW + px];
  }
  const float mb = m >= 0.5f ? 1.f : 0.f;
  mask_bin[i] = mb;
  const float keep = mb < 0.5f ? 1.f : 0.f;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const long long o = (static_cast<long long>(b) * 3 + c) * HW + px;
    float v = image[o];
    if (normalize) v = 2.0f * v - 1.0f;
    init_image[o] = v;
    masked_image[o] = v * keep;
  }
  const int y = static_cast<int>(px / W), x = static_cast<int>(px % W);
  if (y % s == 0 && x % s == 0 && y / s < H / s && x / s < W / s)
    mask_latent[(static_cast<long long>(b) * (H / s) + y / s) * (W / s) + x / s] = f2h(mb);
}

int preprocess_impl(const void* image, const void* mask, int Cm, const void* img_min, int B, int H, int W, int scale,
                    void* init_image, void* mask_bin, void* masked_image, void* mask_latent, cudaStream_t stream) {
  VTON_CHECK_ARG(B > 0 && H > 0 && W > 0 && (Cm == 1 || Cm == 3) && scale > 0 && H % scale == 0 && W % scale == 0,
                 "preprocess: bad shape B=%d H=%d W=%d Cm=%d scale=%d", B, H, W, Cm, scale);
  VTON_CHECK_ARG(image && mask && img_min && init_image && mask_bin && masked_image && mask_latent, "preprocess: null pointer");
  const long long total = static_cast<long long>(B) * H * W;
  preprocess_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(
      static_cast<const float*>(image), static_cast<const float*>(mask), Cm, static_cast<const float*>(img_min), B, H, W,
      scale, static_cast<float*>(init_image), static_cast<float*>(mask_bin), static_cast<float*>(masked_image),
      static_cast<__half*>(mask_latent));
  count_launch();
  VTON_CUDA(cudaGetLastError());
  return kOk;
}

__global__ void postprocess_kernel(const float* x, int nhwc, int B, int H, int W, float* out_pt, uint8_t* out_u8) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long HW = static_cast<long long>(H) * W;
  if (i >= B * HW) return;
  const int b = static_cast<int>(i / HW);
  const long long px = i % HW;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float v = nhwc ? x[i * 3 + c] : x[(static_cast<long long>(b) * 3 + c) * HW + px];
    const float y = fminf(fmaxf(v / 2.f + 0.5f, 0.f), 1.f);
    if (out_pt) out_pt[(static_cast<long long>(b) * 3 + c) * HW + px] = y;
    if (out_u8) out_u8[i * 3 + c] = static_cast<uint8_t>(rintf(y * 255.f));
  }
}

int postprocess_impl(const void* x, int nhwc, int B, int H, int W, void* out_pt, void* out_u8, cudaStream_t stream) {
  VTON_CHECK_ARG(B > 0 && H > 0 && W > 0 && x && (out_pt || out_u8), "postprocess: bad arguments");
  const long long total = static_cast<long long>(B) * H * W;
  postprocess_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(
      static_cast<const float*>(x), nhwc, B, H, W, static_cast<float*>(out_pt), static_cast<uint8_t*>(out_u8));
  count_launch();
  VTON_CUDA(cudaGetLastError());
  return kOk;
}

// ------------------------------------------------------------------------------------------------
// CLIP embedding front ends (SURVEY.md 8f row 2; transformers CLIPVisionEmbeddings / CLIPTextEmbeddings, called from
// src/tryon_pipeline.py:468-470 and :592-596).
// patchify: the stride-P patch convolution of the ViT becomes a GEMM over rows [b, gy, gx] with K = (c, ky, kx) — the
//           order of the conv weight [Cout, 3, P, P] flattened — zero-padded to a multiple of 64 columns.
// token_embed: out[r] = fp16(token_embedding[ids[r]] + position_embedding[r % T]).
// ------------------------------------------------------------------------------------------------
__global__ void patchify_kernel(const __half* x, int C, int Hi, int Wi, int P, int gh, int gw, int K, int ldk, __half* out,
                                long long total) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int col = static_cast<int>(i % ldk);
  const long long row = i / ldk;
  __half v = __float2half(0.f);
  if (col < K) {
    const int kx = col % P, ky = (col / P) % P, c = col / (P * P);
    const int gx = static_cast<int>(row % gw), gy = static_cast<int>((row / gw) % gh);
    const long long b = row / (static_cast<long long>(gw) * gh);
    v = x[((b * C + c) * Hi + gy * P + ky) * Wi + gx * P + kx];
  }
  out[i] = v;
}

int patchify_impl(const void* x, int B, int C, int Hi, int Wi, int P, void* out, int ldk, cudaStream_t stream) {
  VTON_CHECK_ARG(B > 0 && C > 0 && P > 0 && Hi >= P && Wi >= P, "patchify: bad shape");
  const int gh = Hi / P, gw = Wi / P, K = C * P * P;
  VTON_CHECK_ARG(ldk >= K, "patchify: row stride %d < K %d", ldk, K);
  const long long total = static_cast<long long>(B) * gh * gw * ldk;
  patchify_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(
      static_cast<const __half*>(x), C, Hi, Wi, P, gh, gw, K, ldk, static_cast<__half*>(out), total);
  count_launch();
  VTON_CUDA(cudaGetLastError());
  return kOk;
}

__global__ void token_embed_kernel(const long long* ids, int rows, int T, int V, int vocab, const uint4* tok, const uint4* pos,
                                   uint4* out) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<long long>(rows) * V) return;
  const int r = static_cast<int>(i / V), c = static_cast<int>(i % V);
  long long id = ids[r];
  id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
  const uint4 a = tok[id * V + c];
  const uint4 b = pos[static_cast<long long>(r % T) * V + c];
  const uint32_t aw[4] = {a.x, a.y, a.z, a.w}, bw[4] = {b.x, b.y, b.z, b.w};
  uint32_t o[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 fa = unpack_h2(aw[j]), fb = unpack_h2(bw[j]);
    o[j] = pack_h2(fa.x + fb.x, fa.y + fb.y);
  }
  out[i] = make_uint4(o[0], o[1], o[2], o[3]);
}

int token_embed_impl(const void* ids, int rows, int T, int C, int vocab, const void* tok, const void* pos, void* out,
                     cudaStream_t stream) {
  VTON_CHECK_ARG(rows > 0 && T > 0 && C > 0 && C % 8 == 0 && vocab > 0, "token_embed: bad shape rows=%d T=%d C=%d", rows, T, C);
  const int V = C / 8;
  const long long total = static_cast<long long>(rows) * V;
  token_embed_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, stream>>>(
      static_cast<const long long*>(ids), rows, T, V, vocab, static_cast<const uint4*>(tok), static_cast<const uint4*>(pos),
      static_cast<uint4*>(out));
  count_launch();
  VTON_CUDA(cudaGetLastError());
  return kOk;
}

}  // namespace vton
