// GroupNorm(32) (+SiLU) for the VAE's fp32 NHWC activations (SURVEY.md §8 row f, "next": diffusers AutoencoderKL
// ResnetBlock2D.norm1/norm2 + nonlinearity, Attention.group_norm, conv_norm_out; the reference runs the SDXL VAE in fp32,
// src/tryon_pipeline.py:913-915,1076-1093). Same structure as the fp16 kernels of norm.cu — deterministic two-stage
// statistics (per-(sample, chunk, group) partial sums in double, no atomics), then one normalise(+SiLU) pass — with
// fp32 in/out and float4 accesses; HBM-bound: 3 * B*HW*C*4 bytes per call (up to 2.4 GB at 1024x768x128).
// Checked by tests/test_kernels_gpu.py -k "fp32_nhwc or vae_nhwc"; ON by default in the VAE's NHWC route (idm-vton_b200/vae.py).
#include "common.cuh"
#include "host.h"

namespace vton {

constexpr int GN32_THREADS = 512;
constexpr int GN32_GROUPS = 32;

__global__ void __launch_bounds__(GN32_THREADS)
gn32_stats_kernel(const float* __restrict__ x, int HW, int C, int rows_per_cta, double* __restrict__ partial) {
  const int V = C / 4;                       // float4 vectors per row (<= 512)
  const int cpg = C / GN32_GROUPS;
  const int row_lanes = GN32_THREADS / V;
  const int b = blockIdx.y;
  const long long r_begin = static_cast<long long>(blockIdx.x) * rows_per_cta;
  const long long r_end = min(static_cast<long long>(HW), r_begin + rows_per_cta);
  __shared__ float ps[GN32_THREADS * 4];     // [row_lane][C] partial sums
  __shared__ float pq[GN32_THREADS * 4];
  const int v = threadIdx.x % V;
  const int rl = threadIdx.x / V;
  if (rl < row_lanes) {
    // sums of x - s_g, s_g = the sample's first pixel in the group's first channel (the same for every CTA; see
    // gn_fused_kernel): E[x^2] - mean^2 of unshifted fp32 sums loses the variance of a group with a large mean
    float sum[4] = {0.f, 0.f, 0.f, 0.f}, sq[4] = {0.f, 0.f, 0.f, 0.f}, sft[4];
    const float* sample = x + (static_cast<long long>(b) * HW) * C;
#pragma unroll
    for (int j = 0; j < 4; ++j) sft[j] = __ldg(sample + (v * 4 + j) / cpg * cpg);
    const float* base = sample + v * 4;
    for (long long r = r_begin + rl; r < r_end; r += row_lanes) {
      const float4 u = __ldg(reinterpret_cast<const float4*>(base + r * C));
      const float d[4] = {u.x - sft[0], u.y - sft[1], u.z - sft[2], u.w - sft[3]};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        sum[j] += d[j];
        sq[j] += d[j] * d[j];
      }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      ps[rl * C + v * 4 + j] = sum[j];
      pq[rl * C + v * 4 + j] = sq[j];
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += GN32_THREADS) {   // per-channel totals, fixed order over row lanes
    float a = 0.f, q = 0.f;
    for (int l = 0; l < row_lanes; ++l) {
      a += ps[l * C + c];
      q += pq[l * C + c];
    }
    ps[c] = a;
    pq[c] = q;
  }
  __syncthreads();
  if (threadIdx.x < GN32_GROUPS) {
    double a = 0.0, q = 0.0;
    for (int i = 0; i < cpg; ++i) {
      a += static_cast<double>(ps[threadIdx.x * cpg + i]);
      q += static_cast<double>(pq[threadIdx.x * cpg + i]);
    }
    double* dst = partial + ((static_cast<long long>(b) * gridDim.x + blockIdx.x) * GN32_GROUPS + threadIdx.x) * 2;
    dst[0] = a;
    dst[1] = q;
  }
}

// HALF_OUT: the normalised (+SiLU) values are stored as fp16 — the consumer is the fp16-operand convolution
// (conv_tf32.cu, F16IN), whose 10-bit operand mantissa is the one the TF32 convolution would round these values to anyway.
template <bool HALF_OUT>
__global__ void __launch_bounds__(GN32_THREADS)
gn32_apply_kernel(const float* __restrict__ x, int HW, int C, int rows_per_cta, const double* __restrict__ partial,
                  const float* __restrict__ gamma, const float* __restrict__ beta, float eps, int silu,
                  void* __restrict__ out_v) {
  const int V = C / 4;
  const int cpg = C / GN32_GROUPS;
  const int row_lanes = GN32_THREADS / V;
  const int b = blockIdx.y;
  const long long r_begin = static_cast<long long>(blockIdx.x) * rows_per_cta;
  const long long r_end = min(static_cast<long long>(HW), r_begin + rows_per_cta);
  const int v = threadIdx.x % V;
  const int rl = threadIdx.x / V;
  __shared__ float s_mean[GN32_GROUPS], s_rstd[GN32_GROUPS];
  __shared__ double red_a[GN32_THREADS / GN32_GROUPS][GN32_GROUPS], red_q[GN32_THREADS / GN32_GROUPS][GN32_GROUPS];
  {
    const int g = threadIdx.x & (GN32_GROUPS - 1), sl = threadIdx.x / GN32_GROUPS;
    double a = 0.0, q = 0.0;
    for (int ch = sl; ch < static_cast<int>(gridDim.x); ch += GN32_THREADS / GN32_GROUPS) {
      const double2 pv = *reinterpret_cast<const double2*>(
          partial + ((static_cast<long long>(b) * gridDim.x + ch) * GN32_GROUPS + g) * 2);
      a += pv.x;
      q += pv.y;
    }
    red_a[sl][g] = a;
    red_q[sl][g] = q;
  }
  __syncthreads();
  if (threadIdx.x < GN32_GROUPS) {
    double a = 0.0, q = 0.0;
#pragma unroll
    for (int sl = 0; sl < GN32_THREADS / GN32_GROUPS; ++sl) {
      a += red_a[sl][threadIdx.x];
      q += red_q[sl][threadIdx.x];
    }
    const double n = static_cast<double>(cpg) * HW;
    const double dmean = a / n;                   // mean of x - s_g
    double var = q / n - dmean * dmean;
    var = var < 0.0 ? 0.0 : var;
    const float shift = __ldg(x + (static_cast<long long>(b) * HW) * C + threadIdx.x * cpg);
    s_mean[threadIdx.x] = static_cast<float>(shift + dmean);
    s_rstd[threadIdx.x] = static_cast<float>(1.0 / sqrt(var + static_cast<double>(eps)));
  }
  __syncthreads();
  if (rl >= row_lanes) return;
  // y = (x - mean) * (rstd * gamma) + beta: subtracting first keeps a large mean from cancelling in fp32
  float sc[4], sh[4], mu[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int c = v * 4 + j;
    const int g = c / cpg;
    const float gm = gamma ? gamma[c] : 1.f;
    sc[j] = s_rstd[g] * gm;
    sh[j] = beta ? beta[c] : 0.f;
    mu[j] = s_mean[g];
  }
  const long long off = (static_cast<long long>(b) * HW) * C + v * 4;
  for (long long r = r_begin + rl; r < r_end; r += row_lanes) {
    const float4 u = __ldg(reinterpret_cast<const float4*>(x + off + r * C));
    float y[4] = {fmaf(u.x - mu[0], sc[0], sh[0]), fmaf(u.y - mu[1], sc[1], sh[1]), fmaf(u.z - mu[2], sc[2], sh[2]),
                  fmaf(u.w - mu[3], sc[3], sh[3])};
    if (silu) {
#pragma unroll
      for (int j = 0; j < 4; ++j) y[j] = silu_f(y[j]);
    }
    if (HALF_OUT) {
      uint2 o;
      o.x = pack_h2(y[0], y[1]);
      o.y = pack_h2(y[2], y[3]);
      *reinterpret_cast<uint2*>(static_cast<__half*>(out_v) + off + r * C) = o;
    } else {
      *reinterpret_cast<float4*>(static_cast<float*>(out_v) + off + r * C) = make_float4(y[0], y[1], y[2], y[3]);
    }
  }
}

// x: [B, HW, C] fp32 dense NHWC; out: the same shape, fp32 or (out_fp16) fp16, and must not alias x (every apply CTA
// re-reads the shift in row 0 of its sample, which CTA 0 overwrites); gamma/beta: [C] fp32 or null;
// stats_ws: B * chunks(<= 1184) * 64 doubles
int groupnorm_f32_impl(const void* x, int B, int HW, int C, const void* gamma, const void* beta, float eps, int silu,
                       void* stats_ws, long long stats_ws_doubles, void* out, int out_fp16, cudaStream_t stream) {
  VTON_CHECK_ARG(B > 0 && HW > 0 && C > 0, "groupnorm_f32: empty input");
  VTON_CHECK_ARG(C % GN32_GROUPS == 0 && C % 4 == 0 && C / 4 <= GN32_THREADS, "groupnorm_f32: C=%d unsupported (32 groups, C <= 2048, C %% 4 == 0)", C);
  VTON_CHECK_ARG(x && out && stats_ws, "groupnorm_f32: null pointer");
  VTON_CHECK_ARG(B <= 65535, "groupnorm_f32: batch too large");
  int chunks = 1184 / B;                     // 8 CTAs per SM in flight over the whole batch
  if (chunks < 1) chunks = 1;
  if (chunks > cdiv(HW, 16)) chunks = cdiv(HW, 16);
  const int rows_per_cta = cdiv(HW, chunks);
  chunks = cdiv(HW, rows_per_cta);
  VTON_CHECK_ARG(static_cast<long long>(B) * chunks * 64 <= stats_ws_doubles, "groupnorm_f32: stats workspace too small (%lld doubles needed)",
                 static_cast<long long>(B) * chunks * 64);
  dim3 grid(chunks, B);
  gn32_stats_kernel<<<grid, GN32_THREADS, 0, stream>>>(static_cast<const float*>(x), HW, C, rows_per_cta,
                                                       static_cast<double*>(stats_ws));
  if (out_fp16)
    gn32_apply_kernel<true><<<grid, GN32_THREADS, 0, stream>>>(static_cast<const float*>(x), HW, C, rows_per_cta,
                                                             static_cast<const double*>(stats_ws),
                                                             static_cast<const float*>(gamma), static_cast<const float*>(beta),
                                                             eps, silu, out);
  else
    gn32_apply_kernel<false><<<grid, GN32_THREADS, 0, stream>>>(static_cast<const float*>(x), HW, C, rows_per_cta,
                                                              static_cast<const double*>(stats_ws),
                                                              static_cast<const float*>(gamma), static_cast<const float*>(beta),
                                                              eps, silu, out);
  count_launch(2);
  VTON_CUDA(cudaGetLastError());
  return kOk;
}

}  // namespace vton
