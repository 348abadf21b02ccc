// GroupNorm(32) (+SiLU) and LayerNorm for the UNets' NHWC / token-major fp16 activations (sm_90a, HBM-bound).
//
// Reference rounding points (SURVEY.md App. D.1): under torch.cuda.amp.autocast the norms run in fp32 on the fp16
// input and return fp32; SiLU stays fp32; the consuming conv / linear casts to fp16. So both kernels compute in fp32
// and round ONCE to fp16 on store.
//   GroupNorm: diffusers ResnetBlock2D norm1/norm2 (+SiLU), Transformer2DModel.norm (eps 1e-6, no act;
//              src/transformerhacked_tryon.py:148,329), conv_norm_out (src/unet_hacked_tryon.py:744,1384-1385).
//              The input may be the channel-concat of two tensors (up-block skip, src/unet_block_hacked_tryon.py:2346)
//              which is never materialised: both sources are read in place.
//   LayerNorm: BasicTransformerBlock.norm1/2/3 (src/attentionhacked_tryon.py:310,365,390), eps 1e-5.
#include <cuda_fp8.h>

#include "common.cuh"
#include "host.h"

namespace vton {

constexpr int GN_THREADS = 512;
constexpr int GN_GROUPS = 32;

struct GnSrc {
  const __half* x0;
  const __half* x1;
  int C0, C1;  // channels of each source (C1 = 0: single source)
};

__device__ __forceinline__ uint4 gn_load(const GnSrc& s, long long row, int v) {
  const int c = v * 8;
  if (c < s.C0) return *reinterpret_cast<const uint4*>(s.x0 + row * s.C0 + c);
  return *reinterpret_cast<const uint4*>(s.x1 + row * s.C1 + (c - s.C0));
}
__device__ __forceinline__ float gn_scalar(const GnSrc& s, long long row, int c) {
  return h2f(c < s.C0 ? s.x0[row * s.C0 + c] : s.x1[row * s.C1 + (c - s.C0)]);
}

// ONE launch per GroupNorm (round 2; round 1 ran a statistics kernel and an apply kernel = 3 passes over the tensor):
//   phase 1: CTA (chunk, b) streams its rows once, accumulates per-channel sums / sums of squares of x - s_g in a fixed
//            order (s_g = the sample's first pixel in the group's first channel, the same value for every CTA: without the
//            shift, E[x^2] - mean^2 of fp32 sums loses the variance of a group whose mean is large against its spread) and —
//            when its rows fit shared memory (RESIDENT) — parks the raw fp16 rows there; it publishes
//            partial[b][chunk][g] = {sum, sum of squares} (double).
//   barrier: the CTAs of ONE sample meet at a sense-reversing barrier in global memory (count + sense per sample; the
//            last arriver resets the count and flips the sense, so the state is reusable by the next launch / graph
//            replay without host intervention). All CTAs of a launch are co-resident by construction (grid <= SMs x
//            occupancy, see groupnorm_impl), so the spin cannot starve an unscheduled CTA.
//   phase 2: every CTA sums the chunk partials of its sample in a FIXED order (no atomics on data: a CUDA-graph replay is
//            bit-identical to eager launches), derives mean / rstd, and normalises its rows from shared memory (RESIDENT:
//            the tensor is read from global memory once) or by re-reading them (L2-resident for the UNet's sizes).
// HBM traffic: 1 read + 1 write of the tensor; 46 launches per try-on step instead of 92.
struct GnBarrier {
  int count;
  int sense;
};

template <bool RESIDENT>
__global__ void __launch_bounds__(GN_THREADS, 2)
gn_fused_kernel(GnSrc src, int HW, int rows_per_cta, double* partial, GnBarrier* bar, const __half* gamma,
                const __half* beta, float eps, int silu, __half* out) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ uint4 gn_rows[];   // RESIDENT: [rows_per_cta][V] raw rows of this CTA
  const int C = src.C0 + src.C1;
  const int V = C / 8;
  const int cpg = C / GN_GROUPS;
  const int row_lanes = GN_THREADS / V;
  const int b = blockIdx.y;
  const int r_begin = blockIdx.x * rows_per_cta;
  const int r_end = min(HW, r_begin + rows_per_cta);
  __shared__ float ps[GN_THREADS * 8];  // [row_lane][C] partial sums
  __shared__ float pq[GN_THREADS * 8];  // [row_lane][C] partial sums of squares
  __shared__ float s_mean[GN_GROUPS], s_rstd[GN_GROUPS], s_shift[GN_GROUPS];
  __shared__ int s_sense;
  const int v = threadIdx.x % V;
  const int rl = threadIdx.x / V;
  if (threadIdx.x == 0) s_sense = *reinterpret_cast<volatile int*>(&bar[b].sense);   // read BEFORE anyone can flip it
  if (threadIdx.x < GN_GROUPS) s_shift[threadIdx.x] = gn_scalar(src, static_cast<long long>(b) * HW, threadIdx.x * cpg);
  // ---------------- phase 1: statistics of x - s_g (and parking the rows)
  if (rl < row_lanes) {
    float sum[8], sq[8], sft[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      sum[j] = sq[j] = 0.f;
      sft[j] = gn_scalar(src, static_cast<long long>(b) * HW, (v * 8 + j) / cpg * cpg);
    }
    auto acc = [&](const uint4 u) {
      const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = unpack_h2(w[j]);
        const float d0 = f.x - sft[2 * j], d1 = f.y - sft[2 * j + 1];
        sum[2 * j] += d0;
        sq[2 * j] += d0 * d0;
        sum[2 * j + 1] += d1;
        sq[2 * j + 1] += d1 * d1;
      }
    };
    int r = r_begin + rl;
    // six independent 16-byte loads in flight per thread: with 16-32 warps per SM the statistics pass is bound by
    // bytes in flight per SM x memory latency, not by issue (ncu r2: 30 us for 31.5 MB with a 4-deep loop)
    for (; r + 5 * row_lanes < r_end; r += 6 * row_lanes) {
      uint4 u[6];
#pragma unroll
      for (int k = 0; k < 6; ++k) u[k] = gn_load(src, static_cast<long long>(b) * HW + r + k * row_lanes, v);
#pragma unroll
      for (int k = 0; k < 6; ++k) {
        if (RESIDENT) gn_rows[(r + k * row_lanes - r_begin) * V + v] = u[k];
        acc(u[k]);
      }
    }
    for (; r + 1 * row_lanes < r_end; r += 2 * row_lanes) {
      uint4 u[2];
#pragma unroll
      for (int k = 0; k < 2; ++k) u[k] = gn_load(src, static_cast<long long>(b) * HW + r + k * row_lanes, v);
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        if (RESIDENT) gn_rows[(r + k * row_lanes - r_begin) * V + v] = u[k];
        acc(u[k]);
      }
    }
    for (; r < r_end; r += row_lanes) {
      const uint4 u = gn_load(src, static_cast<long long>(b) * HW + r, v);
      if (RESIDENT) gn_rows[(r - r_begin) * V + v] = u;
      acc(u);
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      ps[rl * C + v * 8 + j] = sum[j];
      pq[rl * C + v * 8 + j] = sq[j];
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += GN_THREADS) {  // per-channel totals, fixed order over row lanes
    float a = 0.f, q = 0.f;
    for (int l = 0; l < row_lanes; ++l) {
      a += ps[l * C + c];
      q += pq[l * C + c];
    }
    ps[c] = a;
    pq[c] = q;
  }
  __syncthreads();
  if (threadIdx.x < GN_GROUPS) {
    double a = 0.0, q = 0.0;
    for (int i = 0; i < cpg; ++i) {
      a += static_cast<double>(ps[threadIdx.x * cpg + i]);
      q += static_cast<double>(pq[threadIdx.x * cpg + i]);
    }
    double* dst = partial + ((static_cast<long long>(b) * gridDim.x + blockIdx.x) * GN_GROUPS + threadIdx.x) * 2;
    dst[0] = a;
    dst[1] = q;
    __threadfence();   // the partials are visible device-wide before this CTA arrives at the barrier
  }
  __syncthreads();
  // ---------------- per-sample barrier (sense reversal; bounded spin: a bug must trap, not hang the GPU)
  if (threadIdx.x == 0 && gridDim.x > 1) {
    const int my = s_sense;
    if (atomicAdd(&bar[b].count, 1) == static_cast<int>(gridDim.x) - 1) {
      bar[b].count = 0;
      __threadfence();
      atomicExch(&bar[b].sense, my ^ 1);
    } else {
      const uint64_t t0 = globaltimer_ns();
      uint32_t spins = 0;
      while (*reinterpret_cast<volatile int*>(&bar[b].sense) == my) {
        __nanosleep(64);
        if ((++spins & 0x3ff) == 0 && globaltimer_ns() - t0 > 4000000000ull) {
          printf("b200vton: groupnorm barrier timeout block(%d,%d)\n", blockIdx.x, blockIdx.y);
          __trap();
        }
      }
    }
    __threadfence();
  }
  __syncthreads();
  // ---------------- phase 2: total statistics in a fixed order, then apply
  {
    double* red_a = reinterpret_cast<double*>(ps);   // [16][32] doubles = 4 KB each, ps / pq are free now
    double* red_q = reinterpret_cast<double*>(pq);
    const int g = threadIdx.x & (GN_GROUPS - 1), sl = threadIdx.x / GN_GROUPS;
    double a = 0.0, q = 0.0;
    {
      // the chunk partials of this (slice, group) are fetched five at a time before they are summed (independent L2
      // loads; the order of the additions is fixed): 74 chunks per sample at batch 4 = one batch of five per thread
      constexpr int SLICES = GN_THREADS / GN_GROUPS;
      for (int c0 = sl; c0 < static_cast<int>(gridDim.x); c0 += 5 * SLICES) {
        double2 pv[5];
#pragma unroll
        for (int k = 0; k < 5; ++k) {
          const int ch = c0 + k * SLICES;
          pv[k] = ch < static_cast<int>(gridDim.x)
                      ? __ldcg(reinterpret_cast<const double2*>(
                            partial + ((static_cast<long long>(b) * gridDim.x + ch) * GN_GROUPS + g) * 2))
                      : make_double2(0.0, 0.0);
        }
#pragma unroll
        for (int k = 0; k < 5; ++k) {
          a += pv[k].x;
          q += pv[k].y;
        }
      }
    }
    red_a[sl * GN_GROUPS + g] = a;
    red_q[sl * GN_GROUPS + g] = q;
    __syncthreads();
    if (threadIdx.x < GN_GROUPS) {
      double ta = 0.0, tq = 0.0;
#pragma unroll
      for (int s2 = 0; s2 < GN_THREADS / GN_GROUPS; ++s2) {
        ta += red_a[s2 * GN_GROUPS + threadIdx.x];
        tq += red_q[s2 * GN_GROUPS + threadIdx.x];
      }
      const double n = static_cast<double>(cpg) * HW;
      const double dmean = ta / n;                 // mean of x - s_g
      double var = tq / n - dmean * dmean;
      var = var < 0.0 ? 0.0 : var;
      s_mean[threadIdx.x] = static_cast<float>(s_shift[threadIdx.x] + dmean);
      s_rstd[threadIdx.x] = rsqrtf(static_cast<float>(var) + eps);
    }
    __syncthreads();
  }
  if (rl >= row_lanes) return;
  // y = x * (rstd * gamma) + (beta - mean * rstd * gamma)
  float sc[8], sh[8], mu[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int c = v * 8 + j;
    const int g = c / cpg;
    const float gm = gamma ? h2f(gamma[c]) : 1.f;
    sc[j] = s_rstd[g] * gm;
    sh[j] = beta ? h2f(beta[c]) : 0.f;
    mu[j] = s_mean[g];
  }
  auto apply_row = [&](int r, const uint4 u) {
    const long long row = static_cast<long long>(b) * HW + r;
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
    float y[8];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = unpack_h2(w[j]);
      y[2 * j] = f.x * sc[2 * j] + (sh[2 * j] - mu[2 * j] * sc[2 * j]);
      y[2 * j + 1] = f.y * sc[2 * j + 1] + (sh[2 * j + 1] - mu[2 * j + 1] * sc[2 * j + 1]);
    }
    if (silu) {
#pragma unroll
      for (int j = 0; j < 8; ++j) y[j] = silu_f(y[j]);
    }
    uint4 o;
    o.x = pack_h2(y[0], y[1]);
    o.y = pack_h2(y[2], y[3]);
    o.z = pack_h2(y[4], y[5]);
    o.w = pack_h2(y[6], y[7]);
    *reinterpret_cast<uint4*>(out + row * C + v * 8) = o;
  };
  int r = r_begin + rl;
  for (; r + 3 * row_lanes < r_end; r += 4 * row_lanes) {   // the re-read (L2 hits in the streaming variant) is 4 deep
    uint4 u[4];
#pragma unroll
    for (int k = 0; k < 4; ++k)
      u[k] = RESIDENT ? gn_rows[(r + k * row_lanes - r_begin) * V + v]
                      : gn_load(src, static_cast<long long>(b) * HW + r + k * row_lanes, v);
#pragma unroll
    for (int k = 0; k < 4; ++k) apply_row(r + k * row_lanes, u[k]);
  }
  for (; r < r_end; r += row_lanes)
    apply_row(r, RESIDENT ? gn_rows[(r - r_begin) * V + v] : gn_load(src, static_cast<long long>(b) * HW + r, v));
}

// stats_ws layout (doubles): [max(B,296) * 64] per-(sample, chunk, group) partial sums, then GN_BAR_BYTES of barrier state
// (GnBarrier per sample) that must be ZERO before the first launch on this workspace and is left zero-count afterwards.
constexpr int GN_WS_PARTIAL_DOUBLES = 296 * 64;
constexpr int GN_MAX_BATCH_BARRIER = 4096;

int groupnorm_impl(const void* x0, int C0, const void* x1, int C1, int B, int HW, const void* gamma, const void* beta,
                   float eps, int silu, void* stats_ws, void* out, cudaStream_t stream) {
  const int C = C0 + C1;
  VTON_CHECK_ARG(B > 0 && HW > 0 && C > 0, "groupnorm: empty input");
  VTON_CHECK_ARG(C % GN_GROUPS == 0 && C0 % 8 == 0 && C1 % 8 == 0, "groupnorm: C=%d must divide into 32 groups, sources multiple of 8", C);
  VTON_CHECK_ARG(C / 8 <= GN_THREADS, "groupnorm: C=%d too wide", C);
  VTON_CHECK_ARG(stats_ws != nullptr, "groupnorm: stats workspace required (see include/b200vton.h)");
  VTON_CHECK_ARG(B <= GN_MAX_BATCH_BARRIER, "groupnorm: batch %d > %d", B, GN_MAX_BATCH_BARRIER);
  VTON_CHECK_ARG(aligned_to(x0, 16) && aligned_to(x1, 16) && aligned_to(out, 16),
                 "groupnorm: x0/x1/out must be 16-byte aligned (rows are read and written 8 halves at a time)");
  GnSrc src{static_cast<const __half*>(x0), static_cast<const __half*>(x1), C0, C1};
  static int max_smem = 0, occ_stream = 0;
  if (!max_smem) {
    int dev = 0, optin = 0;
    VTON_CUDA(cudaGetDevice(&dev));
    VTON_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    cudaFuncAttributes fa;
    VTON_CUDA(cudaFuncGetAttributes(&fa, gn_fused_kernel<true>));
    max_smem = optin - static_cast<int>(fa.sharedSizeBytes) - 1024;
    VTON_CUDA(cudaFuncSetAttribute(gn_fused_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
    VTON_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_stream, gn_fused_kernel<false>, GN_THREADS, 0));
    if (occ_stream < 1) occ_stream = 1;
    if (occ_stream > 2) occ_stream = 2;
  }
  double* partial = static_cast<double*>(stats_ws);
  const int ws_rows = B > 296 ? B : 296;
  GnBarrier* bar = reinterpret_cast<GnBarrier*>(partial + static_cast<long long>(ws_rows) * 64);
  // RESIDENT: one CTA per SM, its rows parked in shared memory
  int chunks_r = num_sms() / B;
  if (chunks_r * B > ws_rows) chunks_r = ws_rows / B;   // the partial-sum workspace holds ws_rows (sample, chunk) rows
  if (chunks_r > cdiv(HW, 16)) chunks_r = cdiv(HW, 16);
  bool resident = false;
  int rows_per_cta = 0, chunks = 0;
  if (chunks_r >= 1) {
    rows_per_cta = cdiv(HW, chunks_r);
    if (static_cast<long long>(rows_per_cta) * C * 2 <= max_smem) {
      resident = true;
      chunks = cdiv(HW, rows_per_cta);
    }
  }
  if (!resident) {
    chunks = (num_sms() * occ_stream) / B;   // every CTA of the launch co-resident
    if (chunks * B > ws_rows) chunks = ws_rows / B;
    if (chunks < 1) chunks = 1;         // B > capacity: one CTA per sample, nobody waits for anybody
    if (chunks > cdiv(HW, 16)) chunks = cdiv(HW, 16);
    rows_per_cta = cdiv(HW, chunks);
    chunks = cdiv(HW, rows_per_cta);
  }
  dim3 grid(chunks, B);
  if (resident) {
    VTON_CUDA(launch_kernel(gn_fused_kernel<true>, grid, dim3(GN_THREADS),
                            static_cast<size_t>(rows_per_cta) * C * 2, stream, src, HW, rows_per_cta, partial, bar,
                            static_cast<const __half*>(gamma), static_cast<const __half*>(beta), eps, silu,
                            static_cast<__half*>(out)));
  } else {
    VTON_CUDA(launch_kernel(gn_fused_kernel<false>, grid, dim3(GN_THREADS), 0, stream, src, HW, rows_per_cta, partial, bar,
                            static_cast<const __half*>(gamma), static_cast<const __half*>(beta), eps, silu,
                            static_cast<__half*>(out)));
  }
  count_launch(1);
  return kOk;
}

// ------------------------------------------------------------------------------------------------
// LayerNorm: one warp per row, values held in registers (C <= 2048)
// ------------------------------------------------------------------------------------------------
constexpr int LN_MAX_VEC = 8;  // per lane: up to 8 x 8 halves => C <= 2048

// NV = ceil(C / 256) uint4 loads per lane, a compile-time bound so the row lives in 8*NV registers (C = 640: 24,
// C = 1280: 40) and the SM holds enough warps to cover the load latency.
// QUANT (layernorm_e4m3, the FP8 linears' input): the same arithmetic gives the fp16 row y16; then amax = max|y16|
// over the row, scale = amax / 448 and q = e4m3_rn_satfinite(y16 * (448 / amax)) (an all-zero row: scale 1, q 0).
// `out` (the fp16 row, bit-identical to the plain LayerNorm) is optional then.
template <int NV, bool QUANT>
__global__ void __launch_bounds__(256)
layernorm_kernel(const __half* x, long long ldx, int rows, int C, const __half* gamma, const __half* beta, float eps,
                 __half* out, long long ldo, __nv_fp8_storage_t* q, long long ldq, float* q_scale) {
  pdl_launch_dependents();
  pdl_wait();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row = blockIdx.x * 8 + warp;
  if (row >= rows) return;
  const int V = C / 8;
  float val[NV][8];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int v = lane + i * 32;
    if (v < V) {
      const uint4 u = *reinterpret_cast<const uint4*>(x + row * ldx + v * 8);
      const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = unpack_h2(w[j]);
        val[i][2 * j] = f.x;
        val[i][2 * j + 1] = f.y;
        sum += f.x + f.y;
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float mean = sum / C;
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int v = lane + i * 32;
    if (v < V) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float d = val[i][j] - mean;
        sq += d * d;
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
  const float rstd = rsqrtf(sq / C + eps);
  uint32_t yw[QUANT ? NV : 1][4];   // the fp16 row, kept for the quantization pass
  float amax = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int v = lane + i * 32;
    if (v < V) {
      const uint4 g = gamma ? *reinterpret_cast<const uint4*>(gamma + v * 8) : make_uint4(0x3c003c00u, 0x3c003c00u, 0x3c003c00u, 0x3c003c00u);
      const uint4 bt = beta ? *reinterpret_cast<const uint4*>(beta + v * 8) : make_uint4(0, 0, 0, 0);
      const uint32_t gw[4] = {g.x, g.y, g.z, g.w};
      const uint32_t bw[4] = {bt.x, bt.y, bt.z, bt.w};
      uint32_t ow[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 gg = unpack_h2(gw[j]);
        const float2 bb = unpack_h2(bw[j]);
        const float y0 = (val[i][2 * j] - mean) * rstd * gg.x + bb.x;
        const float y1 = (val[i][2 * j + 1] - mean) * rstd * gg.y + bb.y;
        ow[j] = pack_h2(y0, y1);
        if constexpr (QUANT) {
          const float2 y = unpack_h2(ow[j]);
          amax = fmaxf(amax, fmaxf(fabsf(y.x), fabsf(y.y)));
          yw[i][j] = ow[j];
        }
      }
      if (!QUANT || out != nullptr)
        *reinterpret_cast<uint4*>(out + row * ldo + v * 8) = make_uint4(ow[0], ow[1], ow[2], ow[3]);
    }
  }
  if constexpr (QUANT) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    const float inv = amax > 0.f ? __fdiv_rn(448.0f, amax) : 0.f;
    if (lane == 0) q_scale[row] = amax > 0.f ? __fdiv_rn(amax, 448.0f) : 1.0f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int v = lane + i * 32;
      if (v < V) {
        uint32_t qw[2];
#pragma unroll
        for (int j = 0; j < 4; j += 2) {
          const float2 a = unpack_h2(yw[i][j]), b = unpack_h2(yw[i][j + 1]);
          const __nv_fp8x2_storage_t lo = __nv_cvt_float2_to_fp8x2(make_float2(__fmul_rn(a.x, inv), __fmul_rn(a.y, inv)),
                                                                   __NV_SATFINITE, __NV_E4M3);
          const __nv_fp8x2_storage_t hi = __nv_cvt_float2_to_fp8x2(make_float2(__fmul_rn(b.x, inv), __fmul_rn(b.y, inv)),
                                                                   __NV_SATFINITE, __NV_E4M3);
          qw[j / 2] = static_cast<uint32_t>(lo) | (static_cast<uint32_t>(hi) << 16);
        }
        *reinterpret_cast<uint2*>(q + row * ldq + v * 8) = make_uint2(qw[0], qw[1]);
      }
    }
  }
}

template <bool QUANT>
static int layernorm_launch(const void* x, long long ldx, int rows, int C, const void* gamma, const void* beta, float eps,
                            void* out, long long ldo, void* q, long long ldq, void* q_scale, cudaStream_t stream) {
  const int nv = cdiv(C / 8, 32);
  auto go = [&](auto kern) {
    return launch_kernel(kern, dim3(cdiv(rows, 8)), dim3(256), 0, stream, static_cast<const __half*>(x), ldx, rows, C,
                         static_cast<const __half*>(gamma), static_cast<const __half*>(beta), eps,
                         static_cast<__half*>(out), ldo, static_cast<__nv_fp8_storage_t*>(q), ldq,
                         static_cast<float*>(q_scale));
  };
  cudaError_t le = cudaSuccess;
  switch (nv) {
    case 1: le = go(layernorm_kernel<1, QUANT>); break;
    case 2: le = go(layernorm_kernel<2, QUANT>); break;
    case 3: le = go(layernorm_kernel<3, QUANT>); break;
    case 4: le = go(layernorm_kernel<4, QUANT>); break;
    case 5: le = go(layernorm_kernel<5, QUANT>); break;
    default: le = go(layernorm_kernel<LN_MAX_VEC, QUANT>); break;
  }
  VTON_CUDA(le);
  count_launch();
  return kOk;
}

int layernorm_impl(const void* x, long long ldx, int rows, int C, const void* gamma, const void* beta, float eps,
                   void* out, long long ldo, cudaStream_t stream) {
  VTON_CHECK_ARG(rows > 0 && C > 0, "layernorm: empty input");
  VTON_CHECK_ARG(C % 8 == 0 && C <= LN_MAX_VEC * 256 && ldx % 8 == 0 && ldo % 8 == 0, "layernorm: C=%d unsupported", C);
  VTON_CHECK_ARG(aligned_to(x, 16) && aligned_to(out, 16) && aligned_to(gamma, 16) && aligned_to(beta, 16),
                 "layernorm: x/out/gamma/beta must be 16-byte aligned (read and written 8 halves at a time)");
  return layernorm_launch<false>(x, ldx, rows, C, gamma, beta, eps, out, ldo, nullptr, 0, nullptr, stream);
}

int layernorm_e4m3_impl(const void* x, long long ldx, int rows, int C, const void* gamma, const void* beta, float eps,
                        void* out, long long ldo, void* q, long long ldq, void* q_scale, cudaStream_t stream) {
  VTON_CHECK_ARG(rows > 0 && C > 0, "layernorm_e4m3: empty input");
  VTON_CHECK_ARG(C % 8 == 0 && C <= LN_MAX_VEC * 256 && ldx % 8 == 0 && (!out || ldo % 8 == 0),
                 "layernorm_e4m3: C=%d unsupported", C);
  VTON_CHECK_ARG(q && q_scale, "layernorm_e4m3: q and q_scale must not be null");
  VTON_CHECK_ARG(ldq % 16 == 0 && ldq >= C, "layernorm_e4m3: ldq=%lld must be a multiple of 16 and >= C", ldq);
  VTON_CHECK_ARG(aligned_to(x, 16) && aligned_to(out, 16) && aligned_to(gamma, 16) && aligned_to(beta, 16) &&
                     aligned_to(q, 16) && aligned_to(q_scale, 4),
                 "layernorm_e4m3: x/out/q/gamma/beta must be 16-byte aligned, q_scale 4-byte");
  return layernorm_launch<true>(x, ldx, rows, C, gamma, beta, eps, out, ldo, q, ldq, q_scale, stream);
}

}  // namespace vton
