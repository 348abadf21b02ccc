// fp32 helpers of the VAE's mid-block attention (SURVEY.md 8f row 1; diffusers AutoencoderKL mid_block.attentions[0]: ONE head
// of 512 channels over H*W tokens, exact fp32 in the reference because src/tryon_pipeline.py:913-915,1076-1093 upcasts the
// VAE). idm-vton_b200/vae.py runs its products on the TF32 tensor cores three times with split operands
// (a.b ~ a_lo.b_hi + a_hi.b_lo + a_hi.b_hi); these kernels produce the split operands in ONE pass each instead of the five
// ATen passes per split (the probabilities alone are 100 MB per 2048-query chunk
// and image):
//   split_tf32:          x (* scale) -> hi = tf32(x), lo = tf32(x - hi), both exactly representable in TF32, so the tensor
//                        core (which ignores the 13 low mantissa bits of its fp32 operands) sees them unchanged;
//   softmax_split_tf32:  one row of scores -> softmax in fp32 (max-subtracted, expf, fp32 sum) -> the hi / lo parts of the
//                        probabilities, without writing the fp32 probabilities themselves.
#include "common.cuh"
#include "host.h"

namespace vton {

// round half up on the 13 low mantissa bits, then clear them (the formula of vae._split_tf32)
__device__ __forceinline__ float tf32_round(float x) {
  return __int_as_float((__float_as_int(x) + 4096) & static_cast<int>(0xFFFFE000u));
}

__global__ void split_tf32_kernel(const float* __restrict__ x, long long stride_b, long long per_batch, float scale,
                                  float* __restrict__ hi, float* __restrict__ lo, long long total4) {
  // x: [B] blocks of per_batch contiguous floats, batch stride stride_b (a row slice of a dense [B,N,C] tensor); outputs dense
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total4;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long e = i * 4;
    const long long b = e / per_batch, r = e - b * per_batch;
    float4 v = *reinterpret_cast<const float4*>(x + b * stride_b + r);
    v.x *= scale; v.y *= scale; v.z *= scale; v.w *= scale;
    float4 h, l;
    h.x = tf32_round(v.x); h.y = tf32_round(v.y); h.z = tf32_round(v.z); h.w = tf32_round(v.w);
    l.x = tf32_round(v.x - h.x); l.y = tf32_round(v.y - h.y); l.z = tf32_round(v.z - h.z); l.w = tf32_round(v.w - h.w);
    *reinterpret_cast<float4*>(hi + e) = h;
    *reinterpret_cast<float4*>(lo + e) = l;
  }
}

int split_tf32_impl(const void* x, long long stride_b, int B, long long per_batch, float scale, void* hi, void* lo,
                    cudaStream_t stream) {
  VTON_CHECK_ARG(B > 0 && per_batch > 0 && per_batch % 4 == 0 && stride_b % 4 == 0, "split_tf32: bad shape B=%d per_batch=%lld", B,
                 per_batch);
  VTON_CHECK_ARG((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(hi) & 15) == 0 &&
                     (reinterpret_cast<uintptr_t>(lo) & 15) == 0, "split_tf32: pointers must be 16-byte aligned");
  const long long total4 = static_cast<long long>(B) * per_batch / 4;
  long long blocks = (total4 + 255) / 256;
  if (blocks > num_sms() * 16) blocks = num_sms() * 16;
  split_tf32_kernel<<<static_cast<unsigned>(blocks), 256, 0, stream>>>(static_cast<const float*>(x), stride_b, per_batch, scale,
                                                                      static_cast<float*>(hi), static_cast<float*>(lo), total4);
  count_launch();
  VTON_CUDA(cudaGetLastError());
  return kOk;
}

constexpr int SS_THREADS = 256;

__device__ __forceinline__ float block_reduce(float v, bool is_max, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float u = __shfl_xor_sync(0xffffffffu, v, o);
    v = is_max ? fmaxf(v, u) : v + u;
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();            // red may still be read by the previous reduction
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float r = red[0];
#pragma unroll
  for (int w = 1; w < SS_THREADS / 32; ++w) r = is_max ? fmaxf(r, red[w]) : r + red[w];   // fixed order: deterministic
  return r;
}

// one CTA per row of N scores (N % 4 == 0); the row (48 KB at 12288 keys) is read three times, from L1 / L2 after the first
__global__ void __launch_bounds__(SS_THREADS)
softmax_split_tf32_kernel(const float* __restrict__ s, int N, float* __restrict__ phi, float* __restrict__ plo) {
  __shared__ float red[SS_THREADS / 32];
  const long long row = blockIdx.x;
  const float4* src = reinterpret_cast<const float4*>(s + row * N);
  const int n4 = N >> 2;
  float m = -INFINITY;
  for (int i = threadIdx.x; i < n4; i += SS_THREADS) {
    const float4 v = src[i];
    m = fmaxf(fmaxf(m, fmaxf(v.x, v.y)), fmaxf(v.z, v.w));
  }
  m = block_reduce(m, true, red);
  float sum = 0.f;
  for (int i = threadIdx.x; i < n4; i += SS_THREADS) {
    const float4 v = src[i];
    sum += (expf(v.x - m) + expf(v.y - m)) + (expf(v.z - m) + expf(v.w - m));
  }
  sum = block_reduce(sum, false, red);
  const float inv = 1.0f / sum;
  float4* dh = reinterpret_cast<float4*>(phi + row * N);
  float4* dl = reinterpret_cast<float4*>(plo + row * N);
  for (int i = threadIdx.x; i < n4; i += SS_THREADS) {
    const float4 v = src[i];
    float4 p, h, l;
    p.x = expf(v.x - m) * inv; p.y = expf(v.y - m) * inv; p.z = expf(v.z - m) * inv; p.w = expf(v.w - m) * inv;
    h.x = tf32_round(p.x); h.y = tf32_round(p.y); h.z = tf32_round(p.z); h.w = tf32_round(p.w);
    l.x = tf32_round(p.x - h.x); l.y = tf32_round(p.y - h.y); l.z = tf32_round(p.z - h.z); l.w = tf32_round(p.w - h.w);
    dh[i] = h;
    dl[i] = l;
  }
}

int softmax_split_tf32_impl(const void* s, long long rows, int N, void* phi, void* plo, cudaStream_t stream) {
  VTON_CHECK_ARG(rows > 0 && rows <= 0x7fffffffLL && N > 0 && N % 4 == 0, "softmax_split_tf32: bad shape rows=%lld N=%d", rows, N);
  VTON_CHECK_ARG((reinterpret_cast<uintptr_t>(s) & 15) == 0 && (reinterpret_cast<uintptr_t>(phi) & 15) == 0 &&
                     (reinterpret_cast<uintptr_t>(plo) & 15) == 0, "softmax_split_tf32: pointers must be 16-byte aligned");
  softmax_split_tf32_kernel<<<static_cast<unsigned>(rows), SS_THREADS, 0, stream>>>(static_cast<const float*>(s), N,
                                                                                   static_cast<float*>(phi), static_cast<float*>(plo));
  count_launch();
  VTON_CUDA(cudaGetLastError());
  return kOk;
}

}  // namespace vton
