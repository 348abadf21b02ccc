// Shared pieces of the wgmma GEMM / implicit-conv kernel (gemm.cu): the problem descriptor, the accumulator-row ->
// output-row mapping and the fused epilogue.
#pragma once
#include "common.cuh"

namespace vton {

struct GemmParams {
  __half* out;
  int ld_out;
  int M, N;  // output rows / accumulator columns (GEGLU: N = 2 * out columns)
  const __half* bias;
  const __half* bias_sc;
  const __half* residual;
  int ld_res;
  const __half* rowvec;  // per-sample row vector added after the bias rounding (time embedding), [B, ld_rowvec]
  int ld_rowvec;
  int rows_per_sample;
  int slabs_main;  // 64-wide K slabs accumulated into accumulator 0
  int slabs_sc;    // slabs accumulated into accumulator 1 (1x1 shortcut), 0 = none
  int sc_split;    // shortcut slabs taken from source 0 before switching to source 1
  // conv geometry
  int conv;
  int H, W, B;
  int bw, bh, bb;  // TMA box extent in x / y / batch (bw*bh*bb == 128)
  int tiles_x, tiles_y;
  int cin_slabs;  // Cin / 64
  int cout;       // rows per tap in the packed weight
  int n_tiles;
  int act_gelu;  // v = fp16(act(fp16(acc + bias))) before the later epilogue terms; 1 = erf-GELU (Resampler FeedForward, CLIP
                 // ViT-H / bigG MLPs), 2 = quick-GELU (CLIP ViT-L text MLP)
  int stride;    // conv: input pixel step per output pixel (1, or 2 = Downsample2D: the A map steps by 2 pixels per row)
  // fp32-output convolution (the VAE): out = acc + bias (+ residual), all fp32; `out` above is unused then
  float* out_f32;
  const float* bias_f32;
  const float* res_f32;
};

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int A_BYTES = BM * BK * 2;  // 16 KB

// Accumulator row r_local (0..127) of 128-row tile m_tile -> global output row (-1 = outside) and sample index.
__device__ __forceinline__ void map_row(const GemmParams& p, int m_tile, int r_local, long long* out_row, int* sample) {
  *out_row = -1;
  if (p.conv) {
    const int tx = m_tile % p.tiles_x;
    const int ty = (m_tile / p.tiles_x) % p.tiles_y;
    const int tb = m_tile / (p.tiles_x * p.tiles_y);
    const int lx = r_local % p.bw;
    const int ly = (r_local / p.bw) % p.bh;
    const int lb = r_local / (p.bw * p.bh);
    const int b = tb * p.bb + lb, y = ty * p.bh + ly, x = tx * p.bw + lx;
    if (b < p.B && y < p.H && x < p.W) *out_row = (static_cast<long long>(b) * p.H + y) * p.W + x;
    *sample = b;
  } else {
    const int m = m_tile * BM + r_local;
    if (m < p.M) *out_row = m;
    *sample = p.rows_per_sample > 0 ? m / p.rows_per_sample : 0;
  }
}

// Epilogue specialisation (compile time): which terms exist. EPI_RUNTIME keeps every term behind a runtime test of the
// GemmParams pointers.
enum : int { EPI_BIAS = 1, EPI_ROWVEC = 2, EPI_RES = 4, EPI_RUNTIME = 8 };

// erf-GELU with the Abramowitz-Stegun 7.1.26 rational/exponential form (|abs err| < 2e-7, far below the fp16 rounding
// that follows): ~16 instructions instead of erff's ~40.
__device__ __forceinline__ float gelu_erf_fast(float x) {
  const float ax = fabsf(x) * 0.70710678118654752f;
  const float t = __fdividef(1.0f, fmaf(0.3275911f, ax, 1.0f));
  float poly = fmaf(t, 1.061405429f, -1.453152027f);
  poly = fmaf(poly, t, 1.421413741f);
  poly = fmaf(poly, t, -0.284496736f);
  poly = fmaf(poly, t, 0.254829592f);
  poly *= t;
  float e;
  const float arg = -ax * ax * 1.4426950408889634f;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(arg));
  const float erf_abs = fmaf(-poly, e, 1.0f);
  const float erf_v = copysignf(erf_abs, x);
  return 0.5f * x * (1.0f + erf_v);
}

// chunk c of one accumulator row from the fp32 staging tile in shared memory: accumulator 0 into acc, the gate half /
// shortcut accumulator into acc2
template <int BN, bool GEGLU, int EPI>
__device__ __forceinline__ void epilogue_load(const GemmParams& p, const float* row, const float* row_sc, int c,
                                              uint32_t (&acc)[32], uint32_t (&acc2)[32]) {
#pragma unroll
  for (int i = 0; i < 32; i += 4) {
    const float4 v = *reinterpret_cast<const float4*>(row + c * 32 + i);
    acc[i] = __float_as_uint(v.x), acc[i + 1] = __float_as_uint(v.y), acc[i + 2] = __float_as_uint(v.z), acc[i + 3] = __float_as_uint(v.w);
  }
  const float* src2 = GEGLU ? row + BN / 2 : (((EPI & EPI_RUNTIME) && p.slabs_sc) ? row_sc : nullptr);
  if (src2 != nullptr) {
#pragma unroll
    for (int i = 0; i < 32; i += 4) {
      const float4 v = *reinterpret_cast<const float4*>(src2 + c * 32 + i);
      acc2[i] = __float_as_uint(v.x), acc2[i + 1] = __float_as_uint(v.y), acc2[i + 2] = __float_as_uint(v.z), acc2[i + 3] = __float_as_uint(v.w);
    }
  }
}

__device__ __forceinline__ void add_h8(float (&v)[8], const __half* src) {
  const uint4 u = *reinterpret_cast<const uint4*>(src);
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 a = unpack_h2(w[j]);
    v[2 * j] += a.x;
    v[2 * j + 1] += a.y;
  }
}
__device__ __forceinline__ void add_u4(float (&v)[8], const uint4 u) {   // v += u (8 halves)
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 a = unpack_h2(w[j]);
    v[2 * j] += a.x;
    v[2 * j + 1] += a.y;
  }
}
__device__ __forceinline__ void round_add_u4(float (&v)[8], const uint4 u) {   // v = fp16(v) + u (8 halves)
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 a = unpack_h2(w[j]);
    v[2 * j] = round_h(v[2 * j]) + a.x;
    v[2 * j + 1] = round_h(v[2 * j + 1]) + a.y;
  }
}
__device__ __forceinline__ void round_add_h8(float (&v)[8], const __half* src) {   // v = fp16(v) + src
  const uint4 u = *reinterpret_cast<const uint4*>(src);
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 a = unpack_h2(w[j]);
    v[2 * j] = round_h(v[2 * j]) + a.x;
    v[2 * j + 1] = round_h(v[2 * j + 1]) + a.y;
  }
}

// One 32-column chunk of the fused epilogue for one accumulator row: registers -> (bias, activation, temb, shortcut,
// residual with the reference's fp16 rounding points) -> 16 packed half2 words. Columns >= N of the last tile carry
// don't-care values (the sinks clip them).
template <int BN, bool GEGLU, int EPI>
__device__ __forceinline__ void epilogue_math(const GemmParams& p, int n_tile, long long out_row, int sample, int c,
                                              const uint32_t (&acc)[32], const uint32_t (&acc2)[32], uint32_t (&pk)[16],
                                              const uint4* res_pre = nullptr, const uint4* bias_pre = nullptr) {
  constexpr bool RT = (EPI & EPI_RUNTIME) != 0;
  const bool has_bias = RT ? (p.bias != nullptr) : ((EPI & EPI_BIAS) != 0);
  const bool has_rowvec = RT ? (p.rowvec != nullptr) : ((EPI & EPI_ROWVEC) != 0);
  const bool has_res = RT ? (p.residual != nullptr) : ((EPI & EPI_RES) != 0);
  const int n0 = n_tile * BN;
  const int out_n0 = GEGLU ? n_tile * (BN / 2) : n0;
  const int out_N = GEGLU ? p.N / 2 : p.N;
  // Rows outside the output (a conv box whose batch extent exceeds B, the ragged last M tile) carry a sample index past
  // the [B, ld_rowvec] time-embedding tensor: their values are never stored, so they must not read it either (found by
  // compute-sanitizer in round 2: a 16-byte read up to bb - B rows past the tensor).
  const __half* rowvec_row = (has_rowvec && out_row >= 0) ? p.rowvec + static_cast<long long>(sample) * p.ld_rowvec : nullptr;
  const __half* res_row = (has_res && out_row >= 0) ? p.residual + out_row * p.ld_res : nullptr;
#pragma unroll
  for (int g = 0; g < 4; ++g) {
    const int ncol = out_n0 + c * 32 + g * 8;  // output column of this 8-group
    const bool col_ok = ncol < out_N;
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = __uint_as_float(acc[g * 8 + j]);
    if (GEGLU) {
      const int bcol = n0 + c * 32 + g * 8;  // packed (interleaved) bias index of the value half
      float gt[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) gt[j] = __uint_as_float(acc2[g * 8 + j]);
      if (p.bias && col_ok) {
        add_h8(v, p.bias + bcol);
        add_h8(gt, p.bias + bcol + BN / 2);
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float hv = round_h(v[j]);
        const float gv = round_h(gt[j]);
        v[j] = hv * round_h(gelu_erf_fast(gv));  // fp16(h) * fp16(gelu(fp16(gate)))
      }
    } else {
      if (bias_pre != nullptr) {
        if (has_bias) add_u4(v, bias_pre[g]);   // prefetched by the caller (zeros past N)
      } else if (has_bias && col_ok) {
        add_h8(v, p.bias + ncol);
      }
      if (RT && p.act_gelu) {   // rare (Resampler FeedForward, CLIP MLPs): keep it rolled
#pragma unroll 1
        for (int j = 0; j < 8; ++j) {
          const float x = round_h(v[j]);
          // 1: erf-GELU; 2: quick-GELU x * sigmoid(1.702 x) (the CLIP ViT-L text encoder's activation)
          v[j] = p.act_gelu == 2 ? __fdividef(x, 1.0f + __expf(-1.702f * x)) : gelu_erf_fast(x);
        }
      }
      if (has_rowvec && col_ok && rowvec_row != nullptr) round_add_h8(v, rowvec_row + ncol);
      if (RT && p.slabs_sc) {
        float s[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) s[j] = __uint_as_float(acc2[g * 8 + j]);
        if (p.bias_sc && col_ok) add_h8(s, p.bias_sc + ncol);
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = round_h(s[j]) + round_h(v[j]);
      }
      if (res_pre != nullptr) {   // residual row segment prefetched by the caller (zeros where it does not apply)
        if (has_res) round_add_u4(v, res_pre[g]);
      } else if (has_res && col_ok && res_row != nullptr) {
        round_add_h8(v, res_row + ncol);
      }
    }
    pk[g * 4 + 0] = pack_h2(v[0], v[1]);
    pk[g * 4 + 1] = pack_h2(v[2], v[3]);
    pk[g * 4 + 2] = pack_h2(v[4], v[5]);
    pk[g * 4 + 3] = pack_h2(v[6], v[7]);
  }
}

// Registers -> global, each thread writes the 32-column chunks c = c_first, c_first + c_step, ... of its own row.
template <int BN, bool GEGLU>
__device__ __forceinline__ void epilogue_store(const GemmParams& p, const float* row, const float* row_sc, int n_tile,
                                               long long out_row, int sample, int c_first, int c_step) {
  constexpr int OUT_COLS = GEGLU ? BN / 2 : BN;
  const int out_n0 = GEGLU ? n_tile * (BN / 2) : n_tile * BN;
  const int out_N = GEGLU ? p.N / 2 : p.N;
#pragma unroll 1
  for (int c = c_first; c < OUT_COLS / 32; c += c_step) {
    if (out_row < 0 || out_n0 + c * 32 >= out_N) continue;
    uint32_t acc[32], acc2[32];
    uint32_t pk[16];
    epilogue_load<BN, GEGLU, EPI_RUNTIME>(p, row, row_sc, c, acc, acc2);
    epilogue_math<BN, GEGLU, EPI_RUNTIME>(p, n_tile, out_row, sample, c, acc, acc2, pk);
#pragma unroll
    for (int g = 0; g < 4; ++g) {
      const int ncol = out_n0 + c * 32 + g * 8;
      if (ncol >= out_N) continue;
      *reinterpret_cast<uint4*>(p.out + out_row * p.ld_out + ncol) =
          make_uint4(pk[g * 4], pk[g * 4 + 1], pk[g * 4 + 2], pk[g * 4 + 3]);
    }
  }
}

// ----------------------------------------------------------------------------------------------
// TMA stores (smem -> global, bulk async group); out-of-bounds box elements are clipped by the hardware.
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, uint32_t src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(m)), "r"(src), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* m, uint32_t src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(m)), "r"(src), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait_all() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

}  // namespace vton
