// Shared pieces of the wgmma GEMM / implicit-conv kernel (gemm.cu): the problem descriptor, the accumulator-row ->
// output-row mapping and the fused epilogue that runs on the accumulator fragments.
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
  int total_tiles;  // m tiles x n_tiles; tile t is (m_tile, n_tile) = (t / n_tiles, t % n_tiles)
  int act_gelu;  // v = fp16(act(fp16(acc + bias))) before the later epilogue terms; 1 = erf-GELU (Resampler FeedForward, CLIP
                 // ViT-H / bigG MLPs), 2 = quick-GELU (CLIP ViT-L text MLP)
  int stride;    // conv: input pixel step per output pixel (1, or 2 = Downsample2D: the A map steps by 2 pixels per row)
  // fp32-output convolution (the VAE): out = acc + bias (+ residual), all fp32; `out` above is unused then
  float* out_f32;
  const float* bias_f32;
  const float* res_f32;
  // e4m3 operands (the FP8 linears): acc is scaled to (acc * a_scale[m]) * w_scale[n] before the fp16 epilogue
  const float* a_scale;
  const float* w_scale;
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

// Transposes a 4x4 block of words across a quad (lanes 4k .. 4k+3, q = lane & 3): afterwards w[j] of lane q is what
// lane j held in w[q]. Two exchange rounds (lane bit 0 with index bit 0, then bit 1 with bit 1). Every lane of the warp
// must call it.
__device__ __forceinline__ void quad_transpose(uint32_t (&w)[4], int q) {
  {
    const bool odd = (q & 1) != 0;
    const uint32_t s0 = __shfl_xor_sync(0xffffffffu, odd ? w[0] : w[1], 1);
    const uint32_t s1 = __shfl_xor_sync(0xffffffffu, odd ? w[2] : w[3], 1);
    if (odd) w[0] = s0, w[2] = s1;
    else w[1] = s0, w[3] = s1;
  }
  {
    const bool hi = (q & 2) != 0;
    const uint32_t s0 = __shfl_xor_sync(0xffffffffu, hi ? w[0] : w[2], 2);
    const uint32_t s1 = __shfl_xor_sync(0xffffffffu, hi ? w[1] : w[3], 2);
    if (hi) w[0] = s0, w[1] = s1;
    else w[2] = s0, w[3] = s1;
  }
}

__device__ __forceinline__ float2 ldg_h2(const __half* src) {
  return unpack_h2(__ldg(reinterpret_cast<const uint32_t*>(src)));
}

__device__ __forceinline__ void st_shared_v4(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ uint4 ld_shared_v4(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr) : "memory");
  return v;
}
// Bulk copy (no tensor map) of `bytes` (a multiple of 16, both addresses 16-byte aligned) from global to shared memory,
// completing as transaction bytes on the mbarrier `bar`.
__device__ __forceinline__ void bulk_copy_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(reinterpret_cast<uint64_t>(src)), "r"(bytes), "r"(bar) : "memory");
}

// The fp16 tile between the two halves of the epilogue: 128 rows x OUT_COLS halves in shared memory, row-major in
// 16-byte chunks, so that a residual row lands in it with one bulk copy. The consumers read and write it a quad at a
// time (4 consecutive chunks of rows r and r + 1 in one 8-lane phase: conflict-free with 20 chunks per row, two-way
// where a row holds a multiple of 8 chunks) and the store warps read 8 consecutive chunks of a row at a time.
template <int BN, bool GEGLU>
struct StagingTile {
  static constexpr int OUT_COLS = GEGLU ? BN / 2 : BN;
  static constexpr int CHUNKS_PER_ROW = OUT_COLS / 8;
  static constexpr int BYTES = BM * OUT_COLS * 2;
  __device__ static __forceinline__ uint32_t offset(int r, int chunk) {
    return static_cast<uint32_t>(r * CHUNKS_PER_ROW + chunk) * 16u;
  }
};

// Register half of the fp16 epilogue of one 128 x BN tile, straight from the wgmma accumulator fragment. The thread
// holds rows r_local and r_local + 8 of the tile and, of every 8-column group i, columns 8i + 2q + {0,1} in
// acc[4i .. 4i+3] (q = lane & 3); acc_sc (the shortcut accumulator) has the same layout, and the GEGLU gate of column c
// is column c + BN/2 of the same thread. Per element, with the reference's fp16 rounding points:
//   v = fp16(acc + bias); v = act(v); v = fp16(v + temb[sample]); v = fp16(fp16(acc_sc + bias_sc) + v); v = fp16(v + res)
//   GEGLU: v = fp16(h) * fp16(gelu(fp16(g)))
// Bias and time embedding are read in the fragment shape (one half2 per column pair, the bias once for both rows). The
// packed half2 words of four 8-groups are then transposed across the quad, so each lane owns 8 contiguous columns of one
// row; the residual of those 8 columns, which the store warps have copied into the staging tile during the K loop, is
// added in place and the result written back, 16 bytes per lane.
//
// Only eight consumer warps share an SM, so a global load whose value is needed at once costs its whole latency.
// begin() therefore runs before the tile's K loop: it maps the rows and issues the loads of the tile's bias words,
// which land while the tensor cores work.
// SCALED (e4m3 operands): every accumulator is first scaled to (acc * a_scale[row]) * w_scale[col] in fp32; the row
// scales are loaded in begin(), the column scales of an 8-group where it is scaled (L1 hits after the first row; BN/4
// more registers held across the K loop would not fit at BN = 256). Everything after that is the fp16 epilogue unchanged.
template <int BN, bool GEGLU, bool SC, bool SCALED = false>
struct EpilogueF16 {
  using Staging = StagingTile<BN, GEGLU>;
  static constexpr int OUT_COLS = Staging::OUT_COLS;
  static constexpr int CHUNKS = OUT_COLS / 32;
  static constexpr bool HAS_RES = !GEGLU && !SC;   // a residual comes with neither GEGLU nor a fused shortcut

  int q, n0, out_n0, out_N;
  long long out_row[2];
  int sample[2];
  uint32_t bias[BN / 8];              // half2 of columns n0 + 8i + 2q + {0,1} (GEGLU: value and gate halves alike)
  uint32_t bias_sc[SC ? BN / 8 : 1];
  float a_scale[SCALED ? 2 : 1];      // row scales of rows r_local and r_local + 8

  __device__ __forceinline__ void begin(const GemmParams& p, int m_tile, int n_tile, int r_local) {
    q = threadIdx.x & 3;
    n0 = n_tile * BN;
    out_n0 = GEGLU ? n_tile * (BN / 2) : n0;
    out_N = GEGLU ? p.N / 2 : p.N;
#pragma unroll
    for (int h = 0; h < 2; ++h) map_row(p, m_tile, r_local + 8 * h, &out_row[h], &sample[h]);
    if constexpr (SCALED) {
#pragma unroll
      for (int h = 0; h < 2; ++h) a_scale[h] = out_row[h] >= 0 ? __ldg(p.a_scale + out_row[h]) : 0.0f;
    }
#pragma unroll
    for (int i = 0; i < BN / 8; ++i) {
      const bool ok = n0 + i * 8 < p.N;
      bias[i] = (p.bias && ok) ? __ldg(reinterpret_cast<const uint32_t*>(p.bias + n0 + i * 8 + 2 * q)) : 0u;
      if (SC) bias_sc[i] = (p.bias_sc && ok) ? __ldg(reinterpret_cast<const uint32_t*>(p.bias_sc + n0 + i * 8 + 2 * q)) : 0u;
    }
  }

  // Writes the tile's fp16 output to the staging tile at shared address `staging`, which holds the tile's residual.
  // ACT / ROWVEC: whether the activation / time-embedding code is compiled in at all. The caller picks the variant once
  // per tile (act_gelu != 0 needs ACT, a rowvec needs ROWVEC), so the common path is straight-line code of a few
  // instructions per column pair instead of a walk over rare branches inlined for every pair, which made the epilogue
  // instruction-fetch bound.
  template <bool ACT, bool ROWVEC>
  __device__ __forceinline__ void stage(const GemmParams& p, const float (&acc)[BN / 2], const float (&acc_sc)[BN / 2],
                                        int r_local, uint32_t staging) {
    // Rows outside the output (a conv box whose batch extent exceeds B, the ragged last M tile) carry a sample index past
    // the [B, ld_rowvec] time-embedding tensor: their values are never stored, so they must not read it either.
    const __half* rowvec_row[2];
#pragma unroll
    for (int h = 0; h < 2; ++h)
      rowvec_row[h] = (ROWVEC && p.rowvec && out_row[h] >= 0)
                          ? p.rowvec + static_cast<long long>(sample[h]) * p.ld_rowvec
                          : nullptr;
#pragma unroll
    for (int c = 0; c < CHUNKS; ++c) {
      if (out_n0 + c * 32 >= out_N) break;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        uint32_t w[4];
#pragma unroll
        for (int g = 0; g < 4; ++g) {
          const int i = 4 * c + g;
          const bool col_ok = out_n0 + i * 8 < out_N;
          float v0 = acc[4 * i + 2 * h], v1 = acc[4 * i + 2 * h + 1];
          float2 w_scale[GEGLU ? 2 : 1];   // column scales of the 8-group (GEGLU: and of its gate columns)
          if constexpr (SCALED) {
#pragma unroll
            for (int e = 0; e < (GEGLU ? 2 : 1); ++e) {
              const int col = n0 + (i + e * (BN / 16)) * 8 + 2 * q;
              w_scale[e] = col < p.N ? __ldg(reinterpret_cast<const float2*>(p.w_scale + col)) : make_float2(0.f, 0.f);
            }
            // __fmul_rn: the scaled product is rounded to fp32 before the bias add (no FMA contraction)
            v0 = __fmul_rn(__fmul_rn(v0, a_scale[h]), w_scale[0].x);
            v1 = __fmul_rn(__fmul_rn(v1, a_scale[h]), w_scale[0].y);
          }
          if (GEGLU) {   // packed (interleaved) bias: value half at n0 + 8i, gate half BN/2 further
            float g0 = acc[4 * (i + BN / 16) + 2 * h], g1 = acc[4 * (i + BN / 16) + 2 * h + 1];
            if constexpr (SCALED) {
              g0 = __fmul_rn(__fmul_rn(g0, a_scale[h]), w_scale[GEGLU ? 1 : 0].x);
              g1 = __fmul_rn(__fmul_rn(g1, a_scale[h]), w_scale[GEGLU ? 1 : 0].y);
            }
            if (p.bias && col_ok) {
              const float2 b = unpack_h2(bias[i]), bg = unpack_h2(bias[i + BN / 16]);
              v0 += b.x, v1 += b.y, g0 += bg.x, g1 += bg.y;
            }
            v0 = round_h(v0) * round_h(gelu_erf_fast(round_h(g0)));   // fp16(h) * fp16(gelu(fp16(gate)))
            v1 = round_h(v1) * round_h(gelu_erf_fast(round_h(g1)));
          } else {
            if (p.bias && col_ok) {
              const float2 b = unpack_h2(bias[i]);
              v0 += b.x, v1 += b.y;
            }
            if (ACT && p.act_gelu) {   // rare (Resampler FeedForward, CLIP MLPs)
              const float x0 = round_h(v0), x1 = round_h(v1);
              // 1: erf-GELU; 2: quick-GELU x * sigmoid(1.702 x) (the CLIP ViT-L text encoder's activation)
              v0 = p.act_gelu == 2 ? __fdividef(x0, 1.0f + __expf(-1.702f * x0)) : gelu_erf_fast(x0);
              v1 = p.act_gelu == 2 ? __fdividef(x1, 1.0f + __expf(-1.702f * x1)) : gelu_erf_fast(x1);
            }
            if (ROWVEC && rowvec_row[h] != nullptr && col_ok) {
              const float2 t = ldg_h2(rowvec_row[h] + n0 + i * 8 + 2 * q);
              v0 = round_h(v0) + t.x, v1 = round_h(v1) + t.y;
            }
            if (SC) {
              float s0 = acc_sc[4 * i + 2 * h], s1 = acc_sc[4 * i + 2 * h + 1];
              if (p.bias_sc && col_ok) {
                const float2 b = unpack_h2(bias_sc[i]);
                s0 += b.x, s1 += b.y;
              }
              v0 = round_h(s0) + round_h(v0), v1 = round_h(s1) + round_h(v1);
            }
          }
          w[g] = pack_h2(v0, v1);
        }
        quad_transpose(w, q);
        const uint32_t slot = staging + Staging::offset(r_local + 8 * h, 4 * c + q);
        if (HAS_RES && p.residual) {   // rows and columns outside the output hold stale words here: never stored
          const uint4 u = ld_shared_v4(slot);
          const uint32_t r[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
          for (int j = 0; j < 4; ++j) {   // w already holds fp16(v)
            const float2 a = unpack_h2(w[j]), d = unpack_h2(r[j]);
            w[j] = pack_h2(a.x + d.x, a.y + d.y);
          }
        }
        st_shared_v4(slot, w[0], w[1], w[2], w[3]);
      }
    }
  }
};

// Memory half of the fp16 epilogue, on the 96 threads of warps 9..11 (e = 0..95), which walk the consumers' tile
// schedule. For tile j they map its rows into a shared row table (double-buffered, so one named barrier per tile orders
// its writes and reads). Once all of them are done reading tile j - 1 out of the staging tile, they bulk-copy tile j's
// residual rows into it and arrive on `ready`, which completes when the copies have landed: the residual travels while
// tile j's K loop runs and costs no registers, and the consumers add it as they stage the tile. When the consumers
// have staged it (`staged`), the store warps store it 16 bytes at a time, 8 threads covering 128 contiguous bytes of a
// row. A CTA's last tile has no K loop after it to hide its store behind, so the consumers join in and it is stored by
// all 352 threads. Column groups at or past N and rows outside the output (a conv box whose batch extent exceeds B, the
// ragged last M tile) are neither copied nor stored.
template <int BN, bool GEGLU>
struct EpilogueStore {
  using Staging = StagingTile<BN, GEGLU>;
  static constexpr int THREADS = 96;
  static constexpr int CPR = Staging::CHUNKS_PER_ROW;
  static constexpr int UNITS = BM * CPR;   // 16-byte chunks per tile

  // Thread t of n stores chunks t, t + n, ... of the staged tile; rows: the tile's output rows (-1 = outside).
  __device__ static __forceinline__ void store(const GemmParams& p, const uint8_t* staging_ptr, const int* rows, int out_n0,
                                               int out_N, int t, int n) {
#pragma unroll 4
    for (int u = t; u < UNITS; u += n) {
      const int r = u / CPR, chunk = u % CPR;
      const int row = rows[r];
      const int col = out_n0 + chunk * 8;
      if (row >= 0 && col < out_N)
        *reinterpret_cast<uint4*>(p.out + static_cast<long long>(row) * p.ld_out + col) =
            *reinterpret_cast<const uint4*>(staging_ptr + Staging::offset(r, chunk));
    }
  }

  // The consumers' share (thread t of 256) of storing `tile`, the CTA's last, once both warpgroups have staged it.
  __device__ static __forceinline__ void help_store_last(const GemmParams& p, int tile, const uint8_t* staging_ptr,
                                                         const int* row_table, uint32_t staged_bar, int t) {
    const int j = (tile - blockIdx.x) / gridDim.x;
    mbar_wait(staged_bar, j & 1);
    store(p, staging_ptr, row_table + (j & 1) * BM, (tile % p.n_tiles) * Staging::OUT_COLS, GEGLU ? p.N / 2 : p.N,
          THREADS + t, THREADS + 256);
  }

  __device__ static __forceinline__ void run(const GemmParams& p, uint32_t staging, const uint8_t* staging_ptr,
                                             int* row_table, uint32_t staged_bar, uint32_t ready_bar, int e) {
    const int out_N = GEGLU ? p.N / 2 : p.N;
    int j = 0;
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x, ++j) {
      const int m_tile = tile / p.n_tiles;
      const int out_n0 = (tile % p.n_tiles) * Staging::OUT_COLS;
      int* rows = row_table + (j & 1) * BM;
      for (int r = e; r < BM; r += THREADS) {
        long long out_row;
        int sample;
        map_row(p, m_tile, r, &out_row, &sample);
        rows[r] = static_cast<int>(out_row);
      }
      named_bar_sync(1, THREADS);   // the row table is complete and nobody reads the staging tile any more
      if (p.residual) {
        fence_proxy_async_smem();   // the staging tile's generic reads before the copies' writes
        const uint32_t row_bytes = (out_N - out_n0 < Staging::OUT_COLS ? out_N - out_n0 : Staging::OUT_COLS) * 2u;
        uint32_t bytes = 0;
        for (int r = e; r < BM; r += THREADS) bytes += rows[r] >= 0 ? row_bytes : 0u;
        mbar_expect_tx(ready_bar, bytes);   // arrives, and expects this thread's copies
        for (int r = e; r < BM; r += THREADS) {
          if (rows[r] >= 0)
            bulk_copy_g2s(staging + Staging::offset(r, 0), p.residual + static_cast<long long>(rows[r]) * p.ld_res + out_n0,
                          row_bytes, ready_bar);
        }
      } else {
        mbar_arrive(ready_bar);
      }
      mbar_wait(staged_bar, j & 1);
      const bool last = tile + static_cast<int>(gridDim.x) >= p.total_tiles;
      store(p, staging_ptr, rows, out_n0, out_N, e, last ? THREADS + 256 : THREADS);
    }
  }
};

// fp32-output epilogue (the VAE convolutions) from the same fragment: out = acc + bias (+ residual), all fp32. A thread
// stores float2 pairs, a quad one 32-byte sector per row.
template <int BN>
__device__ __forceinline__ void epilogue_f32(const GemmParams& p, int m_tile, int n_tile, int r_local,
                                             const float (&acc)[BN / 2]) {
  const int q = threadIdx.x & 3;
  const int n0 = n_tile * BN;
  long long out_row[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    int sample;
    map_row(p, m_tile, r_local + 8 * h, &out_row[h], &sample);
  }
#pragma unroll
  for (int i = 0; i < BN / 8; ++i) {
    if (n0 + i * 8 >= p.N) break;
    const int ncol = n0 + i * 8 + 2 * q;
    float2 b = make_float2(0.0f, 0.0f);
    if (p.bias_f32 != nullptr) b = __ldg(reinterpret_cast<const float2*>(p.bias_f32 + ncol));
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (out_row[h] < 0) continue;
      float2 v = make_float2(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]);
      if (p.bias_f32 != nullptr) v.x += b.x, v.y += b.y;
      if (p.res_f32 != nullptr) {   // after the bias, like torch's `x + conv(h)`
        const float2 r = __ldg(reinterpret_cast<const float2*>(p.res_f32 + out_row[h] * p.N + ncol));
        v.x += r.x, v.y += r.y;
      }
      *reinterpret_cast<float2*>(p.out_f32 + out_row[h] * p.N + ncol) = v;
    }
  }
}

}  // namespace vton
