// Flash-style attention on wgmma (sm_90a) for every attention of the project, one kernel:
//
//   * attn1 of src/attentionhacked_tryon.py:334-348 + ip_adapter/attention_processor.py:238-262 — self-attention whose
//     keys/values are [self tokens ; garment tokens]. Segment 0 = this sample's K/V, segment 1 = the cached garment K/V
//     of sample (b - kv1_off) % kv1_count (+ a device step base), or of the row a device table names per sample (a
//     pool of hoisted garment K/V shared by slots at different steps); the torch.cat never happens. Query rows are the
//     N self tokens only (the reference computes and discards the Ng garment query rows).
//   * CFG-uncond samples (b < kv1_off) see ZERO garment features (src/tryon_pipeline.py:1796): K=V=0, so each of the N1
//     tokens adds exp(0 - m) to the softmax denominator and nothing to the numerator. Closed form, no KV traffic.
//   * attn2 (ip_adapter/attention_processor.py:1943-1995, IPAttnProcessor2_0): the text softmax and the IP-token softmax
//     in one launch (segment 0 = text, segment 1 = IP tokens, flash_kernel<4, true>): out = fp16(fp16(O_t) + fp16(ip_scale * fp16(O_i))),
//     the reference's rounding points (cross_attn_impl).
//   * the CLIP towers' encoder self-attention (heads of 64 or 80, optional causal mask; enc_attn_impl).
//
// Head dimension D = 16..96 in steps of 16: a head's columns are fetched as R = ceil(D/64) 128B-swizzled regions of 64
// columns straight out of the projection buffer (the second region runs into the next head's columns, which are never
// used: Q K^T issues exactly D/16 k-steps and the extra output columns of P V are never stored).
//
// One CTA = one (sample, head, 128-query tile), three warpgroups (FA3 layout):
//   * warpgroup 2 is the producer: it gives up registers (setmaxnreg.dec) and one thread issues every TMA load: Q once,
//     then the K/V tiles of 128 keys of segment 0 and segment 1 through a ring of FlashSmem::STAGES stages (3 for D <= 64,
//     2 above: what 227 KB of shared memory holds);
//   * warpgroups 0 and 1 are the consumers, 64 query rows each (setmaxnreg.inc). Per K/V tile j a consumer computes
//     S = Q K_j^T (m64n128k16, both operands in shared memory) into registers, runs the online softmax there (a row lives
//     in the 4 threads of a quad), converts P to fp16 A fragments in registers and accumulates O += P V_j (m64nDNk16,
//     V as the MN-major B operand).
// Overlap: a consumer issues S_{j+1} = Q K_{j+1}^T together with O += P_j V_j and runs the softmax of tile j+1 while
// P_j V_j is still in the tensor cores (wgmma_wait<1>); and the two consumers issue their MMAs in turns ordered by two
// named barriers (ping-pong), so one warpgroup's softmax runs while the other's MMAs do. The arithmetic of every
// element is that of the plain loop (O is rescaled by alpha_j before P_j V_j is added), so the overlap changes no bit.
// Full key tiles take an unmasked softmax; only the last, partial tile of a segment and causal tiles test each key.
// Samples with a real segment 1 (b >= kv1_off, the longest CTAs) are scheduled before the zero-K/V samples.
// With IP (the decoupled text + IP-token cross-attention), segment 1 has its own softmax and the CTA stores
// fp16(fp16(O_0) + fp16(out_scale * fp16(O_1))).
#include <cuda_fp8.h>

#include <algorithm>

#include "common.cuh"
#include "host.h"
#include "wgmma.cuh"

namespace vton {

struct FlashParams {
  __half* out;
  int ld_out;
  int B, H, Nq, N0, N1;
  int D;          // head dimension: head h occupies columns [h*D, h*D + D)
  int kv1_off;    // segment-1 sample index = (b - kv1_off) % kv1_count; negative => zero K/V closed form
  int kv1_count;  // segment-1 sample index is taken modulo this count (with kv1_rows: B1, the rows that exist)
  const int* kv1_base;  // optional device scalar added to the segment-1 sample index (hoisted per-step K/V)
  const int* kv1_rows;  // optional device table: segment-1 sample index = kv1_rows[b - kv1_off] (negative => zero K/V);
                        // replaces the modulo and kv1_base (per-slot rows of a pool of hoisted K/V)
  int causal;    // key j visible to query i iff j <= i (segment 0 only)
  float scale_log2;
  int accumulate;   // out = old + fp16(out_scale * fp16(o)) instead of out = fp16(o)
  float out_scale;
};

constexpr int FA_REGION = 128 * 128;  // 128 rows x 64 halves
constexpr int FA_THREADS = 384;       // consumer warpgroups 0 and 1, producer warpgroup 2
constexpr int FA_PRODUCER_REGS = 40;  // 128 * 40 + 256 * 232 = 64512 <= 65536 registers per SM
constexpr int FA_CONSUMER_REGS = 232;
constexpr uint32_t FA_BAR_TURN = 1;   // named barriers FA_BAR_TURN + wg: consumer wg may issue its MMAs (0 = __syncthreads)
constexpr uint32_t FA_BAR_CVT = 3;    // KV8: the converting warps 9-11 have written a stage's fp16 K/V
constexpr int FA_CVT_THREADS = 96;

// KV8: per stage, a staging area for a segment-1 tile in the FP8 garment K/V format (e4m3 K and V, 64 B x 128 rows
// each, then the 128 K and 128 V exponents), and one more mbarrier per stage (stg_full)
template <int R, bool KV8 = false>
struct FlashSmem {
  static constexpr int STAGES = R == 1 ? 3 : 2;
  static constexpr int OFF_Q = 0;
  static constexpr int OFF_K = OFF_Q + R * FA_REGION;
  static constexpr int OFF_V = OFF_K + STAGES * R * FA_REGION;
  static constexpr int STG_Q = 128 * 64;                       // one e4m3 tile
  static constexpr int STG_BYTES = KV8 ? 2 * STG_Q + 2 * 128 : 0;
  static constexpr int OFF_STG = OFF_V + STAGES * R * FA_REGION;
  static constexpr int OFF_BAR = OFF_STG + STAGES * STG_BYTES;
  static constexpr int TOTAL = OFF_BAR + (KV8 ? 128 : 64) + 1024;
};

__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// The FP8 garment K/V format (INTEGRATION.md, "FP8 garment K/V"): x = fp16(float(q) * 2^e) with q e4m3 and e one int8
// per (token, 64-column group). fp16(2^e) for e in [-24, 8] (subnormal below -14).
__device__ __forceinline__ uint32_t kv8_scale_h2(int e) {
  const uint32_t hb = e >= -14 ? static_cast<uint32_t>(e + 15) << 10 : 1u << (e + 24);
  return hb | (hb << 16);
}
// Two e4m3 codes (low byte first) -> fp16x2, times fp16(2^e) in one rounding: the rule's bits, since both factors are
// exact fp16 numbers
__device__ __forceinline__ uint32_t kv8_dequant2(uint32_t codes, uint32_t scale_h2) {
  const __half2_raw r = __nv_cvt_fp8x2_to_halfraw2(static_cast<__nv_fp8x2_storage_t>(codes & 0xffffu), __NV_E4M3);
  __half2 v(r);
  const __half2 s = *reinterpret_cast<const __half2*>(&scale_h2);
  v = __hmul2_rn(v, s);
  return *reinterpret_cast<uint32_t*>(&v);
}

// KS: Q K^T k-steps (D / 16); IP: segment 1 has a softmax of its own (the text + IP-token cross-attention, D = 64);
// R: 64-column regions per head; DN: P V tile width (64 for D <= 64, 96 otherwise). D > 64 (the CLIP image tower)
// and IP do not overlap a warpgroup's softmax with its own P V: S, P and a 96-wide O (or O and the kept fp16 O_0) do not
// fit the registers together.
// KV8 (D = 64 without IP only): segment 1 is in the FP8 garment K/V format. The TMA thread loads a segment-1 tile's e4m3
// K / V and exponents into the stage's staging area (stg_full), and the producer warpgroup's warps 9-11 write it as
// fp16 into the stage's 128B-swizzled K / V slots, then arrive on kv_full: the consumers read what they read for fp16.
template <int KS, bool IP, int R, int DN, bool KV8>
__device__ __forceinline__ void flash_body(const CUtensorMap* tmQ, const CUtensorMap* tmK0, const CUtensorMap* tmV0,
                                           const CUtensorMap* tmK1, const CUtensorMap* tmV1, const CUtensorMap* tmE,
                                           const FlashParams p) {
  static_assert(!KV8 || (KS == 4 && !IP && R == 1 && DN == 64), "the FP8 segment 1 is for D = 64 without IP");
  using SM = FlashSmem<R, KV8>;
  constexpr int ST = SM::STAGES;
  constexpr bool OVERLAP = DN == 64 && !IP;   // IP runs two tiles, one per softmax: nothing to overlap
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bar_base = smem_base + SM::OFF_BAR;
  const uint32_t q_full = bar_base;
  auto kv_full = [&](int s) { return bar_base + 8u * (1 + s); };
  auto kv_empty = [&](int s) { return bar_base + 8u * (1 + ST + s); };
  auto stg_full = [&](int s) { return bar_base + 8u * (1 + 2 * ST + s); };   // KV8 only

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = threadIdx.x >> 7;
  const int q_tile = blockIdx.x;
  const int h = blockIdx.y;
  // heaviest first: the samples that read a segment 1 (b >= kv1_off) get the lowest block indices
  int b = blockIdx.z;
  if (p.N1 > 0 && p.kv1_off > 0 && p.kv1_off < p.B) {
    b += p.kv1_off;
    if (b >= p.B) b -= p.B;
  }

  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    for (int s = 0; s < ST; ++s) {
      mbar_init(kv_full(s), 1);
      mbar_init(kv_empty(s), 2);   // one arrival per consumer warpgroup
      if constexpr (KV8) mbar_init(stg_full(s), 1);
    }
    fence_barrier_init();
  }
  if (threadIdx.x == 256) {
    tma_prefetch_desc(tmQ);
    tma_prefetch_desc(tmK0);
    tma_prefetch_desc(tmV0);
    if (p.N1 > 0) {
      tma_prefetch_desc(tmK1);
      tma_prefetch_desc(tmV1);
      if constexpr (KV8) tma_prefetch_desc(tmE);
    }
  }
  // Programmatic dependent launch: Q/K/V (and kv1_base / kv1_rows) are written by the previous kernels of the stream
  pdl_wait();
  __syncthreads();
  pdl_launch_dependents();

  const int tiles0 = (p.N0 + 127) >> 7;
  int idx1 = -1;
  if (p.N1 > 0) {
    idx1 = b - p.kv1_off;
    if (idx1 >= 0 && p.kv1_rows) {
      idx1 = p.kv1_rows[idx1];
      if (idx1 >= p.kv1_count) idx1 = -1;   // rows outside [0, B1) read nothing: the zero-K/V closed form
    } else if (idx1 >= 0) {
      idx1 = idx1 % p.kv1_count + (p.kv1_base ? *p.kv1_base : 0);
    }
  }
  const bool zero_kv = (p.N1 > 0) && (idx1 < 0);
  const int tiles1 = (p.N1 > 0 && idx1 >= 0) ? ((p.N1 + 127) >> 7) : 0;
  // causal: key tiles entirely after the last query row of this CTA contribute nothing
  const int total = p.causal ? min(tiles0, q_tile + 1) : tiles0 + tiles1;

  // ===================== producer =====================
  if (wg == 2) {
    setmaxnreg_dec<FA_PRODUCER_REGS>();
    if (threadIdx.x == 256) {
      mbar_expect_tx(q_full, R * FA_REGION);
#pragma unroll
      for (int r = 0; r < R; ++r)
        tma_load_3d(smem_base + SM::OFF_Q + r * FA_REGION, tmQ, q_full, h * p.D + r * 64, q_tile * 128, b);
      // K/V tile j into stage j % ST, once both consumers have released the stage's previous tile
      for (int j = 0; j < total; ++j) {
        const int stage = j % ST;
        if (j >= ST) mbar_wait(kv_empty(stage), ((j / ST) - 1) & 1);
        if constexpr (KV8) {
          if (j >= tiles0) {   // e4m3 K, V and their exponents (K group h, V group H + h) into the staging area
            const uint32_t stg = smem_base + SM::OFF_STG + stage * SM::STG_BYTES;
            const int key0 = (j - tiles0) * 128;
            mbar_expect_tx(stg_full(stage), SM::STG_BYTES);
            tma_load_3d(stg, tmK1, stg_full(stage), h * 64, key0, idx1);
            tma_load_3d(stg + SM::STG_Q, tmV1, stg_full(stage), h * 64, key0, idx1);
            tma_load_3d(stg + 2 * SM::STG_Q, tmE, stg_full(stage), key0, h, idx1);
            tma_load_3d(stg + 2 * SM::STG_Q + 128, tmE, stg_full(stage), key0, p.H + h, idx1);
            continue;
          }
        }
        mbar_expect_tx(kv_full(stage), 2 * R * FA_REGION);
#pragma unroll
        for (int r = 0; r < R; ++r) {
          const uint32_t kdst = smem_base + SM::OFF_K + (stage * R + r) * FA_REGION;
          const uint32_t vdst = smem_base + SM::OFF_V + (stage * R + r) * FA_REGION;
          const int col = h * p.D + r * 64;
          if (j < tiles0) {
            tma_load_3d(kdst, tmK0, kv_full(stage), col, j * 128, b);
            tma_load_3d(vdst, tmV0, kv_full(stage), col, j * 128, b);
          } else {
            tma_load_3d(kdst, tmK1, kv_full(stage), col, (j - tiles0) * 128, idx1);
            tma_load_3d(vdst, tmV1, kv_full(stage), col, (j - tiles0) * 128, idx1);
          }
        }
      }
    } else if constexpr (KV8) {
      if (warp >= 9) {
        // Warps 9-11 turn each staged segment-1 tile into fp16: 2 x 128 rows x 8 chunks of 16 B, chunk c of row r at
        // byte r * 128 + ((c ^ (r & 7)) << 4) of the slot (what a SWIZZLE_128B TMA load writes). The staging area of
        // stage s is refilled only after both consumers released the slot (kv_empty), which is after this arrival.
        const int t = threadIdx.x - 288;
        for (int j = tiles0; j < total; ++j) {
          const int stage = j % ST;
          mbar_wait(stg_full(stage), ((j - tiles0) / ST) & 1);
          const uint32_t stg = smem_base + SM::OFF_STG + stage * SM::STG_BYTES;
#pragma unroll 1   // 40 registers after setmaxnreg.dec: an unrolled loop spills
          for (int c = t; c < 2 * 128 * 8; c += FA_CVT_THREADS) {
            const int kv = c >> 10, r = (c >> 3) & 127, ch = c & 7;
            uint32_t lo, hi;
            int e;
            asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(lo), "=r"(hi) : "r"(stg + kv * SM::STG_Q + r * 64 + ch * 8));
            asm volatile("ld.shared.s8 %0, [%1];" : "=r"(e) : "r"(stg + 2 * SM::STG_Q + kv * 128 + r));
            const uint32_t sc = kv8_scale_h2(e);
            const uint32_t dst = smem_base + (kv ? SM::OFF_V : SM::OFF_K) + stage * FA_REGION + r * 128 + ((ch ^ (r & 7)) << 4);
            asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(dst), "r"(kv8_dequant2(lo, sc)),
                         "r"(kv8_dequant2(lo >> 16, sc)), "r"(kv8_dequant2(hi, sc)), "r"(kv8_dequant2(hi >> 16, sc))
                         : "memory");
          }
          fence_proxy_async_smem();   // generic-proxy writes, read by wgmma through the async proxy
          named_bar_sync(FA_BAR_CVT, FA_CVT_THREADS);
          if (t == 0) mbar_arrive(kv_full(stage));
        }
      }
    }
    return;
  }

  // ===================== consumers =====================
  setmaxnreg_inc<FA_CONSUMER_REGS>();
  const int row0 = wg * 64 + ((warp & 3) << 4) + (lane >> 2);   // this thread's rows: row0 and row0 + 8 of the tile
  const int qi0 = q_tile * 128 + row0, qi1 = qi0 + 8;
  const int cq = (lane & 3) * 2;                                 // first of this thread's two columns per 8-block
  const float sl2 = p.scale_log2;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;    // l: this thread's partial row sums
  float o[DN / 2];
#pragma unroll
  for (int i = 0; i < DN / 2; ++i) o[i] = 0.f;
  uint32_t o_seg0[IP ? DN / 4 : 1];   // IP: the normalised output of segment 0, rounded to fp16 (half2 per register)
#pragma unroll
  for (int i = 0; i < (IP ? DN / 4 : 1); ++i) o_seg0[i] = 0u;
  float s[64];
  uint32_t pa[8][4];

  const uint32_t q_src = smem_base + SM::OFF_Q + wg * (64 * 128);
  auto issue_s = [&](int stage) {
    const uint32_t k_src = smem_base + SM::OFF_K + stage * R * FA_REGION;
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < KS; ++k) {
      const uint32_t off = (k >> 2) * FA_REGION + (k & 3) * 32;
      WgmmaF16SS<128, 0>::mma(s, make_gmma_desc_sw128(q_src + off, 0, 1024), make_gmma_desc_sw128(k_src + off, 0, 1024),
                              k > 0 ? 1 : 0);
    }
    wgmma_commit();
  };
  auto issue_pv = [&](int stage) {
    const uint32_t v_src = smem_base + SM::OFF_V + stage * R * FA_REGION;
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 8; ++kk)   // 16 keys = 16 V rows of 128 B per step
      WgmmaF16RS<DN>::mma(o, pa[kk], make_gmma_desc_sw128(v_src + kk * 2048, FA_REGION, 1024), 1);
    wgmma_commit();
  };
  // Ping-pong: a consumer issues its MMAs between turn_begin and turn_end. Warpgroup 1 opens warpgroup 0's first turn;
  // both consumers take the same number of turns, and warpgroup 1's last arrival would have no matching wait, so it is
  // skipped.
  auto turn_begin = [&]() { named_bar_sync(FA_BAR_TURN + wg, 256); };
  auto turn_end = [&](bool last) {
    if (!(last && wg == 1)) named_bar_arrive(FA_BAR_TURN + (wg ^ 1), 256);
  };
  // Online softmax of tile j in s: new row maxima, alpha, P = exp2(s * sl2 - m * sl2) in place, row sums updated
  auto softmax = [&](int j, float& alpha0, float& alpha1) {
    const int key0 = (j < tiles0) ? j * 128 : (j - tiles0) * 128;
    const int kv_valid = (j < tiles0) ? min(128, p.N0 - key0) : min(128, p.N1 - key0);
    const bool masked = p.causal || kv_valid < 128;
    float mx0 = -INFINITY, mx1 = -INFINITY;
    if (masked) {
#pragma unroll
      for (int i = 0; i < 16; ++i) {
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const int col = i * 8 + cq + u;
          bool ok = col < kv_valid;
          const bool ok0 = ok && (!p.causal || key0 + col <= qi0);
          const bool ok1 = ok && (!p.causal || key0 + col <= qi1);
          if (!ok0) s[4 * i + u] = -INFINITY;
          if (!ok1) s[4 * i + 2 + u] = -INFINITY;
          mx0 = fmaxf(mx0, s[4 * i + u]);
          mx1 = fmaxf(mx1, s[4 * i + 2 + u]);
        }
      }
    } else {
#pragma unroll
      for (int i = 0; i < 16; ++i) {
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          mx0 = fmaxf(mx0, s[4 * i + u]);
          mx1 = fmaxf(mx1, s[4 * i + 2 + u]);
        }
      }
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);
    alpha0 = fast_exp2((m0 - mn0) * sl2);
    alpha1 = fast_exp2((m1 - mn1) * sl2);
    const float ms0 = mn0 * sl2, ms1 = mn1 * sl2;
    m0 = mn0;
    m1 = mn1;
    float sum0 = 0.f, sum1 = 0.f;
    if (masked) {
#pragma unroll
      for (int i = 0; i < 16; ++i) {
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const float x0 = s[4 * i + u], x1 = s[4 * i + 2 + u];
          const float p0 = x0 == -INFINITY ? 0.f : fast_exp2(x0 * sl2 - ms0);
          const float p1 = x1 == -INFINITY ? 0.f : fast_exp2(x1 * sl2 - ms1);
          s[4 * i + u] = p0;
          s[4 * i + 2 + u] = p1;
          sum0 += p0;
          sum1 += p1;
        }
      }
    } else {
#pragma unroll
      for (int i = 0; i < 16; ++i) {
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const float p0 = fast_exp2(s[4 * i + u] * sl2 - ms0);
          const float p1 = fast_exp2(s[4 * i + 2 + u] * sl2 - ms1);
          s[4 * i + u] = p0;
          s[4 * i + 2 + u] = p1;
          sum0 += p0;
          sum1 += p1;
        }
      }
    }
    l0 = l0 * alpha0 + sum0;
    l1 = l1 * alpha1 + sum1;
  };
  // P (fp16, unnormalised, <= 1) as the A fragments of the 8 k-steps of 16 keys
  auto pack_p = [&]() {
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
      pa[kk][0] = pack_h2(s[8 * kk + 0], s[8 * kk + 1]);
      pa[kk][1] = pack_h2(s[8 * kk + 2], s[8 * kk + 3]);
      pa[kk][2] = pack_h2(s[8 * kk + 4], s[8 * kk + 5]);
      pa[kk][3] = pack_h2(s[8 * kk + 6], s[8 * kk + 7]);
    }
  };

  auto rescale_o = [&](float alpha0, float alpha1) {
#pragma unroll
    for (int i = 0; i < DN / 8; ++i) {
      o[4 * i] *= alpha0;
      o[4 * i + 1] *= alpha0;
      o[4 * i + 2] *= alpha1;
      o[4 * i + 3] *= alpha1;
    }
  };
  // IP: at the first tile of segment 1, keep fp16(O_0 / l_0) and restart the softmax (called after softmax(j) with the
  // segment-0 row sums saved in ls0 / ls1)
  auto close_segment0 = [&](float ls0, float ls1) {
    ls0 += __shfl_xor_sync(0xffffffffu, ls0, 1);
    ls0 += __shfl_xor_sync(0xffffffffu, ls0, 2);
    ls1 += __shfl_xor_sync(0xffffffffu, ls1, 1);
    ls1 += __shfl_xor_sync(0xffffffffu, ls1, 2);
    const float i0 = 1.f / ls0, i1 = 1.f / ls1;
#pragma unroll
    for (int i = 0; i < DN / 8; ++i) {
      if constexpr (IP) {
        o_seg0[2 * i] = pack_h2(o[4 * i] * i0, o[4 * i + 1] * i0);
        o_seg0[2 * i + 1] = pack_h2(o[4 * i + 2] * i1, o[4 * i + 3] * i1);
      }
      o[4 * i] = o[4 * i + 1] = o[4 * i + 2] = o[4 * i + 3] = 0.f;
    }
  };

  if (wg == 1) named_bar_arrive(FA_BAR_TURN, 256);
  mbar_wait(q_full, 0);
  if constexpr (OVERLAP) {
    // tile 0: S_0 alone (O is still zero, so no rescale)
    mbar_wait(kv_full(0), 0);
    turn_begin();
    issue_s(0);
    turn_end(false);
    wgmma_wait<0>();
    fence_regs(s);
    {
      float a0, a1;
      softmax(0, a0, a1);
    }
    pack_p();
    for (int j = 1; j < total; ++j) {
      const int stage = j % ST, prev = (j - 1) % ST;
      mbar_wait(kv_full(stage), (j / ST) & 1);
      turn_begin();
      issue_s(stage);
      issue_pv(prev);
      turn_end(false);
      wgmma_wait<1>();   // S_j is in registers; P_{j-1} V_{j-1} may still run
      fence_regs(s);
      const bool seg_start = IP && j == tiles0;
      float ls0 = l0, ls1 = l1;
      if (seg_start) {   // the IP tokens' softmax starts afresh
        m0 = m1 = -INFINITY;
        l0 = l1 = 0.f;
      }
      float alpha0, alpha1;
      softmax(j, alpha0, alpha1);
      wgmma_wait<0>();
      fence_regs(o);
      if ((threadIdx.x & 127) == 0) mbar_arrive(kv_empty(prev));
      if (seg_start)
        close_segment0(ls0, ls1);
      else
        rescale_o(alpha0, alpha1);
      pack_p();
    }
    turn_begin();
    issue_pv((total - 1) % ST);
    turn_end(true);
    wgmma_wait<0>();
    fence_regs(o);
  } else {
    for (int j = 0; j < total; ++j) {
      const int stage = j % ST;
      mbar_wait(kv_full(stage), (j / ST) & 1);
      turn_begin();
      issue_s(stage);
      turn_end(false);
      wgmma_wait<0>();
      fence_regs(s);
      const bool seg_start = IP && j == tiles0;
      float ls0 = l0, ls1 = l1;
      if (seg_start) {
        m0 = m1 = -INFINITY;
        l0 = l1 = 0.f;
      }
      float alpha0, alpha1;
      softmax(j, alpha0, alpha1);
      if (seg_start)
        close_segment0(ls0, ls1);
      else
        rescale_o(alpha0, alpha1);
      pack_p();
      fence_regs(o);
      turn_begin();
      issue_pv(stage);
      turn_end(j == total - 1);
      wgmma_wait<0>();
      fence_regs(o);
      if ((threadIdx.x & 127) == 0) mbar_arrive(kv_empty(stage));
    }
  }

  l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
  l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  if (zero_kv) {
    // N1 all-zero key/value tokens: score 0 each (App. D.3)
    const float mn0 = fmaxf(m0, 0.f), mn1 = fmaxf(m1, 0.f);
    const float alpha0 = fast_exp2((m0 - mn0) * sl2), alpha1 = fast_exp2((m1 - mn1) * sl2);
    l0 = l0 * alpha0 + static_cast<float>(p.N1) * fast_exp2(-mn0 * sl2);
    l1 = l1 * alpha1 + static_cast<float>(p.N1) * fast_exp2(-mn1 * sl2);
#pragma unroll
    for (int i = 0; i < DN / 8; ++i) {
      o[4 * i] *= alpha0;
      o[4 * i + 1] *= alpha0;
      o[4 * i + 2] *= alpha1;
      o[4 * i + 3] *= alpha1;
    }
  }
  const float inv[2] = {1.f / l0, 1.f / l1};
  const int qi[2] = {qi0, qi1};
  const bool two_softmax = IP && tiles1 > 0;
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    if (qi[hr] >= p.Nq) continue;
    __half* dst = p.out + (static_cast<long long>(b) * p.Nq + qi[hr]) * p.ld_out + h * p.D;
#pragma unroll
    for (int i = 0; i < DN / 8; ++i) {
      const int col = i * 8 + cq;
      if (col >= p.D) continue;
      float v0 = o[4 * i + 2 * hr] * inv[hr], v1 = o[4 * i + 2 * hr + 1] * inv[hr];
      if (two_softmax) {
        const float2 t = unpack_h2(o_seg0[IP ? 2 * i + hr : 0]);
        v0 = t.x + round_h(p.out_scale * round_h(v0));
        v1 = t.y + round_h(p.out_scale * round_h(v1));
      } else if (p.accumulate) {
        const float2 a = unpack_h2(*reinterpret_cast<const uint32_t*>(dst + col));
        v0 = a.x + round_h(p.out_scale * round_h(v0));
        v1 = a.y + round_h(p.out_scale * round_h(v1));
      }
      *reinterpret_cast<uint32_t*>(dst + col) = pack_h2(v0, v1);
    }
  }
}

template <int KS, bool IP = false, int R = (KS + 3) / 4, int DN = (KS <= 4 ? 64 : 96)>
__global__ void __launch_bounds__(FA_THREADS, 1)
flash_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK0,
             const __grid_constant__ CUtensorMap tmV0, const __grid_constant__ CUtensorMap tmK1,
             const __grid_constant__ CUtensorMap tmV1, const FlashParams p) {
  flash_body<KS, IP, R, DN, false>(&tmQ, &tmK0, &tmV0, &tmK1, &tmV1, nullptr, p);
}

// Self + garment attention of the try-on blocks with the garment K/V (segment 1) in the FP8 format: tmK1 / tmV1 are
// one-byte maps of the e4m3 K / V (box 64 x 128, no swizzle), tmE the exponents [B1, 2H, lde] (box 128 x 1 x 1).
__global__ void __launch_bounds__(FA_THREADS, 1)
flash_kv8_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK0,
                 const __grid_constant__ CUtensorMap tmV0, const __grid_constant__ CUtensorMap tmK1,
                 const __grid_constant__ CUtensorMap tmV1, const __grid_constant__ CUtensorMap tmE, const FlashParams p) {
  flash_body<4, false, 1, 64, true>(&tmQ, &tmK0, &tmV0, &tmK1, &tmV1, &tmE, p);
}

// Tuning switches of other attention kernels of this library's C ABI. There is one attention kernel here, which always
// runs the ping-pong schedule with 128-query tiles and ex2.approx, so the options "attention_pingpong",
// "attention_q_tiles" and "attention_poly_exp" are accepted and have no effect.
void set_attn_poly(int) {}
void set_attn_qtiles(int) {}
void set_attn_v2(int) {}

static int encode_tokens(CUtensorMap* tm, const void* base, long long ld, int cols, int n, int batch) {
  uint64_t dims[3] = {static_cast<uint64_t>(cols), static_cast<uint64_t>(n), static_cast<uint64_t>(batch)};
  uint64_t strides[2] = {static_cast<uint64_t>(ld) * 2, static_cast<uint64_t>(n) * ld * 2};
  uint32_t box[3] = {64, 128, 1};
  return encode_tmap_f16(tm, base, 3, dims, strides, box);
}

template <int KS, bool IP = false>
static int launch_flash(const CUtensorMap& tmQ, const CUtensorMap& tmK0, const CUtensorMap& tmV0, const CUtensorMap& tmK1,
                        const CUtensorMap& tmV1, const FlashParams& p, cudaStream_t stream) {
  constexpr int R = (KS + 3) / 4;
  auto kern = flash_kernel<KS, IP>;
  static bool configured = false;
  if (!configured) {
    VTON_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, FlashSmem<R>::TOTAL));
    configured = true;
  }
  dim3 grid((p.Nq + 127) / 128, p.H, p.B);
  VTON_CUDA(launch_kernel(kern, grid, dim3(FA_THREADS), FlashSmem<R>::TOTAL, stream, tmQ, tmK0, tmV0, tmK1, tmV1, p));
  count_launch();
  return kOk;
}

// One launch: q [B, Nq, >= H*D] (row stride ldq); k0/v0 [B, N0, .] (ldkv0); k1/v1 [B1, N1, .] (ldkv1) or null.
// ip: segment 1 is the IP tokens of the decoupled cross-attention (D = 64), with a softmax of its own.
static int flash(const void* q, long long ldq, const void* k0, const void* v0, long long ldkv0, const void* k1,
                 const void* v1, long long ldkv1, int B1, void* out, long long ldo, FlashParams p, cudaStream_t stream,
                 bool ip = false) {
  CUtensorMap tmQ, tmK0, tmV0, tmK1, tmV1;
  const int cols = p.H * p.D;
  if (int e = encode_tokens(&tmQ, q, ldq, cols, p.Nq, p.B)) return e;
  if (int e = encode_tokens(&tmK0, k0, ldkv0, cols, p.N0, p.B)) return e;
  if (int e = encode_tokens(&tmV0, v0, ldkv0, cols, p.N0, p.B)) return e;
  tmK1 = tmK0;
  tmV1 = tmV0;
  if (k1 != nullptr) {
    if (int e = encode_tokens(&tmK1, k1, ldkv1, cols, p.N1, B1)) return e;
    if (int e = encode_tokens(&tmV1, v1, ldkv1, cols, p.N1, B1)) return e;
  }
  p.out = static_cast<__half*>(out);
  p.ld_out = static_cast<int>(ldo);
  if (ip) return launch_flash<4, true>(tmQ, tmK0, tmV0, tmK1, tmV1, p, stream);
  switch (p.D / 16) {
    case 1: return launch_flash<1>(tmQ, tmK0, tmV0, tmK1, tmV1, p, stream);
    case 2: return launch_flash<2>(tmQ, tmK0, tmV0, tmK1, tmV1, p, stream);
    case 3: return launch_flash<3>(tmQ, tmK0, tmV0, tmK1, tmV1, p, stream);
    case 4: return launch_flash<4>(tmQ, tmK0, tmV0, tmK1, tmV1, p, stream);
    case 5: return launch_flash<5>(tmQ, tmK0, tmV0, tmK1, tmV1, p, stream);
    case 6: return launch_flash<6>(tmQ, tmK0, tmV0, tmK1, tmV1, p, stream);
  }
  set_last_error("attention: head dim %d unsupported", p.D);
  return kErrUnsupported;
}

// q: [B, Nq, >=H*64] (row stride ldq); k0/v0: [B, N0, .] (ldkv0); k1/v1: [B1, N1, .] (ldkv1); out: [B, Nq, .] (ldo).
// kv1_rows (device int32 [B - kv1_off], or null): sample b >= kv1_off reads segment-1 row kv1_rows[b - kv1_off], in
// place of kv1_mod / kv1_base.
static int attn_common(const void* q, long long ldq, const void* k0, const void* v0, long long ldkv0, const void* k1,
                       const void* v1, long long ldkv1, void* out, long long ldo, int B, int H, int Nq, int N0, int N1,
                       int B1, int kv1_off, int kv1_mod, const void* kv1_base, const void* kv1_rows, float scale,
                       int accumulate, cudaStream_t stream) {
  VTON_CHECK_ARG(B > 0 && H > 0 && Nq > 0 && N0 > 0 && N1 >= 0, "attn: bad sizes B=%d H=%d Nq=%d N0=%d N1=%d", B, H, Nq, N0, N1);
  VTON_CHECK_ARG(ldq % 8 == 0 && ldkv0 % 8 == 0 && ldo % 8 == 0, "attn: row strides must be multiples of 8");
  VTON_CHECK_ARG(aligned_to(out, 4), "attn: out must be 4-byte aligned (stored two halves at a time)");
  VTON_CHECK_ARG(B <= 65535 && H <= 65535, "attn: grid too large");
  const bool has1 = N1 > 0 && B1 > 0 && k1 && v1;
  VTON_CHECK_ARG(N1 == 0 || has1 || kv1_off >= B, "attn: segment 1 declared (N1=%d) but no K/V given", N1);
  VTON_CHECK_ARG(!has1 || ldkv1 % 8 == 0, "attn: ldkv1 must be a multiple of 8");
  FlashParams p{};
  p.B = B;
  p.H = H;
  p.Nq = Nq;
  p.N0 = N0;
  p.N1 = N1;
  p.D = 64;
  p.kv1_off = has1 ? kv1_off : (N1 > 0 ? B : 0);
  p.kv1_count = has1 ? (kv1_rows || kv1_mod <= 0 ? B1 : kv1_mod) : 1;
  p.kv1_base = has1 && !kv1_rows ? static_cast<const int*>(kv1_base) : nullptr;
  p.kv1_rows = has1 ? static_cast<const int*>(kv1_rows) : nullptr;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.accumulate = accumulate;
  p.out_scale = 1.f;
  return flash(q, ldq, k0, v0, ldkv0, has1 ? k1 : nullptr, has1 ? v1 : nullptr, ldkv1, B1, out, ldo, p, stream);
}

int attn_impl(const void* q, long long ldq, const void* k0, const void* v0, long long ldkv0, const void* k1,
              const void* v1, long long ldkv1, void* out, long long ldo, int B, int H, int Nq, int N0, int N1, int B1,
              int kv1_off, int kv1_mod, const void* kv1_base, float scale, int accumulate, cudaStream_t stream) {
  return attn_common(q, ldq, k0, v0, ldkv0, k1, v1, ldkv1, out, ldo, B, H, Nq, N0, N1, B1, kv1_off, kv1_mod, kv1_base,
                     nullptr, scale, accumulate, stream);
}

int attn_rows_impl(const void* q, long long ldq, const void* k0, const void* v0, long long ldkv0, const void* k1,
                   const void* v1, long long ldkv1, void* out, long long ldo, int B, int H, int Nq, int N0, int N1,
                   int B1, int kv1_off, const void* kv1_rows, float scale, int accumulate, cudaStream_t stream) {
  VTON_CHECK_ARG(kv1_rows, "attention_rows: kv1_rows is null");
  VTON_CHECK_ARG(aligned_to(kv1_rows, 4), "attention_rows: kv1_rows must be 4-byte aligned (int32)");
  VTON_CHECK_ARG(N1 > 0 && B1 > 0 && k1 && v1, "attention_rows: needs segment-1 K/V (N1=%d, B1=%d)", N1, B1);
  VTON_CHECK_ARG(kv1_off >= 0 && kv1_off < B, "attention_rows: kv1_off %d outside [0, B=%d)", kv1_off, B);
  return attn_common(q, ldq, k0, v0, ldkv0, k1, v1, ldkv1, out, ldo, B, H, Nq, N0, N1, B1, kv1_off, 0, nullptr,
                     kv1_rows, scale, accumulate, stream);
}

// Decoupled cross-attention of the try-on / garment transformer blocks:
//     out = fp16( fp16(softmax(Q Kt^T * scale) Vt) + fp16(ip_scale * fp16(softmax(Q Ki^T * scale) Vi)) )
// Kt/Vt = the text tokens (attn2.to_k / to_v), Ki/Vi = the IP-Adapter image tokens (to_k_ip / to_v_ip); with Ni = 0 it is
// the plain text cross-attention of the garment UNet (src/attentionhacked_garmnet.py:371-383).
// q/out: [B, Nq, >= H*64]; kt/vt: [B, Nt, .] (row stride ldkv_t); ki/vi: [B, Ni, .] (ldkv_i) or null with Ni = 0
int cross_attn_impl(const void* q, long long ldq, const void* kt, const void* vt, long long ldkv_t, int Nt,
                    const void* ki, const void* vi, long long ldkv_i, int Ni, void* out, long long ldo, int B, int H,
                    int Nq, float scale, float ip_scale, cudaStream_t stream) {
  VTON_CHECK_ARG(B > 0 && H > 0 && Nq > 0, "cross_attn: bad sizes B=%d H=%d Nq=%d", B, H, Nq);
  VTON_CHECK_ARG(Nt > 0 && Nt <= 80 && Ni >= 0 && Ni <= 16, "cross_attn: needs 1 <= Nt <= 80 and Ni <= 16 (got %d, %d)", Nt, Ni);
  VTON_CHECK_ARG(q && kt && vt && out && (Ni == 0 || (ki && vi)), "cross_attn: null pointer");
  VTON_CHECK_ARG(ldq % 8 == 0 && ldkv_t % 8 == 0 && ldo % 8 == 0 && (Ni == 0 || ldkv_i % 8 == 0),
                 "cross_attn: row strides must be multiples of 8");
  VTON_CHECK_ARG(aligned_to(out, 4), "cross_attn: out must be 4-byte aligned (stored two halves at a time)");
  VTON_CHECK_ARG(B <= 65535 && H <= 65535, "cross_attn: grid too large");
  // one launch: Q is read once, segment 0 = the text tokens, segment 1 = the IP tokens of the same sample (kv1_off = 0,
  // kv1_count = B) with a softmax of its own
  FlashParams p{};
  p.B = B;
  p.H = H;
  p.Nq = Nq;
  p.N0 = Nt;
  p.N1 = Ni;
  p.D = 64;
  p.kv1_count = B;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.out_scale = Ni > 0 ? ip_scale : 1.f;
  return flash(q, ldq, kt, vt, ldkv_t, Ni > 0 ? ki : nullptr, Ni > 0 ? vi : nullptr, ldkv_i, B, out, ldo, p, stream,
               Ni > 0);
}

// Self + garment attention with the garment K/V (segment 1) in the FP8 format: k1 / v1 e4m3 [B1, N1, >= H*64] (row
// stride ldkv1 bytes), e1 int8 exponents [B1, 2H, lde1] (group h = K head h, group H + h = V head h). Segment 1 as in
// attn_impl (kv1_mod / kv1_base) or, with kv1_rows, as in attn_rows_impl.
int attn_kv8_impl(const void* q, long long ldq, const void* k0, const void* v0, long long ldkv0, const void* k1,
                  const void* v1, long long ldkv1, const void* e1, long long lde1, void* out, long long ldo, int B, int H,
                  int Nq, int N0, int N1, int B1, int kv1_off, int kv1_mod, const void* kv1_base, const void* kv1_rows,
                  float scale, int accumulate, cudaStream_t stream) {
  VTON_CHECK_ARG(B > 0 && H > 0 && Nq > 0 && N0 > 0 && N1 > 0 && B1 > 0,
                 "attention_kv8: bad sizes B=%d H=%d Nq=%d N0=%d N1=%d B1=%d", B, H, Nq, N0, N1, B1);
  VTON_CHECK_ARG(q && k0 && v0 && k1 && v1 && e1 && out, "attention_kv8: null pointer");
  VTON_CHECK_ARG(ldq % 8 == 0 && ldkv0 % 8 == 0 && ldo % 8 == 0, "attention_kv8: fp16 row strides must be multiples of 8");
  VTON_CHECK_ARG(ldkv1 % 16 == 0 && ldkv1 >= 64LL * H, "attention_kv8: ldkv1 %lld must be a multiple of 16 and >= 64*H",
                 ldkv1);
  VTON_CHECK_ARG(lde1 % 16 == 0 && lde1 >= N1, "attention_kv8: lde1 %lld must be a multiple of 16 and >= N1 = %d", lde1,
                 N1);
  VTON_CHECK_ARG(aligned_to(out, 4), "attention_kv8: out must be 4-byte aligned (stored two halves at a time)");
  VTON_CHECK_ARG(aligned_to(kv1_rows, 4), "attention_kv8: kv1_rows must be 4-byte aligned (int32)");
  VTON_CHECK_ARG(kv1_off >= 0 && kv1_off < B, "attention_kv8: kv1_off %d outside [0, B=%d)", kv1_off, B);
  VTON_CHECK_ARG(B <= 65535 && H <= 65535, "attention_kv8: grid too large");
  FlashParams p{};
  p.B = B;
  p.H = H;
  p.Nq = Nq;
  p.N0 = N0;
  p.N1 = N1;
  p.D = 64;
  p.kv1_off = kv1_off;
  p.kv1_count = kv1_rows || kv1_mod <= 0 ? B1 : kv1_mod;
  p.kv1_base = kv1_rows ? nullptr : static_cast<const int*>(kv1_base);
  p.kv1_rows = static_cast<const int*>(kv1_rows);
  p.scale_log2 = scale * 1.4426950408889634f;
  p.accumulate = accumulate;
  p.out_scale = 1.f;
  p.out = static_cast<__half*>(out);
  p.ld_out = static_cast<int>(ldo);
  CUtensorMap tmQ, tmK0, tmV0, tmK1, tmV1, tmE;
  const int cols = H * 64;
  if (int e = encode_tokens(&tmQ, q, ldq, cols, Nq, B)) return e;
  if (int e = encode_tokens(&tmK0, k0, ldkv0, cols, N0, B)) return e;
  if (int e = encode_tokens(&tmV0, v0, ldkv0, cols, N0, B)) return e;
  {
    const uint64_t dims[3] = {static_cast<uint64_t>(cols), static_cast<uint64_t>(N1), static_cast<uint64_t>(B1)};
    const uint64_t strides[2] = {static_cast<uint64_t>(ldkv1), static_cast<uint64_t>(ldkv1) * N1};
    const uint32_t box[3] = {64, 128, 1};
    if (int e = encode_tmap_u8(&tmK1, k1, 3, dims, strides, box, 0)) return e;
    if (int e = encode_tmap_u8(&tmV1, v1, 3, dims, strides, box, 0)) return e;
  }
  {
    const uint64_t dims[3] = {static_cast<uint64_t>(lde1), static_cast<uint64_t>(2 * H), static_cast<uint64_t>(B1)};
    const uint64_t strides[2] = {static_cast<uint64_t>(lde1), static_cast<uint64_t>(lde1) * 2 * H};
    const uint32_t box[3] = {128, 1, 1};
    if (int e = encode_tmap_u8(&tmE, e1, 3, dims, strides, box, 0)) return e;
  }
  using SM = FlashSmem<1, true>;
  static bool configured = false;
  if (!configured) {
    VTON_CUDA(cudaFuncSetAttribute(flash_kv8_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SM::TOTAL));
    configured = true;
  }
  dim3 grid((Nq + 127) / 128, H, B);
  VTON_CUDA(launch_kernel(flash_kv8_kernel, grid, dim3(FA_THREADS), SM::TOTAL, stream, tmQ, tmK0, tmV0, tmK1, tmV1, tmE, p));
  count_launch();
  return kOk;
}

// The FP8 garment K/V quantizer. A warp takes 4 (token, group) items, 8 lanes each (8 values per lane); items run over
// [rows, G, lde] with the token fastest, so the exponent stores of a warp are contiguous. Items with n >= Ng write the
// exponent padding (0) only.
__global__ void __launch_bounds__(256) quantize_kv_e4m3_kernel(const __half* __restrict__ x, long long ldx, int rows,
                                                                int Ng, int G, int lde, uint8_t* __restrict__ q,
                                                                long long ldq, int8_t* __restrict__ e_out) {
  pdl_wait();
  pdl_launch_dependents();
  const int lane = threadIdx.x & 31, sub = lane & 7;
  const long long n_items = static_cast<long long>(rows) * G * lde;
  const long long warps = static_cast<long long>(gridDim.x) * (blockDim.x >> 5);
  for (long long base = (static_cast<long long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5)) * 4;
       base < n_items; base += warps * 4) {
    const long long it = base + (lane >> 3);
    const bool valid = it < n_items;
    const int n = valid ? static_cast<int>(it % lde) : 0;
    const long long rg = valid ? it / lde : 0;   // row * G + g
    const int g = static_cast<int>(rg % G);
    const bool tok = valid && n < Ng;
    const long long m = (rg / G) * Ng + n;
    float v[8];
    float amax = 0.f;
    if (tok) {
      const uint4 raw = *reinterpret_cast<const uint4*>(x + m * ldx + g * 64 + sub * 8);
      const uint32_t w[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 f = unpack_h2(w[i]);
        v[2 * i] = f.x;
        v[2 * i + 1] = f.y;
        amax = fmaxf(amax, fmaxf(fabsf(f.x), fabsf(f.y)));
      }
    }
    amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 1));
    amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 2));
    amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 4));
    // smallest e with amax <= 448 * 2^e: amax = 1.f * 2^E, 448 = 1.75 * 2^8
    int e = 0;
    if (amax > 0.f) {
      const uint32_t bits = __float_as_uint(amax);
      const int E = static_cast<int>((bits >> 23) & 0xff) - 127;
      e = max(E - ((bits & 0x7fffffu) <= 0x600000u ? 8 : 7), -24);
    }
    if (tok) {
      const float inv = __uint_as_float(static_cast<uint32_t>(127 - e) << 23);   // 2^-e, exact products
      uint32_t packed[2];
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const __nv_fp8x2_storage_t a =
            __nv_cvt_float2_to_fp8x2(make_float2(__fmul_rn(v[4 * i], inv), __fmul_rn(v[4 * i + 1], inv)), __NV_SATFINITE, __NV_E4M3);
        const __nv_fp8x2_storage_t b =
            __nv_cvt_float2_to_fp8x2(make_float2(__fmul_rn(v[4 * i + 2], inv), __fmul_rn(v[4 * i + 3], inv)), __NV_SATFINITE, __NV_E4M3);
        packed[i] = static_cast<uint32_t>(a) | (static_cast<uint32_t>(b) << 16);
      }
      *reinterpret_cast<uint2*>(q + m * ldq + g * 64 + sub * 8) = make_uint2(packed[0], packed[1]);
    }
    if (valid && sub == 0) e_out[rg * lde + n] = static_cast<int8_t>(tok ? e : 0);
  }
}

int quantize_kv_e4m3_impl(const void* x, long long ldx, int M, int G, int Ng, void* q, long long ldq, void* e,
                          long long lde, cudaStream_t stream) {
  VTON_CHECK_ARG(M > 0 && G > 0 && Ng > 0 && M % Ng == 0, "quantize_kv_e4m3: bad sizes M=%d G=%d Ng=%d (M must be a "
                 "multiple of Ng)", M, G, Ng);
  VTON_CHECK_ARG(x && q && e, "quantize_kv_e4m3: null pointer");
  VTON_CHECK_ARG(ldx % 8 == 0 && ldx >= 64LL * G && aligned_to(x, 16),
                 "quantize_kv_e4m3: x must be 16-byte aligned with ldx a multiple of 8 and >= 64*G");
  VTON_CHECK_ARG(ldq % 8 == 0 && ldq >= 64LL * G && aligned_to(q, 8),
                 "quantize_kv_e4m3: q must be 8-byte aligned with ldq a multiple of 8 and >= 64*G");
  VTON_CHECK_ARG(lde >= Ng && lde <= (1LL << 30), "quantize_kv_e4m3: lde %lld must be >= Ng = %d", lde, Ng);
  const int rows = M / Ng;
  const long long items = static_cast<long long>(rows) * G * lde;
  const long long blocks = std::min<long long>((items + 31) / 32, 32LL * num_sms());
  VTON_CUDA(launch_kernel(quantize_kv_e4m3_kernel, dim3(static_cast<unsigned>(blocks)), dim3(256), 0, stream,
                          static_cast<const __half*>(x), ldx, rows, Ng, G, static_cast<int>(lde),
                          static_cast<uint8_t*>(q), ldq, static_cast<int8_t*>(e)));
  count_launch();
  return kOk;
}

// Encoder self-attention of the CLIP towers around the denoising loop: the ViT-H image encoder (16 heads of 80, 257
// tokens) and the two text encoders (heads of 64, 77 tokens, causal mask).
// q / k / v: [B, N, >= H*D] views (row strides ldq / ldkv, e.g. the three column blocks of a fused QKV buffer);
// out: [B, N, H*D] (row stride ldo)
int enc_attn_impl(const void* q, long long ldq, const void* k, const void* v, long long ldkv, void* out, long long ldo,
                  int B, int H, int N, int D, float scale, int causal, cudaStream_t stream) {
  VTON_CHECK_ARG(B > 0 && H > 0 && N > 0, "encoder_attention: bad sizes B=%d H=%d N=%d", B, H, N);
  VTON_CHECK_ARG(D >= 16 && D <= 96 && D % 16 == 0, "encoder_attention: head dim %d unsupported (16..96, multiple of 16)", D);
  VTON_CHECK_ARG(ldq % 8 == 0 && ldkv % 8 == 0 && ldo % 8 == 0, "encoder_attention: row strides must be multiples of 8");
  VTON_CHECK_ARG(aligned_to(out, 4), "encoder_attention: out must be 4-byte aligned (stored two halves at a time)");
  VTON_CHECK_ARG(B <= 65535 && H <= 65535, "encoder_attention: grid too large");
  FlashParams p{};
  p.B = B;
  p.H = H;
  p.Nq = N;
  p.N0 = N;
  p.D = D;
  p.kv1_count = 1;
  p.causal = causal ? 1 : 0;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.out_scale = 1.f;
  return flash(q, ldq, k, v, ldkv, nullptr, nullptr, 0, 0, out, ldo, p, stream);
}

}  // namespace vton
