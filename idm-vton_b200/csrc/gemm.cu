// wgmma GEMM / implicit-GEMM 3x3 convolution for the IDM-VTON UNets and the VAE (sm_90a).
//
//   linear : out[M,N] = epi( A[M,K] . W[N,K]^T )                (K8 in SURVEY.md 2.3: to_q/k/v/out, proj_in/out, FF)
//   conv3x3: out[b,y,x,:] = epi( sum_taps A[b,y+dy,x+dx,:] . W[tap][:, :]^T  (+ 1x1 shortcut in a 2nd accumulator) )
//            (K1/K2/K5: ResnetBlock2D conv1/conv2/conv_shortcut, conv_in, conv_out; NHWC, pad 1, stride 1 or 2)
//   fp32 conv3x3 (the VAE): TF32 operands (or fp16 operands) with fp32 accumulate, bias, residual and output.
//
// A CTA computes 128 x BN output tiles, one after another: the grid is min(tiles, SMs) and CTA b takes tiles b,
// b + gridDim.x, ... (n fastest, so neighbouring CTAs share an A slab in L2). Warps 0..7 are two consumer warpgroups
// (rows 0..63 / 64..127 of the tile) that issue m64nBNk16 (k8 for TF32) wgmma from 128B-swizzled shared memory into
// register accumulators; warp 8 (in a warpgroup of its own, which gives most of its registers to the consumers) is the
// TMA producer. The conv walks K as 9 taps x Cin/64 slabs with a 4-D tensor map over [B,H,W,C]; out-of-bounds box
// elements are zero-filled by TMA, which is the conv's zero padding. The producer runs on into the next tile's slabs
// while the consumers finish a tile, so only a CTA's first tile waits for a load.
// The fp16 epilogue is split in two (gemm_common.cuh). After a tile's K loop each consumer thread does the register
// half on its own accumulator fragment (bias, activation or GEGLU, time embedding, shortcut, residual) and writes the
// tile to a shared-memory staging tile, then goes straight on to the next tile's K loop. Warps 9..11 of the producer's
// warpgroup, which used to only give up their registers, do the memory half: they store the staged tile to global
// memory 16 bytes at a time while the next K loop runs, and then bulk-copy the residual rows of the tile after it into
// the staging tile, so it is there when that tile is staged. Two mbarriers hand the staging tile back and forth
// (`staged`, `ready`). The fp32-output kinds keep their epilogue in the consumers and store from the fragment.
// e4m3 linears (KIND_E4M3, the opt-in FP8 mode): a 128-byte slab row holds 128 e4m3 values, so the ring, the
// descriptors and the 32-byte MMA step are those of the fp16 kind; the MMA is m64nNk32 e4m3 x e4m3 -> fp32 and the
// epilogue scales each accumulator by its row's and column's scale before the fp16 epilogue below. The tensor core
// keeps fewer accumulator bits for e4m3 than fp32 (the error grew with K to 4.5e-3 of the output's scale at K = 5120 on
// an H100), so each slab's 4 MMAs accumulate into a partial sum of their own, which is added to the fp32 register
// accumulator once the slab's MMAs have retired (E4M3_SUB columns at a time: halves at BN = 192 and quarters at BN = 256,
// where a wider partial sum would not fit beside the accumulator without spilling).
// Epilogue rounding points replicate the reference's fp16-autocast path (SURVEY.md App. D.1):
//   v = fp16(acc + bias); v = fp16(v + temb[b,n]); s = fp16(acc_sc + bias_sc); v = fp16(s + v); v = fp16(v + res)
#include "gemm_common.cuh"
#include "host.h"
#include "wgmma.cuh"

namespace vton {

enum : int { KIND_F16 = 0, KIND_F16IN_F32OUT = 1, KIND_TF32 = 2, KIND_E4M3 = 3 };

constexpr bool f16_out(int kind) { return kind == KIND_F16 || kind == KIND_E4M3; }

// Operand ring, then (fp16 output) the staging tile of the epilogue, the barriers and the store warps' row tables.
template <int BN, int STAGES, bool GEGLU, int KIND>
struct SmemLayout {
  static constexpr int B_BYTES = BN * 128;              // BN rows x 128 B (64 halves, 32 floats or 128 e4m3)
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STAGING_OFFSET = STAGES * STAGE_BYTES;
  static constexpr int STAGING_BYTES = f16_out(KIND) ? StagingTile<BN, GEGLU>::BYTES : 0;
  static constexpr int BAR_OFFSET = STAGING_OFFSET + STAGING_BYTES;   // full[STAGES], empty[STAGES], staged, ready
  static constexpr int ROWS_OFFSET = BAR_OFFSET + 256;                // 2 x 128 int32 output rows
  static constexpr int TOTAL = ROWS_OFFSET + (f16_out(KIND) ? 2 * BM * 4 : 0) + 1024;   // + alignment slack
};

// 2 consumer warpgroups + the producer's warpgroup (warp 8 loads; warps 9..11 store the fp16 epilogue, or only hand
// over their registers for the fp32-output kinds). ptxas allots registers per whole warpgroup, 168 a thread at launch
// (64512 for the CTA), which does not hold a 128-float accumulator and the epilogue; so the producer's warpgroup drops
// to 56 and the consumers rise to 224 (128 * 56 + 256 * 224 = 64512).
constexpr int GEMM_THREADS = 384;
constexpr int GEMM_PRODUCER_REGS = 56;
constexpr int GEMM_CONSUMER_REGS = 224;

template <int BN>
constexpr int E4M3_SUB = BN == 256 ? 64 : (BN == 192 ? 96 : BN);

template <int BN, int STAGES, bool GEGLU, bool SC, int KIND>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_conv_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const __grid_constant__ CUtensorMap tmS0, const __grid_constant__ CUtensorMap tmS1,
                 const __grid_constant__ CUtensorMap tmBs, const GemmParams p) {
  using L = SmemLayout<BN, STAGES, GEGLU, KIND>;
  constexpr int KBK = KIND == KIND_TF32 ? 32 : (KIND == KIND_E4M3 ? 128 : 64);   // channels per 128-byte slab row
  constexpr bool F16_EPI = f16_out(KIND);
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bar_base = smem_base + L::BAR_OFFSET;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (STAGES + s); };
  // staging tile handshake for tile j of the CTA's schedule: `ready` completes phase j when the store warps have read
  // tile j - 1 out of the staging tile and tile j's residual has landed in it, `staged` when both consumer warpgroups
  // have written tile j
  const uint32_t staged_bar = bar_base + 8u * (2 * STAGES);
  const uint32_t ready_bar = bar_base + 8u * (2 * STAGES + 1);
  const uint32_t staging = smem_base + L::STAGING_OFFSET;
  // the staging tile and the store warps' row tables as pointers (from the 1024-aligned base)
  auto staging_ptr = [&]() { return smem_raw + (smem_base - smem_u32(smem_raw)) + L::STAGING_OFFSET; };
  auto row_table = [&]() { return reinterpret_cast<int*>(smem_raw + (smem_base - smem_u32(smem_raw)) + L::ROWS_OFFSET); };

  const int warp = threadIdx.x >> 5;

  if (threadIdx.x == 8 * 32) {   // warp 8, lane 0
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if (SC) {
      tma_prefetch_desc(&tmS0);
      tma_prefetch_desc(&tmS1);
      tma_prefetch_desc(&tmBs);
    }
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 2);   // one arrival per consumer warpgroup
    }
    if (F16_EPI) {
      mbar_init(staged_bar, 256);   // every consumer thread, after its staging stores
      mbar_init(ready_bar, EpilogueStore<BN, GEGLU>::THREADS);
    }
    fence_barrier_init();
  }
  pdl_wait();
  __syncthreads();
  pdl_launch_dependents();

  // The producer and both consumer warpgroups walk the same static tile schedule, and each keeps one slab counter `it`
  // that runs on across tiles: slab `it` lives in stage it % STAGES on barrier phase (it / STAGES) & 1.
  if (warp >= 8) {
    // ===================== TMA producer =====================
    setmaxnreg_dec<GEMM_PRODUCER_REGS>();
    if (threadIdx.x == 8 * 32) {
      const int total_slabs = p.slabs_main + (SC ? p.slabs_sc : 0);
      uint32_t it = 0;
      for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
        const int n0 = (tile % p.n_tiles) * BN;
        const int m_tile = tile / p.n_tiles;
        int b0 = 0, y0 = 0, x0 = 0;   // conv tile origin
        if (p.conv) {
          x0 = (m_tile % p.tiles_x) * p.bw;
          y0 = ((m_tile / p.tiles_x) % p.tiles_y) * p.bh;
          b0 = (m_tile / (p.tiles_x * p.tiles_y)) * p.bb;
        }
        for (int s = 0; s < total_slabs; ++s, ++it) {
          const int stage = it % STAGES;
          const uint32_t phase = (it / STAGES) & 1;
          mbar_wait(empty_bar(stage), phase ^ 1);
          const uint32_t a_dst = smem_base + stage * L::STAGE_BYTES;
          const uint32_t b_dst = a_dst + A_BYTES;
          mbar_expect_tx(full_bar(stage), L::STAGE_BYTES);
          if (s < p.slabs_main) {
            if (p.conv) {
              const int tap = s / p.cin_slabs;
              const int c0 = (s - tap * p.cin_slabs) * KBK;
              const int dy = tap / 3 - 1, dx = tap % 3 - 1;
              tma_load_4d(a_dst, &tmA, full_bar(stage), c0, x0 * p.stride + dx, y0 * p.stride + dy, b0);
              tma_load_2d(b_dst, &tmB, full_bar(stage), c0, tap * p.cout + n0);
            } else {
              tma_load_2d(a_dst, &tmA, full_bar(stage), s * KBK, m_tile * BM);
              tma_load_2d(b_dst, &tmB, full_bar(stage), s * KBK, n0);
            }
          } else {
            const int ss = s - p.slabs_main;
            if (ss < p.sc_split)
              tma_load_4d(a_dst, &tmS0, full_bar(stage), ss * BK, x0, y0, b0);
            else
              tma_load_4d(a_dst, &tmS1, full_bar(stage), (ss - p.sc_split) * BK, x0, y0, b0);
            tma_load_2d(b_dst, &tmBs, full_bar(stage), ss * BK, n0);
          }
        }
      }
    } else if (F16_EPI && warp > 8) {
      // ===================== store warps: the memory half of the fp16 epilogue =====================
      EpilogueStore<BN, GEGLU>::run(p, staging, staging_ptr(), row_table(), staged_bar, ready_bar, threadIdx.x - 9 * 32);
    }
    return;
  }

  // ===================== consumers: two warpgroups, 64 accumulator rows each =====================
  setmaxnreg_inc<GEMM_CONSUMER_REGS>();
  const int wg = warp >> 2;
  const int lane = threadIdx.x & 31;
  const int r_local = wg * 64 + ((warp & 3) << 4) + (lane >> 2);   // the thread's first fragment row (the other: + 8)
  float acc[BN / 2];
  float acc_sc[BN / 2];   // shortcut accumulator (dead when !SC)
  uint32_t it = 0;
  // Every slab is released (one arrival per warpgroup on its stage's empty barrier) exactly once, after the wgmma wait
  // that retires it: slab it - 1 after the wait<1> that follows slab it's commit, a tile's last slab after the wait<0>
  // that ends the tile.
  auto release = [&](uint32_t slab) {
    if ((threadIdx.x & 127) == 0) mbar_arrive(empty_bar(slab % STAGES));
  };
  // One K slab per iteration; slabs [s_begin, s_end) of the tile accumulate into accr (a separate loop per accumulator
  // keeps the choice of registers static, so the wgmma pipeline is not serialised).
  auto run_slabs = [&](float (&accr)[BN / 2], int s_begin, int s_end) {
    for (int s = s_begin; s < s_end; ++s, ++it) {
      const int stage = it % STAGES;
      mbar_wait(full_bar(stage), (it / STAGES) & 1);
      const uint32_t a_src = smem_base + stage * L::STAGE_BYTES + wg * (64 * 128);
      const uint32_t b_src = smem_base + stage * L::STAGE_BYTES + A_BYTES;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) {   // 16 halves / 8 floats = 32 bytes per MMA step
        const uint64_t da = make_gmma_desc_sw128(a_src + k * 32, 0, 1024);
        const uint64_t db = make_gmma_desc_sw128(b_src + k * 32, 0, 1024);
        const int scale_d = (s > s_begin || k > 0) ? 1 : 0;
        if constexpr (KIND == KIND_TF32) {
          WgmmaTF32SS<BN>::mma(accr, da, db, scale_d);
        } else {
          WgmmaF16SS<BN, 0>::mma(accr, da, db, scale_d);
        }
      }
      wgmma_commit();
      wgmma_wait<1>();
      if (s > 0) release(it - 1);   // s == 0: the previous slab was the last of the tile before and is released already
    }
  };
  // e4m3: every slab accumulates into `part` (scale_d = 0 on its first MMA; 32 e4m3 = 32 bytes per MMA step), then
  // acc += part after wait<0>; the slab is released right there, as all of its MMAs have retired.
  auto run_slabs_promoted = [&](float (&accr)[BN / 2], int s_begin, int s_end) {
    constexpr int SUB = E4M3_SUB<BN>;
    for (int s = s_begin; s < s_end; ++s, ++it) {
      const int stage = it % STAGES;
      mbar_wait(full_bar(stage), (it / STAGES) & 1);
      const uint32_t a_src = smem_base + stage * L::STAGE_BYTES + wg * (64 * 128);
      const uint32_t b_src = smem_base + stage * L::STAGE_BYTES + A_BYTES;
#pragma unroll
      for (int sub = 0; sub < BN / SUB; ++sub) {
        float part[SUB / 2];
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const uint64_t da = make_gmma_desc_sw128(a_src + k * 32, 0, 1024);
          const uint64_t db = make_gmma_desc_sw128(b_src + sub * SUB * 128 + k * 32, 0, 1024);
          WgmmaE4M3SS<SUB>::mma(part, da, db, k > 0 ? 1 : 0);
        }
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(part);
#pragma unroll
        for (int j = 0; j < SUB / 2; ++j) accr[sub * (SUB / 2) + j] = s > s_begin ? accr[sub * (SUB / 2) + j] + part[j] : part[j];
      }
      release(it);
    }
  };
  for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
    EpilogueF16<BN, GEGLU, SC, KIND == KIND_E4M3> epi;   // fp16 output: the bias loads fly during the K loop
    if constexpr (F16_EPI) epi.begin(p, tile / p.n_tiles, tile % p.n_tiles, r_local);
    if constexpr (KIND == KIND_E4M3) {
      run_slabs_promoted(acc, 0, p.slabs_main);
    } else {
      run_slabs(acc, 0, p.slabs_main);
      if constexpr (SC) run_slabs(acc_sc, p.slabs_main, p.slabs_main + p.slabs_sc);
      wgmma_wait<0>();
      fence_regs(acc);
      if (SC) fence_regs(acc_sc);
      release(it - 1);
    }
    if constexpr (F16_EPI) {
      // The store warps stored tile j - 1 and copied this tile's residual into the staging tile while this tile's K loop
      // ran; once both are done, stage this tile and go straight on to the next tile's slabs.
      mbar_wait(ready_bar, ((tile - blockIdx.x) / gridDim.x) & 1);   // phase j for tile j of this CTA's schedule
      if (!GEGLU && p.act_gelu) epi.template stage<true, true>(p, acc, acc_sc, r_local, staging);
      else if (!GEGLU && p.rowvec) epi.template stage<false, true>(p, acc, acc_sc, r_local, staging);
      else epi.template stage<false, false>(p, acc, acc_sc, r_local, staging);
      mbar_arrive(staged_bar);
      if (tile + static_cast<int>(gridDim.x) >= p.total_tiles)   // the CTA's last tile: help the store warps store it
        EpilogueStore<BN, GEGLU>::help_store_last(p, tile, staging_ptr(), row_table(), staged_bar, threadIdx.x);
    } else {
      epilogue_f32<BN>(p, tile / p.n_tiles, tile % p.n_tiles, r_local, acc);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
template <int BN, int STAGES, bool GEGLU, bool SC, int KIND>
static int launch_variant(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmS0,
                          const CUtensorMap& tmS1, const CUtensorMap& tmBs, const GemmParams& p, cudaStream_t stream) {
  using L = SmemLayout<BN, STAGES, GEGLU, KIND>;
  static_assert(L::TOTAL <= 227 * 1024, "shared memory budget");
  auto kern = gemm_conv_kernel<BN, STAGES, GEGLU, SC, KIND>;
  static bool configured = false;
  if (!configured) {
    VTON_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, L::TOTAL));
    configured = true;
  }
  const int grid = p.total_tiles < num_sms() ? p.total_tiles : num_sms();   // every CTA loops over its share of the tiles
  VTON_CUDA(launch_kernel(kern, dim3(grid), dim3(GEMM_THREADS), L::TOTAL, stream, tmA, tmB, tmS0, tmS1, tmBs, p));
  count_launch();
  return kOk;
}

// force_bn: 0 = automatic tile width; 64 / 128 / 160 / 192 / 256 = that width (an error where the configuration cannot use
// it: GEGLU needs 128 or 256 dividing N, a fused shortcut 64 or 128). The encodings 1000 + width and 2000 + width of the
// C ABI (multi-CTA tile variants) select the same width of the one GEMM kernel, and the options "gemm_2cta_auto" /
// "gemm_cluster4" are accepted and have no effect.
void set_auto_v2(int) {}
void set_cluster4(int) {}

// Tile width: fewest waves of 128 x BN tiles over the SMs, each tile costing ~(BN + 64) per K slab (the 64 stands for
// the A slab every tile loads whatever its width); ties go to the wider tile (fewer bytes per FLOP). Returns 0 for a
// forced width this configuration cannot use.
static int pick_bn(int N, int m_tiles, bool geglu, bool has_shortcut, int force_bn) {
  if (force_bn >= 2000) force_bn -= 2000;
  else if (force_bn >= 1000) force_bn -= 1000;
  auto usable = [&](int bn) {
    if (geglu && ((bn != 256 && bn != 128) || N % bn != 0)) return false;
    if (has_shortcut && bn > 128) return false;   // two register accumulators per thread
    return true;
  };
  if (force_bn) {
    const bool known = force_bn == 64 || force_bn == 128 || force_bn == 160 || force_bn == 192 || force_bn == 256;
    return known && usable(force_bn) ? force_bn : 0;
  }
  const int sms = num_sms();
  const int cands[5] = {256, 192, 160, 128, 64};
  double best = 1e300;
  int best_bn = 0;
  for (int bn : cands) {
    if (!usable(bn)) continue;
    if (bn != 128 && N % bn != 0 && !(bn == 64 && N < 64)) continue;
    const long long tiles = static_cast<long long>(m_tiles) * cdiv(N, bn);
    const long long waves = (tiles + sms - 1) / sms;
    const double cost = static_cast<double>(waves) * (bn + 64);
    if (cost < best * 0.999) {
      best = cost;
      best_bn = bn;
    }
  }
  return best_bn ? best_bn : 128;
}

template <int KIND>
static int dispatch(int bn, bool geglu, const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmS0,
                    const CUtensorMap& tmS1, const CUtensorMap& tmBs, GemmParams& p, int m_tiles,
                    cudaStream_t stream) {
  p.n_tiles = cdiv(p.N, bn);
  p.total_tiles = m_tiles * p.n_tiles;
  if (geglu) {
    if (bn == 128) return launch_variant<128, 6, true, false, KIND>(tmA, tmB, tmS0, tmS1, tmBs, p, stream);
    if (bn == 256) return launch_variant<256, 4, true, false, KIND>(tmA, tmB, tmS0, tmS1, tmBs, p, stream);
    set_last_error("GEGLU epilogue supports BN 128/256 only (got %d)", bn);
    return kErrUnsupported;
  }
  if constexpr (KIND == KIND_F16) {   // the fused shortcut exists for the fp16 convolution only
    if (p.slabs_sc) {
      if (bn == 64) return launch_variant<64, 8, false, true, KIND_F16>(tmA, tmB, tmS0, tmS1, tmBs, p, stream);
      if (bn == 128) return launch_variant<128, 6, false, true, KIND_F16>(tmA, tmB, tmS0, tmS1, tmBs, p, stream);
      set_last_error("shortcut epilogue supports BN 64/128 only (got %d)", bn);
      return kErrUnsupported;
    }
  }
  switch (bn) {
    case 64: return launch_variant<64, 8, false, false, KIND>(tmA, tmB, tmS0, tmS1, tmBs, p, stream);
    case 128: return launch_variant<128, 6, false, false, KIND>(tmA, tmB, tmS0, tmS1, tmBs, p, stream);
    case 160: return launch_variant<160, 5, false, false, KIND>(tmA, tmB, tmS0, tmS1, tmBs, p, stream);
    case 192: return launch_variant<192, 4, false, false, KIND>(tmA, tmB, tmS0, tmS1, tmBs, p, stream);
    case 256: return launch_variant<256, 3, false, false, KIND>(tmA, tmB, tmS0, tmS1, tmBs, p, stream);   // + 64 KB staging
  }
  set_last_error("unsupported BN %d", bn);
  return kErrUnsupported;
}

int gemm_f16_impl(const void* A, long long lda, const void* W, long long ldw, void* out, long long ldo, int M, int N,
                  int K, const void* bias, const void* residual, long long ldr, const void* rowvec, long long ld_rowvec,
                  int rows_per_sample, int flags, int force_bn, cudaStream_t stream) {
  const int geglu = flags & 1;
  VTON_CHECK_ARG(M > 0 && N > 0 && K > 0, "gemm: empty problem M=%d N=%d K=%d", M, N, K);
  VTON_CHECK_ARG(K % 64 == 0, "gemm: K=%d must be a multiple of 64", K);
  VTON_CHECK_ARG(N % 8 == 0 && lda % 8 == 0 && ldw % 8 == 0 && ldo % 8 == 0, "gemm: N/lda/ldw/ldo must be multiples of 8");
  VTON_CHECK_ARG(!geglu || (N % 16 == 0 && !residual && !rowvec), "gemm: bad GEGLU configuration");
  // the epilogue reads bias / residual / rowvec and writes out 8 halves (16 bytes) at a time
  VTON_CHECK_ARG(aligned_to(out, 16) && aligned_to(bias, 16) && aligned_to(residual, 16) && aligned_to(rowvec, 16),
                 "gemm: out/bias/residual/rowvec must be 16-byte aligned");
  VTON_CHECK_ARG((!residual || ldr % 8 == 0) && (!rowvec || ld_rowvec % 8 == 0),
                 "gemm: ldr=%lld / ld_rowvec=%lld must be multiples of 8", ldr, ld_rowvec);
  const int bn = pick_bn(N, cdiv(M, BM), geglu != 0, false, force_bn);
  VTON_CHECK_ARG(bn != 0, "gemm: tile width force_bn=%d unsupported for this problem (N=%d, geglu=%d)", force_bn, N, geglu);
  VTON_CHECK_ARG(!geglu || N % bn == 0, "gemm: GEGLU needs N %% BN == 0 (N=%d, BN=%d)", N, bn);
  CUtensorMap tmA, tmB;
  {
    uint64_t dims[2] = {static_cast<uint64_t>(K), static_cast<uint64_t>(M)};
    uint64_t strides[1] = {static_cast<uint64_t>(lda) * 2};
    uint32_t box[2] = {64, 128};
    if (int e = encode_tmap_f16(&tmA, A, 2, dims, strides, box)) return e;
  }
  {
    uint64_t dims[2] = {static_cast<uint64_t>(K), static_cast<uint64_t>(N)};
    uint64_t strides[1] = {static_cast<uint64_t>(ldw) * 2};
    uint32_t box[2] = {64, static_cast<uint32_t>(bn)};
    if (int e = encode_tmap_f16(&tmB, W, 2, dims, strides, box)) return e;
  }
  GemmParams p{};
  p.out = static_cast<__half*>(out);
  p.ld_out = static_cast<int>(ldo);
  p.M = M;
  p.N = N;
  p.bias = static_cast<const __half*>(bias);
  p.residual = static_cast<const __half*>(residual);
  p.ld_res = static_cast<int>(ldr);
  p.rowvec = static_cast<const __half*>(rowvec);
  p.ld_rowvec = static_cast<int>(ld_rowvec);
  p.rows_per_sample = rows_per_sample;
  p.slabs_main = K / 64;
  p.act_gelu = (flags & 4) ? 2 : ((flags & 2) ? 1 : 0);
  return dispatch<KIND_F16>(bn, geglu != 0, tmA, tmB, tmA, tmA, tmB, p, cdiv(M, BM), stream);
}

// A_q [M, lda] and W_q [N, ldw] e4m3 (lda / ldw in elements = bytes), a_scale [M] and w_scale [N] fp32: the per-row
// (per-token) and per-output-channel scales of the FP8 linears. out = epi((acc * a_scale[m]) * w_scale[n]) with the fp16
// epilogue of gemm_f16_impl (bias, GEGLU, residual); flags & 1 = GEGLU, no other flag.
int gemm_e4m3_impl(const void* A, long long lda, const void* a_scale, const void* W, long long ldw, const void* w_scale,
                   void* out, long long ldo, int M, int N, int K, const void* bias, const void* residual, long long ldr,
                   int flags, int force_bn, cudaStream_t stream) {
  const int geglu = flags & 1;
  VTON_CHECK_ARG(M > 0 && N > 0 && K > 0, "gemm_e4m3: empty problem M=%d N=%d K=%d", M, N, K);
  VTON_CHECK_ARG(K % 128 == 0, "gemm_e4m3: K=%d must be a multiple of 128", K);
  VTON_CHECK_ARG((flags & ~1) == 0, "gemm_e4m3: flags=%d unsupported (only GEGLU = 1)", flags);
  VTON_CHECK_ARG(A && W && out && a_scale && w_scale, "gemm_e4m3: A, W, out, a_scale and w_scale must not be null");
  VTON_CHECK_ARG(lda % 16 == 0 && ldw % 16 == 0, "gemm_e4m3: lda=%lld / ldw=%lld must be multiples of 16 bytes", lda, ldw);
  VTON_CHECK_ARG(N % 8 == 0 && ldo % 8 == 0, "gemm_e4m3: N/ldo must be multiples of 8");
  VTON_CHECK_ARG(!geglu || (N % 16 == 0 && !residual), "gemm_e4m3: bad GEGLU configuration");
  VTON_CHECK_ARG(aligned_to(A, 16) && aligned_to(W, 16) && aligned_to(out, 16) && aligned_to(bias, 16) &&
                     aligned_to(residual, 16) && aligned_to(a_scale, 4) && aligned_to(w_scale, 8),
                 "gemm_e4m3: A/W/out/bias/residual must be 16-byte aligned, a_scale 4-byte, w_scale 8-byte");
  VTON_CHECK_ARG(!residual || ldr % 8 == 0, "gemm_e4m3: ldr=%lld must be a multiple of 8", ldr);
  const int bn = pick_bn(N, cdiv(M, BM), geglu != 0, false, force_bn);
  VTON_CHECK_ARG(bn != 0, "gemm_e4m3: tile width force_bn=%d unsupported for this problem (N=%d, geglu=%d)", force_bn, N,
                 geglu);
  VTON_CHECK_ARG(!geglu || N % bn == 0, "gemm_e4m3: GEGLU needs N %% BN == 0 (N=%d, BN=%d)", N, bn);
  CUtensorMap tmA, tmB;
  {
    uint64_t dims[2] = {static_cast<uint64_t>(K), static_cast<uint64_t>(M)};
    uint64_t strides[1] = {static_cast<uint64_t>(lda)};
    uint32_t box[2] = {128, 128};
    if (int e = encode_tmap_u8(&tmA, A, 2, dims, strides, box)) return e;
  }
  {
    uint64_t dims[2] = {static_cast<uint64_t>(K), static_cast<uint64_t>(N)};
    uint64_t strides[1] = {static_cast<uint64_t>(ldw)};
    uint32_t box[2] = {128, static_cast<uint32_t>(bn)};
    if (int e = encode_tmap_u8(&tmB, W, 2, dims, strides, box)) return e;
  }
  GemmParams p{};
  p.out = static_cast<__half*>(out);
  p.ld_out = static_cast<int>(ldo);
  p.M = M;
  p.N = N;
  p.bias = static_cast<const __half*>(bias);
  p.residual = static_cast<const __half*>(residual);
  p.ld_res = static_cast<int>(ldr);
  p.slabs_main = K / 128;
  p.a_scale = static_cast<const float*>(a_scale);
  p.w_scale = static_cast<const float*>(w_scale);
  return dispatch<KIND_E4M3>(bn, geglu != 0, tmA, tmB, tmA, tmA, tmB, p, cdiv(M, BM), stream);
}

static void pick_box(int B, int H, int W, int* bw, int* bh, int* bb) {
  int w = 1;
  while (w < 128 && W % (w * 2) == 0) w *= 2;
  int h = 1;
  while (w * h < 128 && h * 2 <= H) h *= 2;
  *bw = w;
  *bh = h;
  *bb = 128 / (w * h);
  (void)B;
}

// pixel_step = 2 (stride-2 convolution): the box spans 2*bw x 2*bh input pixels and the TMA traversal stride picks every
// second one, so the tile that lands in shared memory is the same 128 rows x 64 channels as for stride 1 and the
// "im2col" of Downsample2D never exists in memory.
static int encode_nhwc(CUtensorMap* tm, const void* base, int B, int H, int W, int C, int ldc, int bw, int bh, int bb,
                       int pixel_step = 1) {
  uint64_t dims[4] = {static_cast<uint64_t>(C), static_cast<uint64_t>(W), static_cast<uint64_t>(H),
                      static_cast<uint64_t>(B)};
  uint64_t strides[3] = {static_cast<uint64_t>(ldc) * 2, static_cast<uint64_t>(W) * ldc * 2,
                         static_cast<uint64_t>(H) * W * ldc * 2};
  uint32_t box[4] = {64, static_cast<uint32_t>(bw * pixel_step), static_cast<uint32_t>(bh * pixel_step),
                     static_cast<uint32_t>(bb)};
  uint32_t estr[4] = {1, static_cast<uint32_t>(pixel_step), static_cast<uint32_t>(pixel_step), 1};
  return encode_tmap_f16(tm, base, 4, dims, strides, box, pixel_step > 1 ? estr : nullptr);
}

// x: [B,Hin,Win,Cin] (channel stride ldx), w: [9][Cout][Cin] fp16 (tap-major), out: [B*H*W, ldo] with H = (Hin-1)/stride+1
int conv3x3_impl(const void* x, long long ldx, int B, int Hin, int Win, int Cin, const void* w, int Cout, const void* bias,
                 const void* temb, long long ld_temb, const void* sc0, int C0, const void* sc1, int C1, const void* w_sc,
                 const void* bias_sc, const void* residual, long long ldr, void* out, long long ldo, int force_bn,
                 int stride, cudaStream_t stream) {
  VTON_CHECK_ARG(B > 0 && Hin > 0 && Win > 0, "conv3x3: empty input");
  VTON_CHECK_ARG(stride == 1 || stride == 2, "conv3x3: stride %d unsupported", stride);
  VTON_CHECK_ARG(stride == 1 || (!w_sc && !residual), "conv3x3: stride 2 has no shortcut / residual form");
  const int H = (Hin - 1) / stride + 1, W = (Win - 1) / stride + 1;   // output size (padding 1)
  VTON_CHECK_ARG(Cin % 64 == 0, "conv3x3: Cin=%d must be a multiple of 64 (pad channels)", Cin);
  VTON_CHECK_ARG(Cout % 8 == 0 && ldo % 8 == 0 && ldx % 8 == 0, "conv3x3: Cout/ldo/ldx must be multiples of 8");
  VTON_CHECK_ARG(C0 % 64 == 0 && C1 % 64 == 0, "conv3x3: shortcut source channels must be multiples of 64");
  VTON_CHECK_ARG(!(w_sc && residual), "conv3x3: shortcut conv and identity residual are exclusive");
  // the epilogue reads bias / temb / bias_sc / residual and writes out 8 halves (16 bytes) at a time
  VTON_CHECK_ARG(aligned_to(out, 16) && aligned_to(bias, 16) && aligned_to(temb, 16) && aligned_to(bias_sc, 16) &&
                     aligned_to(residual, 16),
                 "conv3x3: out/bias/temb/bias_sc/residual must be 16-byte aligned");
  VTON_CHECK_ARG((!residual || ldr % 8 == 0) && (!temb || ld_temb % 8 == 0),
                 "conv3x3: ldr=%lld / ld_temb=%lld must be multiples of 8", ldr, ld_temb);
  int bw, bh, bb;
  pick_box(B, H, W, &bw, &bh, &bb);
  const int m_tiles_est = (W / bw) * cdiv(H, bh) * cdiv(B, bb);
  const int bn = pick_bn(Cout, m_tiles_est, false, w_sc != nullptr, force_bn);
  VTON_CHECK_ARG(bn != 0, "conv3x3: tile width force_bn=%d unsupported (a fused shortcut takes 64 or 128)", force_bn);
  CUtensorMap tmA, tmB, tmS0, tmS1, tmBs;
  VTON_CHECK_ARG(stride == 1 || (bw * 2 <= 256 && bh * 2 <= 256), "conv3x3: stride-2 box too large");
  if (int e = encode_nhwc(&tmA, x, B, Hin, Win, Cin, static_cast<int>(ldx), bw, bh, bb, stride)) return e;
  {
    uint64_t dims[2] = {static_cast<uint64_t>(Cin), static_cast<uint64_t>(9) * Cout};
    uint64_t strides[1] = {static_cast<uint64_t>(Cin) * 2};
    uint32_t box[2] = {64, static_cast<uint32_t>(bn)};
    if (int e = encode_tmap_f16(&tmB, w, 2, dims, strides, box)) return e;
  }
  tmS0 = tmA;
  tmS1 = tmA;
  tmBs = tmB;
  GemmParams p{};
  if (w_sc) {
    VTON_CHECK_ARG(sc0 && C0 > 0, "conv3x3: shortcut needs a source");
    if (int e = encode_nhwc(&tmS0, sc0, B, H, W, C0, C0, bw, bh, bb)) return e;
    if (sc1 && C1 > 0) {
      if (int e = encode_nhwc(&tmS1, sc1, B, H, W, C1, C1, bw, bh, bb)) return e;
    }
    const int Csc = C0 + (sc1 ? C1 : 0);
    uint64_t dims[2] = {static_cast<uint64_t>(Csc), static_cast<uint64_t>(Cout)};
    uint64_t strides[1] = {static_cast<uint64_t>(Csc) * 2};
    uint32_t box[2] = {64, static_cast<uint32_t>(bn)};
    if (int e = encode_tmap_f16(&tmBs, w_sc, 2, dims, strides, box)) return e;
    p.slabs_sc = Csc / 64;
    p.sc_split = C0 / 64;
  }
  p.out = static_cast<__half*>(out);
  p.ld_out = static_cast<int>(ldo);
  p.M = B * H * W;
  p.N = Cout;
  p.bias = static_cast<const __half*>(bias);
  p.bias_sc = static_cast<const __half*>(bias_sc);
  p.residual = static_cast<const __half*>(residual);
  p.ld_res = static_cast<int>(ldr);
  p.rowvec = static_cast<const __half*>(temb);
  p.ld_rowvec = static_cast<int>(ld_temb);
  p.slabs_main = 9 * (Cin / 64);
  p.conv = 1;
  p.stride = stride;
  p.H = H;
  p.W = W;
  p.B = B;
  p.bw = bw;
  p.bh = bh;
  p.bb = bb;
  p.tiles_x = W / bw;
  p.tiles_y = cdiv(H, bh);
  p.cin_slabs = Cin / 64;
  p.cout = Cout;
  const int m_tiles = p.tiles_x * p.tiles_y * cdiv(B, bb);
  return dispatch<KIND_F16>(bn, false, tmA, tmB, tmS0, tmS1, tmBs, p, m_tiles, stream);
}

// x: [B,H,W,Cin] fp32 NHWC (dense), w: [9][Cout][Cin] fp32 (tap-major), bias: [Cout] fp32 or null, residual: [B,H,W,Cout]
// fp32 NHWC or null (added after the bias), out: [B,H,W,Cout]. The reference upcasts the SDXL VAE to fp32 and PyTorch runs
// its fp32 convolutions as TF32 products with fp32 accumulation; this keeps that arithmetic class.
// in_fp16: x and w are fp16 (same layouts), Cin a multiple of 64; the fp16 operand has the 10-bit mantissa TF32 would
// round an fp32 operand to, so the arithmetic class is the same at twice the MMA rate. Everything else stays fp32.
int conv3x3_f32_impl(const void* x, int B, int H, int W, int Cin, const void* w, int Cout, const void* bias,
                     const void* residual, void* out, int in_fp16, cudaStream_t stream) {
  VTON_CHECK_ARG(B > 0 && H > 0 && W > 0, "conv3x3_f32: empty input");
  VTON_CHECK_ARG(Cin % 32 == 0 && Cout % 32 == 0 && Cout >= 64, "conv3x3_f32: Cin=%d / Cout=%d must be multiples of 32 (Cout >= 64)", Cin, Cout);
  VTON_CHECK_ARG(!in_fp16 || Cin % 64 == 0, "conv3x3_f32: fp16 operands need Cin=%d to be a multiple of 64", Cin);
  VTON_CHECK_ARG(x && w && out, "conv3x3_f32: null pointer");
  const int esz = in_fp16 ? 2 : 4;          // operand element size
  const int bk = in_fp16 ? 64 : 32;         // channels per 128-byte slab row
  int bw, bh, bb;
  pick_box(B, H, W, &bw, &bh, &bb);
  VTON_CHECK_ARG(bw * bh * bb == 128 && bw >= 8, "conv3x3_f32: W=%d H=%d cannot be tiled into 128-pixel boxes", W, H);
  const int m_tiles = (W / bw) * cdiv(H, bh) * cdiv(B, bb);
  const int bn = pick_bn(Cout, m_tiles, false, false, Cout % 256 == 0 ? 256 : 128);
  CUtensorMap tmA, tmB;
  {
    uint64_t dims[4] = {static_cast<uint64_t>(Cin), static_cast<uint64_t>(W), static_cast<uint64_t>(H), static_cast<uint64_t>(B)};
    uint64_t strides[3] = {static_cast<uint64_t>(Cin) * esz, static_cast<uint64_t>(W) * Cin * esz,
                           static_cast<uint64_t>(H) * W * Cin * esz};
    uint32_t box[4] = {static_cast<uint32_t>(bk), static_cast<uint32_t>(bw), static_cast<uint32_t>(bh), static_cast<uint32_t>(bb)};
    if (int e = in_fp16 ? encode_tmap_f16(&tmA, x, 4, dims, strides, box) : encode_tmap_f32(&tmA, x, 4, dims, strides, box)) return e;
  }
  {
    uint64_t dims[2] = {static_cast<uint64_t>(Cin), static_cast<uint64_t>(9) * Cout};
    uint64_t strides[1] = {static_cast<uint64_t>(Cin) * esz};
    uint32_t box[2] = {static_cast<uint32_t>(bk), static_cast<uint32_t>(bn)};
    if (int e = in_fp16 ? encode_tmap_f16(&tmB, w, 2, dims, strides, box) : encode_tmap_f32(&tmB, w, 2, dims, strides, box)) return e;
  }
  GemmParams p{};
  p.out_f32 = static_cast<float*>(out);
  p.bias_f32 = static_cast<const float*>(bias);
  p.res_f32 = static_cast<const float*>(residual);
  p.M = B * H * W;
  p.N = Cout;
  p.slabs_main = 9 * (Cin / bk);
  p.conv = 1;
  p.stride = 1;
  p.H = H;
  p.W = W;
  p.B = B;
  p.bw = bw;
  p.bh = bh;
  p.bb = bb;
  p.tiles_x = W / bw;
  p.tiles_y = cdiv(H, bh);
  p.cin_slabs = Cin / bk;
  p.cout = Cout;
  p.n_tiles = cdiv(Cout, bn);
  p.total_tiles = m_tiles * p.n_tiles;
  if (in_fp16) {
    if (bn == 256) return launch_variant<256, 4, false, false, KIND_F16IN_F32OUT>(tmA, tmB, tmA, tmA, tmB, p, stream);
    return launch_variant<128, 6, false, false, KIND_F16IN_F32OUT>(tmA, tmB, tmA, tmA, tmB, p, stream);
  }
  if (bn == 256) return launch_variant<256, 4, false, false, KIND_TF32>(tmA, tmB, tmA, tmA, tmB, p, stream);
  return launch_variant<128, 6, false, false, KIND_TF32>(tmA, tmB, tmA, tmA, tmB, p, stream);
}

}  // namespace vton
