// FreeU (diffusers 0.25.0 `apply_freeu`, https://arxiv.org/abs/2309.11497) on one resnet input of the try-on UNet's
// up stages 0 and 1 (src/unet_block_hacked_tryon.py:2322-2344,2458-2480), in one launch:
//   hidden[..., :Ch/2] = fp16(float(hidden) * b)                                   (the backbone half, in place)
//   skip_out = fourier_filter(skip, threshold=1, scale=s)
// fourier_filter multiplies the shifted 2-D spectrum of each (sample, channel) plane by s on the 2 x 2 block at the
// centre, i.e. on the frequencies {0, -1} along each axis (only 0 along an axis of size 1). In closed form, with
// theta = 2 pi h / H, phi = 2 pi w / W:
//   out = x + (s - 1) / HW * [A + Re(P e^-i phi) + Re(Q e^-i theta) + Re(R e^-i (theta + phi))],
//   A = sum x, P = sum x e^i phi, Q = sum x e^i theta, R = sum x e^i (theta + phi)
// (P and R drop when W = 1, Q and R when H = 1: the two frequencies of that axis are the same bin). So the filter is
// 7 real sums per channel and one elementwise pass; no FFT, any H and W.
//
// A CTA owns (sample, a group of 8 V channels) over all H x W pixels: V lanes of 16 bytes per pixel, 256 / V pixel
// lanes. It sums in fp32 in a fixed order (per-thread strided pixels, a warp-shuffle tree, the 8 warps in order), with
// no atomics, so the result does not depend on the batch or the launch and the kernel can be captured in a graph.
// Then it re-reads its pixels (from L2) and writes the filtered values, each rounded to fp16 once. The CTA reads all of
// its region before writing it, so skip_out may be skip. The CTAs of a sample also split that sample's hidden half.
#include "common.cuh"
#include "host.h"

namespace vton {

constexpr int kFreeuThreads = 256;
constexpr int kFreeuSums = 7;

struct Twiddle {
  float cw, sw, ch, sh, cr, sr;
};

// cos / sin of phi, theta and theta + phi; the angles are reduced in integers (2w / W in [0, 2)) before sincospif
__device__ __forceinline__ Twiddle twiddle(int p, int H, int W) {
  const int h = p / W, w = p - h * W;
  Twiddle t;
  sincospif(static_cast<float>(2 * w) / static_cast<float>(W), &t.sw, &t.cw);
  sincospif(static_cast<float>(2 * h) / static_cast<float>(H), &t.sh, &t.ch);
  t.cr = t.ch * t.cw - t.sh * t.sw;
  t.sr = t.sh * t.cw + t.ch * t.sw;
  return t;
}

__global__ void __launch_bounds__(kFreeuThreads)
freeu_kernel(__half* hidden, int Ch, const __half* skip, __half* out, int Cs, int H, int W, int V, int groups,
             float b, float s, int use_h, int use_w) {
  __shared__ float red[kFreeuThreads / 32][4][kFreeuSums * 8];
  __shared__ float fin[4][kFreeuSums * 8];
  pdl_wait();
  pdl_launch_dependents();
  const int n = blockIdx.x / groups, g = blockIdx.x - n * groups;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int HW = H * W;

  // ---- backbone half of hidden: 4 halves (8 bytes) per access; Ch % 8 == 0 makes Ch / 2 a multiple of 4
  {
    const int hv = Ch / 8;                           // 4-half vectors per row of the half
    const long long per_sample = static_cast<long long>(HW) * hv;
    __half* hs = hidden + static_cast<long long>(n) * HW * Ch;
    for (long long e = static_cast<long long>(g) * kFreeuThreads + tid; e < per_sample;
         e += static_cast<long long>(groups) * kFreeuThreads) {
      const long long p = e / hv;
      const int v = static_cast<int>(e - p * hv);
      uint2* ptr = reinterpret_cast<uint2*>(hs + p * Ch + 4 * v);
      uint2 u = *ptr;
      const float2 a = unpack_h2(u.x), c = unpack_h2(u.y);
      u.x = pack_h2(__fmul_rn(a.x, b), __fmul_rn(a.y, b));
      u.y = pack_h2(__fmul_rn(c.x, b), __fmul_rn(c.y, b));
      *ptr = u;
    }
  }

  // ---- the 7 sums of each of this CTA's 8 V channels
  const int vl = tid % V, pl = tid / V, P = kFreeuThreads / V;
  const int c0 = (g * V + vl) * 8;
  const long long base = static_cast<long long>(n) * HW * Cs + c0;
  float acc[kFreeuSums][8];
#pragma unroll
  for (int k = 0; k < kFreeuSums; ++k)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[k][j] = 0.f;
  for (int p = pl; p < HW; p += P) {
    const uint4 u = *reinterpret_cast<const uint4*>(skip + base + static_cast<long long>(p) * Cs);
    const Twiddle t = twiddle(p, H, W);
    const uint32_t w4[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float2 x = unpack_h2(w4[q]);
      const float xs[2] = {x.x, x.y};
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int j = 2 * q + r;
        acc[0][j] += xs[r];
        acc[1][j] = fmaf(xs[r], t.cw, acc[1][j]);
        acc[2][j] = fmaf(xs[r], t.sw, acc[2][j]);
        acc[3][j] = fmaf(xs[r], t.ch, acc[3][j]);
        acc[4][j] = fmaf(xs[r], t.sh, acc[4][j]);
        acc[5][j] = fmaf(xs[r], t.cr, acc[5][j]);
        acc[6][j] = fmaf(xs[r], t.sr, acc[6][j]);
      }
    }
  }
  // lanes l and l ^ (V 2^k) hold the same channels
  for (int off = V; off < 32; off <<= 1)
#pragma unroll
    for (int k = 0; k < kFreeuSums; ++k)
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[k][j] += __shfl_xor_sync(0xffffffffu, acc[k][j], off);
  if (lane < V) {
#pragma unroll
    for (int k = 0; k < kFreeuSums; ++k)
#pragma unroll
      for (int j = 0; j < 8; ++j) red[warp][lane][k * 8 + j] = acc[k][j];
  }
  __syncthreads();
  if (tid < V * kFreeuSums * 8) {
    const int v = tid / (kFreeuSums * 8), kj = tid - v * (kFreeuSums * 8), k = kj / 8;
    float sum = 0.f;
#pragma unroll
    for (int w = 0; w < kFreeuThreads / 32; ++w) sum += red[w][v][kj];
    // P (cos / sin of phi) and R vanish along a size-1 width, Q and R along a size-1 height
    const bool keep = k == 0 || ((k == 1 || k == 2) && use_w) || ((k == 3 || k == 4) && use_h) ||
                      (k >= 5 && use_w && use_h);
    fin[v][kj] = keep ? sum * ((s - 1.f) / static_cast<float>(HW)) : 0.f;
  }
  __syncthreads();

  // ---- filtered skip
  float f[kFreeuSums][8];
#pragma unroll
  for (int k = 0; k < kFreeuSums; ++k)
#pragma unroll
    for (int j = 0; j < 8; ++j) f[k][j] = fin[vl][k * 8 + j];
  for (int p = pl; p < HW; p += P) {
    const long long off = base + static_cast<long long>(p) * Cs;
    const uint4 u = *reinterpret_cast<const uint4*>(skip + off);
    const Twiddle t = twiddle(p, H, W);
    const uint32_t w4[4] = {u.x, u.y, u.z, u.w};
    uint32_t o4[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float2 x = unpack_h2(w4[q]);
      float y[2];
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int j = 2 * q + r;
        float c = f[0][j];
        c = fmaf(f[1][j], t.cw, c);
        c = fmaf(f[2][j], t.sw, c);
        c = fmaf(f[3][j], t.ch, c);
        c = fmaf(f[4][j], t.sh, c);
        c = fmaf(f[5][j], t.cr, c);
        c = fmaf(f[6][j], t.sr, c);
        y[r] = (r == 0 ? x.x : x.y) + c;
      }
      o4[q] = pack_h2(y[0], y[1]);
    }
    *reinterpret_cast<uint4*>(out + off) = make_uint4(o4[0], o4[1], o4[2], o4[3]);
  }
}

static bool overlaps(const void* a, long long a_bytes, const void* b, long long b_bytes) {
  const uintptr_t pa = reinterpret_cast<uintptr_t>(a), pb = reinterpret_cast<uintptr_t>(b);
  return pa < pb + static_cast<uintptr_t>(b_bytes) && pb < pa + static_cast<uintptr_t>(a_bytes);
}

int freeu_impl(void* hidden, int Ch, const void* skip, void* skip_out, int Cs, int B, int H, int W, float b, float s,
               cudaStream_t stream) {
  VTON_CHECK_ARG(hidden && skip && skip_out, "freeu: hidden, skip and skip_out are required");
  VTON_CHECK_ARG(B > 0 && H > 0 && W > 0 && Ch > 0 && Cs > 0, "freeu: bad shape B=%d H=%d W=%d Ch=%d Cs=%d", B, H, W,
                 Ch, Cs);
  VTON_CHECK_ARG(Ch % 8 == 0 && Cs % 8 == 0, "freeu: channel counts must be multiples of 8 (Ch=%d, Cs=%d)", Ch, Cs);
  VTON_CHECK_ARG(static_cast<long long>(H) * W < (1LL << 31), "freeu: H x W = %lld is too large",
                 static_cast<long long>(H) * W);
  VTON_CHECK_ARG(aligned_to(hidden, 16) && aligned_to(skip, 16) && aligned_to(skip_out, 16),
                 "freeu: hidden, skip and skip_out must be 16-byte aligned");
  const long long px = static_cast<long long>(B) * H * W;
  const long long hb = px * Ch * 2, sb = px * Cs * 2;
  VTON_CHECK_ARG(!overlaps(hidden, hb, skip, sb) && !overlaps(hidden, hb, skip_out, sb),
                 "freeu: hidden may not overlap skip or skip_out");
  VTON_CHECK_ARG(skip_out == skip || !overlaps(skip, sb, skip_out, sb),
                 "freeu: skip_out must be skip itself or not overlap it");
  // 2 vectors of 16 bytes (one 32-byte sector) per pixel and CTA where the width allows
  const int V = (Cs / 8) % 2 == 0 ? 2 : 1;
  const int groups = Cs / (8 * V);
  VTON_CHECK_ARG(static_cast<long long>(B) * groups < (1LL << 31), "freeu: too many CTAs");
  VTON_CUDA(launch_kernel(freeu_kernel, dim3(static_cast<unsigned>(B * groups)), dim3(kFreeuThreads), 0, stream,
                          static_cast<__half*>(hidden), Ch, static_cast<const __half*>(skip),
                          static_cast<__half*>(skip_out), Cs, H, W, V, groups, b, s, H > 1 ? 1 : 0, W > 1 ? 1 : 0));
  count_launch();
  return kOk;
}

}  // namespace vton
