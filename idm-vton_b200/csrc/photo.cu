// Full-resolution photos (include/b200vton.h, b200vton_resample_u8 / b200vton_paste_u8): Pillow-exact resampling of
// uint8 crops (ImagingResample's 8-bit path: fixed-point coefficients, horizontal pass into a uint8 intermediate, then
// the vertical pass) and the paste of the resampled output back into the photo. Integer arithmetic only, so every
// result is Pillow's to the byte and independent of the launch configuration. b200vton_clip_pixels_u8 turns garment
// images already resampled to the CLIP size into the image encoder's pixels through a 3 x 256 lookup table.
//
// A batch of photos of different sizes runs as one launch per pass: blockIdx.y selects the descriptor, and the CTAs of
// a row stride over that image's outputs. One thread per output byte: neighbouring threads read neighbouring source
// bytes (same row, channels and columns in order), so the loads coalesce in both passes.
#include <algorithm>

#include "../../include/b200vton.h"
#include "host.h"

namespace vton {
namespace {

constexpr int kPrecisionBits = 32 - 8 - 2;     // Pillow's PRECISION_BITS for 8-bit images
constexpr int kThreads = 256;
constexpr int kMaxDescs = 4096;

__device__ __forceinline__ uint8_t clip8(int s) {
  if (s >= (1 << kPrecisionBits << 8)) return 255;
  if (s <= 0) return 0;
  return static_cast<uint8_t>(s >> kPrecisionBits);
}

// Writes output byte (y, x, c) and, when asked for, its fp32 NCHW value (fp32 IEEE division and subtraction, as numpy's
// `a / 255` and torchvision's ToTensor + Normalize([0.5], [0.5]) compute them).
__device__ __forceinline__ void store_out(const b200vton_resample_desc& d, int y, int x, int c, uint8_t v) {
  d.dst[static_cast<long long>(y) * d.dst_pitch + static_cast<long long>(x) * d.channels + c] = v;
  if (d.out_f32) {
    float f = __fdiv_rn(static_cast<float>(v), 255.f);
    if (d.f32_mode == 1) f = __fdiv_rn(__fsub_rn(f, 0.5f), 0.5f);
    d.out_f32[(static_cast<long long>(c) * d.out_h + y) * d.out_w + x] = f;
  }
}

// Pillow's ImagingResampleHorizontal_8bpc over crop rows [tmp_first, tmp_first + tmp_rows): into the intermediate, or
// straight into dst when there is no vertical pass (then tmp_first = 0 and tmp_rows = out_h = crop_h).
__global__ void __launch_bounds__(kThreads) resample_h_kernel(const b200vton_resample_desc* descs,
                                                              const int32_t* tables, uint8_t* ws) {
  const b200vton_resample_desc d = descs[blockIdx.y];
  if (!d.need_x) return;
  const int C = d.channels;
  const long long row = static_cast<long long>(d.out_w) * C;
  const long long total = row * d.tmp_rows;
  const int32_t* bounds = tables + d.bounds_x;
  const int32_t* coefs = tables + d.coefs_x;
  uint8_t* tmp = ws + d.tmp_offset;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int r = static_cast<int>(i / row);
    const int rem = static_cast<int>(i - r * row);
    const int x = rem / C, c = rem - (rem / C) * C;
    const int first = bounds[2 * x], taps = bounds[2 * x + 1];
    const int32_t* k = coefs + static_cast<long long>(x) * d.ksize_x;
    const uint8_t* s = d.src + static_cast<long long>(d.crop_y + d.tmp_first + r) * d.src_pitch +
                       static_cast<long long>(d.crop_x + first) * C + c;
    int ss = 1 << (kPrecisionBits - 1);
    for (int t = 0; t < taps; ++t) ss += static_cast<int>(s[t * C]) * k[t];
    if (d.need_y) tmp[i] = clip8(ss);
    else store_out(d, r, x, c, clip8(ss));
  }
}

// Pillow's ImagingResampleVertical_8bpc on the intermediate (or on the crop itself when there was no horizontal pass);
// with neither pass, Pillow's copy of the crop.
__global__ void __launch_bounds__(kThreads) resample_v_kernel(const b200vton_resample_desc* descs,
                                                              const int32_t* tables, const uint8_t* ws) {
  const b200vton_resample_desc d = descs[blockIdx.y];
  if (d.need_x && !d.need_y) return;      // the horizontal pass wrote dst
  const int C = d.channels;
  const long long row = static_cast<long long>(d.out_w) * C;
  const long long total = row * d.out_h;
  const uint8_t* base;
  long long pitch;
  int row0;                               // source row of crop row 0
  if (d.need_x) {
    base = ws + d.tmp_offset;
    pitch = row;
    row0 = -d.tmp_first;
  } else {
    base = d.src + static_cast<long long>(d.crop_y) * d.src_pitch + static_cast<long long>(d.crop_x) * C;
    pitch = d.src_pitch;
    row0 = 0;
  }
  const int32_t* bounds = tables + d.bounds_y;
  const int32_t* coefs = tables + d.coefs_y;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int y = static_cast<int>(i / row);
    const int rem = static_cast<int>(i - y * row);
    const int x = rem / C, c = rem - (rem / C) * C;
    uint8_t v;
    if (!d.need_y) {
      v = base[static_cast<long long>(y) * pitch + rem];
    } else {
      const int first = bounds[2 * y], taps = bounds[2 * y + 1];
      const int32_t* k = coefs + static_cast<long long>(y) * d.ksize_y;
      const uint8_t* s = base + static_cast<long long>(row0 + first) * pitch + rem;
      int ss = 1 << (kPrecisionBits - 1);
      for (int t = 0; t < taps; ++t) ss += static_cast<int>(s[t * pitch]) * k[t];
      v = clip8(ss);
    }
    store_out(d, y, x, c, v);
  }
}

__global__ void __launch_bounds__(kThreads) paste_kernel(const b200vton_paste_desc* descs) {
  const b200vton_paste_desc d = descs[blockIdx.y];
  const long long row = 3LL * d.width;
  const long long total = row * d.height;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int y = static_cast<int>(i / row);
    const int rem = static_cast<int>(i - y * row);
    const int x = rem / 3;
    const int bx = x - d.box_x, by = y - d.box_y;
    bool take = bx >= 0 && bx < d.box_w && by >= 0 && by < d.box_h;
    if (take && d.mask) take = d.mask[static_cast<long long>(y - d.mask_y) * d.mask_pitch + (x - d.mask_x)] >= 128;
    d.dst[static_cast<long long>(y) * d.dst_pitch + rem] =
        take ? d.image[static_cast<long long>(by) * d.image_pitch + 3LL * bx + (rem - 3 * x)]
             : d.photo[static_cast<long long>(y) * d.photo_pitch + rem];
  }
}

// CLIPImageProcessor's centre crop, rescale and normalize of a batch of CLIP-size images: out[j][c][y][x] =
// table[c][src_j[crop_y + y][crop_x + x][c]]. One thread per output float, in NCHW order, so the stores coalesce.
__global__ void __launch_bounds__(kThreads) clip_pixels_kernel(const b200vton_clip_desc* descs, const float* table,
                                                               float* out) {
  __shared__ float lut[3 * 256];
  for (int i = threadIdx.x; i < 3 * 256; i += blockDim.x) lut[i] = table[i];
  __syncthreads();
  const b200vton_clip_desc d = descs[blockIdx.y];
  constexpr int kPlane = B200VTON_CLIP_SIZE * B200VTON_CLIP_SIZE;
  float* o = out + static_cast<long long>(blockIdx.y) * 3 * kPlane;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < 3 * kPlane; i += gridDim.x * blockDim.x) {
    const int c = i / kPlane, rem = i - c * kPlane;
    const int y = rem / B200VTON_CLIP_SIZE, x = rem - y * B200VTON_CLIP_SIZE;
    const uint8_t v = d.src[static_cast<long long>(d.crop_y + y) * d.src_pitch + 3LL * (d.crop_x + x) + c];
    o[i] = lut[c * 256 + v];
  }
}

unsigned grid_x(long long max_total) {
  const long long want = (max_total + kThreads - 1) / kThreads;
  const long long cap = 8LL * num_sms();
  return static_cast<unsigned>(want < 1 ? 1 : (want < cap ? want : cap));
}

bool in_table(long long off, long long len, long long table_len) { return off >= 0 && len >= 0 && off + len <= table_len; }

}  // namespace

int resample_u8_impl(const b200vton_resample_desc* descs, const void* descs_dev, int n, const int32_t* tables,
                     long long table_len, void* workspace, long long workspace_bytes, cudaStream_t stream) {
  VTON_CHECK_ARG(descs && descs_dev && n > 0 && n <= kMaxDescs, "resample_u8: need 1..%d descriptors (host and device)",
                 kMaxDescs);
  VTON_CHECK_ARG(aligned_to(descs_dev, 8), "resample_u8: descs_dev must be 8-byte aligned");
  long long max_h = 0, max_v = 0;
  bool any_h = false;
  for (int j = 0; j < n; ++j) {
    const b200vton_resample_desc& d = descs[j];
    VTON_CHECK_ARG(d.src && d.dst && (d.channels == 1 || d.channels == 3) && (d.f32_mode == 0 || d.f32_mode == 1),
                   "resample_u8: descriptor %d: null src/dst, channels %d or f32_mode %d", j, d.channels, d.f32_mode);
    VTON_CHECK_ARG(d.src_w > 0 && d.src_h > 0 && d.crop_w > 0 && d.crop_h > 0 && d.crop_x >= 0 && d.crop_y >= 0 &&
                       d.crop_x + d.crop_w <= d.src_w && d.crop_y + d.crop_h <= d.src_h && d.out_w > 0 && d.out_h > 0,
                   "resample_u8: descriptor %d: crop (%d,%d) %dx%d of a %dx%d photo to %dx%d", j, d.crop_x, d.crop_y,
                   d.crop_w, d.crop_h, d.src_w, d.src_h, d.out_w, d.out_h);
    VTON_CHECK_ARG(d.src_pitch >= static_cast<long long>(d.src_w) * d.channels &&
                       d.dst_pitch >= static_cast<long long>(d.out_w) * d.channels,
                   "resample_u8: descriptor %d: pitch below a row", j);
    VTON_CHECK_ARG(d.need_x == (d.out_w != d.crop_w) && d.need_y == (d.out_h != d.crop_h),
                   "resample_u8: descriptor %d: need_x / need_y must be (out != crop) per axis", j);
    if (d.need_x)
      VTON_CHECK_ARG(d.ksize_x > 0 && in_table(d.bounds_x, 2LL * d.out_w, table_len) &&
                         in_table(d.coefs_x, static_cast<long long>(d.out_w) * d.ksize_x, table_len),
                     "resample_u8: descriptor %d: horizontal tables outside the %lld entries", j, table_len);
    if (d.need_y)
      VTON_CHECK_ARG(d.ksize_y > 0 && in_table(d.bounds_y, 2LL * d.out_h, table_len) &&
                         in_table(d.coefs_y, static_cast<long long>(d.out_h) * d.ksize_y, table_len),
                     "resample_u8: descriptor %d: vertical tables outside the %lld entries", j, table_len);
    if (d.need_x) {
      any_h = true;
      if (d.need_y) {
        VTON_CHECK_ARG(workspace && d.tmp_first >= 0 && d.tmp_rows > 0 && d.tmp_first + d.tmp_rows <= d.crop_h &&
                           in_table(d.tmp_offset, static_cast<long long>(d.tmp_rows) * d.out_w * d.channels,
                                    workspace_bytes),
                       "resample_u8: descriptor %d: intermediate rows [%d, +%d) at %lld outside the crop or the "
                       "%lld-byte workspace", j, d.tmp_first, d.tmp_rows, static_cast<long long>(d.tmp_offset),
                       workspace_bytes);
      } else {
        VTON_CHECK_ARG(d.tmp_first == 0 && d.tmp_rows == d.crop_h,
                       "resample_u8: descriptor %d: without a vertical pass every crop row is resampled", j);
      }
      max_h = std::max(max_h, static_cast<long long>(d.tmp_rows) * d.out_w * d.channels);
    }
    max_v = std::max(max_v, static_cast<long long>(d.out_h) * d.out_w * d.channels);
  }
  VTON_CHECK_ARG(tables || !any_h, "resample_u8: tables is null");
  const auto* dd = static_cast<const b200vton_resample_desc*>(descs_dev);
  if (any_h) {
    resample_h_kernel<<<dim3(grid_x(max_h), n), kThreads, 0, stream>>>(dd, tables, static_cast<uint8_t*>(workspace));
    count_launch();
    VTON_CUDA(cudaGetLastError());
  }
  resample_v_kernel<<<dim3(grid_x(max_v), n), kThreads, 0, stream>>>(dd, tables,
                                                                      static_cast<const uint8_t*>(workspace));
  count_launch();
  VTON_CUDA(cudaGetLastError());
  return kOk;
}

int paste_u8_impl(const b200vton_paste_desc* descs, const void* descs_dev, int n, cudaStream_t stream) {
  VTON_CHECK_ARG(descs && descs_dev && n > 0 && n <= kMaxDescs, "paste_u8: need 1..%d descriptors (host and device)",
                 kMaxDescs);
  VTON_CHECK_ARG(aligned_to(descs_dev, 8), "paste_u8: descs_dev must be 8-byte aligned");
  long long max_total = 0;
  for (int j = 0; j < n; ++j) {
    const b200vton_paste_desc& d = descs[j];
    VTON_CHECK_ARG(d.photo && d.dst && d.image && d.width > 0 && d.height > 0 &&
                       d.photo_pitch >= 3LL * d.width && d.dst_pitch >= 3LL * d.width,
                   "paste_u8: descriptor %d: null pointer, empty photo or pitch below a row", j);
    VTON_CHECK_ARG(d.box_w > 0 && d.box_h > 0 && d.box_x >= 0 && d.box_y >= 0 && d.box_x + d.box_w <= d.width &&
                       d.box_y + d.box_h <= d.height && d.image_pitch >= 3LL * d.box_w,
                   "paste_u8: descriptor %d: box (%d,%d) %dx%d outside the %dx%d photo", j, d.box_x, d.box_y, d.box_w,
                   d.box_h, d.width, d.height);
    if (d.mask)
      VTON_CHECK_ARG(d.mask_x <= d.box_x && d.mask_y <= d.box_y && d.mask_x + d.mask_w >= d.box_x + d.box_w &&
                         d.mask_y + d.mask_h >= d.box_y + d.box_h && d.mask_pitch >= d.mask_w,
                     "paste_u8: descriptor %d: the mask does not cover the box", j);
    max_total = std::max(max_total, 3LL * d.width * d.height);
  }
  paste_kernel<<<dim3(grid_x(max_total), n), kThreads, 0, stream>>>(static_cast<const b200vton_paste_desc*>(descs_dev));
  count_launch();
  VTON_CUDA(cudaGetLastError());
  return kOk;
}

int clip_pixels_u8_impl(const b200vton_clip_desc* descs, const void* descs_dev, int n, const float* table, float* out,
                        cudaStream_t stream) {
  VTON_CHECK_ARG(descs && descs_dev && n > 0 && n <= kMaxDescs,
                 "clip_pixels_u8: need 1..%d descriptors (host and device)", kMaxDescs);
  VTON_CHECK_ARG(aligned_to(descs_dev, 8), "clip_pixels_u8: descs_dev must be 8-byte aligned");
  VTON_CHECK_ARG(table && out && aligned_to(table, 4) && aligned_to(out, 4),
                 "clip_pixels_u8: table and out must be non-null and 4-byte aligned");
  constexpr int S = B200VTON_CLIP_SIZE;
  for (int j = 0; j < n; ++j) {
    const b200vton_clip_desc& d = descs[j];
    VTON_CHECK_ARG(d.src && d.src_w > 0 && d.src_h > 0 && d.src_pitch >= 3LL * d.src_w,
                   "clip_pixels_u8: descriptor %d: null src, empty image or pitch below a row", j);
    VTON_CHECK_ARG(d.crop_x >= 0 && d.crop_y >= 0 && d.crop_x + S <= d.src_w && d.crop_y + S <= d.src_h,
                   "clip_pixels_u8: descriptor %d: crop (%d,%d) %dx%d outside the %dx%d image", j, d.crop_x, d.crop_y,
                   S, S, d.src_w, d.src_h);
  }
  clip_pixels_kernel<<<dim3(grid_x(3LL * S * S), n), kThreads, 0, stream>>>(
      static_cast<const b200vton_clip_desc*>(descs_dev), table, out);
  count_launch();
  VTON_CUDA(cudaGetLastError());
  return kOk;
}

}  // namespace vton
