// Host-side plumbing for libb200vton.so: last-error string and TMA descriptor encoding.
// cuTensorMapEncodeTiled is resolved through the runtime (cudaGetDriverEntryPoint), so the library has no link-time
// dependency on libcuda and loads on a machine without a driver (the CPU build/"symbols export" check).
#include "host.h"

#include <atomic>
#include <mutex>

namespace vton {

static thread_local char g_err[512] = "";

void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
const char* get_last_error() { return g_err; }

// Off by default for eager launches, switched on by denoise.py for the kernel nodes of the captured step graph. Every kernel
// launched with the attribute calls griddepcontrol.wait before it reads global memory written by its predecessors.
int num_sms() {
  static std::atomic<int> cache[64];
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  int n = cache[dev].load(std::memory_order_relaxed);
  if (n == 0) {
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) return 132;
    cache[dev].store(n, std::memory_order_relaxed);
  }
  return n;
}

static std::atomic<int> g_pdl{0};
int pdl_enabled() { return g_pdl.load(std::memory_order_relaxed); }
void set_pdl(int on) { g_pdl.store(on ? 1 : 0, std::memory_order_relaxed); }
static std::atomic<long long> g_launches{0};
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
long long launch_count() { return g_launches.load(std::memory_order_relaxed); }

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

static int encode_tmap_any(CUtensorMap* out, CUtensorMapDataType dtype, const void* base, int rank, const uint64_t* dims,
                           const uint64_t* strides_bytes, const uint32_t* box, const uint32_t* elem_strides,
                           int swizzle_bytes) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) {
    set_last_error("cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
    return kErrCuda;
  }
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0) {
    set_last_error("tensor map base %p is not 16-byte aligned", base);
    return kErrInvalid;
  }
  cuuint64_t gdim[5];
  cuuint64_t gstr[4];
  cuuint32_t gbox[5];
  cuuint32_t gel[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    gbox[i] = box[i];
    gel[i] = elem_strides ? elem_strides[i] : 1;
    if (i > 0) {
      gstr[i - 1] = strides_bytes[i - 1];
      if (gstr[i - 1] % 16 != 0) {
        set_last_error("tensor map stride %llu not a multiple of 16 bytes", (unsigned long long)gstr[i - 1]);
        return kErrInvalid;
      }
    }
  }
  CUresult r = fn(out, dtype, static_cast<cuuint32_t>(rank), const_cast<void*>(base), gdim,
                  gstr, gbox, gel, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  swizzle_bytes == 0    ? CU_TENSOR_MAP_SWIZZLE_NONE
                  : swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                                        : CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled failed with CUresult %d (rank %d dims %llu,%llu box %u,%u)", (int)r, rank,
                   (unsigned long long)dims[0], (unsigned long long)dims[1], box[0], box[1]);
    return kErrCuda;
  }
  return kOk;
}

int encode_tmap_f16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                    const uint32_t* box, const uint32_t* elem_strides, int swizzle_bytes) {
  return encode_tmap_any(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, base, rank, dims, strides_bytes, box, elem_strides,
                         swizzle_bytes);
}

int encode_tmap_f32(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                    const uint32_t* box) {
  return encode_tmap_any(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, base, rank, dims, strides_bytes, box, nullptr, 128);
}

int encode_tmap_u8(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                   const uint32_t* box, int swizzle_bytes) {
  return encode_tmap_any(out, CU_TENSOR_MAP_DATA_TYPE_UINT8, base, rank, dims, strides_bytes, box, nullptr, swizzle_bytes);
}

}  // namespace vton
