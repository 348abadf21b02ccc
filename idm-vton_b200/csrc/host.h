// Host-side helpers shared by the C-ABI translation units: error reporting and TMA descriptor encode.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

namespace vton {

// error codes returned through the C ABI (0 = success)
enum : int { kOk = 0, kErrInvalid = 1, kErrCuda = 2, kErrUnsupported = 3 };

void set_last_error(const char* fmt, ...);
const char* get_last_error();

#define VTON_CHECK_ARG(cond, ...)      \
  do {                                 \
    if (!(cond)) {                     \
      vton::set_last_error(__VA_ARGS__); \
      return vton::kErrInvalid;        \
    }                                  \
  } while (0)

#define VTON_CUDA(call)                                                                          \
  do {                                                                                           \
    cudaError_t e__ = (call);                                                                    \
    if (e__ != cudaSuccess) {                                                                    \
      vton::set_last_error("%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__), __FILE__, __LINE__); \
      return vton::kErrCuda;                                                                     \
    }                                                                                            \
  } while (0)

// Encodes a tiled fp16 tensor map with SWIZZLE_128B (inner box = 64 halves = 128 B) or, with swizzle_bytes = 64,
// SWIZZLE_64B (inner box = 32 halves).
// dims/strides innermost-first; strides in BYTES for dims 1..rank-1. Returns 0 on success.
int encode_tmap_f16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                    const uint32_t* box, const uint32_t* elem_strides = nullptr, int swizzle_bytes = 128);

// fp32 elements, SWIZZLE_128B (inner box = 32 floats = 128 B): the TF32 convolution of the VAE.
int encode_tmap_f32(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                    const uint32_t* box);

// One-byte elements (e4m3 operands of the FP8 linears), SWIZZLE_128B (inner box = 128 elements = 128 B), or with
// swizzle_bytes = 0 no swizzle (the FP8 garment K/V tiles and exponents, converted by the attention's producer warps).
int encode_tmap_u8(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                   const uint32_t* box, int swizzle_bytes = 128);

inline int cdiv(int a, int b) { return (a + b - 1) / b; }

// Pointers the kernels access with 16-byte vector loads / stores (epilogue operands, norm rows) must be 16-byte aligned;
// a null pointer (operand absent) passes.
inline bool aligned_to(const void* p, uintptr_t bytes) { return (reinterpret_cast<uintptr_t>(p) & (bytes - 1)) == 0; }

// Streaming multiprocessors of the current device (read once per device: 132 on an H100 SXM, fewer on other parts).
int num_sms();

// Programmatic dependent launch (option "programmatic_launch", default OFF, see host.cu): the hot kernels are launched
// with cudaLaunchAttributeProgrammaticStreamSerialization; they initialise their barriers and prefetch tensor maps, call
// griddepcontrol.wait, only then touch global memory, and call
// griddepcontrol.launch_dependents once they hold all their resources — so the launch latency and part of the set-up
// of kernel n+1 overlap the tail of kernel n (~930 launches per captured denoise step).
int pdl_enabled();
void set_pdl(int on);

template <typename... KArgs, typename... Args>
inline cudaError_t launch_kernel(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                                 Args... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

// Number of kernels this library has launched (or recorded into a capturing stream) since load.
void count_launch(int n = 1);
long long launch_count();

}  // namespace vton
