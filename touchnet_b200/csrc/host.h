// touchnet_b200 :: host-side helpers shared by the C-ABI translation units.
#pragma once

#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace tn {

// thread-local last-error string (tn_last_error()).  Returns `code` so callers can `return fail(...)`.
int fail(int code, const char* fmt, ...);
void clear_error();

enum { TN_OK = 0, TN_ERR_ARG = 1, TN_ERR_CUDA = 2, TN_ERR_UNSUPPORTED = 3 };

#define TN_CHECK_CUDA(expr)                                                                         \
  do {                                                                                              \
    cudaError_t _e = (expr);                                                                        \
    if (_e != cudaSuccess)                                                                          \
      return ::tn::fail(::tn::TN_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), \
                        __FILE__, __LINE__);                                                        \
  } while (0)

#define TN_REQUIRE(cond, ...)                                         \
  do {                                                                \
    if (!(cond)) return ::tn::fail(::tn::TN_ERR_ARG, __VA_ARGS__);    \
  } while (0)

// TMA descriptor encoders (driver entry point resolved lazily through the runtime; no -lcuda link).
// elem_bytes: 1 (FP8, as uint8), 2 (bf16) or 4 (f32).  Strides in bytes (must be multiples of 16).  SWIZZLE_128B iff swizzle128.
int encode_tmap_2d(CUtensorMap* out, const void* ptr, int elem_bytes, uint64_t dim0, uint64_t dim1,
                   uint64_t stride1_bytes, uint32_t box0, uint32_t box1, bool swizzle128);
int encode_tmap_3d(CUtensorMap* out, const void* ptr, int elem_bytes, uint64_t dim0, uint64_t dim1, uint64_t dim2,
                   uint64_t stride1_bytes, uint64_t stride2_bytes, uint32_t box0, uint32_t box1, uint32_t box2,
                   bool swizzle128);

int sm_count();
int gemm_group();   // raster group of the GEMM (tn_set_gemm_group)
int gemm_l2_hints();  // 1: operand loads of the GEMM carry L2 eviction hints (tn_set_gemm_l2_hints)

}  // namespace tn
