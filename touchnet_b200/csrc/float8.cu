// touchnet_b200 :: dynamic per-tensor FP8 quantisation for the FP8 decoder-block GEMMs (torchao's tensorwise recipe).
//
//   tn_fp8_amax_bf16 : amax = max(amax, max |x|) over a bf16 [rows, cols] view.  The caller zeroes the device float;
//                      several calls into one float give one scale for several tensors (the q/k/v weights).
//   tn_fp8_cast_bf16 : s = fmax / max(amax, 1e-12) on the device, then sat_rne(x · s) as e4m3 (fmax 448) or e5m2
//                      (fmax 57344) into the row-major copy, the transposed copy, or both from one read of x; writes 1/s.
//
// |x| of a bf16 is its bit pattern with the sign cleared, and non-negative floats order like their bit patterns (NaN
// above +inf), so the amax is an integer atomicMax: exact, and independent of the order of the blocks.  A NaN in x makes
// the amax, the scale and every quantised value NaN, as the torch restatement
// (x.float() * s).clamp(-fmax, fmax).to(float8) with s = fmax / amax.clamp(min=1e-12) does.
#include <stdio.h>

#include "../../include/touchnet_b200.h"
#include "common.cuh"
#include "host.h"

namespace tn {

constexpr float kFp8MaxE4M3 = 448.f;
constexpr float kFp8MaxE5M2 = 57344.f;
constexpr int kAmaxThreads = 128;
constexpr int kCastTile = 64;              // 64 x 64 elements per CTA
constexpr int kCastThreads = 256;
constexpr int kCastPitch = kCastTile + 8;  // shared-memory row pitch of the byte tile (8-byte aligned rows)

__global__ void __launch_bounds__(kAmaxThreads)
fp8_amax_kernel(const bf16* __restrict__ x, int64_t ldx, int64_t rows, int64_t cols, float* amax) {
  uint32_t m = 0;
  for (int64_t r = blockIdx.x; r < rows; r += gridDim.x)
    for (int64_t c = 8 * int64_t(threadIdx.x); c < cols; c += 8 * kAmaxThreads) {
      const uint4 v = __ldg(reinterpret_cast<const uint4*>(x + r * ldx + c));
      const uint32_t* w = &v.x;
#pragma unroll
      for (int i = 0; i < 4; ++i) m = max(m, max((w[i] & 0x7FFFu) << 16, w[i] & 0x7FFF0000u));
    }
  m = __reduce_max_sync(0xffffffffu, m);
  __shared__ uint32_t wmax[kAmaxThreads / 32];
  if ((threadIdx.x & 31) == 0) wmax[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
#pragma unroll
    for (int i = 1; i < kAmaxThreads / 32; ++i) m = max(m, wmax[i]);
    if (m) atomicMax(reinterpret_cast<unsigned int*>(amax), m);
  }
}

__device__ __forceinline__ float fp8_scale(float amax, float fmax) {
  return __fdiv_rn(fmax, isnan(amax) ? amax : fmaxf(amax, 1e-12f));
}

// two fp32 -> two saturated, round-to-nearest-even 8-bit floats: lo in bits 0-7, hi in bits 8-15
template <bool E5M2>
__device__ __forceinline__ uint32_t cvt_fp8x2(float lo, float hi) {
  uint16_t d;
  if constexpr (E5M2) asm("cvt.rn.satfinite.e5m2x2.f32 %0, %1, %2;" : "=h"(d) : "f"(hi), "f"(lo));
  else asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(d) : "f"(hi), "f"(lo));
  return d;
}

// One 64 x 64 tile per CTA: each thread quantises two 8-element row chunks (writing them to `out` as they are) and
// drops the bytes into a shared tile, from which each thread gathers one 16-row column chunk of the transposed copy.
template <bool E5M2>
__global__ void __launch_bounds__(kCastThreads)
fp8_cast_kernel(const bf16* __restrict__ x, int64_t ldx, int64_t rows, int64_t cols, const float* amax, uint8_t* out,
                int64_t ld_out, uint8_t* out_t, int64_t ld_out_t, float* inv_scale) {
  __shared__ __align__(16) uint8_t tile[kCastTile * kCastPitch];
  const float s = fp8_scale(*amax, E5M2 ? kFp8MaxE5M2 : kFp8MaxE4M3);
  if (inv_scale && blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) *inv_scale = __frcp_rn(s);
  const int64_t r0 = int64_t(blockIdx.y) * kCastTile, c0 = int64_t(blockIdx.x) * kCastTile;
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const int q = int(threadIdx.x) + kCastThreads * j;
    const int rr = q >> 3, cc = 8 * (q & 7);
    const int64_t r = r0 + rr, c = c0 + cc;
    if (r >= rows || c >= cols) continue;   // cols % 16 == 0: a chunk is wholly inside or outside
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(x + r * ldx + c));
    const uint32_t* w = &v.x;
    uint2 b;
    b.x = cvt_fp8x2<E5M2>(__fmul_rn(bf16lo(w[0]), s), __fmul_rn(bf16hi(w[0]), s)) |
          cvt_fp8x2<E5M2>(__fmul_rn(bf16lo(w[1]), s), __fmul_rn(bf16hi(w[1]), s)) << 16;
    b.y = cvt_fp8x2<E5M2>(__fmul_rn(bf16lo(w[2]), s), __fmul_rn(bf16hi(w[2]), s)) |
          cvt_fp8x2<E5M2>(__fmul_rn(bf16lo(w[3]), s), __fmul_rn(bf16hi(w[3]), s)) << 16;
    if (out) *reinterpret_cast<uint2*>(out + r * ld_out + c) = b;
    if (out_t) *reinterpret_cast<uint2*>(tile + rr * kCastPitch + cc) = b;
  }
  if (!out_t) return;
  __syncthreads();
  const int cc = int(threadIdx.x) >> 2, rq = 16 * (int(threadIdx.x) & 3);
  const int64_t c = c0 + cc, r = r0 + rq;
  if (c >= cols || r >= rows) return;        // rows % 16 == 0
  uint32_t w[4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
    w[i] = uint32_t(tile[(rq + 4 * i) * kCastPitch + cc]) | uint32_t(tile[(rq + 4 * i + 1) * kCastPitch + cc]) << 8 |
           uint32_t(tile[(rq + 4 * i + 2) * kCastPitch + cc]) << 16 |
           uint32_t(tile[(rq + 4 * i + 3) * kCastPitch + cc]) << 24;
  *reinterpret_cast<uint4*>(out_t + c * ld_out_t + r) = make_uint4(w[0], w[1], w[2], w[3]);
}

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace tn

using namespace tn;

extern "C" int tn_fp8_amax_bf16(const void* x, int64_t ldx, int64_t rows, int64_t cols, float* amax,
                                tn_stream_t stream_) {
  clear_error();
  TN_REQUIRE(x && amax, "tn_fp8_amax_bf16: null pointer");
  TN_REQUIRE(rows > 0 && cols > 0 && rows % 16 == 0 && cols % 16 == 0,
             "tn_fp8_amax_bf16: rows=%lld cols=%lld must be positive multiples of 16", (long long)rows, (long long)cols);
  TN_REQUIRE(ldx >= cols && ldx % 8 == 0 && aligned16(x), "tn_fp8_amax_bf16: x must be 16 B aligned with ldx >= cols, a multiple of 8");
  const int64_t grid = rows < int64_t(sm_count()) * 16 ? rows : int64_t(sm_count()) * 16;
  fp8_amax_kernel<<<int(grid), kAmaxThreads, 0, static_cast<cudaStream_t>(stream_)>>>(static_cast<const bf16*>(x), ldx,
                                                                                       rows, cols, amax);
  TN_CHECK_CUDA(cudaGetLastError());
  return TN_OK;
}

extern "C" int tn_fp8_cast_bf16(const void* x, int64_t ldx, int64_t rows, int64_t cols, int e5m2, const float* amax,
                                void* out, int64_t ld_out, void* out_t, int64_t ld_out_t, float* inv_scale,
                                tn_stream_t stream_) {
  clear_error();
  TN_REQUIRE(x && amax && (out || out_t), "tn_fp8_cast_bf16: null pointer (x, amax and at least one output)");
  TN_REQUIRE(rows > 0 && cols > 0 && rows % 16 == 0 && cols % 16 == 0,
             "tn_fp8_cast_bf16: rows=%lld cols=%lld must be positive multiples of 16", (long long)rows, (long long)cols);
  TN_REQUIRE(rows / kCastTile < 65535, "tn_fp8_cast_bf16: too many rows");
  TN_REQUIRE(ldx >= cols && ldx % 8 == 0 && aligned16(x), "tn_fp8_cast_bf16: x must be 16 B aligned with ldx >= cols, a multiple of 8");
  TN_REQUIRE(!out || (ld_out >= cols && ld_out % 16 == 0 && aligned16(out)),
             "tn_fp8_cast_bf16: out must be 16 B aligned with ld_out >= cols, a multiple of 16");
  TN_REQUIRE(!out_t || (ld_out_t >= rows && ld_out_t % 16 == 0 && aligned16(out_t)),
             "tn_fp8_cast_bf16: out_t must be 16 B aligned with ld_out_t >= rows, a multiple of 16");
  const dim3 grid(unsigned((cols + kCastTile - 1) / kCastTile), unsigned((rows + kCastTile - 1) / kCastTile));
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  auto kern = e5m2 ? fp8_cast_kernel<true> : fp8_cast_kernel<false>;
  kern<<<grid, kCastThreads, 0, stream>>>(static_cast<const bf16*>(x), ldx, rows, cols, amax, static_cast<uint8_t*>(out),
                                          ld_out, static_cast<uint8_t*>(out_t), ld_out_t, inv_scale);
  TN_CHECK_CUDA(cudaGetLastError());
  return TN_OK;
}
