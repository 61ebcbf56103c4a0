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
//
// Axiswise e4m3 scaling (torchao's rowwise recipe), one power-of-two scale per row or per column:
//   tn_fp8_rowwise_cast_bf16  : per-row amax, s = 2^floor(log2(448 / max(amax, 1e-12))) and the row-major copy, one
//                               read of each row; 1/s per row into a device vector.
//   tn_fp8_colwise_amax_bf16  : amax[c] = max(amax[c], max_r |x[r, c]|), the same exact integer atomicMax per column.
//   tn_fp8_colwise_cast_t_bf16: the transposed copy [cols, rows] with the scale of each column; 1/s per column.
// The scale is torchao's amax_to_scale (division in fp64, result in fp32) rounded down to a power of two, so x · s and
// the dequantisation are exact.  The rounding clears the mantissa of the fp32 scale: for a bf16 amax that is what
// exp2(floor(log2(s))) gives.  A NaN in a row (column) makes that row's (column's) scale and values NaN.
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

// ----------------------------------------------- axiswise (rowwise recipe) -----------------------------------------------
constexpr int kRowThreads = 128;
constexpr int kRowChunks = 8;   // 8-element chunks per thread held in registers: rows up to 8192 are read once
constexpr int kColStrip = 256;  // rows per CTA of the column amax

__device__ __forceinline__ float fp8_pow2_scale(float amax) {
  if (isnan(amax)) return amax;
  const float s = float(double(kFp8MaxE4M3) / fmax(double(amax), 1e-12));   // finite amax: a normal float, or 0
  return __uint_as_float(__float_as_uint(s) & 0x7F800000u);
}

// max |x| of 8 bf16, as an fp32 bit pattern
__device__ __forceinline__ uint32_t absmax8(const uint4& v) {
  const uint32_t* w = &v.x;
  uint32_t m = 0;
#pragma unroll
  for (int i = 0; i < 4; ++i) m = max(m, max((w[i] & 0x7FFFu) << 16, w[i] & 0x7FFF0000u));
  return m;
}

__device__ __forceinline__ uint2 cast8_e4m3(const uint4& v, float s0, float s1, float s2, float s3, float s4, float s5,
                                            float s6, float s7) {
  const uint32_t* w = &v.x;
  uint2 b;
  b.x = cvt_fp8x2<false>(__fmul_rn(bf16lo(w[0]), s0), __fmul_rn(bf16hi(w[0]), s1)) |
        cvt_fp8x2<false>(__fmul_rn(bf16lo(w[1]), s2), __fmul_rn(bf16hi(w[1]), s3)) << 16;
  b.y = cvt_fp8x2<false>(__fmul_rn(bf16lo(w[2]), s4), __fmul_rn(bf16hi(w[2]), s5)) |
        cvt_fp8x2<false>(__fmul_rn(bf16lo(w[3]), s6), __fmul_rn(bf16hi(w[3]), s7)) << 16;
  return b;
}

// One row per CTA: the row's chunks are loaded into registers once, reduced to the amax, then quantised from there.
__global__ void __launch_bounds__(kRowThreads)
fp8_rowwise_cast_kernel(const bf16* __restrict__ x, int64_t ldx, int64_t cols, uint8_t* out, int64_t ld_out,
                        float* inv_scale) {
  const int64_t r = blockIdx.x;
  const bf16* xr = x + r * ldx;
  const int nch = int(cols / 8);
  uint4 v[kRowChunks];
  uint32_t m = 0;
#pragma unroll
  for (int i = 0; i < kRowChunks; ++i) {
    const int ch = int(threadIdx.x) + kRowThreads * i;
    if (ch < nch) {
      v[i] = __ldg(reinterpret_cast<const uint4*>(xr + 8 * ch));
      m = max(m, absmax8(v[i]));
    }
  }
  for (int ch = int(threadIdx.x) + kRowThreads * kRowChunks; ch < nch; ch += kRowThreads)
    m = max(m, absmax8(__ldg(reinterpret_cast<const uint4*>(xr + 8 * ch))));
  m = __reduce_max_sync(0xffffffffu, m);
  __shared__ uint32_t wmax[kRowThreads / 32];
  if ((threadIdx.x & 31) == 0) wmax[threadIdx.x >> 5] = m;
  __syncthreads();
#pragma unroll
  for (int i = 0; i < kRowThreads / 32; ++i) m = max(m, wmax[i]);
  const float s = fp8_pow2_scale(__uint_as_float(m));
  if (threadIdx.x == 0) inv_scale[r] = __frcp_rn(s);
  uint8_t* orow = out + r * ld_out;
#pragma unroll
  for (int i = 0; i < kRowChunks; ++i) {
    const int ch = int(threadIdx.x) + kRowThreads * i;
    if (ch < nch) *reinterpret_cast<uint2*>(orow + 8 * ch) = cast8_e4m3(v[i], s, s, s, s, s, s, s, s);
  }
  for (int ch = int(threadIdx.x) + kRowThreads * kRowChunks; ch < nch; ch += kRowThreads)
    *reinterpret_cast<uint2*>(orow + 8 * ch) =
        cast8_e4m3(__ldg(reinterpret_cast<const uint4*>(xr + 8 * ch)), s, s, s, s, s, s, s, s);
}

// CTA: 64 columns x kColStrip rows; thread (ty, tx) keeps the maxima of chunk tx over rows ty, ty + 32, ...
__global__ void __launch_bounds__(256)
fp8_colwise_amax_kernel(const bf16* __restrict__ x, int64_t ldx, int64_t rows, int64_t cols, float* amax) {
  __shared__ uint32_t red[32][65];
  const int tx = int(threadIdx.x) & 7, ty = int(threadIdx.x) >> 3;
  const int64_t c = int64_t(blockIdx.x) * 64 + 8 * tx;
  const int64_t r0 = int64_t(blockIdx.y) * kColStrip, r1 = min(rows, r0 + kColStrip);
  uint32_t m[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (c < cols)   // cols % 16 == 0: a chunk is wholly inside or outside
    for (int64_t r = r0 + ty; r < r1; r += 32) {
      const uint4 v = __ldg(reinterpret_cast<const uint4*>(x + r * ldx + c));
      const uint32_t* w = &v.x;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        m[2 * i] = max(m[2 * i], (w[i] & 0x7FFFu) << 16);
        m[2 * i + 1] = max(m[2 * i + 1], w[i] & 0x7FFF0000u);
      }
    }
#pragma unroll
  for (int e = 0; e < 8; ++e) red[ty][8 * tx + e] = m[e];
  __syncthreads();
  if (threadIdx.x >= 64) return;
  const int64_t col = int64_t(blockIdx.x) * 64 + threadIdx.x;
  if (col >= cols) return;
  uint32_t mm = 0;
#pragma unroll 8
  for (int i = 0; i < 32; ++i) mm = max(mm, red[i][threadIdx.x]);
  if (mm) atomicMax(reinterpret_cast<unsigned int*>(amax + col), mm);
}

// One 64 x 64 tile per CTA as fp8_cast_kernel, transposed copy only, with the scale of each column.
__global__ void __launch_bounds__(kCastThreads)
fp8_colwise_cast_t_kernel(const bf16* __restrict__ x, int64_t ldx, int64_t rows, int64_t cols, const float* amax,
                          uint8_t* out_t, int64_t ld_out_t, float* inv_scale) {
  __shared__ __align__(16) uint8_t tile[kCastTile * kCastPitch];
  __shared__ float sc[kCastTile];
  const int64_t r0 = int64_t(blockIdx.y) * kCastTile, c0 = int64_t(blockIdx.x) * kCastTile;
  if (threadIdx.x < kCastTile) {
    const int64_t c = c0 + threadIdx.x;
    const float s = c < cols ? fp8_pow2_scale(amax[c]) : 0.f;
    sc[threadIdx.x] = s;
    if (inv_scale && blockIdx.y == 0 && c < cols) inv_scale[c] = __frcp_rn(s);
  }
  __syncthreads();
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const int q = int(threadIdx.x) + kCastThreads * j;
    const int rr = q >> 3, cc = 8 * (q & 7);
    const int64_t r = r0 + rr, c = c0 + cc;
    if (r >= rows || c >= cols) continue;
    const float* s = sc + cc;
    *reinterpret_cast<uint2*>(tile + rr * kCastPitch + cc) =
        cast8_e4m3(__ldg(reinterpret_cast<const uint4*>(x + r * ldx + c)), s[0], s[1], s[2], s[3], s[4], s[5], s[6],
                   s[7]);
  }
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
static bool aligned4(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 3) == 0; }

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

#define TN_AXIS_REQUIRE_X(name)                                                                                      \
  TN_REQUIRE(rows > 0 && cols > 0 && rows % 16 == 0 && cols % 16 == 0,                                           \
             name ": rows=%lld cols=%lld must be positive multiples of 16", (long long)rows, (long long)cols);       \
  TN_REQUIRE(ldx >= cols && ldx % 8 == 0 && aligned16(x), name ": x must be 16 B aligned with ldx >= cols, a multiple of 8")

extern "C" int tn_fp8_rowwise_cast_bf16(const void* x, int64_t ldx, int64_t rows, int64_t cols, void* out,
                                        int64_t ld_out, float* inv_scale, tn_stream_t stream_) {
  clear_error();
  TN_REQUIRE(x && out && inv_scale, "tn_fp8_rowwise_cast_bf16: null pointer (x, out and inv_scale)");
  TN_AXIS_REQUIRE_X("tn_fp8_rowwise_cast_bf16");
  TN_REQUIRE(aligned4(inv_scale), "tn_fp8_rowwise_cast_bf16: inv_scale must be 4 B aligned");
  TN_REQUIRE(rows < (int64_t(1) << 31), "tn_fp8_rowwise_cast_bf16: too many rows");
  TN_REQUIRE(ld_out >= cols && ld_out % 16 == 0 && aligned16(out),
             "tn_fp8_rowwise_cast_bf16: out must be 16 B aligned with ld_out >= cols, a multiple of 16");
  fp8_rowwise_cast_kernel<<<unsigned(rows), kRowThreads, 0, static_cast<cudaStream_t>(stream_)>>>(
      static_cast<const bf16*>(x), ldx, cols, static_cast<uint8_t*>(out), ld_out, inv_scale);
  TN_CHECK_CUDA(cudaGetLastError());
  return TN_OK;
}

extern "C" int tn_fp8_colwise_amax_bf16(const void* x, int64_t ldx, int64_t rows, int64_t cols, float* amax,
                                        tn_stream_t stream_) {
  clear_error();
  TN_REQUIRE(x && amax, "tn_fp8_colwise_amax_bf16: null pointer");
  TN_AXIS_REQUIRE_X("tn_fp8_colwise_amax_bf16");
  TN_REQUIRE(aligned4(amax), "tn_fp8_colwise_amax_bf16: amax must be 4 B aligned (integer atomicMax)");
  TN_REQUIRE((rows + kColStrip - 1) / kColStrip < 65535, "tn_fp8_colwise_amax_bf16: too many rows");
  const dim3 grid(unsigned((cols + 63) / 64), unsigned((rows + kColStrip - 1) / kColStrip));
  fp8_colwise_amax_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream_)>>>(static_cast<const bf16*>(x), ldx, rows,
                                                                                 cols, amax);
  TN_CHECK_CUDA(cudaGetLastError());
  return TN_OK;
}

extern "C" int tn_fp8_colwise_cast_t_bf16(const void* x, int64_t ldx, int64_t rows, int64_t cols, const float* amax,
                                          void* out_t, int64_t ld_out_t, float* inv_scale, tn_stream_t stream_) {
  clear_error();
  TN_REQUIRE(x && amax && out_t, "tn_fp8_colwise_cast_t_bf16: null pointer (x, amax and out_t)");
  TN_AXIS_REQUIRE_X("tn_fp8_colwise_cast_t_bf16");
  TN_REQUIRE(aligned4(amax) && (!inv_scale || aligned4(inv_scale)),
             "tn_fp8_colwise_cast_t_bf16: amax and inv_scale must be 4 B aligned");
  TN_REQUIRE(rows / kCastTile < 65535, "tn_fp8_colwise_cast_t_bf16: too many rows");
  TN_REQUIRE(ld_out_t >= rows && ld_out_t % 16 == 0 && aligned16(out_t),
             "tn_fp8_colwise_cast_t_bf16: out_t must be 16 B aligned with ld_out_t >= rows, a multiple of 16");
  const dim3 grid(unsigned((cols + kCastTile - 1) / kCastTile), unsigned((rows + kCastTile - 1) / kCastTile));
  fp8_colwise_cast_t_kernel<<<grid, kCastThreads, 0, static_cast<cudaStream_t>(stream_)>>>(
      static_cast<const bf16*>(x), ldx, rows, cols, amax, static_cast<uint8_t*>(out_t), ld_out_t, inv_scale);
  TN_CHECK_CUDA(cudaGetLastError());
  return TN_OK;
}
#undef TN_AXIS_REQUIRE_X
