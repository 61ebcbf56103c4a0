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

// ------------------------------------------- skinny-M decode GEMM (rowwise e4m3) -------------------------------------------
// D[M, N] = X[M, K]·W[N, K]ᵀ for the few rows of a cached decode step.  The weight is far too narrow in M for the wgmma
// tiles, so the kernel streams W once per group of up to 64 rows of X:
//   - each CTA quantises its group of X rows into shared memory with the rule of fp8_rowwise_cast_kernel (the same amax,
//     power-of-two scale and sat_rne bytes; rows past M are zero), then loops over 8-column tiles of W (persistent grid);
//   - within a tile the 8 warps split K: warp w takes the 64-byte chunks w, w + 8, ... and accumulates them in order with
//     mma.sync.m16n8k32 e4m3 (16 rows of X per MMA).  Each lane loads one 16-byte piece of a weight row per chunk and
//     feeds its halves to two MMAs; the X bytes are read from shared memory with the same permutation of k, so the sum
//     is over the same products;
//   - the 8 warp partials are added in warp order through shared memory, then the rowwise epilogue runs.
// An output element depends on its row of X, W, inv_sw (and R) only: the MMA's rows are independent, the chunk order is a
// function of K, and nothing is atomic.
constexpr int kDecThreads = 256;
constexpr int kDecWarps = kDecThreads / 32;
constexpr int kDecTileN = 8;                    // output columns per tile (one n8 MMA)
constexpr int kDecMaxMTiles = 4;                // 64 rows of X per group
constexpr int kDecSmemMax = 200 * 1024;

__device__ __forceinline__ void mma_e4m3_16832(float* c, uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                               uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k32.row.col.f32.e4m3.e4m3.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
      "{%0, %1, %2, %3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

// shared-memory pitch of a quantised X row: holds K rounded up to 64 (zero tail), and is 64 mod 128 so that the two rows
// each quarter-warp reads sit in different banks
__host__ __device__ constexpr int dec_pitch(int K) { return (K + 127) / 128 * 128 + 64; }

__host__ __device__ constexpr int dec_smem(int K, int mtiles, int nw) {
  return mtiles * 16 * dec_pitch(K) + mtiles * 16 * 4 + kDecWarps * nw * mtiles * 16 * kDecTileN * 4;
}

// EPI 0: bf16(acc·ia·iw); 1: + R; 2: SwiGLU over W = [Wg; Wu] (2N rows), H only.  MT: 16-row MMA tiles per group.
template <int EPI, int MT>
__global__ void __launch_bounds__(kDecThreads)
fp8_decode_gemm_kernel(const bf16* __restrict__ x, int64_t ldx, const uint8_t* __restrict__ w, int64_t ldw,
                       const float* __restrict__ inv_sw, const bf16* __restrict__ r, int64_t ldr, bf16* __restrict__ d,
                       int64_t ldd, int M, int N, int K) {
  constexpr int NW = EPI == 2 ? 2 : 1;          // weight rows per output column
  constexpr int G = 16 * MT;
  constexpr int U = EPI == 2 && MT > 2 ? 2 : 8 / NW;   // chunks in flight per batch (no spill at 64 SwiGLU rows)
  extern __shared__ __align__(16) uint8_t dsm[];
  const int pitch = dec_pitch(K);
  uint8_t* xq = dsm;
  float* ia = reinterpret_cast<float*>(dsm + G * pitch);
  float* red = ia + G;                          // [warp][NW][G][8]
  const int warp = int(threadIdx.x) >> 5, lane = int(threadIdx.x) & 31;
  const int g = lane >> 2, tig = lane & 3;
  const int m0 = int(blockIdx.y) * G;
  const int kpad = (K + 63) / 64 * 64, nch = kpad / 64, ntiles = N / kDecTileN;

  // the first tile's weight lines start on their way to L2 while X is quantised
  if (int(blockIdx.x) < ntiles)
    for (int c = warp; c < nch; c += kDecWarps) {
      const int k = 64 * c + 16 * tig;
      if (k < K)
#pragma unroll
        for (int j = 0; j < NW; ++j)
          asm volatile("prefetch.global.L2 [%0];" ::"l"(w + (int64_t(j) * N + kDecTileN * blockIdx.x + g) * ldw + k));
    }

  // X rows -> e4m3 in shared memory, one warp per row (fp8_rowwise_cast_kernel's amax, scale and bytes)
  for (int rr = warp; rr < G; rr += kDecWarps) {
    uint8_t* q = xq + rr * pitch;
    const int row = m0 + rr;
    if (row < M) {
      const bf16* xr = x + int64_t(row) * ldx;
      uint32_t m = 0;
      for (int ch = lane; ch < K / 8; ch += 32) m = max(m, absmax8(__ldg(reinterpret_cast<const uint4*>(xr + 8 * ch))));
      m = __reduce_max_sync(0xffffffffu, m);
      const float s = fp8_pow2_scale(__uint_as_float(m));
      if (lane == 0) ia[rr] = __frcp_rn(s);
      for (int ch = lane; ch < K / 8; ch += 32)
        *reinterpret_cast<uint2*>(q + 8 * ch) =
            cast8_e4m3(__ldg(reinterpret_cast<const uint4*>(xr + 8 * ch)), s, s, s, s, s, s, s, s);
      for (int ch = K / 8 + lane; ch < kpad / 8; ch += 32) *reinterpret_cast<uint2*>(q + 8 * ch) = make_uint2(0, 0);
    } else {
      if (lane == 0) ia[rr] = 0.f;
      for (int ch = lane; ch < kpad / 8; ch += 32) *reinterpret_cast<uint2*>(q + 8 * ch) = make_uint2(0, 0);
    }
  }
  __syncthreads();

  for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
    const int n0 = kDecTileN * t;
    float acc[NW][MT][4];
#pragma unroll
    for (int j = 0; j < NW; ++j)
#pragma unroll
      for (int i = 0; i < MT; ++i) acc[j][i][0] = acc[j][i][1] = acc[j][i][2] = acc[j][i][3] = 0.f;
    const uint8_t* wr[NW];
#pragma unroll
    for (int j = 0; j < NW; ++j) wr[j] = w + (int64_t(j) * N + n0 + g) * ldw + 16 * tig;
    for (int c0 = warp; c0 < nch; c0 += kDecWarps * U) {
      uint4 b[U][NW];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int c = c0 + kDecWarps * u;
        const bool ok = c < nch && 64 * c + 16 * tig < K;   // K % 16 == 0: a piece is wholly inside or outside
#pragma unroll
        for (int j = 0; j < NW; ++j)
          b[u][j] = ok ? __ldg(reinterpret_cast<const uint4*>(wr[j] + 64 * c)) : make_uint4(0, 0, 0, 0);
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int c = c0 + kDecWarps * u;
        if (c >= nch) break;                                 // warp-uniform
        const uint8_t* qa = xq + g * pitch + 64 * c + 16 * tig;
#pragma unroll
        for (int i = 0; i < MT; ++i) {
          const uint4 lo = *reinterpret_cast<const uint4*>(qa + 16 * i * pitch);
          const uint4 hi = *reinterpret_cast<const uint4*>(qa + (16 * i + 8) * pitch);
#pragma unroll
          for (int j = 0; j < NW; ++j) {
            mma_e4m3_16832(acc[j][i], lo.x, hi.x, lo.y, hi.y, b[u][j].x, b[u][j].y);
            mma_e4m3_16832(acc[j][i], lo.z, hi.z, lo.w, hi.w, b[u][j].z, b[u][j].w);
          }
        }
      }
    }
#pragma unroll
    for (int j = 0; j < NW; ++j)
#pragma unroll
      for (int i = 0; i < MT; ++i) {
        float* p = red + ((warp * NW + j) * G + 16 * i + g) * kDecTileN + 2 * tig;
        *reinterpret_cast<float2*>(p) = make_float2(acc[j][i][0], acc[j][i][1]);
        *reinterpret_cast<float2*>(p + 8 * kDecTileN) = make_float2(acc[j][i][2], acc[j][i][3]);
      }
    __syncthreads();
    for (int e = int(threadIdx.x); e < G * kDecTileN; e += kDecThreads) {
      const int rr = e / kDecTileN, row = m0 + rr, col = n0 + e % kDecTileN;
      if (row >= M) continue;
      float s[NW];
#pragma unroll
      for (int j = 0; j < NW; ++j) {
        s[j] = red[j * G * kDecTileN + e];
#pragma unroll
        for (int v = 1; v < kDecWarps; ++v) s[j] += red[(v * NW + j) * G * kDecTileN + e];
      }
      // the rowwise wgmma epilogue's order: (acc · 1/s_a) · 1/s_b, rounded to bf16
      float out;
      if constexpr (EPI == 2) {
        const float gt = bf16_round(s[0] * ia[rr] * inv_sw[col]);
        const float up = bf16_round(s[1] * ia[rr] * inv_sw[N + col]);
        out = bf16_round(gt / (1.f + __expf(-gt))) * up;
      } else {
        out = s[0] * ia[rr] * inv_sw[col];
        if constexpr (EPI == 1) out = bf16_round(out) + __bfloat162float(r[int64_t(row) * ldr + col]);
      }
      d[int64_t(row) * ldd + col] = __float2bfloat16_rn(out);
    }
    __syncthreads();
  }
}

template <int EPI, int MT>
static int launch_decode_gemm(const bf16* x, int64_t ldx, const uint8_t* w, int64_t ldw, const float* inv_sw,
                              const bf16* r, int64_t ldr, bf16* d, int64_t ldd, int M, int N, int K,
                              cudaStream_t stream) {
  auto kern = fp8_decode_gemm_kernel<EPI, MT>;
  static bool attr = false;
  if (!attr) {
    TN_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kDecSmemMax));
    attr = true;
  }
  const int smem = dec_smem(K, MT, EPI == 2 ? 2 : 1);
  int per_sm = 0;
  TN_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kDecThreads, smem));
  const int groups = (M + 16 * MT - 1) / (16 * MT), ntiles = N / kDecTileN;
  const int ctas = max(1, max(per_sm, 1) * sm_count() / groups);
  const dim3 grid(unsigned(min(ntiles, ctas)), unsigned(groups));
  kern<<<grid, kDecThreads, smem, stream>>>(x, ldx, w, ldw, inv_sw, r, ldr, d, ldd, M, N, K);
  TN_CHECK_CUDA(cudaGetLastError());
  return TN_OK;
}

template <int EPI>
static int decode_gemm(int mt, const bf16* x, int64_t ldx, const uint8_t* w, int64_t ldw, const float* inv_sw,
                       const bf16* r, int64_t ldr, bf16* d, int64_t ldd, int M, int N, int K, cudaStream_t stream) {
  switch (mt) {
    case 1: return launch_decode_gemm<EPI, 1>(x, ldx, w, ldw, inv_sw, r, ldr, d, ldd, M, N, K, stream);
    case 2: return launch_decode_gemm<EPI, 2>(x, ldx, w, ldw, inv_sw, r, ldr, d, ldd, M, N, K, stream);
    case 3: return launch_decode_gemm<EPI, 3>(x, ldx, w, ldw, inv_sw, r, ldr, d, ldd, M, N, K, stream);
    default: return launch_decode_gemm<EPI, 4>(x, ldx, w, ldw, inv_sw, r, ldr, d, ldd, M, N, K, stream);
  }
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

extern "C" int tn_gemm_fp8_decode(const void* X, int64_t ldx, const void* W, int64_t ldw, const float* inv_sw, int epi,
                                  const void* R, int64_t ldr, void* D, int64_t ldd, int M, int N, int K,
                                  tn_stream_t stream_) {
  clear_error();
  TN_REQUIRE(X && W && inv_sw && D, "tn_gemm_fp8_decode: null pointer (X, W, inv_sw and D)");
  TN_REQUIRE(epi >= 0 && epi <= 2, "tn_gemm_fp8_decode: epi=%d must be 0 (plain), 1 (+ residual) or 2 (SwiGLU)", epi);
  TN_REQUIRE((epi == 1) == (R != nullptr), "tn_gemm_fp8_decode: R is required with epi 1 and only there");
  TN_REQUIRE(M > 0 && N > 0 && K > 0 && N % 16 == 0 && K % 16 == 0,
             "tn_gemm_fp8_decode: M=%d must be positive, N=%d and K=%d positive multiples of 16", M, N, K);
  TN_REQUIRE(dec_smem(K, 1, epi == 2 ? 2 : 1) <= kDecSmemMax, "tn_gemm_fp8_decode: K=%d too large (16 rows of X must "
             "fit in shared memory)", K);
  TN_REQUIRE(ldx >= K && ldx % 8 == 0 && aligned16(X), "tn_gemm_fp8_decode: X must be 16 B aligned with ldx >= K, a "
             "multiple of 8");
  TN_REQUIRE(ldw >= K && ldw % 16 == 0 && aligned16(W), "tn_gemm_fp8_decode: W must be 16 B aligned with ldw >= K, a "
             "multiple of 16");
  TN_REQUIRE(aligned4(inv_sw), "tn_gemm_fp8_decode: inv_sw must be 4 B aligned");
  TN_REQUIRE(ldd >= N && (!R || ldr >= N), "tn_gemm_fp8_decode: ldd and ldr must be >= N");
  const int need = (M + 15) / 16;
  int mt = need < kDecMaxMTiles ? need : kDecMaxMTiles;
  while (mt > 1 && dec_smem(K, mt, epi == 2 ? 2 : 1) > kDecSmemMax) --mt;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const bf16* x = static_cast<const bf16*>(X);
  const uint8_t* w = static_cast<const uint8_t*>(W);
  const bf16* r = static_cast<const bf16*>(R);
  bf16* d = static_cast<bf16*>(D);
  if (epi == 0) return decode_gemm<0>(mt, x, ldx, w, ldw, inv_sw, r, ldr, d, ldd, M, N, K, stream);
  if (epi == 1) return decode_gemm<1>(mt, x, ldx, w, ldw, inv_sw, r, ldr, d, ldd, M, N, K, stream);
  return decode_gemm<2>(mt, x, ldx, w, ldw, inv_sw, r, ldr, d, ldd, M, N, K, stream);
}
