// touchnet_b200 :: data augmentation of the ASR recipe on the GPU, over utterances packed back to back.
//
// Replaces the application half of (the random draws stay on the host, touchnet_b200/augment.py):
//   audio_resample        touchnet/data/functions.py:83-96   -> torchaudio.transforms.Resample (sinc_interp_hann)
//   audio_speed_perturb   touchnet/data/functions.py:99-114  (sox `speed s` + `rate sr` == resampling from sr*s to sr)
//   audiofeat_spec_aug    touchnet/data/functions.py:193-217
//   audiofeat_spec_sub    touchnet/data/functions.py:220-239
//   audiofeat_spec_trim   touchnet/data/functions.py:242-255
//
// resample_kernel: one CTA per tile of RS output samples of one utterance.  The input window the tile needs is staged
// in shared memory with coalesced loads (zero outside the utterance); banks of up to RS_MAX_SMEM_BANK floats (the speed
// perturbation ones) are staged too, larger ones (44.1 / 22.05 kHz) are read through L1/L2.  Outputs are computed in
// phase-major order, so the 32 lanes of a warp share one bank row (broadcast loads) and step through the staged input
// at the odd-or-small stride `orig`; they are written to a staging tile and stored coalesced.  Every output is one
// fmaf chain over the taps in order: no atomics, bit-reproducible.  A 1:1 bank is an exact copy.
// spec_augment_kernel: one warp per output frame; only copies and zeros, so it is bit-exact.
#include <stdlib.h>

#include "../../include/touchnet_b200.h"
#include "common.cuh"
#include "host.h"

namespace tn {

constexpr int RS_THREADS = 256;
constexpr int RS_MAX_BANKS = 16;
constexpr int RS_MAX_SMEM_BANK = 8192;   // floats (32 KB)
constexpr int RS_MAX_TILE = 8192;

struct ResampleBank {
  int orig, nw, width, taps, offset;   // gcd-reduced rates, filter half-width, 2*width + orig, offset into `banks`
};

struct ResampleParams {
  const void* x;
  int x_is_i16;
  const int64_t* in_off;     // [n_utts + 1] input samples
  const int64_t* out_off;    // [n_utts + 1] output samples
  const int64_t* tile_off;   // [n_utts + 1] tiles
  const int32_t* utt_bank;   // [n_utts]
  int n_utts, tile, xs_cap, w_cap;
  const float* banks;
  float* y;
  ResampleBank bank[RS_MAX_BANKS];
};

__device__ __forceinline__ int find_segment(const int64_t* __restrict__ off, int n, int64_t v) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (off[mid] <= v) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__device__ __forceinline__ float load_wav(const void* x, int is_i16, int64_t i) {
  return is_i16 ? float(reinterpret_cast<const int16_t*>(x)[i]) * (1.0f / 32768.0f)
                : reinterpret_cast<const float*>(x)[i];
}

__global__ void __launch_bounds__(RS_THREADS) resample_kernel(const ResampleParams p) {
  extern __shared__ float rs_smem[];
  const int64_t tile = blockIdx.x;
  const int u = find_segment(p.tile_off, p.n_utts, tile);
  const ResampleBank b = p.bank[p.utt_bank[u]];
  const int64_t in0 = p.in_off[u], in_len = p.in_off[u + 1] - in0;
  const int64_t out0 = p.out_off[u], out_len = p.out_off[u + 1] - out0;
  const int64_t t0 = (tile - p.tile_off[u]) * p.tile;
  const int64_t t1 = min(t0 + int64_t(p.tile), out_len);
  const int tid = threadIdx.x;
  if (b.orig == b.nw) {   // 1:1: exact copy (out_len == in_len)
    for (int64_t n = t0 + tid; n < t1; n += RS_THREADS) p.y[out0 + n] = load_wav(p.x, p.x_is_i16, in0 + n);
    return;
  }
  float* ys = rs_smem;                   // [tile]
  float* xs = ys + p.tile;               // [xs_cap]
  float* ws = xs + p.xs_cap;             // [w_cap] (small banks only)
  const int64_t i_first = t0 / b.nw, i_last = (t1 - 1) / b.nw;
  const int n_i = int(i_last - i_first) + 1;
  const int64_t s0 = i_first * b.orig - b.width;
  const int span = (n_i - 1) * b.orig + b.taps;
  for (int s = tid; s < span; s += RS_THREADS) {
    const int64_t g = s0 + s;
    xs[s] = (g >= 0 && g < in_len) ? load_wav(p.x, p.x_is_i16, in0 + g) : 0.f;
  }
  const int bank_len = b.nw * b.taps;
  const bool w_smem = bank_len <= p.w_cap;
  if (w_smem)
    for (int i = tid; i < bank_len; i += RS_THREADS) ws[i] = __ldg(p.banks + b.offset + i);
  __syncthreads();
  const float* w = w_smem ? ws : p.banks + b.offset;
  // phase-major: q -> (phase j, input block i); output n = i*nw + j
  const int nq = b.nw * n_i;
  for (int q = tid; q < nq; q += RS_THREADS) {
    const int j = q / n_i, ii = q - j * n_i;
    const int64_t n = (i_first + ii) * b.nw + j;
    if (n < t0 || n >= t1) continue;
    const float* xr = xs + ii * b.orig;
    const float* wr = w + j * b.taps;
    float acc = 0.f;
    if (w_smem) {
      for (int k = 0; k < b.taps; ++k) acc = fmaf(wr[k], xr[k], acc);
    } else {
      for (int k = 0; k < b.taps; ++k) acc = fmaf(__ldg(wr + k), xr[k], acc);
    }
    ys[n - t0] = acc;
  }
  __syncthreads();
  for (int64_t n = t0 + tid; n < t1; n += RS_THREADS) p.y[out0 + n] = ys[n - t0];
}

// one warp per output frame: source frame = f - pos of the last sub covering f (else f); zero if the source frame is in
// a time mask or the column in a frequency mask (masks are applied before subs in the reference, subs read the masked
// features, trim drops the tail, which the output offsets already encode).
__global__ void __launch_bounds__(256) spec_augment_kernel(const float* __restrict__ in,
                                                           const int64_t* __restrict__ in_off,
                                                           const int64_t* __restrict__ out_off, int n_utts,
                                                           int64_t total_out, int n_feat,
                                                           const int32_t* __restrict__ t_masks, int n_t,
                                                           const int32_t* __restrict__ f_masks, int n_f,
                                                           const int32_t* __restrict__ subs, int n_sub,
                                                           float* __restrict__ out) {
  const int64_t row = int64_t(blockIdx.x) * 8 + warp_id();
  if (row >= total_out) return;
  const uint32_t lane = lane_id();
  const int u = find_segment(out_off, n_utts, row);
  const int f = int(row - out_off[u]);
  int src = f;
  const int32_t* su = subs + int64_t(u) * n_sub * 3;
  for (int s = 0; s < n_sub; ++s)
    if (su[3 * s] <= f && f < su[3 * s + 1]) src = f - su[3 * s + 2];
  bool zero_row = false;
  const int32_t* tm = t_masks + int64_t(u) * n_t * 2;
  for (int t = 0; t < n_t; ++t) zero_row |= (tm[2 * t] <= src && src < tm[2 * t + 1]);
  const int32_t* fm = f_masks + int64_t(u) * n_f * 2;
  const float* xr = in + (in_off[u] + src) * n_feat;
  float* yr = out + row * n_feat;
  for (int c = lane; c < n_feat; c += 32) {
    bool z = zero_row;
    for (int m = 0; m < n_f; ++m) z |= (fm[2 * m] <= c && c < fm[2 * m + 1]);
    yr[c] = z ? 0.f : xr[c];
  }
}

}  // namespace tn

using namespace tn;

extern "C" int tn_resample_f32(const void* x, int x_is_i16, const int64_t* in_offsets, const int64_t* out_offsets,
                               const int64_t* tile_offsets, const int32_t* utt_bank, int n_utts, int64_t n_tiles,
                               int tile, const int32_t* bank_table, int n_banks, const float* banks, float* y,
                               tn_stream_t stream_) {
  clear_error();
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  TN_REQUIRE(x && in_offsets && out_offsets && tile_offsets && utt_bank && bank_table && banks && y,
             "tn_resample_f32: null pointer");
  TN_REQUIRE(n_banks >= 1 && n_banks <= RS_MAX_BANKS, "tn_resample_f32: n_banks=%d out of range (1..%d)", n_banks,
             RS_MAX_BANKS);
  TN_REQUIRE(tile >= 32 && tile <= RS_MAX_TILE && tile % 32 == 0, "tn_resample_f32: tile=%d (multiple of 32, <= %d)",
             tile, RS_MAX_TILE);
  ResampleParams p{};
  int xs_cap = 0, w_cap = 0;
  for (int i = 0; i < n_banks; ++i) {
    const int32_t* t = bank_table + 5 * i;
    ResampleBank b{t[0], t[1], t[2], t[3], t[4]};
    TN_REQUIRE(b.orig >= 1 && b.nw >= 1 && b.width >= 0 && b.offset >= 0,
               "tn_resample_f32: bank %d: bad (orig=%d, new=%d, width=%d, offset=%d)", i, b.orig, b.nw, b.width,
               b.offset);
    if (b.orig == b.nw) {
      TN_REQUIRE(b.orig == 1, "tn_resample_f32: bank %d: a 1:1 bank must be reduced to (1, 1)", i);
    } else {
      TN_REQUIRE(b.taps == 2 * b.width + b.orig, "tn_resample_f32: bank %d: taps=%d != 2*width + orig", i, b.taps);
      const int span = ((tile - 1) / b.nw + 1) * b.orig + b.taps;   // upper bound of the staged input window
      xs_cap = span > xs_cap ? span : xs_cap;
      const int bank_len = b.nw * b.taps;
      if (bank_len <= RS_MAX_SMEM_BANK && bank_len > w_cap) w_cap = bank_len;
    }
    p.bank[i] = b;
  }
  const size_t smem = sizeof(float) * (size_t(xs_cap > 0 ? tile : 0) + xs_cap + w_cap);
  TN_REQUIRE(smem <= 200 * 1024, "tn_resample_f32: ratio needs %zu B of shared memory per tile (max 200 KB)", smem);
  if (n_tiles == 0 || n_utts == 0) return TN_OK;
  p.x = x; p.x_is_i16 = x_is_i16; p.in_off = in_offsets; p.out_off = out_offsets; p.tile_off = tile_offsets;
  p.utt_bank = utt_bank; p.n_utts = n_utts; p.tile = tile; p.xs_cap = xs_cap; p.w_cap = w_cap; p.banks = banks;
  p.y = y;
  if (smem > 48 * 1024)
    TN_CHECK_CUDA(cudaFuncSetAttribute(resample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
  resample_kernel<<<unsigned(n_tiles), RS_THREADS, smem, stream>>>(p);
  TN_CHECK_CUDA(cudaGetLastError());
  return TN_OK;
}

extern "C" int tn_spec_augment_f32(const float* in, const int64_t* in_frame_offsets, const int64_t* out_frame_offsets,
                                   int n_utts, int64_t total_out_frames, int n_feat, const int32_t* t_masks,
                                   int n_t_masks, const int32_t* f_masks, int n_f_masks, const int32_t* subs,
                                   int n_subs, float* out, tn_stream_t stream_) {
  clear_error();
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  TN_REQUIRE(in && in_frame_offsets && out_frame_offsets && out, "tn_spec_augment_f32: null pointer");
  TN_REQUIRE(n_feat >= 1 && n_t_masks >= 0 && n_f_masks >= 0 && n_subs >= 0,
             "tn_spec_augment_f32: bad n_feat=%d / table sizes", n_feat);
  TN_REQUIRE((n_t_masks == 0 || t_masks) && (n_f_masks == 0 || f_masks) && (n_subs == 0 || subs),
             "tn_spec_augment_f32: null mask / sub table");
  if (total_out_frames == 0 || n_utts == 0) return TN_OK;
  spec_augment_kernel<<<unsigned((total_out_frames + 7) / 8), 256, 0, stream>>>(
      in, in_frame_offsets, out_frame_offsets, n_utts, total_out_frames, n_feat, t_masks, n_t_masks, f_masks,
      n_f_masks, subs, n_subs, out);
  TN_CHECK_CUDA(cudaGetLastError());
  return TN_OK;
}
