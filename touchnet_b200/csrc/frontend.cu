// touchnet_b200 :: audio frontend (waveform -> fbank / MFCC / log-mel -> stacked low-frame-rate features) on the GPU.
//
// Replaces, batched over utterances packed back to back in one buffer:
//   audio_compute_fbank                touchnet/data/functions.py:117-134
//       -> torchaudio.compliance.kaldi.fbank  ta:compliance/kaldi.py:514-645 (+ :44-84 framing, :154-217 window)
//   audio_compute_mfcc                 touchnet/data/functions.py:137-156
//       -> torchaudio.compliance.kaldi.mfcc   ta:compliance/kaldi.py:679-800: fbank's log-mel row times the DCT table
//          (the lifter folded in on the host), a compile-time epilogue variant of the two fbank kernels
//   audio_compute_log_mel_spectrogram  touchnet/data/functions.py:159-190 (whisper-style torch.stft path)
//   audiofeat_stack                    touchnet/data/functions.py:258-286
//
// One CTA processes groups of 8 frames: warp w prepares frame w (DC removal, pre-emphasis, window | reflect
// padding, window) into shared memory, then thread k evaluates DFT bin k for all 8 frames at once from a
// shared cos/sin table (the transform length is tiny - 400 or 512 points - so a table-driven DFT with 16 FMAs
// per 3 shared loads beats an FFT's synchronisation cost and handles n_fft = 400 without a mixed-radix plan),
// power spectrum -> sparse mel filter rows -> log.  HBM traffic is the algorithmic minimum: every sample is read
// once per frame that covers it (L1/L2 absorb the 2.5x overlap) and every feature is written once.
#include <math.h>
#include <stdlib.h>

#include "../../include/touchnet_b200.h"
#include "common.cuh"
#include "host.h"

namespace tn {

constexpr int FE_THREADS = 288;   // >= max bins (257) rounded to warps; 9 warps
constexpr int FE_FRAMES = 8;      // frames per group (one per warp 0..7)
constexpr int FE_MAX_NFFT = 512;
constexpr int FE_MAX_BINS = FE_MAX_NFFT / 2 + 1;
constexpr int FE_MAX_MELS = 128;

struct FrontendParams {
  const void* wav;
  int wav_is_i16;
  const int64_t* utt_offsets;
  const int64_t* frame_offsets;
  int n_utts;
  int64_t total_frames;
  int frame_len, frame_shift, n_fft, n_bins, n_mels;
  const float* window;       // [frame_len]
  const float* mel_filters;  // [n_mels, n_bins]
  float preemph;
  float* out;      // [total_frames, n_mels]  (MFCC: [total_frames, n_ceps])
  float* utt_max;  // whisper mode
  const float* dct;  // MFCC: [n_mels, n_ceps] DCT-II table with the lifter folded in
  int n_ceps;
  int pad;           // whisper mode: zero samples appended to every utterance (audiofeat_padding)
};

// the MFCC table [n_mels][n_ceps] is staged in shared memory once per CTA (64 KB at the 128 x 128 limit)
__device__ __forceinline__ void stage_dct(const float* __restrict__ dct, int n_mels, int n_ceps, float* dct_s) {
  for (int i = threadIdx.x; i < n_mels * n_ceps; i += blockDim.x) dct_s[i] = __ldg(dct + i);
}

__device__ __forceinline__ void atomic_max_float(float* addr, float v) {
  if (v >= 0.f) atomicMax(reinterpret_cast<int*>(addr), __float_as_int(v));
  else atomicMin(reinterpret_cast<unsigned int*>(addr), __float_as_uint(v));
}

__device__ __forceinline__ int find_utt(const int64_t* __restrict__ frame_offsets, int n_utts, int64_t frame) {
  int lo = 0, hi = n_utts - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (frame_offsets[mid] <= frame) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// non-zero span [lo, hi) of every (triangular) mel filter row: one warp per row, lanes stride over the bins
__device__ __forceinline__ void mel_spans(const float* __restrict__ filters, int n_mels, int n_bins, int* mel_lo,
                                          int* mel_hi) {
  const int nwarps = blockDim.x >> 5;
  const uint32_t lane = lane_id();
  for (int m = warp_id(); m < n_mels; m += nwarps) {
    const float* w = filters + int64_t(m) * n_bins;
    int lo = n_bins, hi = 0;
    for (int k = lane; k < n_bins; k += 32)
      if (__ldg(w + k) != 0.f) { lo = min(lo, k); hi = max(hi, k + 1); }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      lo = min(lo, __shfl_xor_sync(0xffffffffu, lo, o));
      hi = max(hi, __shfl_xor_sync(0xffffffffu, hi, o));
    }
    if (lane == 0) { mel_lo[m] = lo; mel_hi[m] = hi; }
  }
}

// MODE 0: kaldi fbank (snip_edges, DC removal, pre-emphasis, window, zero-pad to n_fft, log(max(x, eps)))
// MODE 1: whisper log-mel (center + reflect padding, window length == n_fft, log10(max(x, 1e-10)), per-utt max)
// MFCC (MODE 0 only): the log-mel rows stay in shared memory and each output is sum_m y[m] * dct[m][c]
template <int MODE, bool MFCC = false>
__global__ void __launch_bounds__(FE_THREADS) frontend_kernel(const FrontendParams p) {
  extern __shared__ float fe_smem[];
  float2* tab = reinterpret_cast<float2*>(fe_smem);                       // [n_fft] (cos, sin)(2*pi*i/n_fft)
  float* xs = fe_smem + 2 * FE_MAX_NFFT;                                  // [n_fft][8] frame-minor
  float* ps = xs + FE_MAX_NFFT * FE_FRAMES;                               // [8][FE_MAX_BINS+3] power spectra
  int* mel_lo = reinterpret_cast<int*>(ps + FE_FRAMES * (FE_MAX_BINS + 3));  // [n_mels]
  int* mel_hi = mel_lo + FE_MAX_MELS;
  float* lm = xs;                                           // MFCC: [8][FE_MAX_MELS] log-mel rows (xs is dead by then)
  float* dct_s = reinterpret_cast<float*>(mel_hi + FE_MAX_MELS);   // MFCC: [n_mels][n_ceps]
  float* fmax_s = reinterpret_cast<float*>(mel_hi + FE_MAX_MELS);  // MODE 1: [8] log-mel max of each frame of the group
  constexpr int PS_LD = FE_MAX_BINS + 3;

  const int tid = threadIdx.x;
  const uint32_t warp = warp_id(), lane = lane_id();
  const int n_fft = p.n_fft, n_bins = p.n_bins;

  for (int i = tid; i < n_fft; i += FE_THREADS) {
    float s, c;
    sincospif(2.0f * float(i) / float(n_fft), &s, &c);
    tab[i] = make_float2(c, s);
  }
  mel_spans(p.mel_filters, p.n_mels, n_bins, mel_lo, mel_hi);
  if constexpr (MFCC) stage_dct(p.dct, p.n_mels, p.n_ceps, dct_s);
  if constexpr (MODE == 1) if (tid < FE_FRAMES) fmax_s[tid] = -INFINITY;
  __syncthreads();

  const int64_t n_groups = (p.total_frames + FE_FRAMES - 1) / FE_FRAMES;
  for (int64_t grp = blockIdx.x; grp < n_groups; grp += gridDim.x) {
    // ---------------- stage 1: warp w prepares frame w ----------------
    if (warp < FE_FRAMES) {
      const int64_t frame = grp * FE_FRAMES + warp;
      const bool valid = frame < p.total_frames;
      int u = 0;
      int64_t fi = 0, wav0 = 0, wav_n = 0;
      if (valid) {
        u = find_utt(p.frame_offsets, p.n_utts, frame);
        fi = frame - p.frame_offsets[u];
        wav0 = p.utt_offsets[u];
        wav_n = p.utt_offsets[u + 1] - wav0;
      }
      constexpr int PER_LANE = (FE_MAX_NFFT + 31) / 32;  // 16
      float v[PER_LANE];
      float sum = 0.f;
#pragma unroll
      for (int i = 0; i < PER_LANE; ++i) {
        const int j = int(lane) + 32 * i;
        float x = 0.f;
        if (valid && j < p.frame_len) {
          if (MODE == 0) {
            const int64_t idx = fi * p.frame_shift + j;  // snip_edges: every frame fits
            if (p.wav_is_i16) x = float(reinterpret_cast<const int16_t*>(p.wav)[wav0 + idx]);
            else x = reinterpret_cast<const float*>(p.wav)[wav0 + idx] * 32768.f;
          } else {
            // center=True, reflect on the right-padded length wav_n + pad; indices past wav_n are the zero padding
            const int64_t len = wav_n + p.pad;
            int64_t idx = fi * p.frame_shift + j - n_fft / 2;
            if (idx < 0) idx = -idx;
            if (idx >= len) idx = 2 * (len - 1) - idx;
            if (idx < 0) idx = 0;
            if (idx < wav_n) {
              if (p.wav_is_i16) x = float(reinterpret_cast<const int16_t*>(p.wav)[wav0 + idx]) * (1.f / 32768.f);
              else x = reinterpret_cast<const float*>(p.wav)[wav0 + idx];
            }
          }
        }
        v[i] = x;
        sum += x;
      }
      if (MODE == 0) {
        const float mean = warp_sum(sum) / float(p.frame_len);
        // y[j] = (x[j]-mean) - c*(x[max(j-1,0)]-mean); neighbour j-1 lives in lane-1 (or lane 31 of slot i-1)
#pragma unroll
        for (int i = 0; i < PER_LANE; ++i) v[i] -= mean;
#pragma unroll
        for (int i = 0; i < PER_LANE; ++i) {
          const float up = __shfl_up_sync(0xffffffffu, v[i], 1);
          const float wrap = __shfl_sync(0xffffffffu, v[i > 0 ? i - 1 : 0], 31);
          const float prev = (lane > 0) ? up : (i > 0 ? wrap : v[0]);  // replicate-left at j == 0
          const int j = int(lane) + 32 * i;
          float y = v[i] - p.preemph * prev;
          y = (j < p.frame_len) ? y * p.window[j] : 0.f;
          if (j < n_fft) xs[j * FE_FRAMES + warp] = y;
        }
      } else {
#pragma unroll
        for (int i = 0; i < PER_LANE; ++i) {
          const int j = int(lane) + 32 * i;
          if (j < n_fft) xs[j * FE_FRAMES + warp] = (j < p.frame_len) ? v[i] * p.window[j] : 0.f;
        }
      }
    }
    __syncthreads();
    // ---------------- stage 2: thread k -> DFT bin k of all 8 frames ----------------
    if (tid < n_bins) {
      float re[FE_FRAMES], im[FE_FRAMES];
#pragma unroll
      for (int f = 0; f < FE_FRAMES; ++f) { re[f] = 0.f; im[f] = 0.f; }
      int idx = 0;
      const int n_used = (MODE == 0) ? p.frame_len : n_fft;  // samples beyond frame_len are the zero padding
      for (int n = 0; n < n_used; ++n) {
        const float2 cs = tab[idx];
        const float4 a = *reinterpret_cast<const float4*>(xs + n * FE_FRAMES);
        const float4 b = *reinterpret_cast<const float4*>(xs + n * FE_FRAMES + 4);
        re[0] = fmaf(a.x, cs.x, re[0]); im[0] = fmaf(a.x, cs.y, im[0]);
        re[1] = fmaf(a.y, cs.x, re[1]); im[1] = fmaf(a.y, cs.y, im[1]);
        re[2] = fmaf(a.z, cs.x, re[2]); im[2] = fmaf(a.z, cs.y, im[2]);
        re[3] = fmaf(a.w, cs.x, re[3]); im[3] = fmaf(a.w, cs.y, im[3]);
        re[4] = fmaf(b.x, cs.x, re[4]); im[4] = fmaf(b.x, cs.y, im[4]);
        re[5] = fmaf(b.y, cs.x, re[5]); im[5] = fmaf(b.y, cs.y, im[5]);
        re[6] = fmaf(b.z, cs.x, re[6]); im[6] = fmaf(b.z, cs.y, im[6]);
        re[7] = fmaf(b.w, cs.x, re[7]); im[7] = fmaf(b.w, cs.y, im[7]);
        idx += tid;
        if (idx >= n_fft) idx -= n_fft;
      }
#pragma unroll
      for (int f = 0; f < FE_FRAMES; ++f) ps[f * PS_LD + tid] = re[f] * re[f] + im[f] * im[f];
    }
    __syncthreads();
    // ---------------- stage 3: mel filters + log ----------------
    for (int o = tid; o < FE_FRAMES * p.n_mels; o += FE_THREADS) {
      const int f = o / p.n_mels, m = o - f * p.n_mels;
      const int64_t frame = grp * FE_FRAMES + f;
      if (frame < p.total_frames) {
        const float* w = p.mel_filters + int64_t(m) * n_bins;
        float acc = 0.f;
        for (int k = mel_lo[m]; k < mel_hi[m]; ++k) acc = fmaf(ps[f * PS_LD + k], __ldg(w + k), acc);
        float y;
        if (MODE == 0) {
          y = logf(fmaxf(acc, 1.1920928955078125e-07f));  // torch.finfo(float32).eps
        } else {
          y = log10f(fmaxf(acc, 1e-10f));
          atomic_max_float(fmax_s + f, y);
        }
        if constexpr (MFCC) lm[f * FE_MAX_MELS + m] = y;
        else p.out[frame * p.n_mels + m] = y;
      }
    }
    __syncthreads();
    if constexpr (MODE == 1) {
      // one global atomic per frame, not per (frame, mel): a max is exact, so utt_max is the same either way
      if (tid < FE_FRAMES) {
        const int64_t frame = grp * FE_FRAMES + tid;
        if (frame < p.total_frames)
          atomic_max_float(p.utt_max + find_utt(p.frame_offsets, p.n_utts, frame), fmax_s[tid]);
        fmax_s[tid] = -INFINITY;   // read and reset by the same thread; the next group's stage 3 is two barriers away
      }
    }
    if constexpr (MFCC) {
      // ---------------- stage 4: cepstra, m ascending (fixed order: bit-reproducible) ----------------
      for (int o = tid; o < FE_FRAMES * p.n_ceps; o += FE_THREADS) {
        const int f = o / p.n_ceps, c = o - f * p.n_ceps;
        const int64_t frame = grp * FE_FRAMES + f;
        if (frame < p.total_frames) {
          float acc = 0.f;
          for (int m = 0; m < p.n_mels; ++m) acc = fmaf(lm[f * FE_MAX_MELS + m], dct_s[m * p.n_ceps + c], acc);
          p.out[frame * p.n_ceps + c] = acc;
        }
      }
      __syncthreads();
    }
  }
}

__global__ void fill_kernel(float* x, int n, float v) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) x[i] = v;
}

__global__ void __launch_bounds__(256) logmel_finish_kernel(float* __restrict__ feats,
                                                            const int64_t* __restrict__ frame_offsets,
                                                            const float* __restrict__ utt_max, int n_utts,
                                                            int64_t total_frames, int n_mels) {
  const int64_t total = total_frames * n_mels;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += int64_t(gridDim.x) * blockDim.x) {
    const int64_t frame = i / n_mels;
    const int u = find_utt(frame_offsets, n_utts, frame);
    const float x = fmaxf(feats[i], utt_max[u] - 8.0f);
    feats[i] = (x + 4.0f) / 4.0f;
  }
}

// one warp per output row
__global__ void __launch_bounds__(256) feat_stack_kernel(const float* __restrict__ feats,
                                                         const int64_t* __restrict__ frame_offsets,
                                                         const int64_t* __restrict__ out_offsets, int n_utts,
                                                         int64_t total_out_rows, int n_mels, int stack, int stride,
                                                         int normalize, float* __restrict__ out,
                                                         const int64_t* __restrict__ dst_row0, int64_t out_ld) {
  const int64_t row = int64_t(blockIdx.x) * 8 + warp_id();
  if (row >= total_out_rows) return;
  const uint32_t lane = lane_id();
  const int u = find_utt(out_offsets, n_utts, row);
  const int64_t i = row - out_offsets[u];
  const int64_t f0 = frame_offsets[u];
  const int64_t T = frame_offsets[u + 1] - f0;
  const int left = (stack - 1) / 2;
  const int width = stack * n_mels;
  // packed output (row-major, back to back) or scattered into a [B*T, out_ld] batch buffer at dst_row0[u] + i
  float* dst = dst_row0 ? out + (dst_row0[u] + i) * out_ld : out + row * width;
  float sum = 0.f;
  for (int c = lane; c < width; c += 32) {
    const int s = c / n_mels, m = c - s * n_mels;
    int64_t src = i * stride + s - left;
    src = src < 0 ? 0 : (src > T - 1 ? T - 1 : src);
    const float x = feats[(f0 + src) * n_mels + m];
    dst[c] = x;
    sum += x;
  }
  if (!normalize) return;
  const float mean = warp_sum(sum) / float(width);
  float ss = 0.f;
  __syncwarp();
  for (int c = lane; c < width; c += 32) {
    const float d = dst[c] - mean;
    ss += d * d;
  }
  const float stdv = sqrtf(warp_sum(ss) / float(width - 1));  // unbiased, as torch.std
  const float inv = 1.f / (stdv + 1e-5f);
  for (int c = lane; c < width; c += 32) dst[c] = (dst[c] - mean) * inv;
}


// ---------------------------------------------------------------------------------------------------------------
// FFT path (n_fft = 512, the kaldi fbank geometry at 16 kHz): one warp per frame.
//   real 512-point FFT = complex 256-point FFT of z[n] = x[2n] + i x[2n+1] (radix-2 DIT in shared memory, input stored
//   bit-reversed by the framing step, 8 stages x 4 butterflies per lane) + the split step
//   X[k] = (Z[k] + conj Z[256-k])/2 - i/2 * W512^k * (Z[k] - conj Z[256-k]),  k = 0..256.
// ~10 kFLOP per frame instead of ~410 kFLOP for the table DFT; HBM traffic unchanged (the algorithmic minimum).
// ---------------------------------------------------------------------------------------------------------------
constexpr int FF_N = 512, FF_H = 256, FF_WARPS = 8, FF_LOG2H = 8;
constexpr int FF_MAX_UTT_TAB = 512;   // utterances per launch whose offsets are staged in shared memory

__device__ __forceinline__ uint32_t bitrev8(uint32_t x) { return __brev(x) >> 24; }

// MFCC: the log-mel row goes to the warp's (by then dead) FFT buffer instead of HBM, then lane l writes cepstra
// l, l+32, ..
template <bool MFCC>
__global__ void __launch_bounds__(FF_WARPS * 32) fbank_fft_kernel(const FrontendParams p) {
  extern __shared__ float ff_smem[];
  float2* w256 = reinterpret_cast<float2*>(ff_smem);            // [128]  exp(-2*pi*i*k/256)
  float2* w512 = w256 + FF_H / 2;                                // [257]  exp(-2*pi*i*k/512)
  int* mel_lo = reinterpret_cast<int*>(w512 + FF_H + 1 + 1);     // [n_mels]
  int* mel_hi = mel_lo + FE_MAX_MELS;
  int64_t* s_frm_off = reinterpret_cast<int64_t*>(mel_hi + FE_MAX_MELS);   // [FF_MAX_UTT_TAB]
  int64_t* s_utt_off = s_frm_off + FF_MAX_UTT_TAB;                        // [FF_MAX_UTT_TAB]
  float2* zbase = reinterpret_cast<float2*>(s_utt_off + FF_MAX_UTT_TAB);   // per warp: z[256] then ps[260]
  constexpr int PER_WARP = FF_H * 2 + 260;                       // floats
  const uint32_t warp = warp_id(), lane = lane_id();
  float2* z = reinterpret_cast<float2*>(reinterpret_cast<float*>(zbase) + warp * PER_WARP);
  float* ps = reinterpret_cast<float*>(z + FF_H);
  float* lm = reinterpret_cast<float*>(z);                                   // MFCC: [n_mels] log-mel row
  float* dct_s = reinterpret_cast<float*>(zbase) + FF_WARPS * PER_WARP;      // MFCC: [n_mels][n_ceps]
  const int tid = threadIdx.x;
  for (int i = tid; i < FF_H / 2; i += blockDim.x) {
    float sn, cs;
    sincospif(-2.0f * float(i) / float(FF_H), &sn, &cs);
    w256[i] = make_float2(cs, sn);
  }
  for (int i = tid; i <= FF_H; i += blockDim.x) {
    float sn, cs;
    sincospif(-2.0f * float(i) / float(FF_N), &sn, &cs);
    w512[i] = make_float2(cs, sn);
  }
  const int n_bins = FF_H + 1;
  mel_spans(p.mel_filters, p.n_mels, n_bins, mel_lo, mel_hi);
  // utterance offset tables in shared memory: the per-frame binary search then never leaves the SM
  const int n_tab = min(p.n_utts + 1, FF_MAX_UTT_TAB);
  for (int i = tid; i < n_tab; i += blockDim.x) { s_frm_off[i] = p.frame_offsets[i]; s_utt_off[i] = p.utt_offsets[i]; }
  if constexpr (MFCC) stage_dct(p.dct, p.n_mels, p.n_ceps, dct_s);
  __syncthreads();
  const bool tab_ok = p.n_utts + 1 <= FF_MAX_UTT_TAB;
  const int64_t* frm_off = tab_ok ? s_frm_off : p.frame_offsets;
  const int64_t* utt_off = tab_ok ? s_utt_off : p.utt_offsets;

  const int64_t warps_total = int64_t(gridDim.x) * FF_WARPS;
  for (int64_t frame = int64_t(blockIdx.x) * FF_WARPS + warp; frame < p.total_frames; frame += warps_total) {
    // ---- framing: DC removal, pre-emphasis, window; packed bit-reversed into z ----
    const int u = find_utt(frm_off, p.n_utts, frame);
    const int64_t fi = frame - frm_off[u];
    const int64_t wav0 = utt_off[u] + fi * p.frame_shift;
    constexpr int PER_LANE = FF_N / 32;  // 16
    float v[PER_LANE];
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < PER_LANE; ++i) {
      const int j = int(lane) + 32 * i;
      float x = 0.f;
      if (j < p.frame_len) {
        if (p.wav_is_i16) x = float(reinterpret_cast<const int16_t*>(p.wav)[wav0 + j]);
        else x = reinterpret_cast<const float*>(p.wav)[wav0 + j] * 32768.f;
      }
      v[i] = x;
      sum += x;
    }
    const float mean = warp_sum(sum) / float(p.frame_len);
#pragma unroll
    for (int i = 0; i < PER_LANE; ++i) v[i] -= mean;
#pragma unroll
    for (int i = 0; i < PER_LANE; ++i) {
      const float up = __shfl_up_sync(0xffffffffu, v[i], 1);
      const float wrap = __shfl_sync(0xffffffffu, v[i > 0 ? i - 1 : 0], 31);
      const float prev = (lane > 0) ? up : (i > 0 ? wrap : v[0]);
      const int j = int(lane) + 32 * i;
      float y = v[i] - p.preemph * prev;
      y = (j < p.frame_len) ? y * p.window[j] : 0.f;
      // sample j is component (j & 1) of z[j >> 1]; stored at the bit-reversed index for the in-place DIT
      reinterpret_cast<float*>(z)[2 * bitrev8(uint32_t(j) >> 1) + (j & 1)] = y;
    }
    __syncwarp();
    // ---- 8 radix-2 DIT stages, 4 butterflies per lane per stage ----
#pragma unroll
    for (int s = 0; s < FF_LOG2H; ++s) {
      const int half = 1 << s;
#pragma unroll
      for (int q = 0; q < FF_H / 64; ++q) {
        const int t = int(lane) + 32 * q;            // butterfly 0..127
        const int j = t & (half - 1);
        const int i0 = ((t >> s) << (s + 1)) + j;
        const float2 w = w256[j << (FF_LOG2H - 1 - s)];
        const float2 a = z[i0], b = z[i0 + half];
        const float br = b.x * w.x - b.y * w.y, bi = b.x * w.y + b.y * w.x;
        z[i0] = make_float2(a.x + br, a.y + bi);
        z[i0 + half] = make_float2(a.x - br, a.y - bi);
      }
      __syncwarp();
    }
    // ---- split step + power spectrum ----
    for (int k = lane; k <= FF_H; k += 32) {
      const float2 zk = z[k & (FF_H - 1)];
      const float2 zm = z[(FF_H - k) & (FF_H - 1)];
      const float ar = 0.5f * (zk.x + zm.x), ai = 0.5f * (zk.y - zm.y);     // (Zk + conj Zm)/2
      const float dr = 0.5f * (zk.x - zm.x), di = 0.5f * (zk.y + zm.y);     // (Zk - conj Zm)/2
      const float2 w = w512[k];
      // -i * w * d = -i * ((wr*dr - wi*di) + i(wr*di + wi*dr)) = (wr*di + wi*dr) - i (wr*dr - wi*di)
      const float xr = ar + (w.x * di + w.y * dr);
      const float xi = ai - (w.x * dr - w.y * di);
      ps[k] = xr * xr + xi * xi;
    }
    __syncwarp();
    // ---- mel filter rows + log ----
    for (int m = lane; m < p.n_mels; m += 32) {
      const float* wrow = p.mel_filters + int64_t(m) * n_bins;
      float acc = 0.f;
      for (int k = mel_lo[m]; k < mel_hi[m]; ++k) acc = fmaf(ps[k], __ldg(wrow + k), acc);
      const float y = logf(fmaxf(acc, 1.1920928955078125e-07f));
      if constexpr (MFCC) lm[m] = y;
      else p.out[frame * p.n_mels + m] = y;
    }
    if constexpr (MFCC) {
      // ---- cepstra: c[i] = sum_m y[m] * dct[m][i], m ascending (fixed order: bit-reproducible) ----
      __syncwarp();
      constexpr int CPL = FE_MAX_MELS / 32;   // cepstra per lane (n_ceps <= n_mels <= 128)
      float c[CPL];
#pragma unroll
      for (int j = 0; j < CPL; ++j) c[j] = 0.f;
      for (int m = 0; m < p.n_mels; ++m) {
        const float y = lm[m];
        const float* row = dct_s + m * p.n_ceps + lane;
#pragma unroll
        for (int j = 0; j < CPL; ++j)
          if (int(lane) + 32 * j < p.n_ceps) c[j] = fmaf(y, row[32 * j], c[j]);
      }
#pragma unroll
      for (int j = 0; j < CPL; ++j) {
        const int i = int(lane) + 32 * j;
        if (i < p.n_ceps) p.out[frame * p.n_ceps + i] = c[j];
      }
    }
    __syncwarp();
  }
}

// extra shared memory of the MFCC variants: the DCT table (the log-mel rows reuse buffers that are dead by then)
static size_t mfcc_smem(const FrontendParams& p) { return sizeof(float) * size_t(p.n_mels) * p.n_ceps; }

// grid of a persistent MFCC launch: as many CTAs as fit at this table size (the grid-stride loops would otherwise
// run a partial second wave)
static int mfcc_grid(void (*kernel)(FrontendParams), int threads, size_t smem, int64_t n_groups, int64_t* grid) {
  TN_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
  int per_sm = 0;
  TN_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, smem));
  *grid = int64_t(sm_count()) * (per_sm > 0 ? per_sm : 1);
  if (*grid > n_groups) *grid = n_groups;
  return TN_OK;
}

static int launch_fbank_fft(const FrontendParams& p, cudaStream_t stream) {
  const size_t smem = sizeof(float2) * (FF_H / 2 + FF_H + 2) + sizeof(int) * 2 * FE_MAX_MELS +
                      sizeof(int64_t) * 2 * FF_MAX_UTT_TAB + sizeof(float) * FF_WARPS * (FF_H * 2 + 260);
  const int64_t n_groups = (p.total_frames + FF_WARPS - 1) / FF_WARPS;
  int64_t grid = int64_t(sm_count()) * 6;
  if (grid > n_groups) grid = n_groups;
  if (p.dct) {
    const size_t smem_m = smem + mfcc_smem(p);
    const int rc = mfcc_grid(fbank_fft_kernel<true>, FF_WARPS * 32, smem_m, n_groups, &grid);
    if (rc != TN_OK) return rc;
    fbank_fft_kernel<true><<<unsigned(grid), FF_WARPS * 32, smem_m, stream>>>(p);
  } else {
    fbank_fft_kernel<false><<<unsigned(grid), FF_WARPS * 32, smem, stream>>>(p);
  }
  TN_CHECK_CUDA(cudaGetLastError());
  return TN_OK;
}

static int launch_frontend(int mode, const FrontendParams& p, cudaStream_t stream) {
  const size_t smem = sizeof(float) * (2 * FE_MAX_NFFT + FE_MAX_NFFT * FE_FRAMES + FE_FRAMES * (FE_MAX_BINS + 3)) +
                      sizeof(int) * 2 * FE_MAX_MELS;
  const int64_t n_groups = (p.total_frames + FE_FRAMES - 1) / FE_FRAMES;
  int64_t grid = int64_t(sm_count()) * 4;
  if (grid > n_groups) grid = n_groups;
  if (mode == 0 && p.dct) {
    const size_t smem_m = smem + mfcc_smem(p);
    const int rc = mfcc_grid(frontend_kernel<0, true>, FE_THREADS, smem_m, n_groups, &grid);
    if (rc != TN_OK) return rc;
    frontend_kernel<0, true><<<unsigned(grid), FE_THREADS, smem_m, stream>>>(p);
  } else if (mode == 0) {
    frontend_kernel<0><<<unsigned(grid), FE_THREADS, smem, stream>>>(p);
  } else {
    frontend_kernel<1><<<unsigned(grid), FE_THREADS, smem + sizeof(float) * FE_FRAMES, stream>>>(p);
  }
  TN_CHECK_CUDA(cudaGetLastError());
  return TN_OK;
}

}  // namespace tn

using namespace tn;

// fbank (dct == nullptr) or MFCC: shared argument checks and dispatch of tn_fbank_f32 / tn_mfcc_f32
static int kaldi_features(const char* fn, const void* wav, int wav_is_i16, const int64_t* utt_offsets,
                          const int64_t* frame_offsets, int n_utts, int64_t total_frames, int frame_len,
                          int frame_shift, int n_fft, const float* window, const float* mel_filters, int n_mels,
                          float preemph, const float* dct, int n_ceps, float* out, cudaStream_t stream) {
  TN_REQUIRE(wav && utt_offsets && frame_offsets && window && mel_filters && out, "%s: null pointer", fn);
  TN_REQUIRE(n_fft <= FE_MAX_NFFT && n_fft % 2 == 0 && frame_len <= n_fft && frame_len >= 2 && frame_shift > 0,
             "%s: unsupported geometry frame_len=%d n_fft=%d (max %d)", fn, frame_len, n_fft, FE_MAX_NFFT);
  TN_REQUIRE(n_mels > 0 && n_mels <= FE_MAX_MELS, "%s: n_mels=%d out of range (max %d)", fn, n_mels, FE_MAX_MELS);
  if (total_frames == 0 || n_utts == 0) return TN_OK;
  FrontendParams p{};
  p.wav = wav; p.wav_is_i16 = wav_is_i16; p.utt_offsets = utt_offsets; p.frame_offsets = frame_offsets;
  p.n_utts = n_utts; p.total_frames = total_frames; p.frame_len = frame_len; p.frame_shift = frame_shift;
  p.n_fft = n_fft; p.n_bins = n_fft / 2 + 1; p.n_mels = n_mels; p.window = window; p.mel_filters = mel_filters;
  p.preemph = preemph; p.out = out; p.utt_max = nullptr; p.dct = dct; p.n_ceps = n_ceps;
  static const bool force_dft = getenv("TN_FBANK_DFT") != nullptr;   // A/B switch: table DFT instead of the FFT path
  if (n_fft == FF_N && !force_dft) return launch_fbank_fft(p, stream);
  return launch_frontend(0, p, stream);
}

extern "C" int tn_fbank_f32(const void* wav, int wav_is_i16, const int64_t* utt_offsets, const int64_t* frame_offsets,
                            int n_utts, int64_t total_frames, int frame_len, int frame_shift, int n_fft,
                            const float* window, const float* mel_filters, int n_mels, float preemph, float* out,
                            tn_stream_t stream_) {
  clear_error();
  return kaldi_features("tn_fbank_f32", wav, wav_is_i16, utt_offsets, frame_offsets, n_utts, total_frames, frame_len,
                        frame_shift, n_fft, window, mel_filters, n_mels, preemph, nullptr, 0, out,
                        static_cast<cudaStream_t>(stream_));
}

extern "C" int tn_mfcc_f32(const void* wav, int wav_is_i16, const int64_t* utt_offsets, const int64_t* frame_offsets,
                           int n_utts, int64_t total_frames, int frame_len, int frame_shift, int n_fft,
                           const float* window, const float* mel_filters, int n_mels, float preemph, const float* dct,
                           int n_ceps, float* out, tn_stream_t stream_) {
  clear_error();
  TN_REQUIRE(dct, "tn_mfcc_f32: null DCT table");
  TN_REQUIRE(n_ceps >= 1 && n_ceps <= n_mels, "tn_mfcc_f32: n_ceps=%d out of range (1..n_mels=%d)", n_ceps, n_mels);
  return kaldi_features("tn_mfcc_f32", wav, wav_is_i16, utt_offsets, frame_offsets, n_utts, total_frames, frame_len,
                        frame_shift, n_fft, window, mel_filters, n_mels, preemph, dct, n_ceps, out,
                        static_cast<cudaStream_t>(stream_));
}

extern "C" int tn_logmel_power_f32(const void* wav, int wav_is_i16, const int64_t* utt_offsets,
                                   const int64_t* frame_offsets, int n_utts, int64_t total_frames, int n_fft, int hop,
                                   int pad, const float* window, const float* mel_filters, int n_mels, float* out,
                                   float* utt_max, tn_stream_t stream_) {
  clear_error();
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  TN_REQUIRE(wav && utt_offsets && frame_offsets && window && mel_filters && out && utt_max,
             "tn_logmel_power_f32: null pointer");
  TN_REQUIRE(n_fft <= FE_MAX_NFFT && n_fft % 2 == 0 && hop > 0, "tn_logmel_power_f32: unsupported n_fft=%d", n_fft);
  TN_REQUIRE(n_mels > 0 && n_mels <= FE_MAX_MELS, "tn_logmel_power_f32: n_mels=%d out of range", n_mels);
  TN_REQUIRE(pad >= 0, "tn_logmel_power_f32: negative padding %d", pad);
  if (n_utts == 0) return TN_OK;
  fill_kernel<<<(n_utts + 255) / 256, 256, 0, stream>>>(utt_max, n_utts, -INFINITY);
  TN_CHECK_CUDA(cudaGetLastError());
  if (total_frames == 0) return TN_OK;
  FrontendParams p{};
  p.wav = wav; p.wav_is_i16 = wav_is_i16; p.utt_offsets = utt_offsets; p.frame_offsets = frame_offsets;
  p.n_utts = n_utts; p.total_frames = total_frames; p.frame_len = n_fft; p.frame_shift = hop;
  p.n_fft = n_fft; p.n_bins = n_fft / 2 + 1; p.n_mels = n_mels; p.window = window; p.mel_filters = mel_filters;
  p.preemph = 0.f; p.out = out; p.utt_max = utt_max; p.pad = pad;
  return launch_frontend(1, p, stream);
}

extern "C" int tn_logmel_finish_f32(float* feats, const int64_t* frame_offsets, const float* utt_max, int n_utts,
                                    int64_t total_frames, int n_mels, tn_stream_t stream_) {
  clear_error();
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  TN_REQUIRE(feats && frame_offsets && utt_max, "tn_logmel_finish_f32: null pointer");
  if (total_frames == 0) return TN_OK;
  const int64_t total = total_frames * n_mels;
  int64_t blocks = (total + 255) / 256;
  if (blocks > int64_t(sm_count()) * 16) blocks = int64_t(sm_count()) * 16;
  logmel_finish_kernel<<<unsigned(blocks), 256, 0, stream>>>(feats, frame_offsets, utt_max, n_utts, total_frames, n_mels);
  TN_CHECK_CUDA(cudaGetLastError());
  return TN_OK;
}

extern "C" int tn_feat_stack_f32(const float* feats, const int64_t* frame_offsets, const int64_t* out_offsets, int n_utts,
                                 int64_t total_out_rows, int n_mels, int stack, int stride, int normalize, float* out,
                                 const int64_t* dst_row0, int64_t out_ld, tn_stream_t stream_) {
  clear_error();
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  TN_REQUIRE(feats && frame_offsets && out_offsets && out, "tn_feat_stack_f32: null pointer");
  TN_REQUIRE(stack >= 1 && stride >= 1 && n_mels >= 1, "tn_feat_stack_f32: bad stack/stride");
  if (total_out_rows == 0) return TN_OK;
  feat_stack_kernel<<<unsigned((total_out_rows + 7) / 8), 256, 0, stream>>>(feats, frame_offsets, out_offsets, n_utts,
                                                                           total_out_rows, n_mels, stack, stride,
                                                                           normalize, out, dst_row0,
                                                                           out_ld > 0 ? out_ld : int64_t(stack) * n_mels);
  TN_CHECK_CUDA(cudaGetLastError());
  return TN_OK;
}
