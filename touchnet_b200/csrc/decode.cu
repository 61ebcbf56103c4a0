// touchnet_b200 :: autoregressive decoding - split-KV decode attention, KV-cache append, greedy and sampled token
// selection.
//
// Replaces what transformers' `generate(use_cache=True, do_sample=False, num_beams=1)` runs per new token when the
// reference evaluates a model (touchnet/models/touch_audio/inference_touch_audio.py:170-192): the attention of one new
// query row per sequence over the cache (hf: DynamicCache + sdpa), the cache update, and the logits processors
// RepetitionPenaltyLogitsProcessor / NoRepeatNGramLogitsProcessor followed by argmax.
//
// Decode attention is memory bound (one query row per head against S cached keys), so the kernel is organised around
// streaming K/V: grid (split, kv head, batch row); the H/KV query heads that share a kv head are the rows of ONE
// m16n8k16 tile (GQA ratios 1..16), 4 warps each take 16 keys of every 64-key sub-block, K/V sub-blocks arrive through a
// DEC_STAGES-deep cp.async ring.  Every split writes an fp32 partial (O unnormalised, m in the log2 domain, l); a second
// kernel merges the splits in split order (no atomics: bit-reproducible run to run).
//
// Continuous batching (generation.generate_many) adds slot-addressed forms: a K/V scatter of a packed multi-prompt
// prefill into chosen cache slots, the admission of those slots' decoding state, and a selection that holds finished /
// idle slots still and stops a slot at its token limit.  Its sampling form (generate_many with do_sample=True) draws
// from HF's temperature / top-k / top-p distribution with a counter-based Philox stream per prompt.
//
// Speculative decoding (generation.generate with assistant_model) adds the multi-query form of the decode attention
// (Tq new rows per sequence, causal within the block, each row bit-identical to the single-query kernel at its own
// length) and a verify selection: the greedy pick at each of the k + 1 positions of the block over the history
// extended by the draft tokens before it, then the longest accepted prefix plus one token.
#include "../../include/touchnet_b200.h"
#include "attn_common.cuh"
#include "host.h"

#include <curand_philox4x32_x.h>

namespace tn {

constexpr int DEC_THREADS = 128;   // 4 warps x 16 keys of each 64-key sub-block
constexpr int DEC_STAGES = 3;
constexpr int DEC_SUB_TILE = ATT_SUB * ATT_HD * 2;              // 16 KB (one of K, V)
constexpr int DEC_Q_TILE = 16 * ATT_HD * 2;                     // 4 KB
constexpr int DEC_SMEM = DEC_Q_TILE + DEC_STAGES * 2 * DEC_SUB_TILE;
constexpr int DEC_TARGET_CTAS = 4 * 132;   // two resident CTAs per SM, two waves over the 132 SMs of an H100 SXM
constexpr int DEC_MAX_SPLITS = 64;

// split count: a function of the shapes only (never of the current length, so a captured graph stays valid)
static inline int decode_splits(int B, int KV, int S_cap) {
  const int per_row = B * KV;
  int s = (DEC_TARGET_CTAS + per_row - 1) / per_row;
  const int max_by_len = (S_cap + ATT_SUB - 1) / ATT_SUB;
  if (s > max_by_len) s = max_by_len;
  if (s > DEC_MAX_SPLITS) s = DEC_MAX_SPLITS;
  return s < 1 ? 1 : s;
}

struct DecodeParams {
  const bf16* Q;
  const bf16* K;
  const bf16* V;
  int64_t ldq, ld_tok, ld_batch;
  const int32_t* kv_start;
  const int32_t* kv_end;
  float* part_o;    // [B*Tq, H, splits, 128]
  float* part_ml;   // [B*Tq, H, splits, 2]  (m in the log2 domain, l)
  int H, KV, S_cap, splits, chunk;
  float scale_log2;
  int Tq;           // queries per batch row (MULTI only)
};

// MULTI = false: one query per batch row, tile row g = query head g of this kv head.  MULTI = true: Tq queries per batch
// row (query j at cache position kv_end - Tq + j), tile row j*G + g; every tile row has its own key limit, so a row sees
// exactly the keys it would see alone.  Sub-blocks or whole splits past a row's limit are exact no-ops for that row (its
// scores are -inf: m unchanged, alpha = exp2(0) = 1, p = 0; an untouched split leaves l = 0, which the merge skips).
template <bool MULTI>
__global__ void __launch_bounds__(DEC_THREADS, 2) attn_decode_kernel(const DecodeParams p) {
  extern __shared__ __align__(128) uint8_t smem[];
  const uint32_t sb = smem_u32(smem);
  const int split = blockIdx.x, kvh = blockIdx.y, b = blockIdx.z;
  const int tid = int(threadIdx.x), warp = tid >> 5, lane = tid & 31;
  const int G = p.H / p.KV;
  const int lo = max(p.kv_start[b], split * p.chunk);
  const int hi = min(min(p.kv_end[b], p.S_cap), (split + 1) * p.chunk);
  float* pml = p.part_ml + ((int64_t(b) * p.H + kvh * G) * p.splits + split) * 2;
  float* po = p.part_o + ((int64_t(b) * p.H + kvh * G) * p.splits + split) * ATT_HD;
  // MULTI: tile row r = j*G + g is partial row [b*Tq + j, kvh*G + g] (element offset of its (m, l) pair / 2)
  const auto part = [&](int r) { return ((int64_t(b) * p.Tq + r / G) * p.H + kvh * G + r % G) * p.splits + split; };
  if (hi <= lo) {   // nothing of this row's range in this chunk: an empty partial
    if constexpr (MULTI) {
      for (int r = tid; r < p.Tq * G; r += DEC_THREADS) {
        p.part_ml[part(r) * 2] = -INFINITY;
        p.part_ml[part(r) * 2 + 1] = 0.f;
      }
    } else {
      for (int g = tid; g < G; g += DEC_THREADS) {
        pml[int64_t(g) * p.splits * 2] = -INFINITY;
        pml[int64_t(g) * p.splits * 2 + 1] = 0.f;
      }
    }
    return;
  }
  const bf16* Kb = p.K + int64_t(b) * p.ld_batch + kvh * ATT_HD;
  const bf16* Vb = p.V + int64_t(b) * p.ld_batch + kvh * ATT_HD;
  const int kbase = lo & ~(ATT_SUB - 1);
  const int nsub = (hi - kbase + ATT_SUB - 1) / ATT_SUB;
  const uint32_t sQ = sb, sK0 = sb + DEC_Q_TILE, sV0 = sK0 + DEC_STAGES * DEC_SUB_TILE;

  if constexpr (MULTI) {   // tile row j*G + g <- head kvh*G + g of query row b*Tq + j (rows >= Tq*G zero)
    for (int i = tid; i < 16 * 16; i += DEC_THREADS) {
      const int r = i >> 4, ch = i & 15;
      const bool ok = r < p.Tq * G;
      const bf16* src =
          p.Q + (ok ? (int64_t(b) * p.Tq + r / G) * p.ldq + int64_t(kvh * G + r % G) * ATT_HD : 0) + ch * 8;
      cp_async16(sQ + tile_off(r, ch), src, ok ? 16u : 0u);
    }
  } else {                 // the G query heads of this kv head are rows 0..G-1 of a 16-row tile (rows >= G zero)
    load_tile_async<16, DEC_THREADS>(sQ, p.Q + int64_t(b) * p.ldq + int64_t(kvh) * G * ATT_HD, ATT_HD, 0, 0, G, tid);
  }
  auto load_stage = [&](int i) {
    if (i < nsub) {
      const int st = i % DEC_STAGES, k0 = kbase + i * ATT_SUB;
      load_tile_async<ATT_SUB, DEC_THREADS, true>(sK0 + st * DEC_SUB_TILE, Kb, p.ld_tok, k0, lo, hi, tid);
      load_tile_async<ATT_SUB, DEC_THREADS, true>(sV0 + st * DEC_SUB_TILE, Vb, p.ld_tok, k0, lo, hi, tid);
    }
    cp_async_commit();   // empty groups keep the group count uniform
  };
#pragma unroll
  for (int i = 0; i < DEC_STAGES - 1; ++i) load_stage(i);

  const int cq = 2 * (lane & 3);
  float o[16][4];
#pragma unroll
  for (int i = 0; i < 16; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
  float m_a = -INFINITY, m_b = -INFINITY, l_a = 0.f, l_b = 0.f;
  uint32_t qf[8][4];

  for (int i = 0; i < nsub; ++i) {
    cp_async_wait<DEC_STAGES - 2>();
    __syncthreads();                         // stage i landed for every thread; stage i-1 is no longer read
    load_stage(i + DEC_STAGES - 1);
    if (i == 0) {
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) ldsm_a(sQ, 0, kk, qf[kk]);
    }
    const int st = i % DEC_STAGES;
    const uint32_t sK = sK0 + st * DEC_SUB_TILE, sV = sV0 + st * DEC_SUB_TILE;
    const int k0 = kbase + i * ATT_SUB + warp * 16;   // this warp's 16 keys

    float s[2][4];
    mma_scores_nk<1>(s, qf, sK, warp * 16);
    if constexpr (MULTI) {   // per-row key limits: query j sees cache rows < kv_end - Tq + j + 1
      const int hi_a = min(hi, p.kv_end[b] - p.Tq + (lane >> 2) / G + 1);
      const int hi_b = min(hi, p.kv_end[b] - p.Tq + ((lane >> 2) + 8) / G + 1);
      const auto mask = [&](float x, int j, int e) {
        const int key = k0 + 8 * j + cq + (e & 1);
        return (key >= lo && key < (e < 2 ? hi_a : hi_b)) ? x * p.scale_log2 : -INFINITY;
      };
      softmax_step(s, mask, o, m_a, m_b, l_a, l_b);
    } else {
      const auto mask = [&](float x, int j, int e) {
        const int key = k0 + 8 * j + cq + (e & 1);
        return (key >= lo && key < hi) ? x * p.scale_log2 : -INFINITY;
      };
      softmax_step(s, mask, o, m_a, m_b, l_a, l_b);
    }
    mma_acc_kn(o, s, sV, warp * 16);
  }
  cp_async_wait<0>();
  __syncthreads();   // the ring is free: reuse it for the cross-warp merge

  // ---- merge the 4 warps (fixed order) -> this split's partial ----
  l_a = quad_sum(l_a); l_b = quad_sum(l_b);
  float* sO = reinterpret_cast<float*>(smem + DEC_Q_TILE);        // [4 warps][16 rows][128] fp32 = 32 KB
  float* sM = sO + 4 * 16 * ATT_HD;                               // [4][16]
  float* sL = sM + 4 * 16;                                        // [4][16]
  const int ra = lane >> 2;
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const int col = 8 * j + cq;
    float* wa = sO + (warp * 16 + ra) * ATT_HD + col;
    float* wb = sO + (warp * 16 + ra + 8) * ATT_HD + col;
    wa[0] = o[j][0]; wa[1] = o[j][1]; wb[0] = o[j][2]; wb[1] = o[j][3];
  }
  if ((lane & 3) == 0) {
    sM[warp * 16 + ra] = m_a; sM[warp * 16 + ra + 8] = m_b;
    sL[warp * 16 + ra] = l_a; sL[warp * 16 + ra + 8] = l_b;
  }
  __syncthreads();
  for (int i = tid; i < (MULTI ? p.Tq * G : G) * ATT_HD; i += DEC_THREADS) {   // tile rows in use
    const int g = i / ATT_HD, c = i % ATT_HD;
    float M = -INFINITY;
#pragma unroll
    for (int w = 0; w < 4; ++w) M = fmaxf(M, sM[w * 16 + g]);
    const float Mu = M == -INFINITY ? 0.f : M;
    float acc = 0.f, L = 0.f;
#pragma unroll
    for (int w = 0; w < 4; ++w) {
      const float f = fast_exp2(sM[w * 16 + g] - Mu);
      acc += f * sO[(w * 16 + g) * ATT_HD + c];
      L += f * sL[w * 16 + g];
    }
    if constexpr (MULTI) {
      p.part_o[part(g) * ATT_HD + c] = acc;
      if (c == 0) {
        p.part_ml[part(g) * 2] = M;
        p.part_ml[part(g) * 2 + 1] = L;
      }
    } else {
      po[int64_t(g) * p.splits * ATT_HD + c] = acc;
      if (c == 0) {
        pml[int64_t(g) * p.splits * 2] = M;
        pml[int64_t(g) * p.splits * 2 + 1] = L;
      }
    }
  }
}

// one CTA (128 threads = 128 columns) per (row, head): combine the splits in split order
__global__ void __launch_bounds__(ATT_HD) attn_decode_merge_kernel(const float* __restrict__ part_o,
                                                                   const float* __restrict__ part_ml, bf16* __restrict__ O,
                                                                   int64_t ldo, float* __restrict__ lse, int H, int splits) {
  const int h = blockIdx.x, b = blockIdx.y, c = threadIdx.x;
  const float* ml = part_ml + (int64_t(b) * H + h) * splits * 2;
  const float* po = part_o + (int64_t(b) * H + h) * splits * ATT_HD;
  float M = -INFINITY;
  for (int s = 0; s < splits; ++s)
    if (ml[2 * s + 1] > 0.f) M = fmaxf(M, ml[2 * s]);
  float acc = 0.f, L = 0.f;
  if (M != -INFINITY) {
    for (int s = 0; s < splits; ++s) {
      const float l = ml[2 * s + 1];
      if (l > 0.f) {
        const float f = fast_exp2(ml[2 * s] - M);
        acc += f * po[int64_t(s) * ATT_HD + c];
        L += f * l;
      }
    }
  }
  const float inv = L > 0.f ? 1.f / L : 0.f;
  O[int64_t(b) * ldo + int64_t(h) * ATT_HD + c] = __float2bfloat16_rn(acc * inv);
  if (lse && c == 0) lse[int64_t(b) * H + h] = softmax_lse(M, L);
}

// ---------------------------------------------------------------------------------------------------------------
// cache append: rows [end[b] - T_new, end[b]) of batch row b <- source rows b*T_new .. b*T_new + T_new - 1
// ---------------------------------------------------------------------------------------------------------------
// row `src` of K / V -> element offset `dst` of Kc / Vc: `width` bf16 in 16-byte copies over the CTA's threads
__device__ __forceinline__ void copy_kv_row(const bf16* K, int64_t ldk, const bf16* V, int64_t ldv, bf16* Kc, bf16* Vc,
                                            int64_t src, int64_t dst, int width) {
  for (int i = threadIdx.x; i < width / 8; i += blockDim.x) {
    reinterpret_cast<uint4*>(Kc + dst)[i] = reinterpret_cast<const uint4*>(K + src * ldk)[i];
    reinterpret_cast<uint4*>(Vc + dst)[i] = reinterpret_cast<const uint4*>(V + src * ldv)[i];
  }
}

__global__ void kv_append_kernel(const bf16* __restrict__ K, int64_t ldk, const bf16* __restrict__ V, int64_t ldv,
                                 bf16* __restrict__ Kc, bf16* __restrict__ Vc, int64_t ld_tok, int64_t ld_batch,
                                 const int32_t* __restrict__ row_end, int T_new, int S_cap, int width) {
  const int t = blockIdx.x, b = blockIdx.y;
  const int row = row_end[b] - T_new + t;
  if (row < 0 || row >= S_cap) return;
  copy_kv_row(K, ldk, V, ldv, Kc, Vc, int64_t(b) * T_new + t, int64_t(b) * ld_batch + int64_t(row) * ld_tok, width);
}

// ---------------------------------------------------------------------------------------------------------------
// greedy selection with HF's repetition penalty and no-repeat-ngram processors, one CTA per batch row
// ---------------------------------------------------------------------------------------------------------------
constexpr int SEL_THREADS = 1024;
constexpr size_t SEL_MAX_SMEM = 204800;   // 200 KB: the most dynamic shared memory a selection CTA's bitmaps may take

// torch.argmax order: NaN above every number, then the larger value, then the lower index; index -1 = no candidate
__device__ __forceinline__ bool argmax_better(float x, int i, float best, int bi) {
  if (i < 0) return false;
  if (bi < 0) return true;
  const bool nx = x != x, nb = best != best;
  if (nx != nb) return nx;
  if (!nx && x != best) return x > best;
  return i < bi;
}

enum SelectMode { SEL_PLAIN, SEL_SLOTS, SEL_VERIFY };

// HF's processor front, shared by the greedy and the sampling selections: the repetition set and the no-repeat-ngram
// ban of slot b's history as two bitmaps bits[0, words) / bits[words, 2 words).  The history is the slot's
// length[b] ids followed (VERIFY) by draft[0 .. extra).  Returns the history length; ends on a barrier.
template <bool VERIFY>
__device__ __forceinline__ int processor_front(uint32_t* bits, uint32_t* rep, uint32_t* ban, int words, int V,
                                               const int64_t* __restrict__ history, int64_t ld_hist,
                                               const int32_t* __restrict__ length, int b,
                                               const int64_t* __restrict__ draft, int extra, float penalty, int ngram) {
  const int tid = threadIdx.x;
  for (int i = tid; i < 2 * words; i += SEL_THREADS) bits[i] = 0u;
  __syncthreads();
  const int n0 = length[b];
  const int len = n0 + extra;
  const int64_t* h0 = history + int64_t(b) * ld_hist;
  const auto h = [&](int i) { return VERIFY && i >= n0 ? draft[i - n0] : h0[i]; };
  if (penalty != 1.0f) {
    for (int i = tid; i < len; i += SEL_THREADS) {
      const int64_t id = h(i);
      if (id >= 0 && id < V) atomicOr(&rep[id >> 5], 1u << (id & 31));
    }
  }
  if (ngram > 0 && len + 1 >= ngram) {
    // ngram i = h[i .. i+n-1]; its last id is banned when its first n-1 ids equal the last n-1 ids of the sequence
    for (int i = tid; i + ngram <= len; i += SEL_THREADS) {
      bool match = true;
      for (int j = 0; j < ngram - 1 && match; ++j) match = h(i + j) == h(len - ngram + 1 + j);
      const int64_t id = h(i + ngram - 1);
      if (match && id >= 0 && id < V) atomicOr(&ban[id >> 5], 1u << (id & 31));
    }
  }
  __syncthreads();
  return len;
}

// logit v of a row after the processor front: the fp32 value, the repetition penalty, -inf where banned (the loop of
// greedy_select_row spells the same three steps out: written through this helper it compiles to other registers)
__device__ __forceinline__ float processed_logit(const bf16* __restrict__ row, int v, const uint32_t* rep,
                                                 const uint32_t* ban, bool use_pen, float penalty) {
  float x = __bfloat162float(row[v]);
  if (use_pen && (rep[v >> 5] >> (v & 31) & 1u)) x = x < 0.f ? x * penalty : x / penalty;
  if (ban[v >> 5] >> (v & 31) & 1u) x = -INFINITY;
  return x;
}

// The body of the three selection kernels.  Logits row r selects for slot b (r == b without a slot map).  SEL_PLAIN is
// tn_greedy_select_bf16: every row advances, finished rows take pad.  SEL_SLOTS is tn_greedy_select_slots_bf16: a
// finished (or idle) slot does not advance at all (pad in next_ids, nothing else written), and a slot also finishes
// when its length reaches limit[b].  SEL_VERIFY is position `extra` of a speculative block (tn_verify_select_bf16): the
// history is row b followed by the draft tokens draft[0 .. extra), a finished row picks nothing, and the pick goes to
// *pick instead of the decoding state.
template <int MODE>
__device__ __forceinline__ void greedy_select_row(
    const bf16* __restrict__ logits, int64_t ld, int V, int64_t* __restrict__ history, int64_t ld_hist,
    int32_t* __restrict__ length, int64_t* __restrict__ positions, int64_t* __restrict__ next_ids,
    int32_t* __restrict__ finished, const int32_t* __restrict__ limit, float penalty, int ngram, int64_t eos,
    int64_t pad, const int r, const int b, const int64_t* __restrict__ draft = nullptr, int extra = 0,
    int64_t* __restrict__ pick = nullptr) {
  constexpr bool SLOTS = MODE == SEL_SLOTS, VERIFY = MODE == SEL_VERIFY;
  extern __shared__ uint32_t bits[];   // [2][words]: repetition set, banned set
  __shared__ float s_val[SEL_THREADS / 32];
  __shared__ int s_idx[SEL_THREADS / 32];
  const int tid = threadIdx.x;
  if ((SLOTS || VERIFY) && finished[b]) {   // uniform over the CTA: no barrier has been reached yet
    if (tid == 0 && SLOTS) next_ids[b] = pad;
    return;
  }
  const int words = (V + 31) / 32;
  uint32_t* rep = bits;
  uint32_t* ban = bits + words;
  const int len = processor_front<VERIFY>(bits, rep, ban, words, V, history, ld_hist, length, b, draft, extra, penalty,
                                          ngram);
  const bool use_pen = penalty != 1.0f;
  const bf16* row = logits + int64_t(r) * ld;
  float best = -INFINITY;
  int bi = -1;
  for (int v = tid; v < V; v += SEL_THREADS) {   // increasing v per thread: strict '>' keeps the lowest index
    float x = __bfloat162float(row[v]);
    if (use_pen && (rep[v >> 5] >> (v & 31) & 1u)) x = x < 0.f ? x * penalty : x / penalty;
    if (ban[v >> 5] >> (v & 31) & 1u) x = -INFINITY;
    if (argmax_better(x, v, best, bi)) { best = x; bi = v; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (argmax_better(ov, oi, best, bi)) { best = ov; bi = oi; }
  }
  if ((tid & 31) == 0) { s_val[tid >> 5] = best; s_idx[tid >> 5] = bi; }
  __syncthreads();
  if (tid == 0) {
    best = s_val[0]; bi = s_idx[0];
    for (int w = 1; w < SEL_THREADS / 32; ++w) {
      const float ov = s_val[w];
      const int oi = s_idx[w];
      if (argmax_better(ov, oi, best, bi)) { best = ov; bi = oi; }
    }
    if constexpr (VERIFY) {
      *pick = bi;
    } else {
      const int fin = SLOTS ? 0 : finished[b];
      const int64_t tok = fin ? pad : int64_t(bi);
      if (len < ld_hist) history[int64_t(b) * ld_hist + len] = tok;
      next_ids[b] = tok;
      length[b] = len + 1;
      positions[b] += 1;
      if (tok == eos || (SLOTS && len + 1 == limit[b])) finished[b] = 1;
    }
  }
}

__global__ void __launch_bounds__(SEL_THREADS) greedy_select_kernel(
    const bf16* __restrict__ logits, int64_t ld, int V, int64_t* __restrict__ history, int64_t ld_hist,
    int32_t* __restrict__ length, int64_t* __restrict__ positions, int64_t* __restrict__ next_ids,
    int32_t* __restrict__ finished, float penalty, int ngram, int64_t eos, int64_t pad) {
  greedy_select_row<SEL_PLAIN>(logits, ld, V, history, ld_hist, length, positions, next_ids, finished, nullptr, penalty,
                           ngram, eos, pad, blockIdx.x, blockIdx.x);
}

// ---------------------------------------------------------------------------------------------------------------
// speculative verification: the picks of k + 1 positions (grid (k + 1, B)), then per row the accepted prefix
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(SEL_THREADS) verify_pick_kernel(
    const bf16* __restrict__ logits, int64_t ld, int V, int64_t* __restrict__ history, int64_t ld_hist,
    int32_t* __restrict__ length, int32_t* __restrict__ finished, const int64_t* __restrict__ draft, int k,
    int64_t* __restrict__ picks, float penalty, int ngram) {
  const int j = blockIdx.x, b = blockIdx.y;
  const int r = b * (k + 1) + j;
  greedy_select_row<SEL_VERIFY>(logits, ld, V, history, ld_hist, length, nullptr, nullptr, finished, nullptr, penalty,
                                ngram, 0, 0, r, b, draft + int64_t(b) * k, j, picks + r);
}

// The commit of both verify selections, one thread per row: emit picks 0..n, stopping after an eos and at the row's
// limit, then advance the row's state as the slot selection does for one token.  Greedy (verify_pick_kernel's picks):
// n = the leading draft tokens equal to their pick.  SAMPLED (spec_sample_verify_kernel's picks): a pick x >= 0 is an
// accepted draft token, ~t the row's last token t.  A finished row does not advance.
template <bool SAMPLED>
__device__ __forceinline__ void commit_row(const int64_t* __restrict__ picks, const int64_t* __restrict__ draft, int k,
                                           int b, int64_t* __restrict__ history, int64_t ld_hist,
                                           int32_t* __restrict__ length, int64_t* __restrict__ positions,
                                           int64_t* __restrict__ next_ids, int32_t* __restrict__ finished,
                                           const int32_t* __restrict__ limit, int64_t eos, int64_t pad) {
  if (finished[b]) {   // a finished row does not advance
    next_ids[b] = pad;
    return;
  }
  const int len = length[b], lim = limit[b];
  const int64_t* pk = picks + int64_t(b) * (k + 1);
  const int64_t* d = draft + int64_t(b) * k;
  int c = 0;
  int64_t tok;
  bool stop;
  do {
    tok = SAMPLED && pk[c] < 0 ? ~pk[c] : pk[c];
    if (len + c < ld_hist) history[int64_t(b) * ld_hist + len + c] = tok;
    ++c;
    stop = tok == eos || len + c >= lim || c == k + 1 || (SAMPLED ? pk[c - 1] < 0 : d[c - 1] != tok);
  } while (!stop);
  length[b] = len + c;
  positions[b] += c;
  next_ids[b] = tok;
  if (tok == eos || len + c >= lim) finished[b] = 1;
}

__global__ void verify_commit_kernel(const int64_t* __restrict__ picks, const int64_t* __restrict__ draft, int k, int B,
                                     int64_t* __restrict__ history, int64_t ld_hist, int32_t* __restrict__ length,
                                     int64_t* __restrict__ positions, int64_t* __restrict__ next_ids,
                                     int32_t* __restrict__ finished, const int32_t* __restrict__ limit, int64_t eos,
                                     int64_t pad) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  commit_row<false>(picks, draft, k, b, history, ld_hist, length, positions, next_ids, finished, limit, eos, pad);
}

__global__ void spec_commit_kernel(const int64_t* __restrict__ picks, int k, int B, int64_t* __restrict__ history,
                                   int64_t ld_hist, int32_t* __restrict__ length, int64_t* __restrict__ positions,
                                   int64_t* __restrict__ next_ids, int32_t* __restrict__ finished,
                                   const int32_t* __restrict__ limit, int64_t eos, int64_t pad) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  commit_row<true>(picks, picks, k, b, history, ld_hist, length, positions, next_ids, finished, limit, eos, pad);
}

// ---------------------------------------------------------------------------------------------------------------
// continuous batching: slot-addressed admission state, K/V scatter of a packed prefill, slot-aware selection
// ---------------------------------------------------------------------------------------------------------------
constexpr int ADMIT_MAX = TN_ADMIT_MAX;       // documents per admission launch
constexpr int SEL_MAX_MAP = TN_SELECT_MAX_MAP;  // rows of an explicit row -> slot map

// The admission table travels in the launch's parameter block (2 KB), so the entry points validate every slot and
// length on the host and admission needs no host-to-device copy.
struct AdmitTable {
  int n;
  int src_row[ADMIT_MAX], slot[ADMIT_MAX], len[ADMIT_MAX], limit[ADMIT_MAX];
};

struct SlotMap {
  int use_map;                       // 0: row r is slot r
  int slot[SEL_MAX_MAP];
};

__global__ void __launch_bounds__(SEL_THREADS, 1) greedy_select_slots_kernel(
    const bf16* __restrict__ logits, int64_t ld, int V, int64_t* __restrict__ history, int64_t ld_hist,
    int32_t* __restrict__ length, int64_t* __restrict__ positions, int64_t* __restrict__ next_ids,
    int32_t* __restrict__ finished, const int32_t* __restrict__ limit, float penalty, int ngram, int64_t eos,
    int64_t pad, const SlotMap map) {
  const int r = blockIdx.x;
  greedy_select_row<SEL_SLOTS>(logits, ld, V, history, ld_hist, length, positions, next_ids, finished, limit, penalty, ngram,
                          eos, pad, r, map.use_map ? map.slot[r] : r);
}

// ---------------------------------------------------------------------------------------------------------------
// multinomial sampling over cache slots: HF's processors, temperature, top-k, top-p, a counter-based Philox draw
// ---------------------------------------------------------------------------------------------------------------
constexpr int SMP_BINS = 2048;                   // radix digits of 11, 11 and 10 bits over the 32-bit order key
constexpr float SMP_ONE = 1099511627776.f;       // 2^40: fixed-point weight of the row maximum

struct SampleMap {
  SlotMap slots;
  int64_t key[SEL_MAX_MAP];                      // mapped rows: the prompt's stream key, stored into stream_key[slot]
};

// order-preserving uint32 key of a non-NaN float; -0 and +0 are one value, so they get one key
__device__ __forceinline__ uint32_t order_key(float x) {
  const uint32_t u = __float_as_uint(x == 0.f ? 0.f : x);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// exp(x - m) in fixed point (2^40 at the maximum m); 0 below about m - 28.4, where the token is never drawn
__device__ __forceinline__ unsigned long long fixed_weight(float x, float m) {
  return __float2ull_rn(__expf(x - m) * SMP_ONE);
}

// Exact integer weights: u64 for one distribution's weights (<= 2^40 each, V * 2^40 < 2^64 in total), u128 for the
// speculative residual (products of a weight and a total, < 2^100 each).  Warp shuffles of both.
typedef unsigned __int128 u128;
__device__ __forceinline__ unsigned long long shfl_up(unsigned long long x, int o) {
  return __shfl_up_sync(0xffffffffu, x, o);
}
__device__ __forceinline__ unsigned long long shfl_xor(unsigned long long x, int o) {
  return __shfl_xor_sync(0xffffffffu, x, o);
}
__device__ __forceinline__ unsigned long long shfl_idx(unsigned long long x, int l) {
  return __shfl_sync(0xffffffffu, x, l);
}
__device__ __forceinline__ u128 shfl_up(u128 x, int o) {
  return (u128(shfl_up((unsigned long long)(x >> 64), o)) << 64) | shfl_up((unsigned long long)x, o);
}
__device__ __forceinline__ u128 shfl_xor(u128 x, int o) {
  return (u128(shfl_xor((unsigned long long)(x >> 64), o)) << 64) | shfl_xor((unsigned long long)x, o);
}
__device__ __forceinline__ u128 shfl_idx(u128 x, int l) {
  return (u128(shfl_idx((unsigned long long)(x >> 64), l)) << 64) | shfl_idx((unsigned long long)x, l);
}

// Inclusive scan of one W per thread in thread order over the CTA; returns the exclusive prefix, *total the sum.
// Every thread of the CTA calls it (it holds two barriers and reuses `scratch` [33]).
template <typename W>
__device__ __forceinline__ W block_scan(W x, W* scratch, W* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  W inc = x;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const W y = shfl_up(inc, o);
    if (lane >= o) inc += y;
  }
  if (lane == 31) scratch[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    W w = scratch[lane], wi = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const W y = shfl_up(wi, o);
      if (lane >= o) wi += y;
    }
    scratch[lane] = wi - w;                      // exclusive prefix of each warp
    if (lane == 31) scratch[32] = wi;
  }
  __syncthreads();
  *total = scratch[32];
  return scratch[warp] + inc - x;
}

struct BinPick {
  int bin;
  unsigned long long above, total;
};

// The radix step of both thresholds: walking hist[0, nb) from the top bin down, the bin where the running sum reaches
// `need` (the sum of the bins above it < need <= that sum + its own).  need_of(total of the histogram) gives `need`.
template <typename T, typename Need>
__device__ BinPick find_bin(const T* hist, int nb, Need need_of, unsigned long long* scratch, BinPick* out) {
  const int per = nb / SEL_THREADS, top = nb - 1 - per * int(threadIdx.x);   // this thread's bins, descending
  unsigned long long s = 0;
  for (int i = 0; i < per; ++i) s += hist[top - i];
  unsigned long long total;
  unsigned long long a = block_scan(s, scratch, &total);
  const unsigned long long need = need_of(total);
  for (int i = 0; i < per; ++i) {
    const unsigned long long h = hist[top - i];
    if (a < need && a + h >= need) *out = BinPick{top - i, a, total};
    a += h;
  }
  __syncthreads();
  const BinPick p = *out;
  __syncthreads();                               // `out` and `hist` may be rewritten after this
  return p;
}

// Shared memory of the sampling passes (declared by each kernel, used by the passes below)
struct SampleShared {
  unsigned long long* hist;                      // [SMP_BINS]; its first half is also the u32 count histogram
  unsigned long long* scan;                      // [33]
  BinPick* pick;
  float* val;                                    // [SEL_THREADS / 32]
  int* idx;                                      // [SEL_THREADS / 32]
};

// What the passes find in one processed row: its maximum m at bi (argmax_better's order, the pick of a degenerate row)
// and the order key t_key of the kept set's lowest value (a token is kept iff order_key(value) >= t_key).  A row whose
// m is not finite (a NaN, an infinite maximum, every token banned) is degenerate and has no t_key.
struct SampleCut {
  float m;
  int bi;
  uint32_t t_key;
};

// The passes over value(v), v in [0, V) (re-read from L2): the max, fused with the first top-k histogram; two more
// top-k histograms; three top-p mass histograms.  sh.hist must be zero, and a barrier reached, before the call.
template <typename Value>
__device__ __forceinline__ SampleCut sample_cut(Value value, int V, int top_k, float top_p, const SampleShared& sh) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const bool use_k = top_k > 0 && top_k < V, use_p = top_p < 1.0f;
  uint32_t* cnt = reinterpret_cast<uint32_t*>(sh.hist);
  // pass 1: the argmax in argmax_better's order (the pick of a degenerate row) and the first top-k count histogram
  float best = -INFINITY;
  int bi = -1;
  for (int v = tid; v < V; v += SEL_THREADS) {
    const float x = value(v);
    if (argmax_better(x, v, best, bi)) { best = x; bi = v; }
    if (use_k && x == x) atomicAdd(&cnt[order_key(x) >> 21], 1u);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (argmax_better(ov, oi, best, bi)) { best = ov; bi = oi; }
  }
  if (lane == 0) { sh.val[warp] = best; sh.idx[warp] = bi; }
  __syncthreads();
  best = sh.val[0]; bi = sh.idx[0];
  for (int w = 1; w < SEL_THREADS / 32; ++w)
    if (argmax_better(sh.val[w], sh.idx[w], best, bi)) { best = sh.val[w]; bi = sh.idx[w]; }
  const float m = best;
  if (!(m > -INFINITY && m < INFINITY)) return SampleCut{m, bi, 0u};

  // radix digit l covers key bits [shift(l), shift(l) + width(l)); keys whose higher bits equal `pre` take part
  const auto width = [](int l) { return l < 2 ? 11 : 10; };
  const auto shift = [](int l) { return l < 2 ? 21 - 11 * l : 0; };
  const auto in_prefix = [&](uint32_t k, int l, uint32_t pre) {
    return (uint64_t(k) >> (shift(l) + width(l))) == pre;
  };
  const auto digit = [&](uint32_t k, int l) { return (k >> shift(l)) & ((1u << width(l)) - 1u); };

  // top-k: the k-th largest key (ties included: every key >= it is kept)
  uint32_t lo_key = 0u;
  if (use_k) {
    uint32_t pre = 0u;
    unsigned long long need = unsigned(top_k);
    for (int l = 0; l < 3; ++l) {
      if (l > 0) {
        for (int i = tid; i < SMP_BINS; i += SEL_THREADS) cnt[i] = 0u;
        __syncthreads();
        for (int v = tid; v < V; v += SEL_THREADS) {
          const uint32_t k = order_key(value(v));
          if (in_prefix(k, l, pre)) atomicAdd(&cnt[digit(k, l)], 1u);
        }
        __syncthreads();
      }
      const BinPick p = find_bin(cnt, 1 << width(l), [&](unsigned long long) { return need; }, sh.scan, sh.pick);
      need -= p.above;
      pre = (pre << width(l)) | uint32_t(p.bin);
    }
    lo_key = pre;
  }

  // top-p over the top-k set: the lowest value group whose kept mass strictly above it is < top_p * Z (the row maximum
  // always stays); the mass is in fixed point, so every sum below is exact in any order
  uint32_t t_key = lo_key;
  if (use_p) {
    if (top_p <= 0.f) {
      t_key = order_key(m);
    } else {
      uint32_t pre = 0u;
      unsigned long long need = 0;
      for (int l = 0; l < 3; ++l) {
        for (int i = tid; i < SMP_BINS; i += SEL_THREADS) sh.hist[i] = 0ull;
        __syncthreads();
        for (int v = tid; v < V; v += SEL_THREADS) {
          const float x = value(v);
          const uint32_t k = order_key(x);
          if (k >= lo_key && in_prefix(k, l, pre)) {
            const unsigned long long w = fixed_weight(x, m);
            if (w) atomicAdd(&sh.hist[digit(k, l)], w);
          }
        }
        __syncthreads();
        const auto need_of = [&](unsigned long long total) {
          // level 0: ceil(top_p * Z); an integer mass is < top_p * Z iff it is < this
          return l == 0 ? (unsigned long long)ceil(double(top_p) * double(total)) : need;
        };
        const BinPick p = find_bin(sh.hist, 1 << width(l), need_of, sh.scan, sh.pick);
        need = need_of(p.total) - p.above;
        pre = (pre << width(l)) | uint32_t(p.bin);
      }
      t_key = pre;
    }
  }
  return SampleCut{m, bi, t_key};
}

// the fixed-point weight of token v in the distribution `c` of value(): exp(x - m) * 2^40 if kept, else 0
template <typename Value>
__device__ __forceinline__ unsigned long long kept_weight(Value value, int v, const SampleCut& c) {
  const float x = value(v);
  return order_key(x) >= c.t_key ? fixed_weight(x, c.m) : 0ull;
}

// Inverse-CDF draw in index order over the integer weights weight(v) of v in [0, V): each warp sums its index range
// [warp * chunk, warp * chunk + chunk), a block scan gives the total Z, target_of(Z) in [0, Z) picks the token whose
// interval of the prefix sums holds it, and the warp whose range holds the target walks it.  The token is in *s_tok
// after the closing barrier (not written when Z = 0).
template <typename W, typename Weight, typename Target>
__device__ __forceinline__ void draw_index_order(Weight weight, int V, Target target_of, W* scan, int* s_tok) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int words = (V + 31) / 32;
  const int chunk = ((words + 31) / 32) * 32;
  const int v0 = warp * chunk, v1 = min(V, v0 + chunk);
  const auto range_weight = [&](int v) -> W { return v >= v1 ? W(0) : weight(v); };
  W s = 0;
  for (int v = v0 + lane; v < v1; v += 32) s += range_weight(v);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += shfl_xor(s, o);
  W total;
  const W before = block_scan(lane == 0 ? s : W(0), scan, &total);
  const W target = target_of(total);
  const W w_before = shfl_idx(before, 0);
  if (target >= w_before && target - w_before < s) {   // this warp's range holds the target (uniform over the warp)
    W rest = target - w_before;                        // the target's offset past the chunks walked so far
    for (int j = v0; j < v1; j += 32) {
      const W w = range_weight(j + lane);
      W inc = w;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const W y = shfl_up(inc, o);
        if (lane >= o) inc += y;
      }
      const bool hit = rest >= inc - w && rest < inc;
      if (__any_sync(0xffffffffu, hit)) {
        if (hit) *s_tok = j + lane;
        break;
      }
      rest -= shfl_idx(inc, 31);
    }
  }
  __syncthreads();
}

// Philox4x32-10 keyed by the seed at counter (position in the row, purpose, stream key): 64 random bits
constexpr uint32_t RND_TOKEN = 0, RND_ACCEPT = 1, RND_RESIDUAL = 2;   // purposes
__device__ __forceinline__ uint64_t philox_u64(uint64_t seed, int pos, uint32_t purpose, int64_t key) {
  const uint4 rnd = curand_Philox4x32_10(make_uint4(uint32_t(pos), purpose, uint32_t(uint64_t(key)),
                                                    uint32_t(uint64_t(key) >> 32)),
                                         make_uint2(uint32_t(seed), uint32_t(seed >> 32)));
  return (uint64_t(rnd.y) << 32) | rnd.x;
}

// One CTA per logits row; the slot rules, state writes and idle handling of greedy_select_slots_kernel.  Passes over the
// row (re-read from L2): those of sample_cut; the kept mass of each warp's index range; then one warp walks its range to
// the drawn token.
__global__ void __launch_bounds__(SEL_THREADS, 1) sample_select_slots_kernel(
    const bf16* __restrict__ logits, int64_t ld, int V, int64_t* __restrict__ history, int64_t ld_hist,
    int32_t* __restrict__ length, int64_t* __restrict__ positions, int64_t* __restrict__ next_ids,
    int32_t* __restrict__ finished, const int32_t* __restrict__ limit, int64_t* __restrict__ stream_key, float penalty,
    int ngram, float temperature, int top_k, float top_p, uint64_t seed, int64_t eos, int64_t pad,
    const SampleMap map) {
  extern __shared__ uint32_t bits[];             // [2][words]: repetition set, banned set
  __shared__ unsigned long long s_hist[SMP_BINS];
  __shared__ unsigned long long s_scan[33];
  __shared__ BinPick s_pick;
  __shared__ float s_val[SEL_THREADS / 32];
  __shared__ int s_idx[SEL_THREADS / 32];
  __shared__ int s_tok;
  const int r = blockIdx.x, tid = threadIdx.x;
  const int b = map.slots.use_map ? map.slots.slot[r] : r;
  if (finished[b]) {                             // uniform over the CTA: no barrier has been reached yet
    if (tid == 0) next_ids[b] = pad;
    return;
  }
  const int64_t key = map.slots.use_map ? map.key[r] : stream_key[b];
  for (int i = tid; i < SMP_BINS; i += SEL_THREADS) s_hist[i] = 0ull;
  const int words = (V + 31) / 32;
  uint32_t* rep = bits;
  uint32_t* ban = bits + words;
  const int len = processor_front<false>(bits, rep, ban, words, V, history, ld_hist, length, b, nullptr, 0, penalty,
                                         ngram);
  const bool use_pen = penalty != 1.0f, use_temp = temperature != 1.0f;
  const bf16* row = logits + int64_t(r) * ld;
  const auto value = [&](int v) {                // TemperatureLogitsWarper: a true division, as HF divides
    const float x = processed_logit(row, v, rep, ban, use_pen, penalty);
    return use_temp ? x / temperature : x;
  };
  const auto commit = [&](int64_t tok) {         // one thread: the writes of greedy_select_slots_kernel
    if (map.slots.use_map) stream_key[b] = key;
    if (len < ld_hist) history[int64_t(b) * ld_hist + len] = tok;
    next_ids[b] = tok;
    length[b] = len + 1;
    positions[b] += 1;
    if (tok == eos || len + 1 == limit[b]) finished[b] = 1;
  };
  const SampleCut c = sample_cut(value, V, top_k, top_p, SampleShared{s_hist, s_scan, &s_pick, s_val, s_idx});
  // a NaN, an infinite maximum or nothing drawable (every token banned): the greedy kernel's pick
  if (!(c.m > -INFINITY && c.m < INFINITY)) {
    if (tid == 0) commit(c.bi);
    return;
  }
  // the draw in index order: a target in [0, Z)
  draw_index_order<unsigned long long>(
      [&](int v) { return kept_weight(value, v, c); }, V,
      [&](unsigned long long total) { return __umul64hi(philox_u64(seed, len, RND_TOKEN, key), total); }, s_scan,
      &s_tok);
  if (tid == 0) commit(s_tok);
}

// ---------------------------------------------------------------------------------------------------------------
// speculative sampling (Leviathan et al. 2023, Algorithm 1): grid (k + 1, B), then the commit of verify_select
// ---------------------------------------------------------------------------------------------------------------
// floor(r * X / 2^64), exact for X < 2^114 (the 64 x 64 high half carries the low word's share)
__device__ __forceinline__ u128 mul_hi64(uint64_t r, u128 X) {
  return u128(r) * uint64_t(X >> 64) + __umul64hi(r, uint64_t(X));
}

// CTA (j, b): position j of slot b's block, whose context is the slot's history followed by draft[b, 0 .. j).  p is the
// sampling distribution of target row b*(k+1) + j, q that of draft row b*k + j (j < k), both with the same processor
// bitmaps and passes as sample_select_slots_kernel, in 2^40 fixed point: p(v) = wp(v) / Zp, q(v) = wq(v) / Zq.  A
// degenerate draft row drew its greedy pick: q is a point mass there (wq = 1 at that pick, Zq = 1).
//   j < k: accept x = draft[b, j] iff floor(r * wq(x) * Zp / 2^64) < wp(x) * Zq for the 64-bit Philox draw r of
//          (len, RND_ACCEPT): probability min(1, p(x) / q(x)) to within 2^-64.  Accepted: picks[b, j] = x.
//   otherwise (rejected, or j = k): the token drawn from max(0, wp * Zq - wq * Zp) (wq = 0, Zq = 1 at j = k: p itself)
//          in index order with the draw (len, RND_RESIDUAL); picks[b, j] = ~token.
// A degenerate target row stops the row there with its greedy pick: picks[b, j] = ~pick.  Finished slots: nothing.
__global__ void __launch_bounds__(SEL_THREADS, 1) spec_sample_verify_kernel(
    const bf16* __restrict__ logits, int64_t ld, const bf16* __restrict__ dlogits, int64_t ldd, int V,
    const int64_t* __restrict__ draft, int k, const int64_t* __restrict__ history, int64_t ld_hist,
    const int32_t* __restrict__ length, const int32_t* __restrict__ finished, const int64_t* __restrict__ stream_key,
    int64_t* __restrict__ picks, float penalty, int ngram, float temperature, int top_k, float top_p, uint64_t seed) {
  extern __shared__ uint32_t bits[];             // [2][words]: repetition set, banned set
  __shared__ unsigned long long s_hist[SMP_BINS];
  __shared__ u128 s_scan[33];
  __shared__ BinPick s_pick;
  __shared__ float s_val[SEL_THREADS / 32];
  __shared__ int s_idx[SEL_THREADS / 32];
  __shared__ int s_tok;
  __shared__ SampleCut s_cut[2];                 // p, q
  __shared__ unsigned long long s_tot[2];        // Zp, Zq
  __shared__ bool s_point;                       // q is a point mass (a degenerate draft row)
  const int j = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  if (finished[b]) return;                       // uniform over the CTA
  unsigned long long* scan64 = reinterpret_cast<unsigned long long*>(s_scan);
  const SampleShared sh{s_hist, scan64, &s_pick, s_val, s_idx};
  for (int i = tid; i < SMP_BINS; i += SEL_THREADS) s_hist[i] = 0ull;
  const int words = (V + 31) / 32;
  uint32_t* rep = bits;
  uint32_t* ban = bits + words;
  const int64_t* d = draft + int64_t(b) * k;
  const int len = processor_front<true>(bits, rep, ban, words, V, history, ld_hist, length, b, d, j, penalty, ngram);
  const bool use_pen = penalty != 1.0f, use_temp = temperature != 1.0f;
  const bf16* prow = logits + (int64_t(b) * (k + 1) + j) * ld;
  const bf16* qrow = dlogits + (int64_t(b) * k + min(j, k - 1)) * ldd;
  const auto value_p = [&](int v) {
    const float x = processed_logit(prow, v, rep, ban, use_pen, penalty);
    return use_temp ? x / temperature : x;
  };
  const auto value_q = [&](int v) {
    const float x = processed_logit(qrow, v, rep, ban, use_pen, penalty);
    return use_temp ? x / temperature : x;
  };
  const auto total = [&](auto weight) {          // sum of weight(v) over the row (ends on a barrier)
    unsigned long long s = 0, z;
    for (int v = tid; v < V; v += SEL_THREADS) s += weight(v);
    block_scan(s, scan64, &z);
    __syncthreads();
    return z;
  };
  int64_t* out = picks + int64_t(b) * (k + 1) + j;
  {
    const SampleCut P = sample_cut(value_p, V, top_k, top_p, sh);
    if (!(P.m > -INFINITY && P.m < INFINITY)) {
      if (tid == 0) *out = ~int64_t(P.bi);
      return;
    }
    const unsigned long long Zp = total([&](int v) { return kept_weight(value_p, v, P); });
    if (tid == 0) { s_cut[0] = P; s_tot[0] = Zp; }
  }
  if (j < k) {
    for (int i = tid; i < SMP_BINS; i += SEL_THREADS) s_hist[i] = 0ull;
    __syncthreads();
    const SampleCut Q = sample_cut(value_q, V, top_k, top_p, sh);
    const bool q_point = !(Q.m > -INFINITY && Q.m < INFINITY);
    const unsigned long long Zq = q_point ? 1ull : total([&](int v) { return kept_weight(value_q, v, Q); });
    if (tid == 0) { s_cut[1] = Q; s_tot[1] = Zq; s_point = q_point; }
  }
  __syncthreads();
  // p's and q's cuts and totals come back from shared memory: nothing of the p pass stays live in registers across
  // the q pass (a 1024-thread CTA has 64 registers per thread)
  const SampleCut P = s_cut[0];
  const unsigned long long Zp = s_tot[0];
  const SampleCut Q = j < k ? s_cut[1] : SampleCut{0.f, -1, 0u};
  const unsigned long long Zq = j < k ? s_tot[1] : 1ull;
  const bool q_point = j < k && s_point;
  const auto wp = [&](int v) { return kept_weight(value_p, v, P); };
  const auto wq = [&](int v) -> unsigned long long {
    if (j == k) return 0ull;
    if (q_point) return v == Q.bi ? 1ull : 0ull;
    return kept_weight(value_q, v, Q);
  };
  const int64_t key = stream_key[b];
  if (j < k) {
    const int64_t x = d[j];
    const bool drawable = x >= 0 && x < V;
    const u128 A = drawable ? u128(wp(int(x))) * Zq : u128(0);
    const u128 Bq = drawable ? u128(wq(int(x))) * Zp : u128(0);
    if (mul_hi64(philox_u64(seed, len, RND_ACCEPT, key), Bq) < A) {   // uniform over the CTA
      if (tid == 0) *out = x;
      return;
    }
  }
  if (tid == 0) s_tok = P.bi;                    // an empty residual (x not drawable from q, and q == p): p's argmax
  const auto residual = [&](int v) -> u128 {
    const u128 a = u128(wp(v)) * Zq, c = u128(wq(v)) * Zp;
    return a > c ? a - c : u128(0);
  };
  draw_index_order<u128>(residual, V, [&](u128 R) { return mul_hi64(philox_u64(seed, len, RND_RESIDUAL, key), R); },
                         s_scan, &s_tok);
  if (tid == 0) *out = ~int64_t(s_tok);
}

// grid (longest document, documents): row t of document j -> cache row t of slot j, 16-byte copies
__global__ void kv_scatter_kernel(const bf16* __restrict__ K, int64_t ldk, const bf16* __restrict__ V, int64_t ldv,
                                  bf16* __restrict__ Kc, bf16* __restrict__ Vc, int64_t ld_tok, int64_t ld_batch,
                                  const AdmitTable tab, int width) {
  const int t = blockIdx.x, j = blockIdx.y;
  if (t >= tab.len[j]) return;
  copy_kv_row(K, ldk, V, ldv, Kc, Vc, int64_t(tab.src_row[j]) + t,
              int64_t(tab.slot[j]) * ld_batch + int64_t(t) * ld_tok, width);
}

constexpr int ADMIT_THREADS = 256;

// one CTA per admitted document: its slot's decoding state and the prompt ids of its history
__global__ void __launch_bounds__(ADMIT_THREADS) slot_admit_kernel(
    const AdmitTable tab, const int64_t* __restrict__ ids, const int32_t* __restrict__ doc_ids,
    const int64_t* __restrict__ position_ids, int64_t* __restrict__ history, int64_t ld_hist,
    int32_t* __restrict__ kv_start, int32_t* __restrict__ kv_end, int64_t* __restrict__ positions,
    int32_t* __restrict__ finished, int32_t* __restrict__ limit) {
  __shared__ int s_start[ADMIT_THREADS / 32];
  const int j = blockIdx.x, tid = threadIdx.x;
  const int src = tab.src_row[j], b = tab.slot[j], T = tab.len[j];
  const int32_t* doc = doc_ids + src;
  const int32_t last = doc[T - 1];
  int start = 0;                       // first row of the last document = 1 + the last row outside it
  for (int t = tid; t < T; t += ADMIT_THREADS) {
    if (doc[t] != last) start = t + 1;
    history[int64_t(b) * ld_hist + t] = ids[src + t];
  }
  start = __reduce_max_sync(0xffffffffu, start);
  if ((tid & 31) == 0) s_start[tid >> 5] = start;
  __syncthreads();
  if (tid == 0) {
    for (int w = 1; w < ADMIT_THREADS / 32; ++w) start = max(start, s_start[w]);
    kv_start[b] = start;
    kv_end[b] = T;
    positions[b] = position_ids[src + T - 1];
    finished[b] = 0;
    limit[b] = tab.limit[j];
  }
}

}  // namespace tn

using namespace tn;

extern "C" int64_t tn_attn_decode_ws_floats(int B, int H, int KV, int S_cap) {
  if (B <= 0 || H <= 0 || KV <= 0 || S_cap <= 0) return 0;
  return int64_t(B) * H * decode_splits(B, KV, S_cap) * (ATT_HD + 2);
}

extern "C" int64_t tn_attn_decode_multi_ws_floats(int B, int Tq, int H, int KV, int S_cap) {
  if (Tq <= 0) return 0;
  return tn_attn_decode_ws_floats(B, H, KV, S_cap) * Tq;   // the splits of the single-query launch, per query
}

// both decode attention launches: Tq query rows per batch row (MULTI), the split count and chunking of (B, KV, S_cap)
template <bool MULTI>
static int decode_launch(const char* fn, const void* Q, int64_t ldq, const void* K, const void* V, int64_t ld_tok,
                         int64_t ld_batch, const int32_t* kv_start, const int32_t* kv_end, int B, int Tq, int H, int KV,
                         int S_cap, float scale, float* workspace, void* O, int64_t ldo, float* lse, tn_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  TN_REQUIRE(Q && K && V && kv_start && kv_end && workspace && O, "%s: null pointer", fn);
  TN_REQUIRE(B > 0 && H > 0 && KV > 0 && S_cap > 0 && H % KV == 0 && H / KV <= 16,
             "%s: bad dims B=%d H=%d KV=%d S_cap=%d (H/KV must be 1..16)", fn, B, H, KV, S_cap);
  TN_REQUIRE(ldq % 8 == 0 && ld_tok % 8 == 0 && ld_batch % 8 == 0 && ldo % 8 == 0,
             "%s: strides must be multiples of 8", fn);
  TN_REQUIRE(ldq >= int64_t(H) * ATT_HD && ldo >= int64_t(H) * ATT_HD && ld_tok >= int64_t(KV) * ATT_HD &&
                 ld_batch >= ld_tok * S_cap, "%s: stride smaller than the rows it must hold", fn);
  TN_REQUIRE(int64_t(B) * Tq <= 65535, "%s: grid too large (B*Tq = %lld)", fn, (long long)B * Tq);
  const int splits = decode_splits(B, KV, S_cap);
  DecodeParams p{};
  p.Q = static_cast<const bf16*>(Q); p.K = static_cast<const bf16*>(K); p.V = static_cast<const bf16*>(V);
  p.ldq = ldq; p.ld_tok = ld_tok; p.ld_batch = ld_batch;
  p.kv_start = kv_start; p.kv_end = kv_end;
  p.part_o = workspace;
  p.part_ml = workspace + int64_t(B) * Tq * H * splits * ATT_HD;
  p.H = H; p.KV = KV; p.S_cap = S_cap; p.splits = splits;
  p.chunk = ((S_cap + splits - 1) / splits + ATT_SUB - 1) / ATT_SUB * ATT_SUB;
  p.scale_log2 = scale * LOG2E;
  p.Tq = Tq;
  TN_CHECK_CUDA(attn_smem_optin<attn_decode_kernel<MULTI>>(DEC_SMEM));
  attn_decode_kernel<MULTI><<<dim3(splits, KV, B), DEC_THREADS, DEC_SMEM, stream>>>(p);
  TN_CHECK_CUDA(cudaGetLastError());
  attn_decode_merge_kernel<<<dim3(H, B * Tq), ATT_HD, 0, stream>>>(p.part_o, p.part_ml, static_cast<bf16*>(O), ldo, lse,
                                                                   H, splits);
  TN_CHECK_CUDA(cudaGetLastError());
  return TN_OK;
}

extern "C" int tn_attn_decode_bf16(const void* Q, int64_t ldq, const void* K, const void* V, int64_t ld_tok,
                                   int64_t ld_batch, const int32_t* kv_start, const int32_t* kv_end, int B, int H, int KV,
                                   int S_cap, float scale, float* workspace, void* O, int64_t ldo, float* lse,
                                   tn_stream_t stream_) {
  clear_error();
  return decode_launch<false>("tn_attn_decode_bf16", Q, ldq, K, V, ld_tok, ld_batch, kv_start, kv_end, B, 1, H, KV,
                              S_cap, scale, workspace, O, ldo, lse, stream_);
}

extern "C" int tn_attn_decode_multi_bf16(const void* Q, int64_t ldq, const void* K, const void* V, int64_t ld_tok,
                                         int64_t ld_batch, const int32_t* kv_start, const int32_t* kv_end, int B, int Tq,
                                         int H, int KV, int S_cap, float scale, float* workspace, void* O, int64_t ldo,
                                         float* lse, tn_stream_t stream_) {
  clear_error();
  TN_REQUIRE(Tq > 0 && KV > 0 && H % KV == 0 && int64_t(Tq) * (H / KV) <= 16 && Tq <= S_cap,
             "tn_attn_decode_multi_bf16: bad dims Tq=%d H=%d KV=%d S_cap=%d (Tq*H/KV must be 1..16)", Tq, H, KV, S_cap);
  return decode_launch<true>("tn_attn_decode_multi_bf16", Q, ldq, K, V, ld_tok, ld_batch, kv_start, kv_end, B, Tq, H, KV,
                             S_cap, scale, workspace, O, ldo, lse, stream_);
}

// the checks of both K/V copies (`map`: row_end or the admission table): pointers, dims, strides, 16-byte alignment
static int check_kv_copy(const char* fn, const void* K, int64_t ldk, const void* V, int64_t ldv, const void* Kc,
                         const void* Vc, int64_t ld_tok, int64_t ld_batch, const void* map, int B, int S_cap,
                         int width) {
  TN_REQUIRE(K && V && Kc && Vc && map, "%s: null pointer", fn);
  TN_REQUIRE(B > 0 && S_cap > 0 && width > 0 && width % 8 == 0, "%s: bad dims B=%d S_cap=%d width=%d", fn, B, S_cap,
             width);
  TN_REQUIRE(ldk % 8 == 0 && ldv % 8 == 0 && ld_tok % 8 == 0 && ld_batch % 8 == 0 && ldk >= width && ldv >= width &&
                 ld_tok >= width && ld_batch >= ld_tok * S_cap, "%s: bad strides", fn);
  TN_REQUIRE(((uintptr_t(K) | uintptr_t(V) | uintptr_t(Kc) | uintptr_t(Vc)) & 15) == 0,
             "%s: pointers must be 16-byte aligned", fn);
  return TN_OK;
}

extern "C" int tn_kv_append_bf16(const void* K, int64_t ldk, const void* V, int64_t ldv, void* K_cache, void* V_cache,
                                 int64_t ld_tok, int64_t ld_batch, const int32_t* row_end, int B, int T_new, int S_cap,
                                 int width, tn_stream_t stream_) {
  clear_error();
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (const int rc = check_kv_copy("tn_kv_append_bf16", K, ldk, V, ldv, K_cache, V_cache, ld_tok, ld_batch, row_end,
                                   B, S_cap, width)) return rc;
  TN_REQUIRE(T_new > 0 && S_cap >= T_new, "tn_kv_append_bf16: bad dims T_new=%d S_cap=%d", T_new, S_cap);
  TN_REQUIRE(T_new <= 65535 && B <= 65535, "tn_kv_append_bf16: grid too large");
  kv_append_kernel<<<dim3(T_new, B), 128, 0, stream>>>(
      static_cast<const bf16*>(K), ldk, static_cast<const bf16*>(V), ldv, static_cast<bf16*>(K_cache),
      static_cast<bf16*>(V_cache), ld_tok, ld_batch, row_end, T_new, S_cap, width);
  TN_CHECK_CUDA(cudaGetLastError());
  return TN_OK;
}

// both selection launches, one CTA per logits row: processor arguments, bitmap bytes, one-time shared-memory opt-in
template <auto kernel, typename... Args>
static int select_launch(const char* fn, dim3 rows, int V, float penalty, int ngram, tn_stream_t stream, Args... args) {
  TN_REQUIRE(penalty > 0.f, "%s: repetition_penalty must be > 0", fn);
  TN_REQUIRE(ngram >= 0, "%s: no_repeat_ngram_size must be >= 0", fn);
  const size_t smem = size_t(2) * ((V + 31) / 32) * sizeof(uint32_t);
  TN_REQUIRE(smem <= SEL_MAX_SMEM, "%s: vocabulary of %d too large for the shared-memory bitmaps", fn, V);
  static bool configured = false;
  if (!configured) {
    TN_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SEL_MAX_SMEM));
    configured = true;
  }
  kernel<<<rows, SEL_THREADS, smem, static_cast<cudaStream_t>(stream)>>>(args...);
  TN_CHECK_CUDA(cudaGetLastError());
  return TN_OK;
}

extern "C" int tn_greedy_select_bf16(const void* logits, int64_t ld, int B, int V, int64_t* history, int64_t ld_hist,
                                     int32_t* length, int64_t* positions, int64_t* next_ids, int32_t* finished,
                                     float repetition_penalty, int no_repeat_ngram_size, int64_t eos, int64_t pad,
                                     tn_stream_t stream_) {
  clear_error();
  TN_REQUIRE(logits && history && length && positions && next_ids && finished, "tn_greedy_select_bf16: null pointer");
  TN_REQUIRE(B > 0 && V > 0 && ld >= V && ld_hist > 0, "tn_greedy_select_bf16: bad dims B=%d V=%d", B, V);
  return select_launch<greedy_select_kernel>(
      "tn_greedy_select_bf16", B, V, repetition_penalty, no_repeat_ngram_size, stream_, static_cast<const bf16*>(logits),
      ld, V, history, ld_hist, length, positions, next_ids, finished, repetition_penalty, no_repeat_ngram_size, eos, pad);
}

// the checks of both slot selections; the host row -> slot map is checked and copied into `map` (passed by value)
static int slot_select_args(const char* fn, const void* logits, int64_t ld, int n_rows, const int32_t* row_slot, int B,
                            int V, const void* history, int64_t ld_hist, const void* length, const void* positions,
                            const void* next_ids, const void* finished, const void* limit, SlotMap* map) {
  TN_REQUIRE(logits && history && length && positions && next_ids && finished && limit, "%s: null pointer", fn);
  TN_REQUIRE(n_rows > 0 && B > 0 && V > 0 && ld >= V && ld_hist > 0, "%s: bad dims n_rows=%d B=%d V=%d", fn, n_rows, B,
             V);
  TN_REQUIRE(row_slot || n_rows == B, "%s: bad dims: without a row -> slot map n_rows (%d) must equal B (%d)", fn,
             n_rows, B);
  TN_REQUIRE(!row_slot || n_rows <= SEL_MAX_MAP, "%s: at most %d mapped rows, got %d", fn, SEL_MAX_MAP, n_rows);
  map->use_map = row_slot != nullptr;
  for (int r = 0; row_slot && r < n_rows; ++r) {   // the map is host memory: checked here, passed by value
    TN_REQUIRE(row_slot[r] >= 0 && row_slot[r] < B, "%s: slot %d out of range [0, %d)", fn, row_slot[r], B);
    for (int q = 0; q < r; ++q) TN_REQUIRE(row_slot[q] != row_slot[r], "%s: slot %d named twice", fn, row_slot[r]);
    map->slot[r] = row_slot[r];
  }
  return TN_OK;
}

extern "C" int tn_greedy_select_slots_bf16(const void* logits, int64_t ld, int n_rows, const int32_t* row_slot, int B,
                                           int V, int64_t* history, int64_t ld_hist, int32_t* length, int64_t* positions,
                                           int64_t* next_ids, int32_t* finished, const int32_t* limit,
                                           float repetition_penalty, int no_repeat_ngram_size, int64_t eos, int64_t pad,
                                           tn_stream_t stream_) {
  clear_error();
  SlotMap map{};
  if (const int rc = slot_select_args("tn_greedy_select_slots_bf16", logits, ld, n_rows, row_slot, B, V, history, ld_hist,
                                      length, positions, next_ids, finished, limit, &map)) return rc;
  return select_launch<greedy_select_slots_kernel>(
      "tn_greedy_select_slots_bf16", n_rows, V, repetition_penalty, no_repeat_ngram_size, stream_,
      static_cast<const bf16*>(logits), ld, V, history, ld_hist, length, positions, next_ids, finished, limit,
      repetition_penalty, no_repeat_ngram_size, eos, pad, map);
}

extern "C" int tn_sample_select_slots_bf16(const void* logits, int64_t ld, int n_rows, const int32_t* row_slot,
                                           const int64_t* row_key, int B, int V, int64_t* history, int64_t ld_hist,
                                           int32_t* length, int64_t* positions, int64_t* next_ids, int32_t* finished,
                                           const int32_t* limit, int64_t* stream_key, float repetition_penalty,
                                           int no_repeat_ngram_size, float temperature, int top_k, float top_p,
                                           int64_t seed, int64_t eos, int64_t pad, tn_stream_t stream_) {
  clear_error();
  const char* fn = "tn_sample_select_slots_bf16";
  SampleMap map{};
  if (const int rc = slot_select_args(fn, logits, ld, n_rows, row_slot, B, V, history, ld_hist, length, positions,
                                      next_ids, finished, limit, &map.slots)) return rc;
  TN_REQUIRE(stream_key && (row_key || !row_slot), "%s: null pointer (stream_key, or row_key with a row -> slot map)",
             fn);
  TN_REQUIRE(temperature > 0.f && temperature < INFINITY, "%s: temperature must be a finite number > 0", fn);
  TN_REQUIRE(top_k >= 0, "%s: top_k must be >= 0", fn);
  TN_REQUIRE(top_p >= 0.f && top_p <= 1.f, "%s: top_p must be in [0, 1]", fn);
  for (int r = 0; row_slot && r < n_rows; ++r) map.key[r] = row_key[r];
  return select_launch<sample_select_slots_kernel>(
      fn, n_rows, V, repetition_penalty, no_repeat_ngram_size, stream_, static_cast<const bf16*>(logits), ld, V, history,
      ld_hist, length, positions, next_ids, finished, limit, stream_key, repetition_penalty, no_repeat_ngram_size,
      temperature, top_k, top_p, uint64_t(seed), eos, pad, map);
}

extern "C" int tn_verify_select_bf16(const void* logits, int64_t ld, int B, int k, int V, const int64_t* draft,
                                     int64_t* history, int64_t ld_hist, int32_t* length, int64_t* positions,
                                     int64_t* next_ids, int32_t* finished, const int32_t* limit, int64_t* picks,
                                     float repetition_penalty, int no_repeat_ngram_size, int64_t eos, int64_t pad,
                                     tn_stream_t stream_) {
  clear_error();
  TN_REQUIRE(logits && draft && history && length && positions && next_ids && finished && limit && picks,
             "tn_verify_select_bf16: null pointer");
  TN_REQUIRE(B > 0 && k > 0 && V > 0 && ld >= V && ld_hist > 0, "tn_verify_select_bf16: bad dims B=%d k=%d V=%d", B, k,
             V);
  TN_REQUIRE(B <= 65535 && k < 65535, "tn_verify_select_bf16: grid too large (B=%d, k=%d)", B, k);
  const int rc = select_launch<verify_pick_kernel>(
      "tn_verify_select_bf16", dim3(k + 1, B), V, repetition_penalty, no_repeat_ngram_size, stream_,
      static_cast<const bf16*>(logits), ld, V, history, ld_hist, length, finished, draft, k, picks, repetition_penalty,
      no_repeat_ngram_size);
  if (rc != TN_OK) return rc;
  verify_commit_kernel<<<(B + 127) / 128, 128, 0, static_cast<cudaStream_t>(stream_)>>>(
      picks, draft, k, B, history, ld_hist, length, positions, next_ids, finished, limit, eos, pad);
  TN_CHECK_CUDA(cudaGetLastError());
  return TN_OK;
}

extern "C" int tn_spec_sample_verify_bf16(const void* logits, int64_t ld, const void* draft_logits, int64_t ldd, int B,
                                          int k, int V, const int64_t* draft, int64_t* history, int64_t ld_hist,
                                          int32_t* length, int64_t* positions, int64_t* next_ids, int32_t* finished,
                                          const int32_t* limit, const int64_t* stream_key, int64_t* picks,
                                          float repetition_penalty, int no_repeat_ngram_size, float temperature,
                                          int top_k, float top_p, int64_t seed, int64_t eos, int64_t pad,
                                          tn_stream_t stream_) {
  clear_error();
  const char* fn = "tn_spec_sample_verify_bf16";
  TN_REQUIRE(logits && draft_logits && draft && history && length && positions && next_ids && finished && limit &&
                 stream_key && picks, "%s: null pointer", fn);
  TN_REQUIRE(B > 0 && k > 0 && V > 0 && ld >= V && ldd >= V && ld_hist > 0, "%s: bad dims B=%d k=%d V=%d", fn, B, k, V);
  TN_REQUIRE(B <= 65535 && k < 65535, "%s: grid too large (B=%d, k=%d)", fn, B, k);
  TN_REQUIRE(temperature > 0.f && temperature < INFINITY, "%s: temperature must be a finite number > 0", fn);
  TN_REQUIRE(top_k >= 0, "%s: top_k must be >= 0", fn);
  TN_REQUIRE(top_p >= 0.f && top_p <= 1.f, "%s: top_p must be in [0, 1]", fn);
  const int rc = select_launch<spec_sample_verify_kernel>(
      fn, dim3(k + 1, B), V, repetition_penalty, no_repeat_ngram_size, stream_, static_cast<const bf16*>(logits), ld,
      static_cast<const bf16*>(draft_logits), ldd, V, draft, k, history, ld_hist, length, finished, stream_key, picks,
      repetition_penalty, no_repeat_ngram_size, temperature, top_k, top_p, uint64_t(seed));
  if (rc != TN_OK) return rc;
  spec_commit_kernel<<<(B + 127) / 128, 128, 0, static_cast<cudaStream_t>(stream_)>>>(
      picks, k, B, history, ld_hist, length, positions, next_ids, finished, limit, eos, pad);
  TN_CHECK_CUDA(cudaGetLastError());
  return TN_OK;
}

// docs: host [n_docs][4] int32 = (src_row, slot, len, limit); checked against the cache shape, returned by value
static int admit_table(const char* fn, const int32_t* docs, int n_docs, int B, int S_cap, int64_t n_src_rows,
                       AdmitTable* tab, int* max_len) {
  TN_REQUIRE(n_docs > 0 && n_docs <= ADMIT_MAX, "%s: bad dims: %d documents (1..%d per launch)", fn, n_docs, ADMIT_MAX);
  tab->n = n_docs;
  *max_len = 0;
  for (int j = 0; j < n_docs; ++j) {
    const int src = docs[4 * j], slot = docs[4 * j + 1], len = docs[4 * j + 2], lim = docs[4 * j + 3];
    TN_REQUIRE(slot >= 0 && slot < B, "%s: slot %d out of range [0, %d)", fn, slot, B);
    for (int q = 0; q < j; ++q) TN_REQUIRE(tab->slot[q] != slot, "%s: slot %d named twice", fn, slot);
    TN_REQUIRE(len > 0 && len <= S_cap, "%s: bad dims: document of %d rows for a cache of %d", fn, len, S_cap);
    TN_REQUIRE(src >= 0 && int64_t(src) + len <= n_src_rows, "%s: document rows [%d, %d) outside the %lld source rows",
               fn, src, src + len, (long long)n_src_rows);
    TN_REQUIRE(lim > len && lim <= S_cap, "%s: limit %d must be in (%d, %d]", fn, lim, len, S_cap);
    tab->src_row[j] = src; tab->slot[j] = slot; tab->len[j] = len; tab->limit[j] = lim;
    if (len > *max_len) *max_len = len;
  }
  return TN_OK;
}

extern "C" int tn_kv_scatter_bf16(const void* K, int64_t ldk, const void* V, int64_t ldv, int64_t n_src_rows,
                                  void* K_cache, void* V_cache, int64_t ld_tok, int64_t ld_batch, const int32_t* docs,
                                  int n_docs, int B, int S_cap, int width, tn_stream_t stream_) {
  clear_error();
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (const int rc = check_kv_copy("tn_kv_scatter_bf16", K, ldk, V, ldv, K_cache, V_cache, ld_tok, ld_batch, docs,
                                   B, S_cap, width)) return rc;
  TN_REQUIRE(n_src_rows > 0, "tn_kv_scatter_bf16: bad dims: %lld source rows", (long long)n_src_rows);
  AdmitTable tab{};
  int max_len = 0;
  const int rc = admit_table("tn_kv_scatter_bf16", docs, n_docs, B, S_cap, n_src_rows, &tab, &max_len);
  if (rc != TN_OK) return rc;
  kv_scatter_kernel<<<dim3(max_len, n_docs), 128, 0, stream>>>(
      static_cast<const bf16*>(K), ldk, static_cast<const bf16*>(V), ldv, static_cast<bf16*>(K_cache),
      static_cast<bf16*>(V_cache), ld_tok, ld_batch, tab, width);
  TN_CHECK_CUDA(cudaGetLastError());
  return TN_OK;
}

extern "C" int tn_slot_admit(const int32_t* docs, int n_docs, const int64_t* ids, const int32_t* doc_ids,
                             const int64_t* position_ids, int64_t n_src_rows, int64_t* history, int64_t ld_hist,
                             int32_t* kv_start, int32_t* kv_end, int64_t* positions, int32_t* finished, int32_t* limit,
                             int B, tn_stream_t stream_) {
  clear_error();
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  TN_REQUIRE(docs && ids && doc_ids && position_ids && history && kv_start && kv_end && positions && finished && limit,
             "tn_slot_admit: null pointer");
  TN_REQUIRE(B > 0 && ld_hist > 0 && n_src_rows > 0, "tn_slot_admit: bad dims B=%d ld_hist=%lld", B,
             (long long)ld_hist);
  AdmitTable tab{};
  int max_len = 0;
  const int rc = admit_table("tn_slot_admit", docs, n_docs, B, int(ld_hist < INT32_MAX ? ld_hist : INT32_MAX), n_src_rows,
                             &tab, &max_len);
  if (rc != TN_OK) return rc;
  slot_admit_kernel<<<n_docs, ADMIT_THREADS, 0, stream>>>(tab, ids, doc_ids, position_ids, history, ld_hist, kv_start,
                                                          kv_end, positions, finished, limit);
  TN_CHECK_CUDA(cudaGetLastError());
  return TN_OK;
}
