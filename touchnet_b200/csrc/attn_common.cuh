// touchnet_b200 :: shared definitions of the packed-sequence attention kernels (forward, dQ, dK/dV and decode): tile
// loads, fragment MMA loops, the document mask, the online softmax, work items and epilogues.
#pragma once
#include "common.cuh"

namespace tn {

constexpr int ATT_BLK = 128;  // q-block and kv-block size (tokens)
constexpr int ATT_HD = 128;   // head_dim
constexpr float LOG2E = 1.4426950408889634f;
constexpr float LN2 = 0.6931471805599453f;

// meta[b][blk] = {kv_lo, kv_end, q_end, canonical}
//   forward / dQ : q-block `blk` visits kv blocks [kv_lo, kv_end)   (kv_end == 0 -> every row is padding)
//   dK/dV        : kv-block `blk` is visited by q blocks [blk, q_end) (q_end == 0 -> no query attends here)
//   canonical    : 1 iff the row's ids are non-decreasing runs followed only by zeros (TouchNet's layout,
//                  touchnet/models/llama/processing_llama.py:37-40); otherwise ranges are conservative (everything
//                  causal) and every block is masked element-wise by doc-id compare, which is exact for any ids.
struct AttnMeta {
  int32_t kv_lo, kv_end, q_end, canonical;
};

__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm volatile("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// per-position document extent: keys/queries of position t's document live in [start, end)  (start > t for padding)
struct AttnSeg {
  int32_t start, end;
};

// layout of the int32 "meta" buffer built by tn_attn_prep (all offsets in int32 units)
__host__ __device__ inline int64_t attn_meta_flags_off(int B, int nblk) { return int64_t(B) * nblk * 4; }
__host__ __device__ inline int64_t attn_meta_seg_off(int B, int nblk) {
  return (attn_meta_flags_off(B, nblk) + B + 3) / 4 * 4;
}
// cost-ordered work lists of the persistent kernels (entries b*nblk + blk, heaviest first):
//   order_q  : q blocks by kv_end - kv_lo      (forward, dQ)
//   order_kv : kv blocks by q_end - blk        (dK/dV)
__host__ __device__ inline int64_t attn_meta_order_off(int B, int nblk) {
  return attn_meta_seg_off(B, nblk) + int64_t(B) * nblk * ATT_BLK * 2;
}
__host__ __device__ inline int64_t attn_meta_order_kv_off(int B, int nblk) {
  return attn_meta_order_off(B, nblk) + int64_t(B) * nblk;
}
__host__ __device__ inline int64_t attn_meta_total(int B, int nblk) {
  return attn_meta_order_kv_off(B, nblk) + int64_t(B) * nblk;
}

constexpr int ATT_SUB = 64;   // rows streamed per iteration: kv rows (forward, dQ) or q rows (dK/dV)

// [rows x 128] bf16 tile in shared memory: 256 B per row, 16-byte chunk `ch` of row r stored at chunk ch ^ (r & 7), so
// that the eight row addresses of every ldmatrix phase hit distinct banks
__device__ __forceinline__ uint32_t tile_off(int r, int ch) { return uint32_t(r) * 256u + (uint32_t(ch ^ (r & 7)) << 4); }

// cp.async of rows [row0, row0 + ROWS) of a token-major bf16 tensor (128 columns starting at `base`, token stride `ld`
// elements) into a swizzled tile; rows outside [lo, hi) are zero-filled (rows past a sequence, or cache rows outside
// the written range, which may hold anything: a NaN there times a zero probability would still be NaN).  Without
// LOWER the bound lo is 0 and row0 >= 0, so one unsigned compare does; the decode kernel's K/V loads run measurably
// faster with the two signed compares of LOWER than with a single range compare.
template <int ROWS, int NTHREADS, bool LOWER = false>
__device__ __forceinline__ void load_tile_async(uint32_t dst, const bf16* base, int64_t ld, int row0, int lo, int hi,
                                                int tid) {
#pragma unroll
  for (int i = tid; i < ROWS * 16; i += NTHREADS) {
    const int r = i >> 4, ch = i & 15;
    const bool ok = LOWER ? row0 + r >= lo && row0 + r < hi : uint32_t(row0 + r - lo) < uint32_t(hi - lo);
    const bf16* src = base + (ok ? int64_t(row0 + r) * ld : 0) + ch * 8;
    cp_async16(dst + tile_off(r, ch), src, ok ? 16u : 0u);
  }
}

// A fragment (16 x 16, rows r0.., columns 16*kk..) of a swizzled tile for mma.m16n8k16
__device__ __forceinline__ void ldsm_a(uint32_t tile, int r0, int kk, uint32_t (&a)[4]) {
  const int lane = int(threadIdx.x & 31);
  ldsm_x4(tile + tile_off(r0 + (lane & 15), 2 * kk + (lane >> 4)), a[0], a[1], a[2], a[3]);
}
// B fragments of two adjacent n8 tiles when the tile stores B as [n][k] (rows n0.., columns 16*kk..)
__device__ __forceinline__ void ldsm_b_nk(uint32_t tile, int n0, int kk, uint32_t (&b)[4]) {
  const int lane = int(threadIdx.x & 31);
  ldsm_x4(tile + tile_off(n0 + (lane & 7) + ((lane >> 4) << 3), 2 * kk + ((lane >> 3) & 1)), b[0], b[1], b[2], b[3]);
}
// B fragments of two adjacent n8 tiles (columns 16*np..) when the tile stores B as [k][n] (rows k0..k0+15)
__device__ __forceinline__ void ldsm_b_kn(uint32_t tile, int k0, int np, uint32_t (&b)[4]) {
  const int lane = int(threadIdx.x & 31);
  ldsm_x4_t(tile + tile_off(k0 + (lane & 7) + (((lane >> 3) & 1) << 3), 2 * np + (lane >> 4)), b[0], b[1], b[2], b[3]);
}

__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// ---------------------------------------------------------------------------------------------------------------
// Fragment MMA loops.  A warp owns 16 rows; its accumulators follow the mma.m16n8k16 C layout: tile j holds columns
// 8j.., elements 0-1 on row lane/4 and 2-3 on row lane/4 + 8, columns 2*(lane&3) + (e&1).
// ---------------------------------------------------------------------------------------------------------------
// A fragments of a 16 x 16 block of bf16 P / dS values held as two adjacent n8 accumulator tiles
__device__ __forceinline__ void acc_to_a(const float (&x0)[4], const float (&x1)[4], uint32_t (&a)[4]) {
  a[0] = pack_bf16x2(x0[0], x0[1]); a[1] = pack_bf16x2(x0[2], x0[3]);
  a[2] = pack_bf16x2(x1[0], x1[1]); a[3] = pack_bf16x2(x1[2], x1[3]);
}

// A operand of a score product: rows r0.. of a resident swizzled tile, loaded at each k-step ...
struct TileRows {
  uint32_t tile;
  int r0;
};
__device__ __forceinline__ void a_frag(TileRows t, int kk, uint32_t (&a)[4]) { ldsm_a(t.tile, t.r0, kk, a); }
// ... or fragments already held in registers
__device__ __forceinline__ void a_frag(const uint32_t (&f)[8][4], int kk, uint32_t (&a)[4]) {
  a[0] = f[kk][0]; a[1] = f[kk][1]; a[2] = f[kk][2]; a[3] = f[kk][3];
}

// s = A(16 x 128) . B^T over the head dimension, B tile stored [n][k] (rows n0 .. n0 + 16*NP): S = Q.K^T, dP = dO.V^T,
// S^T = K.Q^T, dP^T = V.dO^T
template <int NP, class A>
__device__ __forceinline__ void mma_scores_nk(float (&s)[2 * NP][4], const A& a_src, uint32_t tile, int n0) {
#pragma unroll
  for (int j = 0; j < 2 * NP; ++j) s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
#pragma unroll
  for (int kk = 0; kk < 8; ++kk) {
    uint32_t a[4];
    a_frag(a_src, kk, a);
#pragma unroll
    for (int np = 0; np < NP; ++np) {
      uint32_t bf[4];
      ldsm_b_nk(tile, n0 + np * 16, kk, bf);
      mma_bf16_16816(s[2 * np], a, bf[0], bf[1]);
      mma_bf16_16816(s[2 * np + 1], a, bf[2], bf[3]);
    }
  }
}

// acc(16 x 128) += P(16 x 8*NT) . B, P the score accumulators, B tile stored [k][n] (rows k0 .. k0 + 8*NT):
// O += P.V, dV += P^T.dO, dK += dS^T.Q, dQ += dS.K
template <int NT>
__device__ __forceinline__ void mma_acc_kn(float (&acc)[16][4], const float (&p)[NT][4], uint32_t tile, int k0) {
#pragma unroll
  for (int kk = 0; kk < NT / 2; ++kk) {
    uint32_t a[4];
    acc_to_a(p[2 * kk], p[2 * kk + 1], a);
#pragma unroll
    for (int np = 0; np < 8; ++np) {
      uint32_t bf[4];
      ldsm_b_kn(tile, k0 + kk * 16, np, bf);
      mma_bf16_16816(acc[2 * np], a, bf[0], bf[1]);
      mma_bf16_16816(acc[2 * np + 1], a, bf[2], bf[3]);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Document mask: key k is visible from query q iff k <= q and both lie in the same document (id > 0; 0 is padding)
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool doc_visible(int q, int32_t doc_q, int k, int32_t doc_k) {
  return k <= q && doc_k == doc_q && doc_q > 0;
}
// Score element e of accumulator tile j of a sub-block, scaled to the log2 domain: x * scale_log2, or -inf where
// masked (unless `full`).  The warp's rows are queries (KEY_ROWS false: columns are keys) or keys (KEY_ROWS true:
// columns are queries); this thread's rows are row_a, row_a + 8 with ids doc_a, doc_b, and column c is position
// col0 + c with id col_doc[c].  Applied element by element inside each kernel's softmax loop, so that the compiler
// can split that whole loop on `full`.
// `full` (canonical ids only: every key of the sub-block lies before its first query, and its first key and last query
// are in one document) is written out at each call site: computed by a helper function, it no longer splits the loop
// and the forward kernel runs measurably slower.
template <bool KEY_ROWS>
struct DocMask {
  float scale_log2;
  bool full;
  int row_a;
  int32_t doc_a, doc_b;
  int col0;
  const int32_t* col_doc;
  __device__ __forceinline__ float operator()(float s, int j, int e) const {
    float x = s * scale_log2;
    if (!full) {
      const int c = 8 * j + 2 * int(threadIdx.x & 3) + (e & 1);
      const int row = e < 2 ? row_a : row_a + 8;
      const int32_t dr = e < 2 ? doc_a : doc_b;
      const bool ok = KEY_ROWS ? doc_visible(col0 + c, col_doc[c], row, dr) : doc_visible(row, dr, col0 + c, col_doc[c]);
      x = ok ? x : -INFINITY;
    }
    return x;
  }
};

// ---------------------------------------------------------------------------------------------------------------
// Online softmax (forward and decode), log2 domain: m_* running max, l_* running sum of this thread's rows a, b
// ---------------------------------------------------------------------------------------------------------------
// one step over raw scores s: s <- mask(s, j, e) (scaled, -inf where masked), new running max, rescale of o and l,
// s <- exp2(s - max)
template <int NT, class Mask>
__device__ __forceinline__ void softmax_step(float (&s)[NT][4], const Mask& mask, float (&o)[16][4], float& m_a,
                                             float& m_b, float& l_a, float& l_b) {
  float mx_a = -INFINITY, mx_b = -INFINITY;
#pragma unroll
  for (int j = 0; j < NT; ++j) {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float x = mask(s[j][e], j, e);
      s[j][e] = x;
      if (e < 2) mx_a = fmaxf(mx_a, x); else mx_b = fmaxf(mx_b, x);
    }
  }
  mx_a = quad_max(mx_a); mx_b = quad_max(mx_b);
  const float mn_a = fmaxf(m_a, mx_a), mn_b = fmaxf(m_b, mx_b);
  const float mu_a = mn_a == -INFINITY ? 0.f : mn_a, mu_b = mn_b == -INFINITY ? 0.f : mn_b;
  const float al_a = fast_exp2(m_a - mu_a), al_b = fast_exp2(m_b - mu_b);
  m_a = mn_a; m_b = mn_b;
  l_a *= al_a; l_b *= al_b;
#pragma unroll
  for (int j = 0; j < 16; ++j) { o[j][0] *= al_a; o[j][1] *= al_a; o[j][2] *= al_b; o[j][3] *= al_b; }
#pragma unroll
  for (int j = 0; j < NT; ++j) {
    s[j][0] = fast_exp2(s[j][0] - mu_a); s[j][1] = fast_exp2(s[j][1] - mu_a);
    s[j][2] = fast_exp2(s[j][2] - mu_b); s[j][3] = fast_exp2(s[j][3] - mu_b);
    l_a += s[j][0] + s[j][1];
    l_b += s[j][2] + s[j][3];
  }
}
// natural-log lse from the log2-domain max and the sum; +inf for a row that attends to nothing (its O is exactly 0)
__device__ __forceinline__ float softmax_lse(float m, float l) { return l > 0.f ? (m + __log2f(l)) * LN2 : INFINITY; }

// ---------------------------------------------------------------------------------------------------------------
// Work items and epilogues
// ---------------------------------------------------------------------------------------------------------------
// (block, head, batch row) of this CTA: entry blockIdx.x / nh of the cost-ordered list `order` (heads innermost), or
// the (block, head, batch) grid when `order` is NULL
__device__ __forceinline__ void attn_work_item(const int32_t* order, int nh, int nblk, int& blk, int& h, int& b) {
  if (order) {
    const int e = order[blockIdx.x / nh];
    h = int(blockIdx.x % nh); b = e / nblk; blk = e % nblk;
  } else {
    blk = blockIdx.x; h = blockIdx.y; b = blockIdx.z;
  }
}

// rows [row0, row0 + 128) of `out` (those below `nrows`) = 0: the output of a block no query / key reaches
template <int NTHREADS>
__device__ __forceinline__ void zero_rows(bf16* out, int64_t ld, int row0, int nrows, int tid) {
  for (int i = tid; i < ATT_BLK * 16; i += NTHREADS) {
    const int r = row0 + (i >> 4);
    if (r < nrows) *reinterpret_cast<uint4*>(out + int64_t(r) * ld + (i & 15) * 8) = make_uint4(0, 0, 0, 0);
  }
}

// 16 rows x 128 columns of one warp's accumulator (rows row_a and row_a + 8 of the output, `nrows` valid) -> bf16, times
// `mul`; with rope_cos the inverse rotation  dx_lo = g_lo*cos + g_hi*sin,  dx_hi = g_hi*cos - g_lo*sin  is applied
// (pairs (j, j+64) sit in accumulator tiles j and j+8 of the thread; tables indexed by trow_a / trow_a + 8)
__device__ __forceinline__ void store_acc_rows(bf16* out, int64_t ld, int row_a, int nrows, const float (&acc)[16][4],
                                               float mul, const bf16* rope_cos, const bf16* rope_sin, int64_t trow_a) {
  const int cq = 2 * int(threadIdx.x & 3);
  if (rope_cos == nullptr) {
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      if (row_a < nrows)
        *reinterpret_cast<uint32_t*>(out + int64_t(row_a) * ld + 8 * j + cq) = pack_bf16x2(acc[j][0] * mul, acc[j][1] * mul);
      if (row_a + 8 < nrows)
        *reinterpret_cast<uint32_t*>(out + int64_t(row_a + 8) * ld + 8 * j + cq) = pack_bf16x2(acc[j][2] * mul, acc[j][3] * mul);
    }
    return;
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = row_a + 8 * h;
    if (row >= nrows) continue;
    bf16* o = out + int64_t(row) * ld;
    const int64_t tr = (trow_a + 8 * h) * 64;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int c = 8 * j + cq;
      const uint32_t cw = *reinterpret_cast<const uint32_t*>(rope_cos + tr + c);
      const uint32_t sw = *reinterpret_cast<const uint32_t*>(rope_sin + tr + c);
      float lo[2], hi[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const float gl = acc[j][2 * h + e] * mul, gh = acc[j + 8][2 * h + e] * mul;
        const float cs = e ? bf16hi(cw) : bf16lo(cw), sn = e ? bf16hi(sw) : bf16lo(sw);
        lo[e] = fmaf(gl, cs, gh * sn);
        hi[e] = fmaf(gh, cs, -gl * sn);
      }
      *reinterpret_cast<uint32_t*>(o + c) = pack_bf16x2(lo[0], lo[1]);
      *reinterpret_cast<uint32_t*>(o + c + 64) = pack_bf16x2(hi[0], hi[1]);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Host side
// ---------------------------------------------------------------------------------------------------------------
// Query window of a forward / backward call: the Q-side tensors hold rows [q_blk_off*128, q_blk_off*128 + Tq) of the
// sequence of length T (context parallelism); Tq <= 0 selects the whole sequence.  False when the window leaves it.
inline bool attn_query_window(int T, int& Tq, int& q_blk_off) {
  if (Tq <= 0) { Tq = T; q_blk_off = 0; }
  const int nblk = (T + ATT_BLK - 1) / ATT_BLK;
  return q_blk_off >= 0 && q_blk_off * ATT_BLK + Tq <= nblk * ATT_BLK;
}
// Grid over nb blocks x nh heads x B rows.  Over the whole sequence a 1-D grid walks the cost-ordered list `list`, so
// the last wave is made of the cheapest items; a context-parallel window uses the (block, head, batch) grid and sets
// `order` to NULL.
inline dim3 attn_grid(int T, int Tq, int q_blk_off, const int32_t* list, int nb, int nh, int B, const int32_t*& order) {
  const bool ordered = Tq == T && q_blk_off == 0;
  order = ordered ? list : nullptr;
  return ordered ? dim3(unsigned(nb) * nh * B) : dim3(nb, nh, B);
}
// Opt kernel K in to `bytes` of dynamic shared memory, once per process
template <auto K>
inline cudaError_t attn_smem_optin(int bytes) {
  static const cudaError_t err = cudaFuncSetAttribute(K, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  return err;
}

}  // namespace tn
