// touchnet_b200 :: packed-sequence ("document") causal attention, forward.  head_dim 128, bf16, GQA.
//
// Replaces torch.nn.attention.flex_attention + make_flex_block_causal_mask as reached from
//   hf:integrations/flex_attention.py:136-247, :262-364  (selected by `"attn_implementation": "flex_attention"`,
//   examples/text/pretrain/fineweb-edu/config/Llama-3_2-1B.json:7; touchnet/bin/train.py:129-131)
// mask  allow[b,q,k] = (q >= k) && doc[b,q] == doc[b,k] && doc[b,q] > 0
//
// One CTA = one 128-row q block of one head, 8 warps of 16 query rows each.  Q stays resident in shared memory (its
// fragments in registers); K / V stream through a double-buffered cp.async ring in 64-row sub-blocks.  Per sub-block
// every warp computes S = Q.K^T and O += P.V with mma.sync m16n8k16 (bf16 in, fp32 accumulate in registers) and keeps
// an online softmax in the log2 domain; P goes from the S accumulators straight into A fragments (no shared memory).
// kv blocks outside the [kv_lo, kv_end) range of the q block are never touched (block-level document skipping); sub-
// blocks wholly inside one document below the diagonal skip the mask arithmetic.
#include "../../include/touchnet_b200.h"
#include "attn_common.cuh"
#include "host.h"

#include <stdlib.h>

namespace tn {

// ---------------------------------------------------------------------------------------------------------------
// prep: canonical flag per batch row, then per-block ranges
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) attn_canonical_kernel(const int32_t* __restrict__ doc, int32_t* __restrict__ flags,
                                                              int T) {
  const int b = blockIdx.x;
  const int32_t* d = doc + int64_t(b) * T;
  int bad = 0;
  for (int t = threadIdx.x + 1; t < T; t += blockDim.x) {
    const int32_t cur = d[t], prev = d[t - 1];
    if (cur != 0 && (prev == 0 || cur < prev)) bad = 1;
    if (cur < 0) bad = 1;
  }
  if (threadIdx.x == 0 && T > 0 && d[0] < 0) bad = 1;
  bad = __syncthreads_or(bad);
  if (threadIdx.x == 0) flags[b] = bad ? 0 : 1;
}

// one warp per (b, block)
__global__ void __launch_bounds__(256) attn_meta_kernel(const int32_t* __restrict__ doc, const int32_t* __restrict__ flags,
                                                        AttnMeta* __restrict__ meta, AttnSeg* __restrict__ seg, int B,
                                                        int T, int nblk) {
  const int gw = blockIdx.x * 8 + warp_id();
  if (gw >= B * nblk) return;
  const int b = gw / nblk, blk = gw - b * nblk;
  const uint32_t lane = lane_id();
  const int32_t* d = doc + int64_t(b) * T;
  const int t0 = blk * ATT_BLK;
  const int canonical = flags[b];
  // the 128 ids of this block: lane holds positions t0 + lane + 32*i
  int32_t ids[4];
  uint32_t valid_mask[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int t = t0 + int(lane) + 32 * i;
    ids[i] = (t < T) ? d[t] : 0;
    valid_mask[i] = __ballot_sync(0xffffffffu, ids[i] > 0);
  }
  int first = -1, last = -1;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    if (valid_mask[i]) {
      if (first < 0) first = 32 * i + __ffs(valid_mask[i]) - 1;
      last = 32 * i + 31 - __clz(valid_mask[i]);
    }
  }
  AttnMeta m;
  m.canonical = canonical;
  AttnSeg* segb = seg + (int64_t(b) * nblk + blk) * ATT_BLK;
  if (first < 0 || !canonical) {
    // padding-only block, or ids that are not non-decreasing runs: segments are empty / unused (the kernels mask
    // non-canonical rows element-wise by document id over the whole causal range)
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int t = t0 + int(lane) + 32 * i;
      segb[lane + 32 * i] = AttnSeg{t + 1, t};
    }
    if (first < 0) { m.kv_lo = 0; m.kv_end = 0; m.q_end = 0; }
    else { m.kv_lo = 0; m.kv_end = blk + 1; m.q_end = nblk; }
    if (lane == 0) meta[gw] = m;
    return;
  }
  // ---- backward scan: start of the run containing the first valid row ----
  const int32_t d_first = __shfl_sync(0xffffffffu, ids[first >> 5], first & 31);
  int run_start = t0 + first;
  {
    // inside the block
    bool done = false;
    for (int t = t0 + first - 1; t >= t0 && !done; --t) {  // <= 127 steps, warp-uniform
      const int32_t v = __shfl_sync(0xffffffffu, ids[(t - t0) >> 5], (t - t0) & 31);
      if (v == d_first) run_start = t; else done = true;
    }
    if (!done) {
      int base = t0 - 128;  // earlier blocks, 128 ids per step
      while (base >= 0 && !done) {
        int32_t v[4];
        uint32_t eq[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          v[i] = d[base + int(lane) + 32 * i];
          eq[i] = __ballot_sync(0xffffffffu, v[i] == d_first);
        }
        // canonical => matching ids form a suffix of this window
#pragma unroll
        for (int i = 3; i >= 0; --i) {
          if (done) break;
          if (eq[i] == 0xffffffffu) { run_start = base + 32 * i; }
          else {
            if (eq[i]) run_start = base + 32 * i + (32 - __clz(~eq[i]));
            done = true;
          }
        }
        base -= 128;
      }
    }
  }
  m.kv_lo = run_start / ATT_BLK;
  m.kv_end = blk + 1;
  // ---- forward scan: end (exclusive) of the run containing the last valid column ----
  const int32_t d_last = __shfl_sync(0xffffffffu, ids[last >> 5], last & 31);
  int run_end = t0 + last + 1;
  if (last == ATT_BLK - 1) {
    bool done = false;
    int base = t0 + 128;
    while (base < T && !done) {
      uint32_t eq[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int t = base + int(lane) + 32 * i;
        const int32_t v = (t < T) ? d[t] : 0;
        eq[i] = __ballot_sync(0xffffffffu, v == d_last);
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        if (done) break;
        if (eq[i] == 0xffffffffu) { run_end = base + 32 * i + 32; }
        else {
          if (eq[i]) run_end = base + 32 * i + (__ffs(~eq[i]) - 1);
          done = true;
        }
      }
      base += 128;
    }
  }
  m.q_end = (run_end - 1) / ATT_BLK + 1;
  if (lane == 0) meta[gw] = m;

  // ---- per-position document extents [start, end) ----
  // a run starts at p if p == 0 of the block or id[p] != id[p-1]; it ends after p if id[p+1] != id[p]
  uint32_t sb[4], eb[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int pos = int(lane) + 32 * i;
    const int32_t prev = __shfl_up_sync(0xffffffffu, ids[i], 1);
    const int32_t prev_w = __shfl_sync(0xffffffffu, ids[i > 0 ? i - 1 : 0], 31);
    const int32_t next = __shfl_down_sync(0xffffffffu, ids[i], 1);
    const int32_t next_w = __shfl_sync(0xffffffffu, ids[i < 3 ? i + 1 : 3], 0);
    const int32_t pv = lane > 0 ? prev : (i > 0 ? prev_w : ids[i] /* block edge: resolved by run_start */);
    const int32_t nx = lane < 31 ? next : (i < 3 ? next_w : ids[i] /* block edge: resolved by run_end */);
    sb[i] = __ballot_sync(0xffffffffu, pos > 0 && pv != ids[i]);
    eb[i] = __ballot_sync(0xffffffffu, pos < ATT_BLK - 1 && nx != ids[i]);
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int pos = int(lane) + 32 * i;
    const int t = t0 + pos;
    AttnSeg sg;
    if (ids[i] <= 0) { sg.start = t + 1; sg.end = t; }
    else {
      // last run boundary at or before pos
      int st = -1;
      {
        const uint32_t mcur = sb[i] & (0xffffffffu >> (31 - lane));
        if (mcur) st = 32 * i + 31 - __clz(mcur);
        else {
#pragma unroll
          for (int w = 3; w >= 0; --w)
            if (w < i && st < 0 && sb[w]) st = 32 * w + 31 - __clz(sb[w]);
        }
      }
      sg.start = st >= 0 ? t0 + st : run_start;       // no boundary inside the block: the run began earlier
      int en = -1;
      {
        const uint32_t mcur = eb[i] & (0xffffffffu << lane);
        if (mcur) en = 32 * i + __ffs(mcur) - 1;
        else {
#pragma unroll
          for (int w = 0; w < 4; ++w)
            if (w > i && en < 0 && eb[w]) en = 32 * w + __ffs(eb[w]) - 1;
        }
      }
      sg.end = en >= 0 ? t0 + en + 1 : run_end;        // the run continues past the block (or ends at its last valid id)
    }
    segb[pos] = sg;
  }
}

// cost-ordered work lists (one CTA; N = B*nblk entries, rank by counting: O(N^2 / 1024) compares per thread, once per step)
__global__ void __launch_bounds__(1024) attn_order_kernel(const AttnMeta* __restrict__ meta, int32_t* __restrict__ order_q,
                                                          int32_t* __restrict__ order_kv, int N, int nblk) {
  for (int i = threadIdx.x; i < N; i += blockDim.x) {
    const AttnMeta m = meta[i];
    const int blk = i % nblk;
    const int cq = m.kv_end - m.kv_lo;
    const int ckv = m.q_end > blk ? m.q_end - blk : 0;
    int rq = 0, rkv = 0;
    for (int t = 0; t < N; ++t) {
      const AttnMeta o = meta[t];
      const int oq = o.kv_end - o.kv_lo;
      const int ob = t % nblk;
      const int okv = o.q_end > ob ? o.q_end - ob : 0;
      rq += (oq > cq) || (oq == cq && t < i);
      rkv += (okv > ckv) || (okv == ckv && t < i);
    }
    order_q[rq] = i;
    order_kv[rkv] = i;
  }
}


// ---------------------------------------------------------------------------------------------------------------
// forward kernel
// ---------------------------------------------------------------------------------------------------------------
constexpr int FWD_THREADS = 256;
constexpr int SUB_TILE = ATT_SUB * ATT_HD * 2;   // 16 KB

struct FwdSmem {
  static constexpr int Q = 0;                          // 128 x 128 bf16
  static constexpr int K = Q + ATT_BLK * ATT_HD * 2;   // 2 stages
  static constexpr int V = K + 2 * SUB_TILE;           // 2 stages
  static constexpr int DOC = V + 2 * SUB_TILE;         // 2 x 64 int32
  static constexpr int TOTAL = DOC + 2 * ATT_SUB * 4;
};

struct AttnFwdParams {
  const bf16* Q;
  const bf16* K;
  const bf16* V;
  bf16* O;
  int64_t ldq, ldk, ldv, ldo;
  float* lse;
  const int32_t* doc;
  const AttnMeta* meta;
  const int32_t* order;   // cost-ordered q blocks (tn_attn_prep) for a 1-D grid, heaviest first; NULL = 3-D grid
  int B, T, H, KV, nblk;
  int Tq, q_blk_off;  // context parallelism: the Q/O/lse tensors hold rows [q_blk_off*128, q_blk_off*128 + Tq) of the
                      // global sequence of length T; K/V/doc/meta are global.  Tq == T, off == 0 without CP.
  float scale_log2;   // softmax scale * log2(e)
};

__global__ void __launch_bounds__(FWD_THREADS, 1) attn_fwd_kernel(const AttnFwdParams p) {
  extern __shared__ __align__(128) uint8_t smem[];
  const uint32_t sb = smem_u32(smem);
  int32_t* sDoc = reinterpret_cast<int32_t*>(smem + FwdSmem::DOC);
  int qb, h, b;
  attn_work_item(p.order, p.H, p.nblk, qb, h, b);
  const int gblk = qb + p.q_blk_off;
  const AttnMeta meta = p.meta[b * p.nblk + gblk];
  const int tid = int(threadIdx.x), warp = tid >> 5, lane = tid & 31;
  const int q0 = gblk * ATT_BLK, lrow0 = qb * ATT_BLK;
  const int kvh = h / (p.H / p.KV);
  const int32_t* docb = p.doc + int64_t(b) * p.T;
  bf16* Ob = p.O + int64_t(b) * p.Tq * p.ldo + h * ATT_HD;
  float* lseb = p.lse + (int64_t(b) * p.H + h) * p.Tq;
  const int nsub = meta.kv_end > meta.kv_lo ? (meta.kv_end - meta.kv_lo) * (ATT_BLK / ATT_SUB) : 0;
  if (nsub == 0) {   // padding-only block: O = 0, lse = +inf
    zero_rows<FWD_THREADS>(Ob, p.ldo, lrow0, p.Tq, tid);
    for (int i = tid; i < ATT_BLK; i += FWD_THREADS)
      if (lrow0 + i < p.Tq) lseb[lrow0 + i] = INFINITY;
    return;
  }

  const bf16* Kb = p.K + int64_t(b) * p.T * p.ldk + kvh * ATT_HD;
  const bf16* Vb = p.V + int64_t(b) * p.T * p.ldv + kvh * ATT_HD;
  const int kbase = meta.kv_lo * ATT_BLK;
  load_tile_async<ATT_BLK, FWD_THREADS>(sb + FwdSmem::Q, p.Q + int64_t(b) * p.Tq * p.ldq + h * ATT_HD, p.ldq, lrow0, 0,
                                        p.Tq, tid);
  auto load_kv = [&](int i, int buf) {
    const int k0 = kbase + i * ATT_SUB;
    load_tile_async<ATT_SUB, FWD_THREADS>(sb + FwdSmem::K + buf * SUB_TILE, Kb, p.ldk, k0, 0, p.T, tid);
    load_tile_async<ATT_SUB, FWD_THREADS>(sb + FwdSmem::V + buf * SUB_TILE, Vb, p.ldv, k0, 0, p.T, tid);
    if (tid < ATT_SUB) sDoc[buf * ATT_SUB + tid] = (k0 + tid < p.T) ? docb[k0 + tid] : 0;
    cp_async_commit();
  };
  load_kv(0, 0);

  // this thread's two rows (global positions) and their document ids
  const int ra = warp * 16 + (lane >> 2);
  const int qa = q0 + ra, qb8 = qa + 8;
  const int32_t da = qa < p.T ? docb[qa] : 0, db = qb8 < p.T ? docb[qb8] : 0;
  const int32_t d_last = (q0 + ATT_BLK - 1 < p.T) ? docb[q0 + ATT_BLK - 1] : 0;

  float o[16][4];
#pragma unroll
  for (int i = 0; i < 16; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
  float m_a = -INFINITY, m_b = -INFINITY, l_a = 0.f, l_b = 0.f;
  uint32_t qf[8][4];

  for (int i = 0; i < nsub; ++i) {
    const int buf = i & 1;
    if (i + 1 < nsub) { load_kv(i + 1, buf ^ 1); cp_async_wait<1>(); }
    else cp_async_wait<0>();
    __syncthreads();
    if (i == 0) {
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) ldsm_a(sb + FwdSmem::Q, warp * 16, kk, qf[kk]);
    }
    const uint32_t sK = sb + FwdSmem::K + buf * SUB_TILE, sV = sb + FwdSmem::V + buf * SUB_TILE;
    const int32_t* dk = sDoc + buf * ATT_SUB;
    const int k0 = kbase + i * ATT_SUB;

    float s[8][4];
    mma_scores_nk<4>(s, qf, sK, 0);
    // canonical ids: keys all before the block's first query and in the document of its last query -> no mask
    const bool full = meta.canonical && (k0 + ATT_SUB <= q0) && d_last > 0 && dk[0] == d_last;
    softmax_step(s, DocMask<false>{p.scale_log2, full, qa, da, db, k0, dk}, o, m_a, m_b, l_a, l_b);
    mma_acc_kn(o, s, sV, 0);
    __syncthreads();   // buffer `buf` is refilled by the next iteration's prefetch
  }

  // ---- O / l -> global, lse ----
  // (written out rather than through store_acc_rows: with that helper the kernel compiles to a main loop that ran
  // about 2 % slower at T = 32768 on an H100 80GB HBM3 at 700 W)
  l_a = quad_sum(l_a); l_b = quad_sum(l_b);
  const float inv_a = l_a > 0.f ? 1.f / l_a : 0.f, inv_b = l_b > 0.f ? 1.f / l_b : 0.f;
  const int la = lrow0 + ra, lb = la + 8, cq = 2 * (lane & 3);
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const int col = 8 * j + cq;
    if (la < p.Tq) *reinterpret_cast<uint32_t*>(Ob + int64_t(la) * p.ldo + col) = pack_bf16x2(o[j][0] * inv_a, o[j][1] * inv_a);
    if (lb < p.Tq) *reinterpret_cast<uint32_t*>(Ob + int64_t(lb) * p.ldo + col) = pack_bf16x2(o[j][2] * inv_b, o[j][3] * inv_b);
  }
  if ((lane & 3) == 0) {
    if (la < p.Tq) lseb[la] = softmax_lse(m_a, l_a);
    if (lb < p.Tq) lseb[lb] = softmax_lse(m_b, l_b);
  }
}

}  // namespace tn

using namespace tn;

extern "C" int64_t tn_attn_meta_ints(int B, int T) {
  return attn_meta_total(B, (T + ATT_BLK - 1) / ATT_BLK);
}

extern "C" int tn_attn_prep(const int32_t* doc_ids, int32_t* meta, int B, int T, tn_stream_t stream_) {
  clear_error();
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  TN_REQUIRE(doc_ids && meta, "tn_attn_prep: null pointer");
  TN_REQUIRE(B > 0 && T > 0, "tn_attn_prep: empty batch");
  const int nblk = (T + ATT_BLK - 1) / ATT_BLK;
  int32_t* flags = meta + attn_meta_flags_off(B, nblk);
  AttnSeg* seg = reinterpret_cast<AttnSeg*>(meta + attn_meta_seg_off(B, nblk));
  attn_canonical_kernel<<<B, 1024, 0, stream>>>(doc_ids, flags, T);
  TN_CHECK_CUDA(cudaGetLastError());
  const int warps = B * nblk;
  attn_meta_kernel<<<(warps + 7) / 8, 256, 0, stream>>>(doc_ids, flags, reinterpret_cast<AttnMeta*>(meta), seg, B, T, nblk);
  TN_CHECK_CUDA(cudaGetLastError());
  attn_order_kernel<<<1, 1024, 0, stream>>>(reinterpret_cast<const AttnMeta*>(meta), meta + attn_meta_order_off(B, nblk),
                                            meta + attn_meta_order_kv_off(B, nblk), B * nblk, nblk);
  TN_CHECK_CUDA(cudaGetLastError());
  return TN_OK;
}

extern "C" int tn_attn_fwd_bf16(const void* Q, int64_t ldq, const void* K, int64_t ldk, const void* V, int64_t ldv,
                                void* O, int64_t ldo, float* lse, const int32_t* doc_ids, const int32_t* meta, int B,
                                int T, int H, int KV, float scale, int Tq, int q_blk_off, tn_stream_t stream_) {
  clear_error();
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  TN_REQUIRE(Q && K && V && O && lse && doc_ids && meta, "tn_attn_fwd_bf16: null pointer");
  TN_REQUIRE(B > 0 && T > 0 && H > 0 && KV > 0 && H % KV == 0, "tn_attn_fwd_bf16: bad dims B=%d T=%d H=%d KV=%d", B, T, H, KV);
  TN_REQUIRE(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 8 == 0, "tn_attn_fwd_bf16: strides must be multiples of 8");
  TN_REQUIRE(ldq >= int64_t(H) * ATT_HD && ldo >= int64_t(H) * ATT_HD && ldk >= int64_t(KV) * ATT_HD &&
                 ldv >= int64_t(KV) * ATT_HD, "tn_attn_fwd_bf16: token stride smaller than heads*128");
  TN_REQUIRE(attn_query_window(T, Tq, q_blk_off), "tn_attn_fwd_bf16: query window outside the sequence");
  const int nblk = (T + ATT_BLK - 1) / ATT_BLK, nqb = (Tq + ATT_BLK - 1) / ATT_BLK;
  AttnFwdParams p{};
  p.Q = static_cast<const bf16*>(Q); p.K = static_cast<const bf16*>(K); p.V = static_cast<const bf16*>(V);
  p.O = static_cast<bf16*>(O);
  p.ldq = ldq; p.ldk = ldk; p.ldv = ldv; p.ldo = ldo;
  p.lse = lse; p.doc = doc_ids; p.meta = reinterpret_cast<const AttnMeta*>(meta);
  p.B = B; p.T = T; p.H = H; p.KV = KV; p.nblk = nblk;
  p.Tq = Tq; p.q_blk_off = q_blk_off;
  p.scale_log2 = scale * LOG2E;
  const dim3 grid = attn_grid(T, Tq, q_blk_off, meta + attn_meta_order_off(B, nblk), nqb, H, B, p.order);
  TN_CHECK_CUDA(attn_smem_optin<attn_fwd_kernel>(FwdSmem::TOTAL));
  attn_fwd_kernel<<<grid, FWD_THREADS, FwdSmem::TOTAL, stream>>>(p);
  TN_CHECK_CUDA(cudaGetLastError());
  return TN_OK;
}
