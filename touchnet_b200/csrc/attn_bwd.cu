// touchnet_b200 :: packed-sequence ("document") causal attention, backward.  head_dim 128, bf16, GQA.
//
// Backward of the FlexAttention call the reference reaches through hf:integrations/flex_attention.py:262-364
// (autograd of torch.nn.attention.flex_attention with the block-causal document mask of :136-247).
//
// Three launches, no atomics, deterministic:
//   attn_delta_kernel   delta[b,h,t] = sum_d O.dO
//   attn_dkdv_kernel    one CTA per (kv block, kv head), walked heaviest first: K and V stay resident in shared memory,
//                       the CTA loops over the q heads of the GQA group and the 64-row q sub-blocks that attend to the
//                       block (cp.async double buffer); S^T = K.Q^T, dP^T = V.dO^T, dV += P^T.dO, dK += dS^T.Q
//   attn_dq_kernel      one CTA per (q block, head): Q and dO resident, K/V streamed; S = Q.K^T, dP = dO.V^T, dQ += dS.K
// 8 warps per CTA, 16 resident rows per warp; every product is an mma.sync m16n8k16 (bf16 in, fp32 accumulate in
// registers) and P / dS go from the score accumulators straight into A fragments.  The mask is the exact document
// compare (q >= k, same id, id > 0); sub-blocks wholly inside one document off the diagonal skip it.
#include "../../include/touchnet_b200.h"
#include "attn_common.cuh"
#include "host.h"

namespace tn {

constexpr int BWD_THREADS = 256;
constexpr int RES_TILE = ATT_BLK * ATT_HD * 2;   // 32 KB resident tile
constexpr int STR_TILE = ATT_SUB * ATT_HD * 2;   // 16 KB streamed tile

struct DkdvSmem {
  static constexpr int K = 0;
  static constexpr int V = K + RES_TILE;
  static constexpr int Q = V + RES_TILE;        // 2 stages
  static constexpr int DO = Q + 2 * STR_TILE;   // 2 stages
  static constexpr int COL = DO + 2 * STR_TILE; // 2 x {lse2[64], delta[64], doc[64]}
  static constexpr int TOTAL = COL + 2 * 3 * ATT_SUB * 4;
};
struct DqSmem {
  static constexpr int Q = 0;
  static constexpr int DO = Q + RES_TILE;
  static constexpr int K = DO + RES_TILE;       // 2 stages
  static constexpr int V = K + 2 * STR_TILE;    // 2 stages
  static constexpr int DOC = V + 2 * STR_TILE;  // 2 x 64 int32
  static constexpr int TOTAL = DOC + 2 * ATT_SUB * 4;
};

struct AttnBwdParams {
  const bf16* Q;
  const bf16* K;
  const bf16* V;
  const bf16* dO;
  int64_t ldq, ldk, ldv, lddo;
  const int32_t* doc;
  const AttnMeta* meta;
  const float* lse;
  const float* delta;
  bf16* out1;   // dKdV: dV ; dQ: dQ
  bf16* out2;   // dKdV: dK
  int64_t ld1, ld2;
  int B, T, H, KV, nblk;
  int Tq, q_blk_off;   // context parallelism: Q/dO/dQ/lse/delta hold rows [q_blk_off*128, +Tq) of the global sequence
  float scale, scale_log2;
  // fused inverse RoPE (backward of hf apply_rotary_pos_emb, modeling_llama.py:151-168) on dQ and dK in the epilogue:
  // cos/sin [rows, 64] bf16 indexed like the output tensor's rows (NULL = gradients w.r.t. the rotated q/k)
  const bf16* rope_cos;
  const bf16* rope_sin;
  // cost-ordered work list (tn_attn_prep: kv blocks by number of attending q blocks for dK/dV, q blocks by number of kv
  // blocks for dQ; entries b*nblk + blk, heaviest first) walked by a 1-D grid, so that the last wave is made of the
  // cheapest items; NULL = (block, head, batch) grid (context-parallel windows)
  const int32_t* order;
};

__global__ void __launch_bounds__(256) attn_delta_kernel(const bf16* __restrict__ O, int64_t ldo,
                                                         const bf16* __restrict__ dO, int64_t lddo,
                                                         float* __restrict__ delta, int B, int T, int H) {
  // half-warp per (b, t, h): 16 lanes x 8 elements
  const int64_t pair = (int64_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 4;
  const int sub = threadIdx.x & 15;
  const int64_t total = int64_t(B) * T * H;
  float acc = 0.f;
  if (pair < total) {
    const int h = int(pair % H);
    const int64_t bt = pair / H;
    const uint4 a = *reinterpret_cast<const uint4*>(O + bt * ldo + int64_t(h) * ATT_HD + sub * 8);
    const uint4 g = *reinterpret_cast<const uint4*>(dO + bt * lddo + int64_t(h) * ATT_HD + sub * 8);
    acc = bf16lo(a.x) * bf16lo(g.x) + bf16hi(a.x) * bf16hi(g.x) + bf16lo(a.y) * bf16lo(g.y) + bf16hi(a.y) * bf16hi(g.y) +
          bf16lo(a.z) * bf16lo(g.z) + bf16hi(a.z) * bf16hi(g.z) + bf16lo(a.w) * bf16lo(g.w) + bf16hi(a.w) * bf16hi(g.w);
  }
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (pair < total && sub == 0) {
    const int h = int(pair % H);
    const int64_t bt = pair / H;
    const int64_t b = bt / T, t = bt - b * T;
    delta[(b * H + h) * T + t] = acc;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// dK / dV
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(BWD_THREADS, 1) attn_dkdv_kernel(const AttnBwdParams p) {
  extern __shared__ __align__(128) uint8_t smem[];
  const uint32_t sb = smem_u32(smem);
  float* sCol = reinterpret_cast<float*>(smem + DkdvSmem::COL);
  int blk, kvh, b;
  attn_work_item(p.order, p.KV, p.nblk, blk, kvh, b);
  const AttnMeta meta = p.meta[b * p.nblk + blk];
  const int tid = int(threadIdx.x), warp = tid >> 5, lane = tid & 31;
  const int k0 = blk * ATT_BLK;
  const int G = p.H / p.KV;
  const int32_t* docb = p.doc + int64_t(b) * p.T;
  bf16* dVb = p.out1 + int64_t(b) * p.T * p.ld1 + kvh * ATT_HD;
  bf16* dKb = p.out2 + int64_t(b) * p.T * p.ld2 + kvh * ATT_HD;
  // local query rows [lq0, lq1) that may attend to this block: q blocks [blk, q_end) inside the query window
  const int qoff = p.q_blk_off * ATT_BLK;
  const int lq0 = max(k0 - qoff, 0);
  const int lq1 = min(meta.q_end * ATT_BLK - qoff, p.Tq);
  const int nsub = lq1 > lq0 ? (lq1 - lq0 + ATT_SUB - 1) / ATT_SUB : 0;
  const int n = G * nsub;
  if (n == 0) {   // no query attends here: dK = dV = 0
    zero_rows<BWD_THREADS>(dVb, p.ld1, k0, p.T, tid);
    zero_rows<BWD_THREADS>(dKb, p.ld2, k0, p.T, tid);
    return;
  }
  load_tile_async<ATT_BLK, BWD_THREADS>(sb + DkdvSmem::K, p.K + int64_t(b) * p.T * p.ldk + kvh * ATT_HD, p.ldk, k0, 0, p.T,
                                        tid);
  load_tile_async<ATT_BLK, BWD_THREADS>(sb + DkdvSmem::V, p.V + int64_t(b) * p.T * p.ldv + kvh * ATT_HD, p.ldv, k0, 0, p.T,
                                        tid);
  auto load_q = [&](int it, int buf) {
    const int h = kvh * G + it / nsub;
    const int r0 = lq0 + (it % nsub) * ATT_SUB;
    load_tile_async<ATT_SUB, BWD_THREADS>(sb + DkdvSmem::Q + buf * STR_TILE, p.Q + int64_t(b) * p.Tq * p.ldq + h * ATT_HD,
                                          p.ldq, r0, 0, p.Tq, tid);
    load_tile_async<ATT_SUB, BWD_THREADS>(sb + DkdvSmem::DO + buf * STR_TILE, p.dO + int64_t(b) * p.Tq * p.lddo + h * ATT_HD,
                                          p.lddo, r0, 0, p.Tq, tid);
    if (tid < ATT_SUB) {
      const int r = r0 + tid;
      const bool ok = r < p.Tq && qoff + r < p.T;
      const int64_t li = (int64_t(b) * p.H + h) * p.Tq + r;
      float* col = sCol + buf * 3 * ATT_SUB;
      col[tid] = ok ? p.lse[li] * LOG2E : INFINITY;    // +inf -> P = 0
      col[ATT_SUB + tid] = ok ? p.delta[li] : 0.f;
      reinterpret_cast<int32_t*>(col)[2 * ATT_SUB + tid] = ok ? docb[qoff + r] : 0;
    }
    cp_async_commit();
  };
  load_q(0, 0);

  const int ka = k0 + warp * 16 + (lane >> 2), kb8 = ka + 8;
  const int32_t da = ka < p.T ? docb[ka] : 0, db = kb8 < p.T ? docb[kb8] : 0;
  const int32_t d_first = docb[k0];
  const int cq = 2 * (lane & 3);
  float dv[16][4], dk[16][4];
#pragma unroll
  for (int j = 0; j < 16; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) { dv[j][e] = 0.f; dk[j][e] = 0.f; }

  for (int it = 0; it < n; ++it) {
    const int buf = it & 1;
    if (it + 1 < n) { load_q(it + 1, buf ^ 1); cp_async_wait<1>(); }
    else cp_async_wait<0>();
    __syncthreads();
    const uint32_t sQ = sb + DkdvSmem::Q + buf * STR_TILE, sDO = sb + DkdvSmem::DO + buf * STR_TILE;
    const float* col = sCol + buf * 3 * ATT_SUB;
    const int32_t* cdoc = reinterpret_cast<const int32_t*>(col) + 2 * ATT_SUB;
    const int gq0 = qoff + lq0 + (it % nsub) * ATT_SUB;   // global position of streamed column 0

    // S^T = K.Q^T (rows = keys, columns = queries)
    float s[8][4];
    mma_scores_nk<4>(s, TileRows{sb + DkdvSmem::K, warp * 16}, sQ, 0);
    // P^T = exp2(S^T * scale_log2 - lse2[q]); masked -> 0
    const bool full = meta.canonical && (k0 + ATT_BLK <= gq0) && d_first > 0 && cdoc[ATT_SUB - 1] == d_first;
    const DocMask<true> mask{p.scale_log2, full, ka, da, db, gq0, cdoc};
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) s[j][e] = fast_exp2(mask(s[j][e], j, e) - col[8 * j + cq + (e & 1)]);
    // dV += P^T.dO
    mma_acc_kn(dv, s, sDO, 0);
    // dP^T = V.dO^T, dS^T = P^T * (dP^T - delta[q])
    float dp[8][4];
    mma_scores_nk<4>(dp, TileRows{sb + DkdvSmem::V, warp * 16}, sDO, 0);
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) dp[j][e] = s[j][e] * (dp[j][e] - col[ATT_SUB + 8 * j + cq + (e & 1)]);
    // dK += dS^T.Q
    mma_acc_kn(dk, dp, sQ, 0);
    __syncthreads();   // buffer `buf` is refilled by the next iteration's prefetch
  }
  // dV unscaled; dK carries the softmax scale (and the inverse RoPE when requested)
  store_acc_rows(dVb, p.ld1, ka, p.T, dv, 1.f, nullptr, nullptr, 0);
  store_acc_rows(dKb, p.ld2, ka, p.T, dk, p.scale, p.rope_cos, p.rope_sin, int64_t(b) * p.T + ka);
}

// ---------------------------------------------------------------------------------------------------------------
// dQ
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(BWD_THREADS, 1) attn_dq_kernel(const AttnBwdParams p) {
  extern __shared__ __align__(128) uint8_t smem[];
  const uint32_t sb = smem_u32(smem);
  int32_t* sDoc = reinterpret_cast<int32_t*>(smem + DqSmem::DOC);
  int qb, h, b;
  attn_work_item(p.order, p.H, p.nblk, qb, h, b);
  const int gblk = qb + p.q_blk_off;
  const AttnMeta meta = p.meta[b * p.nblk + gblk];
  const int tid = int(threadIdx.x), warp = tid >> 5, lane = tid & 31;
  const int q0 = gblk * ATT_BLK, lrow0 = qb * ATT_BLK;
  const int kvh = h / (p.H / p.KV);
  const int32_t* docb = p.doc + int64_t(b) * p.T;
  bf16* dQb = p.out1 + int64_t(b) * p.Tq * p.ld1 + h * ATT_HD;
  const int nsub = meta.kv_end > meta.kv_lo ? (meta.kv_end - meta.kv_lo) * (ATT_BLK / ATT_SUB) : 0;
  if (nsub == 0) {
    zero_rows<BWD_THREADS>(dQb, p.ld1, lrow0, p.Tq, tid);
    return;
  }
  const bf16* Kb = p.K + int64_t(b) * p.T * p.ldk + kvh * ATT_HD;
  const bf16* Vb = p.V + int64_t(b) * p.T * p.ldv + kvh * ATT_HD;
  const int kbase = meta.kv_lo * ATT_BLK;
  load_tile_async<ATT_BLK, BWD_THREADS>(sb + DqSmem::Q, p.Q + int64_t(b) * p.Tq * p.ldq + h * ATT_HD, p.ldq, lrow0, 0, p.Tq,
                                        tid);
  load_tile_async<ATT_BLK, BWD_THREADS>(sb + DqSmem::DO, p.dO + int64_t(b) * p.Tq * p.lddo + h * ATT_HD, p.lddo, lrow0, 0,
                                        p.Tq, tid);
  auto load_kv = [&](int i, int buf) {
    const int k0 = kbase + i * ATT_SUB;
    load_tile_async<ATT_SUB, BWD_THREADS>(sb + DqSmem::K + buf * STR_TILE, Kb, p.ldk, k0, 0, p.T, tid);
    load_tile_async<ATT_SUB, BWD_THREADS>(sb + DqSmem::V + buf * STR_TILE, Vb, p.ldv, k0, 0, p.T, tid);
    if (tid < ATT_SUB) sDoc[buf * ATT_SUB + tid] = (k0 + tid < p.T) ? docb[k0 + tid] : 0;
    cp_async_commit();
  };
  load_kv(0, 0);

  const int ra = warp * 16 + (lane >> 2);
  const int qa = q0 + ra, qb8 = qa + 8;
  const int32_t da = qa < p.T ? docb[qa] : 0, db = qb8 < p.T ? docb[qb8] : 0;
  const int32_t d_last = (q0 + ATT_BLK - 1 < p.T) ? docb[q0 + ATT_BLK - 1] : 0;
  const int la = lrow0 + ra, lb = la + 8;
  const float* lseb = p.lse + (int64_t(b) * p.H + h) * p.Tq;
  const float* delb = p.delta + (int64_t(b) * p.H + h) * p.Tq;
  const float l2a = la < p.Tq ? lseb[la] * LOG2E : INFINITY;
  const float l2b = lb < p.Tq ? lseb[lb] * LOG2E : INFINITY;
  const float dla = la < p.Tq ? delb[la] : 0.f, dlb = lb < p.Tq ? delb[lb] : 0.f;
  float dq[16][4];
#pragma unroll
  for (int j = 0; j < 16; ++j) dq[j][0] = dq[j][1] = dq[j][2] = dq[j][3] = 0.f;

  for (int i = 0; i < nsub; ++i) {
    const int buf = i & 1;
    if (i + 1 < nsub) { load_kv(i + 1, buf ^ 1); cp_async_wait<1>(); }
    else cp_async_wait<0>();
    __syncthreads();
    const uint32_t sK = sb + DqSmem::K + buf * STR_TILE, sV = sb + DqSmem::V + buf * STR_TILE;
    const int32_t* dkd = sDoc + buf * ATT_SUB;
    const int k0 = kbase + i * ATT_SUB;

    float s[8][4], dp[8][4];
    mma_scores_nk<4>(s, TileRows{sb + DqSmem::Q, warp * 16}, sK, 0);
    mma_scores_nk<4>(dp, TileRows{sb + DqSmem::DO, warp * 16}, sV, 0);
    const bool full = meta.canonical && (k0 + ATT_SUB <= q0) && d_last > 0 && dkd[0] == d_last;
    const DocMask<false> mask{p.scale_log2, full, qa, da, db, k0, dkd};
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float pr = fast_exp2(mask(s[j][e], j, e) - (e < 2 ? l2a : l2b));
        dp[j][e] = pr * (dp[j][e] - (e < 2 ? dla : dlb));
      }
    }
    // dQ += dS.K
    mma_acc_kn(dq, dp, sK, 0);
    __syncthreads();
  }
  store_acc_rows(dQb, p.ld1, la, p.Tq, dq, p.scale, p.rope_cos, p.rope_sin, int64_t(b) * p.Tq + la);
}

}  // namespace tn

using namespace tn;

extern "C" int tn_attn_bwd_bf16(const void* Q, int64_t ldq, const void* K, int64_t ldk, const void* V, int64_t ldv,
                                const void* O, int64_t ldo, const void* dO, int64_t lddo, const float* lse, float* delta,
                                void* dQ, int64_t lddq, void* dK, int64_t lddk, void* dV, int64_t lddv,
                                const int32_t* doc_ids, const int32_t* meta, int B, int T, int H, int KV, float scale,
                                int Tq, int q_blk_off, const void* rope_cos_q, const void* rope_sin_q,
                                const void* rope_cos_k, const void* rope_sin_k, tn_stream_t stream_) {
  clear_error();
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  TN_REQUIRE(Q && K && V && O && dO && lse && delta && dQ && dK && dV && doc_ids && meta, "tn_attn_bwd_bf16: null pointer");
  TN_REQUIRE((rope_cos_q == nullptr) == (rope_sin_q == nullptr) && (rope_cos_k == nullptr) == (rope_sin_k == nullptr),
             "tn_attn_bwd_bf16: cos and sin tables come in pairs");
  TN_REQUIRE(B > 0 && T > 0 && H > 0 && KV > 0 && H % KV == 0, "tn_attn_bwd_bf16: bad dims");
  TN_REQUIRE(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 8 == 0 && lddo % 8 == 0 && lddq % 8 == 0 &&
                 lddk % 8 == 0 && lddv % 8 == 0, "tn_attn_bwd_bf16: strides must be multiples of 8");
  TN_REQUIRE(attn_query_window(T, Tq, q_blk_off), "tn_attn_bwd_bf16: query window outside the sequence");
  const int nblk = (T + ATT_BLK - 1) / ATT_BLK, nqb = (Tq + ATT_BLK - 1) / ATT_BLK;

  {
    const int64_t pairs = int64_t(B) * Tq * H;
    const int64_t threads = pairs * 16;
    attn_delta_kernel<<<unsigned((threads + 255) / 256), 256, 0, stream>>>(
        static_cast<const bf16*>(O), ldo, static_cast<const bf16*>(dO), lddo, delta, B, Tq, H);
    TN_CHECK_CUDA(cudaGetLastError());
  }

  AttnBwdParams p{};
  p.doc = doc_ids; p.meta = reinterpret_cast<const AttnMeta*>(meta); p.lse = lse; p.delta = delta;
  p.Q = static_cast<const bf16*>(Q); p.K = static_cast<const bf16*>(K); p.V = static_cast<const bf16*>(V);
  p.dO = static_cast<const bf16*>(dO);
  p.ldq = ldq; p.ldk = ldk; p.ldv = ldv; p.lddo = lddo;
  p.B = B; p.T = T; p.H = H; p.KV = KV; p.nblk = nblk;
  p.Tq = Tq; p.q_blk_off = q_blk_off;
  p.scale = scale; p.scale_log2 = scale * LOG2E;

  TN_CHECK_CUDA(attn_smem_optin<attn_dkdv_kernel>(DkdvSmem::TOTAL));
  TN_CHECK_CUDA(attn_smem_optin<attn_dq_kernel>(DqSmem::TOTAL));
  {
    AttnBwdParams pk = p;
    pk.out1 = static_cast<bf16*>(dV); pk.ld1 = lddv; pk.out2 = static_cast<bf16*>(dK); pk.ld2 = lddk;
    pk.rope_cos = static_cast<const bf16*>(rope_cos_k); pk.rope_sin = static_cast<const bf16*>(rope_sin_k);
    const dim3 grid = attn_grid(T, Tq, q_blk_off, meta + attn_meta_order_kv_off(B, nblk), nblk, KV, B, pk.order);
    attn_dkdv_kernel<<<grid, BWD_THREADS, DkdvSmem::TOTAL, stream>>>(pk);
    TN_CHECK_CUDA(cudaGetLastError());
  }
  {
    AttnBwdParams pq = p;
    pq.out1 = static_cast<bf16*>(dQ); pq.ld1 = lddq; pq.out2 = nullptr; pq.ld2 = 0;
    pq.rope_cos = static_cast<const bf16*>(rope_cos_q); pq.rope_sin = static_cast<const bf16*>(rope_sin_q);
    const dim3 grid = attn_grid(T, Tq, q_blk_off, meta + attn_meta_order_off(B, nblk), nqb, H, B, pq.order);
    attn_dq_kernel<<<grid, BWD_THREADS, DqSmem::TOTAL, stream>>>(pq);
    TN_CHECK_CUDA(cudaGetLastError());
  }
  return TN_OK;
}
