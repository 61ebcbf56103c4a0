// touchnet_b200 :: wgmma GEMM for the projection / MLP matmuls of the packed decoder layer.
//
// Replaces the cuBLASLt calls behind F.linear at
//   hf:models/llama/modeling_llama.py:251-289 (q/k/v/o_proj), :182-184 (gate/up/down_proj)
//   touchnet/models/touch_audio/modeling_touch_audio.py:127 (projector)
// and their autograd backward (dgrad, wgrad).
//
// Design (H100, one CTA per SM, persistent, warp-specialised):
//   warpgroup 0     : TMA producer - one thread streams 128 x 64 A and BN x 64 B tiles (128B swizzle) into a STAGES-deep
//                     shared-memory ring guarded by full / empty mbarriers; it runs ahead into the next tile while the
//                     consumers are still in the epilogue of the current one.  setmaxnreg gives its registers away.
//   warpgroups 1, 2 : consumers - each issues wgmma.m64n{BN}k16 on its 64 rows of the 128 x BN tile (fp32 accumulator in
//                     registers), then writes the finished values into 64-row swizzled staging sub-tiles in shared memory
//                     that TMA stores push to global memory; the stores drain while the next tile's MMAs run
// BN = 256 (m64n256: half the shared-memory operand traffic per FLOP of the 128-wide tile) or 128, chosen on the host from
// the wave count of the shape (pick_bn).  Operands may be K-major or MN-major (the transpose bits of wgmma), so
// forward, dgrad and wgrad all run on the tensors where they lie: no transposes, no copies.  Epilogues: D = acc (+R) in
// bf16 or fp32, SwiGLU (gate and up halves of one tile), SwiGLU backward on the dH accumulator, RoPE on the q/k columns of
// the fused QKV projection.  Each output element sums its k-blocks in the same order at either tile width.
// FP8 (OP != 0): the same kernel on 8-bit operands, both K-major (8-bit wgmma has no transpose bits).  A stage holds
// 128 k (the same 128-byte swizzled rows, stage bytes and stage count) and takes four wgmma k32 steps; the epilogue
// starts by multiplying the accumulator with the two per-tensor inverse scales read from device memory.  Forward
// (e4m3 A) accumulates in the wgmma accumulator alone; dgrad and wgrad (e5m2 A) add each stage's partial sum into a
// separate fp32 accumulator, because the 8-bit MMAs accumulate with reduced precision.  That doubles the accumulator
// registers, so the promoted form runs on the 128-wide tile only.
// Rowwise FP8 (OP 3, 4): both operands e4m3 with one scale per row of A and per row of B (torchao's rowwise recipe,
// torch._scaled_mm's scale_a [M,1] / scale_b [1,N]); the dequantisation multiplies each accumulator element with the
// 1/s of its row and its column, read from two device vectors, ahead of the same epilogues.  OP 3 accumulates like
// OP 1 (forward), OP 4 promotes like OP 2 (dgrad, wgrad).
#include <stdio.h>
#include <stdlib.h>

#include "../../include/touchnet_b200.h"
#include "common.cuh"
#include "host.h"

namespace tn {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int GEMM_THREADS = 384;
constexpr int A_BYTES = BM * BK * 2;              // 16 KB
constexpr int SUB_BYTES = 64 * 128;               // one staging sub-tile: 64 rows x 128 B (64 bf16 or 32 fp32 columns)
constexpr int STAGING_BYTES = 2 * 2 * SUB_BYTES;  // two sub-tile buffers per consumer warpgroup
constexpr int SMEM_LIMIT = 227 * 1024;
template <int BN>
struct TileCfg {
  static constexpr int B_BYTES = BN * BK * 2;     // 16 KB (BN 128) / 32 KB (BN 256)
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STAGES = (SMEM_LIMIT - STAGING_BYTES - 256 - 1024) / STAGE_BYTES;   // 6 / 4
  static constexpr int SMEM = STAGES * STAGE_BYTES + STAGING_BYTES + 256 + 1024;          // + barriers + alignment slack
};

// EPI: 0 = bf16 D = acc (+R);  1 = SwiGLU (cols [0,BN/2) gate, [BN/2,BN) up -> G, U, H);  2 = fp32 D = acc (+R);
//      3 = SwiGLU backward on the dH accumulator: dG = (dH*U) * silu'(G), dU = dH * silu(G)  (same rounding points as
//          tn_swiglu_bwd_bf16 applied to the bf16-rounded dH, so the fused and the two-kernel paths agree bit for bit)
struct GemmParams {
  int M, N, K;
  int num_m, num_n, num_k;
  int group;                 // raster: tiles walk `group` M blocks x all N blocks before moving down (L2 reuse of A)
  uint64_t hint_a, hint_b;   // L2 policy of the operand loads (tn_set_gemm_l2_hints)
  const void* R;             // residual, read in the accumulator layout (may alias the output: in-place accumulation)
  int64_t ldr;
  int has_g, has_u;          // EPI 1: G / U are written too
  // segmented operands: several weight tensors that are separate nn.Parameters (q/k/v projections) behave as one GEMM
  //   b_seg 1: B = [B0;B1;B2] stacked along N (fused QKV forward)       -> D columns [0,off1) [off1,off2) [off2,N)
  //   b_seg 2: B = [B0;B1;B2] stacked along K (fused QKV dgrad)         -> A columns ...
  //   d_seg 1: D = [D0;D1;D2] stacked along M (fused QKV wgrad: one dW per parameter)
  int b_seg, d_seg;
  int off1, off2;
  // fused RoPE in the epilogue of the QKV forward (hf apply_rotary_pos_emb, modeling_llama.py:151-168): output columns
  // below rope_end (the q and k segments, heads of 128 columns) are rotated with the per-row cos/sin tables
  // [M, 64] bf16 (tn_rope_table); same bf16 rounding points as the unfused kernel -> bit-identical results
  const bf16* rope_cos;
  const bf16* rope_sin;
  int rope_end;
  // EPI 3: saved G / U ([M, N] bf16, row stride ld_gu)
  const bf16* aux_g;
  const bf16* aux_u;
  int64_t ld_gu;
  // FP8: 1/s of the A and B operands (device floats written by tn_fp8_cast_bf16)
  // rowwise FP8: vectors of 1/s per row of A [M] and per row of B [N] (the QKV forward: the rows of [Wq;Wk;Wv],
  // indexed by the output column; EPI 1: [2N], the gate rows then the up rows)
  const float* inv_sa;
  const float* inv_sb;
  // plain epilogue (EPI 0 / 2): output columns [n_store, N) - less than one 16-byte chunk, when the row length in bytes
  // is not a multiple of 16 - are written with ordinary stores to d (row stride ldd), because the TMA store writes
  // whole 16-byte chunks and would write past N into the caller's memory; the output map then ends at n_store.
  // n_store = N: no such columns.
  int n_store;
  void* d;
  int64_t ldd;
};

// Operand and output tensor maps.  d[]: EPI 0/2 the output (d_seg: one map per segment), EPI 1 H / G / U, EPI 3 dG / dU;
// output boxes are one staging sub-tile (64 rows x 128 B, 128B swizzle).
struct GemmMaps {
  CUtensorMap a, b[3], d[3];
};

__device__ __forceinline__ void decode_tile(int tile, int num_m, int num_n, int group, int& m_blk, int& n_blk) {
  const int per_group = group * num_n;
  const int g = tile / per_group;
  const int first_m = g * group;
  const int gsize = min(num_m - first_m, group);
  const int r = tile - g * per_group;
  m_blk = first_m + (r % gsize);
  n_blk = r / gsize;
}

// OP: operand type and accumulation.  0 = bf16;  1 = e4m3 A, e4m3 B, accumulated in the wgmma accumulator (forward);
//     2 = e5m2 A, e4m3 B, stage partial sums promoted into a separate fp32 accumulator (dgrad / wgrad, BN 128 only);
//     3 = OP 1 and 4 = e4m3 A promoted as OP 2, both with per-row scales (rowwise recipe)
template <int BN, bool A_MN, bool B_MN, int EPI, int OP = 0>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_kernel(const __grid_constant__ GemmMaps tm, const GemmParams p) {
  static_assert(OP == 0 || (!A_MN && !B_MN), "8-bit operands are K-major");
  static_assert((OP != 2 && OP != 4) || BN == 128, "the promoted accumulator fits the 128-wide tile only");
  using C = TileCfg<BN>;
  constexpr int STAGES = C::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sA = smem;
  uint8_t* sB = smem + STAGES * A_BYTES;
  uint8_t* sStage = smem + STAGES * C::STAGE_BYTES;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(sStage + STAGING_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;

  const int wg = int(threadIdx.x) >> 7;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm.a);
    tma_prefetch_desc(&tm.b[0]);
    if (EPI == 1 || p.b_seg) { tma_prefetch_desc(&tm.b[1]); }
    if (p.b_seg) tma_prefetch_desc(&tm.b[2]);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 8);   // one arrive per consumer warp
    }
    fence_barrier_init();
  }
  __syncthreads();

  const int num_tiles = p.num_m * p.num_n;
  constexpr int TN = (EPI == 1) ? BN / 2 : BN;   // output columns per tile

  if (wg == 0) {
    // ===================== TMA producer =====================
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        int m_blk, n_blk;
        decode_tile(tile, p.num_m, p.num_n, p.group, m_blk, n_blk);
        const int m0 = m_blk * BM;
        int n0 = n_blk * TN;
        const CUtensorMap* bmap = &tm.b[0];
        if (p.b_seg == 1) {   // weight segment that owns these output columns
          const int sg = (n0 >= p.off1) + (n0 >= p.off2);
          bmap = &tm.b[sg];
          n0 -= sg == 0 ? 0 : (sg == 1 ? p.off1 : p.off2);
        }
        for (int kb = 0; kb < p.num_k; ++kb) {
          mbar_wait_nocall(&empty_bar[stage], phase ^ 1);
          mbar_arrive_expect_tx(&full_bar[stage], C::STAGE_BYTES);
          uint8_t* a_dst = sA + stage * A_BYTES;
          uint8_t* b_dst = sB + stage * C::B_BYTES;
          const int k0 = kb * (OP ? 2 * BK : BK);   // k per stage: 128-byte operand rows either way
          int kb0 = k0;   // k coordinate inside the selected B segment
          if (p.b_seg == 2) {
            const int sg = (k0 >= p.off1) + (k0 >= p.off2);
            bmap = &tm.b[sg];
            kb0 = k0 - (sg == 0 ? 0 : (sg == 1 ? p.off1 : p.off2));
          }
          if (!A_MN) {
            tma_load_2d(a_dst, &tm.a, &full_bar[stage], k0, m0, p.hint_a);   // box {64 k, 128 m}
          } else {
            tma_load_2d(a_dst, &tm.a, &full_bar[stage], m0, k0, p.hint_a);   // boxes {64 m, 64 k}
            tma_load_2d(a_dst + 8192, &tm.a, &full_bar[stage], m0 + 64, k0, p.hint_a);
          }
          if (EPI == 1) {
            tma_load_2d(b_dst, &tm.b[0], &full_bar[stage], k0, n0, p.hint_b);                 // BN/2 gate rows
            tma_load_2d(b_dst + C::B_BYTES / 2, &tm.b[1], &full_bar[stage], k0, n0, p.hint_b);  // BN/2 up rows
          } else if (!B_MN) {
            tma_load_2d(b_dst, bmap, &full_bar[stage], kb0, n0, p.hint_b);                    // box {64 k, BN n}
          } else {
#pragma unroll
            for (int i = 0; i < BN / 64; ++i)                                                   // boxes {64 n, 64 k}
              tma_load_2d(b_dst + i * 8192, bmap, &full_bar[stage], n0 + 64 * i, kb0, p.hint_b);
          }
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // ===================== consumers =====================
  setmaxnreg_inc<232>();
  const int c = wg - 1;                          // 64-row half of the tile
  const int t = int(threadIdx.x) & 127;
  const int lane = t & 31, warp = t >> 5;
  const int r_loc = warp * 16 + (lane >> 2);     // accumulator row inside the warpgroup's 64 (h = 0; h = 1 adds 8)
  const int cq = 2 * (lane & 3);
  uint8_t* stg = sStage + c * (2 * SUB_BYTES);
  int sbuf = 0;
  int stage = 0;
  uint32_t phase = 0;
  float acc[BN / 2];

  // Staging sub-tiles out.  `fill` writes the accumulator values of one sub-tile (two for a pair) into the staging
  // buffers; an optional `pass` then walks the staged rows coalesced (thread t: chunk t % 8 of rows t / 8 + 16 i) and
  // combines them with global operands (residual, G / U, cos / sin), so those loads never sit next to the live
  // accumulator.  The buffers then go to the async proxy and out as TMA stores, one bulk group per buffer.  Before a
  // buffer is rewritten, thread 0 (bulk groups are per thread) waits until the store that last read it is done.
  auto emit = [&](bool pair, auto&& fill, bool has_pass, auto&& pass, auto&& store) {
    uint8_t* buf = pair ? stg : stg + sbuf * SUB_BYTES;
    if (t == 0) {
      if (pair) tma_store_wait_read<0>();
      else tma_store_wait_read<1>();
    }
    named_bar_sync(1 + c, 128);
    fill(buf);
    if (has_pass) {
      named_bar_sync(1 + c, 128);
      pass(buf);
    }
    fence_proxy_async_smem();
    named_bar_sync(1 + c, 128);
    if (t == 0) store(buf);
    sbuf = pair ? 0 : sbuf ^ 1;
  };
  auto no_pass = [](uint8_t*) {};
  auto store1 = [&](const CUtensorMap* map, int x0, int y0) {
    return [=](uint8_t* buf) { tma_store_2d(map, buf, x0, y0); tma_store_commit(); };
  };
  auto store2 = [&](const CUtensorMap* m0, int x0, const CUtensorMap* m1, int x1, int y0) {
    return [=](uint8_t* buf) {
      tma_store_2d(m0, buf, x0, y0); tma_store_commit();
      tma_store_2d(m1, buf + SUB_BYTES, x1, y0); tma_store_commit();
    };
  };
  // 128B swizzle of the staging rows (the TMA store map's layout): 16-byte chunk q of row r sits at chunk q ^ (r & 7);
  // r & 7 == lane / 4 for both accumulator rows of a thread, so each warp-wide store touches all 32 banks once
  auto put_bf16x2 = [&](uint8_t* buf, int jj, int h, uint32_t v) {   // columns 8jj + cq, +1 of a 64-column sub-tile
    *reinterpret_cast<uint32_t*>(buf + (r_loc + 8 * h) * 128 + ((jj ^ (lane >> 2)) << 4) + 2 * cq) = v;
  };
  auto put_f32x2 = [&](uint8_t* buf, int jj, int h, float lo, float hi) {   // columns 8jj + cq, +1 of a 32-column one
    const int q = 2 * jj + (cq >> 2);
    *reinterpret_cast<float2*>(buf + (r_loc + 8 * h) * 128 + ((q ^ (lane >> 2)) << 4) + 4 * (cq & 3)) =
        make_float2(lo, hi);
  };
  auto chunk = [&](uint8_t* buf, int rr) {   // the pass's 16-byte chunk (t % 8) of staged row rr
    return reinterpret_cast<uint4*>(buf + rr * 128 + (((t & 7) ^ (rr & 7)) << 4));
  };
  auto stage_bf16 = [&](int s) {   // bf16-rounded accumulator columns [64s, 64s + 64)
    return [&, s](uint8_t* buf) {
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
#pragma unroll
        for (int h = 0; h < 2; ++h)
          put_bf16x2(buf, jj, h, pack_bf16x2(acc[4 * (8 * s + jj) + 2 * h], acc[4 * (8 * s + jj) + 2 * h + 1]));
    };
  };
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    int m_blk, n_blk;
    decode_tile(tile, p.num_m, p.num_n, p.group, m_blk, n_blk);
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    int prev = -1;
    for (int kb = 0; kb < p.num_k; ++kb) {
      mbar_wait_nocall(&full_bar[stage], phase);
      const uint32_t a_addr = smem_u32(sA + stage * A_BYTES) + uint32_t(c) * 8192u;
      const uint32_t b_addr = smem_u32(sB + stage * C::B_BYTES);
      wgmma_fence();
      if constexpr (OP == 2 || OP == 4) {
        float part[BN / 2];                      // this stage's partial sum
#pragma unroll
        for (int k = 0; k < 4; ++k)
          wgmma_fp8_m64n128<OP == 2>(part, make_sdesc_sw128(a_addr + k * 32, 16, 1024),
                                  make_sdesc_sw128(b_addr + k * 32, 16, 1024), k > 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(part);
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] += part[i];
      } else {
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) {
          const uint64_t da = A_MN ? make_sdesc_sw128(a_addr + k * 2048, 8192, 1024) : make_sdesc_sw128(a_addr + k * 32, 16, 1024);
          const uint64_t db = B_MN ? make_sdesc_sw128(b_addr + k * 2048, 8192, 1024) : make_sdesc_sw128(b_addr + k * 32, 16, 1024);
          if constexpr (OP == 1 || OP == 3) {
            if constexpr (BN == 256) wgmma_fp8_m64n256<false>(acc, da, db, 1u);
            else wgmma_fp8_m64n128<false>(acc, da, db, 1u);
          } else if constexpr (BN == 256) {
            wgmma_m64n256<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, da, db, 1u);
          } else {
            wgmma_m64n128<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, da, db, 1u);
          }
        }
        wgmma_commit();
        wgmma_wait<1>();                         // the previous k-block's MMAs have retired: its slot can be refilled
        wgmma_fence_regs(acc);
      }
      if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
      prev = stage;
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc);
    if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
    if constexpr (OP == 1 || OP == 2) {   // dequantise: acc · (1/s_a)·(1/s_b), ahead of every epilogue
      const float sc = *p.inv_sa * *p.inv_sb;
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] *= sc;
    } else if constexpr (OP >= 3) {       // acc(m, n) · (1/s_a[m]) · (1/s_b[n]); rows / columns past M / N are clipped
      const int row = m_blk * BM + c * 64 + r_loc;
      float sa[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) sa[h] = row + 8 * h < p.M ? p.inv_sa[row + 8 * h] : 0.f;
      // the 1/s of columns 8j + cq, +1: lane L loads those of j = 8g + L/4 for the threads with lane % 4 == L % 4 and
      // hands them out by shuffle (one coalesced load per 8 j; per-j loads would be hoisted next to the live
      // accumulator and spill on the 256-wide tile)
#pragma unroll
      for (int g = 0; g < BN / 64; ++g) {
        const int jl = 8 * g + (lane >> 2);
        const bool up = EPI == 1 && jl >= BN / 16;       // SwiGLU: the up half of the tile
        const int col = n_blk * TN + 8 * (up ? jl - BN / 16 : jl) + cq;
        const float2 sb = col < p.N ? *reinterpret_cast<const float2*>(p.inv_sb + (up ? p.N : 0) + col)
                                    : make_float2(0.f, 0.f);
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          const int j = 8 * g + jj, src = (jj << 2) | (lane & 3);
          const float bx = __shfl_sync(0xffffffffu, sb.x, src), by = __shfl_sync(0xffffffffu, sb.y, src);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            acc[4 * j + 2 * h] = acc[4 * j + 2 * h] * sa[h] * bx;
            acc[4 * j + 2 * h + 1] = acc[4 * j + 2 * h + 1] * sa[h] * by;
          }
        }
      }
      wgmma_fence_regs(acc);   // keeps the products here: sunk into the epilogue, the 64 scales would stay live there
    }

    // ---------------- epilogue: registers -> swizzled staging (-> coalesced pass) -> TMA store ----------------
    const int m0 = m_blk * BM;
    const int n0 = n_blk * TN;
    const int y0 = m0 + c * 64;                  // first row of this warpgroup; the stores clip rows >= M, cols >= N
    if (y0 >= p.M) continue;                     // warpgroup-uniform
    if (EPI == 1) {
#pragma unroll
      for (int s = 0; s < TN / 64; ++s) {
        const int x0 = n0 + 64 * s;
        if (x0 >= p.N) break;
        // mimic the unfused reference rounding: g,u -> bf16; silu(g) -> bf16; * u -> bf16
        auto gate = [&](int jj, int h, int e) { return bf16_round(acc[4 * (8 * s + jj) + 2 * h + e]); };
        auto up = [&](int jj, int h, int e) { return bf16_round(acc[4 * (8 * s + jj + BN / 16) + 2 * h + e]); };
        emit(false, [&](uint8_t* buf) {
#pragma unroll
          for (int jj = 0; jj < 8; ++jj)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              float hh[2];
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const float g = gate(jj, h, e);
                hh[e] = bf16_round(g / (1.f + __expf(-g))) * up(jj, h, e);
              }
              put_bf16x2(buf, jj, h, pack_bf16x2(hh[0], hh[1]));
            }
        }, false, no_pass, store1(&tm.d[0], x0, y0));
        if (p.has_g)
          emit(false, [&](uint8_t* buf) {
#pragma unroll
            for (int jj = 0; jj < 8; ++jj)
#pragma unroll
              for (int h = 0; h < 2; ++h) put_bf16x2(buf, jj, h, pack_bf16x2(gate(jj, h, 0), gate(jj, h, 1)));
          }, false, no_pass, store1(&tm.d[1], x0, y0));
        if (p.has_u)
          emit(false, [&](uint8_t* buf) {
#pragma unroll
            for (int jj = 0; jj < 8; ++jj)
#pragma unroll
              for (int h = 0; h < 2; ++h) put_bf16x2(buf, jj, h, pack_bf16x2(up(jj, h, 0), up(jj, h, 1)));
          }, false, no_pass, store1(&tm.d[2], x0, y0));
      }
    } else if (EPI == 3) {
      // dH (bf16-rounded, as the unfused path stores it) staged in buffer 0; the pass reads it with G / U and writes dG
      // over it and dU into buffer 1
#pragma unroll
      for (int s = 0; s < BN / 64; ++s) {
        const int x0 = n0 + 64 * s;
        if (x0 >= p.N) break;
        emit(true, stage_bf16(s), true, [&](uint8_t* buf) {
          // 4-byte pieces (a warp per row): next to the live accumulator there is no room for wider ones
#pragma unroll 1
          for (int i = 0; i < 16; ++i) {
            const int rr = (t >> 5) + 4 * i, row = y0 + rr, col = x0 + 2 * lane;
            if (row >= p.M || col >= p.N) continue;   // N % 8 == 0: whole pairs
            const int off = rr * 128 + (((lane >> 2) ^ (rr & 7)) << 4) + 4 * (lane & 3);
            uint32_t* pd = reinterpret_cast<uint32_t*>(buf + off);
            uint32_t* pu = reinterpret_cast<uint32_t*>(buf + SUB_BYTES + off);
            const uint32_t dw = *pd;
            const uint32_t gw = *reinterpret_cast<const uint32_t*>(p.aux_g + int64_t(row) * p.ld_gu + col);
            const uint32_t uw = *reinterpret_cast<const uint32_t*>(p.aux_u + int64_t(row) * p.ld_gu + col);
            float rg[2], ru[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const float d = e ? bf16hi(dw) : bf16lo(dw);
              const float g = e ? bf16hi(gw) : bf16lo(gw);
              const float u = e ? bf16hi(uw) : bf16lo(uw);
              const float sig = 1.f / (1.f + __expf(-g));
              ru[e] = d * bf16_round(g * sig);
              rg[e] = bf16_round(d * u) * (sig * (1.f + g * (1.f - sig)));
            }
            *pd = pack_bf16x2(rg[0], rg[1]);
            *pu = pack_bf16x2(ru[0], ru[1]);
          }
        }, store2(&tm.d[0], x0, &tm.d[1], x0, y0));
      }
    } else if (EPI == 0 && p.rope_cos != nullptr && n0 < p.rope_end) {
      // RoPE tile: BN / 128 whole heads.  Both halves of a head (columns j and j + 64 pair up) are staged as bf16, then
      // the pass rotates them with the row's cos / sin and writes o1 over the first half and o2 over the second.
#pragma unroll
      for (int hd = 0; hd < BN / 128; ++hd) {
        const int x0 = n0 + 128 * hd;
        emit(true, [&](uint8_t* buf) {
          stage_bf16(2 * hd)(buf);
          stage_bf16(2 * hd + 1)(buf + SUB_BYTES);
        }, true, [&](uint8_t* buf) {
#pragma unroll 1
          for (int i = 0; i < 4; ++i) {
            const int rr = (t >> 3) + 16 * i, row = y0 + rr, cc = 8 * (t & 7);
            if (row >= p.M) continue;
            uint4* pa = chunk(buf, rr);
            uint4* pb = chunk(buf + SUB_BYTES, rr);
            const uint4 av = *pa, bv = *pb;
            const uint4 cv = *reinterpret_cast<const uint4*>(p.rope_cos + int64_t(row) * 64 + cc);
            const uint4 sv = *reinterpret_cast<const uint4*>(p.rope_sin + int64_t(row) * 64 + cc);
            const uint32_t* aw = &av.x;
            const uint32_t* bw = &bv.x;
            const uint32_t* cw = &cv.x;
            const uint32_t* sw = &sv.x;
            uint4 o1, o2;
            uint32_t* o1w = &o1.x;
            uint32_t* o2w = &o2.x;
#pragma unroll
            for (int w = 0; w < 4; ++w) {
              float r1[2], r2[2];
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const float a = e ? bf16hi(aw[w]) : bf16lo(aw[w]), b = e ? bf16hi(bw[w]) : bf16lo(bw[w]);
                const float cs = e ? bf16hi(cw[w]) : bf16lo(cw[w]), sn = e ? bf16hi(sw[w]) : bf16lo(sw[w]);
                r1[e] = bf16_round(a * cs) + bf16_round(-b * sn);
                r2[e] = bf16_round(b * cs) + bf16_round(a * sn);
              }
              o1w[w] = pack_bf16x2(r1[0], r1[1]);
              o2w[w] = pack_bf16x2(r2[0], r2[1]);
            }
            *pa = o1;
            *pb = o2;
          }
        }, store2(&tm.d[0], x0, &tm.d[0], x0 + 64, y0));
      }
    } else {
      const CUtensorMap* dmap = &tm.d[0];
      int yd = y0;
      if (p.d_seg == 1) {   // output rows belong to one of several gradient tensors (segments are multiples of 256)
        const int sg = (m0 >= p.off1) + (m0 >= p.off2);
        dmap = &tm.d[sg];
        yd -= sg == 0 ? 0 : (sg == 1 ? p.off1 : p.off2);
      }
      constexpr int SW = EPI == 2 ? 32 : 64;   // columns per sub-tile
      constexpr int CW = SW / 8;               // columns per 16-byte chunk
#pragma unroll
      for (int s = 0; s < BN / SW; ++s) {
        const int x0 = n0 + SW * s;
        if (x0 >= p.N) break;
        auto fill = [&](uint8_t* buf) {
#pragma unroll
          for (int jj = 0; jj < SW / 8; ++jj)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const float lo = acc[4 * ((SW / 8) * s + jj) + 2 * h], hi = acc[4 * ((SW / 8) * s + jj) + 2 * h + 1];
              if (EPI == 2) put_f32x2(buf, jj, h, lo, hi);
              else put_bf16x2(buf, jj, h, pack_bf16x2(lo, hi));
            }
        };
        // + R: fp32 acc + R, or (reference order) the bf16-rounded product + R rounded again
        auto add_residual = [&](uint8_t* buf) {
#pragma unroll 1
          for (int i = 0; i < 4; ++i) {
            const int rr = (t >> 3) + 16 * i, row = y0 + rr, col = x0 + CW * (t & 7);
            if (row >= p.M || col >= p.N) continue;
            uint4* pd = chunk(buf, rr);
            uint4 v = *pd;
            if (EPI == 2) {
              const float* rp = static_cast<const float*>(p.R) + int64_t(row) * p.ldr + col;
              float* f = reinterpret_cast<float*>(&v);
              if (col + 4 <= p.N) {
                const float4 r = *reinterpret_cast<const float4*>(rp);
                f[0] += r.x; f[1] += r.y; f[2] += r.z; f[3] += r.w;
              } else {
#pragma unroll
                for (int e = 0; e < 4; ++e)
                  if (col + e < p.N) f[e] += rp[e];
              }
            } else {
              const bf16* rp = static_cast<const bf16*>(p.R) + int64_t(row) * p.ldr + col;
              uint4 r = make_uint4(0, 0, 0, 0);
              uint32_t* rw = &r.x;
              if (col + 8 <= p.N) {
                r = *reinterpret_cast<const uint4*>(rp);
              } else {   // ragged N: the pairs that exist (the columns past N are clipped by the store)
#pragma unroll
                for (int e = 0; e < 8; e += 2)
                  if (col + e < p.N)
                    rw[e / 2] = uint32_t(__bfloat16_as_ushort(rp[e])) |
                                (col + e + 1 < p.N ? uint32_t(__bfloat16_as_ushort(rp[e + 1])) << 16 : 0u);
              }
              uint32_t* vw = &v.x;
#pragma unroll
              for (int w = 0; w < 4; ++w)
                vw[w] = pack_bf16x2(bf16lo(vw[w]) + bf16lo(rw[w]), bf16hi(vw[w]) + bf16hi(rw[w]));
            }
            *pd = v;
          }
        };
        emit(false, fill, p.R != nullptr, add_residual, [=](uint8_t* buf) {
          if (x0 < p.n_store) tma_store_2d(dmap, buf, x0, yd);   // the map ends at n_store: it clips the rest
          tma_store_commit();
        });
      }
      if (p.n_store < p.N && n0 + BN > p.n_store && t < 64 && y0 + t < p.M) {
        // the ragged tail [n_store, N) of the last column tile (only tn_gemm_bf16 sets n_store < N, without segments):
        // one 16-byte chunk of each row of the sub-tile staged last, read after the accumulator is dead; the next
        // emit() synchronises the warpgroup before it writes that buffer again
        const int xt = p.n_store - (p.n_store - n0) % SW;          // first column of that sub-tile
        const uint8_t* sub = stg + (sbuf ^ 1) * SUB_BYTES;
        const int q = (p.n_store - xt) / CW;
        const uint4 v = *reinterpret_cast<const uint4*>(sub + t * 128 + ((q ^ (t & 7)) << 4));
        const int64_t off = int64_t(y0 + t) * p.ldd + p.n_store;
#pragma unroll
        for (int e = 0; e < CW - 1; ++e)
          if (p.n_store + e < p.N) {
            if (EPI == 2) static_cast<float*>(p.d)[off + e] = reinterpret_cast<const float*>(&v)[e];
            else static_cast<bf16*>(p.d)[off + e] = reinterpret_cast<const bf16*>(&v)[e];
          }
      }
    }
  }
  if (t == 0) tma_store_wait<0>();   // staging must stay valid until the last stores have read it
}

template <int BN, bool A_MN, bool B_MN, int EPI, int OP = 0>
static int launch_gemm(const GemmMaps& tm, const GemmParams& p, cudaStream_t stream) {
  auto kern = gemm_kernel<BN, A_MN, B_MN, EPI, OP>;
  constexpr int smem = TileCfg<BN>::SMEM;
  static bool configured = false;  // per instantiation
  if (!configured) {
    TN_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    configured = true;
  }
  const int tiles = p.num_m * p.num_n;
  const int grid = tiles < sm_count() ? tiles : sm_count();
  kern<<<grid, GEMM_THREADS, smem, stream>>>(tm, p);
  TN_CHECK_CUDA(cudaGetLastError());
  return TN_OK;
}

template <bool A_MN, bool B_MN, int EPI>
static int launch_gemm(int bn, const GemmMaps& tm, const GemmParams& p, cudaStream_t stream) {
  return bn == 256 ? launch_gemm<256, A_MN, B_MN, EPI>(tm, p, stream) : launch_gemm<128, A_MN, B_MN, EPI>(tm, p, stream);
}

// Tile width from the shape: a 128x256 tile does the work of two 128x128 tiles in kWideTileCost of the time of one, so
// the wide tile wins unless halving the tile count costs more in the last, partly idle wave than it saves per tile
// (e.g. 3072x3072: 576 narrow tiles in 5 waves vs 288 wide tiles in 3).  `out_div` = accumulator columns per output
// column (2 for SwiGLU).  A pure function of the shape, so equal shapes always get equal tiles.
constexpr double kWideTileCost = 1.8;
static int pick_bn(int M, int N, int out_div) {
  const int64_t sms = sm_count();
  const int64_t nm = (M + BM - 1) / BM;
  const int64_t wide = nm * ((N + 256 / out_div - 1) / (256 / out_div));
  const int64_t narrow = nm * ((N + 128 / out_div - 1) / (128 / out_div));
  const int64_t w_wide = (wide + sms - 1) / sms, w_narrow = (narrow + sms - 1) / sms;
  return double(w_wide) * kWideTileCost <= double(w_narrow) ? 256 : 128;
}

static GemmParams base_params(int M, int N, int K, int tile_n, int kb = BK) {
  GemmParams p{};
  p.M = M; p.N = N; p.K = K;
  p.num_m = (M + BM - 1) / BM;
  p.num_n = (N + tile_n - 1) / tile_n;
  p.num_k = (K + kb - 1) / kb;
  p.n_store = N;
  p.group = gemm_group();
  // L2 policy: inside a raster group the `group` A strips are re-read by every wave, a B strip is consumed within
  // about one wave -> A evict-last, B evict-first (tn_set_gemm_l2_hints; default off)
  p.hint_a = gemm_l2_hints() ? kEvictLast : kEvictNormal;
  p.hint_b = gemm_l2_hints() ? kEvictFirst : kEvictNormal;
  return p;
}

// K-major operand [rows, K] (K contiguous) -> box {64 k, box_rows}; MN-major operand [K, rows] -> box {64 rows, 64 k}
static int map_operand(CUtensorMap* m, const void* ptr, int mn, uint64_t rows, uint64_t K, int64_t ld, uint32_t box_rows) {
  if (!mn) return encode_tmap_2d(m, ptr, 2, K, rows, uint64_t(ld) * 2, 64, box_rows, true);
  return encode_tmap_2d(m, ptr, 2, rows, K, uint64_t(ld) * 2, 64, 64, true);
}

// K-major 8-bit operand [rows, K] (K contiguous, ld bytes) -> box {128 k, box_rows}: the same 128-byte rows
static int map_operand_fp8(CUtensorMap* m, const void* ptr, uint64_t rows, uint64_t K, int64_t ld, uint32_t box_rows) {
  return encode_tmap_2d(m, ptr, 1, K, rows, uint64_t(ld), 128, box_rows, true);
}

// FP8 launches: `op` is gemm_kernel's OP (1-4).  The promoted forms (2, 4) run on the 128 tile, and so do the rowwise
// SwiGLU and fp32-output forms (EPI 1, 2), which spill on the 256 tile: the per-column scales cost registers there.
template <int EPI>
static bool fp8_wide_ok(int op) { return op == 1 || (op == 3 && EPI != 1 && EPI != 2); }
template <int EPI>
static int fp8_bn(int op, int M, int N, int out_div) { return fp8_wide_ok<EPI>(op) ? pick_bn(M, N, out_div) : 128; }

// Rowwise forms exist where an entry point can reach them: the SwiGLU forward (EPI 1) never promotes, the dSwiGLU
// backward (EPI 3) always does.
template <int EPI>
static int launch_fp8(int op, int bn, const GemmMaps& tm, const GemmParams& p, cudaStream_t stream) {
  if (op == 1)
    return bn == 256 ? launch_gemm<256, false, false, EPI, 1>(tm, p, stream)
                     : launch_gemm<128, false, false, EPI, 1>(tm, p, stream);
  if (op == 2) return launch_gemm<128, false, false, EPI, 2>(tm, p, stream);
  if constexpr (EPI != 3) {
    if (op == 3) {
      if constexpr (EPI != 1 && EPI != 2)
        if (bn == 256) return launch_gemm<256, false, false, EPI, 3>(tm, p, stream);
      return launch_gemm<128, false, false, EPI, 3>(tm, p, stream);
    }
  }
  if constexpr (EPI != 1)
    if (op == 4) return launch_gemm<128, false, false, EPI, 4>(tm, p, stream);
  return fail(TN_ERR_UNSUPPORTED, "FP8 GEMM: operand mode %d is not built for epilogue %d", op, EPI);
}

static GemmParams fp8_params(int M, int N, int K, int tile_n, const float* inv_sa, const float* inv_sb) {
  GemmParams p = base_params(M, N, K, tile_n, 2 * BK);
  p.inv_sa = inv_sa; p.inv_sb = inv_sb;
  return p;
}

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// output [rows, cols] (row stride ld elements) -> box of one staging sub-tile: 64 rows x (64 bf16 | 32 fp32) columns
static int map_output(CUtensorMap* m, const void* ptr, int f32, uint64_t rows, uint64_t cols, int64_t ld) {
  return encode_tmap_2d(m, ptr, f32 ? 4 : 2, cols, rows, uint64_t(ld) * (f32 ? 4 : 2), f32 ? 32 : 64, 64, true);
}

}  // namespace tn

using namespace tn;

extern "C" int tn_gemm_bf16(const void* A, int64_t lda, int a_mn, const void* B, int64_t ldb, int b_mn, void* D,
                            int64_t ldd, int d_f32, const void* R, int64_t ldr, int M, int N, int K,
                            tn_stream_t stream_) {
  clear_error();
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  TN_REQUIRE(A && B && D, "tn_gemm_bf16: null pointer");
  TN_REQUIRE(M > 0 && N > 0 && K > 0, "tn_gemm_bf16: empty problem M=%d N=%d K=%d", M, N, K);
  TN_REQUIRE(lda % 8 == 0 && ldb % 8 == 0, "tn_gemm_bf16: lda/ldb must be multiples of 8 elements (16 B)");
  TN_REQUIRE(ldd % (d_f32 ? 4 : 8) == 0 && (!R || ldr % (d_f32 ? 4 : 8) == 0), "tn_gemm_bf16: ldd/ldr alignment");
  TN_REQUIRE((reinterpret_cast<uintptr_t>(D) & 15) == 0 && (!R || (reinterpret_cast<uintptr_t>(R) & 15) == 0),
             "tn_gemm_bf16: D/R must be 16 B aligned");
  TN_REQUIRE(!(a_mn && !b_mn), "tn_gemm_bf16: (a_mn=1, b_mn=0) layout is not instantiated");

  const int bn = pick_bn(M, N, 1);
  GemmParams p = base_params(M, N, K, bn);
  p.R = R; p.ldr = ldr;
  p.n_store = N & ~(d_f32 ? 3 : 7);   // whole 16-byte chunks go out by TMA, the rest by ordinary stores
  p.d = D; p.ldd = ldd;
  GemmMaps tm;
  int rc;
  if ((rc = map_operand(&tm.a, A, a_mn, uint64_t(M), uint64_t(K), lda, BM))) return rc;
  if ((rc = map_operand(&tm.b[0], B, b_mn, uint64_t(N), uint64_t(K), ldb, bn))) return rc;
  if ((rc = map_output(&tm.d[0], D, d_f32, uint64_t(M), uint64_t(p.n_store > 0 ? p.n_store : N), ldd))) return rc;
  tm.b[1] = tm.b[2] = tm.b[0];
  tm.d[1] = tm.d[2] = tm.d[0];

#define TN_GEMM_DISPATCH(AMN_, BMN_)                              \
  (d_f32 ? launch_gemm<AMN_, BMN_, 2>(bn, tm, p, stream)          \
         : launch_gemm<AMN_, BMN_, 0>(bn, tm, p, stream))
  if (!a_mn && !b_mn) return TN_GEMM_DISPATCH(false, false);
  if (!a_mn && b_mn) return TN_GEMM_DISPATCH(false, true);
  return TN_GEMM_DISPATCH(true, true);
#undef TN_GEMM_DISPATCH
}

extern "C" int tn_gemm_swiglu_bf16(const void* X, int64_t ldx, const void* Wg, const void* Wu, int64_t ldw, void* G,
                                   void* U, void* H, int64_t ldh, int M, int N, int K, tn_stream_t stream_) {
  clear_error();
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  TN_REQUIRE(X && Wg && Wu && H, "tn_gemm_swiglu_bf16: null pointer");
  TN_REQUIRE(M > 0 && N > 0 && K > 0, "tn_gemm_swiglu_bf16: empty problem");
  TN_REQUIRE(ldx % 8 == 0 && ldw % 8 == 0 && ldh % 8 == 0, "tn_gemm_swiglu_bf16: leading dims must be multiples of 8");
  TN_REQUIRE((reinterpret_cast<uintptr_t>(H) & 15) == 0 && (!G || (reinterpret_cast<uintptr_t>(G) & 15) == 0) &&
                 (!U || (reinterpret_cast<uintptr_t>(U) & 15) == 0),
             "tn_gemm_swiglu_bf16: outputs must be 16 B aligned");
  const int bn = pick_bn(M, N, 2);
  GemmParams p = base_params(M, N, K, bn / 2);
  p.has_g = G != nullptr; p.has_u = U != nullptr;
  GemmMaps tm;
  int rc;
  if ((rc = map_operand(&tm.a, X, 0, uint64_t(M), uint64_t(K), ldx, BM))) return rc;
  if ((rc = map_operand(&tm.b[0], Wg, 0, uint64_t(N), uint64_t(K), ldw, bn / 2))) return rc;
  if ((rc = map_operand(&tm.b[1], Wu, 0, uint64_t(N), uint64_t(K), ldw, bn / 2))) return rc;
  tm.b[2] = tm.b[1];
  if ((rc = map_output(&tm.d[0], H, 0, uint64_t(M), uint64_t(N), ldh))) return rc;
  tm.d[1] = tm.d[2] = tm.d[0];
  if (G && (rc = map_output(&tm.d[1], G, 0, uint64_t(M), uint64_t(N), ldh))) return rc;
  if (U && (rc = map_output(&tm.d[2], U, 0, uint64_t(M), uint64_t(N), ldh))) return rc;
  return launch_gemm<false, false, 1>(bn, tm, p, stream);
}

// Down-proj dgrad with the SwiGLU backward in its epilogue: dH = dY[M,K].W[K,N] (W = down_proj.weight [d, ffn], MN-major B),
// dG / dU [M,N] from the accumulator and the saved G / U.
extern "C" int tn_gemm_dswiglu_bf16(const void* dY, int64_t lddy, const void* W, int64_t ldw, const void* G, const void* U,
                                    int64_t ldgu, void* dG, void* dU, int64_t lddg, int M, int N, int K,
                                    tn_stream_t stream_) {
  clear_error();
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  TN_REQUIRE(dY && W && G && U && dG && dU, "tn_gemm_dswiglu_bf16: null pointer");
  TN_REQUIRE(M >= 256 && N >= 256 && K > 0, "tn_gemm_dswiglu_bf16: needs M, N >= 256 (use tn_gemm_bf16 + tn_swiglu_bwd_bf16 below that)");
  TN_REQUIRE(lddy % 8 == 0 && ldw % 8 == 0 && ldgu % 8 == 0 && lddg % 8 == 0 && N % 8 == 0,
             "tn_gemm_dswiglu_bf16: leading dims and N must be multiples of 8");
  TN_REQUIRE(((reinterpret_cast<uintptr_t>(G) | reinterpret_cast<uintptr_t>(U) | reinterpret_cast<uintptr_t>(dG) |
               reinterpret_cast<uintptr_t>(dU)) & 15) == 0, "tn_gemm_dswiglu_bf16: G, U, dG, dU must be 16 B aligned");
  const int bn = pick_bn(M, N, 1);   // the tile tn_gemm_bf16 would use for dH
  GemmParams p = base_params(M, N, K, bn);
  p.aux_g = static_cast<const bf16*>(G); p.aux_u = static_cast<const bf16*>(U); p.ld_gu = ldgu;
  GemmMaps tm;
  int rc;
  if ((rc = map_operand(&tm.a, dY, 0, uint64_t(M), uint64_t(K), lddy, BM))) return rc;
  if ((rc = map_operand(&tm.b[0], W, 1, uint64_t(N), uint64_t(K), ldw, bn))) return rc;
  tm.b[1] = tm.b[2] = tm.b[0];
  if ((rc = map_output(&tm.d[0], dG, 0, uint64_t(M), uint64_t(N), lddg))) return rc;
  if ((rc = map_output(&tm.d[1], dU, 0, uint64_t(M), uint64_t(N), lddg))) return rc;
  tm.d[2] = tm.d[1];
  return launch_gemm<false, true, 3>(bn, tm, p, stream);
}

// Three weights / gradients treated as one operand (see GemmParams).  mode: 0 = forward  D[M, n0+n1+n2] = A·[B0;B1;B2]ᵀ
// (B K-major), 1 = dgrad  D[M,N] = [A0|A1|A2]·[B0;B1;B2] (A = one [M, k0+k1+k2] buffer, B MN-major, segmented along K),
// 2 = wgrad  [D0;D1;D2] = Aᵀ·X (A = one [Mred, m0+m1+m2] buffer MN-major, B MN-major, D segmented along M).
extern "C" int tn_gemm_qkv_bf16(int mode, const void* A, int64_t lda, const void* B0, const void* B1, const void* B2,
                                int64_t ldb, void* D0, void* D1, void* D2, int64_t ldd, int d_f32, int s0, int s1, int s2,
                                int M, int N, int K, const void* rope_cos, const void* rope_sin, tn_stream_t stream_) {
  clear_error();
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  TN_REQUIRE(A && B0 && D0, "tn_gemm_qkv_bf16: null pointer");
  TN_REQUIRE(mode >= 0 && mode <= 2, "tn_gemm_qkv_bf16: mode must be 0 (forward), 1 (dgrad) or 2 (wgrad)");
  TN_REQUIRE(s0 > 0 && s1 > 0 && s2 > 0 && s0 % 256 == 0 && s1 % 256 == 0 && s2 % 256 == 0,
             "tn_gemm_qkv_bf16: segment sizes (%d,%d,%d) must be positive multiples of 256", s0, s1, s2);
  const int tot = s0 + s1 + s2;
  TN_REQUIRE((mode == 0 && N == tot) || (mode == 1 && K == tot) || (mode == 2 && M == tot),
             "tn_gemm_qkv_bf16: segments do not add up to the segmented dimension");
  TN_REQUIRE(M >= 256 && N >= 256 && lda % 8 == 0 && ldb % 8 == 0 && ldd % (d_f32 ? 4 : 8) == 0,
             "tn_gemm_qkv_bf16: needs M,N >= 256 and 16-byte aligned leading dimensions");
  TN_REQUIRE(mode == 2 || (B1 && B2), "tn_gemm_qkv_bf16: B1/B2 required");
  TN_REQUIRE(mode != 2 || (D1 && D2), "tn_gemm_qkv_bf16: D1/D2 required for wgrad");
  TN_REQUIRE((rope_cos == nullptr) == (rope_sin == nullptr), "tn_gemm_qkv_bf16: cos and sin tables come in pairs");
  TN_REQUIRE(rope_cos == nullptr || mode == 0, "tn_gemm_qkv_bf16: fused RoPE exists for the forward projection only");
  const void* Bs[3] = {B0, B1, B2};
  const int seg[3] = {s0, s1, s2};
  const int bn = pick_bn(M, N, 1);
  GemmParams p = base_params(M, N, K, bn);
  p.off1 = s0; p.off2 = s0 + s1;
  GemmMaps tm;
  int rc;
  if (mode == 0) {
    if (rope_cos) {
      p.rope_cos = static_cast<const bf16*>(rope_cos); p.rope_sin = static_cast<const bf16*>(rope_sin);
      p.rope_end = s0 + s1;
    }
    p.b_seg = 1;
    if ((rc = map_operand(&tm.a, A, 0, uint64_t(M), uint64_t(K), lda, BM))) return rc;
    for (int i = 0; i < 3; ++i)
      if ((rc = map_operand(&tm.b[i], Bs[i], 0, uint64_t(seg[i]), uint64_t(K), ldb, bn))) return rc;
    if ((rc = map_output(&tm.d[0], D0, 0, uint64_t(M), uint64_t(N), ldd))) return rc;
    tm.d[1] = tm.d[2] = tm.d[0];
    return launch_gemm<false, false, 0>(bn, tm, p, stream);
  }
  if (mode == 1) {
    p.b_seg = 2;
    if ((rc = map_operand(&tm.a, A, 0, uint64_t(M), uint64_t(K), lda, BM))) return rc;
    for (int i = 0; i < 3; ++i)   // B_i stored [seg_i (K), N] row-major, N contiguous
      if ((rc = map_operand(&tm.b[i], Bs[i], 1, uint64_t(N), uint64_t(seg[i]), ldb, bn))) return rc;
    if ((rc = map_output(&tm.d[0], D0, 0, uint64_t(M), uint64_t(N), ldd))) return rc;
    tm.d[1] = tm.d[2] = tm.d[0];
    return launch_gemm<false, true, 0>(bn, tm, p, stream);
  }
  p.d_seg = 1;
  void* Ds[3] = {D0, D1, D2};
  if ((rc = map_operand(&tm.a, A, 1, uint64_t(M), uint64_t(K), lda, BM))) return rc;
  if ((rc = map_operand(&tm.b[0], B0, 1, uint64_t(N), uint64_t(K), ldb, bn))) return rc;
  tm.b[1] = tm.b[2] = tm.b[0];
  for (int i = 0; i < 3; ++i)   // one map per gradient tensor [seg_i, N]
    if ((rc = map_output(&tm.d[i], Ds[i], d_f32, uint64_t(seg[i]), uint64_t(N), ldd))) return rc;
  return d_f32 ? launch_gemm<true, true, 2>(bn, tm, p, stream) : launch_gemm<true, true, 0>(bn, tm, p, stream);
}

// ---------------------------------------------------------------------------------------------------------------
// FP8 twins of the entry points above: K-major 8-bit operands, outputs and epilogues as in the bf16 entry points.
// Tensorwise (tn_*_fp8): A e4m3, or e5m2 with a_e5m2 (promoted accumulation); B e4m3; 1/s_a and 1/s_b are single
// device floats (tn_fp8_cast_bf16).  Rowwise (tn_*_fp8_rowwise): A and B e4m3, 1/s_a and 1/s_b are device vectors
// over the rows of A and of B (tn_fp8_rowwise_cast_bf16, tn_fp8_colwise_cast_t_bf16).  Every dimension and leading
// dimension is a multiple of 16 (TMA rows of 8-bit elements are 16-byte aligned).
// ---------------------------------------------------------------------------------------------------------------
#define TN_FP8_REQUIRE_COMMON(name, A, lda, B, ldb, inv_sa, inv_sb, M, N, K)                                          \
  TN_REQUIRE(A && B && inv_sa && inv_sb, "%s: null pointer", name);                                                 \
  TN_REQUIRE(M > 0 && N > 0 && K > 0 && M % 16 == 0 && N % 16 == 0 && K % 16 == 0,                                   \
             "%s: M=%d N=%d K=%d must be positive multiples of 16", name, M, N, K);                                   \
  TN_REQUIRE(lda % 16 == 0 && ldb % 16 == 0 && aligned16(A) && aligned16(B),                                        \
             "%s: A and B must be 16 B aligned with leading dims that are multiples of 16", name)
// rowwise scale vectors are read in pairs
#define TN_FP8_REQUIRE_VEC(name, v) \
  TN_REQUIRE((reinterpret_cast<uintptr_t>(v) & 7) == 0, "%s: scale vectors must be 8 B aligned", name)

static int gemm_fp8(const char* name, int op, const void* A, int64_t lda, const void* B, int64_t ldb, void* D,
                    int64_t ldd, int d_f32, const void* R, int64_t ldr, int M, int N, int K, const float* inv_sa,
                    const float* inv_sb, cudaStream_t stream) {
  TN_REQUIRE(D, "%s: null pointer", name);
  TN_FP8_REQUIRE_COMMON(name, A, lda, B, ldb, inv_sa, inv_sb, M, N, K);
  TN_REQUIRE(ldd % (d_f32 ? 4 : 8) == 0 && (!R || ldr % (d_f32 ? 4 : 8) == 0), "%s: ldd/ldr alignment", name);
  TN_REQUIRE(aligned16(D) && (!R || aligned16(R)), "%s: D/R must be 16 B aligned", name);
  if (op >= 3) { TN_FP8_REQUIRE_VEC(name, inv_sa); TN_FP8_REQUIRE_VEC(name, inv_sb); }
  const int bn = d_f32 ? fp8_bn<2>(op, M, N, 1) : fp8_bn<0>(op, M, N, 1);
  GemmParams p = fp8_params(M, N, K, bn, inv_sa, inv_sb);
  p.R = R; p.ldr = ldr;
  GemmMaps tm;
  int rc;
  if ((rc = map_operand_fp8(&tm.a, A, uint64_t(M), uint64_t(K), lda, BM))) return rc;
  if ((rc = map_operand_fp8(&tm.b[0], B, uint64_t(N), uint64_t(K), ldb, bn))) return rc;
  if ((rc = map_output(&tm.d[0], D, d_f32, uint64_t(M), uint64_t(N), ldd))) return rc;
  tm.b[1] = tm.b[2] = tm.b[0];
  tm.d[1] = tm.d[2] = tm.d[0];
  return d_f32 ? launch_fp8<2>(op, bn, tm, p, stream) : launch_fp8<0>(op, bn, tm, p, stream);
}

static int gemm_swiglu_fp8(const char* name, int op, const void* X, int64_t ldx, const void* Wg, const void* Wu,
                           int64_t ldw, void* G, void* U, void* H, int64_t ldh, int M, int N, int K, const float* inv_sx,
                           const float* inv_sw, cudaStream_t stream) {
  TN_REQUIRE(Wu && H, "%s: null pointer", name);
  TN_FP8_REQUIRE_COMMON(name, X, ldx, Wg, ldw, inv_sx, inv_sw, M, N, K);
  TN_REQUIRE(ldh % 8 == 0 && aligned16(Wu), "%s: ldh must be a multiple of 8, Wu 16 B aligned", name);
  TN_REQUIRE(aligned16(H) && (!G || aligned16(G)) && (!U || aligned16(U)), "%s: outputs must be 16 B aligned", name);
  if (op >= 3) { TN_FP8_REQUIRE_VEC(name, inv_sx); TN_FP8_REQUIRE_VEC(name, inv_sw); }
  const int bn = fp8_bn<1>(op, M, N, 2);
  GemmParams p = fp8_params(M, N, K, bn / 2, inv_sx, inv_sw);
  p.has_g = G != nullptr; p.has_u = U != nullptr;
  GemmMaps tm;
  int rc;
  if ((rc = map_operand_fp8(&tm.a, X, uint64_t(M), uint64_t(K), ldx, BM))) return rc;
  if ((rc = map_operand_fp8(&tm.b[0], Wg, uint64_t(N), uint64_t(K), ldw, bn / 2))) return rc;
  if ((rc = map_operand_fp8(&tm.b[1], Wu, uint64_t(N), uint64_t(K), ldw, bn / 2))) return rc;
  tm.b[2] = tm.b[1];
  if ((rc = map_output(&tm.d[0], H, 0, uint64_t(M), uint64_t(N), ldh))) return rc;
  tm.d[1] = tm.d[2] = tm.d[0];
  if (G && (rc = map_output(&tm.d[1], G, 0, uint64_t(M), uint64_t(N), ldh))) return rc;
  if (U && (rc = map_output(&tm.d[2], U, 0, uint64_t(M), uint64_t(N), ldh))) return rc;
  return launch_fp8<1>(op, bn, tm, p, stream);
}

static int gemm_dswiglu_fp8(const char* name, int op, const void* dY, int64_t lddy, const void* W, int64_t ldw,
                            const void* G, const void* U, int64_t ldgu, void* dG, void* dU, int64_t lddg, int M, int N,
                            int K, const float* inv_sa, const float* inv_sb, cudaStream_t stream) {
  TN_REQUIRE(G && U && dG && dU, "%s: null pointer", name);
  TN_FP8_REQUIRE_COMMON(name, dY, lddy, W, ldw, inv_sa, inv_sb, M, N, K);
  TN_REQUIRE(M >= 256 && N >= 256, "%s: needs M, N >= 256", name);
  TN_REQUIRE(ldgu % 8 == 0 && lddg % 8 == 0, "%s: ldgu and lddg must be multiples of 8", name);
  TN_REQUIRE(aligned16(G) && aligned16(U) && aligned16(dG) && aligned16(dU), "%s: G, U, dG, dU must be 16 B aligned",
             name);
  if (op >= 3) { TN_FP8_REQUIRE_VEC(name, inv_sa); TN_FP8_REQUIRE_VEC(name, inv_sb); }
  const int bn = fp8_bn<3>(op, M, N, 1);
  GemmParams p = fp8_params(M, N, K, bn, inv_sa, inv_sb);
  p.aux_g = static_cast<const bf16*>(G); p.aux_u = static_cast<const bf16*>(U); p.ld_gu = ldgu;
  GemmMaps tm;
  int rc;
  if ((rc = map_operand_fp8(&tm.a, dY, uint64_t(M), uint64_t(K), lddy, BM))) return rc;
  if ((rc = map_operand_fp8(&tm.b[0], W, uint64_t(N), uint64_t(K), ldw, bn))) return rc;
  tm.b[1] = tm.b[2] = tm.b[0];
  if ((rc = map_output(&tm.d[0], dG, 0, uint64_t(M), uint64_t(N), lddg))) return rc;
  if ((rc = map_output(&tm.d[1], dU, 0, uint64_t(M), uint64_t(N), lddg))) return rc;
  tm.d[2] = tm.d[1];
  return launch_fp8<3>(op, bn, tm, p, stream);
}

// `op_fwd` is the OP of mode 0, `op_bwd` that of modes 1 and 2
static int gemm_qkv_fp8(const char* name, int op_fwd, int op_bwd, int mode, const void* A, int64_t lda,
                        const void* B0, const void* B1, const void* B2, int64_t ldb, void* D0, void* D1, void* D2,
                        int64_t ldd, int d_f32, int s0, int s1, int s2, int M, int N, int K, const void* rope_cos,
                        const void* rope_sin, const float* inv_sa, const float* inv_sb, cudaStream_t stream) {
  TN_REQUIRE(D0, "%s: null pointer", name);
  TN_FP8_REQUIRE_COMMON(name, A, lda, B0, ldb, inv_sa, inv_sb, M, N, K);
  TN_REQUIRE(mode >= 0 && mode <= 2, "%s: mode must be 0 (forward), 1 (dgrad) or 2 (wgrad)", name);
  TN_REQUIRE(s0 > 0 && s1 > 0 && s2 > 0 && s0 % 256 == 0 && s1 % 256 == 0 && s2 % 256 == 0,
             "%s: segment sizes (%d,%d,%d) must be positive multiples of 256", name, s0, s1, s2);
  const int tot = s0 + s1 + s2;
  TN_REQUIRE((mode == 0 && N == tot) || (mode == 1 && K == tot) || (mode == 2 && M == tot),
             "%s: segments do not add up to the segmented dimension", name);
  TN_REQUIRE(M >= 256 && N >= 256 && ldd % (d_f32 ? 4 : 8) == 0,
             "%s: needs M,N >= 256 and 16-byte aligned leading dimensions", name);
  TN_REQUIRE(mode == 2 || (B1 && B2 && aligned16(B1) && aligned16(B2)), "%s: B1/B2 required, 16 B aligned", name);
  TN_REQUIRE(mode != 2 || (D1 && D2), "%s: D1/D2 required for wgrad", name);
  TN_REQUIRE((rope_cos == nullptr) == (rope_sin == nullptr), "%s: cos and sin tables come in pairs", name);
  TN_REQUIRE(rope_cos == nullptr || mode == 0, "%s: fused RoPE exists for the forward projection only", name);
  const int op = mode == 0 ? op_fwd : op_bwd;
  if (op >= 3) { TN_FP8_REQUIRE_VEC(name, inv_sa); TN_FP8_REQUIRE_VEC(name, inv_sb); }
  const void* Bs[3] = {B0, B1, B2};
  const int seg[3] = {s0, s1, s2};
  const int bn = mode == 2 && d_f32 ? fp8_bn<2>(op, M, N, 1) : fp8_bn<0>(op, M, N, 1);
  GemmParams p = fp8_params(M, N, K, bn, inv_sa, inv_sb);
  p.off1 = s0; p.off2 = s0 + s1;
  GemmMaps tm;
  int rc;
  if ((rc = map_operand_fp8(&tm.a, A, uint64_t(M), uint64_t(K), lda, BM))) return rc;
  if (mode == 2) {
    p.d_seg = 1;
    void* Ds[3] = {D0, D1, D2};
    if ((rc = map_operand_fp8(&tm.b[0], B0, uint64_t(N), uint64_t(K), ldb, bn))) return rc;
    tm.b[1] = tm.b[2] = tm.b[0];
    for (int i = 0; i < 3; ++i)
      if ((rc = map_output(&tm.d[i], Ds[i], d_f32, uint64_t(seg[i]), uint64_t(N), ldd))) return rc;
    return d_f32 ? launch_fp8<2>(op, bn, tm, p, stream) : launch_fp8<0>(op, bn, tm, p, stream);
  }
  if (mode == 0) {
    if (rope_cos) {
      p.rope_cos = static_cast<const bf16*>(rope_cos); p.rope_sin = static_cast<const bf16*>(rope_sin);
      p.rope_end = s0 + s1;
    }
    p.b_seg = 1;
    for (int i = 0; i < 3; ++i)
      if ((rc = map_operand_fp8(&tm.b[i], Bs[i], uint64_t(seg[i]), uint64_t(K), ldb, bn))) return rc;
  } else {
    p.b_seg = 2;
    for (int i = 0; i < 3; ++i)
      if ((rc = map_operand_fp8(&tm.b[i], Bs[i], uint64_t(N), uint64_t(seg[i]), ldb, bn))) return rc;
  }
  TN_REQUIRE(!d_f32, "%s: modes 0 and 1 write bf16", name);
  if ((rc = map_output(&tm.d[0], D0, 0, uint64_t(M), uint64_t(N), ldd))) return rc;
  tm.d[1] = tm.d[2] = tm.d[0];
  return launch_fp8<0>(op, bn, tm, p, stream);
}
#undef TN_FP8_REQUIRE_VEC
#undef TN_FP8_REQUIRE_COMMON

extern "C" int tn_gemm_fp8(const void* A, int64_t lda, int a_e5m2, const void* B, int64_t ldb, void* D, int64_t ldd,
                           int d_f32, const void* R, int64_t ldr, int M, int N, int K, const float* inv_sa,
                           const float* inv_sb, tn_stream_t stream_) {
  clear_error();
  return gemm_fp8("tn_gemm_fp8", a_e5m2 ? 2 : 1, A, lda, B, ldb, D, ldd, d_f32, R, ldr, M, N, K, inv_sa, inv_sb,
                  static_cast<cudaStream_t>(stream_));
}

extern "C" int tn_gemm_swiglu_fp8(const void* X, int64_t ldx, int x_e5m2, const void* Wg, const void* Wu, int64_t ldw,
                                  void* G, void* U, void* H, int64_t ldh, int M, int N, int K, const float* inv_sx,
                                  const float* inv_sw, tn_stream_t stream_) {
  clear_error();
  return gemm_swiglu_fp8("tn_gemm_swiglu_fp8", x_e5m2 ? 2 : 1, X, ldx, Wg, Wu, ldw, G, U, H, ldh, M, N, K, inv_sx,
                         inv_sw, static_cast<cudaStream_t>(stream_));
}

// W is the K-major transposed copy of down_proj.weight: [N = ffn, K = d]
extern "C" int tn_gemm_dswiglu_fp8(const void* dY, int64_t lddy, int dy_e5m2, const void* W, int64_t ldw, const void* G,
                                   const void* U, int64_t ldgu, void* dG, void* dU, int64_t lddg, int M, int N, int K,
                                   const float* inv_sa, const float* inv_sb, tn_stream_t stream_) {
  clear_error();
  return gemm_dswiglu_fp8("tn_gemm_dswiglu_fp8", dy_e5m2 ? 2 : 1, dY, lddy, W, ldw, G, U, ldgu, dG, dU, lddg, M, N, K,
                          inv_sa, inv_sb, static_cast<cudaStream_t>(stream_));
}

// Modes as tn_gemm_qkv_bf16, all operands K-major: 1 = dgrad with B_i the [N, s_i] column blocks of Wᵀ (row stride
// ldb), 2 = wgrad with A = the transposed gradient [s0+s1+s2, K] and B0 = the transposed layer input [N, K].
extern "C" int tn_gemm_qkv_fp8(int mode, const void* A, int64_t lda, int a_e5m2, const void* B0, const void* B1,
                               const void* B2, int64_t ldb, void* D0, void* D1, void* D2, int64_t ldd, int d_f32, int s0,
                               int s1, int s2, int M, int N, int K, const void* rope_cos, const void* rope_sin,
                               const float* inv_sa, const float* inv_sb, tn_stream_t stream_) {
  clear_error();
  const int op = a_e5m2 ? 2 : 1;
  return gemm_qkv_fp8("tn_gemm_qkv_fp8", op, op, mode, A, lda, B0, B1, B2, ldb, D0, D1, D2, ldd, d_f32, s0, s1, s2, M,
                      N, K, rope_cos, rope_sin, inv_sa, inv_sb, static_cast<cudaStream_t>(stream_));
}

// Rowwise: inv_sa [M] and inv_sb [N] (SwiGLU: inv_sw [2N], the gate rows then the up rows; QKV mode 0: inv_sb over the
// rows of [Wq;Wk;Wv], N long).  `promoted` selects the separate fp32 accumulator (dgrad, wgrad); the dSwiGLU GEMM and
// QKV modes 1 and 2 always promote, the SwiGLU GEMM and QKV mode 0 never do.
extern "C" int tn_gemm_fp8_rowwise(const void* A, int64_t lda, const void* B, int64_t ldb, void* D, int64_t ldd,
                                   int d_f32, const void* R, int64_t ldr, int M, int N, int K, const float* inv_sa,
                                   const float* inv_sb, int promoted, tn_stream_t stream_) {
  clear_error();
  return gemm_fp8("tn_gemm_fp8_rowwise", promoted ? 4 : 3, A, lda, B, ldb, D, ldd, d_f32, R, ldr, M, N, K, inv_sa,
                  inv_sb, static_cast<cudaStream_t>(stream_));
}

extern "C" int tn_gemm_swiglu_fp8_rowwise(const void* X, int64_t ldx, const void* Wg, const void* Wu, int64_t ldw,
                                          void* G, void* U, void* H, int64_t ldh, int M, int N, int K,
                                          const float* inv_sx, const float* inv_sw, tn_stream_t stream_) {
  clear_error();
  return gemm_swiglu_fp8("tn_gemm_swiglu_fp8_rowwise", 3, X, ldx, Wg, Wu, ldw, G, U, H, ldh, M, N, K, inv_sx, inv_sw,
                         static_cast<cudaStream_t>(stream_));
}

extern "C" int tn_gemm_dswiglu_fp8_rowwise(const void* dY, int64_t lddy, const void* W, int64_t ldw, const void* G,
                                           const void* U, int64_t ldgu, void* dG, void* dU, int64_t lddg, int M, int N,
                                           int K, const float* inv_sa, const float* inv_sb, tn_stream_t stream_) {
  clear_error();
  return gemm_dswiglu_fp8("tn_gemm_dswiglu_fp8_rowwise", 4, dY, lddy, W, ldw, G, U, ldgu, dG, dU, lddg, M, N, K,
                          inv_sa, inv_sb, static_cast<cudaStream_t>(stream_));
}

extern "C" int tn_gemm_qkv_fp8_rowwise(int mode, const void* A, int64_t lda, const void* B0, const void* B1,
                                       const void* B2, int64_t ldb, void* D0, void* D1, void* D2, int64_t ldd, int d_f32,
                                       int s0, int s1, int s2, int M, int N, int K, const void* rope_cos,
                                       const void* rope_sin, const float* inv_sa, const float* inv_sb,
                                       tn_stream_t stream_) {
  clear_error();
  return gemm_qkv_fp8("tn_gemm_qkv_fp8_rowwise", 3, 4, mode, A, lda, B0, B1, B2, ldb, D0, D1, D2, ldd, d_f32, s0, s1,
                      s2, M, N, K, rope_cos, rope_sin, inv_sa, inv_sb, static_cast<cudaStream_t>(stream_));
}
