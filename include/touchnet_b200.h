/* touchnet_b200 — C ABI of the H100-native (sm_90a) TouchNet hot path.
 *
 * This header is the drop-in boundary: every entry point replaces one third-party kernel call site that the
 * reference (xingchensong/TouchNet) reaches from Python.  "Reference interface" below names the reference
 * file:line the call replaces (paths relative to the TouchNet checkout; `hf:` = transformers 4.51.3,
 * `ta:` = torchaudio).
 *
 * Conventions
 *   - all pointers are DEVICE pointers owned by the caller (PyTorch caching allocator); kernels never allocate
 *     and never synchronise; work is enqueued on `stream` (a cudaStream_t / CUstream; NULL = legacy default).
 *   - bf16 tensors are row-major with explicit leading dimensions (in elements).
 *   - return value 0 = success; non-zero = error, message via tn_last_error() (thread-local).
 *   - entry points are re-entrant and stream-ordered (FSDP2 side streams, activation-checkpoint recompute and the
 *     autograd device thread may all call concurrently on different streams).
 */
#ifndef TOUCHNET_B200_H
#define TOUCHNET_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TOUCHNET_B200_VERSION 100

typedef void* tn_stream_t; /* cudaStream_t */

const char* tn_last_error(void);
int tn_version(void);
/* 0 iff the current CUDA device is compute capability 9.0 (H100). */
int tn_device_check(void);
/* Persistent kernels (the GEMMs) launch one CTA per SM; under FSDP2 the NCCL all-gather / reduce-scatter kernels of the
 * neighbouring layers need SMs of their own to overlap with them.  Leave `sms` SMs unused by persistent grids
 * (0 = default, single GPU).  Process-wide. */
int tn_set_sm_margin(int sms);
/* Tuning knob: raster group of the GEMM = number of 128-row M blocks whose tiles are walked across all N blocks before
 * moving on (default 8; decides which operand strips stay L2-resident between waves).  Results do not depend on it. */
int tn_set_gemm_group(int m_blocks);
int tn_set_gemm_split_tail(int on);  /* accepted for API compatibility; the GEMM has no half-tile tail mode */
int tn_set_gemm_l2_hints(int on);   /* 1: A strips evict-last, B strips evict-first in the GEMM's TMA loads (default 0) */

/* ---------------------------------------------------------------------------------------------------------------
 * GEMM  D[M,N] = A·Bᵀ (+ R)          wgmma / TMA, bf16 in, fp32 accumulate.
 *   a_mn = 0: A stored [M,K] (K contiguous, lda)      a_mn = 1: A stored [K,M] (M contiguous, lda)
 *   b_mn = 0: B stored [N,K] (K contiguous, ldb)      b_mn = 1: B stored [K,N] (N contiguous, ldb)
 *   d_f32 = 0: D (and R) bf16;  d_f32 = 1: D (and R) fp32.  R optional (NULL), may alias D (accumulate).
 *   forward  y = x·Wᵀ      : a_mn=0, b_mn=0   (F.linear; hf:models/llama/modeling_llama.py:251-289 q/k/v/o_proj,
 *                                               :182-184 down_proj; touchnet/models/touch_audio/modeling_touch_audio.py:127 projector)
 *   dgrad    dx = dy·W     : a_mn=0, b_mn=1
 *   wgrad    dW = dyᵀ·x    : a_mn=1, b_mn=1
 */
int tn_gemm_bf16(const void* A, int64_t lda, int a_mn, const void* B, int64_t ldb, int b_mn, void* D, int64_t ldd,
                 int d_f32, const void* R, int64_t ldr, int M, int N, int K, tn_stream_t stream);

/* Fused gate/up projection + SwiGLU:  G = X·Wgᵀ, U = X·Wuᵀ, H = silu(G)⊙U   (all bf16, [M,N]; X [M,K]; Wg,Wu [N,K]).
 * G and U may be NULL (inference: only H is written).
 * Reference interface: hf:models/llama/modeling_llama.py:182-184 LlamaMLP.forward (gate_proj, up_proj, act_fn, mul). */
int tn_gemm_swiglu_bf16(const void* X, int64_t ldx, const void* Wg, const void* Wu, int64_t ldw, void* G, void* U,
                        void* H, int64_t ldh, int M, int N, int K, tn_stream_t stream);

/* q/k/v projections as ONE launch although the three weights stay separate parameters (HF FQNs, FSDP2, DCP):
 *   mode 0 forward  D0[M, s0+s1+s2] = A[M,K] · [B0;B1;B2]ᵀ         (B_i [s_i, K]; q|k|v land side by side in one buffer)
 *   mode 1 dgrad    D0[M, N]        = A[M, s0+s1+s2] · [B0;B1;B2]   (A = dq|dk|dv side by side; B_i [s_i, N])
 *   mode 2 wgrad    D_i[s_i, N]     = A[:, seg_i]ᵀ · B0[Mred=K, N]  (A = dq|dk|dv [K, s0+s1+s2]; B0 = layer input x)
 * Segment sizes must be multiples of 256.  hf:models/llama/modeling_llama.py:251-289 (q_proj, k_proj, v_proj).
 * mode 0 with rope_cos/rope_sin ([M, 64] bf16 tables of tn_rope_table): the epilogue also applies RoPE to the q and k
 * segments (hf apply_rotary_pos_emb :151-168) with the rounding points of the unfused bf16 ops (bit-identical). */
/* Down-proj dgrad fused with the SwiGLU backward (hf LlamaMLP.forward modeling_llama.py:182-184, backward of
 * `down(silu(gate) * up)`): dH = dY[M,K] . W[K,N] (W = down_proj.weight, [d, ffn] row-major) never leaves the chip -
 * the epilogue turns the accumulator tile into dG = (dH*U)*silu'(G) and dU = dH*silu(G) with the rounding points of
 * tn_gemm_bf16 + tn_swiglu_bwd_bf16 (bit-identical to that two-kernel path).  Needs M, N >= 256. */
int tn_gemm_dswiglu_bf16(const void* dY, int64_t lddy, const void* W, int64_t ldw, const void* G, const void* U,
                         int64_t ldgu, void* dG, void* dU, int64_t lddg, int M, int N, int K, tn_stream_t stream);
int tn_gemm_qkv_bf16(int mode, const void* A, int64_t lda, const void* B0, const void* B1, const void* B2, int64_t ldb,
                     void* D0, void* D1, void* D2, int64_t ldd, int d_f32, int s0, int s1, int s2, int M, int N, int K,
                     const void* rope_cos, const void* rope_sin, tn_stream_t stream);

/* FP8 twins of the four GEMM entry points above (torchao's tensorwise recipe, opt-in through the model config key
 * `float8_training`).  Same arguments without the *_mn flags: every operand is K-major 8-bit (A e4m3, or e5m2 when
 * a_e5m2 / x_e5m2 / dy_e5m2 is set; B always e4m3), and two device floats 1/s_a, 1/s_b (tn_fp8_cast_bf16) multiply the
 * fp32 accumulator ahead of the epilogue.  An e4m3 A (forward) accumulates in the tensor-core accumulator alone; an e5m2
 * A (dgrad, wgrad) adds each 128-k partial sum into a separate fp32 accumulator.  All dimensions and leading dimensions
 * are multiples of 16.
 *   tn_gemm_fp8        : D[M,N] = A[M,K]·B[N,K]ᵀ (+R), bf16 or fp32 D.
 *   tn_gemm_swiglu_fp8 : G, U, H of tn_gemm_swiglu_bf16 from X[M,K] and Wg, Wu [N,K].
 *   tn_gemm_dswiglu_fp8: dG, dU of tn_gemm_dswiglu_bf16; W = the transposed down_proj weight [N = ffn, K = d].
 *   tn_gemm_qkv_fp8    : modes of tn_gemm_qkv_bf16.  Mode 1: B_i = [N, s_i] column blocks of Wᵀ = [Wq;Wk;Wv]ᵀ
 *                        (row stride ldb).  Mode 2: A = the transposed gradient [s0+s1+s2, K], B0 = the transposed
 *                        layer input [N, K]. */
int tn_gemm_fp8(const void* A, int64_t lda, int a_e5m2, const void* B, int64_t ldb, void* D, int64_t ldd, int d_f32,
                const void* R, int64_t ldr, int M, int N, int K, const float* inv_sa, const float* inv_sb,
                tn_stream_t stream);
int tn_gemm_swiglu_fp8(const void* X, int64_t ldx, int x_e5m2, const void* Wg, const void* Wu, int64_t ldw, void* G,
                       void* U, void* H, int64_t ldh, int M, int N, int K, const float* inv_sx, const float* inv_sw,
                       tn_stream_t stream);
int tn_gemm_dswiglu_fp8(const void* dY, int64_t lddy, int dy_e5m2, const void* W, int64_t ldw, const void* G,
                        const void* U, int64_t ldgu, void* dG, void* dU, int64_t lddg, int M, int N, int K,
                        const float* inv_sa, const float* inv_sb, tn_stream_t stream);
int tn_gemm_qkv_fp8(int mode, const void* A, int64_t lda, int a_e5m2, const void* B0, const void* B1, const void* B2,
                    int64_t ldb, void* D0, void* D1, void* D2, int64_t ldd, int d_f32, int s0, int s1, int s2, int M,
                    int N, int K, const void* rope_cos, const void* rope_sin, const float* inv_sa, const float* inv_sb,
                    tn_stream_t stream);

/* Dynamic per-tensor FP8 scaling (bf16 [rows, cols] views, rows and cols multiples of 16):
 *   tn_fp8_amax_bf16: *amax = max(*amax, max|x|) (atomic; the caller zeroes it; several calls share one amax).
 *   tn_fp8_cast_bf16: s = fmax / max(*amax, 1e-12) (fmax 448 e4m3, 57344 e5m2 with e5m2 = 1); out = sat_rne(x·s)
 *                     row-major [rows, cols] and/or out_t = its transpose [cols, rows] (either may be NULL); *inv_scale
 *                     = 1/s if inv_scale is not NULL.  NaN stays NaN. */
int tn_fp8_amax_bf16(const void* x, int64_t ldx, int64_t rows, int64_t cols, float* amax, tn_stream_t stream);
int tn_fp8_cast_bf16(const void* x, int64_t ldx, int64_t rows, int64_t cols, int e5m2, const float* amax, void* out,
                     int64_t ld_out, void* out_t, int64_t ld_out_t, float* inv_scale, tn_stream_t stream);

/* Rowwise FP8 (torchao's rowwise recipe, opt-in through the model config key `float8_recipe_name`): e4m3 operands with
 * one power-of-two scale per row along the GEMM's reduction axis, s = 2^floor(log2(448 / max(amax, 1e-12))) with the
 * division in fp64 and the result in fp32.  bf16 [rows, cols] views, rows and cols multiples of 16; NaN stays NaN.
 *   tn_fp8_rowwise_cast_bf16  : out = sat_rne(x · s_row) row-major [rows, cols], inv_scale[rows] = 1/s_row.
 *   tn_fp8_colwise_amax_bf16  : amax[c] = max(amax[c], max_r |x[r,c]|) (atomic; the caller zeroes amax[cols]; several
 *                               calls share one vector).
 *   tn_fp8_colwise_cast_t_bf16: out_t = sat_rne(x · s_col)ᵀ [cols, rows] with s_col from amax[cols]; inv_scale[cols] =
 *                               1/s_col if inv_scale is not NULL.
 * GEMMs: as the tensorwise twins with A and B e4m3 and 1/s vectors over the rows of A (inv_sa [M]) and of B (inv_sb
 * [N]; SwiGLU: inv_sw [2N], the gate rows then the up rows; QKV mode 0: over the rows of [Wq;Wk;Wv]).  Each accumulator
 * element is multiplied with the 1/s of its row and column.  tn_gemm_fp8_rowwise accumulates in the tensor-core
 * accumulator, or with `promoted` in a separate fp32 accumulator per 128-k stage; dSwiGLU and QKV modes 1 and 2 always
 * promote, SwiGLU and QKV mode 0 never do.  Scale vectors are 8 B aligned. */
int tn_fp8_rowwise_cast_bf16(const void* x, int64_t ldx, int64_t rows, int64_t cols, void* out, int64_t ld_out,
                             float* inv_scale, tn_stream_t stream);
int tn_fp8_colwise_amax_bf16(const void* x, int64_t ldx, int64_t rows, int64_t cols, float* amax, tn_stream_t stream);
int tn_fp8_colwise_cast_t_bf16(const void* x, int64_t ldx, int64_t rows, int64_t cols, const float* amax, void* out_t,
                               int64_t ld_out_t, float* inv_scale, tn_stream_t stream);
int tn_gemm_fp8_rowwise(const void* A, int64_t lda, const void* B, int64_t ldb, void* D, int64_t ldd, int d_f32,
                        const void* R, int64_t ldr, int M, int N, int K, const float* inv_sa, const float* inv_sb,
                        int promoted, tn_stream_t stream);
int tn_gemm_swiglu_fp8_rowwise(const void* X, int64_t ldx, const void* Wg, const void* Wu, int64_t ldw, void* G,
                               void* U, void* H, int64_t ldh, int M, int N, int K, const float* inv_sx,
                               const float* inv_sw, tn_stream_t stream);
int tn_gemm_dswiglu_fp8_rowwise(const void* dY, int64_t lddy, const void* W, int64_t ldw, const void* G, const void* U,
                                int64_t ldgu, void* dG, void* dU, int64_t lddg, int M, int N, int K,
                                const float* inv_sa, const float* inv_sb, tn_stream_t stream);
int tn_gemm_qkv_fp8_rowwise(int mode, const void* A, int64_t lda, const void* B0, const void* B1, const void* B2,
                            int64_t ldb, void* D0, void* D1, void* D2, int64_t ldd, int d_f32, int s0, int s1, int s2,
                            int M, int N, int K, const void* rope_cos, const void* rope_sin, const float* inv_sa,
                            const float* inv_sb, tn_stream_t stream);

/* Skinny-M rowwise FP8 GEMM for cached decode steps: D[M,N] = X[M,K]·Wᵀ with X bf16 and W e4m3 rows as
 * tn_fp8_rowwise_cast_bf16 writes them (inv_sw their 1/s).  The kernel quantises each row of X with that cast's rule (the
 * same power-of-two scale and sat_rne bytes) and accumulates over K in a fixed order, so each element of D depends only
 * on its row of X, W, inv_sw and R[m,n]: not on M, the row's position or the other rows.  Epilogues in the rounding
 * order of the rowwise wgmma GEMMs: epi 0 D = bf16(acc·1/s_x·1/s_w); epi 1 D = bf16(that + R) (R bf16 [M,N], ldr);
 * epi 2 (SwiGLU) W = [Wg;Wu] (2N rows, inv_sw [2N] stacked the same way), D = H = silu(G)⊙U as
 * tn_gemm_swiglu_fp8_rowwise computes it, G and U not stored.  Any M >= 1; N and K multiples of 16; ldw a multiple of
 * 16.  Allocates nothing and never syncs the host (graph-capturable). */
int tn_gemm_fp8_decode(const void* X, int64_t ldx, const void* W, int64_t ldw, const float* inv_sw, int epi,
                       const void* R, int64_t ldr, void* D, int64_t ldd, int M, int N, int K, tn_stream_t stream);

/* SwiGLU backward (elementwise): dG = dH⊙U⊙silu'(G), dU = dH⊙silu(G).  bf16 [M,N] contiguous rows (ld). */
int tn_swiglu_bwd_bf16(const void* G, const void* U, const void* dH, void* dG, void* dU, int64_t rows, int64_t cols,
                       int64_t ld, tn_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------------
 * RMSNorm (+ fused residual add).   hf:models/llama/modeling_llama.py:62-67 LlamaRMSNorm.forward and the residual
 * adds of LlamaDecoderLayer.forward :303-333.
 *   fwd: if R != NULL: S = X + R (bf16, written to S_out if non-NULL) else S = X;
 *        Y = w ⊙ bf16(S · rsqrt(mean(S²)+eps));  rstd[row] (fp32) saved for backward.
 *   bwd: dS = rstd·(w⊙dY) − rstd³/d · S · Σ(w⊙dY⊙S)  (+ dS_extra if non-NULL: gradient flowing through the residual
 *        branch), dW_partial[num_partials, d] fp32 partial sums (workspace; num_partials = tn_rmsnorm_bwd_num_partials())
 *        and, if dW != NULL, dW[d] = their column sums in a fixed order (a second, tiny kernel on the same stream).
 */
int tn_rmsnorm_fwd_bf16(const void* X, const void* R, const void* w, int w_is_f32, void* S_out, void* Y, float* rstd,
                        int64_t rows, int d, float eps, tn_stream_t stream);
int tn_rmsnorm_bwd_bf16(const void* S, const void* dY, const void* dS_extra, const void* w, int w_is_f32,
                        const float* rstd, void* dS, float* dW_partial, int num_partials, float* dW, int64_t rows, int d,
                        tn_stream_t stream);
int tn_rmsnorm_bwd_num_partials(void);

/* ---------------------------------------------------------------------------------------------------------------
 * RoPE.  hf:models/llama/modeling_llama.py:124-168 (LlamaRotaryEmbedding.forward + apply_rotary_pos_emb), called at
 * touchnet/models/llama/pipeline_llama.py:83.  position_ids restart per packed document
 * (touchnet/models/llama/processing_llama.py:98).
 *   tn_rope_table: cos/sin[b*T+t, j] = bf16(cos/sin(position_ids[b,t] · inv_freq[j]) · attention_scaling), j < hd/2
 *   tn_rope_apply: in-place x ← x·cos + rotate_half(x)·sin on X [rows, n_heads, hd] (row stride ldx elements);
 *                  inverse != 0 applies the transpose rotation (backward).
 */
int tn_rope_table(const int64_t* position_ids, const float* inv_freq, float attention_scaling, void* cos_out,
                  void* sin_out, int64_t rows, int half_dim, tn_stream_t stream);
int tn_rope_apply_bf16(void* X, int64_t ldx, const void* cos_tab, const void* sin_tab, int64_t rows, int n_heads,
                       int head_dim, int inverse, tn_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Packed-sequence (block-causal "document") attention, head_dim = 128, bf16, GQA.
 * Reference interface: hf:integrations/flex_attention.py:136-247 make_flex_block_causal_mask + :262-364
 * flex_attention_forward (selected by "attn_implementation": "flex_attention",
 * examples/text/pretrain/fineweb-edu/config/Llama-3_2-1B.json:7; checked at touchnet/bin/train.py:129-131).
 *   mask: allow[b,q,k] = (q >= k) && doc[b,q] == doc[b,k] && doc[b,q] > 0      (doc = attention_mask ids, int32)
 *   Q [B,T,H,128], K/V [B,T,KV,128], O [B,T,H,128] with strides (elements): token stride ld*, batch stride = T*ld*.
 *   lse [B,H,T] fp32 (natural log; +inf for fully-masked rows whose O is exactly 0).
 *   Context parallelism (touchnet/utils/distributed.py:292-315 shards the sequence over the `cp` mesh): Tq > 0 makes
 *   Q / O / dO / dQ / lse / delta hold only the Tq query rows starting at global position q_blk_off*128, while K / V /
 *   dK / dV / doc_ids / meta stay global (T rows); Tq <= 0 means Tq = T, offset 0.
 *   tn_attn_prep builds, on the device with no host sync, the per-block kv/q ranges, a per-row "canonical" flag and
 *   the per-position document extents [start,end) the kernels mask with; meta: int32 buffer of tn_attn_meta_ints(B,T)
 *   elements.
 */
int64_t tn_attn_meta_ints(int B, int T);
int tn_attn_prep(const int32_t* doc_ids, int32_t* meta, int B, int T, tn_stream_t stream);
int tn_attn_fwd_bf16(const void* Q, int64_t ldq, const void* K, int64_t ldk, const void* V, int64_t ldv, void* O,
                     int64_t ldo, float* lse, const int32_t* doc_ids, const int32_t* meta, int B, int T, int H, int KV,
                     float scale, int Tq, int q_blk_off, tn_stream_t stream);
/* backward: delta [B,H,T] fp32 workspace; dQ [B,T,H,128], dK/dV [B,T,KV,128] bf16.  Optional fused inverse RoPE: with
 * rope_cos_q/sin_q ([B*Tq, 64] bf16 tables of tn_rope_table) dQ is returned w.r.t. the UN-rotated q, likewise
 * rope_cos_k/sin_k ([B*T, 64]) for dK (backward of hf apply_rotary_pos_emb, modeling_llama.py:151-168); NULL = off. */
int tn_attn_bwd_bf16(const void* Q, int64_t ldq, const void* K, int64_t ldk, const void* V, int64_t ldv, const void* O,
                     int64_t ldo, const void* dO, int64_t lddo, const float* lse, float* delta, void* dQ, int64_t lddq,
                     void* dK, int64_t lddk, void* dV, int64_t lddv, const int32_t* doc_ids, const int32_t* meta, int B,
                     int T, int H, int KV, float scale, int Tq, int q_blk_off, const void* rope_cos_q,
                     const void* rope_sin_q, const void* rope_cos_k, const void* rope_sin_k, tn_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Autoregressive decoding (touchnet_b200/generation.py).  Reference interface: the greedy `model.generate(use_cache=True,
 * do_sample=False, num_beams=1, repetition_penalty, no_repeat_ngram_size, ...)` of
 * touchnet/models/touch_audio/inference_touch_audio.py:170-192 (hf: DynamicCache + sdpa attention of the new token,
 * RepetitionPenaltyLogitsProcessor, NoRepeatNGramLogitsProcessor, argmax).
 *   Cache K/V: [B, S_cap, KV, 128] bf16 with token stride ld_tok and batch stride ld_batch (elements).
 *   tn_attn_decode: one query row per batch row, Q [B, H*128] (row stride ldq, RoPE already applied) against cache rows
 *     [kv_start[b], kv_end[b]) (device int32).  Split-KV: the split count depends on (B, KV, S_cap) only; `workspace`
 *     holds tn_attn_decode_ws_floats(B, H, KV, S_cap) floats.  O [B, H*128] bf16; lse [B, H] fp32 (optional, natural
 *     log) with the conventions of tn_attn_fwd_bf16 (O = 0, lse = +inf for an empty range).  H/KV in 1..16.
 *     Bit-reproducible (splits are merged in a fixed order).
 *   tn_kv_append: cache rows [row_end[b] - T_new, row_end[b]) of batch row b <- source rows b*T_new .. b*T_new+T_new-1 of
 *     K / V (row strides ldk / ldv, `width` = KV*128 columns copied).
 *   tn_greedy_select: per row b, over the bf16 logits [B, V] (row stride ld) cast to fp32: repetition penalty on every id
 *     of history[b, 0:length[b]] (score < 0 ? score*p : score/p), no-repeat-ngram ban (n = no_repeat_ngram_size, 0 = off),
 *     argmax (lowest index on ties); finished rows take `pad`.  Then history[b, length[b]] = next_ids[b] = token,
 *     length[b] += 1, positions[b] += 1, finished[b] |= (token == eos).
 */
int64_t tn_attn_decode_ws_floats(int B, int H, int KV, int S_cap);
int tn_attn_decode_bf16(const void* Q, int64_t ldq, const void* K, const void* V, int64_t ld_tok, int64_t ld_batch,
                        const int32_t* kv_start, const int32_t* kv_end, int B, int H, int KV, int S_cap, float scale,
                        float* workspace, void* O, int64_t ldo, float* lse, tn_stream_t stream);
int tn_kv_append_bf16(const void* K, int64_t ldk, const void* V, int64_t ldv, void* K_cache, void* V_cache,
                      int64_t ld_tok, int64_t ld_batch, const int32_t* row_end, int B, int T_new, int S_cap, int width,
                      tn_stream_t stream);
int tn_greedy_select_bf16(const void* logits, int64_t ld, int B, int V, int64_t* history, int64_t ld_hist,
                          int32_t* length, int64_t* positions, int64_t* next_ids, int32_t* finished,
                          float repetition_penalty, int no_repeat_ngram_size, int64_t eos, int64_t pad,
                          tn_stream_t stream);

/* Speculative decoding (generation.generate with assistant_model): a draft model proposes k tokens per row, the target
 * scores the k + 1 rows next_ids, d_0 .. d_{k-1} in one step and keeps the longest prefix that matches its own picks.
 *   tn_attn_decode_multi: Tq query rows per batch row, Q [B*Tq, H*128]: row b*Tq + j is query j of batch row b, at cache
 *     position kv_end[b] - Tq + j, attending to cache rows [kv_start[b], kv_end[b] - Tq + j + 1) (causal within the new
 *     block).  Row j's O / lse are bit-identical to tn_attn_decode_bf16 with kv_end = kv_end[b] - Tq + j + 1: same
 *     split count and chunks (functions of B, KV, S_cap), same merge order.  `workspace` holds
 *     tn_attn_decode_multi_ws_floats(B, Tq, H, KV, S_cap) floats.  Tq * H/KV in 1..16 (one m16 tile per kv head).
 *   tn_verify_select: logits [B*(k+1), V] (row b*(k+1) + j), draft [B, k] int64 (device).  For a row with finished == 0,
 *     picks[b, j] is the pick of tn_greedy_select on logits row b*(k+1) + j over history[b, 0:length[b]] followed by
 *     draft[b, 0:j]; n = the number of leading j < k with draft[b, j] == picks[b, j].  The row emits picks[b, 0..n],
 *     cut after the first eos and when length reaches limit[b]: they are written to history[b, length[b]..],
 *     length and positions advance by their count, next_ids = the last one, finished = 1 if it is eos or length ==
 *     limit[b].  A finished row does not advance (next_ids = pad, nothing else written).  picks [B, k+1] int64 is
 *     written for every row that is not finished.
 */
int64_t tn_attn_decode_multi_ws_floats(int B, int Tq, int H, int KV, int S_cap);
int tn_attn_decode_multi_bf16(const void* Q, int64_t ldq, const void* K, const void* V, int64_t ld_tok,
                              int64_t ld_batch, const int32_t* kv_start, const int32_t* kv_end, int B, int Tq, int H,
                              int KV, int S_cap, float scale, float* workspace, void* O, int64_t ldo, float* lse,
                              tn_stream_t stream);
int tn_verify_select_bf16(const void* logits, int64_t ld, int B, int k, int V, const int64_t* draft, int64_t* history,
                          int64_t ld_hist, int32_t* length, int64_t* positions, int64_t* next_ids, int32_t* finished,
                          const int32_t* limit, int64_t* picks, float repetition_penalty, int no_repeat_ngram_size,
                          int64_t eos, int64_t pad, tn_stream_t stream);

/* Continuous batching (generation.generate_many): a cache of B slots whose rows are refilled with new prompts while
 * the other slots keep decoding.  `docs` is a HOST table [n_docs][4] int32 = (src_row, slot, len, limit), at most
 * TN_ADMIT_MAX documents per call, distinct slots in [0, B), 0 < len < limit <= S_cap; it is checked here and passed to
 * the kernel by value (no device copy, nothing allocated).
 *   tn_kv_scatter: cache rows [0, len) of slot `slot` <- source rows [src_row, src_row + len) of K / V (the packed prefill
 *     of the admitted prompts; n_src_rows rows, strides and alignment as tn_kv_append).  A bit-exact copy; nothing else
 *     in the cache is written.
 *   tn_slot_admit: for each document, history[slot, 0:len) = ids[src_row:src_row+len), kv_start[slot] = first row of
 *     the prompt's last document (its last run of equal doc_ids), kv_end[slot] = len, positions[slot] =
 *     position_ids[src_row + len - 1], finished[slot] = 0, limit[slot] = limit.  Slots not named are not touched.
 *   tn_greedy_select_slots: the selection of tn_greedy_select on n_rows logits rows; row r selects for slot
 *     row_slot[r] (HOST array, at most TN_SELECT_MAX_MAP rows, distinct slots) or, with row_slot = NULL and n_rows == B,
 *     for slot r.  A slot with finished != 0 (finished or idle) does not advance: next_ids = pad, no history write,
 *     length and positions unchanged.  A slot finishes when it emits eos or when length + 1 == limit[slot].
 */
#define TN_ADMIT_MAX 128
#define TN_SELECT_MAX_MAP 256
int tn_kv_scatter_bf16(const void* K, int64_t ldk, const void* V, int64_t ldv, int64_t n_src_rows, void* K_cache,
                       void* V_cache, int64_t ld_tok, int64_t ld_batch, const int32_t* docs, int n_docs, int B, int S_cap,
                       int width, tn_stream_t stream);
int tn_slot_admit(const int32_t* docs, int n_docs, const int64_t* ids, const int32_t* doc_ids, const int64_t* position_ids,
                  int64_t n_src_rows, int64_t* history, int64_t ld_hist, int32_t* kv_start, int32_t* kv_end,
                  int64_t* positions, int32_t* finished, int32_t* limit, int B, tn_stream_t stream);
int tn_greedy_select_slots_bf16(const void* logits, int64_t ld, int n_rows, const int32_t* row_slot, int B, int V,
                                int64_t* history, int64_t ld_hist, int32_t* length, int64_t* positions, int64_t* next_ids,
                                int32_t* finished, const int32_t* limit, float repetition_penalty,
                                int no_repeat_ngram_size, int64_t eos, int64_t pad, tn_stream_t stream);

/* Multinomial sampling over cache slots (generation.generate_many with do_sample=True).
 *   tn_sample_select_slots: tn_greedy_select_slots with the argmax replaced by a draw from HF's sampling distribution:
 *     the processed fp32 logits divided by temperature (> 0; 1 skips it), then top-k (0 or >= V skips it: every token
 *     >= the k-th largest value is kept, ties included), then top-p in [0, 1] (1 skips it: a group of equal values v is
 *     kept iff the kept mass of the values <= v is > (1 - top_p) times the kept total; the maximum always stays), then
 *     softmax.  Token weights are exp(x - max) in 2^40 fixed point, so every sum is exact in any order; a token whose
 *     weight rounds to 0 (total probability < V * 2^-40) is never drawn.  The draw is Philox4x32-10 with key = seed and
 *     counter (length[slot], 0, stream key): a 64-bit r picks the target floor(r * Z / 2^64) in the kept total Z and the
 *     token is the one whose interval of the prefix sums in index order holds it.  The stream key of a mapped row is
 *     row_key[r] (HOST array beside row_slot), stored into stream_key[slot]; other rows read stream_key[slot] (device,
 *     [B] int64).  A row with a NaN, an infinite maximum or every token banned takes tn_greedy_select's pick.
 */
int tn_sample_select_slots_bf16(const void* logits, int64_t ld, int n_rows, const int32_t* row_slot,
                                const int64_t* row_key, int B, int V, int64_t* history, int64_t ld_hist, int32_t* length,
                                int64_t* positions, int64_t* next_ids, int32_t* finished, const int32_t* limit,
                                int64_t* stream_key, float repetition_penalty, int no_repeat_ngram_size,
                                float temperature, int top_k, float top_p, int64_t seed, int64_t eos, int64_t pad,
                                tn_stream_t stream);

/* Speculative sampling (generation.generate_many with assistant_model and do_sample=True; Leviathan et al. 2023,
 * Algorithm 1) over B slots and k draft tokens per slot.
 *   tn_spec_sample_verify: logits [B*(k+1), V] of the model (row b*(k+1) + j) and draft_logits [B*k, V] of the draft
 *     (row b*k + j, the logits the draft drew draft[b, j] from), draft [B, k] int64 (device).  For a slot with
 *     finished == 0, p_j and q_j are tn_sample_select_slots's distributions (same processors, temperature, top_k,
 *     top_p and 2^40 fixed-point weights) of target row j and draft row j over history[b, 0:length[b]] followed by
 *     draft[b, 0:j].  Position j < k accepts draft[b, j] = x iff floor(r * wq(x) * Zp / 2^64) < wp(x) * Zq in exact
 *     integers, r the 64-bit Philox4x32-10 draw (key seed, counter (length[b] + j, 1, stream_key[b])): probability
 *     min(1, p_j(x) / q_j(x)) within 2^-64.  At the first rejection n (or n = k) the row emits one token drawn from
 *     max(0, wp * Zq - wq * Zp) (p_k itself at n = k) in index order with the draw of counter (length[b] + n, 2,
 *     stream_key[b]).  A target row with a NaN, an infinite maximum or every token banned emits its greedy pick and
 *     stops there; a degenerate draft row's q is a point mass on its greedy pick.  The emitted tokens (accepted
 *     drafts, then the last) are committed as tn_verify_select commits its picks: cut after the first eos and when
 *     length reaches limit[b].  A finished slot does not advance (next_ids = pad, nothing else written).
 *     picks [B, k+1] int64 (device scratch) receives, for each slot not finished, x at an accepted position and ~t at
 *     the position that emitted t (later positions are computed but never read).
 */
int tn_spec_sample_verify_bf16(const void* logits, int64_t ld, const void* draft_logits, int64_t ldd, int B, int k,
                               int V, const int64_t* draft, int64_t* history, int64_t ld_hist, int32_t* length,
                               int64_t* positions, int64_t* next_ids, int32_t* finished, const int32_t* limit,
                               const int64_t* stream_key, int64_t* picks, float repetition_penalty,
                               int no_repeat_ngram_size, float temperature, int top_k, float top_p, int64_t seed,
                               int64_t eos, int64_t pad, tn_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Audio frontend.
 *   tn_fbank: touchnet/data/functions.py:117-134 audio_compute_fbank → ta:compliance/kaldi.py:514-645 (snip_edges,
 *     remove DC, pre-emphasis, povey window, |rfft|², HTK mel bank, log) batched over utterances packed back to back.
 *     wav: fp32 in [-1,1] (wav_is_i16 = 0; scaled by 2^15 like functions.py:125) or int16 PCM (wav_is_i16 = 1).
 *     utt_offsets[n_utts+1]: sample offsets; frame_offsets[n_utts+1]: output row offsets (m_i = 1+(N_i-win)/shift).
 *     window [frame_len] and mel_filters [n_mels, n_fft/2+1] are supplied by the host mirror (povey window and HTK
 *     mel bank computed exactly as ta:compliance/kaldi.py:90-103 and :436-511 do).
 *   tn_logmel: touchnet/data/functions.py:159-190 audio_compute_log_mel_spectrogram (whisper-style: hann STFT,
 *     center/reflect, power, Slaney mel (caller supplies filters [n_mels, n_fft/2+1] fp32), log10, per-utterance
 *     max-8 clamp, (x+4)/4).  Two passes: tn_logmel_power writes log10 mel + per-utterance max (atomic), then
 *     tn_logmel_finish applies the clamp/affine in place.
 *   tn_feat_stack: touchnet/data/functions.py:258-286 audiofeat_stack (left/right replicate padding, stack/stride,
 *     optional per-row mean / unbiased-std normalisation).  dst_row0 == NULL: rows are written packed back to back;
 *     otherwise utterance u's rows go to out[(dst_row0[u] + i) * out_ld ...], i.e. straight into the
 *     input_features [B*T, F] buffer at the positions batch_pairaudio_pairtext_packed assigns
 *     (touchnet/models/touch_audio/processing_touch_audio.py:200).
 */
int tn_fbank_f32(const void* wav, int wav_is_i16, const int64_t* utt_offsets, const int64_t* frame_offsets, int n_utts,
                 int64_t total_frames, int frame_len, int frame_shift, int n_fft, const float* window,
                 const float* mel_filters, int n_mels, float preemph, float* out, tn_stream_t stream);
/*   tn_mfcc: touchnet/data/functions.py:137-156 audio_compute_mfcc → ta:compliance/kaldi.py mfcc with the arguments
 *     the reference leaves at their defaults (use_energy off, cepstral_lifter 22, no htk_compat, no mean subtraction):
 *     tn_fbank's log-mel row y (same arguments, same arithmetic) times dct [n_mels, n_ceps] fp32, the orthonormal
 *     DCT-II of torchaudio's _get_dct_matrix with the lifter folded into its columns by the host.  out is
 *     [total_frames, n_ceps]; the log-mel row never leaves the chip.  c[i] = sum_m y[m] * dct[m][i] in ascending m:
 *     bit-reproducible.  1 <= n_ceps <= n_mels (the reference asserts the same).
 */
int tn_mfcc_f32(const void* wav, int wav_is_i16, const int64_t* utt_offsets, const int64_t* frame_offsets, int n_utts,
                int64_t total_frames, int frame_len, int frame_shift, int n_fft, const float* window,
                const float* mel_filters, int n_mels, float preemph, const float* dct /*[n_mels, n_ceps], lifter folded in*/,
                int n_ceps, float* out, tn_stream_t stream);
/*   tn_logmel_power: wav is fp32 in [-1,1] (wav_is_i16 = 0, used as is: functions.py:168 does not scale it) or int16
 *     PCM (wav_is_i16 = 1, times 2^-15, so the same bits as fp32 pcm / 32768).  Every utterance is right-padded with
 *     pad >= 0 zero samples (functions.py:169-170 audiofeat_padding) without a copy: frames reflect-index the padded
 *     length N_i + pad and read 0 at or past N_i.  frame_offsets counts (N_i + pad) / hop rows per utterance.
 */
int tn_logmel_power_f32(const void* wav, int wav_is_i16, const int64_t* utt_offsets, const int64_t* frame_offsets,
                        int n_utts, int64_t total_frames, int n_fft, int hop, int pad, const float* window,
                        const float* mel_filters, int n_mels, float* out, float* utt_max, tn_stream_t stream);
int tn_logmel_finish_f32(float* feats, const int64_t* frame_offsets, const float* utt_max, int n_utts,
                         int64_t total_frames, int n_mels, tn_stream_t stream);
int tn_feat_stack_f32(const float* feats, const int64_t* frame_offsets, const int64_t* out_offsets, int n_utts,
                      int64_t total_out_rows, int n_mels, int stack, int stride, int normalize, float* out,
                      const int64_t* dst_row0, int64_t out_ld, tn_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Data augmentation of the ASR recipe (touchnet/data/functions.py:83-114 audio_resample / audio_speed_perturb and
 * :193-255 audiofeat_spec_aug / audiofeat_spec_sub / audiofeat_spec_trim), applied to utterances packed back to back.
 * The random draws are made on the host in the reference's order (touchnet_b200/augment.py); these apply them.
 *   tn_resample_f32: polyphase FIR of torchaudio.transforms.Resample.  Utterance u uses bank_table[utt_bank[u]] =
 *     (orig, new, width, taps, offset) - gcd-reduced rates, filter half-width, taps = 2*width + orig, offset of its
 *     [new, taps] fp32 bank in `banks` - and writes y[i*new + j] = sum_k w[j][k] * x[i*orig - width + k] for its
 *     out_offsets[u+1] - out_offsets[u] outputs (x is zero outside the utterance).  x is fp32 or int16 (scaled by
 *     2^-15).  A (1, 1) bank is an exact copy.  Speed perturbation s at rate sr is the bank (sr*s -> sr).
 *     bank_table is a HOST array of n_banks <= 16 rows; tile_offsets[u] = first tile of utterance u, tile = output
 *     samples per tile (multiple of 32).  Fixed summation order: bit-reproducible.
 *   tn_spec_augment_f32: out of place.  Output frame f of utterance u (frames in_frame_offsets -> out_frame_offsets,
 *     the output already trimmed) = input frame f - pos of the last sub (start, end, pos) with start <= f < end, else
 *     f; zero if that source frame lies in a time mask [start, end) or the column in a frequency mask.  Tables are per
 *     utterance, fixed width: t_masks [n_utts][n_t_masks][2], f_masks [n_utts][n_f_masks][2], subs
 *     [n_utts][n_subs][3] int32 (empty entries: start == end).
 */
int tn_resample_f32(const void* x, int x_is_i16, const int64_t* in_offsets, const int64_t* out_offsets,
                    const int64_t* tile_offsets, const int32_t* utt_bank, int n_utts, int64_t n_tiles, int tile,
                    const int32_t* bank_table, int n_banks, const float* banks, float* y, tn_stream_t stream);
int tn_spec_augment_f32(const float* in, const int64_t* in_frame_offsets, const int64_t* out_frame_offsets, int n_utts,
                        int64_t total_out_frames, int n_feat, const int32_t* t_masks, int n_t_masks,
                        const int32_t* f_masks, int n_f_masks, const int32_t* subs, int n_subs, float* out,
                        tn_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Small fused elementwise helpers on the path.
 *   tn_embed_add: E = embed[input_ids] + P   (touchnet/models/touch_audio/modeling_touch_audio.py:124-131), with the
 *     NaN check of :133-134 folded in (nan_flag[0] set to 1 if any NaN; read lazily by the caller, no sync here).
 *   tn_cast_f32_bf16: fp32 master → bf16 working copy (what FSDP2 MixedPrecisionPolicy does at all-gather,
 *     touchnet/models/helper_func.py:163).
 */
int tn_embed_add_bf16(const int64_t* input_ids, const void* embed, int embed_is_f32, const void* P, void* E,
                      int32_t* nan_flag, int64_t rows, int d, int64_t vocab, tn_stream_t stream);
int tn_cast_f32_bf16(const float* src, void* dst, int64_t n, tn_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Pack-loss cross-entropy next to the path (SURVEY 8(f) rank 1).  touchnet/loss/__init__.py:7-28 +
 * touchnet/loss/cross_entropy.py:12-50 + touchnet/utils/metrics.py:26-50, without fp32 logits:
 *   fwd: lse[r] = logsumexp(logits[r,:]) (fp32), ce[r] = lse[r] - logits[r,label[r]] (0 where label is the ignore
 *        index, i.e. outside [0,V)), argmax[r] (optional, for the accuracy metric).
 *   bwd: IN PLACE  logits[r,:] <- (softmax(logits[r,:]) - onehot(label[r])) * scale * grad_scalar[0] / sentence_lens[r]
 *        (rows with an ignored label become 0).  grad_scalar: device pointer to the upstream scalar gradient (or NULL = 1).
 */
int tn_pack_ce_fwd_bf16(const void* logits, int64_t ld, const int64_t* labels, float* lse, float* ce, int32_t* argmax,
                        int64_t M, int V, tn_stream_t stream);
int tn_pack_ce_bwd_bf16(void* logits, int64_t ld, const int64_t* labels, const int64_t* sentence_lens, const float* lse,
                        const float* grad_scalar, float scale, int64_t M, int V, tn_stream_t stream);
/* vocabulary-parallel backward (tensor-parallel lm_head with loss parallel, ref: touchnet/utils/distributed.py:322-323,
 * touchnet/models/llama/parallelize_llama.py:127-131): `logits` holds columns [v0, v0+V_local) of a V_total-wide vocabulary,
 * labels are GLOBAL ids, lse the GLOBAL logsumexp (all-reduced by the caller from per-shard tn_pack_ce_fwd_bf16 results). */
int tn_pack_ce_bwd_vp_bf16(void* logits, int64_t ld, const int64_t* labels_global, const int64_t* sentence_lens,
                           const float* lse_global, const float* grad_scalar, float scale, int64_t M, int V_local, int64_t v0,
                           int64_t V_total, tn_stream_t stream);
/* fwd and bwd (upstream gradient 1) of the above in ONE launch over a chunk of rows: the building block of the fused
 * lm_head + loss (touchnet_b200/loss.py::FusedLinearCEFn - the reference's best path is Liger's fused-linear-cross-entropy,
 * touchnet/bin/train.py:443-445, which never materialises [B,T,V] logits either).  IN PLACE like the bwd entry point. */
int tn_pack_ce_fused_bf16(void* logits, int64_t ld, const int64_t* labels, const int64_t* sentence_lens, float* lse,
                          float* ce, int32_t* argmax, float scale, int64_t M, int V, tn_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------------
 * BEST-RQ tokenizer (SURVEY 8(f) rank 2): labels of audio pre-training.  touchnet/tokenizer/tokenizer.py:289-299.
 *   codes[t] = argmin_v || normalize(feats[t,:] @ proj) - codebook[v,:] ||_2   (lowest index on ties, like torch.argmin)
 *   feats [T, D] fp32 (row stride ld), proj [D, E], codebook [V, E] (rows already L2-normalised, :267), E in {8,16,32}.
 */
int tn_bestrq_tokenize_f32(const float* feats, int64_t ld, const float* proj, const float* codebook, int64_t T, int D,
                           int E, int V, int32_t* codes, tn_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Optimizer step next to the path (SURVEY 8(f) rank 4), on the rank-local fp32 shards.
 *   tn_sumsq_f32: partials[0..*n_partials_used) = block-wise sums of x[i]^2 (deterministic; the caller adds them up, sums
 *     over tensors / ranks and takes the root) - replaces torch.nn.utils.get_total_norm in
 *     touchnet/utils/distributed.py:426-491.  `partials` holds tn_sumsq_num_partials() floats.
 *   tn_scale_f32: x *= scale[0] (device scalar, no-op when it is 1) - clip_grads_with_norm_ of the same function.
 *   tn_adamw_f32: one AdamW step (decoupled weight decay, bias corrections passed in) replacing
 *     torch.optim.AdamW(..., fused=True) as built by touchnet/utils/optimizer.py:127-172; `grad_scale` (device scalar or
 *     NULL) multiplies the gradient on the fly (the clip coefficient, so clipping needs no pass of its own) and
 *     `param_bf16` (or NULL) receives the bf16 working copy of the updated parameter.
 */
int tn_sumsq_num_partials(void);
int tn_sumsq_f32(const float* x, int64_t n, float* partials, int* n_partials_used, tn_stream_t stream);
int tn_scale_f32(float* x, int64_t n, const float* scale, tn_stream_t stream);
int tn_scale_bf16(void* x, int64_t n, const float* scale, tn_stream_t stream);   /* same, bf16 data (no-op when scale is 1) */
int tn_adamw_f32(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, void* param_bf16, int64_t n,
                 float lr, float beta1, float beta2, float eps, float weight_decay, float bias_correction1,
                 float bias_correction2_sqrt, const float* grad_scale, tn_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Device-side assembly of the integer side of a packed batch (SURVEY 8(f) rank 3): the per-document slice assignments of
 * touchnet/models/llama/processing_llama.py:64-102 and touchnet/models/touch_audio/processing_touch_audio.py:176-206.
 * The host keeps the greedy placement (row / offset / document id per document) and ships the concatenated text tokens;
 * the five [B,T] int64 buffers are filled here: defaults pad / -100 / 0 / 0 / 1, then per document
 *   position_ids = 0..total-1, attention_mask = sid, sentence_lens = n_txt over its `audio + n_txt` positions,
 *   input_ids = [bos, tokens...], labels = [tokens..., eos] over the text positions (n_txt = n_tokens + 1).
 */
int tn_pack_layout_i64(const int32_t* doc_row, const int32_t* doc_off, const int32_t* doc_audio, const int32_t* doc_sid,
                       const int64_t* tok_off, const int64_t* tokens, int n_docs, int B, int T, int64_t pad, int64_t bos,
                       int64_t eos, int64_t* input_ids, int64_t* labels, int64_t* position_ids, int64_t* attention_mask,
                       int64_t* sentence_lens, tn_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Data-parallel collectives over NVLink peer memory (SURVEY 8(e) "NCCL's or your own"; touchnet_b200/fsdp_comm.py).  What FSDP2 does
 * through NCCL around every decoder block (touchnet/models/helper_func.py:134-202: fp32 gradient reduce-scatter, bf16
 * parameter all-gather) as pull kernels on buffers every rank has mapped (torch symmetric memory):
 *   tn_peer_reduce_scatter_f32: out[i] = scale * sum_{p<n_peers} inputs[p][shard_offset + i], i < numel, summed in rank
 *     order (bit-reproducible); inputs = HOST array of n_peers device pointers (peer-mapped), shard_offset % 4 == 0.
 *   tn_peer_all_gather: out[p*bytes_each + j] = inputs[p][j]; bytes_each % 16 == 0.
 * max_ctas bounds the grid (default 32) so that the GEMMs these overlap with keep their SMs.  Cross-rank ordering (inputs
 * complete before the call, buffers not reused before every rank's call has finished) is the caller's barrier.
 */
int tn_peer_reduce_scatter_f32(const void* const* inputs, int n_peers, int64_t shard_offset, float* out, int64_t numel,
                               float scale, int max_ctas, tn_stream_t stream);
int tn_peer_all_gather(const void* const* inputs, int n_peers, int64_t bytes_each, void* out, int max_ctas,
                       tn_stream_t stream);
/* out[i] = scale * sum_k float(inputs[k][i]): bf16 chunks (local memory), fp32 accumulation in input order - the reduce step
 * of the direct-push reduce-scatter of touchnet_b200/fsdp_comm.py (same sum as FSDP2's fp32 reduce of bf16 gradients). */
int tn_reduce_bf16_to_f32(const void* const* inputs, int n_inputs, float* out, int64_t numel, float scale, int max_ctas,
                          tn_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* TOUCHNET_B200_H */
