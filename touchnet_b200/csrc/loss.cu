// touchnet_b200 :: "pack loss" cross-entropy next to the path (SURVEY 8(f) rank 1).
//
// Replaces   touchnet/loss/__init__.py:7-28   (torch.compile'd F.cross_entropy(pred.float(), reduction="none"))
//            touchnet/loss/cross_entropy.py:12-50 (per-token CE / sentence_len, summed, / num_sentence)
//            touchnet/utils/metrics.py:26-50   (argmax accuracy)
// without ever materialising fp32 logits: forward streams the bf16 logits once (online max / sum-exp / argmax per row),
// backward streams them once more and overwrites them in place with dlogits = (softmax - onehot) * w_row * g.
// HBM-bound: 2 bytes/logit forward, 4 bytes/logit backward (the reference path moves >= 26 bytes/logit).
#include <math.h>

#include "../../include/touchnet_b200.h"
#include "common.cuh"
#include "host.h"

namespace tn {

constexpr int CE_THREADS = 512;

struct MaxSum {
  float m, s;
  int idx;
};

__device__ __forceinline__ MaxSum ms_merge(const MaxSum& a, const MaxSum& b) {
  MaxSum r;
  if (a.m > b.m || (a.m == b.m && a.idx < b.idx)) { r.m = a.m; r.idx = a.idx; } else { r.m = b.m; r.idx = b.idx; }
  r.s = (a.m == -INFINITY ? 0.f : a.s * __expf(a.m - r.m)) + (b.m == -INFINITY ? 0.f : b.s * __expf(b.m - r.m));
  return r;
}

// Online max / sum-exp / first argmax of one bf16 row: per-thread loop over 16-byte vectors and the V % 8 tail, warp
// butterfly, one partial per warp in red[], barrier.  Thread 0 then merges them with merge_partials inside the caller's
// own thread-0 block: a merge in here would open a second thread-0 region, which lengthens the fused kernel.
__device__ __forceinline__ void row_partials(const bf16* __restrict__ x, int V, MaxSum* red) {
  const int nvec = V >> 3;
  MaxSum acc{-INFINITY, 0.f, 0x7fffffff};
  for (int i = threadIdx.x; i < nvec; i += CE_THREADS) {
    const uint4 v = reinterpret_cast<const uint4*>(x)[i];
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    float f[8];
#pragma unroll
    for (int j = 0; j < 4; ++j) { f[2 * j] = bf16lo(w[j]); f[2 * j + 1] = bf16hi(w[j]); }
    float vm = f[0];
    int vi = 0;
#pragma unroll
    for (int j = 1; j < 8; ++j) if (f[j] > vm) { vm = f[j]; vi = j; }
    if (vm > acc.m) {
      acc.s = (acc.m == -INFINITY) ? 0.f : acc.s * __expf(acc.m - vm);
      acc.m = vm;
      acc.idx = i * 8 + vi;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) acc.s += __expf(f[j] - acc.m);
  }
  for (int c = nvec * 8 + threadIdx.x; c < V; c += CE_THREADS) {   // tail (V % 8)
    const float f = __bfloat162float(x[c]);
    if (f > acc.m) { acc.s = (acc.m == -INFINITY) ? 0.f : acc.s * __expf(acc.m - f); acc.m = f; acc.idx = c; }
    acc.s += __expf(f - acc.m);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    MaxSum other;
    other.m = __shfl_xor_sync(0xffffffffu, acc.m, o);
    other.s = __shfl_xor_sync(0xffffffffu, acc.s, o);
    other.idx = __shfl_xor_sync(0xffffffffu, acc.idx, o);
    acc = ms_merge(acc, other);
  }
  if (lane_id() == 0) red[warp_id()] = acc;
  __syncthreads();
}

// The row's statistics from the warp partials, merged in warp order (ties keep the lower column).
__device__ __forceinline__ MaxSum merge_partials(const MaxSum* red) {
  MaxSum t = red[0];
  for (int w = 1; w < CE_THREADS / 32; ++w) t = ms_merge(t, red[w]);
  return t;
}

// Overwrites the row with dlogits[j] = (exp(x[j] - lse) - [j == lab]) * w, all zeros when !valid.  lab is the label's local
// column; outside [0, V) the one-hot lands in no column of this row.
__device__ __forceinline__ void write_grad(bf16* __restrict__ x, int V, float lse, float w, bool valid, int64_t lab) {
  const int nvec = V >> 3;
  for (int i = threadIdx.x; i < nvec; i += CE_THREADS) {
    uint4 v = reinterpret_cast<const uint4*>(x)[i];
    uint32_t ws[4] = {v.x, v.y, v.z, v.w};
    uint32_t o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float p0 = valid ? __expf(bf16lo(ws[j]) - lse) * w : 0.f;
      float p1 = valid ? __expf(bf16hi(ws[j]) - lse) * w : 0.f;
      const int c = i * 8 + 2 * j;
      if (c == lab) p0 -= w;
      if (c + 1 == lab) p1 -= w;
      o[j] = pack_bf16x2(p0, p1);
    }
    reinterpret_cast<uint4*>(x)[i] = make_uint4(o[0], o[1], o[2], o[3]);
  }
  for (int c = nvec * 8 + threadIdx.x; c < V; c += CE_THREADS) {
    float p = valid ? __expf(__bfloat162float(x[c]) - lse) * w : 0.f;
    if (c == lab) p -= w;
    x[c] = __float2bfloat16_rn(p);
  }
}

__global__ void __launch_bounds__(CE_THREADS) pack_ce_fwd_kernel(const bf16* __restrict__ logits, int64_t ld,
                                                                 const int64_t* __restrict__ labels,
                                                                 float* __restrict__ lse_out, float* __restrict__ ce_out,
                                                                 int32_t* __restrict__ argmax_out, int V) {
  __shared__ MaxSum red[CE_THREADS / 32];
  const int64_t row = blockIdx.x;
  const bf16* x = logits + row * ld;
  row_partials(x, V, red);
  if (threadIdx.x == 0) {
    const MaxSum t = merge_partials(red);
    const float lse = t.m + logf(t.s);
    lse_out[row] = lse;
    const int64_t lab = labels[row];
    ce_out[row] = (lab >= 0 && lab < V) ? lse - __bfloat162float(x[lab]) : 0.f;   // ignore_index (-100) -> 0
    if (argmax_out) argmax_out[row] = t.idx;
  }
}

// dlogits[r, j] = (exp(x - lse_r) - [j == label_r]) * w_r,  w_r = scale * g / sentence_len_r  (0 for ignored rows)
__global__ void __launch_bounds__(CE_THREADS) pack_ce_bwd_kernel(bf16* __restrict__ logits, int64_t ld,
                                                                 const int64_t* __restrict__ labels,
                                                                 const int64_t* __restrict__ sentence_lens,
                                                                 const float* __restrict__ lse_in,
                                                                 const float* __restrict__ grad_scalar, float scale,
                                                                 int V, int64_t v0, int64_t v_total) {
  // vocabulary-parallel form (tensor parallel lm_head, ref loss_parallel: touchnet/utils/distributed.py:322-323): this tensor
  // holds columns [v0, v0 + V) of a v_total-wide vocabulary, labels are global ids, lse is the GLOBAL logsumexp; a row is
  // valid iff its label is in [0, v_total), the one-hot lands here only if the label is one of OUR columns
  const int64_t row = blockIdx.x;
  const int64_t lab_g = labels[row];
  const bool valid = lab_g >= 0 && lab_g < v_total;
  const float g = grad_scalar ? grad_scalar[0] : 1.f;
  const float w = valid ? scale * g / float(sentence_lens ? sentence_lens[row] : 1) : 0.f;
  write_grad(logits + row * ld, V, lse_in[row], w, valid, lab_g - v0);
}

// Fused form for the chunked lm_head + loss (touchnet_b200/loss.py::FusedLinearCEFn): one CTA per row, pass 1 = the forward
// reduction above, pass 2 re-reads the row (256 KB at V = 128 k: it is still in L2) and overwrites it with
// dlogits = (softmax - onehot) * scale / sentence_len, i.e. the gradient for an upstream gradient of 1.
__global__ void __launch_bounds__(CE_THREADS) pack_ce_fused_kernel(bf16* __restrict__ logits, int64_t ld,
                                                                   const int64_t* __restrict__ labels,
                                                                   const int64_t* __restrict__ sentence_lens,
                                                                   float* __restrict__ lse_out, float* __restrict__ ce_out,
                                                                   int32_t* __restrict__ argmax_out, float scale, int V) {
  __shared__ MaxSum red[CE_THREADS / 32];
  __shared__ float s_lse;
  const int64_t row = blockIdx.x;
  bf16* x = logits + row * ld;
  row_partials(x, V, red);
  const int64_t lab = labels[row];
  const bool valid = lab >= 0 && lab < V;
  if (threadIdx.x == 0) {
    const MaxSum t = merge_partials(red);
    const float lse = t.m + logf(t.s);
    s_lse = lse;
    lse_out[row] = lse;
    ce_out[row] = valid ? lse - __bfloat162float(x[lab]) : 0.f;
    if (argmax_out) argmax_out[row] = t.idx;
  }
  __syncthreads();
  const float lse = s_lse;
  const float w = valid ? scale / float(sentence_lens ? sentence_lens[row] : 1) : 0.f;
  write_grad(x, V, lse, w, valid, lab);
}

}  // namespace tn

using namespace tn;

// Argument checks every entry point shares: the pointers it dereferences (`args_ok` covers all but the logits) and
// 16-byte aligned logits rows for the vector loads.
static int check_logits(const char* fn, const void* logits, int64_t ld, bool args_ok) {
  TN_REQUIRE(logits && args_ok, "%s: null pointer", fn);
  TN_REQUIRE(ld % 8 == 0 && (reinterpret_cast<uintptr_t>(logits) & 15) == 0, "%s: logits rows must be 16 B aligned", fn);
  return TN_OK;
}

extern "C" int tn_pack_ce_fwd_bf16(const void* logits, int64_t ld, const int64_t* labels, float* lse, float* ce,
                                   int32_t* argmax, int64_t M, int V, tn_stream_t stream_) {
  clear_error();
  if (int rc = check_logits("tn_pack_ce_fwd_bf16", logits, ld, labels && lse && ce)) return rc;
  if (M == 0) return TN_OK;
  pack_ce_fwd_kernel<<<unsigned(M), CE_THREADS, 0, static_cast<cudaStream_t>(stream_)>>>(
      static_cast<const bf16*>(logits), ld, labels, lse, ce, argmax, V);
  TN_CHECK_CUDA(cudaGetLastError());
  return TN_OK;
}

extern "C" int tn_pack_ce_bwd_bf16(void* logits, int64_t ld, const int64_t* labels, const int64_t* sentence_lens,
                                   const float* lse, const float* grad_scalar, float scale, int64_t M, int V,
                                   tn_stream_t stream_) {
  clear_error();
  if (int rc = check_logits("tn_pack_ce_bwd_bf16", logits, ld, labels && lse)) return rc;
  if (M == 0) return TN_OK;
  pack_ce_bwd_kernel<<<unsigned(M), CE_THREADS, 0, static_cast<cudaStream_t>(stream_)>>>(
      static_cast<bf16*>(logits), ld, labels, sentence_lens, lse, grad_scalar, scale, V, 0, V);
  TN_CHECK_CUDA(cudaGetLastError());
  return TN_OK;
}

extern "C" int tn_pack_ce_bwd_vp_bf16(void* logits, int64_t ld, const int64_t* labels_global, const int64_t* sentence_lens,
                                      const float* lse_global, const float* grad_scalar, float scale, int64_t M, int V_local,
                                      int64_t v0, int64_t V_total, tn_stream_t stream_) {
  clear_error();
  if (int rc = check_logits("tn_pack_ce_bwd_vp_bf16", logits, ld, labels_global && lse_global)) return rc;
  TN_REQUIRE(v0 >= 0 && v0 + V_local <= V_total, "tn_pack_ce_bwd_vp_bf16: column range outside the vocabulary");
  if (M == 0) return TN_OK;
  pack_ce_bwd_kernel<<<unsigned(M), CE_THREADS, 0, static_cast<cudaStream_t>(stream_)>>>(
      static_cast<bf16*>(logits), ld, labels_global, sentence_lens, lse_global, grad_scalar, scale, V_local, v0, V_total);
  TN_CHECK_CUDA(cudaGetLastError());
  return TN_OK;
}

extern "C" int tn_pack_ce_fused_bf16(void* logits, int64_t ld, const int64_t* labels, const int64_t* sentence_lens,
                                     float* lse, float* ce, int32_t* argmax, float scale, int64_t M, int V,
                                     tn_stream_t stream_) {
  clear_error();
  if (int rc = check_logits("tn_pack_ce_fused_bf16", logits, ld, labels && lse && ce)) return rc;
  if (M == 0) return TN_OK;
  pack_ce_fused_kernel<<<unsigned(M), CE_THREADS, 0, static_cast<cudaStream_t>(stream_)>>>(
      static_cast<bf16*>(logits), ld, labels, sentence_lens, lse, ce, argmax, scale, V);
  TN_CHECK_CUDA(cudaGetLastError());
  return TN_OK;
}
