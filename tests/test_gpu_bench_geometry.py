"""GPU parity at the geometry bench.py measures (llama32_3b_asr: d=3072, H=24, KV=8, head_dim 128, ffn=8192, T=8192
packed audio+text documents) and at the edges of the attention kernels' tiling.

  1. one decoder layer (ops.decoder_layer) at the benchmark geometry, forward and backward, fp32 and bf16 master
     weights, on the fused path (segmented QKV GEMM with RoPE in its epilogue, attention on strided views of the qkv
     buffer, attention backward with the inverse RoPE in its epilogues writing into one dqkv buffer, segmented QKV
     dgrad / wgrad) vs an fp32 autograd reference built from oracle/model_oracle.py pieces, with a bf16 rounding-point
     reference as the error floor;
  2. the packed-document attention forward / backward vs an fp64 reference, element-wise, over generated layouts, GQA
     ratios 1..16, operands as the decoder block hands them and four score regimes; the AttnPlan metadata vs a plain
     restatement of its contract;
  3. split-KV decode attention at long contexts (64 splits, G = 3, 8, 16) vs an fp64 reference.

Layouts, the metadata restatement and the fp64 references with their bounds live in tests/test_attn_geometry_cpu.py."""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import model_oracle as mo
from tests.gpu_util import rel_err, require_cuda
from tests.test_attn_geometry_cpu import (HD, LAYOUT_SETS, attention_reference, bench_doc_ids, decode_reference, layout,
                                          meta_offsets, random_doc_ids, restate_attn_meta, run_positions, work_order)
from touchnet_b200 import _lib, ops

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
SCALE = HD ** -0.5
LLAMA3 = {"rope_type": "llama3", "factor": 32.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0,
          "original_max_position_embeddings": 8192}


def _rope_tables(pos, H, KV, dev):
    """bf16 cos/sin [rows, 64] with the benchmark model's llama3 rope scaling."""
    inv, sc = mo.rope_inv_freq(mo.OracleConfig(3072, 8192, 1, H, KV, HD, 128256, rope_theta=500000.0,
                                               rope_scaling=dict(LLAMA3)))
    return ops.rope_table(pos.to(dev), inv.to(dev), sc)


def _within(name, got, ref, bound):
    """Element-wise |got - ref| <= bound (NaN fails); reports the worst row and the largest err / bound."""
    err = (got.double() - ref).abs()
    ok = err <= bound
    ratio = float((err / bound.clamp_min(1e-300)).nan_to_num(math.inf).max())
    if not bool(ok.all()):
        bad_rows = (~ok).reshape(ok.shape[0], -1).any(-1).nonzero().flatten()
        raise AssertionError(f"{name}: {int((~ok).sum())} elements over their bound in {bad_rows.numel()} rows "
                             f"(first rows {bad_rows[:8].tolist()}), max err/bound {ratio:.3g}")
    return ratio


# ---------------------------------------------------------------------------------------------------------------
# 1. decoder layer at the benchmark geometry
# ---------------------------------------------------------------------------------------------------------------
D, NH, NKV, FFN, EPS = 3072, 24, 8, 8192, 1e-5
LAYER_NAMES = ("ln1", "wq", "wk", "wv", "wo", "ln2", "wg", "wu", "wd")
# Largest allowed (our error) / (bf16 rounding-point reference's error), both against the fp32 reference.  Measured on
# one H100 80GB HBM3 (SXM, 700 W power limit), fp32 and bf16 master weights alike: 0.998 at most over the eleven
# tensors (the output; the gradients 0.92-0.998), 1.08 at most over the 8192 output rows.
LAYER_FACTOR = 1.25
ROW_FACTOR = 1.5


def _layer_reference(x, w, cos, sin, doc, dout, dtype):
    """The decoder layer (hf LlamaDecoderLayer, oracle/model_oracle.py::decoder_layer) in `dtype` by autograd, with
    attention one document at a time (oracle `attention`, dense per document) instead of a [T, T] mask."""
    T = x.shape[0]
    xr = x.detach().to(dtype).requires_grad_(True)
    wr = {k: v.detach().to(dtype).requires_grad_(True) for k, v in w.items()}
    h = mo.rms_norm(xr, wr["ln1"], EPS)
    q = F.linear(h, wr["wq"]).view(1, T, NH, HD).transpose(1, 2)
    k = F.linear(h, wr["wk"]).view(1, T, NKV, HD).transpose(1, 2)
    v = F.linear(h, wr["wv"]).view(1, T, NKV, HD).transpose(1, 2)
    q, k = mo.apply_rope(q, k, torch.cat([cos, cos], -1).to(dtype)[None], torch.cat([sin, sin], -1).to(dtype)[None])
    pieces, idxs = [], []
    for i in torch.unique(doc[doc > 0]).tolist():
        idx = (doc[0] == i).nonzero().squeeze(1)
        n = idx.numel()
        allow = torch.ones(1, n, n, dtype=torch.bool, device=x.device).tril()
        o_d, _ = mo.attention(q[:, :, idx], k[:, :, idx], v[:, :, idx], allow, SCALE)
        pieces.append(o_d.reshape(n, NH * HD))
        idxs.append(idx)
    o = torch.zeros(T, NH * HD, dtype=dtype, device=x.device).index_copy(0, torch.cat(idxs), torch.cat(pieces))
    x1 = xr + F.linear(o, wr["wo"])
    out = x1 + mo.mlp(mo.rms_norm(x1, wr["ln2"], EPS), wr["wg"], wr["wu"], wr["wd"])
    out.backward(dout.to(dtype))
    return out.detach(), xr.grad, {k: wr[k].grad for k in LAYER_NAMES}


@pytest.mark.parametrize("master_dtype", [torch.float32, torch.bfloat16])
def test_decoder_layer_at_benchmark_geometry(master_dtype):
    """ops.decoder_layer, d=3072, H=24, KV=8, ffn=8192, no bias, one layer, on the benchmark's packing (B=1, T=8192,
    bench.py::make_host_batch) with its llama3-scaled RoPE tables, fp32 or bf16 master weights.

    The layer must take the benchmark's path (checked through _lib._hooks): tn_gemm_qkv_bf16 mode 0 with the rope
    tables, attention forward on views of that buffer (row stride (H+2KV)*128), tn_attn_bwd_bf16 with rope tables
    writing into views of one dqkv buffer, tn_gemm_qkv_bf16 modes 1 (dgrad) and 2 (wgrad, fp32 or bf16 outputs).

    Reference: the same layer by autograd in fp32 on the bf16-rounded linear weights (norm weights as the kernels read
    them: the master values), TF32 off.  Floor: the same layer in bf16 (HF's rounding points).  With e(t) = relative L2
    error against the fp32 reference, every compared tensor - output, input gradient, the nine parameter gradients
    (both RMSNorm weights included) - must satisfy e(ours) <= LAYER_FACTOR * e(bf16 reference), and every output row
    (valid or padding) its own row-wise error within ROW_FACTOR of the bf16 reference's error on that row, so that an
    error confined to one document cannot hide in the global norm.

    Calibration: the measured ratios are recorded beside LAYER_FACTOR / ROW_FACTOR."""
    dev = require_cuda()
    doc, pos = (t.to(dev) for t in bench_doc_ids())
    T = doc.shape[1]
    g = torch.Generator(device=dev).manual_seed(3072)
    rn = lambda *s: torch.randn(*s, generator=g, device=dev)
    master = {"ln1": 1 + 0.1 * rn(D), "wq": 0.02 * rn(NH * HD, D), "wk": 0.02 * rn(NKV * HD, D),
              "wv": 0.02 * rn(NKV * HD, D), "wo": 0.02 * rn(D, NH * HD), "ln2": 1 + 0.1 * rn(D),
              "wg": 0.02 * rn(FFN, D), "wu": 0.02 * rn(FFN, D), "wd": 0.02 * rn(D, FFN)}
    P = {k: torch.nn.Parameter(v.to(master_dtype)) for k, v in master.items()}
    x = rn(T, D).to(BF16).requires_grad_(True)
    dout = rn(T, D).to(BF16)
    cos, sin = _rope_tables(pos, NH, NKV, dev)
    plan = ops.AttnPlan(doc)
    calls = []
    hook = lambda name, phase, args: calls.append((name, args)) if phase == "pre" else None
    _lib._hooks.append(hook)
    try:
        out = ops.decoder_layer(x, P["ln1"], P["wq"], P["wk"], P["wv"], None, None, None, P["wo"], P["ln2"], P["wg"],
                                P["wu"], P["wd"], cos, sin, plan, NH, NKV, EPS)
        out.backward(dout)
        torch.cuda.synchronize()
    finally:
        _lib._hooks.remove(hook)
    # ---- the benchmarked path ----
    width = (NH + 2 * NKV) * HD
    qkv = [a for n, a in calls if n == "tn_gemm_qkv_bf16"]
    assert sorted(a[0] for a in qkv) == [0, 1, 2], [a[0] for a in qkv]
    fwd = next(a for a in qkv if a[0] == 0)
    assert fwd[18] is not None and fwd[19] is not None, "RoPE must run in the QKV GEMM epilogue"
    wgrad = next(a for a in qkv if a[0] == 2)
    assert wgrad[11] == int(master_dtype == torch.float32), "segmented wgrad output dtype"
    att_f = [a for n, a in calls if n == "tn_attn_fwd_bf16"]
    assert len(att_f) == 1 and att_f[0][1] == width and att_f[0][3] == width and att_f[0][5] == width
    att_b = [a for n, a in calls if n == "tn_attn_bwd_bf16"]
    assert len(att_b) == 1 and all(a is not None for a in att_b[0][27:31]), "inverse RoPE in the attention backward"
    assert att_b[0][13] == att_b[0][15] == att_b[0][17] == width, "dq/dk/dv are views of one dqkv buffer"
    assert not any(n == "tn_rope_apply_bf16" for n, _ in calls)
    # ---- values ----
    ref_w = {k: (v.detach().float() if k.startswith("ln") else v.detach().bfloat16().float()) for k, v in P.items()}
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        r32 = _layer_reference(x, ref_w, cos, sin, doc, dout, torch.float32)
        r16 = _layer_reference(x, {k: v.bfloat16() for k, v in ref_w.items()}, cos, sin, doc, dout, BF16)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    checks = [("out", out.detach(), r32[0], r16[0]), ("dx", x.grad, r32[1], r16[1])]
    checks += [("d" + k, P[k].grad, r32[2][k], r16[2][k]) for k in LAYER_NAMES]
    ratios = {}
    for name, ours, ref, floor in checks:
        assert ours is not None and torch.isfinite(ours.float()).all(), name
        if name.startswith("d") and name != "dx":
            assert ours.dtype == master_dtype, (name, ours.dtype)
        e, f = rel_err(ours.float(), ref), rel_err(floor.float(), ref)
        ratios[name] = (e, f)
        assert e <= LAYER_FACTOR * f, (name, e, f)
    row = lambda a: (a.float() - r32[0]).double().norm(dim=1) / r32[0].double().norm(dim=1)
    e_row, f_row = row(out.detach()), row(r16[0])
    worst = int((e_row / f_row).argmax())
    print("layer", master_dtype, {k: f"{e:.3g}/{f:.3g}={e / f:.3g}" for k, (e, f) in ratios.items()},
          f"row max {float(e_row[worst] / f_row[worst]):.3g} at {worst}")
    assert (e_row <= ROW_FACTOR * f_row).all(), ("row", worst, float(e_row[worst]), float(f_row[worst]))


# ---------------------------------------------------------------------------------------------------------------
# 2. training attention kernels vs fp64, element-wise
# ---------------------------------------------------------------------------------------------------------------
def _doc_starts(doc):
    prev = torch.cat([torch.zeros_like(doc[:, :1]), doc[:, :-1]], 1)
    return (doc > 0) & ((doc != prev) | (torch.arange(doc.shape[1], device=doc.device) == 0))


def _operands(regime, doc, pos, H, KV, seed):
    """q [B*T,H,128], k/v [B*T,KV,128], do [B*T,H,128] fp32 for a score regime:
      normal  N(0,1) everywhere (logits std ~1)
      scaled  q, k times sqrt(10): logits std ~10
      sink    q share a direction mu; the first key of every document is 2*mu: its logit is ~11 above the rest
      rising  q share mu, key t of a document carries 2.8e-3*t*mu: logits climb ~2 per 64-key sub-block, so the running
              maximum (and the rescale) changes in every sub-block."""
    B, T = doc.shape
    dev = doc.device
    g = torch.Generator(device=dev).manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g, device=dev)
    q, k, v, do = rn(B * T, H, HD), rn(B * T, KV, HD), rn(B * T, KV, HD), rn(B * T, H, HD)
    mu = torch.sign(rn(HD))
    if regime == "scaled":
        q, k = q * math.sqrt(10), k * math.sqrt(10)
    elif regime == "sink":
        q = q + 0.5 * mu
        st = _doc_starts(doc).reshape(-1)
        k[st] = 2 * mu + 0.1 * k[st]
    elif regime == "rising":
        q = q + mu
        k = k + 2.8e-3 * pos.reshape(-1, 1, 1).float() * mu
    return q, k, v, do


ATTN_CASES = {
    # name: (layout set, H, KV, score regime, operands)
    "g1_edges_normal_strided": ("edges", 2, 2, "normal", "strided"),
    "g2_noncanonical_scaled_strided_rope": ("noncanonical", 4, 2, "scaled", "strided_rope"),
    "g3_bench_normal_strided_rope": ("bench", 24, 8, "normal", "strided_rope"),
    "g3_bench_sink_strided": ("bench", 24, 8, "sink", "strided"),
    "g3_edges_rising_strided_rope": ("edges", 6, 2, "rising", "strided_rope"),
    "g3_noncanonical_normal_contiguous": ("noncanonical", 3, 1, "normal", "contiguous"),
    "g4_mixed_sink_strided_rope": ("mixed", 8, 2, "sink", "strided_rope"),
    "g8_edges_scaled_strided_rope": ("edges", 8, 1, "scaled", "strided_rope"),
    "g8_bench_rising_strided": ("bench", 16, 2, "rising", "strided"),
    "g16_noncanonical_rising_strided": ("noncanonical", 16, 1, "rising", "strided"),
    "g16_mixed_normal_strided_rope": ("mixed", 16, 1, "normal", "strided_rope"),
}

def _run_attention(q, k, v, do, doc, H, KV, mode, rope):
    """Forward + backward as the decoder block runs them (mode 'strided*': q/k/v views of one [B*T, (H+2KV)*128]
    buffer, dq/dk/dv views of one NaN-poisoned dqkv buffer) or on contiguous tensors."""
    rows = q.shape[0]
    plan = ops.AttnPlan(doc)
    if mode == "contiguous":
        qb, kb, vb = (t.reshape(rows, -1).to(BF16).contiguous() for t in (q, k, v))
        o, lse = ops.attn_fwd(qb, kb, vb, plan, H, KV, SCALE)
        dq, dk, dv = ops.attn_bwd(qb, kb, vb, o, do, lse, plan, H, KV, SCALE, rope=rope)
        return (qb, kb, vb), o, lse, (dq, dk, dv), torch.cat([dq, dk, dv], 1)
    nq, nkv = H * HD, KV * HD
    qkv = torch.cat([q.reshape(rows, -1), k.reshape(rows, -1), v.reshape(rows, -1)], 1).to(BF16)
    qb, kb, vb = qkv[:, :nq], qkv[:, nq:nq + nkv], qkv[:, nq + nkv:]
    o, lse = ops.attn_fwd(qb, kb, vb, plan, H, KV, SCALE)
    dqkv = torch.full_like(qkv, float("nan"))
    out = (dqkv[:, :nq], dqkv[:, nq:nq + nkv], dqkv[:, nq + nkv:])
    ops.attn_bwd(qb, kb, vb, o, do, lse, plan, H, KV, SCALE, out=out, rope=rope)
    return (qb, kb, vb), o, lse, out, dqkv


@pytest.mark.parametrize("name", list(ATTN_CASES))
def test_attention_kernels_match_fp64_per_row(name):
    """attn_fwd / attn_bwd vs tests/test_attn_geometry_cpu.py::attention_reference: fp64, one document at a time, on
    the same bf16 operands (rotated q/k; with `rope=` the gradients w.r.t. the un-rotated q/k).  Every element of every
    valid query row of O and dQ, every LSE entry and every element of every key row of dK and dV must lie within the
    element-wise bound derived there from the bf16 rounding of P, of dS and of the outputs (plus fp32 accumulation);
    padding query rows give O = 0, LSE = +inf, dQ = 0 exactly, keys no query attends dK = dV = 0 exactly, and every
    element of the dqkv buffer is written.  Two runs are bit-identical.
    Measured on one H100 80GB HBM3 (SXM, 700 W), largest err/bound over all cases: O 0.82, LSE 0.008, dQ 0.18,
    dK 0.24, dV 0.78 (printed per case)."""
    dev = require_cuda()
    lay, H, KV, regime, mode = ATTN_CASES[name]
    doc = layout(lay).to(dev)
    pos = run_positions(doc.cpu()).to(dev)
    B, T = doc.shape
    q, k, v, do = _operands(regime, doc, pos, H, KV, seed=len(name) * 131 + H)
    do = do.reshape(B * T, -1).to(BF16)
    rope = _rope_tables(pos, H, KV, dev) if mode.endswith("rope") else None
    (qb, kb, vb), o, lse, (dq, dk, dv), dqkv = _run_attention(q, k, v, do, doc, H, KV, mode, rope)
    (_, _, _), o2, lse2, _, dqkv2 = _run_attention(q, k, v, do, doc, H, KV, mode, rope)
    torch.cuda.synchronize()
    assert torch.equal(o, o2) and torch.equal(lse, lse2) and torch.equal(dqkv, dqkv2), "two runs differ"
    assert not torch.isnan(dqkv).any(), "the backward left part of the dqkv buffer unwritten"
    ref = attention_reference(qb, kb, vb, do, doc, H, KV, SCALE, rope)
    valid = (doc > 0).reshape(-1)
    assert torch.all(o[~valid] == 0) and torch.all(dq[~valid] == 0)
    vm = (doc > 0)[:, None, :].expand(B, H, T)
    assert torch.all(lse[~vm] == math.inf)
    r = {"o": _within("o", o, ref["o"], ref["o_bound"]),
         "lse": _within("lse", lse[vm], ref["lse"][vm], ref["lse_bound"][vm]),
         "dq": _within("dq", dq, ref["dq"], ref["dq_bound"]),
         "dk": _within("dk", dk, ref["dk"], ref["dk_bound"]),
         "dv": _within("dv", dv, ref["dv"], ref["dv_bound"])}
    print("attention", name, {k_: f"{x:.3g}" for k_, x in r.items()})


def test_attn_plan_metadata_matches_its_contract():
    """AttnPlan.meta vs tests/test_attn_geometry_cpu.py::restate_attn_meta (kv_lo, kv_end, q_end, canonical per
    block; the canonical flag per row) and ::work_order (both cost-ordered work lists are permutations, ordered by
    non-increasing cost, ties by entry index), over 300 seeded random layouts and the named layout sets.  The
    per-position document-extent table is not compared: no kernel reads it."""
    dev = require_cuda()
    docs = [random_doc_ids(s) for s in range(300)] + [layout(n) for n in LAYOUT_SETS]
    for i, doc in enumerate(docs):
        B, T = doc.shape
        plan = ops.AttnPlan(doc.to(dev))
        meta = plan.meta.cpu()
        off = meta_offsets(B, T)
        nblk, N = off["nblk"], B * off["nblk"]
        assert meta.numel() == off["total"], (i, meta.numel(), off["total"])
        exp = restate_attn_meta(doc)
        got = [[tuple(x) for x in row] for row in meta[:N * 4].view(B, nblk, 4).tolist()]
        assert got == exp, (i, doc.shape, [(b, j, got[b][j], exp[b][j]) for b in range(B) for j in range(nblk)
                                           if got[b][j] != exp[b][j]][:4])
        assert meta[off["flags"]:off["flags"] + B].tolist() == [row[0][3] for row in exp], i
        oq, okv = work_order(exp)
        assert meta[off["order_q"]:off["order_q"] + N].tolist() == oq, i
        assert meta[off["order_kv"]:off["order_kv"] + N].tolist() == okv, i


# ---------------------------------------------------------------------------------------------------------------
# 3. split-KV decode at long contexts
# ---------------------------------------------------------------------------------------------------------------
def decode_splits(B, KV, S_cap):
    """decode.cu's split rule: ~4*132 CTAs over (split, kv head, row), at most one split per 64 cache rows, at most 64."""
    s = -(-4 * 132 // (B * KV))
    return max(1, min(s, -(-S_cap // 64), 64))


def decode_chunk(B, KV, S_cap):
    """Cache rows per split: ceil(S_cap / splits) rounded up to whole 64-key blocks."""
    per_split = -(-S_cap // decode_splits(B, KV, S_cap))
    return -(-per_split // 64) * 64


DECODE_CASES = {
    # name: (H, KV, S_cap, [(start, end) per batch row], splits)
    "bench_generate_S8192_full": (24, 8, 8192, [(0, 8192)], 64),
    "bench_generate_S32768_full": (24, 8, 32768, [(0, 32768)], 64),
    "bench_generate_S32768_mid_split": (24, 8, 32768, [(1061, 32461)], 64),     # 1061 = 2*512 + 37, 32461 = 63*512 + 205
    "g16_S32768": (16, 1, 32768, [(13, 32700)], 64),
    "g8_ragged": (16, 2, 4096, [(100, 3999), (2047, 2048)], 64),
    "g3_lengths_1_and_0": (6, 2, 2048, [(5, 6), (700, 700), (0, 0), (0, 2048)], 32),
}


@pytest.mark.parametrize("name", list(DECODE_CASES))
def test_decode_attention_long_context_matches_fp64(name):
    """ops.attn_decode vs tests/test_attn_geometry_cpu.py::decode_reference (fp64), element-wise within its bound (P
    rounded to bf16 before P.V, fp32 sums, output rounding).  Each case states the split count that decode.cu's rule
    (restated in `decode_splits`, and tied to the library through tn_attn_decode_ws_floats) gives for its shapes: the
    benchmark model's generate() (B=1, KV=8, H=24) runs 64 splits; the full ranges put keys in every split, the others
    start and end mid-split and mid-64-key block, have length 1 or are empty (O = 0, LSE = +inf exactly).  Every cache
    row outside a row's range is NaN and must not leak.  Two runs are bit-identical.
    Measured on one H100 80GB HBM3 (SXM, 700 W), largest err/bound over all cases: O 0.08, LSE 0.002."""
    dev = require_cuda()
    H, KV, S_cap, ranges, splits = DECODE_CASES[name]
    B = len(ranges)
    assert decode_splits(B, KV, S_cap) == splits
    assert _lib.load().tn_attn_decode_ws_floats(B, H, KV, S_cap) == B * H * splits * (HD + 2)
    chunk = decode_chunk(B, KV, S_cap)
    for lo, hi in ranges:
        if hi - lo == S_cap:
            assert all(lo < (s + 1) * chunk and s * chunk < hi for s in range(splits)), "a split without keys"
    g = torch.Generator(device=dev).manual_seed(S_cap + H)
    cache = torch.randn(2, B, S_cap, KV * HD, generator=g, device=dev).to(BF16)
    kc, vc = cache[0], cache[1]
    start = torch.tensor([r[0] for r in ranges], dtype=torch.int32, device=dev)
    end = torch.tensor([r[1] for r in ranges], dtype=torch.int32, device=dev)
    for b, (lo, hi) in enumerate(ranges):
        kc[b, :lo] = float("nan"); vc[b, :lo] = float("nan")
        kc[b, hi:] = float("nan"); vc[b, hi:] = float("nan")
    q = torch.randn(B, H * HD, generator=g, device=dev).to(BF16)
    o, lse = ops.attn_decode(q, kc, vc, start, end, H, KV, SCALE, lse=True)
    o2, lse2 = ops.attn_decode(q, kc, vc, start, end, H, KV, SCALE, lse=True)
    torch.cuda.synchronize()
    assert torch.equal(o, o2) and torch.equal(lse, lse2), "two runs differ"
    ro, rlse, ob, lb = decode_reference(q, kc, vc, start, end, H, KV, SCALE)
    empty = torch.tensor([hi <= lo for lo, hi in ranges], device=dev)
    assert torch.all(o[empty] == 0) and torch.all(lse[empty] == math.inf)
    ratios = (_within("o", o, ro, ob), _within("lse", lse[~empty], rlse[~empty], lb[~empty]))
    print("decode", name, f"splits {splits} chunk {chunk}", [f"{x:.3g}" for x in ratios])
