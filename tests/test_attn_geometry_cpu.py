"""Layouts, plain restatements and fp64 references for the attention tests at the benchmark geometry
(tests/test_gpu_bench_geometry.py), and the CPU checks that these helpers are what they claim to be.

  * layout generator  - named packed-document layouts with the edges where block-tiled kernels go wrong (document
                        boundaries at offsets 0, 1, 63, 64, 65, 127 of the 128-row block, length-1 documents, documents
                        over three or more blocks, padding on and off a block boundary, all-padding rows, T = 1000,
                        non-canonical ids) plus the benchmark's own packing, and a seeded random layout generator;
  * AttnPlan contract - `restate_attn_meta` / `meta_offsets` restate, in plain Python, the per-block ranges and the
                        canonical flag documented in touchnet_b200/csrc/attn_common.cuh, and `work_order` the two
                        cost-ordered work lists;
  * fp64 references   - `attention_reference` (O, LSE, dQ/dK/dV by autograd, one document at a time) and
                        `decode_reference` (split-KV decode), each with an element-wise error bound derived from where
                        the kernels round (see `attention_reference`).
"""
import math
import random

import pytest
import torch

from oracle import model_oracle as mo
from touchnet_b200 import batching

BLK, SUB, HD = 128, 64, 128          # attention block, streamed sub-block, head_dim (attn_common.cuh)
U_BF16 = 2.0 ** -8                   # unit roundoff of bf16 (8 significant bits, round to nearest)
EPS_ACC = 2.0 ** -23                 # error per fp32 accumulation step, one ulp (tensor-core adds need not round to nearest)
E_DOT = 2.0 ** -15                   # relative error of a 128-term fp32 dot product (128 * 2^-23 = 2^-16), doubled for the
                                     # fp32 multiply by the log2-domain scale and the ex2.approx / lg2.approx instructions
E_TRANSC = 2.0 ** -20                # absolute error of ex2.approx + lg2.approx in the log-sum-exp


# ---------------------------------------------------------------------------------------------------------------
# layouts: [B, T] int64 document ids (0 = padding)
# ---------------------------------------------------------------------------------------------------------------
def ids_from_runs(T, runs):
    """Row of length T from (id, length) runs laid end to end; the rest is padding."""
    ids = []
    for i, n in runs:
        ids += [i] * n
    assert len(ids) <= T, (len(ids), T)
    return ids + [0] * (T - len(ids))


def ids_from_cuts(T, cuts, pad_from):
    """Documents 1, 2, ... starting at 0 and at every cut; padding from `pad_from`."""
    edges = [0] + list(cuts) + [pad_from]
    return ids_from_runs(T, [(i + 1, edges[i + 1] - edges[i]) for i in range(len(edges) - 1)])


# Document starts at 1, 63, 64, 65, 127, 128, 129, ... (offsets 0, 1, 63, 64, 65, 127 mod 128); length-1 documents at
# [0,1), [63,64), [64,65), [127,128), [128,129), [639,640); [129,577) covers blocks 1..4; padding from 961 (offset 65).
EDGE_CUTS = [1, 63, 64, 65, 127, 128, 129, 577, 639, 640, 897]
EDGE_PAD = 961


def layout_rows(name):
    """(T, rows) of a named layout set (every set has B > 1 rows with different layouts except 'bench')."""
    T = 1000                                                                      # not a multiple of 64
    if name == "edges":
        return T, [ids_from_cuts(T, EDGE_CUTS, EDGE_PAD),
                   ids_from_runs(T, [(1, 300), (2, 84)]),                         # padding from 384 = 3 * 128
                   [0] * T]                                                       # all padding
    if name == "noncanonical":
        return T, [[0] * 200 + [1] * 800,                                         # left padding, as in prefill
                   ids_from_runs(T, [(1, 300), (0, 33), (1, 367), (2, 300)]),    # id 1 again after padding
                   ids_from_runs(T, [(3, 130), (2, 370), (1, 499)])]             # decreasing ids, one padding row
    if name == "mixed":
        return T, [[1] * T,                                                       # one document over all 8 blocks
                   ids_from_runs(T, [(1, 100), (2, 100), (1, 200), (3, 65), (2, 500)])]  # ids interleaved
    if name == "bench":
        return 8192, [bench_doc_ids()[0][0].tolist()]
    raise KeyError(name)


LAYOUT_SETS = ("edges", "noncanonical", "mixed", "bench")


def layout(name):
    T, rows = layout_rows(name)
    return torch.tensor(rows, dtype=torch.int64)


def run_positions(doc):
    """Position of every token inside its run of equal non-zero ids (0 on padding): the RoPE positions."""
    B, T = doc.shape
    pos = torch.zeros(B, T, dtype=torch.int64)
    for b in range(B):
        ids = doc[b].tolist()
        p = 0
        for t in range(T):
            p = p + 1 if t > 0 and ids[t] == ids[t - 1] else 0
            pos[b, t] = p if ids[t] > 0 else 0
    return pos


_BENCH = {}


def bench_doc_ids(seed=2025):
    """Document ids and positions of the benchmark's packing (bench.py::make_host_batch, B=1, T=8192)."""
    if seed not in _BENCH:
        buf, _ = batching.plan_audio_text_batch(seed, 1, 8192, 128256, stride=4, max_s=30.0)
        _BENCH[seed] = (buf["attention_mask"].clone(), buf["position_ids"].clone())
    return _BENCH[seed]


def random_doc_ids(seed):
    """A seeded layout for the AttnPlan metadata comparison: T around the block edges or arbitrary, 1-4 rows, each
    packed (lengths 1, ~64, ~128 or long), padded, all-padding, left-padded, with an id repeated after padding, with
    decreasing ids, or arbitrary small ids."""
    r = random.Random(seed)
    T = r.choice([1, 2, 63, 64, 65, 127, 128, 129, 255, 256, 257, 383, 1000, r.randint(1, 2100), r.randint(1, 2100)])
    rows = []
    for _ in range(r.randint(1, 4)):
        lens, n = [], 0
        while n < T:
            k = r.choice([1, r.randint(2, 9), r.randint(62, 66), r.randint(126, 130), r.randint(100, 900)])
            lens.append(min(k, T - n))
            n += lens[-1]
        ids = []
        for i, k in enumerate(lens):
            ids += [i + 1] * k
        kind = r.choice(["packed", "padded", "padded", "all_pad", "left_pad", "reappear", "decreasing", "random"])
        if kind == "padded":
            cut = r.randint(0, T)
            ids = ids[:cut] + [0] * (T - cut)
        elif kind == "all_pad":
            ids = [0] * T
        elif kind == "left_pad":
            cut = r.randint(1, T)
            ids = [0] * cut + [1] * (T - cut)
        elif kind == "reappear":
            a = r.randint(0, T)
            b = r.randint(a, T)
            ids = ids[:a] + [0] * (b - a) + [ids[a - 1] if a > 0 else 1] * (T - b)
        elif kind == "decreasing":
            top = max(ids) + 1
            ids = [top - i for i in ids]
        elif kind == "random":
            ids = []
            while len(ids) < T:
                ids += [r.randint(0, 3)] * r.randint(1, 80)
            ids = ids[:T]
        rows.append(ids)
    return torch.tensor(rows, dtype=torch.int64)


# ---------------------------------------------------------------------------------------------------------------
# AttnPlan metadata, restated from the contract in attn_common.cuh
# ---------------------------------------------------------------------------------------------------------------
def is_canonical(ids):
    """Non-decreasing runs of positive ids followed only by zeros."""
    k = next((t for t, x in enumerate(ids) if x == 0), len(ids))
    head, tail = ids[:k], ids[k:]
    return all(x > 0 for x in head) and all(a <= b for a, b in zip(head, head[1:])) and all(x == 0 for x in tail)


def restate_attn_meta(doc):
    """[B][nblk] tuples (kv_lo, kv_end, q_end, canonical):
      forward / dQ : q block `blk` visits kv blocks [kv_lo, kv_end); kv_end == 0 when every row of the block is padding
      dK / dV      : kv block `blk` is visited by q blocks [blk, q_end); q_end == 0 when no query attends to it
      canonical    : the row's ids are non-decreasing runs followed only by zeros; otherwise the ranges are the whole
                     causal range (kv_lo = 0, kv_end = blk + 1, q_end = nblk) and the kernels mask element-wise.
    For canonical rows kv_lo is the block of the first key of the document of the block's first valid row, q_end the
    block after the last query of the document of its last valid key."""
    B, T = doc.shape
    nblk = (T + BLK - 1) // BLK
    out = []
    for b in range(B):
        ids = doc[b].tolist()
        canon = int(is_canonical(ids))
        start, end = [0] * T, [0] * T
        for t in range(T):
            start[t] = start[t - 1] if t > 0 and ids[t] == ids[t - 1] else t
        for t in reversed(range(T)):
            end[t] = end[t + 1] if t + 1 < T and ids[t] == ids[t + 1] else t + 1
        row = []
        for blk in range(nblk):
            valid = [t for t in range(blk * BLK, min(T, (blk + 1) * BLK)) if ids[t] > 0]
            if not valid:
                row.append((0, 0, 0, canon))
            elif not canon:
                row.append((0, blk + 1, nblk, canon))
            else:
                row.append((start[valid[0]] // BLK, blk + 1, (end[valid[-1]] + BLK - 1) // BLK, canon))
        out.append(row)
    return out


def meta_offsets(B, T):
    """int32 offsets of the parts of AttnPlan.meta: AttnMeta[B*nblk], flags[B] (padded to 4), the per-position extent
    table (B*nblk*128 pairs), order_q[B*nblk], order_kv[B*nblk]."""
    nblk = (T + BLK - 1) // BLK
    flags = B * nblk * 4
    seg = (flags + B + 3) // 4 * 4
    order_q = seg + B * nblk * BLK * 2
    order_kv = order_q + B * nblk
    return {"nblk": nblk, "flags": flags, "order_q": order_q, "order_kv": order_kv, "total": order_kv + B * nblk}


def work_order(meta_rows):
    """The two cost-ordered work lists over entries b*nblk + blk, heaviest first, ties by entry index:
    order_q by kv_end - kv_lo (forward, dQ), order_kv by max(q_end - blk, 0) (dK/dV)."""
    flat = [(blk, m) for row in meta_rows for blk, m in enumerate(row)]
    cq = [m[1] - m[0] for _, m in flat]
    ckv = [max(m[2] - blk, 0) for blk, m in flat]
    n = len(flat)
    return sorted(range(n), key=lambda i: (-cq[i], i)), sorted(range(n), key=lambda i: (-ckv[i], i))


# ---------------------------------------------------------------------------------------------------------------
# fp64 references with element-wise error bounds
# ---------------------------------------------------------------------------------------------------------------
def rope_fp64(x, cos, sin):
    """hf apply_rotary_pos_emb (half split) on x [..., n, 128] with [n, 64] tables, in fp64."""
    c, s = cos.double(), sin.double()
    lo, hi = x[..., :64], x[..., 64:]
    return torch.cat([lo * c - hi * s, hi * c + lo * s], -1)


def rope_vjp(g, cos, sin):
    """Gradient w.r.t. the un-rotated input, through RoPE with these tables (autograd of rope_fp64)."""
    u = torch.zeros_like(g, requires_grad=True)
    with torch.enable_grad():
        return torch.autograd.grad(rope_fp64(u, cos, sin), u, g)[0]


def _abs_rope_t(b, cos, sin):
    """|R|^T applied to a non-negative bound: what a bound on the rotated gradient becomes after the inverse rotation."""
    c, s = cos.double().abs(), sin.double().abs()
    lo, hi = b[..., :64], b[..., 64:]
    return torch.cat([lo * c + hi * s, lo * s + hi * c], -1)


def attention_reference(q, k, v, do, doc, H, KV, scale, rope=None):
    """fp64 document attention on the bf16 operands, one document (one id value) at a time:
    allow[q, k] = (q >= k) & (doc[q] == doc[k]) & (doc[q] > 0).  q/do [B*T, H*128], k/v [B*T, KV*128] (any row stride);
    rope = (cos, sin) [B*T, 64]: dQ/dK are returned w.r.t. the un-rotated q/k (the kernels' epilogue contract).
    Returns a dict of o, lse, dq, dk, dv and, for each, an element-wise bound `<name>_bound` on |kernel - reference|.
    Padding queries: O = 0, LSE = +inf, dQ = 0; keys no query attends: dK = dV = 0 (bounds 0: exact).

    Bounds.  u = 2^-8 (bf16), n_i = keys of query row i, N = G * document length (terms of a dK/dV sum), all products
    fp32-accumulated (error n * 2^-23 relative to the sum of magnitudes), A = scale * |Q||K|^T:
      e_s,i   = 2^-15 * max_j A_ij                                error of the fp32 logits of row i (128-term dots)
      e_p,i   = u + n_i 2^-23 + 2 e_s,i                           relative error of P as rounded to bf16 for P.V
      O       : e_p,i (P|V|)_ic + u |O_ic|                        P rounding, accumulation, output rounding
      LSE     : e_s,i + n_i 2^-23 + 2^-20 + 2^-23 |lse_i|         logits, sum of exponentials, ex2 / lg2 approximations
      e_b,i   = e_p,i + LSE bound_i                               P recomputed in the backward from the forward's LSE
      Δδ_i    = sum_c |dO_ic| O bound_ic + 2^-16 (|dO||O|)_i      delta = rowsum(dO * O) from the bf16 O
      ΔdS_ij  = (u + e_b,i)|dS_ij| + P_ij (2^-16 (|dO||V|^T)_ij + Δδ_i)     dS = P (dP - delta), rounded to bf16
      dQ      : scale (ΔdS|K| + n_i 2^-23 |dS||K|) + u |dQ|
      dK      : scale (ΔdS^T|Q| + N 2^-23 |dS|^T|Q|) + u |dK|     (summed over the G heads of the group)
      dV      : (e_b P)^T|dO| + N 2^-23 P^T|dO| + u |dV|
    With rope the dQ/dK bounds before output rounding go through |R|^T and the output term is u |R|^T|g|.  These are
    worst-case sums of magnitudes; the kernels' errors are random-signed and land well inside (see the GPU tests)."""
    B, T = doc.shape
    G = H // KV
    dev = q.device
    f64 = torch.float64
    rows_all = B * T
    r = {"o": torch.zeros(rows_all, H, HD, dtype=f64, device=dev), "lse": torch.full((B, H, T), math.inf, dtype=f64, device=dev),
         "dq": torch.zeros(rows_all, H, HD, dtype=f64, device=dev), "dk": torch.zeros(rows_all, KV, HD, dtype=f64, device=dev),
         "dv": torch.zeros(rows_all, KV, HD, dtype=f64, device=dev)}
    for name in list(r):
        r[name + "_bound"] = torch.zeros_like(r[name]) if name != "lse" else torch.zeros(B, H, T, dtype=f64, device=dev)
    for b in range(B):
        d = doc[b]
        for i in torch.unique(d[d > 0]).tolist():
            idx = (d == i).nonzero().squeeze(1)
            rows = b * T + idx
            n = idx.numel()
            Q = q[rows].to(f64).view(n, H, HD).transpose(0, 1).detach().requires_grad_(True)
            K = k[rows].to(f64).view(n, KV, HD).transpose(0, 1).detach().requires_grad_(True)
            V = v[rows].to(f64).view(n, KV, HD).transpose(0, 1).detach().requires_grad_(True)
            dO = do[rows].to(f64).view(n, H, HD).transpose(0, 1)
            causal = torch.ones(n, n, dtype=torch.bool, device=dev).tril()
            with torch.enable_grad():
                Kg, Vg = K.repeat_interleave(G, 0), V.repeat_interleave(G, 0)
                S = (Q @ Kg.transpose(1, 2) * scale).masked_fill(~causal, -math.inf)
                lse = torch.logsumexp(S, -1)
                P = torch.exp(S - lse[..., None])
                O = P @ Vg
                O.backward(dO)
            with torch.no_grad():
                Q0, K0, Kg, Vg, S, P, O = Q.detach(), K.detach(), Kg.detach(), Vg.detach(), S.detach(), P.detach(), O.detach()
                aQ, aK, aV, adO = Q0.abs(), Kg.abs(), Vg.abs(), dO.abs()
                n_i = torch.arange(1, n + 1, device=dev, dtype=f64)                        # keys of each query row
                N = G * n * EPS_ACC
                e_s = E_DOT * (scale * (aQ @ aK.transpose(1, 2))).masked_fill(~causal, 0).amax(-1)   # [H, n]
                e_p = U_BF16 + n_i * EPS_ACC + 2 * e_s
                o_b = e_p[..., None] * (P @ aV) + U_BF16 * O.abs()
                lse_b = e_s + n_i * EPS_ACC + E_TRANSC + EPS_ACC * lse.abs()
                e_b = e_p + lse_b
                dS = P * (dO @ Vg.transpose(1, 2) - (dO * O).sum(-1)[..., None])
                aS = dS.abs()
                ddelta = (adO * o_b).sum(-1) + 2 * E_DOT * (adO * O.abs()).sum(-1)
                ddS = (U_BF16 + e_b)[..., None] * aS + P * (2 * E_DOT * (adO @ aV.transpose(1, 2)) + ddelta[..., None])
                dq_b = scale * (ddS @ aK + (n_i * EPS_ACC)[:, None] * (aS @ aK))
                dk_b = (scale * (ddS.transpose(1, 2) @ aQ + N * (aS.transpose(1, 2) @ aQ))).view(KV, G, n, HD).sum(1)
                dv_b = ((e_b[..., None] * P).transpose(1, 2) @ adO + N * (P.transpose(1, 2) @ adO)).view(KV, G, n, HD).sum(1)
                dq, dk, dv = Q.grad, K.grad, V.grad
                tok = lambda x: x.transpose(0, 1)                                             # [heads, n, 128] -> [n, heads, 128]
                if rope is not None:
                    c, s = rope[0][rows][:, None], rope[1][rows][:, None]
                    dq_rot, dk_rot = tok(dq), tok(dk)
                    r["dq"][rows] = rope_vjp(dq_rot, c, s)
                    r["dk"][rows] = rope_vjp(dk_rot, c, s)
                    r["dq_bound"][rows] = _abs_rope_t(tok(dq_b) + U_BF16 * dq_rot.abs(), c, s)
                    r["dk_bound"][rows] = _abs_rope_t(tok(dk_b) + U_BF16 * dk_rot.abs(), c, s)
                else:
                    r["dq"][rows] = tok(dq)
                    r["dk"][rows] = tok(dk)
                    r["dq_bound"][rows] = tok(dq_b) + U_BF16 * tok(dq).abs()
                    r["dk_bound"][rows] = tok(dk_b) + U_BF16 * tok(dk).abs()
                r["dv"][rows] = tok(dv)
                r["dv_bound"][rows] = tok(dv_b) + U_BF16 * tok(dv).abs()
                r["o"][rows] = tok(O)
                r["o_bound"][rows] = tok(o_b)
                r["lse"][b][:, idx] = lse
                r["lse_bound"][b][:, idx] = lse_b
    for name in ("o", "dq"):
        r[name] = r[name].view(rows_all, H * HD)
        r[name + "_bound"] = r[name + "_bound"].view(rows_all, H * HD)
    for name in ("dk", "dv"):
        r[name] = r[name].view(rows_all, KV * HD)
        r[name + "_bound"] = r[name + "_bound"].view(rows_all, KV * HD)
    return r


def decode_reference(q, k_cache, v_cache, kv_start, kv_end, H, KV, scale):
    """fp64 attention of one query row per batch row over cache rows [start, end): (o [B, H*128], lse [B, H],
    o_bound, lse_bound) with the bounds of `attention_reference` for n = end - start keys (an empty range: O = 0,
    LSE = +inf, exact)."""
    B = q.shape[0]
    G = H // KV
    f64 = torch.float64
    dev = q.device
    o = torch.zeros(B, H, HD, dtype=f64, device=dev)
    o_b = torch.zeros_like(o)
    lse = torch.full((B, H), math.inf, dtype=f64, device=dev)
    lse_b = torch.zeros(B, H, dtype=f64, device=dev)
    for b in range(B):
        lo, hi = int(kv_start[b]), int(kv_end[b])
        if hi <= lo:
            continue
        n = hi - lo
        K = k_cache[b, lo:hi].to(f64).view(n, KV, HD).transpose(0, 1).repeat_interleave(G, 0)   # [H, n, 128]
        V = v_cache[b, lo:hi].to(f64).view(n, KV, HD).transpose(0, 1).repeat_interleave(G, 0)
        Q = q[b].to(f64).view(H, 1, HD)
        S = (Q @ K.transpose(1, 2) * scale)[:, 0]                                                # [H, n]
        l = torch.logsumexp(S, -1)
        P = torch.exp(S - l[:, None])
        O = (P[:, None] @ V)[:, 0]
        e_s = E_DOT * (scale * (Q.abs() @ K.abs().transpose(1, 2)))[:, 0].amax(-1)
        e_p = U_BF16 + n * EPS_ACC + 2 * e_s
        o[b], lse[b] = O, l
        o_b[b] = e_p[:, None] * (P[:, None] @ V.abs())[:, 0] + U_BF16 * O.abs()
        lse_b[b] = e_s + n * EPS_ACC + E_TRANSC + EPS_ACC * l.abs()
    return o.view(B, H * HD), lse, o_b.view(B, H * HD), lse_b


# ---------------------------------------------------------------------------------------------------------------
# CPU checks of the helpers
# ---------------------------------------------------------------------------------------------------------------
def _doc_starts(ids):
    return [t for t in range(len(ids)) if ids[t] > 0 and (t == 0 or ids[t - 1] != ids[t])]


def test_layouts_cover_the_block_edges():
    T, (edge, pad_on, all_pad) = layout_rows("edges")
    assert T % SUB != 0
    starts = _doc_starts(edge)
    assert {s % BLK for s in starts} >= {0, 1, 63, 64, 65, 127}
    assert {128, 129} <= set(starts)
    runs = [(s, next((t for t in range(s, T) if edge[t] != edge[s]), T)) for s in starts]
    assert sum(1 for s, e in runs if e - s == 1) >= 5                                  # length-1 documents
    assert any(e // BLK - s // BLK >= 3 for s, e in runs)                              # over three or more blocks
    assert EDGE_PAD % BLK != 0 and edge[EDGE_PAD - 1] > 0 and set(edge[EDGE_PAD:]) == {0}   # padding off a boundary
    assert pad_on[383] > 0 and set(pad_on[384:]) == {0}                                # padding on a boundary
    assert set(all_pad) == {0}
    for name in ("noncanonical", "mixed"):
        T, rows = layout_rows(name)
        assert len(rows) > 1 and len({tuple(r) for r in rows}) == len(rows)
    T, (left, reap, dec) = layout_rows("noncanonical")
    assert left[0] == 0 and left[-1] == 1 and not is_canonical(left)
    assert reap[299] == 1 and reap[300] == 0 and reap[333] == 1 and not is_canonical(reap)
    assert dec[0] > dec[200] > dec[600] and not is_canonical(dec)
    assert is_canonical(edge) and is_canonical(pad_on) and is_canonical(all_pad)


def test_bench_layout_is_the_benchmark_packing():
    doc, pos = bench_doc_ids()
    assert doc.shape == (1, 8192)
    ids = doc[0].tolist()
    assert is_canonical(ids) and ids[-1] == 0                                          # a padding tail
    lens = [ids.count(i) for i in set(ids) - {0}]
    assert len(lens) >= 5 and max(lens) <= 1100                                        # documents of at most ~1000 tokens
    assert torch.equal(run_positions(doc), pos)


def test_meta_restatement_matches_hand_derived_ranges():
    """docs [0,300) [300,800) [800,900), padding [900,1024): the ranges test_gpu_attention.py checks on the GPU."""
    doc = torch.tensor([ids_from_runs(1024, [(1, 300), (2, 500), (3, 100)])])
    m = restate_attn_meta(doc)[0]
    assert m[2][:2] == (0, 3) and m[3][:2] == (2, 4) and m[6][:2] == (2, 7) and m[7][:2] == (6, 8)
    assert m[2][2] == 7 and m[0][2] == 3 and m[7][2] == 8 and all(x[3] == 1 for x in m)
    left = restate_attn_meta(torch.tensor([[0] * 200 + [1] * 56]))[0]
    assert left == [(0, 0, 0, 0), (0, 2, 2, 0)]                                       # block 0 is all padding
    assert restate_attn_meta(torch.zeros(1, 129, dtype=torch.int64))[0] == [(0, 0, 0, 1), (0, 0, 0, 1)]
    oq, okv = work_order(restate_attn_meta(doc))
    assert sorted(oq) == list(range(8)) and oq[0] == 6                                 # block 6 visits 5 kv blocks


def test_random_layouts_cover_every_kind():
    kinds = {"canonical": 0, "noncanonical": 0, "all_pad": 0, "partial_block": 0}
    for seed in range(300):
        doc = random_doc_ids(seed)
        for row in doc.tolist():
            kinds["canonical" if is_canonical(row) else "noncanonical"] += 1
            kinds["all_pad"] += set(row) == {0}
        kinds["partial_block"] += doc.shape[1] % BLK != 0
    assert min(kinds.values()) >= 20, kinds


def _small_case(seed, B=2, T=150, H=4, KV=2):
    g = torch.Generator().manual_seed(seed)
    doc = torch.tensor([ids_from_runs(T, [(1, 1), (2, 70), (3, 60)]), [0] * 20 + [1] * 60 + [0] * 10 + [1] * 60])
    mk = lambda c: torch.randn(B * T, c * HD, generator=g).bfloat16()
    return doc, mk(H), mk(KV), mk(KV), mk(H), H, KV


def test_attention_reference_matches_the_oracle():
    """fp64 reference vs oracle/model_oracle.py::attention (dense mask, fp32) and its autograd, with and without RoPE."""
    doc, q, k, v, do, H, KV = _small_case(0)
    B, T = doc.shape
    scale = HD ** -0.5
    pos = run_positions(doc)
    inv, sc = mo.rope_inv_freq(mo.OracleConfig(256, 8, 1, H, KV, HD, 8, rope_theta=500000.0))
    cos, sin = mo.rope_cos_sin(pos, inv, sc, torch.bfloat16)
    cos, sin = cos[..., :64].reshape(B * T, 64), sin[..., :64].reshape(B * T, 64)
    for rope in (None, (cos, sin)):
        ref = attention_reference(q, k, v, do, doc, H, KV, scale, rope)
        qf = q.float().view(B, T, H, HD).transpose(1, 2).requires_grad_(True)
        kf = k.float().view(B, T, KV, HD).transpose(1, 2).requires_grad_(True)
        vf = v.float().view(B, T, KV, HD).transpose(1, 2).requires_grad_(True)
        o, lse = mo.attention(qf, kf, vf, mo.doc_causal_allow(doc), scale)
        o.backward(do.float().view(B, T, H, HD))
        gq, gk = qf.grad, kf.grad
        if rope is not None:   # q/k are the rotated operands: back through the oracle's RoPE to the un-rotated ones
            c = torch.cat([cos, cos], -1).float().view(B, T, HD)
            s = torch.cat([sin, sin], -1).float().view(B, T, HD)
            uq, uk = torch.zeros_like(qf, requires_grad=True), torch.zeros_like(kf, requires_grad=True)
            gq, gk = torch.autograd.grad(mo.apply_rope(uq, uk, c, s), (uq, uk), (gq, gk))
        gq = gq.transpose(1, 2).reshape(B * T, -1)
        gk = gk.transpose(1, 2).reshape(B * T, -1)
        valid = (doc > 0)[:, None, :].expand(B, H, T)
        assert torch.allclose(ref["o"].float(), o.reshape(B * T, -1), atol=1e-5)
        assert torch.allclose(ref["lse"][valid].float(), lse[valid], atol=1e-5)
        assert torch.isinf(ref["lse"][~valid]).all() and torch.isinf(lse[~valid]).all()
        assert torch.allclose(ref["dq"].float(), gq, atol=1e-4)
        assert torch.allclose(ref["dk"].float(), gk, atol=1e-4)
        assert torch.allclose(ref["dv"].float(), vf.grad.transpose(1, 2).reshape(B * T, -1), atol=1e-4)
        assert torch.all(ref["dq"][(doc == 0).reshape(-1)] == 0)


def _kernel_like_forward(q, k, v, doc, H, KV, scale, drop_last_key_of_subblock=False):
    """The forward's rounding points restated in fp32: unnormalised P rounded to bf16 before P.V, fp32 row sums,
    output rounded to bf16; optionally with the last key of every non-final 64-key sub-block dropped."""
    B, T = doc.shape
    G = H // KV
    o = torch.zeros(B * T, H, HD)
    for b in range(B):
        d = doc[b]
        for i in torch.unique(d[d > 0]).tolist():
            idx = (d == i).nonzero().squeeze(1)
            n, rows = idx.numel(), b * T + idx
            Q = q[rows].float().view(n, H, HD).transpose(0, 1)
            K = k[rows].float().view(n, KV, HD).transpose(0, 1).repeat_interleave(G, 0)
            V = v[rows].float().view(n, KV, HD).transpose(0, 1).repeat_interleave(G, 0)
            allow = torch.ones(n, n, dtype=torch.bool).tril()
            if drop_last_key_of_subblock:
                last = (idx % SUB == SUB - 1) & (idx // SUB < idx.max() // SUB)
                allow &= ~last[None, :]
            S = (Q @ K.transpose(1, 2) * scale).masked_fill(~allow, -math.inf)
            p = torch.exp(S - S.amax(-1, keepdim=True))
            o[rows] = ((p.bfloat16().float() @ V) / p.sum(-1, keepdim=True)).bfloat16().float().transpose(0, 1)
    return o.view(B * T, H * HD)


def test_output_bound_holds_for_the_rounding_it_models_and_fails_for_a_dropped_key():
    doc, q, k, v, do, H, KV = _small_case(1)
    scale = HD ** -0.5
    ref = attention_reference(q, k, v, do, doc, H, KV, scale)
    err = (_kernel_like_forward(q, k, v, doc, H, KV, scale).double() - ref["o"]).abs()
    assert (err <= ref["o_bound"]).all(), float((err / ref["o_bound"].clamp_min(1e-300)).max())
    bad = (_kernel_like_forward(q, k, v, doc, H, KV, scale, True).double() - ref["o"]).abs()
    assert (bad > ref["o_bound"]).any()


def test_decode_reference_matches_softmax():
    g = torch.Generator().manual_seed(3)
    B, S, H, KV = 3, 300, 6, 2
    kc = torch.randn(B, S, KV * HD, generator=g).bfloat16()
    vc = torch.randn(B, S, KV * HD, generator=g).bfloat16()
    q = torch.randn(B, H * HD, generator=g).bfloat16()
    start, end = torch.tensor([0, 17, 40]), torch.tensor([300, 18, 40])
    o, lse, ob, lb = decode_reference(q, kc, vc, start, end, H, KV, HD ** -0.5)
    for b in range(2):
        lo, hi = int(start[b]), int(end[b])
        kk = kc[b, lo:hi].float().view(hi - lo, KV, HD).repeat_interleave(3, 1)
        vv = vc[b, lo:hi].float().view(hi - lo, KV, HD).repeat_interleave(3, 1)
        s = torch.einsum("hd,shd->hs", q[b].float().view(H, HD), kk) * HD ** -0.5
        assert torch.allclose(lse[b].float(), torch.logsumexp(s, -1), atol=1e-5)
        assert torch.allclose(o[b].float(), torch.einsum("hs,shd->hd", s.softmax(-1), vv).reshape(-1), atol=1e-5)
    assert torch.all(o[2] == 0) and torch.isinf(lse[2]).all() and torch.all(ob[2] == 0)
    assert (ob[:2] > 0).all() and (lb[:2] > 0).all()
