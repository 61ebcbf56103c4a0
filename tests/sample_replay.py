"""Exact CPU replay of the draws of tn_sample_select_slots_bf16 and tn_spec_sample_verify_bf16 (DESIGN §3.4): a
restatement, in numpy and Python integers, of what the kernels compute, so that the GPU tests can check every draw
token for token instead of by its statistics.

The kernels are integer machines except for one instruction.  A processed logit is IEEE fp32 arithmetic (the bf16 cast,
the repetition penalty, the no-repeat-ngram ban to -inf, x / temperature); the top-k and top-p thresholds are exact
order keys over fixed-point masses; a draw is umulhi(r, Z) over integer prefix sums in index order; an acceptance is an
exact 128-bit compare.  The weight of a token is

    W = cvt.rni.u64(ex2.approx.f32(y) * 2^40),   y = fl(fl(x - m) * 0x3FB8AA3B)   (0x3FB8AA3B = log2(e) in fp32)

and only ex2.approx cannot be reproduced bit for bit.  The replay carries each weight as the interval
[rni(2^(y+40) (1 - EPS)), rni(2^(y+40) (1 + EPS))] with EPS = 2^-22 (2 ulp of an fp32 significand) as the bound on the
relative error of ex2.approx.f32; a kernel weight outside it shows up as a draw outside its predicted set.  Every
result that depends on the weights is therefore a set: one token for almost every draw, more where the draw falls
within a few ulps of a boundary.  The tests bound how often a set has more than one element.

`mut` arguments name deliberately wrong variants of the replay (MUTATIONS); the CPU tests use them to show that a
kernel with that defect would disagree with the true replay on a stated share of the draws."""
import numpy as np

M32 = 0xFFFFFFFF
M64 = (1 << 64) - 1
EPS = 2.0 ** -22
LOG2E_F32 = np.array([0x3FB8AA3B], dtype=np.uint32).view(np.float32)[0]
PLAIN, ACCEPT, RESIDUAL = 0, 1, 2             # Philox purposes

MUTATIONS = ("counter_plus_1", "swap_purposes", "swap_seed_words", "swap_r_words", "value_order", "topk_drop_ties",
             "topp_inclusive", "residual_q_minus_p")


# ---------------------------------------------------------------------------------------------------------------
# Philox4x32-10 (Salmon et al. 2011), vectorised over rows in uint64 arithmetic
# ---------------------------------------------------------------------------------------------------------------
def philox4x32_10(ctr, key):
    """ctr: 4 words, key: 2 words (ints or arrays of values < 2^32) -> the 4 output words as uint64 arrays."""
    m = np.uint64(M32)
    c = [np.asarray(w, dtype=np.uint64) & m for w in ctr]
    k0, k1 = (np.asarray(w, dtype=np.uint64) & m for w in key)
    for i in range(10):
        if i:
            k0 = (k0 + np.uint64(0x9E3779B9)) & m
            k1 = (k1 + np.uint64(0xBB67AE85)) & m
        p0 = np.uint64(0xD2511F53) * c[0]     # 32 x 32 -> 64 bits: exact in uint64
        p1 = np.uint64(0xCD9E8D57) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & m, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & m]
    return c


def draw_bits(seed, pos, purpose, key, mut=()):
    """The kernels' 64 random bits r for (seed, position, purpose, stream key): Philox4x32-10 at counter (pos, purpose,
    key lo, key hi) under key (seed lo, seed hi), r = (out.y << 32) | out.x.  seed is a Python int (its two's-complement
    bits), pos and key ints or int64 arrays.  Returns uint64 (an array when pos or key is one)."""
    s = int(seed) & M64
    pos = np.asarray(pos, dtype=np.int64) + (1 if "counter_plus_1" in mut else 0)
    ku = np.asarray(key, dtype=np.int64).astype(np.uint64)
    sk = (s >> 32, s & M32) if "swap_seed_words" in mut else (s & M32, s >> 32)
    out = philox4x32_10((pos.astype(np.uint64), purpose, ku, ku >> np.uint64(32)), sk)
    hi, lo = (out[0], out[1]) if "swap_r_words" in mut else (out[1], out[0])
    return (hi << np.uint64(32)) | lo


# ---------------------------------------------------------------------------------------------------------------
# the processed row and its kept sets
# ---------------------------------------------------------------------------------------------------------------
def processed(row, hist, penalty=1.0, ngram=0, temperature=1.0):
    """fp32 [V] values of one logits row (fp32 of its bf16 values) after the repetition penalty and the no-repeat-ngram
    ban over the history ids `hist`, then x / temperature (skipped at 1), each step in fp32 as the kernels do it."""
    x = np.array(row, dtype=np.float32)
    V = x.size
    h = np.asarray(hist, dtype=np.int64)
    n = h.size
    with np.errstate(all="ignore"):
        p = np.float32(penalty)
        if p != 1:
            ids = np.unique(h[(h >= 0) & (h < V)])
            v = x[ids]
            x[ids] = np.where(v < 0, v * p, v / p)
        if ngram > 0 and n + 1 >= ngram:
            if ngram == 1:
                banned = h
            elif n >= ngram:
                win = np.lib.stride_tricks.sliding_window_view(h, ngram)
                banned = win[(win[:, :-1] == h[n - ngram + 1:]).all(1), -1]
            else:
                banned = h[:0]
            x[banned[(banned >= 0) & (banned < V)]] = -np.inf
        t = np.float32(temperature)
        if t != 1:
            x = x / t
    return x.astype(np.float32)


def order_key(x):
    """The kernels' order-preserving uint32 key of fp32 values (-0 and +0 share one key)."""
    x = np.where(np.asarray(x, dtype=np.float32) == 0, np.float32(0), x).astype(np.float32)
    u = x.view(np.uint32)
    return np.where(u >> np.uint32(31) != 0, ~u, u | np.uint32(0x80000000)).astype(np.uint32)


def argmax_pick(x):
    """argmax_better's pick: a NaN above every number, then the larger value, ties to the lowest index."""
    nan = np.isnan(x)
    return int(np.argmax(nan)) if nan.any() else int(np.argmax(x))


def weight_bounds(x, m):
    """[lo, hi] int64 of each token's fixed-point weight W = rni(ex2.approx(y) * 2^40) (module docstring)."""
    with np.errstate(all="ignore"):
        y = ((x - np.float32(m)).astype(np.float32) * LOG2E_F32).astype(np.float32)
        t = np.exp2(y.astype(np.float64) + 40.0)
    e = EPS + 2.0 ** -50                      # and the fp64 rounding of t
    return np.rint(t * (1 - e)).astype(np.int64), np.rint(t * (1 + e)).astype(np.int64)


class Dist:
    """The sampling distribution of one processed row.  degenerate: the row's maximum is not finite (a NaN, an infinite
    maximum, every token banned) and `pick` is argmax_better's pick.  Otherwise `cuts` lists the possible kept sets
    (bool [V]; more than one only where the top-p cut is within the weights' error of its threshold), `lo` / `hi` the
    weight bounds of every token, and `values` the processed row."""

    def __init__(self, x, top_k, top_p, mut=()):
        self.values = x
        self.pick = argmax_pick(x)
        m = x[self.pick]
        self.degenerate = not np.isfinite(m)
        if self.degenerate:
            return
        V = x.size
        key = order_key(x)
        kept = np.ones(V, dtype=bool)
        if 0 < top_k < V:
            if "topk_drop_ties" in mut:                               # exactly k: ties at the boundary by index
                kept = np.zeros(V, dtype=bool)
                kept[np.argsort(~key, kind="stable")[:top_k]] = True
            else:
                kept = key >= np.partition(key, V - top_k)[V - top_k]
        self.lo, self.hi = weight_bounds(x, m)
        tp = np.float32(top_p)
        if not tp < 1:
            self.cuts = [kept]
        elif tp <= 0:
            self.cuts = [kept & (key >= order_key(m))]                # the tied maxima
        else:
            self.cuts = [kept & (key >= t) for t in _top_p_cuts(key, kept, self.lo, self.hi, tp, mut)]
        self._order = np.argsort(~key, kind="stable") if "value_order" in mut else None
        self._prefix = {}

    def weights(self, c):
        """(lo, hi) weight bounds under cut c (0 outside it)."""
        kept = self.cuts[c]
        return np.where(kept, self.lo, 0), np.where(kept, self.hi, 0)

    def draw(self, r):
        """The set of tokens the draw with random bits r can give, over every possible cut."""
        if self.degenerate:
            return {self.pick}
        out = set()
        for c in range(len(self.cuts)):
            if c not in self._prefix:
                self._prefix[c] = _Prefix(*self.weights(c), self._order)
            out |= self._prefix[c].draw(int(r))
        return out


def _top_p_cuts(key, kept, lo, hi, top_p, mut):
    """Possible threshold keys of the top-p cut over the kept set: the lowest value group whose kept mass strictly
    above it is < need = ceil(top_p * Z) (fp64 product, as the kernel computes it), with the masses as intervals."""
    ks = key[kept]
    order = np.argsort(~ks, kind="stable")                            # descending value
    ks, l, h = ks[order], lo[kept][order], hi[kept][order]
    starts = np.flatnonzero(np.r_[True, ks[1:] != ks[:-1]])
    gk, gl, gh = ks[starts], np.add.reduceat(l, starts), np.add.reduceat(h, starts)
    ZL, ZH = int(gl.sum()), int(gh.sum())
    nL, nH = (int(np.ceil(np.float64(top_p) * float(z))) for z in (ZL, ZH))
    AL = np.cumsum(gl) - gl                                           # kept mass strictly above each group
    AH = np.cumsum(gh) - gh
    if "topp_inclusive" in mut:                                       # keep a group only if it fits entirely
        AL, AH = AL + gl, AH + gh
        AL[0] = AH[0] = 0                                             # the row maximum always stays
        may, must = AL <= nH, AH <= nL
    else:
        may, must = AL < nH, AH < nL
    G = gk.size
    return [gk[g] for g in range(G) if may[g] and (g == G - 1 or not must[g + 1])]


class _Prefix:
    """Index-order (or `order`) prefix sums of interval weights, and the draw over them.  Token i (in draw order) holds
    the target floor(r Z / 2^64) iff r (w + S) >= (2^64 - r) P and r S < (2^64 - r)(P + w), with P the weight before it,
    w its own and S the weight after it (Z = P + w + S); with P, w and S in their intervals it can hold the target iff
    (2^64 - r) P_lo <= r (S_hi + w_hi) and (2^64 - r)(P_hi + w_hi) > r S_lo.  Both sides are monotone in i."""

    def __init__(self, lo, hi, order=None):
        self.idx = np.arange(lo.size) if order is None else order
        lo, hi = lo[self.idx], hi[self.idx]
        if lo.dtype != object and int(hi.sum()) >= 1 << 62:
            lo, hi = lo.astype(object), hi.astype(object)
        self.hi = hi
        self.PL = np.cumsum(lo) - lo                                  # weight before, low
        self.PHi = np.cumsum(hi)                                      # weight before and own, high
        self.SLx = lo.sum() - np.cumsum(lo)                           # weight after, low
        self.SHi = hi.sum() - self.PHi + hi                           # weight after and own, high

    def draw(self, r):
        a, n = (1 << 64) - r, self.hi.size
        f1 = lambda i: a * int(self.PL[i]) <= r * int(self.SHi[i])     # noqa: E731  true up to some index
        f2 = lambda i: a * int(self.PHi[i]) > r * int(self.SLx[i])     # noqa: E731  true from some index
        lo_, hi_ = 0, n                                               # i1 = the last i with f1
        while lo_ < hi_:
            mid = (lo_ + hi_) // 2
            lo_, hi_ = (mid + 1, hi_) if f1(mid) else (lo_, mid)
        i1 = lo_ - 1
        lo_, hi_ = 0, n                                               # i2 = the first i with f2
        while lo_ < hi_:
            mid = (lo_ + hi_) // 2
            lo_, hi_ = (lo_, mid) if f2(mid) else (mid + 1, hi_)
        i2 = lo_
        if i2 > i1:
            return set()
        cand = i2 + np.flatnonzero(np.asarray(self.hi[i2:i1 + 1] > 0, dtype=bool))
        return {int(self.idx[i]) for i in cand}


# ---------------------------------------------------------------------------------------------------------------
# tn_sample_select_slots_bf16
# ---------------------------------------------------------------------------------------------------------------
def select_commit(state, b, tok, length, eos, key=None):
    """sample_select_slots' writes for advancing slot b (state: dict of numpy arrays, changed in place)."""
    if length < state["history"].shape[1]:
        state["history"][b, length] = tok
    state["next_ids"][b] = tok
    state["length"][b] = length + 1
    state["positions"][b] += 1
    if tok == eos or length + 1 == state["limit"][b]:
        state["finished"][b] = 1
    if key is not None:
        state["stream_key"][b] = key


# ---------------------------------------------------------------------------------------------------------------
# tn_spec_sample_verify_bf16 (Leviathan et al. 2023, Algorithm 1)
# ---------------------------------------------------------------------------------------------------------------
def _mulhi(r, X):
    return (r * X) >> 64


def spec_position(p_row, q_row, hist, x, seed, pos, key, knobs, mut=()):
    """The possible picks of one verify position: x (the draft token at this position, None at j = k) accepted, or ~t
    for an emitted token t.  hist: the slot's history followed by the draft tokens before this position; pos: its
    length (the counter position); knobs: (penalty, ngram, temperature, top_k, top_p)."""
    penalty, ngram, t, top_k, top_p = knobs
    P = Dist(processed(p_row, hist, penalty, ngram, t), top_k, top_p, mut)
    if P.degenerate:
        return {~P.pick}
    V = P.values.size
    Q = None if x is None else Dist(processed(q_row, hist, penalty, ngram, t), top_k, top_p, mut)
    same = Q is not None and not Q.degenerate and np.array_equal(P.values, Q.values, equal_nan=True)
    purposes = (RESIDUAL, ACCEPT) if "swap_purposes" in mut else (ACCEPT, RESIDUAL)
    r_acc = int(draw_bits(seed, pos, purposes[0], key, mut))
    r_res = int(draw_bits(seed, pos, purposes[1], key, mut))
    out = set()
    pairs = [(c, c) for c in range(len(P.cuts))] if same else \
        [(c, d) for c in range(len(P.cuts)) for d in range(1 if Q is None or Q.degenerate else len(Q.cuts))]
    for c, d in pairs:
        pl, ph = P.weights(c)
        ZpL, ZpH = int(pl.sum()), int(ph.sum())
        if Q is None:                                                 # j = k: q = 0, Zq = 1
            ql = qh = np.zeros(V, dtype=np.int64)
            ZqL = ZqH = 1
        elif Q.degenerate:                                            # a point mass at the draft's greedy pick
            ql = np.zeros(V, dtype=np.int64)
            ql[Q.pick] = 1
            qh, ZqL, ZqH = ql, 1, 1
        else:
            ql, qh = Q.weights(d)
            ZqL, ZqH = int(ql.sum()), int(qh.sum())
        reject = True
        if x is not None:
            if 0 <= x < V:
                if same:                                              # p == q: A == B = w(x) Z, accepted iff w(x) > 0
                    acc = {int(ph[x]) > 0, int(pl[x]) > 0}
                else:
                    acc = {_mulhi(r_acc, int(ql[x]) * ZpL) < int(ph[x]) * ZqH,
                           _mulhi(r_acc, int(qh[x]) * ZpH) < int(pl[x]) * ZqL}
            else:
                acc = {False}
            if True in acc:
                out.add(int(x))
            reject = False in acc
        if not reject:
            continue
        if same:                                                      # the residual is exactly 0
            out.add(~P.pick)
            continue
        a = (pl.astype(object) * ZqL, ph.astype(object) * ZqH)
        b = (ql.astype(object) * ZpL, qh.astype(object) * ZpH)
        if "residual_q_minus_p" in mut:
            a, b = b[::-1], a[::-1]
        rl = np.maximum(a[0] - b[1], 0)
        rh = np.maximum(a[1] - b[0], 0)
        if int(rl.sum()) == 0:                                        # possibly empty: p's argmax
            out.add(~P.pick)
        if int(rh.sum()) > 0:
            out |= {~t for t in _Prefix(rl, rh, P._order).draw(r_res)}
    return out


def spec_commit(picks, k, length, limit, eos):
    """commit_row for the kernel's picks of one slot: (emitted tokens, finished)."""
    toks = []
    for c in range(k + 1):
        pk = int(picks[c])
        tok = ~pk if pk < 0 else pk
        toks.append(tok)
        n = len(toks)
        if tok == eos or length + n >= limit or n == k + 1 or pk < 0:
            return toks, tok == eos or length + n >= limit
    raise AssertionError("unreachable")
