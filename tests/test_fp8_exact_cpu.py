"""CPU: the exact-operand helpers of tests/test_gpu_fp8_exact.py (tests/fp8_exact.py), and the power of its bitwise
comparisons.

- every case meets the precondition Σ_k |a_mk · b_nk| ≤ 2^12 (in quanta), and an emulated accumulator that keeps 13
  significant bits, truncating after aligning to the largest exponent, reproduces the exact product on sampled rows
  and columns of every case;
- on the promotion witness that accumulator is exact with per-128-k promotion and not exact without it;
- the row and column exponents differ from their neighbours, and a reference computed the way a subtly wrong kernel
  would (a neighbour's scale, the gate scale on the up half, a neighbouring QKV segment's scale, the last k stage
  dropped, the last M or N tile lost) differs from the exact one in at least half of the elements it touches;
- the restated tile choices: at 132 SMs the cases reach the 128- and the 256-wide tile where the kernels have both,
  and every row-group size of the decode kernel, at its group boundaries."""
import functools

import pytest
import torch

from tests import fp8_exact as fx

SMS = 132


@functools.lru_cache(maxsize=None)
def _ab(M, N, K, seed=0):
    return fx.int_a(M, K, seed), fx.int_b(N, K, seed + 1)


def _cases():
    """(name, M, N, K) of every GEMM the GPU file runs on exact operands (one entry per operand pair)."""
    out = [("plain", *s) for s in fx.PLAIN]
    for M, N, K in fx.SWIGLU:
        out += [("swiglu", M, N, K), ("swiglu", M, 2 * N, K)]
    for geom in fx.QKV:
        out += [("qkv%d" % mode, *s) for mode, s in fx.qkv_gemms(*geom).items()]
    out += [("decode", 200, 2 * N, K) for N, K in fx.DEC_NK]
    out += [("decode", 17, 48, fx.dec_max_k(epi)) for epi in (0, 2)]
    return out


def _samples(n):
    idx = sorted(set(range(min(8, n))) | set(range(max(n - 8, 0), n)) | {n // 2})
    return torch.tensor(idx)


def test_helpers_restate_the_kernel_constants():
    assert fx.dec_max_k(0) == fx.dec_max_k(1) == 12416 and fx.dec_max_k(2) == 12160
    assert fx.a_stride(16) == 1 and fx.a_stride(3088) == 8 and fx.a_stride(8208) == 16
    # tensorwise folding keeps every value a normal e4m3 number: 1 · 2^-6 .. 3 · 2^6
    v = torch.tensor([1.0, 3.0]) * torch.tensor([2.0 ** fx.E_LO, 2.0 ** fx.E_HI])[:, None]
    assert torch.equal(fx.fp8(v, torch.float8_e4m3fn).float(), v) and float(v.max()) <= 448
    a = fx.int_x(40, 48, 0, zero_row=7)
    assert bool((a[torch.arange(40) != 7].abs().amax(1) == 3).all()) and not bool(a[7].any())


@pytest.mark.parametrize("n", [16, 272, 3088, 8208])
def test_exponents_differ_from_neighbours(n):
    e = fx.exponents(n, seed=n)
    assert int(e.min()) >= fx.E_LO and int(e.max()) <= fx.E_HI
    assert fx.neighbour_spread(e) >= 0.8
    assert len(set(e.tolist())) == fx.E_HI - fx.E_LO + 1 or n < 64
    gu = fx.exponents(2 * n, seed=1, extra=[(n, n)])        # SwiGLU: gate rows, then up rows
    assert bool((gu[:n] != gu[n:]).all())
    nq, nkv = 512, 256
    q = fx.exponents(nq + 2 * nkv, seed=2, extra=fx.qkv_extra(nq, nkv))
    assert bool((q[nq:nq + nkv] != q[:nkv]).all()) and bool((q[nq + nkv:] != q[nq:nq + nkv]).all())


@pytest.mark.parametrize("case", _cases(), ids=lambda c: "%s-%dx%dx%d" % c)
def test_precondition_and_13_bit_accumulation(case):
    """Σ|products| ≤ 2^12 on every element (the bound is max row sum of |A| times max |B|), nonzeros in the last k
    stage of every row of A, and the 13-bit accumulator exact (with and without promotion) on sampled elements."""
    _, M, N, K = case
    a, b = _ab(M, N, K)
    assert fx.abs_bound(a, b) <= fx.CAP
    last = (K - 1) // fx.KSTAGE * fx.KSTAGE
    assert bool(a[:, last:].abs().sum(1).gt(0).all())
    ra, rb = a[_samples(M)], b[_samples(N)]
    ref = fx.exact(ra, rb)
    assert torch.equal(fx.emulate_acc(ra, rb), ref)
    assert torch.equal(fx.emulate_acc(ra, rb, promote=True), ref)


@pytest.mark.parametrize("shape", [fx.WITNESS_PLAIN] + list(fx.qkv_gemms(*fx.WITNESS_QKV).values()))
def test_witness_needs_promotion(shape):
    M, N, K = shape
    a, b = fx.witness(M, N, K, seed=5)
    ref = fx.exact(a, b)
    assert bool((ref.abs() < 256).all()) and float((ref != 0).float().mean()) > 0.5
    stage = lambda lo, hi: fx.exact(a[:, lo:hi], b[:, lo:hi])
    for lo in range(fx.KSTAGE, K - fx.KSTAGE, fx.KSTAGE):
        assert float(fx.exact(a[:, lo:lo + fx.KSTAGE].abs(), b[:, lo:lo + fx.KSTAGE].abs()).max()) <= fx.CAP
    assert float(stage(0, fx.KSTAGE).abs().min()) == fx.WITNESS == float(stage(K - fx.KSTAGE, K).abs().min())
    assert bool((fx.exact(a[:, :fx.KSTAGE].abs(), b[:, :fx.KSTAGE].abs()) == fx.WITNESS).all())
    for t, dt in ((a, torch.float8_e4m3fn), (a, torch.float8_e5m2), (b, torch.float8_e4m3fn)):
        fx.fp8(t, dt)
    ra, rb = a[_samples(M)], b[_samples(N)]
    r = fx.exact(ra, rb)
    assert torch.equal(fx.emulate_acc(ra, rb, promote=True), r)
    fast = fx.emulate_acc(ra, rb)
    assert float((fast != r).float().mean()) > 0.5


# ---------------------------------------------------------------------------------------------------------------
# mutations: a reference computed as a subtly wrong kernel would compute it
# ---------------------------------------------------------------------------------------------------------------
def _scaled(S, ea, eb):
    return S * torch.exp2((ea[:, None] + eb[None, :]).double())


def _differ(ref, mut, mask):
    """Fraction of the masked elements whose bf16 values differ."""
    d = fx.bf16(ref) != fx.bf16(mut)
    return float(d[mask].float().mean())


def _shift(e, d):
    """e[i + d] where that exists (else e[i]), and the mask of the entries that moved."""
    n = e.numel()
    src = torch.arange(n) + d
    ok = (src >= 0) & (src < n)
    return torch.where(ok, e[src.clamp(0, n - 1)], e), ok


@pytest.mark.parametrize("shape", fx.PLAIN[:4], ids=lambda s: "%dx%dx%d" % s)
def test_mutated_references_differ(shape):
    M, N, K = shape
    a, b = _ab(M, N, K)
    ea, eb = fx.exponents(M, 2), fx.exponents(N, 3)
    S = fx.exact(a, b)
    ref = _scaled(S, ea, eb)
    full = torch.ones(M, N, dtype=torch.bool)
    res = {}
    for d in (1, -1, 8, -8):
        e2, ok = _shift(eb, d)
        res["column n%+d" % d] = _differ(ref, _scaled(S, ea, e2), full & ok[None, :])
    for d in (8, -8):
        e2, ok = _shift(ea, d)
        if ok.any():
            res["row m%+d" % d] = _differ(ref, _scaled(S, e2, eb), full & ok[:, None])
    k0 = (K - 1) // fx.KSTAGE * fx.KSTAGE
    res["last k stage dropped"] = _differ(ref, _scaled(fx.exact(a[:, :k0], b[:, :k0]), ea, eb), full)
    m0 = (M - 1) // fx.BM * fx.BM
    rows = torch.arange(M)[:, None].expand(M, N) >= m0
    res["last M tile lost"] = _differ(ref, torch.where(rows, torch.zeros_like(ref), ref), rows)
    for bn in (128, 256):
        n0 = (N - 1) // bn * bn
        cols = torch.arange(N)[None, :].expand(M, N) >= n0
        res["last N tile (%d) lost" % bn] = _differ(ref, torch.where(cols, torch.zeros_like(ref), ref), cols)
    print(shape, {k: round(v, 3) for k, v in res.items()})
    for k, v in res.items():
        assert v >= 0.5, (k, v)


def test_mutated_swiglu_and_qkv_scales_differ():
    M, N, K = fx.SWIGLU[0]
    a, bu = _ab(M, N, K, seed=4)
    e = fx.exponents(2 * N, 3, extra=[(N, N)])
    ea = fx.exponents(M, 2)
    S = fx.exact(a, bu)
    up, gate_for_up = _scaled(S, ea, e[N:]), _scaled(S, ea, e[:N])
    f_gu = _differ(up, gate_for_up, torch.ones(M, N, dtype=torch.bool))
    M, d, nq, nkv = fx.QKV[0]
    tot = nq + 2 * nkv
    a, b = _ab(M, tot, d, seed=6)
    e = fx.exponents(tot, 3, extra=fx.qkv_extra(nq, nkv))
    ea = fx.exponents(M, 2)
    S = fx.exact(a, b)
    ref = _scaled(S, ea, e)
    # column n of the k (v) segment with the scale at the same offset in the q (k) segment, and back
    n = torch.arange(tot)
    for name, src, ok in (("k from q", n - nq, (n >= nq) & (n < nq + nkv)), ("v from k", n - nkv, n >= nq + nkv),
                          ("q from k", n + nq, n < nkv)):
        e2 = torch.where(ok, e[src.clamp(0, tot - 1)], e)
        f = _differ(ref, _scaled(S, ea, e2), ok[None, :].expand(M, tot))
        print(name, round(f, 3))
        assert f >= 0.5, (name, f)
    print("gate scale on the up half", round(f_gu, 3))
    assert f_gu >= 0.5


# ---------------------------------------------------------------------------------------------------------------
# tile restatements
# ---------------------------------------------------------------------------------------------------------------
def test_cases_reach_both_tile_widths_at_132_sms():
    for op in (1, 3):
        assert {fx.fp8_tile(op, 0, M, N, SMS) for M, N, _ in fx.PLAIN} == {128, 256}, op
    assert {fx.fp8_tile(1, 2, M, N, SMS) for M, N, _ in fx.PLAIN} == {128, 256}
    assert {fx.fp8_tile(1, 1, M, N, SMS) for M, N, _ in fx.SWIGLU} == {128, 256}
    # the promoted forms, and the rowwise SwiGLU and fp32 forms, only have the 128-wide tile
    assert {fx.fp8_tile(op, epi, M, N, SMS) for op, epi in ((2, 0), (4, 2), (3, 1), (3, 2))
            for M, N, _ in fx.PLAIN + fx.SWIGLU} == {128}
    # the two ragged 256-wide cases: a 16-column tail (N = 3088) and a 16-row tail (M = 8208)
    assert fx.pick_bn(8208, 3088, 1, SMS) == 256 and 3088 % 256 == 16 and 8208 % 128 == 16
    assert fx.pick_bn(8208, 3072, 1, SMS) == 256
    # the same shapes keep their tiles with 7 SMs held back (the tile-walk test)
    assert fx.pick_bn(8208, 3088, 1, SMS - 7) == 256


@pytest.mark.parametrize("epi", [0, 1, 2])
def test_decode_cases_reach_every_row_group_and_its_boundaries(epi):
    assert [fx.dec_mt(200, K, epi) for K in (8192, 5120, 3072, 768)] == [1, 2, 3, 4]
    seen = {}
    for N, K in fx.DEC_NK:
        for M in fx.DEC_M:
            mt = fx.dec_mt(M, K, epi)
            seen.setdefault(mt, set()).add(M % (16 * mt) if M >= 16 * mt else None)
            assert fx.dec_smem(K, mt, 2 if epi == 2 else 1) <= fx.DEC_SMEM_MAX
    for mt in (1, 2, 3, 4):
        assert {0, 1} <= seen[mt], (mt, seen[mt])
    K = fx.dec_max_k(epi)
    assert fx.dec_smem(K + 16, 1, 2 if epi == 2 else 1) > fx.DEC_SMEM_MAX >= fx.dec_smem(K, 1, 2 if epi == 2 else 1)
