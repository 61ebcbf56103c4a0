"""GPU: every FP8 GEMM entry point on operands whose product is exact (tests/fp8_exact.py), compared bit for bit.

Each row of A and of B carries its own power-of-two factor (a rowwise 1/s, or folded into the 8-bit values for the
tensorwise GEMMs), so a kernel that gives an element the wrong row or column scale, drops a k stage or loses a tile
changes most of the elements it touches (tests/test_fp8_exact_cpu.py measures this on the references).

  plain      gemm_fp8 (e4m3 and e5m2 A) and gemm_fp8_rowwise (promoted or not), bf16 and fp32 out, from a single tile
             to the 256-wide tile with a 16-column or 16-row tail; a strided residual and an `out=` column block
  fused      SwiGLU (G, U exact; H equal to the bf16 SwiGLU epilogue on them), dSwiGLU (equal to swiglu_bwd on the
             exact dH), QKV modes 0 (with and without RoPE), 1 and 2, in both recipes
  decode     gemm_fp8_decode, epilogues 0-2, every row-group size and its boundaries, strided x and residual, the
             largest K that fits shared memory (and the next one raising)
  settings   raster group and SM margin leave the bits unchanged
  rounding   non-power-of-two scales: the documented rounding order, bit for bit
  control    torch._scaled_mm on the same bytes and scales is exact too (the accumulator-width premise)
  witness    the promoted forms add each 128-k stage into fp32 (exact); whether the forward forms do is printed
"""
import functools

import pytest
import torch

from tests import fp8_exact as fx
from tests.gpu_util import require_cuda
from touchnet_b200 import _lib, ops

pytestmark = pytest.mark.gpu
F8E4M3, F8E5M2, BF16 = torch.float8_e4m3fn, torch.float8_e5m2, torch.bfloat16
COMPARED = [0]


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print(f"\nfp8 exact: {COMPARED[0]} output elements compared bit for bit")


def _eq(got, ref, what=""):
    assert got.dtype == ref.dtype and got.shape == ref.shape, (what, got.dtype, ref.dtype, got.shape, ref.shape)
    if not torch.equal(got, ref):
        bad = (got != ref) & ~(torch.isnan(got.float()) & torch.isnan(ref.float()))
        idx = bad.nonzero()[:4].tolist()
        raise AssertionError(f"{what}: {int(bad.sum())} of {ref.numel()} elements differ, first at {idx}: "
                             f"{[float(got[tuple(i)]) for i in idx]} vs {[float(ref[tuple(i)]) for i in idx]}")
    COMPARED[0] += ref.numel()


def _dev():
    return require_cuda()


def _scalar(v):
    return torch.tensor(float(v), device=_dev())


@functools.lru_cache(maxsize=4)
def _ints(M, N, K, seed):
    dev = _dev()
    a, b = fx.int_a(M, K, seed, dev), fx.int_b(N, K, seed + 1, dev)
    assert fx.abs_bound(a, b) <= fx.CAP
    return a, b


def _rowwise(M, N, K, seed=0, extra=()):
    """e4m3 A, B, their 1/s vectors (2^e per row) and the exact product in fp64."""
    a, b = _ints(M, N, K, seed)
    ia = fx.pow2(fx.exponents(M, seed + 2), a.device)
    ib = fx.pow2(fx.exponents(N, seed + 3, extra), a.device)
    return fx.fp8(a, F8E4M3), fx.fp8(b, F8E4M3), ia, ib, fx.exact(a, b, ia, ib)


def _tensorwise(M, N, K, a_dt, seed=0):
    """8-bit A (e4m3 or e5m2), e4m3 B with the row exponents folded into the values, scalar 1/s, exact product."""
    a, b = _ints(M, N, K, seed)
    av = a * fx.pow2(fx.exponents(M, seed + 2), a.device)[:, None]
    bv = b * fx.pow2(fx.exponents(N, seed + 3), a.device)[:, None]
    ia, ib = _scalar(2.0 ** -(seed % 5 + 1)), _scalar(2.0 ** (seed % 3 + 1))
    return fx.fp8(av, a_dt), fx.fp8(bv, F8E4M3), ia, ib, fx.exact(av, bv) * float(ia * ib)


def _out(ref, f32):
    return ref.float() if f32 else fx.bf16(ref)


# plain GEMM forms and their OP in gemm_kernel (1, 2 tensorwise with an e4m3 / e5m2 A; 3, 4 rowwise, 4 promoted)
FORMS = {"e4m3": 1, "e5m2": 2, "rowwise": 3, "rowwise_promoted": 4}


def _plain(form, M, N, K, seed=0):
    if form in ("e4m3", "e5m2"):
        a8, b8, ia, ib, ref = _tensorwise(M, N, K, F8E4M3 if form == "e4m3" else F8E5M2, seed)
        run = lambda **kw: ops.gemm_fp8(a8, b8, ia, ib, **kw)
    else:
        a8, b8, ia, ib, ref = _rowwise(M, N, K, seed)
        run = lambda **kw: ops.gemm_fp8_rowwise(a8, b8, ia, ib, promoted=form == "rowwise_promoted", **kw)
    return run, ref, (a8, b8, ia, ib)


# ---------------------------------------------------------------------------------------------------------------
# plain GEMMs
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("f32", [False, True], ids=["bf16", "f32"])
@pytest.mark.parametrize("form", list(FORMS))
@pytest.mark.parametrize("shape", fx.PLAIN, ids=lambda s: "%dx%dx%d" % s)
def test_plain_gemm_is_exact(shape, form, f32):
    M, N, K = shape
    run, ref, _ = _plain(form, M, N, K)
    bn = fx.fp8_tile(FORMS[form], 2 if f32 else 0, M, N, fx.sm_count())
    print(f"{form} {'f32' if f32 else 'bf16'} {M}x{N}x{K}: {bn}-wide tile")
    _eq(run(out_f32=f32), _out(ref, f32), form)


@pytest.mark.parametrize("f32", [False, True], ids=["bf16", "f32"])
@pytest.mark.parametrize("form", list(FORMS))
@pytest.mark.parametrize("shape", [(144, 528, 112), (8208, 3088, 3088)], ids=lambda s: "%dx%dx%d" % s)
def test_strided_residual_and_output_column_block(shape, form, f32):
    """residual with row stride > N; `out` the first N columns of a wider buffer whose other columns keep a
    sentinel.  Expected: bf16(bf16(D) + R) in bf16, D + R in fp32."""
    M, N, K = shape
    dev = _dev()
    run, ref, _ = _plain(form, M, N, K, seed=1)
    dt = torch.float32 if f32 else BF16
    g = torch.Generator(device=dev).manual_seed(7)
    r = torch.randn(M, N + 48, device=dev, generator=g).to(dt)[:, :N]
    buf = torch.full((M, N + 80), 3.0e30, device=dev, dtype=dt)
    sentinel = buf[:, N:].clone()
    got = run(out_f32=f32, residual=r, out=buf[:, :N])
    assert got.data_ptr() == buf.data_ptr()
    want = ref.float() + r if f32 else (fx.bf16(ref).float() + r.float()).bfloat16()
    _eq(buf[:, :N], want, form)
    assert torch.equal(buf[:, N:], sentinel)


# ---------------------------------------------------------------------------------------------------------------
# SwiGLU, dSwiGLU, QKV
# ---------------------------------------------------------------------------------------------------------------
def _swiglu_epilogue(g, u):
    """H of the bf16 gemm_swiglu epilogue on given bf16 G, U: with X = I its accumulator is exactly G / U (one nonzero
    product per sum), so H is the epilogue's rounding of those values (rows padded to a multiple of 16 with zeros)."""
    M, N = g.shape
    Mp = -(-M // 16) * 16
    pad = lambda t: torch.cat([t, t.new_zeros(Mp - M, N)]) if Mp != M else t
    eye = torch.eye(Mp, device=g.device, dtype=BF16)
    _, _, h = ops.gemm_swiglu(eye, pad(g).t().contiguous(), pad(u).t().contiguous())
    return h[:M]


@pytest.mark.parametrize("rowwise", [False, True], ids=["tensorwise", "rowwise"])
@pytest.mark.parametrize("shape", fx.SWIGLU, ids=lambda s: "%dx%dx%d" % s)
def test_swiglu_is_exact(shape, rowwise):
    M, N, K = shape
    dev = _dev()
    a, _ = _ints(M, N, K, 0)
    bg, bu = fx.int_b(N, K, 11, dev), fx.int_b(N, K, 12, dev)
    assert max(fx.abs_bound(a, bg), fx.abs_bound(a, bu)) <= fx.CAP
    ea, ew = fx.exponents(M, 2), fx.exponents(2 * N, 3, extra=[(N, N)])
    sa, sw = fx.pow2(ea, dev), fx.pow2(ew, dev)
    if rowwise:
        x8, wg8, wu8 = fx.fp8(a, F8E4M3), fx.fp8(bg, F8E4M3), fx.fp8(bu, F8E4M3)
        run = lambda need: ops.gemm_swiglu_fp8_rowwise(x8, wg8, wu8, sa, sw, need_gu=need)
        g_ref, u_ref = fx.exact(a, bg, sa, sw[:N]), fx.exact(a, bu, sa, sw[N:])
    else:
        av, gv, uv = a * sa[:, None], bg * sw[:N, None], bu * sw[N:, None]
        x8, wg8, wu8 = fx.fp8(av, F8E4M3), fx.fp8(gv, F8E4M3), fx.fp8(uv, F8E4M3)
        ix, iw = _scalar(0.25), _scalar(2.0)
        run = lambda need: ops.gemm_swiglu_fp8(x8, wg8, wu8, ix, iw, need_gu=need)
        g_ref, u_ref = fx.exact(av, gv) * 0.5, fx.exact(av, uv) * 0.5
    op = 3 if rowwise else 1
    print(f"swiglu {'rowwise' if rowwise else 'tensorwise'} {M}x{N}x{K}: {fx.fp8_tile(op, 1, M, N, fx.sm_count())}-wide")
    g, u, h = run(True)
    g_ref, u_ref = fx.bf16(g_ref), fx.bf16(u_ref)
    _eq(g, g_ref, "G")
    _eq(u, u_ref, "U")
    h_ref = _swiglu_epilogue(g_ref, u_ref)
    _eq(h, h_ref, "H")
    _eq(run(False)[2], h_ref, "H without G, U")


@pytest.mark.parametrize("rowwise", [False, True], ids=["tensorwise", "rowwise"])
@pytest.mark.parametrize("shape", fx.SWIGLU, ids=lambda s: "%dx%dx%d" % s)
def test_dswiglu_is_exact(shape, rowwise, monkeypatch):
    M, N, K = shape
    dev = _dev()
    monkeypatch.setattr(ops, "_FUSE_DSWIGLU", True)
    gen = torch.Generator(device=dev).manual_seed(3)
    g = torch.randn(M, N, device=dev, generator=gen).bfloat16()
    u = torch.randn(M, N, device=dev, generator=gen).bfloat16()
    if rowwise:
        a8, b8, ia, ib, ref = _rowwise(M, N, K, seed=2)
        dg, du = ops.gemm_dswiglu_fp8_rowwise(a8, b8, g, u, ia, ib)
    else:
        a8, b8, ia, ib, ref = _tensorwise(M, N, K, F8E5M2, seed=2)
        dg, du = ops.gemm_dswiglu_fp8(a8, b8, g, u, ia, ib)
    dg_ref, du_ref = ops.swiglu_bwd(g, u, fx.bf16(ref))
    _eq(dg, dg_ref, "dG")
    _eq(du, du_ref, "dU")


def _rope(M, dev):
    pos = torch.arange(M, device=dev) % 2048
    inv = 1.0 / (500000.0 ** (torch.arange(0, 128, 2, device=dev).float() / 128))
    return ops.rope_table(pos, inv)


@pytest.mark.parametrize("rowwise", [False, True], ids=["tensorwise", "rowwise"])
@pytest.mark.parametrize("geom", fx.QKV, ids=lambda g: "M%d-d%d-q%d-kv%d" % g)
def test_qkv_three_modes_are_exact(geom, rowwise):
    M, d, nq, nkv = geom
    dev = _dev()
    shapes = fx.qkv_gemms(*geom)
    # mode 0: x [M, d] against [Wq;Wk;Wv] [tot, d]; the weight rows' exponents differ across segment boundaries too
    Mm, Nm, Km = shapes[0]
    if rowwise:
        x8, w8, ix, iw, ref = _rowwise(Mm, Nm, Km, seed=20, extra=fx.qkv_extra(nq, nkv))
        fwd = lambda rope=None: ops.gemm_qkv_fwd_fp8_rowwise(x8, w8[:nq], w8[nq:nq + nkv], w8[nq + nkv:], ix, iw, rope)
    else:
        x8, w8, ix, iw, ref = _tensorwise(Mm, Nm, Km, F8E4M3, seed=20)
        fwd = lambda rope=None: ops.gemm_qkv_fwd_fp8(x8, w8[:nq], w8[nq:nq + nkv], w8[nq + nkv:], ix, iw, rope)
    op = 3 if rowwise else 1
    print(f"qkv {'rowwise' if rowwise else 'tensorwise'} {geom}: mode 0 {fx.fp8_tile(op, 0, Mm, Nm, fx.sm_count())}-wide")
    qkv = fx.bf16(ref)
    _eq(fwd(), qkv, "mode 0")
    cos, sin = _rope(M, dev)
    qkv_r = qkv.clone()
    ops.rope_apply_(qkv_r[:, :nq], cos, sin, nq // 128, 128)
    ops.rope_apply_(qkv_r[:, nq:nq + nkv], cos, sin, nkv // 128, 128)
    _eq(fwd((cos, sin)), qkv_r, "mode 0 + RoPE")
    # mode 1: dqkv [M, tot] against Wᵀ [d, tot], nonzeros of dqkv in every K segment
    Mm, Nm, Km = shapes[1]
    if rowwise:
        a8, b8, ia, ib, ref = _rowwise(Mm, Nm, Km, seed=21)
        dx = ops.gemm_qkv_dgrad_fp8_rowwise(a8, b8, nq, nkv, ia, ib)
    else:
        a8, b8, ia, ib, ref = _tensorwise(Mm, Nm, Km, F8E5M2, seed=21)
        dx = ops.gemm_qkv_dgrad_fp8(a8, b8, nq, nkv, ia, ib)
    for lo, hi in ((0, nq), (nq, nq + nkv), (nq + nkv, Km)):
        assert bool((a8[:, lo:hi].float() != 0).any(1).all())
    _eq(dx, fx.bf16(ref), "mode 1")
    # mode 2: dqkvᵀ [tot, M] against xᵀ [d, M] into three gradients, fp32 and bf16
    Mm, Nm, Km = shapes[2]
    if rowwise:
        a8, b8, ia, ib, ref = _rowwise(Mm, Nm, Km, seed=22)
        wgrad = lambda f32: ops.gemm_qkv_wgrad_fp8_rowwise(a8, b8, f32, nq, nkv, ia, ib)
    else:
        a8, b8, ia, ib, ref = _tensorwise(Mm, Nm, Km, F8E5M2, seed=22)
        wgrad = lambda f32: ops.gemm_qkv_wgrad_fp8(a8, b8, f32, nq, nkv, ia, ib)
    for f32 in (False, True):
        outs = wgrad(f32)
        assert [t.shape[0] for t in outs] == [nq, nkv, nkv]
        _eq(torch.cat(outs), _out(ref, f32), "mode 2")


# ---------------------------------------------------------------------------------------------------------------
# the skinny-M decode GEMM
# ---------------------------------------------------------------------------------------------------------------
ZERO_ROW = 7


@functools.lru_cache(maxsize=2)
def _decode_operands(N, K, epi):
    """bf16 x [200, K] inside a wider buffer (row stride K + 32): row m is an integer row times 2^e_m with a 3 in it,
    so the kernel's row quantisation is exact; row ZERO_ROW is zero.  e4m3 W [rows, K] with 1/s 2^e per row."""
    dev = _dev()
    rows = 2 * N if epi == 2 else N
    xi, wi = fx.int_x(200, K, 30, dev, zero_row=ZERO_ROW), fx.int_b(rows, K, 31, dev)
    assert fx.abs_bound(xi, wi) <= fx.CAP
    xv = xi * fx.pow2(fx.exponents(200, 32), dev)[:, None]
    buf = torch.zeros(200, K + 32, device=dev, dtype=BF16)
    buf[:, :K] = xv.bfloat16()
    assert torch.equal(buf[:, :K].float(), xv)
    iw = fx.pow2(fx.exponents(rows, 33, [(N, N)] if epi == 2 else ()), dev)
    return buf[:, :K], fx.fp8(wi, F8E4M3), iw, fx.exact(xv, wi, None, iw)


def _decode_ref(ref, N, epi, r=None):
    if epi == 2:
        return _swiglu_epilogue(fx.bf16(ref[:, :N]), fx.bf16(ref[:, N:]))
    out = fx.bf16(ref)
    return out if r is None else (out.float() + r.float()).bfloat16()


@pytest.mark.parametrize("epi", [0, 1, 2])
@pytest.mark.parametrize("NK", fx.DEC_NK, ids=lambda s: "N%d-K%d" % s)
def test_decode_is_exact(NK, epi):
    N, K = NK
    dev = _dev()
    x_all, w8, iw, ref_all = _decode_operands(N, K, epi)
    rbuf = torch.randn(200, N + 16, device=dev).bfloat16()
    tiles = {}
    for M in fx.DEC_M:
        x, r = x_all[:M], (rbuf[:M, :N] if epi == 1 else None)
        assert x.stride(0) > K and (r is None or r.stride(0) > N)
        got = ops.gemm_fp8_decode(x, w8, iw, residual=r, swiglu=epi == 2)
        _eq(got, _decode_ref(ref_all[:M], N, epi, r), f"decode M={M}")
        if M > ZERO_ROW:
            assert torch.equal(got[ZERO_ROW], r[ZERO_ROW] if epi == 1 else torch.zeros_like(got[ZERO_ROW]))
        tiles[M] = fx.dec_mt(M, K, epi)
    print(f"decode epi {epi} N {N} K {K}: 16-row tiles per group {tiles}")


@pytest.mark.parametrize("epi", [0, 1, 2])
def test_decode_largest_k_is_exact_and_the_next_raises(epi):
    dev = _dev()
    N, K, M = 48, fx.dec_max_k(epi), 17
    rows = 2 * N if epi == 2 else N
    xi, wi = fx.int_x(M, K, 40, dev, zero_row=3), fx.int_b(rows, K, 41, dev)
    assert fx.abs_bound(xi, wi) <= fx.CAP
    xv = xi * fx.pow2(fx.exponents(M, 42), dev)[:, None]
    iw = fx.pow2(fx.exponents(rows, 43, [(N, N)] if epi == 2 else ()), dev)
    r = torch.randn(M, N, device=dev).bfloat16() if epi == 1 else None
    got = ops.gemm_fp8_decode(xv.bfloat16(), fx.fp8(wi, F8E4M3), iw, residual=r, swiglu=epi == 2)
    _eq(got, _decode_ref(fx.exact(xv, wi, None, iw), N, epi, r), f"decode K={K}")
    K2 = K + 16
    with pytest.raises(_lib.TouchNetB200Error, match="too large"):
        ops.gemm_fp8_decode(torch.zeros(M, K2, device=dev, dtype=BF16), torch.zeros(rows, K2, device=dev, dtype=F8E4M3),
                            iw, residual=r, swiglu=epi == 2)


# ---------------------------------------------------------------------------------------------------------------
# tile-walk settings
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("form", ["e4m3", "rowwise"])
def test_raster_group_and_sm_margin_leave_the_bits(form):
    """65 M blocks: groups 1, 3, 5, 7 and 64 (3, 7 and 64 do not divide 65), then SM margins 0 and 7.  The library's
    defaults (group 8, margin 0) are restored afterwards."""
    M, N, K = 8208, 3088, 3088
    run, ref, _ = _plain(form, M, N, K)
    want = fx.bf16(ref)
    _eq(run(), want, "default settings")
    try:
        for group in (1, 3, 5, 7, 64):
            _lib.call("tn_set_gemm_group", group)
            _eq(run(), want, f"group {group}")
        _lib.call("tn_set_gemm_group", 8)
        for margin in (7, 0):
            _lib.call("tn_set_sm_margin", margin)
            print(f"{form} {M}x{N}x{K} at SM margin {margin}: "
                  f"{fx.fp8_tile(FORMS[form], 0, M, N, fx.sm_count(margin))}-wide tile")
            _eq(run(), want, f"margin {margin}")
    finally:
        _lib.call("tn_set_gemm_group", 8)
        _lib.call("tn_set_sm_margin", 0)


# ---------------------------------------------------------------------------------------------------------------
# rounding order with non-power-of-two scales
# ---------------------------------------------------------------------------------------------------------------
def _nonpow2(n, seed, dev):
    """fp32 [n] in [0.5, 2) · 2^e, e in [-6, 6]: normal, not powers of two."""
    g = torch.Generator().manual_seed(seed)
    u = 0.5 + 1.5 * torch.rand(n, generator=g)
    return (u * torch.exp2(fx.exponents(n, seed).float())).float().to(dev)


@pytest.mark.parametrize("family", ["tensorwise", "rowwise", "decode"])
def test_rounding_order(family):
    """tensorwise fl(acc · fl(ia · ib)); rowwise and decode fl(fl(acc · ia[m]) · ib[n]); then bf16, or bf16 plus the
    residual as bf16(bf16(D) + R); fp32 D + R."""
    dev = _dev()
    M, N, K = 144, 272, 144
    a, b = _ints(M, N, K, 50)
    S = fx.exact(a, b).float()                     # exact integers
    r16 = torch.randn(M, N, device=dev).bfloat16()
    r32 = torch.randn(M, N, device=dev)
    a8, b8 = fx.fp8(a, F8E4M3), fx.fp8(b, F8E4M3)
    if family == "tensorwise":
        ia, ib = _nonpow2(1, 51, dev)[0].clone(), _nonpow2(1, 52, dev)[0].clone()
        d32 = S * (ia * ib)
        run = lambda **kw: ops.gemm_fp8(a8, b8, ia, ib, **kw)
    elif family == "rowwise":
        ia, ib = _nonpow2(M, 53, dev), _nonpow2(N, 54, dev)
        d32 = (S * ia[:, None]) * ib[None, :]
        run = lambda **kw: ops.gemm_fp8_rowwise(a8, b8, ia, ib, promoted=False, **kw)
    else:
        xi = fx.int_x(M, K, 55, dev)
        xv = xi * fx.pow2(fx.exponents(M, 56), dev)[:, None]
        wi = fx.int_b(2 * N, K, 57, dev)
        iw = _nonpow2(2 * N, 58, dev)
        S2 = fx.exact(xv, wi).float()              # acc · (1/s_x): exact
        d = S2 * iw[None, :]
        _eq(ops.gemm_fp8_decode(xv.bfloat16(), fx.fp8(wi[:N], F8E4M3), iw[:N]), d[:, :N].bfloat16(), "decode")
        _eq(ops.gemm_fp8_decode(xv.bfloat16(), fx.fp8(wi[:N], F8E4M3), iw[:N], residual=r16),
            (d[:, :N].bfloat16().float() + r16.float()).bfloat16(), "decode + R")
        _eq(ops.gemm_fp8_decode(xv.bfloat16(), fx.fp8(wi, F8E4M3), iw, swiglu=True),
            _swiglu_epilogue(d[:, :N].bfloat16(), d[:, N:].bfloat16()), "decode SwiGLU")
        return
    assert bool((d32.abs()[d32 != 0] > 2.0 ** -126).all())
    _eq(run(), d32.bfloat16(), family)
    _eq(run(residual=r16), (d32.bfloat16().float() + r16.float()).bfloat16(), family + " + R")
    _eq(run(out_f32=True), d32, family + " fp32")
    _eq(run(out_f32=True, residual=r32), d32 + r32, family + " fp32 + R")


# ---------------------------------------------------------------------------------------------------------------
# control: cuBLAS / CUTLASS through torch._scaled_mm on the same bytes and scales
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fast", [False, True], ids=["promoted", "fast"])
@pytest.mark.parametrize("form", ["e4m3", "e5m2", "rowwise"])
@pytest.mark.parametrize("shape", fx.PLAIN, ids=lambda s: "%dx%dx%d" % s)
def test_scaled_mm_control_is_exact(shape, form, fast):
    """If this fails, the operands' exactness premise (an accumulator of >= 13 significant bits) does not hold."""
    M, N, K = shape
    _, ref, (a8, b8, ia, ib) = _plain(form, M, N, K)
    if form == "rowwise":
        sa, sb = ia[:, None].contiguous(), ib[None, :].contiguous()
    else:
        sa, sb = ia.reshape(()), ib.reshape(())
    got = torch._scaled_mm(a8, b8.t(), scale_a=sa, scale_b=sb, out_dtype=BF16, use_fast_accum=fast)
    _eq(got, fx.bf16(ref), f"_scaled_mm {form} fast={fast}")


# ---------------------------------------------------------------------------------------------------------------
# promotion witness
# ---------------------------------------------------------------------------------------------------------------
def _witness(M, N, K, seed, rowwise, a_dt=F8E4M3, extra=()):
    dev = _dev()
    a, b = fx.witness(M, N, K, seed, dev)
    if rowwise:
        ia = fx.pow2(fx.exponents(M, seed + 2), dev)
        ib = fx.pow2(fx.exponents(N, seed + 3, extra), dev)
        return fx.fp8(a, a_dt), fx.fp8(b, F8E4M3), ia, ib, fx.exact(a, b, ia, ib)
    ia, ib = _scalar(0.5), _scalar(4.0)
    return fx.fp8(a, a_dt), fx.fp8(b, F8E4M3), ia, ib, fx.exact(a, b) * 2.0


def test_promoted_forms_add_each_stage_in_fp32(monkeypatch):
    monkeypatch.setattr(ops, "_FUSE_DSWIGLU", True)
    dev = _dev()
    M, N, K = fx.WITNESS_PLAIN
    a8, b8, ia, ib, ref = _witness(M, N, K, 60, False, F8E5M2)
    for f32 in (False, True):
        _eq(ops.gemm_fp8(a8, b8, ia, ib, out_f32=f32), _out(ref, f32), "gemm_fp8 e5m2")
    a8, b8, ia, ib, ref = _witness(M, N, K, 61, True)
    for f32 in (False, True):
        _eq(ops.gemm_fp8_rowwise(a8, b8, ia, ib, promoted=True, out_f32=f32), _out(ref, f32), "rowwise promoted")
    g = torch.randn(M, N, device=dev).bfloat16()
    u = torch.randn(M, N, device=dev).bfloat16()
    a8, b8, ia, ib, ref = _witness(M, N, K, 62, False, F8E5M2)
    want = ops.swiglu_bwd(g, u, fx.bf16(ref))
    for got, w in zip(ops.gemm_dswiglu_fp8(a8, b8, g, u, ia, ib), want):
        _eq(got, w, "dswiglu tensorwise")
    a8, b8, ia, ib, ref = _witness(M, N, K, 63, True)
    want = ops.swiglu_bwd(g, u, fx.bf16(ref))
    for got, w in zip(ops.gemm_dswiglu_fp8_rowwise(a8, b8, g, u, ia, ib), want):
        _eq(got, w, "dswiglu rowwise")
    Mq, d, nq, nkv = fx.WITNESS_QKV
    shapes = fx.qkv_gemms(*fx.WITNESS_QKV)
    for rowwise in (False, True):
        a8, b8, ia, ib, ref = _witness(*shapes[1], 64, rowwise, F8E4M3 if rowwise else F8E5M2)
        dgrad = ops.gemm_qkv_dgrad_fp8_rowwise if rowwise else ops.gemm_qkv_dgrad_fp8
        _eq(dgrad(a8, b8, nq, nkv, ia, ib), fx.bf16(ref), "qkv mode 1")
        a8, b8, ia, ib, ref = _witness(*shapes[2], 65, rowwise, F8E4M3 if rowwise else F8E5M2)
        wgrad = ops.gemm_qkv_wgrad_fp8_rowwise if rowwise else ops.gemm_qkv_wgrad_fp8
        for f32 in (False, True):
            _eq(torch.cat(wgrad(a8, b8, f32, nq, nkv, ia, ib)), _out(ref, f32), "qkv mode 2")


def test_forward_forms_on_the_witness_are_reported():
    """The forward forms accumulate in the wgmma accumulator; whether they keep the small sum is printed only."""
    M, N, K = fx.WITNESS_PLAIN
    res = {}

    def note(name, got, ref):
        bad = int((got != ref).sum())
        res[name] = "exact" if bad == 0 else f"{bad} of {ref.numel()} differ"

    a8, b8, ia, ib, ref = _witness(M, N, K, 70, False)
    note("gemm_fp8 e4m3 (fp32 out)", ops.gemm_fp8(a8, b8, ia, ib, out_f32=True), ref.float())
    a8, b8, ia, ib, ref = _witness(M, N, K, 71, True)
    note("gemm_fp8_rowwise (fp32 out)", ops.gemm_fp8_rowwise(a8, b8, ia, ib, promoted=False, out_f32=True), ref.float())
    Mq, d, nq, nkv = fx.WITNESS_QKV
    for rowwise in (False, True):
        a8, b8, ia, ib, ref = _witness(*fx.qkv_gemms(*fx.WITNESS_QKV)[0], 72, rowwise,
                                       extra=fx.qkv_extra(nq, nkv))
        fwd = ops.gemm_qkv_fwd_fp8_rowwise if rowwise else ops.gemm_qkv_fwd_fp8
        note(f"qkv mode 0 {'rowwise' if rowwise else 'tensorwise'}",
             fwd(a8, b8[:nq], b8[nq:nq + nkv], b8[nq + nkv:], ia, ib), fx.bf16(ref))
    for k, v in res.items():
        print(f"witness, forward form {k}: {v}")
