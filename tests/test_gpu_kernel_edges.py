"""GPU parity at the edges of the bf16 GEMM and the decoder layer's elementwise kernels, element by element against the
fp64 references of tests/test_kernel_edges_cpu.py (where the bounds and their derivations live), and bit for bit
where the result is defined exactly:

  1. tn_gemm_bf16 at decode-sized M (M < 64 leaves the second consumer warpgroup idle), a single partial k-block
     (K < 64), ragged N into a padded output (the fused lm_head + loss), forward / dgrad / wgrad; and the invariants the
     callers rely on: row independence, TMA's zero fill past K, untouched pad columns, the ragged-N residual epilogue;
  2. RMSNorm at d > 4096 (the NV = 32 forward, the 1024-thread backward), d < 256 and rows past the backward's grid;
  3. RoPE at head_dim 32 / 64 (the zero-padded-heads path) on strided rows;
  4. the SwiGLU backward where exp(-g) leaves fp32's range;
  5. the embedding add and the fp32 -> bf16 cast at their edges;
  6. strided rows (column slices, gradients coming back through torch.cat) through the autograd functions.

Each element-wise check prints its largest err / bound."""
import pytest
import torch

from oracle import model_oracle as mo
from tests.gpu_util import rel_err, require_cuda
from tests.test_gpu_bench_geometry import _within
from tests.test_kernel_edges_cpu import (bits_equal, gemm_bound, gemm_reference, rmsnorm_bwd_bound,
                                         rmsnorm_bwd_reference, rmsnorm_fwd_at, rmsnorm_fwd_bound,
                                         rmsnorm_fwd_reference, rstd_bound,
                                         swiglu_bwd_bound, swiglu_bwd_reference, swiglu_gates)
from touchnet_b200 import _lib, ops

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
EPS = 1e-5
SMALL_M = (1, 3, 8, 63, 64, 65, 127, 129)


def _gen(seed, dev):
    return torch.Generator(device=dev).manual_seed(seed)


def _strided(rows, cols, gen, dev, scale=1.0, dtype=BF16, fill=float("nan")):
    """[rows, cols] view with a row stride rounded up to 8 elements (16 B), the pad columns holding `fill`."""
    ld = (cols + 7) // 8 * 8
    buf = torch.full((rows, ld), fill, device=dev, dtype=dtype)
    buf[:, :cols] = (scale * torch.randn(rows, cols, generator=gen, device=dev)).to(dtype)
    return buf[:, :cols]


# ---------------------------------------------------------------------------------------------------------------
# 1. GEMM
# ---------------------------------------------------------------------------------------------------------------
# (layout, M, N, K, fp32 output).  fwd: a [M, K], b [N, K]; dgrad: b [K, N] (b_mn); wgrad: a [K, M], b [K, N] (a_mn,
# b_mn) with K a handful of tokens.  N = 3072 takes the 128-wide tile at these M, N = 128256 (lm_head) the 256-wide one;
# N = 1003 writes into a padded row stride whose pad columns must keep their sentinel.
GEMM_CASES = [
    ("fwd", 1, 3072, 72, False), ("fwd", 3, 3072, 8, False), ("fwd", 8, 128256, 56, False),
    ("fwd", 63, 3072, 3072, False), ("fwd", 64, 1003, 72, False), ("fwd", 65, 128256, 3072, False),
    ("fwd", 127, 3072, 56, False), ("fwd", 129, 1003, 3072, True), ("fwd", 1, 128256, 8, True),
    ("dgrad", 1, 3072, 3072, False), ("dgrad", 63, 3072, 72, False), ("dgrad", 65, 1003, 56, False),
    ("dgrad", 8, 128256, 72, False), ("dgrad", 127, 3072, 8, True), ("dgrad", 129, 3072, 3072, False),
    ("wgrad", 3072, 3072, 1, True), ("wgrad", 128, 3072, 5, False), ("wgrad", 1003, 3072, 71, True),
    ("wgrad", 3072, 1003, 71, False), ("wgrad", 64, 128256, 5, True),
]


@pytest.mark.parametrize("layout,M,N,K,f32", GEMM_CASES)
def test_gemm_edges_against_fp64(layout, M, N, K, f32):
    dev = require_cuda()
    gen = _gen(M * 131 + N + K, dev)
    a_mn, b_mn = layout == "wgrad", layout != "fwd"
    a = _strided(K, M, gen, dev) if a_mn else _strided(M, K, gen, dev)
    b = _strided(K, N, gen, dev, 0.05) if b_mn else _strided(N, K, gen, dev, 0.05)
    ld = (N + 7) // 8 * 8 + 8
    buf = torch.full((M, ld), -7.0, device=dev, dtype=torch.float32 if f32 else BF16)
    out = ops.gemm(a, b, a_mn=a_mn, b_mn=b_mn, out_f32=f32, out=buf[:, :N])
    ref, absprod = gemm_reference(a, b, a_mn=a_mn, b_mn=b_mn)
    ratio = _within(f"gemm {layout} M={M} N={N} K={K}", out, ref, gemm_bound(ref, absprod, K, f32))
    assert bool((buf[:, N:] == -7.0).all()), "columns of the output buffer past N were written"
    print(f"gemm {layout} M={M} N={N} K={K} f32={f32}: max err/bound {ratio:.3g}")


@pytest.mark.parametrize("f32", [False, True])
def test_gemm_ragged_n_leaves_pad_columns_alone(f32):
    """N = 1003, 1001 and 5 into a row stride of 1008, the pad columns pre-filled with a sentinel: they keep it (whole
    16-byte chunks of a row go out by TMA, the ragged rest by ordinary stores), and the first N columns equal the GEMM
    at N = 1008 cut to N."""
    dev = require_cuda()
    gen = _gen(14, dev)
    M, K, LD = 130, 256, 1008
    a = torch.randn(M, K, generator=gen, device=dev).to(BF16)
    for N in (1003, 1001, 5):
        b8 = (0.05 * torch.randn(LD, K, generator=gen, device=dev)).to(BF16)
        b = b8[:N]
        buf = torch.full((M, LD), 12288.0, device=dev, dtype=torch.float32 if f32 else BF16)
        out = ops.gemm(a, b, out_f32=f32, out=buf[:, :N])
        assert bool((buf[:, N:] == 12288.0).all()), N
        assert torch.equal(out, ops.gemm(a, b8, out_f32=f32)[:, :N]), N
        ref, absprod = gemm_reference(a, b)
        _within(f"gemm ragged N={N} f32={f32}", out, ref, gemm_bound(ref, absprod, K, f32))


@pytest.mark.parametrize("layout", ["fwd", "dgrad"])
def test_gemm_rows_are_independent(layout):
    """gemm(a[:m], b) == gemm(a, b)[:m] bit for bit: at M = 1024 the 256-wide tile, at small m the 128-wide one; both
    sum the k-blocks in the same order, and a row never meets another (continuous batching relies on this)."""
    dev = require_cuda()
    gen = _gen(11, dev)
    K, N = 3072, 3072
    a = torch.randn(1024, K, generator=gen, device=dev).to(BF16)
    b = (0.05 * torch.randn((K, N) if layout == "dgrad" else (N, K), generator=gen, device=dev)).to(BF16)
    full = ops.gemm(a, b, b_mn=layout == "dgrad")
    for m in SMALL_M:
        part = ops.gemm(a[:m], b, b_mn=layout == "dgrad")
        assert torch.equal(part, full[:m]), (layout, m)


@pytest.mark.parametrize("layout", ["fwd", "dgrad"])
def test_gemm_partial_kblock_is_zero_filled(layout):
    """K = 72 on strided slices of 128-wide operands whose columns 72..127 hold NaN == the same GEMM on the operands
    zero-padded to K = 128: the second k-block's missing 56 columns come from TMA's zero fill, not from memory."""
    dev = require_cuda()
    gen = _gen(12, dev)
    M, N, K, KP = 65, 3072, 72, 128
    aw = torch.full((M, KP), float("nan"), device=dev, dtype=BF16)
    aw[:, :K] = torch.randn(M, K, generator=gen, device=dev).to(BF16)
    bw = torch.full((KP, N) if layout == "dgrad" else (N, KP), float("nan"), device=dev, dtype=BF16)
    if layout == "dgrad":
        bw[:K] = (0.05 * torch.randn(K, N, generator=gen, device=dev)).to(BF16)
        b, bp = bw[:K], torch.cat([bw[:K], torch.zeros(KP - K, N, device=dev, dtype=BF16)])
    else:
        bw[:, :K] = (0.05 * torch.randn(N, K, generator=gen, device=dev)).to(BF16)
        b, bp = bw[:, :K], torch.nn.functional.pad(bw[:, :K], (0, KP - K))
    ap = torch.nn.functional.pad(aw[:, :K], (0, KP - K))
    got = ops.gemm(aw[:, :K], b, b_mn=layout == "dgrad")
    assert torch.equal(got, ops.gemm(ap, bp, b_mn=layout == "dgrad"))
    assert not torch.isnan(got).any()


def test_gemm_ragged_n_output_and_residual():
    """N = 1003 into a row stride of 1008 (the fused lm_head + loss): the pad columns keep their sentinel and the first
    1003 equal the GEMM at N = 1008 cut to 1003 columns; the ragged-N residual epilogue in bf16 equals
    bf16(plain + r), in fp32 plain + r, also in place (out is the residual, as the loss's chunked wgrad runs it)."""
    dev = require_cuda()
    gen = _gen(13, dev)
    M, K, N, LD = 200, 256, 1003, 1008
    a = torch.randn(M, K, generator=gen, device=dev).to(BF16)
    b8 = (0.05 * torch.randn(LD, K, generator=gen, device=dev)).to(BF16)
    b = b8[:N]
    for f32 in (False, True):
        dt = torch.float32 if f32 else BF16
        buf = torch.full((M, LD), 12288.0, device=dev, dtype=dt)
        plain = ops.gemm(a, b, out_f32=f32, out=buf[:, :N])
        assert bool((buf[:, N:] == 12288.0).all())
        assert torch.equal(plain, ops.gemm(a, b8, out_f32=f32)[:, :N])
        rbuf = torch.full((M, LD), float("nan"), device=dev, dtype=dt)
        rbuf[:, :N] = torch.randn(M, N, generator=gen, device=dev).to(dt)
        r = rbuf[:, :N]
        got = ops.gemm(a, b, out_f32=f32, residual=r, out=torch.empty(M, LD, device=dev, dtype=dt)[:, :N])
        want = plain + r if f32 else (plain.float() + r.float()).to(BF16)
        assert torch.equal(got, want), f32
    # in place, fp32: forward layout with ragged N, and the loss's wgrad form dW[V, d] += dlogitsᵀ·h (V = 1003 rows)
    acc = rbuf.clone()
    want = plain + acc[:, :N]
    ops.gemm(a, b, out_f32=True, residual=acc[:, :N], out=acc[:, :N])
    assert torch.equal(acc[:, :N], want) and bool(acc[:, N:].isnan().all())
    dlog = _strided(300, N, gen, dev)
    h = torch.randn(300, 512, generator=gen, device=dev).to(BF16)
    dw = torch.randn(N, 512, generator=gen, device=dev)
    want = ops.gemm(dlog, h, a_mn=True, b_mn=True, out_f32=True) + dw
    ops.gemm(dlog, h, a_mn=True, b_mn=True, out_f32=True, residual=dw, out=dw)
    assert torch.equal(dw, want)


# ---------------------------------------------------------------------------------------------------------------
# 2. RMSNorm
# ---------------------------------------------------------------------------------------------------------------
NORM_CASES = [(8, 1), (8, 2100), (24, 7), (24, 529), (4104, 1), (4104, 529), (5120, 7), (5120, 2100), (8192, 529),
              (8192, 2100)]


@pytest.mark.parametrize("d,rows", NORM_CASES)
@pytest.mark.parametrize("w_f32", [False, True])
@pytest.mark.parametrize("with_residual", [False, True])
def test_rmsnorm_edges_against_fp64(d, rows, w_f32, with_residual):
    dev = require_cuda()
    gen = _gen(d * 7 + rows, dev)
    x = torch.randn(rows, d, generator=gen, device=dev).to(BF16)
    w = (1 + 0.1 * torch.randn(d, generator=gen, device=dev)).to(torch.float32 if w_f32 else BF16)
    r = torch.randn(rows, d, generator=gen, device=dev).to(BF16) if with_residual else None
    y, s, rstd = ops.rmsnorm_fwd(x, w, EPS, residual=r)
    if with_residual:
        assert torch.equal(s, x + r)                                  # bf16 add, bit exact
    y_ref, rstd_ref = rmsnorm_fwd_reference(s, w, EPS)
    tag = f"rmsnorm d={d} rows={rows} w_f32={w_f32} res={with_residual}"
    assert torch.equal(y, rmsnorm_fwd_at(s, w, rstd)), "y is not HF's rounding points at the kernel's own rstd"
    ratios = [_within(tag + " y", y, y_ref, rmsnorm_fwd_bound(s, w, rstd_ref, y_ref)),
              _within(tag + " rstd", rstd, rstd_ref, rstd_bound(rstd_ref, d))]
    dy = torch.randn(rows, d, generator=gen, device=dev).to(BF16)
    extra = torch.randn(rows, d, generator=gen, device=dev).to(BF16) if with_residual else None
    ds, dw = ops.rmsnorm_bwd(s, dy, w, rstd, ds_extra=extra)
    ds_ref, ds0, dw_ref = rmsnorm_bwd_reference(s, dy, w, rstd, EPS, extra)
    ds_b, dw_b = rmsnorm_bwd_bound(s, dy, w, rstd, ds0, extra)
    ratios += [_within(tag + " ds", ds, ds_ref, ds_b), _within(tag + " dw", dw, dw_ref, dw_b)]
    print(tag, "max err/bound y, rstd, ds, dw:", [f"{q:.3g}" for q in ratios])


# ---------------------------------------------------------------------------------------------------------------
# 3. RoPE
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("hd", [32, 64])
@pytest.mark.parametrize("inverse", [False, True])
def test_rope_small_head_dim_on_strided_rows(hd, inverse):
    """head_dim 32 / 64 (the zero-padded-heads path of the decoder block), rows with a stride past heads·hd whose extra
    columns hold a sentinel: bit exact against HF's bf16 formula (q·cos + rotate_half(q)·sin, sin negated for the
    inverse), sentinel untouched."""
    dev = require_cuda()
    gen = _gen(hd + inverse, dev)
    H, rows, pad = 3, 777, 24
    cfg = mo.OracleConfig(H * hd, 8, 1, H, H, hd, 8, rope_theta=500000.0)
    inv, sc = mo.rope_inv_freq(cfg)
    pos = (torch.arange(rows, device=dev) * 7 % 4099)[None]
    cos, sin = ops.rope_table(pos, inv.to(dev), sc)
    assert cos.shape == (rows, hd // 2)
    buf = torch.full((rows, H * hd + pad), 3.0, device=dev, dtype=BF16)
    buf[:, :H * hd] = torch.randn(rows, H * hd, generator=gen, device=dev).to(BF16)
    x = buf[:, :H * hd]
    q0 = x.clone()
    ops.rope_apply_(x, cos, sin, H, hd, inverse=inverse)
    c = torch.cat([cos, cos], -1)[None]
    s = torch.cat([sin, sin], -1)[None]
    q = q0.view(1, rows, H, hd).transpose(1, 2)
    ref, _ = mo.apply_rope(q, q, c, -s if inverse else s)
    assert torch.equal(x.view(1, rows, H, hd), ref.transpose(1, 2))
    assert bool((buf[:, H * hd:] == 3.0).all())


# ---------------------------------------------------------------------------------------------------------------
# 4. SwiGLU backward
# ---------------------------------------------------------------------------------------------------------------
def test_swiglu_backward_large_gates_against_fp64():
    """Gates with ±0, ±88..±100 (exp(-g) past fp32's range either way) and silu''s zero spliced into randn, u and dh
    randn: dg, du within 2 bf16 ulps of the fp64 restatement (swiglu_bwd_bound says why 2), no NaN, and where exp(-g)
    overflows (g <= -89) the same zeros torch's fp32 silu gives."""
    dev = require_cuda()
    gen = torch.Generator().manual_seed(5)
    rows, cols = 300, 1024
    g = swiglu_gates(rows * cols, gen).view(rows, cols).to(dev)
    u = torch.randn(rows, cols, generator=gen).to(BF16).to(dev)
    dh = (4 * torch.randn(rows, cols, generator=gen)).to(BF16).to(dev)
    dg, du = ops.swiglu_bwd(g, u, dh)
    dg_ref, du_ref = swiglu_bwd_reference(g, u, dh)
    ratios = (_within("swiglu dg", dg, dg_ref, swiglu_bwd_bound(dg_ref)),
              _within("swiglu du", du, du_ref, swiglu_bwd_bound(du_ref)))
    big_neg = g.float() <= -89
    assert bool((dg[big_neg] == 0).all() and (du[big_neg] == 0).all())
    print("swiglu_bwd max err/bound dg, du:", [f"{q:.3g}" for q in ratios])


# ---------------------------------------------------------------------------------------------------------------
# 5. embedding add, fp32 -> bf16 cast
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("table", ["f32", "bf16", "none"])
def test_embed_add_edges(table):
    """Ids outside [0, vocab) give a zero embedding row; no table (ids None) gives E = 0 + proj; a bf16 table is read
    as is, an fp32 one rounded to bf16 first; 4100 x 1280 is more work than the grid cap (132 SMs x 16 CTAs x 256
    threads x 8 elements) so the grid-stride loop runs; NaN from the table (not only from proj) raises the flag.  Bits
    compared, NaN by position."""
    dev = require_cuda()
    gen = _gen(21, dev)
    V, d, rows = 1000, 1280, 4100
    emb = torch.randn(V, d, generator=gen, device=dev)
    if table == "bf16":
        emb = emb.to(BF16)
    ids = torch.randint(0, V, (rows,), generator=gen, device=dev)
    ids[:6] = torch.tensor([-1, V, V + 5, -(2 ** 40), 2 ** 40, V - 1])
    proj = torch.randn(rows, d, generator=gen, device=dev).to(BF16)
    proj[7, :8] = -0.0
    flag = torch.zeros(1, dtype=torch.int32, device=dev)
    if table == "none":
        e = ops.embed_add(None, None, proj, rows, d, flag)
        ref = torch.zeros(rows, d, device=dev, dtype=BF16) + proj
    else:
        e = ops.embed_add(ids, emb, proj, rows, d, flag)
        ok = (ids >= 0) & (ids < V)
        rows_e = torch.zeros(rows, d, device=dev, dtype=BF16)
        rows_e[ok] = emb[ids[ok]].to(BF16)
        ref = rows_e + proj
    assert bits_equal(e, ref) and int(flag.item()) == 0
    if table != "none":
        e_only = ops.embed_add(ids, emb, None, rows, d, flag)          # no projector rows: the table alone
        assert bits_equal(e_only, rows_e) and int(flag.item()) == 0
        emb[ids[50], 17] = float("nan")                                 # NaN from the table
        e = ops.embed_add(ids, emb, proj, rows, d, flag)
        rows_e[ok] = emb[ids[ok]].to(BF16)
        assert bits_equal(e, rows_e + proj) and int(flag.item()) == 1
        assert bool(torch.isnan(e[:, 17]).any())


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 6, 7, 8, 13, 100003])
def test_cast_bf16_edges(n):
    """n < 4 (no vector part) and n % 4 in {1, 2, 3}, with ±inf, values that overflow bf16, fp32 subnormals, ±0 and NaN
    at the front (the vector part, or the tail alone when n < 4) and at the back (the tail): the bits of torch's
    round-to-nearest-even cast, NaN by position."""
    dev = require_cuda()
    gen = torch.Generator().manual_seed(n)
    special = torch.tensor([float("inf"), -float("inf"), 3.4e38, -3.4e38, 1e-40, -1e-40, -0.0, 0.0, float("nan"),
                            1.0 + 2 ** -8, 1.0 + 3 * 2 ** -8, 2.0 ** -133], dtype=torch.float32)
    x = 3 * torch.randn(n, generator=gen)
    k = min(n, len(special))
    x[:k] = special[:k]
    if n >= 2 * len(special):
        x[n - k:] = special.flip(0)
    got = ops.cast_bf16(x.to(dev))
    assert bits_equal(got.cpu(), x.to(BF16))


def test_cast_bf16_rejects_misaligned_source():
    dev = require_cuda()
    buf = torch.zeros(64, device=dev)
    with pytest.raises(_lib.TouchNetB200Error):
        ops.cast_bf16(buf[1:33])                                         # 4 bytes past a 16-byte boundary


# ---------------------------------------------------------------------------------------------------------------
# 6. strided rows through the autograd functions
# ---------------------------------------------------------------------------------------------------------------
# Each input is a column slice of a wider tensor and each output is fed into torch.cat, so that the input and the
# gradient coming back are row-strided views inside larger allocations.  The results must equal the same calls on
# contiguous copies bit for bit, and fp32 autograd of the same function within bf16 noise.
def _through_cat(fn, x_wide, d, gen, extra_cols=8):
    """Run fn on x_wide[:, :d] (a leaf's column slice), cat its output with noise, backward; return the output, the
    gradient of the slice (from the leaf's grad) and the upstream gradient used for fn's output."""
    xl = x_wide.detach().clone().requires_grad_(True)
    y = fn(xl[..., :d])
    z = torch.randn(*y.shape[:-1], extra_cols, generator=gen, device=y.device).to(y.dtype)
    gout = torch.randn(*y.shape[:-1], y.shape[-1] + extra_cols, generator=gen, device=y.device).to(y.dtype)
    torch.cat([y, z], -1).backward(gout)
    assert bool((xl.grad[..., d:] == 0).all())
    return y.detach(), xl.grad[..., :d], gout[..., :y.shape[-1]]


def _contiguous_run(fn, x, gy):
    xc = x.detach().clone().requires_grad_(True)
    y = fn(xc)
    y.backward(gy.contiguous())
    return y.detach(), xc.grad


def _param_grads_and_reset(params):
    out = [p.grad.clone() for p in params]
    for p in params:
        p.grad = None
    return out


def test_rms_norm_strided_rows():
    dev = require_cuda()
    gen = _gen(31, dev)
    R, d = 300, 1024
    w = torch.nn.Parameter(1 + 0.1 * torch.randn(d, generator=gen, device=dev))
    x_wide = torch.randn(R, 2 * d, generator=gen, device=dev).to(BF16)
    fn = lambda t: ops.rms_norm(t, w, EPS)
    y, dx, gy = _through_cat(fn, x_wide, d, gen)
    (dw,) = _param_grads_and_reset([w])
    x = x_wide[:, :d]
    yc, dxc = _contiguous_run(fn, x, gy)
    (dwc,) = _param_grads_and_reset([w])
    assert torch.equal(y, yc) and torch.equal(dx, dxc) and torch.equal(dw, dwc)
    xf = x.float().requires_grad_(True)
    wf = w.detach().to(BF16).float().requires_grad_(True)
    yf = wf * (xf * torch.rsqrt(xf.square().mean(-1, keepdim=True) + EPS))
    yf.backward(gy.float())
    assert float((y.float() - yf).abs().max()) <= 2 ** -6 * float(yf.abs().max())
    assert rel_err(dx.float(), xf.grad) < 1e-2 and rel_err(dw, wf.grad) < 1e-2


def test_swiglu_mlp_in_strided_rows():
    dev = require_cuda()
    gen = _gen(32, dev)
    R, d, n = 300, 512, 1024
    wg = torch.nn.Parameter(0.05 * torch.randn(n, d, generator=gen, device=dev))
    wu = torch.nn.Parameter(0.05 * torch.randn(n, d, generator=gen, device=dev))
    x_wide = torch.randn(R, d + 64, generator=gen, device=dev).to(BF16)
    fn = lambda t: ops.swiglu_mlp_in(t, wg, wu)
    h, dx, gh = _through_cat(fn, x_wide, d, gen)
    dwg, dwu = _param_grads_and_reset([wg, wu])
    x = x_wide[:, :d]
    hc, dxc = _contiguous_run(fn, x, gh)
    dwgc, dwuc = _param_grads_and_reset([wg, wu])
    assert torch.equal(h, hc) and torch.equal(dx, dxc) and torch.equal(dwg, dwgc) and torch.equal(dwu, dwuc)
    xf = x.float().requires_grad_(True)
    wgf = wg.detach().to(BF16).float().requires_grad_(True)
    wuf = wu.detach().to(BF16).float().requires_grad_(True)
    hf = torch.nn.functional.silu(xf @ wgf.t()) * (xf @ wuf.t())
    hf.backward(gh.float())
    assert rel_err(h.float(), hf) < 1e-2
    assert rel_err(dx.float(), xf.grad) < 1e-2 and rel_err(dwg, wgf.grad) < 1e-2 and rel_err(dwu, wuf.grad) < 1e-2


def test_decoder_layer_strided_rows():
    dev = require_cuda()
    gen = _gen(33, dev)
    T, d, H, KV, hd, ffn = 256, 256, 2, 1, 128, 512
    rn = lambda *s: torch.randn(*s, generator=gen, device=dev)
    names = ("ln1", "wq", "wk", "wv", "wo", "ln2", "wg", "wu", "wd")
    shapes = {"ln1": (d,), "wq": (H * hd, d), "wk": (KV * hd, d), "wv": (KV * hd, d), "wo": (d, H * hd), "ln2": (d,),
              "wg": (ffn, d), "wu": (ffn, d), "wd": (d, ffn)}
    P = {k: torch.nn.Parameter(1 + 0.1 * rn(*s) if k.startswith("ln") else 0.05 * rn(*s)) for k, s in shapes.items()}
    doc = torch.ones(1, T, dtype=torch.int64, device=dev)
    doc[0, 150:] = 2
    pos = torch.cat([torch.arange(150), torch.arange(T - 150)]).to(dev)[None]
    inv, sc = mo.rope_inv_freq(mo.OracleConfig(d, ffn, 1, H, KV, hd, 8, rope_theta=500000.0))
    cos, sin = ops.rope_table(pos, inv.to(dev), sc)
    plan = ops.AttnPlan(doc)
    fn = lambda t: ops.decoder_layer(t, P["ln1"], P["wq"], P["wk"], P["wv"], None, None, None, P["wo"], P["ln2"],
                                     P["wg"], P["wu"], P["wd"], cos, sin, plan, H, KV, EPS)
    x_wide = rn(T, 2 * d).to(BF16)
    out, dx, gout = _through_cat(fn, x_wide, d, gen)
    grads = _param_grads_and_reset([P[k] for k in names])
    x = x_wide[:, :d]
    outc, dxc = _contiguous_run(fn, x, gout)
    gradsc = _param_grads_and_reset([P[k] for k in names])
    assert torch.equal(out, outc) and torch.equal(dx, dxc)
    assert all(torch.equal(a, b) for a, b in zip(grads, gradsc))
    # fp32 autograd of the oracle layer on the same bf16 weights
    full = {"input_layernorm.weight": "ln1", "self_attn.q_proj.weight": "wq", "self_attn.k_proj.weight": "wk",
            "self_attn.v_proj.weight": "wv", "self_attn.o_proj.weight": "wo", "post_attention_layernorm.weight": "ln2",
            "mlp.gate_proj.weight": "wg", "mlp.up_proj.weight": "wu", "mlp.down_proj.weight": "wd"}
    pf = {k: P[v].detach().to(BF16).float().requires_grad_(True) for k, v in full.items()}
    xf = x.float()[None].requires_grad_(True)
    cfg = mo.OracleConfig(d, ffn, 1, H, KV, hd, 8, rms_norm_eps=EPS, rope_theta=500000.0)
    c = torch.cat([cos, cos], -1).float()[None]
    s = torch.cat([sin, sin], -1).float()[None]
    of = mo.decoder_layer(xf, pf, "", cfg, c, s, mo.doc_causal_allow(doc))
    of.backward(gout.float()[None])
    assert rel_err(out.float(), of[0]) < 1e-2 and rel_err(dx.float(), xf.grad[0]) < 2e-2
    for k, v in full.items():
        assert rel_err(grads[names.index(v)].float(), pf[k].grad) < 3e-2, k
