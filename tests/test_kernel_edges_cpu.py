"""fp64 references and element-wise error bounds for the bf16 GEMM, RMSNorm and the SwiGLU backward, shared with
tests/test_gpu_kernel_edges.py, and the checks that those bounds have teeth: a CPU emulation of each kernel's rounding
points stays within its bound, and a kernel that is wrong in one of the ways listed below does not.

  * GEMM (tn_gemm_bf16): D = op(A)·op(B), fp32 accumulation over 64-wide k-blocks, bf16 or fp32 output.
    Bound: 2^-8·|ref| (bf16 output rounding: half an ulp is up to 2^-8 of the value) + K·2^-23·(|A|·|B|) (fp32
    accumulation of K products; 2^-23 rather than 2^-24 leaves room for the tensor cores' truncating adds).  fp32
    output: the second term only.
    Mutations: one k-block dropped at K = 72; one output row taken from the wrong input row.
  * RMSNorm forward: y = bf16(t·w), t = bf16(x·rstd) (HF's rounding points) with rstd in fp64.  Bound: one step of the
    inner rounding point t (the kernel's fp32 rstd can flip it) carried through w, |w|·ulp(t), plus the two outer
    roundings, 1.5·ulp(y); rstd itself within d·2^-23 relative.  Mutation: the reduction stopped at 4096 columns.
  * RMSNorm backward: dS by fp64 autograd, dW as the sum of dy·bf16(x·rstd) over rows.  Bounds: output rounding plus
    (terms summed)·2^-23·(sum of their absolute values), see rmsnorm_bwd_bound.
  * SwiGLU backward: du = bf16(dh·bf16(silu(g))), dg = bf16(bf16(dh·u)·silu'(g)) with sigmoid in fp64.  Bound: 2 bf16
    ulps, see swiglu_bwd_bound.  Mutation: silu' with g in place of sig."""
import math

import torch

BF16 = torch.bfloat16
U23 = 2.0 ** -23
FLT_MAX = float(torch.finfo(torch.float32).max)
KBLOCK = 64                      # k-block of the GEMM mainloop (BK in gemm.cu)
NORM_PARTIALS = 528              # tn_rmsnorm_bwd_num_partials(): CTAs of the RMSNorm backward, each summing its rows


def bf16_ulp(v: torch.Tensor) -> torch.Tensor:
    """Spacing of bf16 numbers at |v| (fp64): 2^(e - 7) for |v| in [2^e, 2^(e+1)), 2^-133 in the subnormal range."""
    e = torch.floor(torch.log2(v.double().abs().clamp_min(2.0 ** -126)))
    return torch.exp2(e - 7)


def violations(got: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor) -> int:
    """Elements with |got - ref| > bound (NaN counts)."""
    err = (got.double() - ref.double()).abs()
    return int((~(err <= bound)).sum())


def bits_equal(got: torch.Tensor, ref: torch.Tensor) -> bool:
    """Same bits everywhere (so -0 differs from +0), except that a NaN only has to meet a NaN."""
    if got.shape != ref.shape or got.dtype != ref.dtype:
        return False
    gn, rn = torch.isnan(got), torch.isnan(ref)
    if not torch.equal(gn, rn):
        return False
    ib = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[got.element_size()]
    return torch.equal(got[~gn].view(ib), ref[~rn].view(ib))


# ---------------------------------------------------------------------------------------------------------------
# GEMM
# ---------------------------------------------------------------------------------------------------------------
def _operands(a, b, a_mn, b_mn):
    """op(A) [M, K] and op(B) [K, N] as fp64: a is [M, K] ([K, M] if a_mn), b is [N, K] ([K, N] if b_mn)."""
    A = (a.t() if a_mn else a).double()
    B = (b if b_mn else b.t()).double()
    return A, B


def gemm_reference(a, b, *, a_mn=False, b_mn=False):
    """(op(A)·op(B), |op(A)|·|op(B)|) in fp64 on the bf16 operands."""
    A, B = _operands(a, b, a_mn, b_mn)
    return A @ B, A.abs() @ B.abs()


def gemm_bound(ref, absprod, K: int, out_f32: bool):
    acc = K * U23 * absprod
    return acc if out_f32 else acc + 2.0 ** -8 * ref.abs()


def gemm_emulate(a, b, *, a_mn=False, b_mn=False, out_f32=False, drop_kblock=None, row_from=None):
    """The kernel's rounding points on the CPU: one fp32 partial product per 64-wide k-block, added into an fp32
    accumulator in k order, rounded to bf16 at the end.  drop_kblock / row_from=(dst, src) are the mutations."""
    A, B = (t.float() for t in _operands(a, b, a_mn, b_mn))
    acc = torch.zeros(A.shape[0], B.shape[1], dtype=torch.float32)
    for i, k0 in enumerate(range(0, A.shape[1], KBLOCK)):
        if i != drop_kblock:
            acc = acc + A[:, k0:k0 + KBLOCK] @ B[k0:k0 + KBLOCK]
    if row_from is not None:
        acc[row_from[0]] = acc[row_from[1]]
    return acc if out_f32 else acc.to(BF16)


# ---------------------------------------------------------------------------------------------------------------
# RMSNorm
# ---------------------------------------------------------------------------------------------------------------
def rstd_reference(x, eps):
    xd = x.double()
    return torch.rsqrt(xd.square().mean(-1) + eps)


def rmsnorm_fwd_reference(x, w, eps):
    """(y, rstd): HF's rounding points y = bf16(bf16(x·rstd)·bf16(w)) evaluated with the fp64 rstd."""
    rstd = rstd_reference(x, eps)
    t = (x.double() * rstd[:, None]).to(BF16).double()
    return (t * w.to(BF16).double()).to(BF16), rstd


def rmsnorm_fwd_bound(x, w, rstd_ref, y_ref):
    """|w|·ulp(t) + 1.5·ulp(y).  An fp32 rstd, any fp32 rstd, lands x·rstd on the other side of a bf16 rounding midpoint
    of t now and then; where y = t·w falls a binade below t (|w| < 1) that one step of t is two ulps of y, and the
    outer roundings add up to 1.5 more (the kernel's y may sit a binade above the reference's)."""
    t = (x.double() * rstd_ref[:, None]).to(BF16).double()
    return w.to(BF16).double().abs() * bf16_ulp(t) + 1.5 * bf16_ulp(y_ref)


def rmsnorm_fwd_at(x, w, rstd):
    """HF's rounding points at a given fp32 rstd, exactly as the kernel evaluates them: fp32 x·rstd rounded to bf16,
    times bf16(w) rounded once."""
    return ((x.float() * rstd.float()[:, None]).to(BF16).float() * w.to(BF16).float()).to(BF16)


def rstd_bound(rstd_ref, d: int):
    return d * U23 * rstd_ref


def rmsnorm_fwd_emulate(x, w, eps, reduce_cols=None):
    """fp32 sum of squares, fp32 rstd, the two bf16 roundings.  reduce_cols: the mutation that stops the sum early."""
    xf = x.float()
    d = x.shape[1]
    ss = xf[:, :reduce_cols].square().sum(-1)
    rstd = torch.rsqrt(ss / d + eps)
    return ((xf * rstd[:, None]).to(BF16).float() * w.to(BF16).float()).to(BF16), rstd


def rmsnorm_bwd_reference(x, dy, w, rstd_k, eps, extra=None):
    """(ds, ds_no_extra, dw) by fp64 autograd of y = w·(x·rstd) with the exact rstd; the forward's bf16 cast of x·rstd
    is the identity for dS (as in HF's autograd) and, for dW, sits at the value the kernel rounded: bf16(x·rstd_k) with
    the forward's fp32 rstd_k."""
    xd = x.double().requires_grad_(True)
    wd = w.to(BF16).double().requires_grad_(True)
    xn = xd * torch.rsqrt(xd.square().mean(-1, keepdim=True) + eps)
    xn_b = (x.float() * rstd_k.float()[:, None]).to(BF16).double()
    (wd * (xn + (xn_b - xn).detach())).backward(dy.double())
    ds = xd.grad
    return (ds if extra is None else ds + extra.double()), ds, wd.grad


def rmsnorm_bwd_bound(x, dy, w, rstd_k, ds_no_extra, extra=None):
    """(dS bound, dW bound).
    dS_i = rstd·(g_i - xn_i·Σ_j g_j·xn_j / d) with g = dy·w, xn = x·rstd.  With a_i = rstd·|g_i| and
    b_i = rstd³·|x_i|·Σ_j |g_j·x_j| / d: the kernel's rstd (relative error δ = d·2^-23, the forward's bound) moves the
    first term by δ·a_i and the second by 3δ·b_i; the d-term fp32 dot product adds d·2^-23·b_i; a few fp32 roundings
    2^-22·(a_i + b_i).  Output: bf16 rounding of that (2^-8·|ref| covers the half ulp of the fp32 value, twice the
    compute error for its own rounding), and with the fused residual gradient a second bf16 rounding of the sum.
    dW_j = Σ_rows dy·bf16(xn): each CTA sums its rows in fp32, the partials are summed in 32 lanes then across them:
    (ceil(rows / 528) + 17 + 32)·2^-23·Σ_rows |dy·bf16(xn)|."""
    rows, d = x.shape
    rstd = rstd_k.double()[:, None]
    g = (dy.double() * w.to(BF16).double()).abs()
    xa = x.double().abs()
    a = rstd * g
    b = rstd ** 3 * xa * (g * xa).sum(-1, keepdim=True) / d
    delta = d * U23
    E = delta * a + (3 * delta + d * U23) * b + 2.0 ** -22 * (a + b)
    ds_bound = 2.0 ** -8 * ds_no_extra.abs() + 2 * E
    if extra is not None:
        ds_bound = ds_bound + 2.0 ** -8 * (ds_no_extra + extra.double()).abs()
    xn_b = (x.float() * rstd_k.float()[:, None]).to(BF16).double()
    n_add = math.ceil(rows / NORM_PARTIALS) + math.ceil(NORM_PARTIALS / 32) + 32
    dw_bound = n_add * U23 * (dy.double() * xn_b).abs().sum(0)
    return ds_bound, dw_bound


def rmsnorm_bwd_emulate(x, dy, w, rstd_k, extra=None):
    """The kernel's rounding points on the CPU (fp32 throughout, bf16 output, bf16 add of the residual gradient)."""
    xf, g = x.float(), dy.float() * w.to(BF16).float()
    r = rstd_k.float()[:, None]
    xn = xf * r
    mean_dot = (g * xn).sum(-1, keepdim=True) / x.shape[1]
    ds = (r * (g - xn * mean_dot)).to(BF16)
    if extra is not None:
        ds = (ds.float() + extra.float()).to(BF16)
    dw = (dy.float() * xn.to(BF16).float()).sum(0)
    return ds, dw


# ---------------------------------------------------------------------------------------------------------------
# SwiGLU backward
# ---------------------------------------------------------------------------------------------------------------
def swiglu_bwd_reference(g, u, dh):
    """(dg, du) at the kernel's (and the unfused HF ops') bf16 rounding points, everything between them in fp64.
    exp(-g) is taken in fp32's range, as the kernel and torch's fp32 silu take it: beyond FLT_MAX (g <= -89 in bf16)
    it is inf, so sigmoid, silu(g) and silu'(g) are zero there."""
    gd = g.double()
    e = torch.exp(-gd)
    e = torch.where(e > FLT_MAX, torch.full_like(e, math.inf), e)
    sig = 1.0 / (1.0 + e)
    silu_b = (gd * sig).to(BF16).double()
    du = (dh.double() * silu_b).to(BF16)
    dg = ((dh.double() * u.double()).to(BF16).double() * (sig * (1.0 + gd * (1.0 - sig)))).to(BF16)
    return dg, du


def swiglu_bwd_bound(ref):
    """2 bf16 ulps.  The kernel's sigmoid comes from __expf, whose error (2 + 1.2·|g| fp32 ulps, under 2^-15 relative
    for |g| <= 100) is far below a bf16 ulp, and from IEEE fp32 divides and products.  For du that can flip the inner
    rounding point bf16(silu(g)) by one ulp (at most 2^-7 relative), which moves dh·silu(g) by at most 2 ulps of the
    result, and output rounding cannot then add a third.  For dg the inner point bf16(dh·u) is exact, and the fp32
    error of silu'(g), even at the bf16 gate closest to its zero (g = -1.28125, where its terms cancel 740-fold), stays
    below one ulp: the output may land one ulp off.  2 ulps cover both."""
    return 2 * bf16_ulp(ref)


def swiglu_bwd_emulate(g, u, dh, mutate_sig=False):
    """The kernel's arithmetic in fp32 (torch's exp in place of __expf).  mutate_sig: silu' = g·(1 + g·(1 - sig))."""
    gf, uf, dhf = g.float(), u.float(), dh.float()
    sig = 1.0 / (1.0 + torch.exp(-gf))
    du = (dhf * (gf * sig).to(BF16).float()).to(BF16)
    lead = gf if mutate_sig else sig
    dg = ((dhf * uf).to(BF16).float() * (lead * (1.0 + gf * (1.0 - sig)))).to(BF16)
    return dg, du


def swiglu_gates(n: int, gen: torch.Generator) -> torch.Tensor:
    """randn gates with the edges spliced in: ±0, ±88..±100 (exp(-g) over and under fp32's range) and the bf16 gates
    on either side of silu''s zero."""
    edge = [0.0, -0.0, 88.0, 88.5, 89.0, 90.0, 95.0, 100.0, -88.0, -88.5, -89.0, -90.0, -95.0, -100.0,
            -1.2734375, -1.28125, 20.0, -20.0]
    g = torch.randn(n, generator=gen)
    g[:len(edge)] = torch.tensor(edge)
    return g.to(BF16)


# ---------------------------------------------------------------------------------------------------------------
# teeth, without a GPU
# ---------------------------------------------------------------------------------------------------------------
def _gen(seed):
    return torch.Generator().manual_seed(seed)


def test_bf16_ulp_and_bits_helpers():
    v = torch.tensor([1.0, 1.5, 2.0, 0.75, 2.0 ** -130, 0.0], dtype=torch.float64)
    assert bf16_ulp(v).tolist() == [2.0 ** -7, 2.0 ** -7, 2.0 ** -6, 2.0 ** -8, 2.0 ** -133, 2.0 ** -133]
    a = torch.tensor([0.0, 1.0, float("nan")], dtype=BF16)
    assert bits_equal(a, a.clone())
    assert not bits_equal(a, torch.tensor([-0.0, 1.0, float("nan")], dtype=BF16))     # signed zero counts
    assert not bits_equal(a, torch.tensor([0.0, float("nan"), 1.0], dtype=BF16))      # NaN positions count


def test_gemm_bound_holds_for_emulation_and_catches_mutations():
    gen = _gen(0)
    M, N, K = 9, 40, 72
    a = torch.randn(M, K, generator=gen).to(BF16)
    b = (0.1 * torch.randn(N, K, generator=gen)).to(BF16)
    for out_f32 in (False, True):
        ref, absprod = gemm_reference(a, b)
        bound = gemm_bound(ref, absprod, K, out_f32)
        assert violations(gemm_emulate(a, b, out_f32=out_f32), ref, bound) == 0
        assert violations(gemm_emulate(a, b, out_f32=out_f32, drop_kblock=1), ref, bound) > 0
        assert violations(gemm_emulate(a, b, out_f32=out_f32, row_from=(3, 4)), ref, bound) > 0
    # the other layouts through the same reference: dgrad (b [K, N]) and wgrad (a [K, M], b [K, N]) with few tokens
    bk = b.t().contiguous()
    ref, absprod = gemm_reference(a, bk, b_mn=True)
    assert violations(gemm_emulate(a, bk, b_mn=True), ref, gemm_bound(ref, absprod, K, False)) == 0
    at, bt = a[:5].contiguous(), (0.1 * torch.randn(5, N, generator=gen)).to(BF16)
    ref, absprod = gemm_reference(at, bt, a_mn=True, b_mn=True)
    assert ref.shape == (K, N)
    bound = gemm_bound(ref, absprod, 5, True)
    assert violations(gemm_emulate(at, bt, a_mn=True, b_mn=True, out_f32=True), ref, bound) == 0
    assert violations(gemm_emulate(at, bt, a_mn=True, b_mn=True, out_f32=True, row_from=(0, 1)), ref, bound) > 0


def test_rmsnorm_bounds_hold_for_emulation_and_catch_mutations():
    gen = _gen(1)
    eps = 1e-5
    for rows, d in ((7, 8), (5, 24), (6, 8192)):
        x = torch.randn(rows, d, generator=gen).to(BF16)
        w = (1 + 0.1 * torch.randn(d, generator=gen))
        y_ref, rstd_ref = rmsnorm_fwd_reference(x, w, eps)
        y, rstd = rmsnorm_fwd_emulate(x, w, eps)
        assert violations(y, y_ref, rmsnorm_fwd_bound(x, w, rstd_ref, y_ref)) == 0
        assert torch.equal(y, rmsnorm_fwd_at(x, w, rstd))
        assert violations(rstd, rstd_ref, rstd_bound(rstd_ref, d)) == 0
        dy = torch.randn(rows, d, generator=gen).to(BF16)
        extra = torch.randn(rows, d, generator=gen).to(BF16)
        for ex in (None, extra):
            ds_ref, ds0, dw_ref = rmsnorm_bwd_reference(x, dy, w, rstd, eps, ex)
            ds_b, dw_b = rmsnorm_bwd_bound(x, dy, w, rstd, ds0, ex)
            ds, dw = rmsnorm_bwd_emulate(x, dy, w, rstd, ex)
            assert violations(ds, ds_ref, ds_b) == 0 and violations(dw, dw_ref, dw_b) == 0
    # the reduction stopped at 4096 columns of an 8192-wide row
    y, rstd = rmsnorm_fwd_emulate(x, w, eps, reduce_cols=4096)
    assert violations(y, y_ref, rmsnorm_fwd_bound(x, w, rstd_ref, y_ref)) > 0
    assert violations(rstd, rstd_ref, rstd_bound(rstd_ref, 8192)) > 0


def test_swiglu_bound_holds_for_emulation_and_catches_mutation():
    gen = _gen(2)
    n = 4096
    g = swiglu_gates(n, gen)
    u = torch.randn(n, generator=gen).to(BF16)
    dh = torch.randn(n, generator=gen).to(BF16)
    dg_ref, du_ref = swiglu_bwd_reference(g, u, dh)
    dg, du = swiglu_bwd_emulate(g, u, dh)
    assert violations(dg, dg_ref, swiglu_bwd_bound(dg_ref)) == 0
    assert violations(du, du_ref, swiglu_bwd_bound(du_ref)) == 0
    assert not (torch.isnan(dg).any() or torch.isnan(du).any())
    dg_m, _ = swiglu_bwd_emulate(g, u, dh, mutate_sig=True)
    assert violations(dg_m, dg_ref, swiglu_bwd_bound(dg_ref)) > 0
