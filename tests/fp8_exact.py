"""Operands whose FP8 GEMM product is exact, their exact references, and restatements of the kernels' tile choices;
shared by tests/test_fp8_exact_cpu.py and tests/test_gpu_fp8_exact.py.

Exact operands.  A and B hold small integers (A in {±1, ±2, ±3}, B in {±1, ±2}), exact in e4m3 and e5m2.  A row m
of A is nonzero only at k ≡ m (mod `a_stride(K)`), so that Σ_k |a_mk · b_nk| ≤ CAP = 2^12 for every (m, n).  Each
row of A and each row of B then gets a power-of-two factor 2^e, e in [-6, 6]: as a rowwise 1/s (the rowwise GEMMs and
the decode kernel), or folded into the 8-bit values (the tensorwise GEMMs, whose 1/s are scalars).  Every product of
an output element is then an integer multiple of one quantum q = 2^(e_m + e_n), and every partial sum, in any order,
is a multiple of q below CAP · q: an accumulator that keeps 13 significant bits adds it exactly.  Every correct kernel
therefore reproduces the exact product bit for bit, whatever its summation order; the bf16 result is the exact value
(exactly representable in fp32) rounded to nearest even.

The exponents are drawn so that a row's (column's) e differs from that of its neighbours at ±1, ±8 and ±64: a kernel
that applies a neighbour's scale, or a wrong segment's, changes almost every element it touches.

Promotion witness.  Stage 0 (k < 128) holds one product of 2^16 per element, the last 128-k stage one of -2^16, and
the stages between hold small products.  A kernel that adds each stage's partial sum into an fp32 accumulator returns
the small sum exactly; one that accumulates across stages in the tensor core, with ~14 bits aligned to the 2^16 term,
loses it.

The tile restatements mirror csrc/gemm.cu (`pick_bn`, `fp8_wide_ok`) and csrc/float8.cu (`dec_pitch`, `dec_smem`, the
row-group choice of `tn_gemm_fp8_decode`)."""
import functools
import math

import torch

CAP = 2 ** 12                    # Σ|products| per element, in quanta
E_LO, E_HI = -6, 6               # exponent range of the row / column factors
NEIGHBOURS = (1, 8, 64)          # offsets at which neighbouring exponents differ
A_MAX, B_MAX = 3, 2              # largest |entry| of A and of B
KSTAGE = 128                     # k per mainloop stage of the FP8 wgmma GEMMs
BM = 128                         # M rows per wgmma tile
WIDE_TILE_COST = 1.8             # gemm.cu kWideTileCost
WITNESS = 2 ** 16                # the large product of the promotion witness


# ---------------------------------------------------------------------------------------------------------------
# operands
# ---------------------------------------------------------------------------------------------------------------
def exponents(n: int, seed: int, extra=()) -> torch.Tensor:
    """int64 [n] in [E_LO, E_HI], each drawn uniformly from the values not taken by the entries already drawn at -1,
    -8 and -64, so every entry differs from its neighbours at ±1, ±8 and ±64.  `extra`: (start, shift) pairs, entry
    i >= start also differs from entry i - shift (the up half of a SwiGLU scale vector from the gate half, a QKV
    segment from the one before it)."""
    return _exponents(n, seed, tuple(extra)).clone()


@functools.lru_cache(maxsize=64)
def _exponents(n, seed, extra):
    g = torch.Generator().manual_seed(seed)
    vals = list(range(E_LO, E_HI + 1))
    draws = torch.randint(0, 1 << 30, (n,), generator=g).tolist()
    e = []
    for i in range(n):
        taken = {e[i - d] for d in NEIGHBOURS if i - d >= 0}
        taken |= {e[i - s] for start, s in extra if i >= start and i - s >= 0}
        free = [v for v in vals if v not in taken]
        e.append(free[draws[i] % len(free)])
    return torch.tensor(e, dtype=torch.int64)


def neighbour_spread(e: torch.Tensor) -> float:
    """Fraction of entries whose exponent differs from every existing neighbour at ±1, ±8 and ±64."""
    ok = torch.ones(e.numel(), dtype=torch.bool)
    for d in NEIGHBOURS:
        if d < e.numel():
            diff = e[d:] != e[:-d]
            ok[d:] &= diff
            ok[:-d] &= diff
    return float(ok.float().mean())


def a_stride(K: int) -> int:
    """Smallest power of two S such that a row of A with a nonzero at every k ≡ m (mod S) stays under CAP."""
    s = 1
    while math.ceil(K / s) * A_MAX * B_MAX > CAP:
        s *= 2
    return s


def _gen(device, seed):
    return torch.Generator(device=device).manual_seed(seed)


def int_a(M: int, K: int, seed: int, device="cpu", stride=None) -> torch.Tensor:
    """float32 [M, K] of integers: row m is ±1, ±2 or ±3 at k ≡ m (mod stride), 0 elsewhere.  Every residue class
    of k occurs in every run of `stride` columns, so each row has nonzeros in the last (partial) k stage."""
    s = a_stride(K) if stride is None else stride
    g = _gen(device, seed)
    nk = -(-K // s)
    m = torch.arange(M, device=device)
    k = (m % s)[:, None] + s * torch.arange(nk, device=device)[None, :]      # [M, nk]: the nonzero columns of row m
    v = _signed(M, nk, A_MAX, g, device)
    ok = k < K
    a = torch.zeros(M, K, device=device)
    a[m[:, None].expand(M, nk)[ok], k[ok]] = v[ok]
    return a


def _signed(rows, cols, vmax, g, device):
    """float32 [rows, cols] uniform over ±1 .. ±vmax."""
    mag = torch.randint(1, vmax + 1, (rows, cols), device=device, generator=g, dtype=torch.int8)
    sign = torch.randint(0, 2, (rows, cols), device=device, generator=g, dtype=torch.int8)
    return (mag * (2 * sign - 1)).float()


def int_b(N: int, K: int, seed: int, device="cpu") -> torch.Tensor:
    """float32 [N, K] of ±1 and ±2."""
    return _signed(N, K, B_MAX, _gen(device, seed), device)


def int_x(M: int, K: int, seed: int, device="cpu", zero_row=None) -> torch.Tensor:
    """int_a with a 3 in every row (its amax: the decode kernel's row scale is then 2^(e - 7) for a row scaled by
    2^e, and its bytes are ±128, ±256, ±384) and row `zero_row` all zero."""
    a = int_a(M, K, seed, device)
    m = torch.arange(M, device=device)
    a[m, m % a_stride(K)] = 3.0
    if zero_row is not None and zero_row < M:
        a[zero_row] = 0
    return a


def abs_bound(a: torch.Tensor, b: torch.Tensor) -> float:
    """An upper bound of max_{m,n} Σ_k |a_mk · b_nk| (in quanta): the largest row sum of |a| times max |b|."""
    return float(a.abs().double().sum(1).max()) * float(b.abs().max())


def witness(M: int, N: int, K: int, seed: int, device="cpu"):
    """(A, B) float32 integers for the promotion witness: A[:, 0] = 256 and A[:, K-1] = -256 against B = 256 there,
    so stage 0 holds +2^16 and the last stage -2^16; in each stage between, A row m is ±1 at 4 of its 128 k, B ±1.
    The exact product is the small sum, |S| ≤ 4 · (stages - 2) < 256 (bf16-exact)."""
    assert K % KSTAGE == 0 and K >= 3 * KSTAGE
    g = _gen(device, seed)
    a = torch.zeros(M, K, device=device)
    m = torch.arange(M, device=device)
    for st in range(1, K // KSTAGE - 1):
        for j in range(4):
            k = st * KSTAGE + (m * 5 + 32 * j) % KSTAGE
            a[m, k] = (torch.randint(0, 2, (M,), device=device, generator=g) * 2 - 1).float()
    b = (torch.randint(0, 2, (N, K), device=device, generator=g) * 2 - 1).float()
    a[:, 0], a[:, K - 1] = 256.0, -256.0
    b[:, 0], b[:, K - 1] = 256.0, 256.0
    return a, b


def pow2(e: torch.Tensor, device=None) -> torch.Tensor:
    """float32 2^e."""
    return torch.exp2(e.double()).float().to(device if device is not None else e.device)


def fp8(x: torch.Tensor, dtype) -> torch.Tensor:
    """x as an 8-bit float; asserts that every value is exact."""
    q = x.to(dtype)
    assert torch.equal(q.float(), x.float()), "value not exact in " + str(dtype)
    return q


# ---------------------------------------------------------------------------------------------------------------
# references
# ---------------------------------------------------------------------------------------------------------------
def exact(a: torch.Tensor, b: torch.Tensor, ia=None, ib=None) -> torch.Tensor:
    """(A · diag(ia)) (B · diag(ib))ᵀ in fp64 on the operands' device (ia [M], ib [N]; None: ones)."""
    A, B = a.double(), b.double()
    if ia is not None:
        A = A * ia.double()[:, None]
    if ib is not None:
        B = B * ib.double()[:, None]
    return A @ B.t()


def bf16(x: torch.Tensor) -> torch.Tensor:
    """The bf16 result of an exact value: fp32 first (exact here), then round to nearest even."""
    return x.float().bfloat16()


# ---------------------------------------------------------------------------------------------------------------
# emulated accumulation
# ---------------------------------------------------------------------------------------------------------------
def emulate_acc(a: torch.Tensor, b: torch.Tensor, bits: int = 13, group: int = 32, promote: bool = False):
    """fp64 [m, n]: Σ_k a_mk · b_nk through an accumulator with `bits` significant bits.  Every `group` k (one wgmma
    k32 step) the accumulator and the group's products are aligned to the largest exponent among them, truncated
    toward zero to `bits` bits below it, and added.  promote: the accumulator restarts at every 128-k stage and the
    stage sums are added in exact arithmetic (an fp32 accumulator is exact for these integers below 2^24)."""
    A, B = a.double(), b.double()
    K = A.shape[1]
    total = torch.zeros(A.shape[0], B.shape[0], dtype=torch.float64)
    acc = torch.zeros_like(total)
    for k0 in range(0, K, group):
        if promote and k0 % KSTAGE == 0 and k0:
            total, acc = total + acc, torch.zeros_like(acc)
        t = torch.cat([acc[..., None], A[:, None, k0:k0 + group] * B[None, :, k0:k0 + group]], -1)
        mx = t.abs().amax(-1)
        e = torch.where(mx > 0, torch.floor(torch.log2(mx.clamp_min(1e-300))), torch.zeros_like(mx))
        qn = torch.exp2(e - (bits - 1))[..., None]
        acc = (torch.trunc(t / qn) * qn).sum(-1)
    total = total + acc
    if promote:
        assert float(total.abs().max()) < 2 ** 24
    return total


# ---------------------------------------------------------------------------------------------------------------
# restated tile choices
# ---------------------------------------------------------------------------------------------------------------
def sm_count(margin: int = 0) -> int:
    """SMs the library launches on: the device's count minus tn_set_sm_margin's margin (at least 2)."""
    n = torch.cuda.get_device_properties(0).multi_processor_count
    return max(n - margin, 2)


def pick_bn(M: int, N: int, out_div: int, sms: int) -> int:
    """gemm.cu pick_bn: the 256-wide tile unless its last, partly idle wave costs more than it saves."""
    nm = -(-M // BM)
    wide = nm * -(-N // (256 // out_div))
    narrow = nm * -(-N // (128 // out_div))
    return 256 if -(-wide // sms) * WIDE_TILE_COST <= -(-narrow // sms) else 128


# gemm_kernel's OP: 1 tensorwise e4m3 A, 2 tensorwise e5m2 A (promoted), 3 rowwise, 4 rowwise promoted;
# EPI: 0 bf16 (+R, RoPE, segments), 1 SwiGLU, 2 fp32, 3 dSwiGLU
def fp8_tile(op: int, epi: int, M: int, N: int, sms: int) -> int:
    """gemm.cu fp8_bn: the promoted forms, and the rowwise SwiGLU and fp32 forms, run on the 128-wide tile."""
    wide_ok = op == 1 or (op == 3 and epi not in (1, 2))
    return pick_bn(M, N, 2 if epi == 1 else 1, sms) if wide_ok else 128


DEC_SMEM_MAX = 200 * 1024        # float8.cu kDecSmemMax
DEC_WARPS, DEC_TILE_N, DEC_MAX_MT = 8, 8, 4


def dec_pitch(K: int) -> int:
    return (K + 127) // 128 * 128 + 64


def dec_smem(K: int, mt: int, nw: int) -> int:
    return mt * 16 * dec_pitch(K) + mt * 16 * 4 + DEC_WARPS * nw * mt * 16 * DEC_TILE_N * 4


def dec_mt(M: int, K: int, epi: int) -> int:
    """16-row MMA tiles per row group of tn_gemm_fp8_decode: as many as the rows need, at most 4, fewer where shared
    memory would overflow."""
    nw = 2 if epi == 2 else 1
    mt = min(-(-M // 16), DEC_MAX_MT)
    while mt > 1 and dec_smem(K, mt, nw) > DEC_SMEM_MAX:
        mt -= 1
    return mt


def dec_max_k(epi: int) -> int:
    """Largest multiple of 16 that tn_gemm_fp8_decode accepts (16 rows of X in shared memory)."""
    nw = 2 if epi == 2 else 1
    K = 16
    while dec_smem(K + 16, 1, nw) <= DEC_SMEM_MAX:
        K += 16
    return K


# ---------------------------------------------------------------------------------------------------------------
# the cases of tests/test_gpu_fp8_exact.py
# ---------------------------------------------------------------------------------------------------------------
# (M, N, K): a single tile, partial M / N tiles, a partial 128-k stage (K = 144, 112, 3088, 8208), and two shapes
# that pick the 256-wide tile at 132 SMs with a 16-column (N = 3088) or 16-row (M = 8208) tail
PLAIN = [(16, 16, 16), (48, 272, 144), (144, 528, 112), (272, 3088, 3088), (8208, 3088, 3088), (8208, 3072, 8208)]
SWIGLU = [(272, 272, 144), (8208, 8192, 3072)]          # (M, N per half, K); the dSwiGLU GEMMs: (M, N, K)
QKV = [(272, 272, 512, 256), (8208, 3072, 3072, 1024)]  # (M, d, nq, nkv); every QKV launch needs M, N >= 256
DEC_M = [1, 15, 16, 17, 47, 48, 49, 64, 65, 200]
DEC_NK = [(16, 16), (48, 80), (3072, 768), (1024, 5120), (5120, 3072), (3072, 8192)]
WITNESS_PLAIN = (256, 256, 512)
WITNESS_QKV = (512, 512, 512, 256)                      # (M, d, nq, nkv): every launch has K >= 512


def qkv_gemms(M, d, nq, nkv):
    """(M, N, K) of the three QKV launches: forward, dgrad (K segmented), wgrad (M segmented)."""
    tot = nq + 2 * nkv
    return {0: (M, tot, d), 1: (M, d, tot), 2: (tot, d, M)}


def qkv_extra(nq, nkv):
    """`exponents` pairs for a vector over the rows of [Wq;Wk;Wv]: each segment differs from the one before."""
    return [(nq, nq), (nq + nkv, nkv)]
