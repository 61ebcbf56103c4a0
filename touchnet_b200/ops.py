"""Host-side op layer: thin, allocation-only wrappers around the C ABI (include/touchnet_b200.h) and the autograd
Functions built from them.  PyTorch is plumbing here (device memory, streams, autograd bookkeeping); every FLOP and
every byte moved on the hot path happens inside libtouchnet_b200.so.  There is no fallback: a missing library or a
non-CUDA tensor raises.

Reference call sites each op replaces are listed in include/touchnet_b200.h.
"""
from __future__ import annotations

import math
import os
from typing import Optional

import torch

from . import _lib

BF16 = torch.bfloat16


def _st() -> int:
    return torch.cuda.current_stream().cuda_stream


def _chk(t: torch.Tensor, name: str, dtype=None):
    if not t.is_cuda:
        raise _lib.TouchNetB200Error(f"{name} must be a CUDA tensor (touchnet_b200 has no CPU path)")
    if dtype is not None and t.dtype != dtype:
        raise _lib.TouchNetB200Error(f"{name} must be {dtype}, got {t.dtype}")


def _rows2d(t: torch.Tensor) -> torch.Tensor:
    """View as [rows, cols] with unit inner stride (no copy unless the input is not row-contiguous)."""
    t2 = t.reshape(-1, t.shape[-1])
    if t2.stride(-1) != 1 or (t2.shape[0] > 1 and t2.stride(0) < t2.shape[1]):
        t2 = t2.contiguous()
    return t2


def _dense_rows(t: torch.Tensor) -> torch.Tensor:
    """2-D `t` with row stride equal to its width, for the kernels that address row r at r * cols (RMSNorm, the SwiGLU
    backward, the embedding add).  Copies only when `t` is not already laid out so; `_rows2d` views with a wider row
    stride (a column slice, a gradient coming back through torch.cat) are the case this exists for."""
    if t.stride(-1) == 1 and (t.shape[0] <= 1 or t.stride(0) == t.shape[1]):
        return t
    return t.contiguous()


# ---------------------------------------------------------------------------------------------------------------
# bf16 working copies of fp32 master weights (what FSDP2's MixedPrecisionPolicy does at all-gather time,
# ref: touchnet/models/helper_func.py:163; at 1 GPU the reference stays fp32, SURVEY 9.1 - we compute in bf16 always)
# ---------------------------------------------------------------------------------------------------------------
def cast_bf16(src: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    _chk(src, "src", torch.float32)
    src = src.contiguous()
    if out is None:
        out = torch.empty(src.shape, dtype=BF16, device=src.device)
    _lib.call("tn_cast_f32_bf16", src.data_ptr(), out.data_ptr(), src.numel(), _st())
    torch.autograd.graph.increment_version(out)   # raw-pointer write: a graph that saved `out` for backward must notice
    return out


def bf16_weight(w: torch.Tensor) -> torch.Tensor:
    """bf16 working copy of a parameter: the tensor itself if already bf16 (FSDP2 mixed precision hands the modules
    bf16 unsharded parameters), else a cast of the fp32 master cached ON THE PARAMETER OBJECT (attribute `_tn_bf16` =
    (version, tensor, event, epoch), keyed by the parameter's version counter) so that it lives and dies with the parameter and
    one step casts once.  Call it with the nn.Parameter itself (module level), not from inside an autograd Function.
    If the copy was produced ahead of time on the side stream (`prefetch_bf16_weights`), the current stream is made to
    wait for it here."""
    if w.dtype == BF16:
        w = w.detach()
        return w if w.is_contiguous() else w.contiguous()
    ent = getattr(w, "_tn_bf16", None)
    ok = ent is not None and ent[1].shape == w.shape and ent[1].device == w.device
    if ok and ent[0] == w._version and ent[3] == _CACHE_EPOCH:
        if ent[2] is not None:
            torch.cuda.current_stream().wait_event(ent[2])
            w._tn_bf16 = (ent[0], ent[1], None, ent[3])
        return ent[1]
    out = cast_bf16(w.detach(), ent[1] if ok else None)
    w._tn_bf16 = (w._version, out, None, _CACHE_EPOCH)
    return out


# FSDP2 refills its unsharded fp32 parameters (param_dtype=None) under `_unsafe_preserve_version_counter`, so the version
# key alone would serve stale copies there: models that find themselves FSDP-managed bump this epoch every forward.
_CACHE_EPOCH = 0


def begin_forward(module: torch.nn.Module) -> None:
    """Called at the top of the model forwards: starts a new cache epoch when parameters are FSDP-managed (casts happen
    once per forward, like the all-gather), else issues the side-stream prefetch of stale fp32 master weights."""
    global _CACHE_EPOCH
    try:
        from torch.distributed.fsdp import FSDPModule
        managed = any(isinstance(m, FSDPModule) for m in module.modules())
    except ImportError:
        managed = False
    if managed:
        _CACHE_EPOCH += 1
    else:
        prefetch_bf16_weights(module)


def invalidate_bf16_cache(module: torch.nn.Module) -> None:
    """Force a fresh fp32->bf16 cast on next use (bench.py calls this every step: the cast is part of the step, as the
    all-gather-time cast is under FSDP2).  The buffers are kept and overwritten."""
    for p in module.parameters():
        ent = getattr(p, "_tn_bf16", None)
        if ent is not None:
            p._tn_bf16 = (-1, ent[1], None, _CACHE_EPOCH)


_CAST_STREAM: dict = {}


def _is_dtensor(t) -> bool:
    try:
        from torch.distributed.tensor import DTensor
    except Exception:       # torch built without distributed
        return False
    return isinstance(t, DTensor)


def prefetch_bf16_weights(module: torch.nn.Module) -> int:
    """Issue the fp32->bf16 casts of every stale >=2-D fp32 parameter of `module` on a side stream, in parameter order,
    so that these HBM-bound copies overlap the tensor-bound GEMMs of the layers in front of them (the same idea as
    FSDP2's all-gather prefetch).  Consumers synchronise per parameter through an event (see bf16_weight).
    Returns the number of casts issued."""
    params, seen = [], set()
    for m in module.modules():          # nn.Linear weights are the only tensors consumed through bf16_weight()
        w = getattr(m, "weight", None) if isinstance(m, torch.nn.Linear) else None
        if w is None or w.dtype != torch.float32 or not w.is_cuda or id(w) in seen:
            continue
        if _is_dtensor(w) or w.untyped_storage().size() == 0:
            continue                    # FSDP2/TP-managed: the all-gather delivers bf16 (MixedPrecisionPolicy), nothing to cast
        seen.add(id(w))
        params.append(w)
    todo = []
    for p in params:
        ent = getattr(p, "_tn_bf16", None)
        ok = ent is not None and ent[1].shape == p.shape and ent[1].device == p.device
        if not (ok and ent[0] == p._version and ent[3] == _CACHE_EPOCH):
            todo.append((p, ent[1] if ok else None))
    if not todo:
        return 0
    dev = todo[0][0].device
    side = _CAST_STREAM.get(dev)
    if side is None:
        side = _CAST_STREAM[dev] = torch.cuda.Stream(device=dev)
    cur = torch.cuda.current_stream(dev)
    side.wait_stream(cur)          # everything that still reads the old copies (or writes the masters) is ahead of us
    with torch.cuda.stream(side):
        for p, buf in todo:
            out = cast_bf16(p.detach(), buf)
            out.record_stream(cur)
            ev = torch.cuda.Event()
            ev.record(side)
            p._tn_bf16 = (p._version, out, ev, _CACHE_EPOCH)
    return len(todo)


# ---------------------------------------------------------------------------------------------------------------
# raw ops (no autograd)
# ---------------------------------------------------------------------------------------------------------------
def gemm(a: torch.Tensor, b: torch.Tensor, *, a_mn: bool = False, b_mn: bool = False, out_f32: bool = False,
         residual: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None, M=None, N=None, K=None):
    """D[M,N] = op(A)·op(B) (+R).  a: [M,K] (a_mn=False) or [K,M] (a_mn=True); b: [N,K] or [K,N] (b_mn=True)."""
    _chk(a, "a", BF16); _chk(b, "b", BF16)
    assert a.dim() == 2 and b.dim() == 2 and a.stride(1) == 1 and b.stride(1) == 1
    if M is None:
        M, K = (a.shape[1], a.shape[0]) if a_mn else (a.shape[0], a.shape[1])
        N, Kb = (b.shape[1], b.shape[0]) if b_mn else (b.shape[0], b.shape[1])
        assert K == Kb, (a.shape, b.shape, a_mn, b_mn)
    dt = torch.float32 if out_f32 else BF16
    if out is None:
        out = torch.empty((M, N), dtype=dt, device=a.device)
    assert out.dtype == dt and out.stride(1) == 1
    if residual is not None:
        assert residual.dtype == dt and residual.stride(-1) == 1
        residual = residual.reshape(M, N) if residual.dim() != 2 else residual
    _lib.call("tn_gemm_bf16", a.data_ptr(), a.stride(0), int(a_mn), b.data_ptr(), b.stride(0), int(b_mn),
              out.data_ptr(), out.stride(0), int(out_f32), None if residual is None else residual.data_ptr(),
              0 if residual is None else residual.stride(0), M, N, K, _st())
    return out


def gemm_swiglu(x: torch.Tensor, wg: torch.Tensor, wu: torch.Tensor, need_gu: bool = True):
    """G = x·Wgᵀ, U = x·Wuᵀ, H = silu(G)⊙U in one wgmma kernel (SwiGLU in the epilogue)."""
    _chk(x, "x", BF16); _chk(wg, "wg", BF16); _chk(wu, "wu", BF16)
    M, K = x.shape
    N = wg.shape[0]
    assert wg.shape == wu.shape == (N, K) and wg.stride(0) == wu.stride(0)
    h = torch.empty((M, N), dtype=BF16, device=x.device)
    g = torch.empty_like(h) if need_gu else None
    u = torch.empty_like(h) if need_gu else None
    _lib.call("tn_gemm_swiglu_bf16", x.data_ptr(), x.stride(0), wg.data_ptr(), wu.data_ptr(), wg.stride(0),
              None if g is None else g.data_ptr(), None if u is None else u.data_ptr(), h.data_ptr(), N, M, N, K, _st())
    return g, u, h


_FUSE_QKV = os.environ.get("TN_FUSED_QKV", "1") != "0"   # A/B switch for measurements


def qkv_fusable(M: int, nq: int, nkv: int) -> bool:
    """The three projections run as one GEMM launch when every segment is a whole number of 256-wide tiles."""
    return _FUSE_QKV and M >= 256 and nq % 256 == 0 and nkv % 256 == 0


def gemm_qkv_fwd(x, wq, wk, wv, rope=None):
    """qkv[M, nq+2nkv] = x·[Wq;Wk;Wv]ᵀ in one launch (weights stay separate tensors).  rope = (cos, sin) tables
    [M, 64]: RoPE is applied to the q and k columns in the GEMM epilogue."""
    M, K = x.shape
    nq, nkv = wq.shape[0], wk.shape[0]
    out = torch.empty((M, nq + 2 * nkv), dtype=BF16, device=x.device)
    _lib.call("tn_gemm_qkv_bf16", 0, x.data_ptr(), x.stride(0), wq.data_ptr(), wk.data_ptr(), wv.data_ptr(), wq.stride(0),
              out.data_ptr(), None, None, out.stride(0), 0, nq, nkv, nkv, M, nq + 2 * nkv, K,
              None if rope is None else rope[0].data_ptr(), None if rope is None else rope[1].data_ptr(), _st())
    return out


def gemm_qkv_dgrad(dqkv, wq, wk, wv):
    """dx[M, d] = dq·Wq + dk·Wk + dv·Wv with dq|dk|dv side by side in `dqkv`."""
    M, Kt = dqkv.shape
    d = wq.shape[1]
    out = torch.empty((M, d), dtype=BF16, device=dqkv.device)
    _lib.call("tn_gemm_qkv_bf16", 1, dqkv.data_ptr(), dqkv.stride(0), wq.data_ptr(), wk.data_ptr(), wv.data_ptr(),
              wq.stride(0), out.data_ptr(), None, None, out.stride(0), 0, wq.shape[0], wk.shape[0], wv.shape[0], M, d, Kt,
              None, None, _st())
    return out


def gemm_qkv_wgrad(dqkv, x, f32: bool, nq: int | None = None, nkv: int | None = None):
    """(dWq, dWk, dWv) = (dqᵀ·x, dkᵀ·x, dvᵀ·x) in one launch; fp32 outputs for fp32 master weights, else bf16.
    Segment sizes default to the GQA split implied by the buffer width (nq + 2*nkv) when nq is given."""
    Mred, Mt = dqkv.shape
    d = x.shape[1]
    if nq is None:
        raise _lib.TouchNetB200Error("gemm_qkv_wgrad needs the q segment width")
    nkv = (Mt - nq) // 2 if nkv is None else nkv
    dt = torch.float32 if f32 else BF16
    outs = [torch.empty((n, d), dtype=dt, device=x.device) for n in (nq, nkv, nkv)]
    _lib.call("tn_gemm_qkv_bf16", 2, dqkv.data_ptr(), dqkv.stride(0), x.data_ptr(), None, None, x.stride(0),
              outs[0].data_ptr(), outs[1].data_ptr(), outs[2].data_ptr(), d, int(f32), nq, nkv, nkv, Mt, d, Mred, None,
              None, _st())
    return outs


# The fused launch's epilogue (strided G/U loads, 2 exp per element, two stores) is not hidden behind the mainloop, so the
# default is the two-kernel path (plain dgrad + SwiGLU-backward pass); the fused form is bit-identical and tested, behind
# TN_FUSED_DSWIGLU=1.
_FUSE_DSWIGLU = os.environ.get("TN_FUSED_DSWIGLU", "0") != "0"


def gemm_dswiglu(dy: torch.Tensor, wd: torch.Tensor, g: torch.Tensor, u: torch.Tensor):
    """(dG, dU) of hm = silu(g)*u given dy = d(hm . Wd^T): the down-proj dgrad GEMM dH = dy . Wd with the SwiGLU backward
    in its epilogue (dH never written).  Takes the two-kernel path below M, N = 256 or without TN_FUSED_DSWIGLU=1."""
    M, K = dy.shape
    N = wd.shape[1]
    if not (_FUSE_DSWIGLU and M >= 256 and N >= 256 and N % 8 == 0 and g.stride(0) == u.stride(0)):
        return swiglu_bwd(g, u, gemm(dy, wd, b_mn=True))
    dg = torch.empty_like(g)
    du = torch.empty_like(u)
    assert dg.stride(0) == du.stride(0)
    _lib.call("tn_gemm_dswiglu_bf16", dy.data_ptr(), dy.stride(0), wd.data_ptr(), wd.stride(0), g.data_ptr(), u.data_ptr(),
              g.stride(0), dg.data_ptr(), du.data_ptr(), dg.stride(0), M, N, K, _st())
    return dg, du


# ---------------------------------------------------------------------------------------------------------------
# FP8 (torchao's tensorwise recipe): dynamic per-tensor scales that never leave the device, K-major 8-bit operands
# ---------------------------------------------------------------------------------------------------------------
F8E4M3, F8E5M2 = torch.float8_e4m3fn, torch.float8_e5m2


def fp8_amax(x: torch.Tensor, amax: torch.Tensor) -> None:
    """amax = max(amax, max|x|) over a bf16 [rows, cols] view; `amax` is a device float the caller zeroed."""
    _chk(x, "x", BF16)
    _lib.call("tn_fp8_amax_bf16", x.data_ptr(), x.stride(0), x.shape[0], x.shape[1], amax.data_ptr(), _st())


def fp8_cast(x: torch.Tensor, amax: torch.Tensor, e5m2: bool, row: bool = True, t: bool = True, inv=None, out=None,
             out_t=None):
    """sat_rne(x · s) with s = fmax / max(amax, 1e-12): the row-major copy [rows, cols] (row=True) and / or the
    transposed copy [cols, rows] (t=True), e5m2 or e4m3, from one read of bf16 x; 1/s goes to `inv` if given.
    Returns (row-major or None, transposed or None)."""
    _chk(x, "x", BF16)
    rows, cols = x.shape
    dt = F8E5M2 if e5m2 else F8E4M3
    if row and out is None:
        out = torch.empty((rows, cols), dtype=dt, device=x.device)
    if t and out_t is None:
        out_t = torch.empty((cols, rows), dtype=dt, device=x.device)
    _lib.call("tn_fp8_cast_bf16", x.data_ptr(), x.stride(0), rows, cols, int(e5m2), amax.data_ptr(), _lib.ptr(out),
              0 if out is None else out.stride(0), _lib.ptr(out_t), 0 if out_t is None else out_t.stride(0),
              _lib.ptr(inv), _st())
    return out, out_t


def _fp8_operands(a: torch.Tensor, b: torch.Tensor) -> int:
    """Checks the operand types of an FP8 GEMM; returns 1 if A is e5m2 (a gradient: promoted accumulation)."""
    if b.dtype != F8E4M3:
        raise _lib.TouchNetB200Error(f"the B operand of an FP8 GEMM must be float8_e4m3fn, got {b.dtype} (e5m2 B is not supported)")
    if a.dtype not in (F8E4M3, F8E5M2):
        raise _lib.TouchNetB200Error(f"the A operand of an FP8 GEMM must be float8_e4m3fn or float8_e5m2, got {a.dtype}")
    _chk(a, "a"); _chk(b, "b")
    assert a.dim() == 2 and b.dim() == 2 and a.stride(1) == 1 and b.stride(1) == 1
    return int(a.dtype == F8E5M2)


def gemm_fp8(a, b, inv_a, inv_b, *, out_f32: bool = False, residual=None, out=None):
    """D[M,N] = a[M,K]·b[N,K]ᵀ · inv_a · inv_b (+R): both operands K-major 8-bit, inv_* device floats (1/s)."""
    a_e5m2 = _fp8_operands(a, b)
    (M, K), N = a.shape, b.shape[0]
    assert b.shape[1] == K, (a.shape, b.shape)
    dt = torch.float32 if out_f32 else BF16
    if out is None:
        out = torch.empty((M, N), dtype=dt, device=a.device)
    _lib.call("tn_gemm_fp8", a.data_ptr(), a.stride(0), a_e5m2, b.data_ptr(), b.stride(0), out.data_ptr(), out.stride(0),
              int(out_f32), _lib.ptr(residual), 0 if residual is None else residual.stride(0), M, N, K, inv_a.data_ptr(),
              inv_b.data_ptr(), _st())
    return out


def gemm_swiglu_fp8(x, wg, wu, inv_x, inv_w, need_gu: bool = True):
    """gemm_swiglu on 8-bit x [M,K] and wg / wu [N,K] (one scale for both weights: they share a tile)."""
    x_e5m2 = _fp8_operands(x, wg)
    _fp8_operands(x, wu)
    M, K = x.shape
    N = wg.shape[0]
    assert wg.shape == wu.shape == (N, K) and wg.stride(0) == wu.stride(0)
    h = torch.empty((M, N), dtype=BF16, device=x.device)
    g = torch.empty_like(h) if need_gu else None
    u = torch.empty_like(h) if need_gu else None
    _lib.call("tn_gemm_swiglu_fp8", x.data_ptr(), x.stride(0), x_e5m2, wg.data_ptr(), wu.data_ptr(), wg.stride(0),
              _lib.ptr(g), _lib.ptr(u), h.data_ptr(), N, M, N, K, inv_x.data_ptr(), inv_w.data_ptr(), _st())
    return g, u, h


def gemm_dswiglu_fp8(dy, wd_t, g, u, inv_a, inv_b):
    """(dG, dU) from the down-proj dgrad dH = dy[M,K]·wd_t[N,K]ᵀ (wd_t: the transposed down_proj weight) with the SwiGLU
    backward in the epilogue; below M, N = 256 or without TN_FUSED_DSWIGLU=1 the plain FP8 GEMM + swiglu_bwd."""
    dy_e5m2 = _fp8_operands(dy, wd_t)
    M, K = dy.shape
    N = wd_t.shape[0]
    if not (_FUSE_DSWIGLU and M >= 256 and N >= 256 and g.stride(0) == u.stride(0)):
        return swiglu_bwd(g, u, gemm_fp8(dy, wd_t, inv_a, inv_b))
    dg = torch.empty_like(g)
    du = torch.empty_like(u)
    _lib.call("tn_gemm_dswiglu_fp8", dy.data_ptr(), dy.stride(0), dy_e5m2, wd_t.data_ptr(), wd_t.stride(0), g.data_ptr(),
              u.data_ptr(), g.stride(0), dg.data_ptr(), du.data_ptr(), dg.stride(0), M, N, K, inv_a.data_ptr(),
              inv_b.data_ptr(), _st())
    return dg, du


def gemm_qkv_fwd_fp8(x, wq, wk, wv, inv_x, inv_w, rope=None):
    """gemm_qkv_fwd on 8-bit x [M,K] and wq / wk / wv [n_i, K] (one shared weight scale)."""
    a_e5m2 = _fp8_operands(x, wq)
    M, K = x.shape
    nq, nkv = wq.shape[0], wk.shape[0]
    out = torch.empty((M, nq + 2 * nkv), dtype=BF16, device=x.device)
    _lib.call("tn_gemm_qkv_fp8", 0, x.data_ptr(), x.stride(0), a_e5m2, wq.data_ptr(), wk.data_ptr(), wv.data_ptr(),
              wq.stride(0), out.data_ptr(), None, None, out.stride(0), 0, nq, nkv, nkv, M, nq + 2 * nkv, K,
              None if rope is None else rope[0].data_ptr(), None if rope is None else rope[1].data_ptr(),
              inv_x.data_ptr(), inv_w.data_ptr(), _st())
    return out


def gemm_qkv_dgrad_fp8(dqkv, w_t, nq: int, nkv: int, inv_a, inv_b):
    """dx[M, d] = dqkv[M, nq+2nkv]·w_t[d, nq+2nkv]ᵀ, w_t = [Wq;Wk;Wv]ᵀ, as the K-segmented launch."""
    a_e5m2 = _fp8_operands(dqkv, w_t)
    M, Kt = dqkv.shape
    d = w_t.shape[0]
    out = torch.empty((M, d), dtype=BF16, device=dqkv.device)
    _lib.call("tn_gemm_qkv_fp8", 1, dqkv.data_ptr(), dqkv.stride(0), a_e5m2, w_t.data_ptr(), w_t[:, nq:].data_ptr(),
              w_t[:, nq + nkv:].data_ptr(), w_t.stride(0), out.data_ptr(), None, None, out.stride(0), 0, nq, nkv, nkv,
              M, d, Kt, None, None, inv_a.data_ptr(), inv_b.data_ptr(), _st())
    return out


def gemm_qkv_wgrad_fp8(dqkv_t, x_t, f32: bool, nq: int, nkv: int, inv_a, inv_b):
    """(dWq, dWk, dWv) = row blocks of dqkv_t[nq+2nkv, M]·x_t[d, M]ᵀ in one launch (fp32 for fp32 master weights)."""
    a_e5m2 = _fp8_operands(dqkv_t, x_t)
    Mt, Mred = dqkv_t.shape
    d = x_t.shape[0]
    dt = torch.float32 if f32 else BF16
    outs = [torch.empty((n, d), dtype=dt, device=x_t.device) for n in (nq, nkv, nkv)]
    _lib.call("tn_gemm_qkv_fp8", 2, dqkv_t.data_ptr(), dqkv_t.stride(0), a_e5m2, x_t.data_ptr(), None, None,
              x_t.stride(0), outs[0].data_ptr(), outs[1].data_ptr(), outs[2].data_ptr(), d, int(f32), nq, nkv, nkv, Mt, d,
              Mred, None, None, inv_a.data_ptr(), inv_b.data_ptr(), _st())
    return outs


# Rowwise recipe (torchao's "rowwise"): every operand e4m3 with one power-of-two scale per row along the GEMM's reduction
# axis; the 1/s vectors stay on the device.
def _fp8_axis_input(x: torch.Tensor) -> None:
    """A bf16 [rows, cols] view with unit inner stride.  These checks come before the device checks of the callers."""
    if x.dtype != BF16 or x.dim() != 2 or x.stride(1) != 1:
        raise _lib.TouchNetB200Error(f"x must be a 2-D bfloat16 view with unit inner stride, got {x.dtype} "
                                     f"{tuple(x.shape)} strides {tuple(x.stride())}")


def _fp8_vec(v: torch.Tensor, n: int, name: str) -> None:
    """A contiguous float32 vector of n entries (amaxes or 1/s)."""
    if v.dtype != torch.float32 or v.dim() != 1 or v.numel() != n or not v.is_contiguous():
        raise _lib.TouchNetB200Error(f"{name} must be a contiguous float32 vector of {n}, got {v.dtype} "
                                     f"{tuple(v.shape)}")


def _fp8_copy(t: torch.Tensor, shape, name: str) -> None:
    """An e4m3 output [rows, cols] (a column block of a wider buffer is fine) with unit inner stride."""
    if t.dtype != F8E4M3 or tuple(t.shape) != tuple(shape) or t.stride(1) != 1:
        raise _lib.TouchNetB200Error(f"{name} must be float8_e4m3fn {tuple(shape)} with unit inner stride, got "
                                     f"{t.dtype} {tuple(t.shape)}")


def fp8_rowwise_cast(x: torch.Tensor, out=None, inv=None):
    """The e4m3 row-major copy of bf16 x [rows, cols], one scale per row; returns (copy, 1/s [rows])."""
    _fp8_axis_input(x)
    rows, cols = x.shape
    out = torch.empty((rows, cols), dtype=F8E4M3, device=x.device) if out is None else out
    inv = torch.empty(rows, dtype=torch.float32, device=x.device) if inv is None else inv
    _fp8_copy(out, (rows, cols), "out")
    _fp8_vec(inv, rows, "inv")
    for t, n in ((x, "x"), (out, "out"), (inv, "inv")):
        _chk(t, n)
    _lib.call("tn_fp8_rowwise_cast_bf16", x.data_ptr(), x.stride(0), rows, cols, out.data_ptr(), out.stride(0),
              inv.data_ptr(), _st())
    return out, inv


def fp8_colwise_amax(x: torch.Tensor, amax: torch.Tensor) -> None:
    """amax[c] = max(amax[c], max_r |x[r, c]|) over bf16 x [rows, cols]; `amax` [cols] is zeroed by the caller."""
    _fp8_axis_input(x)
    _fp8_vec(amax, x.shape[1], "amax")
    _chk(x, "x"); _chk(amax, "amax")
    _lib.call("tn_fp8_colwise_amax_bf16", x.data_ptr(), x.stride(0), x.shape[0], x.shape[1], amax.data_ptr(), _st())


def fp8_colwise_cast_t(x: torch.Tensor, amax: torch.Tensor, out_t=None, inv=None):
    """The e4m3 transposed copy [cols, rows] of bf16 x, one scale per column of x from `amax` [cols]; returns
    (copy, 1/s [cols])."""
    _fp8_axis_input(x)
    rows, cols = x.shape
    _fp8_vec(amax, cols, "amax")
    out_t = torch.empty((cols, rows), dtype=F8E4M3, device=x.device) if out_t is None else out_t
    inv = torch.empty(cols, dtype=torch.float32, device=x.device) if inv is None else inv
    _fp8_copy(out_t, (cols, rows), "out_t")
    _fp8_vec(inv, cols, "inv")
    for t, n in ((x, "x"), (amax, "amax"), (out_t, "out_t"), (inv, "inv")):
        _chk(t, n)
    _lib.call("tn_fp8_colwise_cast_t_bf16", x.data_ptr(), x.stride(0), rows, cols, amax.data_ptr(), out_t.data_ptr(),
              out_t.stride(0), inv.data_ptr(), _st())
    return out_t, inv


def _fp8_rowwise_operands(a: torch.Tensor, b: torch.Tensor) -> None:
    if a.dtype != F8E4M3 or b.dtype != F8E4M3:
        raise _lib.TouchNetB200Error(f"both operands of a rowwise FP8 GEMM are float8_e4m3fn, got {a.dtype} and {b.dtype}")
    _chk(a, "a"); _chk(b, "b")
    assert a.dim() == 2 and b.dim() == 2 and a.stride(1) == 1 and b.stride(1) == 1


def gemm_fp8_rowwise(a, b, inv_a, inv_b, *, promoted: bool, out_f32: bool = False, residual=None, out=None):
    """D[M,N] = a[M,K]·b[N,K]ᵀ · inv_a[m] · inv_b[n] (+R): e4m3 operands, 1/s vectors over the rows of a and b.
    `promoted`: per-stage partial sums in a separate fp32 accumulator (dgrad, wgrad)."""
    _fp8_rowwise_operands(a, b)
    (M, K), N = a.shape, b.shape[0]
    assert b.shape[1] == K and inv_a.numel() == M and inv_b.numel() == N, (a.shape, b.shape)
    dt = torch.float32 if out_f32 else BF16
    if out is None:
        out = torch.empty((M, N), dtype=dt, device=a.device)
    _lib.call("tn_gemm_fp8_rowwise", a.data_ptr(), a.stride(0), b.data_ptr(), b.stride(0), out.data_ptr(), out.stride(0),
              int(out_f32), _lib.ptr(residual), 0 if residual is None else residual.stride(0), M, N, K, inv_a.data_ptr(),
              inv_b.data_ptr(), int(promoted), _st())
    return out


def gemm_swiglu_fp8_rowwise(x, wg, wu, inv_x, inv_w, need_gu: bool = True):
    """gemm_swiglu on e4m3 x [M,K] and wg / wu [N,K]; inv_w [2N] holds the 1/s of the gate rows, then the up rows."""
    _fp8_rowwise_operands(x, wg)
    _fp8_rowwise_operands(x, wu)
    M, K = x.shape
    N = wg.shape[0]
    assert wg.shape == wu.shape == (N, K) and wg.stride(0) == wu.stride(0) and inv_w.numel() == 2 * N
    h = torch.empty((M, N), dtype=BF16, device=x.device)
    g = torch.empty_like(h) if need_gu else None
    u = torch.empty_like(h) if need_gu else None
    _lib.call("tn_gemm_swiglu_fp8_rowwise", x.data_ptr(), x.stride(0), wg.data_ptr(), wu.data_ptr(), wg.stride(0),
              _lib.ptr(g), _lib.ptr(u), h.data_ptr(), N, M, N, K, inv_x.data_ptr(), inv_w.data_ptr(), _st())
    return g, u, h


def gemm_dswiglu_fp8_rowwise(dy, wd_t, g, u, inv_a, inv_b):
    """gemm_dswiglu_fp8 with rowwise scales (promoted accumulation)."""
    _fp8_rowwise_operands(dy, wd_t)
    M, K = dy.shape
    N = wd_t.shape[0]
    if not (_FUSE_DSWIGLU and M >= 256 and N >= 256 and g.stride(0) == u.stride(0)):
        return swiglu_bwd(g, u, gemm_fp8_rowwise(dy, wd_t, inv_a, inv_b, promoted=True))
    dg = torch.empty_like(g)
    du = torch.empty_like(u)
    _lib.call("tn_gemm_dswiglu_fp8_rowwise", dy.data_ptr(), dy.stride(0), wd_t.data_ptr(), wd_t.stride(0), g.data_ptr(),
              u.data_ptr(), g.stride(0), dg.data_ptr(), du.data_ptr(), dg.stride(0), M, N, K, inv_a.data_ptr(),
              inv_b.data_ptr(), _st())
    return dg, du


def gemm_qkv_fwd_fp8_rowwise(x, wq, wk, wv, inv_x, inv_w, rope=None):
    """gemm_qkv_fwd on e4m3 x [M,K] and wq / wk / wv [n_i, K]; inv_w: the 1/s of the rows of [Wq;Wk;Wv]."""
    _fp8_rowwise_operands(x, wq)
    M, K = x.shape
    nq, nkv = wq.shape[0], wk.shape[0]
    out = torch.empty((M, nq + 2 * nkv), dtype=BF16, device=x.device)
    _lib.call("tn_gemm_qkv_fp8_rowwise", 0, x.data_ptr(), x.stride(0), wq.data_ptr(), wk.data_ptr(), wv.data_ptr(),
              wq.stride(0), out.data_ptr(), None, None, out.stride(0), 0, nq, nkv, nkv, M, nq + 2 * nkv, K,
              None if rope is None else rope[0].data_ptr(), None if rope is None else rope[1].data_ptr(),
              inv_x.data_ptr(), inv_w.data_ptr(), _st())
    return out


def gemm_qkv_dgrad_fp8_rowwise(dqkv, w_t, nq: int, nkv: int, inv_a, inv_b):
    """gemm_qkv_dgrad_fp8 with rowwise scales: inv_a over the rows of dqkv, inv_b over the rows of w_t."""
    _fp8_rowwise_operands(dqkv, w_t)
    M, Kt = dqkv.shape
    d = w_t.shape[0]
    out = torch.empty((M, d), dtype=BF16, device=dqkv.device)
    _lib.call("tn_gemm_qkv_fp8_rowwise", 1, dqkv.data_ptr(), dqkv.stride(0), w_t.data_ptr(), w_t[:, nq:].data_ptr(),
              w_t[:, nq + nkv:].data_ptr(), w_t.stride(0), out.data_ptr(), None, None, out.stride(0), 0, nq, nkv, nkv,
              M, d, Kt, None, None, inv_a.data_ptr(), inv_b.data_ptr(), _st())
    return out


def gemm_qkv_wgrad_fp8_rowwise(dqkv_t, x_t, f32: bool, nq: int, nkv: int, inv_a, inv_b):
    """gemm_qkv_wgrad_fp8 with rowwise scales: inv_a over the rows of dqkv_t, inv_b over the rows of x_t."""
    _fp8_rowwise_operands(dqkv_t, x_t)
    Mt, Mred = dqkv_t.shape
    d = x_t.shape[0]
    dt = torch.float32 if f32 else BF16
    outs = [torch.empty((n, d), dtype=dt, device=x_t.device) for n in (nq, nkv, nkv)]
    _lib.call("tn_gemm_qkv_fp8_rowwise", 2, dqkv_t.data_ptr(), dqkv_t.stride(0), x_t.data_ptr(), None, None,
              x_t.stride(0), outs[0].data_ptr(), outs[1].data_ptr(), outs[2].data_ptr(), d, int(f32), nq, nkv, nkv, Mt,
              d, Mred, None, None, inv_a.data_ptr(), inv_b.data_ptr(), _st())
    return outs


def gemm_fp8_decode(x, w8, inv_w, residual=None, swiglu: bool = False):
    """The skinny-M rowwise GEMM of cached decode steps: bf16 x [M, K] (quantised row by row inside the kernel, with
    fp8_rowwise_cast's rule) times e4m3 w8 [N, K] with 1/s inv_w [N]; returns bf16 [M, N], plus the bf16 `residual`
    [M, N] if given.  swiglu=True: w8 = [Wg; Wu] [2N, K], inv_w [2N] stacked the same way, returns H = silu(G)⊙U [M, N].
    Each output row depends on its row of x only.  Any M; N and K multiples of 16."""
    _fp8_axis_input(x)
    if w8.dtype != F8E4M3 or w8.dim() != 2 or w8.stride(1) != 1:
        raise _lib.TouchNetB200Error(f"w8 must be a 2-D float8_e4m3fn view with unit inner stride, got {w8.dtype} "
                                     f"{tuple(w8.shape)}")
    (M, K), rows = x.shape, w8.shape[0]
    if w8.shape[1] != K:
        raise _lib.TouchNetB200Error(f"x {tuple(x.shape)} and w8 {tuple(w8.shape)} differ in K")
    if swiglu and (residual is not None or rows % 2):
        raise _lib.TouchNetB200Error("swiglu takes the stacked [Wg; Wu] (an even row count) and no residual")
    N = rows // 2 if swiglu else rows
    _fp8_vec(inv_w, rows, "inv_w")
    if M < 1 or N % 16 or K % 16 or N == 0 or K == 0:
        raise _lib.TouchNetB200Error(f"gemm_fp8_decode: N={N} and K={K} must be positive multiples of 16, M={M} >= 1")
    out = torch.empty((M, N), dtype=BF16, device=x.device)
    if residual is not None:
        if residual.dtype != BF16 or tuple(residual.shape) != (M, N) or residual.stride(1) != 1:
            raise _lib.TouchNetB200Error(f"residual must be bfloat16 {(M, N)} with unit inner stride, got "
                                         f"{residual.dtype} {tuple(residual.shape)}")
        _chk(residual, "residual")
    for t, n in ((x, "x"), (w8, "w8"), (inv_w, "inv_w")):
        _chk(t, n)
    _lib.call("tn_gemm_fp8_decode", x.data_ptr(), x.stride(0), w8.data_ptr(), w8.stride(0), inv_w.data_ptr(),
              2 if swiglu else int(residual is not None), _lib.ptr(residual),
              0 if residual is None else residual.stride(0), out.data_ptr(), out.stride(0), M, N, K, _st())
    return out


def _fp8_quant(xs, st, slot: int, e5m2: bool, row: bool = True, t: bool = True):
    """Quantise the bf16 tensors `xs` with one dynamic scale, the amax over all of them, kept in row `slot` of the
    device scale table st [n, 2] = (amax, 1/s).  Returns [(row-major, transposed)] per tensor."""
    amax = st[slot, 0]
    for x in xs:
        fp8_amax(x, amax)
    return [fp8_cast(x, amax, e5m2, row, t, inv=st[slot, 1]) for x in xs]


def _fp8_dims(*dims, key: str = "float8_training"):
    """Every GEMM dimension of the FP8 block (and the row count) is a multiple of 16: 16-byte 8-bit TMA rows."""
    bad = [int(v) for v in dims if int(v) % 16]
    if bad:
        raise _lib.TouchNetB200Error(f"{key}: GEMM dimensions must be multiples of 16, got {bad}")


# forward scale-table rows of the FP8 block: (amax, 1/s) of each GEMM input
_F8_H1, _F8_WQKV, _F8_O, _F8_WO, _F8_H2, _F8_WGU, _F8_HM, _F8_WD = range(8)
# backward rows: the incoming gradients
_F8_D2, _F8_DG, _F8_DU, _F8_DX1, _F8_DQKV = range(5)


def swiglu_bwd(g, u, dh, dg_out=None, du_out=None):
    """(dG, dU) of hm = silu(g)*u.  The kernel reads and writes all five [M, N] tensors with one row stride, N."""
    M, N = g.shape
    g, u, dh = _dense_rows(g), _dense_rows(u), _dense_rows(dh)
    dg = torch.empty((M, N), dtype=BF16, device=g.device) if dg_out is None else dg_out
    du = torch.empty((M, N), dtype=BF16, device=g.device) if du_out is None else du_out
    for t, name in ((dg, "dg_out"), (du, "du_out")):
        if t.shape != (M, N) or t.stride(-1) != 1 or (M > 1 and t.stride(0) != N):
            raise _lib.TouchNetB200Error(f"swiglu_bwd: {name} must be [{M}, {N}] with row stride {N}")
    _lib.call("tn_swiglu_bwd_bf16", g.data_ptr(), u.data_ptr(), dh.data_ptr(), dg.data_ptr(), du.data_ptr(), M, N,
              N, _st())
    return dg, du


def rmsnorm_fwd(x: torch.Tensor, w: torch.Tensor, eps: float, residual: Optional[torch.Tensor] = None):
    """Returns (y, s, rstd): s = x (+ residual) is the tensor that was normalised."""
    _chk(x, "x", BF16)
    rows, d = x.shape
    x = _dense_rows(x)
    if residual is not None:
        residual = _dense_rows(residual)
    y = torch.empty_like(x)
    rstd = torch.empty(rows, dtype=torch.float32, device=x.device)
    s = torch.empty_like(x) if residual is not None else x
    w = w.detach()
    _lib.call("tn_rmsnorm_fwd_bf16", x.data_ptr(), None if residual is None else residual.data_ptr(), w.data_ptr(),
              int(w.dtype == torch.float32), s.data_ptr() if residual is not None else None, y.data_ptr(),
              rstd.data_ptr(), rows, d, float(eps), _st())
    return y, s, rstd


_norm_partials = None


def rmsnorm_bwd(s: torch.Tensor, dy: torch.Tensor, w: torch.Tensor, rstd: torch.Tensor,
                ds_extra: Optional[torch.Tensor] = None):
    """Returns (ds, dw) with ds = d/ds RMSNorm (+ ds_extra: the gradient arriving through the residual branch)."""
    global _norm_partials
    if _norm_partials is None:
        _norm_partials = _lib.load().tn_rmsnorm_bwd_num_partials()
    rows, d = s.shape
    s, dy = _dense_rows(s), _dense_rows(dy)
    if ds_extra is not None:
        ds_extra = _dense_rows(ds_extra)
    ds = torch.empty_like(s)
    part = torch.empty((_norm_partials, d), dtype=torch.float32, device=s.device)
    dw = torch.empty(d, dtype=torch.float32, device=s.device)
    w = w.detach()
    _lib.call("tn_rmsnorm_bwd_bf16", s.data_ptr(), dy.data_ptr(), None if ds_extra is None else ds_extra.data_ptr(),
              w.data_ptr(), int(w.dtype == torch.float32), rstd.data_ptr(), ds.data_ptr(), part.data_ptr(),
              _norm_partials, dw.data_ptr(), rows, d, _st())
    return ds, dw


def rope_table(position_ids: torch.Tensor, inv_freq: torch.Tensor, scaling: float = 1.0):
    """cos/sin tables [B*T, hd/2] bf16 for per-document positions."""
    _chk(position_ids, "position_ids", torch.int64)
    pos = position_ids.reshape(-1).contiguous()
    inv = inv_freq.detach().to(device=pos.device, dtype=torch.float32).contiguous()
    rows, half = pos.numel(), inv.numel()
    cos = torch.empty((rows, half), dtype=BF16, device=pos.device)
    sin = torch.empty_like(cos)
    _lib.call("tn_rope_table", pos.data_ptr(), inv.data_ptr(), float(scaling), cos.data_ptr(), sin.data_ptr(), rows, half, _st())
    return cos, sin


def rope_apply_(x: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor, n_heads: int, head_dim: int, inverse: bool = False):
    """In-place RoPE on x [rows, n_heads*head_dim] (row stride arbitrary)."""
    _chk(x, "x", BF16)
    rows = x.shape[0]
    assert x.stride(1) == 1 and cos.shape == (rows, head_dim // 2)
    _lib.call("tn_rope_apply_bf16", x.data_ptr(), x.stride(0), cos.data_ptr(), sin.data_ptr(), rows, n_heads, head_dim,
              int(inverse), _st())
    return x


class AttnPlan:
    """Per-step packing metadata shared by every layer: int32 document ids + per-block kv/q ranges, built on device."""

    def __init__(self, doc_ids: torch.Tensor, Tq: Optional[int] = None, q_blk_off: int = 0):
        """doc_ids: GLOBAL [B,T] document ids.  Tq / q_blk_off: context-parallel query window (rows
        [q_blk_off*128, q_blk_off*128 + Tq) of the sequence live on this rank); default = the whole sequence."""
        _chk(doc_ids, "attention_mask (document ids)")
        assert doc_ids.dim() == 2
        self.B, self.T = doc_ids.shape
        self.Tq = self.T if Tq is None else int(Tq)
        self.q_blk_off = int(q_blk_off)
        self.cp_group = None
        self.tp = None            # tensor_parallel.TPContext when the block runs tensor + sequence parallel
        self.doc = doc_ids.to(torch.int32).contiguous()
        n_ints = int(_lib.load().tn_attn_meta_ints(self.B, self.T))
        self.meta = torch.empty(n_ints, dtype=torch.int32, device=doc_ids.device)
        _lib.call("tn_attn_prep", self.doc.data_ptr(), self.meta.data_ptr(), self.B, self.T, _st())


def attn_fwd(q, k, v, plan: AttnPlan, H: int, KV: int, scale: float):
    """q [B*Tq, H*128], k/v [B*T, KV*128] (row strides arbitrary) -> o [B*Tq, H*128], lse [B,H,Tq].
    Tq == T unless the plan describes a context-parallel query window (plan.Tq, plan.q_blk_off)."""
    B, T = plan.B, plan.T
    Tq = plan.Tq
    o = torch.empty((B * Tq, H * 128), dtype=BF16, device=q.device)
    lse = torch.empty((B, H, Tq), dtype=torch.float32, device=q.device)
    _lib.call("tn_attn_fwd_bf16", q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0), v.data_ptr(), v.stride(0),
              o.data_ptr(), o.stride(0), lse.data_ptr(), plan.doc.data_ptr(), plan.meta.data_ptr(), B, T, H, KV,
              float(scale), Tq, plan.q_blk_off, _st())
    return o, lse


def attn_bwd(q, k, v, o, do, lse, plan: AttnPlan, H: int, KV: int, scale: float, out=None, rope=None):
    """`out` = (dq, dk, dv) preallocated (possibly strided views of one [B*T, (H+2KV)*128] buffer).
    `rope` = (cos, sin) tables: the kernels' epilogues apply the inverse rotation, i.e. dq/dk come back w.r.t. the
    un-rotated projections (only without context parallelism, where dK rows and table rows coincide)."""
    B, T = plan.B, plan.T
    Tq = plan.Tq
    if out is None:
        dq = torch.empty((B * Tq, H * 128), dtype=BF16, device=q.device)
        dk = torch.empty((B * T, KV * 128), dtype=BF16, device=q.device)
        dv = torch.empty_like(dk)
    else:
        dq, dk, dv = out
    delta = torch.empty((B, H, Tq), dtype=torch.float32, device=q.device)
    if do.stride(1) != 1:
        do = do.contiguous()
    _lib.call("tn_attn_bwd_bf16", q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0), v.data_ptr(), v.stride(0),
              o.data_ptr(), o.stride(0), do.data_ptr(), do.stride(0), lse.data_ptr(), delta.data_ptr(),
              dq.data_ptr(), dq.stride(0), dk.data_ptr(), dk.stride(0), dv.data_ptr(), dv.stride(0),
              plan.doc.data_ptr(), plan.meta.data_ptr(), B, T, H, KV, float(scale), Tq, plan.q_blk_off,
              None if rope is None else rope[0].data_ptr(), None if rope is None else rope[1].data_ptr(),
              None if rope is None else rope[0].data_ptr(), None if rope is None else rope[1].data_ptr(), _st())
    return dq, dk, dv


def attn_decode(q, k_cache, v_cache, kv_start, kv_end, H: int, KV: int, scale: float, workspace=None, lse: bool = False):
    """Split-KV attention of one query row per batch row: q [B, H*128] (rotated) against cache rows [kv_start[b],
    kv_end[b]) of k_cache / v_cache [B, S_cap, KV*128] (token and batch strides shared by both) -> o [B, H*128]
    (and lse [B, H] if asked)."""
    _chk(q, "q", BF16); _chk(k_cache, "k_cache", BF16); _chk(v_cache, "v_cache", BF16)
    B, S_cap = k_cache.shape[0], k_cache.shape[1]
    assert k_cache.stride() == v_cache.stride() and k_cache.stride(2) == 1 and q.stride(1) == 1
    if workspace is None:
        workspace = torch.empty(int(_lib.load().tn_attn_decode_ws_floats(B, H, KV, S_cap)), dtype=torch.float32,
                                device=q.device)
    o = torch.empty((B, H * 128), dtype=BF16, device=q.device)
    lse_t = torch.empty((B, H), dtype=torch.float32, device=q.device) if lse else None
    _lib.call("tn_attn_decode_bf16", q.data_ptr(), q.stride(0), k_cache.data_ptr(), v_cache.data_ptr(),
              k_cache.stride(1), k_cache.stride(0), kv_start.data_ptr(), kv_end.data_ptr(), B, H, KV, S_cap, float(scale),
              workspace.data_ptr(), o.data_ptr(), o.stride(0), None if lse_t is None else lse_t.data_ptr(), _st())
    return (o, lse_t) if lse else o


def attn_decode_multi(q, k_cache, v_cache, kv_start, kv_end, Tq: int, H: int, KV: int, scale: float, workspace=None,
                      lse: bool = False):
    """attn_decode for Tq new rows per batch row: q [B*Tq, H*128], row b*Tq + j at cache position kv_end[b] - Tq + j,
    attends to cache rows [kv_start[b], kv_end[b] - Tq + j + 1) -> o [B*Tq, H*128] (and lse [B*Tq, H]); each row is
    bit-identical to attn_decode at its own length."""
    _chk(q, "q", BF16); _chk(k_cache, "k_cache", BF16); _chk(v_cache, "v_cache", BF16)
    B, S_cap = k_cache.shape[0], k_cache.shape[1]
    assert k_cache.stride() == v_cache.stride() and k_cache.stride(2) == 1 and q.stride(1) == 1
    if workspace is None:
        workspace = torch.empty(int(_lib.load().tn_attn_decode_multi_ws_floats(B, Tq, H, KV, S_cap)),
                                dtype=torch.float32, device=q.device)
    o = torch.empty((B * Tq, H * 128), dtype=BF16, device=q.device)
    lse_t = torch.empty((B * Tq, H), dtype=torch.float32, device=q.device) if lse else None
    _lib.call("tn_attn_decode_multi_bf16", q.data_ptr(), q.stride(0), k_cache.data_ptr(), v_cache.data_ptr(),
              k_cache.stride(1), k_cache.stride(0), kv_start.data_ptr(), kv_end.data_ptr(), B, int(Tq), H, KV, S_cap,
              float(scale), workspace.data_ptr(), o.data_ptr(), o.stride(0), None if lse_t is None else lse_t.data_ptr(),
              _st())
    return (o, lse_t) if lse else o


def _kv_copy_dims(k, v, k_cache, v_cache):
    """The checks both K/V copies make; returns the cache's (B, S_cap, width)."""
    _chk(k, "k", BF16); _chk(v, "v", BF16); _chk(k_cache, "k_cache", BF16)
    B, S_cap, width = k_cache.shape
    assert k_cache.stride() == v_cache.stride() and k.shape[1] == width and k.stride(1) == 1 and v.stride(1) == 1
    return B, S_cap, width


def kv_append(k, v, k_cache, v_cache, row_end, T_new: int):
    """Cache rows [row_end[b] - T_new, row_end[b]) of batch row b <- rows b*T_new .. of k / v [B*T_new, KV*128]."""
    B, S_cap, width = _kv_copy_dims(k, v, k_cache, v_cache)
    _chk(row_end, "row_end", torch.int32)
    _lib.call("tn_kv_append_bf16", k.data_ptr(), k.stride(0), v.data_ptr(), v.stride(0), k_cache.data_ptr(),
              v_cache.data_ptr(), k_cache.stride(1), k_cache.stride(0), row_end.data_ptr(), B, int(T_new), S_cap, width,
              _st())


def _select_dims(logits, history, length, positions, next_ids, finished):
    """The checks both selections make of the logits and the decoding state; returns the logits' (rows, V)."""
    _chk(logits, "logits", BF16); _chk(history, "history", torch.int64); _chk(length, "length", torch.int32)
    _chk(positions, "positions", torch.int64); _chk(next_ids, "next_ids", torch.int64)
    _chk(finished, "finished", torch.int32)
    assert logits.stride(1) == 1 and history.stride(1) == 1
    return logits.shape


def greedy_select(logits, history, length, positions, next_ids, finished, repetition_penalty: float,
                  no_repeat_ngram_size: int, eos: int, pad: int):
    """Greedy next token of every row (HF repetition penalty + no-repeat-ngram + argmax on fp32-cast bf16 logits [B, V]),
    written into history / next_ids; advances length and positions, updates finished (all device tensors, in place)."""
    B, V = _select_dims(logits, history, length, positions, next_ids, finished)
    assert history.shape[0] == B
    _lib.call("tn_greedy_select_bf16", logits.data_ptr(), logits.stride(0), B, V, history.data_ptr(), history.stride(0),
              length.data_ptr(), positions.data_ptr(), next_ids.data_ptr(), finished.data_ptr(),
              float(repetition_penalty), int(no_repeat_ngram_size), int(eos), int(pad), _st())


def verify_select(logits, draft, history, length, positions, next_ids, finished, limit, repetition_penalty: float,
                  no_repeat_ngram_size: int, eos: int, pad: int, picks=None):
    """Speculative verification over logits [B*(k+1), V] and the draft tokens draft [B, k]: position j's greedy pick
    over the history extended by draft[:, :j], then per row the accepted prefix plus one token (cut after eos and at
    limit) written into the decoding state.  Returns picks [B, k+1] (rows not finished)."""
    n, V = _select_dims(logits, history, length, positions, next_ids, finished)
    _chk(draft, "draft", torch.int64); _chk(limit, "limit", torch.int32)
    B, k = draft.shape
    assert n == B * (k + 1) and history.shape[0] == B and draft.is_contiguous()
    if picks is None:
        picks = torch.empty((B, k + 1), dtype=torch.int64, device=logits.device)
    _lib.call("tn_verify_select_bf16", logits.data_ptr(), logits.stride(0), B, k, V, draft.data_ptr(),
              history.data_ptr(), history.stride(0), length.data_ptr(), positions.data_ptr(), next_ids.data_ptr(),
              finished.data_ptr(), limit.data_ptr(), picks.data_ptr(), float(repetition_penalty),
              int(no_repeat_ngram_size), int(eos), int(pad), _st())
    return picks


def spec_sample_verify(logits, draft_logits, draft, history, length, positions, next_ids, finished, limit, stream_key,
                       repetition_penalty: float, no_repeat_ngram_size: int, temperature: float, top_k: int,
                       top_p: float, seed: int, eos: int, pad: int, picks=None):
    """Speculative sampling over logits [B*(k+1), V], the draft's logits draft_logits [B*k, V] and its tokens draft
    [B, k] (see tn_spec_sample_verify_bf16): each draft token is accepted with probability min(1, p/q), the first
    rejection emits a token of the residual max(0, p - q) (all accepted: one of p_k), and the emitted tokens are
    committed as verify_select commits its picks.  Returns picks [B, k+1] (x accepted, ~t emitted; rows not finished)."""
    n, V = _select_dims(logits, history, length, positions, next_ids, finished)
    _chk(draft_logits, "draft_logits", BF16); _chk(draft, "draft", torch.int64); _chk(limit, "limit", torch.int32)
    _chk(stream_key, "stream_key", torch.int64)
    B, k = draft.shape
    assert n == B * (k + 1) and tuple(draft_logits.shape) == (B * k, V) and draft_logits.stride(1) == 1
    assert history.shape[0] == B and draft.is_contiguous()
    if picks is None:
        picks = torch.empty((B, k + 1), dtype=torch.int64, device=logits.device)
    _lib.call("tn_spec_sample_verify_bf16", logits.data_ptr(), logits.stride(0), draft_logits.data_ptr(),
              draft_logits.stride(0), B, k, V, draft.data_ptr(), history.data_ptr(), history.stride(0),
              length.data_ptr(), positions.data_ptr(), next_ids.data_ptr(), finished.data_ptr(), limit.data_ptr(),
              stream_key.data_ptr(), picks.data_ptr(), float(repetition_penalty), int(no_repeat_ngram_size),
              float(temperature), int(top_k), float(top_p), int(seed), int(eos), int(pad), _st())
    return picks


def _host_i32(rows) -> torch.Tensor:
    """A small int32 table in host memory (the continuous-batching entry points copy it into the launch)."""
    return torch.tensor(rows, dtype=torch.int32).reshape(-1).contiguous()


def kv_scatter(k, v, k_cache, v_cache, docs):
    """Cache rows [0, len) of slot `slot` <- rows [src_row, src_row + len) of k / v [rows, KV*128], for each
    (src_row, slot, len, limit) in `docs` (a list; limit is not used here)."""
    B, S_cap, width = _kv_copy_dims(k, v, k_cache, v_cache)
    tab = _host_i32(docs)
    _lib.call("tn_kv_scatter_bf16", k.data_ptr(), k.stride(0), v.data_ptr(), v.stride(0), k.shape[0], k_cache.data_ptr(),
              v_cache.data_ptr(), k_cache.stride(1), k_cache.stride(0), tab.data_ptr(), len(docs), B, S_cap, width, _st())


def slot_admit(docs, ids, doc_ids, position_ids, history, kv_start, kv_end, positions, finished, limit):
    """Decoding state of the slots named in `docs` [(src_row, slot, len, limit)] from the packed prompt row (ids /
    position_ids int64, doc_ids int32, all [rows]); other slots are not touched."""
    _chk(ids, "ids", torch.int64); _chk(doc_ids, "doc_ids", torch.int32); _chk(position_ids, "position_ids", torch.int64)
    _chk(history, "history", torch.int64); _chk(kv_start, "kv_start", torch.int32); _chk(limit, "limit", torch.int32)
    assert history.stride(1) == 1
    tab = _host_i32(docs)
    _lib.call("tn_slot_admit", tab.data_ptr(), len(docs), ids.data_ptr(), doc_ids.data_ptr(), position_ids.data_ptr(),
              ids.numel(), history.data_ptr(), history.stride(0), kv_start.data_ptr(), kv_end.data_ptr(),
              positions.data_ptr(), finished.data_ptr(), limit.data_ptr(), history.shape[0], _st())


def greedy_select_slots(logits, history, length, positions, next_ids, finished, limit, repetition_penalty: float,
                        no_repeat_ngram_size: int, eos: int, pad: int, row_slot=None):
    """greedy_select over cache slots: logits row r selects for slot row_slot[r] (a list; None = slot r).  Finished or
    idle slots do not advance (pad in next_ids); a slot finishes on eos or when its length reaches limit."""
    n, V = _select_dims(logits, history, length, positions, next_ids, finished)
    _chk(limit, "limit", torch.int32)
    tab = None if row_slot is None else _host_i32(row_slot)
    _lib.call("tn_greedy_select_slots_bf16", logits.data_ptr(), logits.stride(0), n, None if tab is None else tab.data_ptr(),
              history.shape[0], V, history.data_ptr(), history.stride(0), length.data_ptr(), positions.data_ptr(),
              next_ids.data_ptr(), finished.data_ptr(), limit.data_ptr(), float(repetition_penalty),
              int(no_repeat_ngram_size), int(eos), int(pad), _st())


def sample_select_slots(logits, history, length, positions, next_ids, finished, limit, stream_key,
                        repetition_penalty: float, no_repeat_ngram_size: int, temperature: float, top_k: int,
                        top_p: float, seed: int, eos: int, pad: int, row_slot=None, row_key=None):
    """greedy_select_slots with the argmax replaced by a multinomial draw (temperature, top-k, top-p; see
    tn_sample_select_slots_bf16).  stream_key [B] int64 holds each slot's stream key; a mapped row r (row_slot given)
    draws with row_key[r] and stores it into stream_key[row_slot[r]].  The draw of a slot is a function of (seed, its
    stream key, its length, its processed logits) only."""
    n, V = _select_dims(logits, history, length, positions, next_ids, finished)
    _chk(limit, "limit", torch.int32); _chk(stream_key, "stream_key", torch.int64)
    tab = None if row_slot is None else _host_i32(row_slot)
    keys = None if row_key is None else torch.tensor(row_key, dtype=torch.int64).reshape(-1).contiguous()
    _lib.call("tn_sample_select_slots_bf16", logits.data_ptr(), logits.stride(0), n,
              None if tab is None else tab.data_ptr(), None if keys is None else keys.data_ptr(), history.shape[0], V,
              history.data_ptr(), history.stride(0), length.data_ptr(), positions.data_ptr(), next_ids.data_ptr(),
              finished.data_ptr(), limit.data_ptr(), stream_key.data_ptr(), float(repetition_penalty),
              int(no_repeat_ngram_size), float(temperature), int(top_k), float(top_p), int(seed), int(eos), int(pad),
              _st())


def embed_add(input_ids: Optional[torch.Tensor], embed: Optional[torch.Tensor], proj: Optional[torch.Tensor],
              rows: int, d: int, nan_flag: Optional[torch.Tensor] = None):
    """E = embed[input_ids] + proj (either may be None)."""
    dev = (proj if proj is not None else input_ids).device
    e = torch.empty((rows, d), dtype=BF16, device=dev)
    emb = None if embed is None else embed.detach()
    if proj is not None:
        proj = _dense_rows(proj)
    _lib.call("tn_embed_add_bf16", None if input_ids is None else input_ids.data_ptr(),
              None if emb is None else emb.data_ptr(), int(emb is not None and emb.dtype == torch.float32),
              None if proj is None else proj.data_ptr(), e.data_ptr(),
              None if nan_flag is None else nan_flag.data_ptr(), rows, d, 0 if emb is None else emb.shape[0], _st())
    return e


# ---------------------------------------------------------------------------------------------------------------
# autograd Functions
# ---------------------------------------------------------------------------------------------------------------
def _wgrad(dy2: torch.Tensor, x2: torch.Tensor, f32: bool) -> torch.Tensor:
    """dW[N,K] = dyᵀ·x, in the parameter's dtype (fp32 master -> fp32 gradient straight from the fp32 accumulator)."""
    return gemm(dy2, x2, a_mn=True, b_mn=True, out_f32=f32)


class LinearFn(torch.autograd.Function):
    """y = x·Wᵀ (+ bias) (+ residual).  F.linear at hf:modeling_llama.py:251-289,182-184;
    ref: touchnet/models/touch_audio/modeling_touch_audio.py:127 (projector).
    `w` is the parameter (gradient target, master dtype), `wb` its bf16 working copy (non-differentiable)."""

    @staticmethod
    def forward(ctx, x, w, wb, bias, residual):
        x2 = _rows2d(x)
        if x2.dtype != BF16:
            x2 = x2.to(BF16)
        r2 = None if residual is None else _rows2d(residual)
        y = gemm(x2, wb, residual=r2)
        if bias is not None:
            y += bias.to(BF16)
        ctx.save_for_backward(x2, wb)
        ctx.w_dtype = w.dtype
        ctx.has_bias = bias is not None
        ctx.has_res = residual is not None
        ctx.x_shape = x.shape
        ctx.x_dtype = x.dtype
        return y.view(*x.shape[:-1], w.shape[0])

    @staticmethod
    def backward(ctx, dy):
        x2, wb = ctx.saved_tensors
        dy2 = _rows2d(dy)
        if dy2.dtype != BF16:
            dy2 = dy2.to(BF16)
        dx = dw = db = dr = None
        if ctx.needs_input_grad[0]:
            dx = gemm(dy2, wb, b_mn=True).view(ctx.x_shape).to(ctx.x_dtype)
        if ctx.needs_input_grad[1]:
            dw = gemm(dy2, x2, a_mn=True, b_mn=True, out_f32=(ctx.w_dtype == torch.float32))
        if ctx.has_bias and ctx.needs_input_grad[3]:
            db = dy2.float().sum(0).to(ctx.w_dtype)
        if ctx.has_res and ctx.needs_input_grad[4]:
            dr = dy
        return dx, dw, None, db, dr


def linear(x, w, bias=None, residual=None):
    return LinearFn.apply(x, w, bf16_weight(w), bias, residual)


class RMSNormFn(torch.autograd.Function):
    """hf: LlamaRMSNorm.forward modeling_llama.py:62-67."""

    @staticmethod
    def forward(ctx, x, w, eps):
        x2 = _rows2d(x)
        y, _, rstd = rmsnorm_fwd(x2, w, eps)
        ctx.save_for_backward(x2, w, rstd)
        return y.view(x.shape)

    @staticmethod
    def backward(ctx, dy):
        x2, w, rstd = ctx.saved_tensors
        ds, dw = rmsnorm_bwd(x2, _rows2d(dy), w, rstd)
        return ds.view(dy.shape), dw.to(w.dtype), None


def rms_norm(x, w, eps):
    return RMSNormFn.apply(x, w, eps)


class PackedAttentionFn(torch.autograd.Function):
    """RoPE + block-causal document attention on projected q/k/v ([B*T, heads*128] GEMM outputs, rotated in place).
    hf: apply_rotary_pos_emb :151-168 + flex_attention_forward (integrations/flex_attention.py:262-364).
    q and k are OVERWRITTEN with their rotated values: hand in tensors nothing else reads (the projection outputs; an
    nn.Linear does not need its own output for backward).  The decoder block does not use this node (it fuses RoPE into
    the QKV GEMM epilogue); it is the stand-alone form for callers that keep separate projections."""

    @staticmethod
    def forward(ctx, q, k, v, cos, sin, plan, H, KV, scale):
        rope_apply_(q, cos, sin, H, 128)
        rope_apply_(k, cos, sin, KV, 128)
        o, lse = attn_fwd(q, k, v, plan, H, KV, scale)
        ctx.save_for_backward(q, k, v, o, lse, cos, sin)
        ctx.plan, ctx.H, ctx.KV, ctx.scale = plan, H, KV, scale
        return o

    @staticmethod
    def backward(ctx, do):
        q, k, v, o, lse, cos, sin = ctx.saved_tensors
        dq, dk, dv = attn_bwd(q, k, v, o, do, lse, ctx.plan, ctx.H, ctx.KV, ctx.scale, rope=(cos, sin))
        return dq, dk, dv, None, None, None, None, None, None


class AttentionFn(torch.autograd.Function):
    """Document-masked attention on already-rotated q/k (the HF attention-interface seam hands RoPE'd tensors)."""

    @staticmethod
    def forward(ctx, q, k, v, plan, H, KV, scale):
        o, lse = attn_fwd(q, k, v, plan, H, KV, scale)
        ctx.save_for_backward(q, k, v, o, lse)
        ctx.plan, ctx.H, ctx.KV, ctx.scale = plan, H, KV, scale
        return o

    @staticmethod
    def backward(ctx, do):
        q, k, v, o, lse = ctx.saved_tensors
        dq, dk, dv = attn_bwd(q, k, v, o, do, lse, ctx.plan, ctx.H, ctx.KV, ctx.scale)
        return dq, dk, dv, None, None, None, None


class SwiGLUFn(torch.autograd.Function):
    """hmid = silu(x·Wgᵀ) ⊙ (x·Wuᵀ), one kernel.  hf: LlamaMLP.forward modeling_llama.py:182-184."""

    @staticmethod
    def forward(ctx, x, wg, wu, wgb, wub):
        x2 = _rows2d(x)
        g, u, h = gemm_swiglu(x2, wgb, wub)
        ctx.save_for_backward(x2, wgb, wub, g, u)
        ctx.f32 = wg.dtype == torch.float32
        return h.view(*x.shape[:-1], wg.shape[0])

    @staticmethod
    def backward(ctx, dh):
        x2, wgb, wub, g, u = ctx.saved_tensors
        dg, du = swiglu_bwd(g, u, _rows2d(dh))
        dx = gemm(dg, wgb, b_mn=True)
        dx = gemm(du, wub, b_mn=True, residual=dx, out=dx)
        return dx.view(*dh.shape[:-1], x2.shape[1]), _wgrad(dg, x2, ctx.f32), _wgrad(du, x2, ctx.f32), None, None


def swiglu_mlp_in(x, wg, wu):
    return SwiGLUFn.apply(x, wg, wu, bf16_weight(wg), bf16_weight(wu))


def _pad_heads(x: torch.Tensor, heads: int, hd: int) -> torch.Tensor:
    """[rows, heads*hd] -> [rows, heads*128] with every head zero-padded to the 128 columns the attention kernels are built
    for: zero q/k columns add nothing to the scores, zero v columns give zero output columns - the result is exact."""
    out = torch.zeros((x.shape[0], heads, 128), dtype=x.dtype, device=x.device)
    out[:, :, :hd] = x.reshape(x.shape[0], heads, hd)
    return out.view(x.shape[0], heads * 128)


def _unpad_heads(x: torch.Tensor, heads: int, hd: int) -> torch.Tensor:
    return x.view(x.shape[0], heads, 128)[:, :, :hd].reshape(x.shape[0], heads * hd)


def block_forward(x2, ln1, wqb, wkb, wvb, bq, bk, bv, wob, ln2, wgb, wub, wdb, cos, sin, H, KV, eps, hd, attend, tp=None,
                  need_gu=True, qkv_rows=None, fp8: bool = False, fp8_recipe: str = "tensorwise"):
    """Forward of one pre-norm decoder block on rows x2 [M, d] with bf16 working weights - the body shared by training
    (DecoderLayerFn), prompt prefill and cached decoding (generation.py), which differ only in `attend(q, k, v) ->
    (o, lse, k, v)`: q/k/v arrive projected, rotated and (head_dim < 128) zero-padded to 128-wide heads.
    `qkv_rows` (default M) is the row count the QKV path (fused with the RoPE epilogue, or not) is chosen for: a
    speculative verify step passes the decode step's B so that every row is computed as the decode step computes it.
    Returns (out, saved) with saved = (rstd1, h1, q, k, v, o, lse, x1, rstd2, h2, g, u, hm) for the backward.
    fp8=True (training only, no tensor parallelism): the seven projections run as FP8 GEMMs on dynamically scaled e4m3
    copies of their inputs and weights; h1, h2 and hm in `saved` are then the transposed e4m3 copies the weight
    gradients need, and saved ends with (oᵀ in e4m3, the recipe's saved scales).  `fp8_recipe`: "tensorwise" (one
    scale per tensor, e5m2 gradients) or "rowwise" (per-row power-of-two scales, e4m3 throughout), or for cached FP8
    inference a RowwiseInference object (nothing saved for a backward)."""
    if fp8:
        return _block_forward_fp8(x2, ln1, wqb, wkb, wvb, bq, bk, bv, wob, ln2, wgb, wub, wdb, cos, sin, H, KV, eps, hd,
                                  attend, fp8_recipe)
    h1, _, rstd1 = rmsnorm_fwd(x2, ln1, eps)
    if tp is not None:
        h1 = tp.gather_rows(h1, keep=True)                               # [B*T, d]: every row, for the local heads
    nq, nkv = wqb.shape[0], wkb.shape[0]
    rows = h1.shape[0] if qkv_rows is None else qkv_rows
    rope_in_gemm = qkv_fusable(rows, nq, nkv) and bq is None and hd == 128   # RoPE in the QKV GEMM epilogue
    if qkv_fusable(rows, nq, nkv):
        qkv = gemm_qkv_fwd(h1, wqb, wkb, wvb, rope=(cos, sin) if rope_in_gemm else None)
        q, k, v = qkv[:, :nq], qkv[:, nq:nq + nkv], qkv[:, nq + nkv:]
    else:
        q = gemm(h1, wqb); k = gemm(h1, wkb); v = gemm(h1, wvb)
    if bq is not None:
        q += bq.to(BF16); k += bk.to(BF16); v += bv.to(BF16)
    if not rope_in_gemm:
        rope_apply_(q, cos, sin, H, hd)
        rope_apply_(k, cos, sin, KV, hd)
    if hd != 128:      # head_dim 64 (Llama-3.2-1B, the reference's example config) etc.: zero-padded heads, 128-wide kernels
        q, k, v = _pad_heads(q, H, hd), _pad_heads(k, KV, hd), _pad_heads(v, KV, hd)
    o, lse, k, v = attend(q, k, v)
    if tp is None:
        x1 = gemm(o if hd == 128 else _unpad_heads(o, H, hd), wob, residual=x2)
    else:                                                                # partial sums over tp -> this rank's rows
        x1 = tp.gemm_reduce_scatter(o, wob, x2)
    h2, _, rstd2 = rmsnorm_fwd(x1, ln2, eps)
    if tp is not None:
        h2 = tp.gather_rows(h2, keep=True)
    g, u, hm = gemm_swiglu(h2, wgb, wub, need_gu)
    if tp is None:
        out = gemm(hm, wdb, residual=x1)
    else:
        out = tp.gemm_reduce_scatter(hm, wdb, x1)
    return out, (rstd1, h1, q, k, v, o, lse, x1, rstd2, h2, g, u, hm)


FP8_RECIPES = ("tensorwise", "rowwise")


def check_fp8_recipe(name: str) -> str:
    """The recipe names the FP8 block accepts (the model config key `float8_recipe_name`)."""
    if name not in FP8_RECIPES:
        raise _lib.TouchNetB200Error(f"float8_recipe_name must be 'tensorwise' or 'rowwise', got {name!r}")
    return name


def _seg(inv, off: int, n: int):
    """The 1/s of rows [off, off + n) of a quantised operand: a per-tensor scale covers them all."""
    return inv if inv.dim() == 0 else inv[off:off + n]


class _Tensorwise:
    """torchao's tensorwise recipe: one dynamic scale per tensor, e4m3 activations and weights, e5m2 gradients.  The
    q/k/v weights share one scale, as do gate/up, and dq|dk|dv: the fused QKV dgrad sums over the three stacked weights
    and the SwiGLU tile holds gate and up rows, so one post-accumulation scale must cover them.  The forward's scale
    table [8, 2] = (amax, 1/s) is saved; the backward re-quantises the transposed weights at its amaxes."""

    def __init__(self, dev, dims, saved=None):
        self.fwd = torch.zeros((8, 2), dtype=torch.float32, device=dev) if saved is None else saved
        self.bwd = None if saved is None else torch.zeros((5, 2), dtype=torch.float32, device=dev)
        self.state = self.fwd

    @staticmethod
    def qkv_plan(M, nq, nkv, rope_ok):
        """(one QKV launch, RoPE in its epilogue) for M rows; rope_ok: no q/k/v bias and head_dim 128."""
        fused = qkv_fusable(M, nq, nkv)
        return fused, fused and rope_ok

    def act(self, x, slot):
        """(row-major copy, 1/s, transposed copy, 1/s) of a forward activation."""
        ((x8, x_t),) = _fp8_quant([x], self.fwd, slot, False)
        return x8, self.fwd[slot, 1], x_t, self.fwd[slot, 1]

    def grad(self, dy, slot):
        ((d8, d_t),) = _fp8_quant([dy], self.bwd, slot, True)
        return d8, self.bwd[slot, 1], d_t, self.bwd[slot, 1]

    def saved_inv(self, slot):
        return self.fwd[slot, 1]

    def weights(self, ws, slot):
        """Row-major copies of a weight group; returns (copies, 1/s of each, 1/s of the stacked group)."""
        inv = self.fwd[slot, 1]
        return [w for w, _ in _fp8_quant(ws, self.fwd, slot, False, t=False)], [inv] * len(ws), inv

    def weight_t(self, ws, slot):
        """The transposed copy [in, Σ out] of the stacked group and its 1/s."""
        if len(ws) == 1:
            return _fp8_weight_t(ws[0], self.fwd, slot), self.fwd[slot, 1]
        w_t = torch.empty((ws[0].shape[1], sum(w.shape[0] for w in ws)), dtype=F8E4M3, device=ws[0].device)
        off = 0
        for w in ws:
            _fp8_weight_t(w, self.fwd, slot, out_t=w_t[:, off:off + w.shape[0]])
            off += w.shape[0]
        return w_t, self.fwd[slot, 1]

    def qkv_grad(self, dys, slot):
        """(dq|dk|dv row-major, 1/s, transposed, 1/s) with one scale over the three."""
        M, tot, dev = dys[0].shape[0], sum(dy.shape[1] for dy in dys), dys[0].device
        d8 = torch.empty((M, tot), dtype=F8E5M2, device=dev)
        d_t = torch.empty((tot, M), dtype=F8E5M2, device=dev)
        for dy in dys:
            fp8_amax(dy, self.bwd[slot, 0])
        off = 0
        for dy in dys:
            n = dy.shape[1]
            fp8_cast(dy, self.bwd[slot, 0], True, inv=self.bwd[slot, 1], out=d8[:, off:off + n], out_t=d_t[off:off + n])
            off += n
        return d8, self.bwd[slot, 1], d_t, self.bwd[slot, 1]

    def gemm(self, a, b, inv_a, inv_b, **kw):
        return gemm_fp8(a, b, inv_a, inv_b, **kw)

    def swiglu(self, x, wg, wu, inv_x, inv_w):
        return gemm_swiglu_fp8(x, wg, wu, inv_x, inv_w)

    def dswiglu(self, dy, wd_t, g, u, inv_a, inv_b):
        return gemm_dswiglu_fp8(dy, wd_t, g, u, inv_a, inv_b)

    def qkv_fwd(self, x, wq, wk, wv, inv_x, inv_w, rope):
        return gemm_qkv_fwd_fp8(x, wq, wk, wv, inv_x, inv_w, rope=rope)

    def qkv_dgrad(self, dqkv, w_t, nq, nkv, inv_a, inv_b):
        return gemm_qkv_dgrad_fp8(dqkv, w_t, nq, nkv, inv_a, inv_b)

    def qkv_wgrad(self, dqkv_t, x_t, f32, nq, nkv, inv_a, inv_b):
        return gemm_qkv_wgrad_fp8(dqkv_t, x_t, f32, nq, nkv, inv_a, inv_b)


class _Rowwise:
    """torchao's rowwise recipe: every operand e4m3, one power-of-two scale per row along the GEMM's reduction axis.
    Activations and gradients get a row-scaled copy and a column-scaled transposed copy (for wgrad), weights a
    row-scaled copy (forward) and a column-scaled transposed one (dgrad).  dq|dk|dv share each row's scale, and the
    transposed [Wq;Wk;Wv] each column's, because the fused QKV dgrad sums over the stacked rows.  The forward saves the
    1/s of its transposed copies (h1, o, h2, hm) in one vector; forward GEMMs accumulate in the tensor-core accumulator,
    backward GEMMs promote."""

    def __init__(self, dev, dims, saved=None):
        d, n_o, ffn = dims
        off, self.t_off = 0, {}
        for slot, n in ((_F8_H1, d), (_F8_O, n_o), (_F8_H2, d), (_F8_HM, ffn)):
            self.t_off[slot] = (off, n)
            off += n
        self.state = torch.empty(off, dtype=torch.float32, device=dev) if saved is None else saved
        self.promoted = saved is not None

    qkv_plan = staticmethod(_Tensorwise.qkv_plan)

    def saved_inv(self, slot):
        off, n = self.t_off[slot]
        return self.state[off:off + n]

    def _quant(self, x, inv_t=None):
        x8, inv = fp8_rowwise_cast(x)
        amax = torch.zeros(x.shape[1], dtype=torch.float32, device=x.device)
        fp8_colwise_amax(x, amax)
        x_t, inv_t = fp8_colwise_cast_t(x, amax, inv=inv_t)
        return x8, inv, x_t, inv_t

    def act(self, x, slot):
        return self._quant(x, self.saved_inv(slot))

    def grad(self, dy, slot):
        return self._quant(dy)

    def weights(self, ws, slot):
        inv = torch.empty(sum(w.shape[0] for w in ws), dtype=torch.float32, device=ws[0].device)
        w8s, invs, off = [], [], 0
        for w in ws:
            n = w.shape[0]
            w8s.append(fp8_rowwise_cast(w, inv=inv[off:off + n])[0])
            invs.append(inv[off:off + n])
            off += n
        return w8s, invs, inv

    def weight_t(self, ws, slot):
        dev, d = ws[0].device, ws[0].shape[1]
        amax = torch.zeros(d, dtype=torch.float32, device=dev)
        for w in ws:
            fp8_colwise_amax(w, amax)
        w_t = torch.empty((d, sum(w.shape[0] for w in ws)), dtype=F8E4M3, device=dev)
        inv = torch.empty(d, dtype=torch.float32, device=dev)
        off = 0
        for w in ws:
            fp8_colwise_cast_t(w, amax, out_t=w_t[:, off:off + w.shape[0]], inv=inv)
            off += w.shape[0]
        return w_t, inv

    def qkv_grad(self, dys, slot):
        return self._quant(torch.cat(dys, dim=1))

    def gemm(self, a, b, inv_a, inv_b, **kw):
        return gemm_fp8_rowwise(a, b, inv_a, inv_b, promoted=self.promoted, **kw)

    def swiglu(self, x, wg, wu, inv_x, inv_w):
        return gemm_swiglu_fp8_rowwise(x, wg, wu, inv_x, inv_w)

    def dswiglu(self, dy, wd_t, g, u, inv_a, inv_b):
        return gemm_dswiglu_fp8_rowwise(dy, wd_t, g, u, inv_a, inv_b)

    def qkv_fwd(self, x, wq, wk, wv, inv_x, inv_w, rope):
        return gemm_qkv_fwd_fp8_rowwise(x, wq, wk, wv, inv_x, inv_w, rope=rope)

    def qkv_dgrad(self, dqkv, w_t, nq, nkv, inv_a, inv_b):
        return gemm_qkv_dgrad_fp8_rowwise(dqkv, w_t, nq, nkv, inv_a, inv_b)

    def qkv_wgrad(self, dqkv_t, x_t, f32, nq, nkv, inv_a, inv_b):
        return gemm_qkv_wgrad_fp8_rowwise(dqkv_t, x_t, f32, nq, nkv, inv_a, inv_b)


_FP8_RECIPE_CLASSES = {"tensorwise": _Tensorwise, "rowwise": _Rowwise}


def cached_block_forward(x2, weights, cos, sin, H, KV, eps, hd, attend, qkv_rows=None, float8=None, step=False):
    """One block of cached decoding (generation.py) on its bf16 working weights: block_forward without the tensors
    a backward needs, or with `float8` (the block's float8_inference_weights) the FP8 block under RowwiseInference."""
    if float8 is None:
        return block_forward(x2, *weights, cos, sin, H, KV, eps, hd, attend, need_gu=False, qkv_rows=qkv_rows)
    return _block_forward_fp8(x2, *weights, cos, sin, H, KV, eps, hd, attend, RowwiseInference(float8, step))


def float8_inference_weights(wqb, wkb, wvb, wob, wgb, wub, wdb):
    """The e4m3 copies of one block's projections for cached FP8 inference (the model config key `float8_inference`),
    made once per generate call: {slot: (stacked rows, their 1/s, row count of each weight)} for [Wq;Wk;Wv], Wo,
    [Wg;Wu] and Wd.  Row scales make the stacked copy equal to the copies of its parts."""
    _fp8_dims(wqb.shape[1], wqb.shape[0], wkb.shape[0], wob.shape[1], wgb.shape[0], key="float8_inference")
    out = {}
    for slot, ws in ((_F8_WQKV, (wqb, wkb, wvb)), (_F8_WO, (wob,)), (_F8_WGU, (wgb, wub)), (_F8_WD, (wdb,))):
        w = ws[0] if len(ws) == 1 else torch.cat(ws)
        out[slot] = (*fp8_rowwise_cast(w), [t.shape[0] for t in ws])
    return out


class RowwiseInference:
    """The rowwise recipe for cached decoding: weights from float8_inference_weights, activations as a row-scaled copy only
    (nothing is saved for a backward).  A prompt pass (`step=False`: prefill, generate_many admissions; rows padded to a
    multiple of 16 by the caller) runs the rowwise wgmma kernels as the rowwise training forward does; a cached step
    (`step=True`: decode, draft and verify steps, any row count) runs tn_gemm_fp8_decode on the bf16 rows, which
    quantises them with the same rule, so a row's result does not depend on the other rows of the step.  Always rowwise:
    a per-tensor activation scale would tie each row to its neighbours (slots, draft rows)."""

    state = None

    def __init__(self, weights8, step: bool):
        self.w8, self.step = weights8, step

    def qkv_plan(self, M, nq, nkv, rope_ok):
        """(one QKV launch, RoPE in its epilogue): a cached step runs one decode launch over [Wq;Wk;Wv]."""
        return (True, False) if self.step else _Rowwise.qkv_plan(M, nq, nkv, rope_ok)

    def act(self, x, slot):
        return (x, None, None, None) if self.step else (*fp8_rowwise_cast(x), None, None)

    def weights(self, ws, slot):
        w8, inv, sizes = self.w8[slot]
        parts, invs, off = [], [], 0
        for n in sizes:
            parts.append(w8[off:off + n])
            invs.append(inv[off:off + n])
            off += n
        return parts, invs, inv

    def gemm(self, a, b, inv_a, inv_b, residual=None):
        if self.step:
            return gemm_fp8_decode(a, b, inv_b, residual=residual)
        return gemm_fp8_rowwise(a, b, inv_a, inv_b, promoted=False, residual=residual)

    def swiglu(self, x, wg, wu, inv_x, inv_w):
        if self.step:
            return None, None, gemm_fp8_decode(x, self.w8[_F8_WGU][0], inv_w, swiglu=True)
        return gemm_swiglu_fp8_rowwise(x, wg, wu, inv_x, inv_w, need_gu=False)

    def qkv_fwd(self, x, wq, wk, wv, inv_x, inv_w, rope):
        if self.step:
            return gemm_fp8_decode(x, self.w8[_F8_WQKV][0], inv_w)
        return gemm_qkv_fwd_fp8_rowwise(x, wq, wk, wv, inv_x, inv_w, rope=rope)


def _fp8_recipe(name, dev, wqb, wob, wgb, saved=None):
    return _FP8_RECIPE_CLASSES[check_fp8_recipe(name)](dev, (wqb.shape[1], wob.shape[1], wgb.shape[0]), saved)


def _block_forward_fp8(x2, ln1, wqb, wkb, wvb, bq, bk, bv, wob, ln2, wgb, wub, wdb, cos, sin, H, KV, eps, hd, attend,
                       recipe="tensorwise"):
    """block_forward with FP8 projections (see there) under `recipe`: a name (_Tensorwise, _Rowwise), or a recipe
    object (RowwiseInference)."""
    nq, nkv, d, ffn = wqb.shape[0], wkb.shape[0], wqb.shape[1], wgb.shape[0]
    if isinstance(recipe, str):
        _fp8_dims(x2.shape[0], d, nq, nkv, wob.shape[1], ffn)
        rc = _fp8_recipe(recipe, x2.device, wqb, wob, wgb)
    else:
        rc = recipe
    h1, _, rstd1 = rmsnorm_fwd(x2, ln1, eps)
    h1_8, ih1, h1_t, _ = rc.act(h1, _F8_H1)
    wqkv8, iwqkv, iwqkv_all = rc.weights([wqb, wkb, wvb], _F8_WQKV)
    fused, rope_in_gemm = rc.qkv_plan(h1.shape[0], nq, nkv, bq is None and hd == 128)
    if fused:
        qkv = rc.qkv_fwd(h1_8, *wqkv8, ih1, iwqkv_all, (cos, sin) if rope_in_gemm else None)
        q, k, v = qkv[:, :nq], qkv[:, nq:nq + nkv], qkv[:, nq + nkv:]
    else:
        q, k, v = (rc.gemm(h1_8, w8, ih1, iw) for w8, iw in zip(wqkv8, iwqkv))
    if bq is not None:
        q += bq.to(BF16); k += bk.to(BF16); v += bv.to(BF16)
    if not rope_in_gemm:
        rope_apply_(q, cos, sin, H, hd)
        rope_apply_(k, cos, sin, KV, hd)
    if hd != 128:
        q, k, v = _pad_heads(q, H, hd), _pad_heads(k, KV, hd), _pad_heads(v, KV, hd)
    o, lse, k, v = attend(q, k, v)
    o8, io, o_t, _ = rc.act(o if hd == 128 else _unpad_heads(o, H, hd), _F8_O)
    (wo8,), (iwo,), _ = rc.weights([wob], _F8_WO)
    x1 = rc.gemm(o8, wo8, io, iwo, residual=x2)
    h2, _, rstd2 = rmsnorm_fwd(x1, ln2, eps)
    h2_8, ih2, h2_t, _ = rc.act(h2, _F8_H2)
    (wg8, wu8), _, iwgu = rc.weights([wgb, wub], _F8_WGU)
    g, u, hm = rc.swiglu(h2_8, wg8, wu8, ih2, iwgu)
    hm8, ihm, hm_t, _ = rc.act(hm, _F8_HM)
    (wd8,), (iwd,), _ = rc.weights([wdb], _F8_WD)
    out = rc.gemm(hm8, wd8, ihm, iwd, residual=x1)
    return out, (rstd1, h1_t, q, k, v, o, lse, x1, rstd2, h2_t, g, u, hm_t, o_t, rc.state)


def _fp8_weight_t(wb, st, slot, out_t=None):
    """The transposed e4m3 copy of bf16 weight wb [N, K] -> [K, N], at the scale the forward used (row `slot` of st)."""
    return fp8_cast(wb, st[slot, 0], False, row=False, out_t=out_t)[1]


def _block_backward_fp8(ctx, saved, d2):
    """Weight and input gradients of the FP8 block under ctx.fp8_recipe: every incoming gradient is quantised (dq|dk|dv
    as one operand, which the fused QKV dgrad sums over), dgrad = dY·Wᵀ and wgrad = dYᵀ·Xᵀ as FP8 GEMMs on K-major
    copies."""
    (x2, ln1, ln2, wqb, wkb, wvb, wob, wgb, wub, wdb, cos, sin, rstd1, h1_t, q, k, v, o, lse, x1, rstd2, h2_t, g, u,
     hm_t, o_t, state) = saved
    H, KV, f32, hd = ctx.H, ctx.KV, ctx.f32, ctx.hd
    rb = _fp8_recipe(ctx.fp8_recipe, d2.device, wqb, wob, wgb, saved=state)
    # ---- MLP ----
    d2_8, id2, d2_t, id2_t = rb.grad(d2, _F8_D2)
    wd_t, iwd_t = rb.weight_t([wdb], _F8_WD)
    dg, du = rb.dswiglu(d2_8, wd_t, g, u, id2, iwd_t)
    dwd = rb.gemm(d2_t, hm_t, id2_t, rb.saved_inv(_F8_HM), out_f32=f32)
    del d2_8, d2_t, wd_t
    dg8, idg, dg_t, idg_t = rb.grad(dg, _F8_DG)
    du8, idu, du_t, idu_t = rb.grad(du, _F8_DU)
    del dg, du
    wg_t, iwg_t = rb.weight_t([wgb], _F8_WGU)
    dh2 = rb.gemm(dg8, wg_t, idg, iwg_t)
    wu_t, iwu_t = rb.weight_t([wub], _F8_WGU)
    dh2 = rb.gemm(du8, wu_t, idu, iwu_t, residual=dh2, out=dh2)
    dwg = rb.gemm(dg_t, h2_t, idg_t, rb.saved_inv(_F8_H2), out_f32=f32)
    dwu = rb.gemm(du_t, h2_t, idu_t, rb.saved_inv(_F8_H2), out_f32=f32)
    del dg8, dg_t, du8, du_t, wg_t, wu_t
    dx1, dln2 = rmsnorm_bwd(x1, dh2, ln2, rstd2, ds_extra=d2)
    # ---- attention ----
    dx1_8, idx1, dx1_t, idx1_t = rb.grad(dx1, _F8_DX1)
    wo_t, iwo_t = rb.weight_t([wob], _F8_WO)
    do = rb.gemm(dx1_8, wo_t, idx1, iwo_t)
    dwo = rb.gemm(dx1_t, o_t, idx1_t, rb.saved_inv(_F8_O), out_f32=f32)
    del dx1_8, dx1_t, wo_t
    if hd != 128:   # padded heads: gradients of the padded tensors, un-padded, then the inverse rotation at head_dim hd
        dq, dk, dv = attn_bwd(q, k, v, o, _pad_heads(do, H, hd), lse, ctx.plan, H, KV, ctx.scale)
        dq, dk, dv = _unpad_heads(dq, H, hd), _unpad_heads(dk, KV, hd), _unpad_heads(dv, KV, hd)
        rope_apply_(dq, cos, sin, H, hd, inverse=True)
        rope_apply_(dk, cos, sin, KV, hd, inverse=True)
    else:
        dq, dk, dv = attn_bwd(q, k, v, o, do, lse, ctx.plan, H, KV, ctx.scale, rope=(cos, sin))
    del do
    nq, nkv = wqb.shape[0], wkb.shape[0]
    M = d2.shape[0]
    dqkv8, idqkv, dqkv_t, idqkv_t = rb.qkv_grad((dq, dk, dv), _F8_DQKV)
    w_t, iw_t = rb.weight_t([wqb, wkb, wvb], _F8_WQKV)   # [Wq;Wk;Wv]ᵀ
    if qkv_fusable(M, nq, nkv):
        dh1 = rb.qkv_dgrad(dqkv8, w_t, nq, nkv, idqkv, iw_t)
        dwq, dwk, dwv = rb.qkv_wgrad(dqkv_t, h1_t, f32, nq, nkv, idqkv_t, rb.saved_inv(_F8_H1))
    else:
        dh1 = None
        dws = []
        for off, n in zip((0, nq, nq + nkv), (nq, nkv, nkv)):
            dh1 = rb.gemm(dqkv8[:, off:off + n], w_t[:, off:off + n], idqkv, iw_t, residual=dh1, out=dh1)
            dws.append(rb.gemm(dqkv_t[off:off + n], h1_t, _seg(idqkv_t, off, n), rb.saved_inv(_F8_H1), out_f32=f32))
        dwq, dwk, dwv = dws
    dbq = dbk = dbv = None
    if ctx.has_bias:
        dbq = dq.float().sum(0).to(ctx.w_dtype); dbk = dk.float().sum(0).to(ctx.w_dtype); dbv = dv.float().sum(0).to(ctx.w_dtype)
    dx, dln1 = rmsnorm_bwd(x2, dh1, ln1, rstd1, ds_extra=dx1)
    return dx, dln1.to(ln1.dtype), dwq, dwk, dwv, dbq, dbk, dbv, dwo, dln2.to(ln2.dtype), dwg, dwu, dwd


class DecoderLayerFn(torch.autograd.Function):
    """One pre-norm decoder block as a single autograd node (hf: LlamaDecoderLayer.forward modeling_llama.py:303-333):
    7 kernel launches forward, residual adds fused into the o_proj / down_proj GEMM epilogues, q/k/v projections one
    segmented GEMM, the residual-branch gradient fused into the RMSNorm backward kernel.  Parameters stay separate
    nn.Linear weights (HF FQNs) so FSDP2 / DCP / convert_* of the reference keep working
    (ref: touchnet/models/helper_func.py:134-202).  Use `decoder_layer(...)`: it resolves the bf16 working copies of the
    fp32 master weights on the parameter objects and passes them in as non-differentiable inputs."""

    @staticmethod
    def forward(ctx, x, ln1, wq, wk, wv, bq, bk, bv, wo, ln2, wg, wu, wd, wqb, wkb, wvb, wob, wgb, wub, wdb, cos, sin,
                plan, H, KV, eps, hd=128, fp8=False, fp8_recipe="tensorwise"):
        x2 = _rows2d(x)
        scale = 1.0 / math.sqrt(hd)
        if hd != 128 and (hd > 128 or hd % 8 or plan.tp is not None or plan.cp_group is not None):
            raise _lib.TouchNetB200Error(f"head_dim {hd}: only multiples of 8 up to 128, without tensor / context parallelism")
        tp = plan.tp                # tensor + sequence parallel: x holds T/tp rows, weights are this rank's shards
        if tp is not None and plan.cp_group is not None:
            raise _lib.TouchNetB200Error("tensor parallelism and context parallelism cannot be combined in one block")
        if fp8 and (tp is not None or plan.cp_group is not None):
            raise _lib.TouchNetB200Error("float8_training does not support tensor or context parallelism")

        def attend(q, k, v):
            if plan.cp_group is None:
                o, lse = attn_fwd(q, k, v, plan, H, KV, scale)
                return o, lse, k, v
            # context parallel: K/V of all cp ranks are gathered, the kernel runs on this rank's query window
            from . import context_parallel as _cp
            return _cp.cp_attn_fwd(q, k, v, plan, H, KV, scale)

        out, saved = block_forward(x2, ln1, wqb, wkb, wvb, bq, bk, bv, wob, ln2, wgb, wub, wdb, cos, sin, H, KV, eps, hd,
                                   attend, tp, fp8=fp8, fp8_recipe=fp8_recipe)
        ctx.save_for_backward(x2, ln1, ln2, wqb, wkb, wvb, wob, wgb, wub, wdb, cos, sin, *saved)
        ctx.plan, ctx.H, ctx.KV, ctx.scale, ctx.has_bias, ctx.hd, ctx.fp8 = plan, H, KV, scale, bq is not None, hd, fp8
        ctx.f32 = wq.dtype == torch.float32
        ctx.w_dtype = wq.dtype
        ctx.fp8_recipe = fp8_recipe
        return out.view(x.shape)

    @staticmethod
    def backward(ctx, dout):
        d2 = _rows2d(dout)
        if d2.dtype != BF16:
            d2 = d2.to(BF16)
        if ctx.fp8:
            dx, *grads = _block_backward_fp8(ctx, ctx.saved_tensors, d2)
            return (dx.view(dout.shape), *grads) + (None,) * 16
        (x2, ln1, ln2, wqb, wkb, wvb, wob, wgb, wub, wdb, cos, sin, rstd1, h1, q, k, v, o, lse, x1, rstd2, h2, g, u,
         hm) = ctx.saved_tensors
        H, KV, f32 = ctx.H, ctx.KV, ctx.f32
        tp = ctx.plan.tp
        # ---- MLP ----
        d2f = d2 if tp is None else tp.gather_rows(d2)     # backward of the forward reduce-scatter
        dg, du = gemm_dswiglu(d2f, wdb, g, u)          # down-proj dgrad, SwiGLU backward in its epilogue
        dwd = _wgrad(d2f, hm, f32)
        del d2f
        dh2 = gemm(dg, wgb, b_mn=True)
        dh2 = gemm(du, wub, b_mn=True, residual=dh2, out=dh2)
        dwg = _wgrad(dg, h2, f32)
        dwu = _wgrad(du, h2, f32)
        del dg, du
        if tp is not None:
            dh2 = tp.reduce_scatter(dh2)               # backward of the forward all-gather
        dx1, dln2 = rmsnorm_bwd(x1, dh2, ln2, rstd2, ds_extra=d2)
        # ---- attention ----
        dx1f = dx1 if tp is None else tp.gather_rows(dx1)
        hd = ctx.hd
        do = gemm(dx1f, wob, b_mn=True)
        dwo = _wgrad(dx1f, o if hd == 128 else _unpad_heads(o, H, hd), f32)
        if hd != 128:
            do = _pad_heads(do, H, hd)
        del dx1f
        nq, nkv = wqb.shape[0], wkb.shape[0]
        fused = qkv_fusable(h1.shape[0], nq, nkv)
        if ctx.plan.cp_group is not None:
            from . import context_parallel as _cp
            dq, dk, dv = _cp.cp_attn_bwd(q, k, v, o, do, lse, ctx.plan, H, KV, ctx.scale)   # dK/dV reduce-scattered
            if fused:
                dqkv = torch.cat([dq, dk, dv], dim=1)
                dq, dk, dv = dqkv[:, :nq], dqkv[:, nq:nq + nkv], dqkv[:, nq + nkv:]
            rope_apply_(dq, cos, sin, H, 128, inverse=True)
            rope_apply_(dk, cos, sin, KV, 128, inverse=True)
        elif hd != 128:   # padded heads: gradients of the padded tensors, un-padded, then the inverse rotation at head_dim hd
            dqp, dkp, dvp = attn_bwd(q, k, v, o, do, lse, ctx.plan, H, KV, ctx.scale)
            dq, dk, dv = _unpad_heads(dqp, H, hd), _unpad_heads(dkp, KV, hd), _unpad_heads(dvp, KV, hd)
            rope_apply_(dq, cos, sin, H, hd, inverse=True)
            rope_apply_(dk, cos, sin, KV, hd, inverse=True)
            if fused:
                dqkv = torch.cat([dq, dk, dv], dim=1)
                dq, dk, dv = dqkv[:, :nq], dqkv[:, nq:nq + nkv], dqkv[:, nq + nkv:]
        elif fused:   # inverse RoPE happens in the attention-backward epilogues
            dqkv = torch.empty((h1.shape[0], nq + 2 * nkv), dtype=BF16, device=x2.device)
            dq, dk, dv = dqkv[:, :nq], dqkv[:, nq:nq + nkv], dqkv[:, nq + nkv:]
            attn_bwd(q, k, v, o, do, lse, ctx.plan, H, KV, ctx.scale, out=(dq, dk, dv), rope=(cos, sin))
        else:
            dq, dk, dv = attn_bwd(q, k, v, o, do, lse, ctx.plan, H, KV, ctx.scale, rope=(cos, sin))
        if fused:
            dh1 = gemm_qkv_dgrad(dqkv, wqb, wkb, wvb)
            dwq, dwk, dwv = gemm_qkv_wgrad(dqkv, h1, f32, nq, nkv)
        else:
            dh1 = gemm(dq, wqb, b_mn=True)
            dh1 = gemm(dk, wkb, b_mn=True, residual=dh1, out=dh1)
            dh1 = gemm(dv, wvb, b_mn=True, residual=dh1, out=dh1)
            dwq = _wgrad(dq, h1, f32); dwk = _wgrad(dk, h1, f32); dwv = _wgrad(dv, h1, f32)
        dbq = dbk = dbv = None
        if ctx.has_bias:
            dbq = dq.float().sum(0).to(ctx.w_dtype); dbk = dk.float().sum(0).to(ctx.w_dtype); dbv = dv.float().sum(0).to(ctx.w_dtype)
        if tp is not None:
            dh1 = tp.reduce_scatter(dh1)
        dx, dln1 = rmsnorm_bwd(x2, dh1, ln1, rstd1, ds_extra=dx1)
        if tp is not None:                             # replicated norm weights, sequence-sharded rows: sum the partials
            tp.all_reduce_(dln1)
            tp.all_reduce_(dln2)
        return (dx.view(dout.shape), dln1.to(ln1.dtype), dwq, dwk, dwv, dbq, dbk, dbv, dwo, dln2.to(ln2.dtype), dwg, dwu,
                dwd) + (None,) * 16


def decoder_layer(x, ln1, wq, wk, wv, bq, bk, bv, wo, ln2, wg, wu, wd, cos, sin, plan, H, KV, eps, hd=128, fp8=False, *,
                  float8_recipe_name="tensorwise"):
    """`fp8`: the seven projections in FP8 (the `float8_training` model config key; see block_forward), under
    `float8_recipe_name` (the config key of that name: "tensorwise" or "rowwise")."""
    if fp8:
        check_fp8_recipe(float8_recipe_name)
    return DecoderLayerFn.apply(x, ln1, wq, wk, wv, bq, bk, bv, wo, ln2, wg, wu, wd, bf16_weight(wq), bf16_weight(wk),
                                bf16_weight(wv), bf16_weight(wo), bf16_weight(wg), bf16_weight(wu), bf16_weight(wd),
                                cos, sin, plan, H, KV, eps, hd, fp8, float8_recipe_name)
