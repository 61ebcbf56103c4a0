"""Pack-loss cross-entropy and accuracy behind the reference's `loss_fn` / `acc_fn` slots of TrainSpec
(ref: touchnet/utils/train_spec.py:37-38).

    cross_entropy_loss(pred, labels, sentence_lens, num_sentence) -> (loss_per_sample, loss_per_token)
        ref: touchnet/loss/cross_entropy.py:12-50 (+ the compiled fp32-upcast CE of touchnet/loss/__init__.py:7-28)
    accuracy(pred, labels) -> fraction of non-ignored positions whose argmax equals the label
        ref: touchnet/utils/metrics.py:26-50

The CUDA kernels (csrc/loss.cu) stream the bf16 logits once forward (online logsumexp + argmax) and once backward,
overwriting them in place with the logit gradient; no fp32 copy of the [B,T,V] tensor is ever made.  In-place is safe in
the reference's loop order: loss_fn and acc_fn run, `del pred`, then backward (ref: touchnet/bin/train.py:447-455).

Fused lm_head + loss (SURVEY 8(f) rank 1 as written: "no [B,T,V] logits"): when the model runs with
`fused_linear_ce` (modeling.py) its `pred.logits` is a `LazyLogits` handle (final hidden states + lm_head weight) and
`cross_entropy_loss` runs `FusedLinearCEFn`: per chunk of `FUSED_CE_CHUNK` token rows - lm_head GEMM into ONE reusable
[chunk, V] bf16 buffer, `tn_pack_ce_fused_bf16` (loss statistics + argmax + in-place logit gradient), dgrad GEMM into
dh[chunk], wgrad GEMM accumulating into dW - the way the incumbent's best path does it (Liger fused-linear-cross-entropy,
ref: touchnet/bin/train.py:443-445).  The [B,T,V] tensor never exists; backward only scales dh / dW by the upstream
gradient (a no-op kernel when that is 1).
"""
from __future__ import annotations

import weakref

import torch

from . import _lib

# argmax of the logits the loss kernel saw last: (weak reference to the caller's logits tensor, its version, argmax).
# Keyed on the live tensor OBJECT, not on its address - a freed tensor's address is reused by the next logits.
_LAST_ARGMAX = None


def _st() -> int:
    return torch.cuda.current_stream().cuda_stream


def _pack_ce_fwd(x: torch.Tensor, labels: torch.Tensor):
    """(lse, ce, argmax) [M] of the bf16 CUDA logits x [M, V] (unit column stride); contiguous int64 labels outside
    [0, V) are ignored (ce 0)."""
    if not x.is_cuda or x.dtype != torch.bfloat16:
        raise _lib.TouchNetB200Error("pack-loss CE needs bf16 CUDA logits (no CPU path)")
    assert x.stride(1) == 1
    M, V = x.shape
    lse = torch.empty(M, dtype=torch.float32, device=x.device)
    ce = torch.empty_like(lse)
    am = torch.empty(M, dtype=torch.int32, device=x.device)
    _lib.call("tn_pack_ce_fwd_bf16", x.data_ptr(), x.stride(0), labels.data_ptr(), lse.data_ptr(), ce.data_ptr(),
              am.data_ptr(), M, V, _st())
    return lse, ce, am


def _pack_ce_bwd_(ctx, g_loss, *vp):
    """Backward of _PackCEFn / _VocabParallelCEFn: overwrites ctx.logits in place with dlogits and returns them in the
    forward's shape.  vp = (v0, v_total) selects the vocabulary-parallel kernel."""
    lab, sl, lse = ctx.saved_tensors
    x = ctx.logits
    g = g_loss.reshape(1).float().contiguous()
    _lib.call("tn_pack_ce_bwd_vp_bf16" if vp else "tn_pack_ce_bwd_bf16", x.data_ptr(), x.stride(0), lab.data_ptr(),
              sl.data_ptr(), lse.data_ptr(), g.data_ptr(), float(ctx.inv_ns), x.shape[0], x.shape[1], *vp, _st())
    torch.autograd.graph.increment_version(x)   # the kernel overwrote the caller's logits with their gradient: make
    ctx.logits = None                           # autograd (and accuracy()'s cache key) see the mutation
    return x.view(ctx.shape)


class _PackCEFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, labels, sentence_lens, inv_num_sentence):
        x = logits.view(-1, logits.shape[-1])
        lab = labels.reshape(-1).contiguous()
        sl = sentence_lens.reshape(-1).contiguous()
        lse, ce, am = _pack_ce_fwd(x, lab)
        ctx.save_for_backward(lab, sl, lse)
        ctx.logits = x                      # NOT save_for_backward: backward overwrites it in place on purpose
        ctx.inv_ns = inv_num_sentence
        ctx.shape = logits.shape
        ctx.mark_non_differentiable(ce, am)
        loss_per_sample = (ce / sl.float()).sum() * inv_num_sentence
        return loss_per_sample, ce, am

    @staticmethod
    def backward(ctx, g_loss, _g_ce, _g_am):
        return _pack_ce_bwd_(ctx, g_loss), None, None, None


FUSED_CE_CHUNK = 4096     # token rows per chunk: the [chunk, V] buffer is 1 GB at V = 128 k instead of 2.1 GB for T = 8192;
                          # smaller chunks shorten the K of the accumulating fp32 lm_head wgrad, whose read-modify-write of
                          # the whole fp32 dW per chunk then costs more than the mainloop


class LazyLogits:
    """`pred.logits` of a model running with the fused lm_head + loss: NOT a tensor - the final hidden states and the
    lm_head weight, from which `cross_entropy_loss` / `accuracy` compute what the reference computes from logits.
    `materialize()` gives the real (differentiable) [B,T,V] tensor for any other consumer."""

    def __init__(self, hidden: torch.Tensor, weight: torch.Tensor):
        self.hidden, self.weight = hidden, weight
        self.shape = torch.Size((*hidden.shape[:-1], weight.shape[0]))
        self.dtype, self.device = torch.bfloat16, hidden.device
        self._stats = None          # (ce [M], argmax [M]) of the last fused pass

    def materialize(self) -> torch.Tensor:
        from . import ops
        return ops.linear(self.hidden, self.weight)

    def dim(self) -> int:
        return len(self.shape)

    def size(self, i=None):
        return self.shape if i is None else self.shape[i]

    def __repr__(self):
        return f"LazyLogits(shape={tuple(self.shape)}, fused lm_head + loss; .materialize() for the tensor)"


class VocabParallelLogits:
    """`pred.logits` of a tensor-parallel model running loss parallel: this rank's vocabulary columns [v0, v0 + V/tp) of the
    logits ([B, T, V/tp] bf16, part of the autograd graph) + the tp group.  Not a tensor; `materialize()` all-gathers."""

    def __init__(self, local: torch.Tensor, group, v0: int, v_total: int):
        self.local, self.group, self.v0, self.v_total = local, group, int(v0), int(v_total)
        self.shape = torch.Size((*local.shape[:-1], v_total))
        self.dtype, self.device = local.dtype, local.device
        self._stats = None

    def materialize(self) -> torch.Tensor:
        import torch.distributed as dist
        n = dist.get_world_size(self.group)
        parts = [torch.empty_like(self.local) for _ in range(n)]
        dist.all_gather(parts, self.local.detach().contiguous(), group=self.group)
        return torch.cat(parts, dim=-1)

    def dim(self) -> int:
        return len(self.shape)


class _VocabParallelCEFn(torch.autograd.Function):
    """Pack-loss cross-entropy on vocabulary-sharded logits.  Per shard: tn_pack_ce_fwd_bf16 (local logsumexp, local label
    term, local argmax); across the tp group: three [M]-sized all-reduces (max of the local logsumexps, sum of the rescaled
    exponentials, the label logit from its owner); backward: tn_pack_ce_bwd_vp_bf16 in place on the local columns."""

    @staticmethod
    def forward(ctx, local, labels, sentence_lens, inv_num_sentence, group, v0, v_total):
        import torch.distributed as dist
        Vl = local.shape[-1]
        x = local.view(-1, Vl)
        lab = labels.reshape(-1).contiguous()
        sl = sentence_lens.reshape(-1).contiguous()
        lab_l = lab - v0                                                  # out of [0, Vl): "ignored" by the local kernel
        lse_l, ce_l, am_l = _pack_ce_fwd(x, lab_l)
        mine = (lab_l >= 0) & (lab_l < Vl)
        m = lse_l.clone()
        dist.all_reduce(m, op=dist.ReduceOp.MAX, group=group)
        ssum = torch.exp(lse_l - m)
        dist.all_reduce(ssum, op=dist.ReduceOp.SUM, group=group)
        lse = m + torch.log(ssum)
        xlab = torch.where(mine, lse_l - ce_l, torch.zeros_like(lse_l))      # the label's logit, from the rank that owns it
        dist.all_reduce(xlab, op=dist.ReduceOp.SUM, group=group)
        valid = (lab >= 0) & (lab < v_total)
        ce = torch.where(valid, lse - xlab, torch.zeros_like(lse))
        # global argmax: best local value of every rank, lowest vocabulary index wins ties (torch.argmax semantics)
        best = x.gather(1, am_l.long()[:, None]).squeeze(1).float()
        n = dist.get_world_size(group)
        vals = [torch.empty_like(best) for _ in range(n)]
        idxs = [torch.empty_like(am_l) for _ in range(n)]
        dist.all_gather(vals, best, group=group)
        dist.all_gather(idxs, am_l + v0, group=group)
        vals, idxs = torch.stack(vals), torch.stack(idxs)
        win = vals.argmax(0)                                               # first (lowest-rank = lowest-index) maximum
        am = idxs.gather(0, win[None]).squeeze(0)
        ctx.save_for_backward(lab, sl, lse)
        ctx.logits, ctx.inv_ns, ctx.shape, ctx.v0, ctx.v_total = x, inv_num_sentence, local.shape, v0, v_total
        ctx.mark_non_differentiable(ce, am)
        return (ce / sl.float()).sum() * inv_num_sentence, ce, am

    @staticmethod
    def backward(ctx, g_loss, _g_ce, _g_am):
        return _pack_ce_bwd_(ctx, g_loss, ctx.v0, ctx.v_total), None, None, None, None, None, None


class FusedLinearCEFn(torch.autograd.Function):
    """loss_per_sample(h, W) of ref: touchnet/loss/cross_entropy.py:12-50 with logits = h . W^T never materialised.
    Gradients for an upstream gradient of 1 are produced during forward, chunk by chunk; backward scales them."""

    @staticmethod
    def forward(ctx, h, w, wb, labels, sentence_lens, inv_num_sentence, chunk):
        from . import ops
        d = h.shape[-1]
        h2 = ops._rows2d(h)
        if h2.dtype != torch.bfloat16:
            h2 = h2.to(torch.bfloat16)
        M, V = h2.shape[0], wb.shape[0]
        dev = h2.device
        lab = labels.reshape(-1).contiguous()
        sl = sentence_lens.reshape(-1).contiguous()
        assert lab.numel() == M and sl.numel() == M, "labels / sentence_lens must cover every token row"
        lse = torch.empty(M, dtype=torch.float32, device=dev)
        ce = torch.empty(M, dtype=torch.float32, device=dev)
        am = torch.empty(M, dtype=torch.int32, device=dev)
        need_dh, need_dw = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        f32 = w.dtype == torch.float32
        dh = torch.empty((M, d), dtype=torch.bfloat16, device=dev) if need_dh else None
        dw = torch.empty((V, d), dtype=w.dtype, device=dev) if need_dw else None
        chunk = max(256, int(chunk))
        ldv = (V + 7) // 8 * 8                                    # 16-byte aligned rows for any vocabulary size
        buf = torch.empty((min(chunk, M), ldv), dtype=torch.bfloat16, device=dev)
        for r0 in range(0, M, chunk):
            r1 = min(M, r0 + chunk)
            n = r1 - r0
            x = buf[:n, :V]
            ops.gemm(h2[r0:r1], wb, out=x)                                       # logits of this chunk
            _lib.call("tn_pack_ce_fused_bf16", x.data_ptr(), x.stride(0), lab[r0:r1].data_ptr(), sl[r0:r1].data_ptr(),
                      lse[r0:r1].data_ptr(), ce[r0:r1].data_ptr(), am[r0:r1].data_ptr(), float(inv_num_sentence), n, V,
                      _st())                                                    # x now holds dlogits (upstream grad 1)
            if need_dh:
                ops.gemm(x, wb, b_mn=True, out=dh[r0:r1])                        # dh = dlogits . W
            if need_dw:                                                         # dW (+)= dlogits^T . h
                ops.gemm(x, h2[r0:r1], a_mn=True, b_mn=True, out_f32=f32, residual=dw if r0 > 0 else None, out=dw)
        ctx.save_for_backward(dh, dw)
        ctx.h_shape, ctx.h_dtype = h.shape, h.dtype
        ctx.mark_non_differentiable(ce, am)
        loss_per_sample = (ce / sl.float()).sum() * inv_num_sentence
        return loss_per_sample, ce, am

    @staticmethod
    def backward(ctx, g_loss, _g_ce, _g_am):
        dh, dw = ctx.saved_tensors
        g = g_loss.reshape(1).float().contiguous()
        if dh is not None:
            _lib.call("tn_scale_bf16", dh.data_ptr(), dh.numel(), g.data_ptr(), _st())     # no-op kernel when g == 1
            torch.autograd.graph.increment_version(dh)
            dh = dh.view(ctx.h_shape).to(ctx.h_dtype)
        if dw is not None:
            name = "tn_scale_f32" if dw.dtype == torch.float32 else "tn_scale_bf16"
            _lib.call(name, dw.data_ptr(), dw.numel(), g.data_ptr(), _st())
            torch.autograd.graph.increment_version(dw)
        return dh, dw, None, None, None, None, None


def fused_linear_cross_entropy(hidden: torch.Tensor, weight: torch.Tensor, labels: torch.Tensor,
                               sentence_lens: torch.Tensor, inv_num_sentence: float, chunk: int = 0):
    """(loss_per_sample, ce [M], argmax [M]) for logits = hidden . weight^T without materialising them."""
    from . import ops
    if not hidden.is_cuda:
        raise _lib.TouchNetB200Error("fused lm_head + loss needs CUDA tensors (no CPU path)")
    return FusedLinearCEFn.apply(hidden, weight, ops.bf16_weight(weight), labels, sentence_lens, float(inv_num_sentence),
                                 chunk or FUSED_CE_CHUNK)


def _handle_loss(pred, labels, sentence_lens, inv_num_sentence: float, detach: bool = False):
    """(loss_per_sample, ce, argmax) of a LazyLogits / VocabParallelLogits handle; keeps (ce, argmax) on it for accuracy().
    detach: statistics only, on detached inputs (the fused pass then computes neither dh nor dW)."""
    if isinstance(pred, LazyLogits):
        h, w = (pred.hidden.detach(), pred.weight.detach()) if detach else (pred.hidden, pred.weight)
        out = fused_linear_cross_entropy(h, w, labels, sentence_lens, inv_num_sentence)
    else:
        local = pred.local.detach() if detach else pred.local
        out = _VocabParallelCEFn.apply(local, labels, sentence_lens, inv_num_sentence, pred.group, pred.v0, pred.v_total)
    pred._stats = out[1:]
    return out


def cross_entropy_loss(pred, labels: torch.Tensor, sentence_lens: torch.Tensor, num_sentence: int,
                       ignore_index: int = -100):
    """Same contract as ref: touchnet/loss/cross_entropy.py:12-50.  Returns (loss_per_sample, loss_per_token).
    `pred` is the model's `pred.logits`: a bf16 [B,T,V] tensor, or a LazyLogits handle (fused lm_head + loss)."""
    assert ignore_index < 0, "labels outside [0, V) are ignored (the reference uses -100)"
    global _LAST_ARGMAX
    inv_num_sentence = 1.0 / max(int(num_sentence), 1)
    if isinstance(pred, (LazyLogits, VocabParallelLogits)):
        loss_per_sample, ce, am = _handle_loss(pred, labels, sentence_lens, inv_num_sentence)
    else:
        loss_per_sample, ce, am = _PackCEFn.apply(pred, labels, sentence_lens, inv_num_sentence)
        _LAST_ARGMAX = (weakref.ref(pred), pred._version, am)
    with torch.no_grad():
        num_tokens = (labels != ignore_index).sum()
        tot = ce.sum()
        loss_per_token = torch.where((tot > 1e-6) & (num_tokens > 0), tot / num_tokens.clamp(min=1), torch.zeros_like(tot))
    return loss_per_sample, loss_per_token


def _masked_accuracy(am: torch.Tensor, labels: torch.Tensor, ignore_index: int) -> torch.Tensor:
    lab = labels.reshape(-1)
    mask = lab != ignore_index
    num = ((am.long() == lab) & mask).sum()
    den = mask.sum()
    return torch.where(den > 0, num / den.clamp(min=1), torch.zeros_like(num, dtype=torch.float32)).detach()


def accuracy(pred: torch.Tensor, labels: torch.Tensor, ignore_index: int = -100) -> torch.Tensor:
    """Same contract as ref: touchnet/utils/metrics.py:26-50; reuses the argmax the loss kernel already produced."""
    if isinstance(pred, (LazyLogits, VocabParallelLogits)):
        if pred._stats is None:        # accuracy asked before / without the loss: one statistics-only pass
            with torch.no_grad():
                ones = torch.ones(labels.numel(), dtype=torch.int64, device=labels.device)
                _handle_loss(pred, labels, ones, 1.0, detach=True)
        return _masked_accuracy(pred._stats[1], labels, ignore_index)
    x = pred.view(-1, pred.shape[-1])
    ent = _LAST_ARGMAX
    if ent is not None and ent[0]() is pred and ent[1] == pred._version and ent[2].numel() == x.shape[0]:
        am = ent[2]
    else:
        am = _pack_ce_fwd(x, labels.reshape(-1).contiguous())[2]
    return _masked_accuracy(am, labels, ignore_index)
