"""GPU parity: fused pack-loss cross-entropy / accuracy vs the reference formulas (torch fp32 on the same bf16 logits).
ref: touchnet/loss/cross_entropy.py:12-50, touchnet/utils/metrics.py:26-50.  Tolerances: loss rel 1e-4;
dlogits max err <= 2^-8 relative to the row scale (bf16 output); accuracy / argmax exact."""
import pytest
import torch
import torch.nn.functional as F

from tests.gpu_util import require_cuda
from touchnet_b200 import loss as tl

pytestmark = pytest.mark.gpu


def ref_loss(pred, labels, sentence_lens, num_sentence):
    B = pred.shape[0]
    ce = F.cross_entropy(pred.flatten(0, 1).float(), labels.flatten(0, 1), reduction="none", ignore_index=-100)
    num_tokens = (labels != -100).sum()
    lpt = ce.sum() / num_tokens if (ce.sum() > 1e-6 and num_tokens > 0) else torch.zeros_like(ce.sum())
    lps = torch.sum(torch.sum(ce.reshape(B, -1) / sentence_lens, dim=-1)) / num_sentence
    return lps, lpt


@pytest.mark.parametrize("B,T,V", [(2, 256, 1000), (1, 512, 128256), (3, 77, 156032), (2, 64, 1003)])
def test_pack_ce_matches_reference(B, T, V):
    dev = require_cuda()
    torch.manual_seed(B * T + V)
    if V % 8 != 0:
        base = torch.randn(B, T, V + (8 - V % 8), device=dev).bfloat16()
        logits = base[..., :V]                                       # row stride stays 16-byte aligned, V has a tail
    else:
        logits = (torch.randn(B, T, V, device=dev) * 2).bfloat16()
    labels = torch.randint(0, V, (B, T), device=dev)
    labels[:, -T // 4:] = -100
    labels[0, :3] = -100
    sl = torch.randint(1, 50, (B, T), device=dev)
    ns = 7
    lg_ref = logits.detach().float().requires_grad_(True)
    lps_ref, lpt_ref = ref_loss(lg_ref, labels, sl, ns)
    lps_ref.backward()
    acc_ref = ((lg_ref.argmax(-1) == labels) & (labels != -100)).sum() / (labels != -100).sum()

    lg = logits.detach().clone().requires_grad_(True) if V % 8 == 0 else logits.detach().requires_grad_(True)
    lps, lpt = tl.cross_entropy_loss(lg, labels, sl, ns)
    acc = tl.accuracy(lg, labels)
    assert abs(float(lps) - float(lps_ref)) <= 1e-4 * abs(float(lps_ref)) + 1e-6
    assert abs(float(lpt) - float(lpt_ref)) <= 1e-4 * abs(float(lpt_ref)) + 1e-6
    assert float(acc) == pytest.approx(float(acc_ref), abs=1e-7)
    (lps * 3.0).backward()
    g, g_ref = lg.grad.float(), lg_ref.grad * 3.0
    scale = g_ref.abs().amax(dim=-1, keepdim=True).clamp(min=1e-12)
    assert float(((g - g_ref).abs() / scale).max()) <= 2 ** -7
    assert torch.all(g[labels == -100] == 0)


def test_argmax_ties_pick_first_like_torch():
    dev = require_cuda()
    logits = torch.zeros(1, 4, 1024, device=dev, dtype=torch.bfloat16)
    logits[0, 0, 5] = 1; logits[0, 0, 900] = 1        # tie: torch.argmax returns the first
    logits[0, 1, 1023] = 3
    labels = torch.tensor([[5, 1023, 0, -100]], device=dev)
    acc = tl.accuracy(logits, labels)
    assert float(acc) == pytest.approx(float(((logits.float().argmax(-1) == labels) & (labels != -100)).sum() / 3))


@pytest.mark.parametrize("M,d,V,chunk,master", [(3000, 512, 128256, 1024, torch.float32), (2500, 256, 156032, 1024, torch.bfloat16),
                                               (700, 256, 1003, 256, torch.float32)])
def test_fused_linear_cross_entropy_matches_pack_loss_oracle(M, d, V, chunk, master):
    """Fused lm_head + pack-loss (no [M,V] logits: chunked GEMM -> tn_pack_ce_fused_bf16 -> dgrad / accumulating wgrad) vs
    the oracle's pack_loss on fp32 logits of the same bf16 operands (ref: touchnet/loss/cross_entropy.py:12-50), at the
    vocabularies of BASELINE cfg 2 (128256) and cfg 3 (156032) and at one that is not a multiple of 8; several chunks with
    a ragged last one.  Tolerances: loss rel 2e-4 (bf16 logits), dh / dW relative L2 < 1.5e-2 (bf16 dlogits), argmax exact
    wherever the fp32 top-2 margin exceeds the bf16 rounding of the logits."""
    from oracle import model_oracle as mo
    dev = require_cuda()
    torch.manual_seed(M + V)
    h = (torch.randn(M, d, device=dev) * 1.0).bfloat16()
    w = (torch.randn(V, d, device=dev) * 0.05).to(master)
    labels = torch.randint(0, V, (M,), device=dev)
    labels[-M // 5:] = -100
    labels[:2] = -100
    sl = torch.randint(1, 40, (M,), device=dev)
    ns = 11
    hp = h.detach().clone().requires_grad_(True)
    wp = w.detach().clone().requires_grad_(True)
    lps, ce, am = tl.fused_linear_cross_entropy(hp, wp, labels, sl, 1.0 / ns, chunk=chunk)
    (lps * 2.0).backward()
    # oracle: fp32 logits of the bf16-rounded operands
    hr = h.float().requires_grad_(True)
    wr = w.bfloat16().float().requires_grad_(True)
    logits = hr @ wr.t()
    ref = mo.pack_loss(logits, labels, sl, ns)
    (ref * 2.0).backward()
    assert abs(float(lps) - float(ref)) <= 2e-4 * abs(float(ref)) + 1e-6, (float(lps), float(ref))
    rel = lambda a, b: float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))
    assert rel(hp.grad.float(), hr.grad) < 1.5e-2, rel(hp.grad.float(), hr.grad)
    assert wp.grad.dtype == master
    assert rel(wp.grad.float(), wr.grad) < 1.5e-2, rel(wp.grad.float(), wr.grad)
    assert torch.all(hp.grad[labels == -100] == 0)
    top2 = logits.detach().topk(2, dim=-1).values
    decisive = (top2[:, 0] - top2[:, 1]) > 2 ** -6 * top2[:, 0].abs() + 1e-3
    assert torch.equal(am.long()[decisive], logits.detach().argmax(-1)[decisive])
    ce_ref = torch.nn.functional.cross_entropy(logits.detach(), labels, reduction="none", ignore_index=-100)
    assert float((ce - ce_ref).abs().max()) < 3e-2


def test_lazy_logits_route_through_loss_and_accuracy_like_real_logits():
    """The "*_b200" specs' model returns a LazyLogits handle in training mode; loss_fn / acc_fn (ref: train.py:447-450)
    give what they give on materialised logits, and parameter gradients agree (same kernels, chunked accumulation)."""
    from types import SimpleNamespace as NS
    from touchnet_b200 import modeling
    from tests.gpu_util import packed_doc_ids, rel_err
    dev = require_cuda()
    cfg = NS(hidden_size=256, intermediate_size=512, num_hidden_layers=1, num_attention_heads=2, num_key_value_heads=1,
             head_dim=128, vocab_size=5000, rms_norm_eps=1e-5, rope_theta=500000.0, rope_scaling=None, attention_bias=False,
             tie_word_embeddings=False, initializer_range=0.02, model_type="llama", pad_token_id=0)
    B, T = 2, 384
    doc, pos = packed_doc_ids(B, T, [[100, 200, 50], [384]], dev)
    torch.manual_seed(3)
    ids = torch.randint(1, cfg.vocab_size, (B, T), device=dev)
    labels = torch.randint(0, cfg.vocab_size, (B, T), device=dev)
    labels[doc == 0] = -100
    sl = torch.ones(B, T, dtype=torch.int64, device=dev) * 7

    def run(fused):
        torch.manual_seed(2025)
        m = modeling.B200LlamaForCausalLM(cfg).to(dev)
        m.post_init()
        with torch.no_grad():
            for p in m.parameters():
                if p.dim() == 2:
                    p.normal_(0, 0.05)
        m.fused_linear_ce = fused
        m.train()
        pred = m(input_ids=ids, attention_mask=doc, position_ids=pos)
        assert isinstance(pred.logits, tl.LazyLogits) == fused
        if fused:
            assert tuple(pred.logits.shape) == (B, T, cfg.vocab_size)
        lps, lpt = tl.cross_entropy_loss(pred.logits, labels, sl, 5)
        acc = tl.accuracy(pred.logits, labels)
        lps.backward()
        return float(lps), float(lpt), float(acc), {n: p.grad.float().clone() for n, p in m.named_parameters()}

    l0, t0, a0, g0 = run(False)
    l1, t1, a1, g1 = run(True)
    assert abs(l0 - l1) <= 1e-5 * abs(l0) and abs(t0 - t1) <= 1e-5 * abs(t0) and a0 == a1
    for n in g0:
        assert rel_err(g1[n], g0[n]) < 2e-3, (n, rel_err(g1[n], g0[n]))
    # eval mode / no_grad: real logits come back (dev loop, generation)
    m = modeling.B200LlamaForCausalLM(cfg).to(dev)
    m.post_init()
    m.fused_linear_ce = True
    m.eval()
    with torch.no_grad():
        assert isinstance(m(input_ids=ids, attention_mask=doc, position_ids=pos).logits, torch.Tensor)
    # the Liger-route contract: shift_labels in, pred.loss out (token mean), logits None
    m.train()
    pred = m(input_ids=ids, attention_mask=doc, position_ids=pos, shift_labels=labels)
    assert pred.logits is None
    ref = torch.nn.functional.cross_entropy(m.eval()(input_ids=ids, attention_mask=doc, position_ids=pos).logits.float()
                                            .view(-1, cfg.vocab_size), labels.view(-1), ignore_index=-100)
    assert abs(float(pred.loss) - float(ref)) <= 2e-3 * abs(float(ref))


def _ce_rows(M, V, seed):
    """bf16 logits [M, V] on a 16-byte aligned row stride, labels with ignored rows and one row of equal logits (argmax
    ties), random sentence lengths."""
    dev = require_cuda()
    g = torch.Generator(device=dev).manual_seed(seed)
    ld = (V + 7) // 8 * 8
    x = (torch.randn(M, ld, device=dev, generator=g) * 2).bfloat16()[:, :V]
    x[3] = 0.5
    labels = torch.randint(0, V, (M,), device=dev, generator=g)
    labels[-M // 5:] = -100
    labels[:2] = -100
    sl = torch.randint(1, 50, (M,), device=dev, generator=g)
    return x, labels, sl


def _bits(t):
    return t.view({torch.bfloat16: torch.int16, torch.float32: torch.int32}.get(t.dtype, t.dtype))


@pytest.mark.parametrize("M,V", [(4096, 128256), (1000, 156032), (700, 1003)])
def test_fused_ce_kernel_is_bit_identical_to_the_two_pass_kernels(M, V):
    """tn_pack_ce_fused_bf16 = tn_pack_ce_fwd_bf16 then tn_pack_ce_bwd_bf16 at an upstream gradient of 1: the same lse,
    ce, argmax and logit gradient, bit for bit."""
    from touchnet_b200 import _lib
    x, labels, sl = _ce_rows(M, V, M + V)
    scale = 1.0 / 7
    st = torch.cuda.current_stream().cuda_stream
    out = []
    for fused in (True, False):
        xi = torch.empty(M, x.stride(0), dtype=x.dtype, device=x.device)[:, :V].copy_(x)
        lse = torch.empty(M, dtype=torch.float32, device=x.device)
        ce = torch.empty_like(lse)
        am = torch.empty(M, dtype=torch.int32, device=x.device)
        if fused:
            _lib.call("tn_pack_ce_fused_bf16", xi.data_ptr(), xi.stride(0), labels.data_ptr(), sl.data_ptr(),
                      lse.data_ptr(), ce.data_ptr(), am.data_ptr(), scale, M, V, st)
        else:
            one = torch.ones(1, dtype=torch.float32, device=x.device)
            _lib.call("tn_pack_ce_fwd_bf16", xi.data_ptr(), xi.stride(0), labels.data_ptr(), lse.data_ptr(),
                      ce.data_ptr(), am.data_ptr(), M, V, st)
            _lib.call("tn_pack_ce_bwd_bf16", xi.data_ptr(), xi.stride(0), labels.data_ptr(), sl.data_ptr(),
                      lse.data_ptr(), one.data_ptr(), scale, M, V, st)
        out.append((lse, ce, am, xi))
    assert int(out[0][2][3]) == 0                                   # the equal row: first index wins
    for name, a, b in zip(("lse", "ce", "argmax", "dlogits"), *out):
        assert torch.equal(_bits(a), _bits(b)), name


@pytest.mark.parametrize("M,bounds", [(600, (0, 40000, 85000, 128256)), (500, (0, 256, 1003)),
                                      (300, (0, 8, 4096, 9000, 12347))])
def test_vocab_parallel_bwd_shards_equal_the_full_bwd(M, bounds):
    """tn_pack_ce_bwd_vp_bf16 on each column slice [v0, v1) of a row (global labels, the full row's lse) writes exactly
    what tn_pack_ce_bwd_bf16 writes into those columns of the full row; labels in other shards and ignored rows included."""
    from touchnet_b200 import _lib
    V = bounds[-1]
    x, labels, sl = _ce_rows(M, V, M + len(bounds))
    labels[5], labels[6], labels[7] = bounds[1], bounds[1] - 1, V - 1       # labels on shard edges
    st = torch.cuda.current_stream().cuda_stream
    lse = torch.empty(M, dtype=torch.float32, device=x.device)
    ce = torch.empty_like(lse)
    _lib.call("tn_pack_ce_fwd_bf16", x.data_ptr(), x.stride(0), labels.data_ptr(), lse.data_ptr(), ce.data_ptr(), None,
              M, V, st)
    g = torch.full((1,), 3.0, dtype=torch.float32, device=x.device)
    full = torch.empty(M, x.stride(0), dtype=x.dtype, device=x.device)[:, :V].copy_(x)
    _lib.call("tn_pack_ce_bwd_bf16", full.data_ptr(), full.stride(0), labels.data_ptr(), sl.data_ptr(), lse.data_ptr(),
              g.data_ptr(), 0.2, M, V, st)
    shards = torch.empty(M, x.stride(0), dtype=x.dtype, device=x.device)[:, :V].copy_(x)
    for v0, v1 in zip(bounds[:-1], bounds[1:]):
        xs = shards[:, v0:v1]
        _lib.call("tn_pack_ce_bwd_vp_bf16", xs.data_ptr(), xs.stride(0), labels.data_ptr(), sl.data_ptr(), lse.data_ptr(),
                  g.data_ptr(), 0.2, M, v1 - v0, v0, V, st)
    assert torch.equal(_bits(shards), _bits(full))
    assert torch.all(full[labels == -100] == 0)
