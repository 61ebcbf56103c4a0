"""GPU: FP8 quantisation kernels, FP8 GEMM entry points and the FP8 decoder block (config key `float8_training`)."""
import math

import pytest
import torch

from tests.gpu_util import packed_doc_ids, rel_err, require_cuda
from tests.test_float8_cpu import F8E4M3, F8E5M2, quant, recipe_layer, scale_of
from touchnet_b200 import ops

pytestmark = pytest.mark.gpu


def _amax_cast(x, e5m2):
    amax = torch.zeros((), device=x.device)
    inv = torch.zeros((), device=x.device)
    ops.fp8_amax(x, amax)
    q, qt = ops.fp8_cast(x, amax, e5m2, inv=inv)
    return amax, inv, q, qt


def _same_bits(a, b):
    """bitwise equal, NaN positions equal (NaN encodings may differ in sign)"""
    na, nb = torch.isnan(a.float()), torch.isnan(b.float())
    assert torch.equal(na, nb)
    assert torch.equal(a.view(torch.uint8)[~na], b.view(torch.uint8)[~nb])


@pytest.mark.parametrize("e5m2", [False, True])
@pytest.mark.parametrize("shape", [(8192, 3072), (3072, 8192), (48, 80)])
def test_amax_and_cast_are_bit_exact(e5m2, shape):
    dev = require_cuda()
    g = torch.Generator(device=dev).manual_seed(0)
    x = (torch.randn(shape, device=dev, generator=g) * 3).bfloat16()
    # saturation, ±0, subnormals of the target format after scaling, and a few large outliers
    x.view(-1)[:8] = torch.tensor([0.0, -0.0, 1e-30, -1e-30, 1e-8, -1e-8, 3e-6, -7e-7], dtype=torch.bfloat16)
    amax, inv, q, qt = _amax_cast(x, e5m2)
    ref_amax = x.float().abs().max()
    assert float(amax) == float(ref_amax)
    s = scale_of(ref_amax, e5m2)
    ref = quant(x, s, e5m2)
    _same_bits(q, ref)
    _same_bits(qt, ref.t().contiguous())
    assert float(inv) == float(torch.reciprocal(s))
    # a second call into the same amax with a larger tensor raises it; a fixed amax saturates the rest
    small = torch.zeros((), device=dev); small.fill_(float(ref_amax) / 4)
    q2, _ = ops.fp8_cast(x, small, e5m2, t=False)
    _same_bits(q2, quant(x, scale_of(small, e5m2), e5m2))
    # NaN stays NaN (and poisons the scale, as in the torch restatement)
    xn = x.clone()
    xn[3, 5] = float("nan")
    amax_n, inv_n, qn, qnt = _amax_cast(xn, e5m2)
    assert math.isnan(float(amax_n))
    assert torch.isnan(quant(xn, scale_of(amax_n, e5m2), e5m2).float()).all()
    assert torch.isnan(qn.float()).all() and torch.isnan(qnt.float()).all()


def _operands(M, N, K, a_e5m2, seed=0):
    dev = require_cuda()
    g = torch.Generator(device=dev).manual_seed(seed)
    a = torch.randn(M, K, device=dev, generator=g).bfloat16()
    b = (torch.randn(N, K, device=dev, generator=g) * 0.02).bfloat16()
    _, ia, a8, _ = _amax_cast(a, a_e5m2)
    _, ib, b8, _ = _amax_cast(b, False)
    return a8, b8, ia, ib


def _check_vs_references(got, a8, b8, ia, ib, fast, bar_floor=1e-3):
    ref = (a8.float() @ b8.float().t()) * (ia * ib)
    sm = torch._scaled_mm(a8, b8.t(), scale_a=ia.reshape(1).float(), scale_b=ib.reshape(1).float(),
                          out_dtype=torch.float32, use_fast_accum=fast)
    e_ours, e_sm = rel_err(got.float(), ref), rel_err(sm, ref)
    assert e_ours <= 2 * e_sm + bar_floor, (e_ours, e_sm)
    return e_ours, e_sm


@pytest.mark.parametrize("M,N,K,a_e5m2", [(8192, 8192, 3072, True), (3072, 3072, 8192, True), (8192, 3072, 8192, False)])
def test_gemm_fp8_matches_dequantised_matmul_and_scaled_mm(M, N, K, a_e5m2):
    """down dgrad 8192x8192x3072 and o_proj wgrad 3072x3072x8192 promoted (e5m2 A), a forward shape fast."""
    a8, b8, ia, ib = _operands(M, N, K, a_e5m2)
    got = ops.gemm_fp8(a8, b8, ia, ib, out_f32=True)
    _check_vs_references(got, a8, b8, ia, ib, fast=not a_e5m2)


def test_swiglu_fp8_forward_shape_and_fused_epilogue():
    """gate/up forward 8192x16384x3072 (M x 2·ffn x K): G / U against the references; H bitwise equal to the bf16
    SwiGLU applied to those G / U (the epilogue's rounding points)."""
    M, N, K = 8192, 8192, 3072
    dev = require_cuda()
    a8, wg8, ia, iw = _operands(M, N, K, False)
    wu8 = (wg8.float() * -0.5).to(F8E4M3)
    g, u, h = ops.gemm_swiglu_fp8(a8, wg8, wu8, ia, iw)
    _check_vs_references(g, a8, wg8, ia, iw, fast=True, bar_floor=4e-3)   # + bf16 rounding of G
    gp = ops.gemm_fp8(a8, wg8, ia, iw, out_f32=True)
    up = ops.gemm_fp8(a8, wu8, ia, iw, out_f32=True)
    assert torch.equal(g, gp.bfloat16()) and torch.equal(u, up.bfloat16())
    # H: the bf16 SwiGLU epilogue applied to G and U.  An identity X makes the bf16 launch's accumulator exactly G / U
    # (one non-zero product per sum), so its H is the epilogue on those values, bit for bit.
    rows = 1024
    eye = torch.eye(rows, device=dev, dtype=torch.bfloat16)
    _, _, h_ref = ops.gemm_swiglu(eye, g[:rows].t().contiguous(), u[:rows].t().contiguous())
    assert torch.equal(h[:rows], h_ref)


def test_residual_and_dswiglu_epilogues_match_the_plain_gemm():
    dev = require_cuda()
    M, N, K = 1024, 768, 512
    a8, b8, ia, ib = _operands(M, N, K, True)
    r = torch.randn(M, N, device=dev).bfloat16()
    plain = ops.gemm_fp8(a8, b8, ia, ib)
    fused = ops.gemm_fp8(a8, b8, ia, ib, residual=r)
    assert torch.equal(fused, (plain.float() + r.float()).bfloat16())
    g = torch.randn(M, N, device=dev).bfloat16()
    u = torch.randn(M, N, device=dev).bfloat16()
    ops._FUSE_DSWIGLU, old = True, ops._FUSE_DSWIGLU
    try:
        dg, du = ops.gemm_dswiglu_fp8(a8, b8, g, u, ia, ib)
    finally:
        ops._FUSE_DSWIGLU = old
    dg2, du2 = ops.swiglu_bwd(g, u, plain)
    assert torch.equal(dg, dg2) and torch.equal(du, du2)


@pytest.mark.parametrize("M,N,K,a_e5m2", [(8208, 3072, 3072, False), (8208, 3072, 3088, True), (3072, 3072, 8208, True),
                                           (3088, 1040, 8208, True)])
def test_gemm_fp8_ragged_shapes(M, N, K, a_e5m2):
    """Multiples of 16 that are not multiples of 128: a partial 128-k stage (TMA zero fill) and partial M / N tiles."""
    a8, b8, ia, ib = _operands(M, N, K, a_e5m2)
    _check_vs_references(ops.gemm_fp8(a8, b8, ia, ib, out_f32=True), a8, b8, ia, ib, fast=not a_e5m2)


def test_qkv_fp8_ragged_rows():
    """The QKV launches at B·T = 8208: forward and dgrad with a partial M tile, wgrad with a partial 128-k stage."""
    M, d, nq, nkv = 8208, 3072, 3072, 1024
    tot = nq + 2 * nkv
    h8, w8, ih, iw = _operands(M, tot, d, False)
    qkv = ops.gemm_qkv_fwd_fp8(h8, w8[:nq].contiguous(), w8[nq:nq + nkv].contiguous(), w8[nq + nkv:].contiguous(), ih, iw)
    _check_vs_references(qkv, h8, w8, ih, iw, fast=True, bar_floor=4e-3)
    dq8, wt8, idq, iwt = _operands(M, d, tot, True, seed=1)
    _check_vs_references(ops.gemm_qkv_dgrad_fp8(dq8, wt8, nq, nkv, idq, iwt), dq8, wt8, idq, iwt, fast=False,
                         bar_floor=4e-3)
    dqt8, ht8, idt, iht = _operands(tot, d, M, True, seed=2)
    dws = ops.gemm_qkv_wgrad_fp8(dqt8, ht8, True, nq, nkv, idt, iht)
    _check_vs_references(torch.cat(dws), dqt8, ht8, idt, iht, fast=False)


def test_qkv_fp8_three_modes():
    dev = require_cuda()
    M, d, nq, nkv = 8192, 3072, 3072, 1024
    tot = nq + 2 * nkv
    h8, w8, ih, iw = _operands(M, tot, d, False)
    wq, wk, wv = w8[:nq], w8[nq:nq + nkv], w8[nq + nkv:]
    qkv = ops.gemm_qkv_fwd_fp8(h8, wq.contiguous(), wk.contiguous(), wv.contiguous(), ih, iw)
    _check_vs_references(qkv, h8, w8, ih, iw, fast=True, bar_floor=4e-3)
    # RoPE epilogue: bitwise equal to the plain launch followed by the rope kernel
    pos = torch.arange(M, device=dev) % 2048
    inv = 1.0 / (500000.0 ** (torch.arange(0, 128, 2, device=dev).float() / 128))
    cos, sin = ops.rope_table(pos, inv)
    qkv_r = ops.gemm_qkv_fwd_fp8(h8, wq.contiguous(), wk.contiguous(), wv.contiguous(), ih, iw, rope=(cos, sin))
    ref = qkv.clone()
    ops.rope_apply_(ref[:, :nq], cos, sin, nq // 128, 128)
    ops.rope_apply_(ref[:, nq:nq + nkv], cos, sin, nkv // 128, 128)
    assert torch.equal(qkv_r, ref)
    # dgrad: dqkv [M, tot] e5m2 x Wᵀ [d, tot]
    dq8, wt8, idq, iwt = _operands(M, d, tot, True, seed=1)
    dx = ops.gemm_qkv_dgrad_fp8(dq8, wt8, nq, nkv, idq, iwt)
    _check_vs_references(dx, dq8, wt8, idq, iwt, fast=False, bar_floor=4e-3)
    # wgrad: dqkvᵀ [tot, M] e5m2 x h1ᵀ [d, M]
    dqt8, ht8, idt, iht = _operands(tot, d, M, True, seed=2)
    dws = ops.gemm_qkv_wgrad_fp8(dqt8, ht8, True, nq, nkv, idt, iht)
    _check_vs_references(torch.cat(dws), dqt8, ht8, idt, iht, fast=False)


# ---------------------------------------------------------------------------------------------------------------
# the block and the model
# ---------------------------------------------------------------------------------------------------------------
def _block_inputs(cfg, B, T, lens, seed=0):
    from tests.test_float8_cpu import _params
    dev = require_cuda()
    p = {k: v.to(dev) for k, v in _params(cfg, seed, std=0.02).items()}   # the models' initializer_range
    g = torch.Generator(device=dev).manual_seed(seed + 1)
    x = torch.randn(B, T, cfg.hidden_size, device=dev, generator=g)
    doc, pos = packed_doc_ids(B, T, lens, dev)
    dout = torch.randn(B, T, cfg.hidden_size, device=dev, generator=g).bfloat16()
    return p, x, doc, pos, dout


def _run(p, cfg, x, doc, pos, dout, fp8):
    from touchnet_b200.modeling import B200RotaryEmbedding  # noqa: F401  (rope tables via the kernel)
    w = {k: v.clone().requires_grad_(True) for k, v in p.items()}
    inv = 1.0 / (cfg.rope_theta ** (torch.arange(0, cfg.head_dim, 2, device=x.device).float() / cfg.head_dim))
    cos, sin = ops.rope_table(pos, inv)
    plan = ops.AttnPlan(doc)
    xb = x.bfloat16().requires_grad_(True)
    out = ops.decoder_layer(xb, w["input_layernorm.weight"], w["self_attn.q_proj.weight"], w["self_attn.k_proj.weight"],
                            w["self_attn.v_proj.weight"], None, None, None, w["self_attn.o_proj.weight"],
                            w["post_attention_layernorm.weight"], w["mlp.gate_proj.weight"], w["mlp.up_proj.weight"],
                            w["mlp.down_proj.weight"], cos, sin, plan, cfg.num_attention_heads,
                            cfg.num_key_value_heads, cfg.rms_norm_eps, cfg.head_dim, fp8)
    out.backward(dout)
    return out, xb.grad, {k: v.grad for k, v in w.items()}


def _bench_cfg():
    from tests.test_float8_cpu import _cfg
    return _cfg(d=3072, ffn=8192, H=24, KV=8, hd=128)


def test_block_at_bench_geometry_against_the_recipe_and_bitwise_repeatable():
    """One Llama-3.2-3B-ASR block on a packed row of documents: output, dx and every weight gradient against the fp32
    restatement of the recipe, closer than the bf16 block is; two runs bitwise identical; no host sync in forward +
    backward.  T = 4096 keeps the dense fp32 attention of the restatement within memory."""
    from oracle import model_oracle as mo
    cfg = _bench_cfg()
    T = 4096
    lens = [[1500, 700, 1100, 796]]
    p, x, doc, pos, dout = _block_inputs(cfg, 1, T, lens)
    torch.cuda.set_sync_debug_mode("error")
    try:
        out, dx, gr = _run(p, cfg, x, doc, pos, dout, True)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    out2, dx2, gr2 = _run(p, cfg, x, doc, pos, dout, True)
    assert torch.equal(out, out2) and torch.equal(dx, dx2)
    for k in gr:
        assert torch.equal(gr[k], gr2[k]), k
    w = {k: v.clone().requires_grad_(True) for k, v in p.items()}
    xr = x.bfloat16().float().requires_grad_(True)
    inv = 1.0 / (cfg.rope_theta ** (torch.arange(0, 128, 2, device=x.device).float() / 128))
    cos, sin = mo.rope_cos_sin(pos, inv, 1.0, torch.float32)
    v = doc[0] > 0
    y = recipe_layer(xr, w, "", cfg, cos, sin, mo.doc_causal_allow(doc))
    y.backward(dout.float())
    def errs_of(out, dx, gr):
        e = {"out": rel_err(out.float()[0, v], y.detach()[0, v]), "dx": rel_err(dx.float()[0, v], xr.grad[0, v])}
        e.update({k: rel_err(gr[k].float(), w[k].grad) for k in gr})
        return e

    errs = errs_of(out, dx, gr)
    errs_bf16 = errs_of(*_run(p, cfg, x, doc, pos, dout, False))
    print("fp8 block vs recipe:", {k: round(e, 4) for k, e in errs.items()})
    print("bf16 block vs recipe:", {k: round(e, 4) for k, e in errs_bf16.items()})
    # the recipe's quantisation is what the FP8 block reproduces and the bf16 block does not
    assert errs["out"] < errs_bf16["out"] and errs["dx"] < errs_bf16["dx"]
    for k, e in errs.items():
        assert e < 1.5e-1, (k, e)


def test_fp8_model_against_bf16_loss_gradients_and_training():
    """2-layer model: loss within 1e-2 of bf16 and weight-gradient cosine > 0.97; 30 AdamW steps on a fixed packed
    batch: both losses fall and FP8 stays within 10 % of bf16 (the measured values are in the asserts' comments)."""
    from types import SimpleNamespace as NS
    from touchnet_b200 import modeling
    dev = require_cuda()
    text = NS(hidden_size=1024, intermediate_size=4096, num_hidden_layers=2, num_attention_heads=8, num_key_value_heads=2,
              head_dim=128, vocab_size=2048, rms_norm_eps=1e-5, rope_theta=500000.0, rope_scaling=None,
              attention_bias=False, tie_word_embeddings=False, initializer_range=0.02, model_type="llama", pad_token_id=0)
    torch.manual_seed(0)
    base = modeling.B200LlamaForCausalLM(text).to(dev)
    base.post_init()
    B, T = 1, 2048
    g = torch.Generator().manual_seed(3)
    ids = torch.randint(1, 2048, (B, T), generator=g).to(dev)
    doc, pos = packed_doc_ids(B, T, [[700, 500, 848]], dev)
    tgt = torch.roll(ids, -1, 1)

    def loss_of(m):
        logits = m(input_ids=ids, attention_mask=doc, position_ids=pos).logits.float()
        return torch.nn.functional.cross_entropy(logits.view(-1, logits.shape[-1]), tgt.view(-1))

    import copy
    runs = {}
    for fp8 in (False, True):
        m = copy.deepcopy(base)
        m.float8_training = fp8
        l0 = loss_of(m)
        l0.backward()
        grads = {n: q.grad.detach().clone() for n, q in m.named_parameters() if q.grad is not None}
        opt = torch.optim.AdamW(m.parameters(), lr=3e-5)   # at 3e-4 both runs memorise the batch (loss ~3e-3)
        hist = []
        for _ in range(30):
            opt.zero_grad(set_to_none=True)
            ops.invalidate_bf16_cache(m)
            l = loss_of(m)
            l.backward()
            opt.step()
            hist.append(float(l))
        runs[fp8] = (float(l0), grads, hist)
    (lb, gb, hb), (lf, gf, hf) = runs[False], runs[True]
    print(f"loss bf16 {lb:.5f} fp8 {lf:.5f} rel {abs(lf - lb) / abs(lb):.3e}")
    assert abs(lf - lb) / abs(lb) < 1e-2
    coss = {n: float(torch.nn.functional.cosine_similarity(gb[n].flatten().float(), gf[n].flatten().float(), 0))
            for n in gb if "layers" in n and gb[n].dim() == 2}
    print("weight-gradient cosine fp8 vs bf16:", {n.split("layers.")[1]: round(c, 4) for n, c in coss.items()})
    # e5m2 keeps 2 mantissa bits: each quantised gradient carries ~4 % relative noise per element, which bounds the
    # cosine of the smallest-signal weights (measured minimum 0.978 on an H100)
    assert min(coss.values()) > 0.97
    dev_max = max(abs(a - b) / b for a, b in zip(hf, hb))
    print(f"30 AdamW steps: bf16 {hb[0]:.4f}->{hb[-1]:.4f} fp8 {hf[0]:.4f}->{hf[-1]:.4f} max rel dev {dev_max:.3e}")
    assert hb[-1] < hb[0] and hf[-1] < hf[0]
    # the same 30 steps in torch: the fp32 oracle against the fp32 restatement of the recipe (recipe_layer).  The gap
    # between those two is what the recipe itself costs on this batch, with no kernel involved (measured: 8.9 %).
    eb, ef = (_emulated_training(base, text, ids, doc, pos, tgt, fp8) for fp8 in (False, True))
    emu_dev = max(abs(a - b) / b for a, b in zip(ef, eb))
    print(f"30 AdamW steps, torch emulation: fp32 {eb[0]:.4f}->{eb[-1]:.4f} recipe {ef[0]:.4f}->{ef[-1]:.4f} "
          f"max rel dev {emu_dev:.3e}")
    assert dev_max < 1.5 * emu_dev + 1e-2
    # measured on an H100: 9.0 % at step 30 (bf16 7.843 -> 1.524, FP8 7.842 -> 1.661), with the first-step losses 1.7e-4
    # apart; 2 % was not met.  The torch emulation below shows the same gap without any kernel.
    assert dev_max < 1e-1


def _emulated_training(base, text, ids, doc, pos, tgt, fp8, steps=30):
    """30 AdamW steps (lr 3e-5) of the 2-layer model in fp32 torch: oracle layers, or recipe_layer for fp8."""
    import torch.nn.functional as F
    from oracle import model_oracle as mo
    cfg = mo.OracleConfig(text.hidden_size, text.intermediate_size, text.num_hidden_layers, text.num_attention_heads,
                          text.num_key_value_heads, text.head_dim, text.vocab_size, rms_norm_eps=text.rms_norm_eps,
                          rope_theta=text.rope_theta)
    p = {k: v.detach().clone().float().requires_grad_(True) for k, v in base.state_dict().items()
         if "rotary" not in k}
    cos, sin = mo.rope_cos_sin(pos, base.model.rotary_emb.inv_freq, 1.0, torch.float32)
    allow = mo.doc_causal_allow(doc)
    layer = recipe_layer if fp8 else mo.decoder_layer
    opt = torch.optim.AdamW(list(p.values()), lr=3e-5)
    hist = []
    for _ in range(steps):
        opt.zero_grad(set_to_none=True)
        x = F.embedding(ids, p["model.embed_tokens.weight"])
        for i in range(cfg.num_hidden_layers):
            x = layer(x, p, f"model.layers.{i}.", cfg, cos, sin, allow)
        logits = F.linear(mo.rms_norm(x, p["model.norm.weight"], cfg.rms_norm_eps), p["lm_head.weight"])
        l = F.cross_entropy(logits.view(-1, logits.shape[-1]), tgt.view(-1))
        l.backward()
        opt.step()
        hist.append(float(l))
    return hist


@pytest.mark.parametrize("nproc", [1, 2])
def test_fp8_under_fsdp2_matches_single_gpu(nproc):
    """FSDP2 with bf16 all-gather (nproc = 1: a one-rank mesh, still the bf16-parameter path): each rank's loss equals
    the single-GPU FP8 run on its row bit for bit, the reduced gradients agree to bf16 rounding."""
    import os
    import subprocess
    import sys
    if torch.cuda.device_count() < nproc:
        pytest.skip(f"needs {nproc} GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}", "--master-addr",
           "127.0.0.1", "--master-port", str(29561 + nproc), os.path.join(root, "tools", "check_fsdp_fp8.py")]
    r = subprocess.run(cmd, cwd=root, capture_output=True, text=True, timeout=600)
    print(r.stdout[-2000:])
    assert r.returncode == 0 and "FSDP FP8 OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]


def test_generate_is_unchanged_by_the_switch():
    from types import SimpleNamespace as NS
    from touchnet_b200 import modeling
    dev = require_cuda()
    text = NS(hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=2, num_key_value_heads=1,
              head_dim=128, vocab_size=320, rms_norm_eps=1e-5, rope_theta=500000.0, rope_scaling=None,
              attention_bias=False, tie_word_embeddings=False, initializer_range=0.02, model_type="llama", pad_token_id=0)
    torch.manual_seed(0)
    m = modeling.B200LlamaForCausalLM(text).to(dev)
    m.post_init()
    ids = torch.randint(3, 320, (2, 40), device=dev)
    a = m.generate(ids, max_new_tokens=8, eos_token_id=1, pad_token_id=0)
    m.float8_training = True
    b = m.generate(ids, max_new_tokens=8, eos_token_id=1, pad_token_id=0)
    assert torch.equal(a, b)
