"""GPU: the rowwise FP8 recipe (config key `float8_recipe_name = "rowwise"`): axiswise casts, rowwise GEMM entry
points, the block and the model."""
import copy

import pytest
import torch

import tests.test_gpu_float8 as tw
from tests.gpu_util import packed_doc_ids, rel_err, require_cuda
from tests.test_float8_cpu import recipe_layer
from tests.test_float8_rowwise_cpu import rowwise_recipe_layer, rw_cols, rw_rows
from touchnet_b200 import ops

pytestmark = pytest.mark.gpu


def _same(a, b):
    assert torch.allclose(a, b, rtol=0, atol=0, equal_nan=True)


@pytest.mark.parametrize("shape", [(8192, 3072), (3072, 8192), (48, 80), (32, 8336)])
def test_axiswise_casts_are_bit_exact(shape):
    """Row cast, column amax and column-scaled transposed cast against the torch restatement: a zero row, a NaN that
    poisons one row and one column, shapes that are multiples of 16 but not of 64, and rows longer than the
    register-resident 8192."""
    dev = require_cuda()
    g = torch.Generator(device=dev).manual_seed(0)
    x = (torch.randn(shape, device=dev, generator=g) * 3).bfloat16()
    x[0] = 0
    x[1, :8] = torch.tensor([0.0, -0.0, 1e-30, -1e-30, 1e-8, -1e-8, 3e-6, -7e-7], dtype=torch.bfloat16)
    x[2, 3] = 2.0 ** 60
    x[5, 7] = float("nan")
    q, inv = ops.fp8_rowwise_cast(x)
    rq, s = rw_rows(x)
    tw._same_bits(q, rq)
    _same(inv, (1.0 / s).flatten())
    assert float(inv[0]) == 2.0 ** -48 and torch.isnan(inv[5]) and not torch.isnan(inv[4])
    amax = torch.zeros(shape[1], device=dev)
    ops.fp8_colwise_amax(x, amax)
    _same(amax, x.float().abs().amax(0))
    ops.fp8_colwise_amax(x[:16], amax)           # a second call into the same vector keeps the maxima
    _same(amax, x.float().abs().amax(0))
    qt, invt = ops.fp8_colwise_cast_t(x, amax)
    rq, s = rw_cols(x)
    tw._same_bits(qt, rq.t().contiguous())
    _same(invt, (1.0 / s).flatten())
    assert torch.isnan(invt[7]) and torch.isnan(qt[7].float()).all()


def _operands(M, N, K, seed=0):
    dev = require_cuda()
    g = torch.Generator(device=dev).manual_seed(seed)
    a = torch.randn(M, K, device=dev, generator=g).bfloat16()
    a[:, :K // 16] *= 10                          # columns of outliers: the row scales differ from the tensor's
    # each B row its own power of two, so that the column scales of the product differ from each other
    b = torch.randn(N, K, device=dev, generator=g) * 0.02
    b = (b * torch.exp2(torch.randint(-3, 5, (N, 1), device=dev, generator=g).float())).bfloat16()
    a8, ia = ops.fp8_rowwise_cast(a)
    b8, ib = ops.fp8_rowwise_cast(b)
    return a8, b8, ia, ib


def _reference(a8, b8, ia, ib):
    return (a8.float() @ b8.float().t()) * ia[:, None] * ib[None, :]


def _check(got, a8, b8, ia, ib, fast):
    """bf16 output: within 2x torch._scaled_mm's rowwise error, both against the dequantised fp32 product."""
    ref = _reference(a8, b8, ia, ib)
    sa, sb = ia[:, None].contiguous(), ib[None, :].contiguous()
    sm = torch._scaled_mm(a8, b8.t(), scale_a=sa, scale_b=sb, out_dtype=torch.bfloat16, use_fast_accum=fast)
    e_ours, e_sm = rel_err(got.float(), ref), rel_err(sm.float(), ref)
    assert e_ours <= 2 * e_sm, (e_ours, e_sm)


def _check_f32(got, a8, b8, ia, ib):
    e = rel_err(got, _reference(a8, b8, ia, ib))
    assert e < 1e-3, e


# bench shapes (DESIGN §6: T = 8192, d 3072, q 3072, kv 1024, ffn 8192) and ragged multiples of 16
@pytest.mark.parametrize("M,N,K,promoted,f32", [
    (8192, 3072, 3072, False, False), (8192, 3072, 8192, False, False),        # o fwd, down fwd
    (8192, 8192, 3072, True, False), (8192, 3072, 8192, True, False),          # down dgrad, gate/up dgrad
    (8192, 3072, 3072, True, False),                                           # o dgrad
    (3072, 3072, 8192, True, True), (3072, 8192, 8192, True, True), (8192, 3072, 8192, True, True),   # wgrads
    (8208, 3072, 3088, False, False), (8208, 3072, 3088, True, False), (3088, 1040, 8208, True, True)])
def test_gemm_fp8_rowwise(M, N, K, promoted, f32):
    a8, b8, ia, ib = _operands(M, N, K)
    got = ops.gemm_fp8_rowwise(a8, b8, ia, ib, promoted=promoted, out_f32=f32)
    if f32:
        _check_f32(got, a8, b8, ia, ib)
    else:
        _check(got, a8, b8, ia, ib, fast=not promoted)


@pytest.mark.parametrize("promoted", [False, True])
def test_residual_and_dswiglu_epilogues_match_the_plain_gemm(promoted):
    dev = require_cuda()
    M, N, K = 1040, 784, 528
    a8, b8, ia, ib = _operands(M, N, K)
    r = torch.randn(M, N, device=dev).bfloat16()
    plain = ops.gemm_fp8_rowwise(a8, b8, ia, ib, promoted=promoted)
    fused = ops.gemm_fp8_rowwise(a8, b8, ia, ib, promoted=promoted, residual=r)
    assert torch.equal(fused, (plain.float() + r.float()).bfloat16())
    if promoted:
        g = torch.randn(M, N, device=dev).bfloat16()
        u = torch.randn(M, N, device=dev).bfloat16()
        ops._FUSE_DSWIGLU, old = True, ops._FUSE_DSWIGLU
        try:
            dg, du = ops.gemm_dswiglu_fp8_rowwise(a8, b8, g, u, ia, ib)
        finally:
            ops._FUSE_DSWIGLU = old
        dg2, du2 = ops.swiglu_bwd(g, u, plain)
        assert torch.equal(dg, dg2) and torch.equal(du, du2)


@pytest.mark.parametrize("M", [8192, 1040])
def test_swiglu_rowwise_takes_gate_and_up_scales(M):
    """G / U equal the plain rowwise GEMMs with their own weight scales; H is the bf16 SwiGLU of G and U."""
    dev = require_cuda()
    N, K = 8192 if M == 8192 else 784, 3072 if M == 8192 else 528
    a8, wg8, ia, ig = _operands(M, N, K)
    wu = (torch.randn(N, K, device=dev) * 0.5).bfloat16()       # other magnitudes: other row scales
    wu8, iu = ops.fp8_rowwise_cast(wu)
    g, u, h = ops.gemm_swiglu_fp8_rowwise(a8, wg8, wu8, ia, torch.cat([ig, iu]))
    assert torch.equal(g, ops.gemm_fp8_rowwise(a8, wg8, ia, ig, promoted=False))
    assert torch.equal(u, ops.gemm_fp8_rowwise(a8, wu8, ia, iu, promoted=False))
    _check(g, a8, wg8, ia, ig, fast=True)
    rows = 1024
    eye = torch.eye(rows, device=dev, dtype=torch.bfloat16)
    _, _, h_ref = ops.gemm_swiglu(eye, g[:rows].t().contiguous(), u[:rows].t().contiguous())
    assert torch.equal(h[:rows], h_ref)


@pytest.mark.parametrize("M", [8192, 8208])
def test_qkv_rowwise_three_modes(M):
    dev = require_cuda()
    d, nq, nkv = 3072, 3072, 1024
    tot = nq + 2 * nkv
    h8, w8, ih, iw = _operands(M, tot, d)
    wq, wk, wv = w8[:nq].contiguous(), w8[nq:nq + nkv].contiguous(), w8[nq + nkv:].contiguous()
    qkv = ops.gemm_qkv_fwd_fp8_rowwise(h8, wq, wk, wv, ih, iw)
    _check(qkv, h8, w8, ih, iw, fast=True)
    assert torch.equal(qkv[:, nq:nq + nkv], ops.gemm_fp8_rowwise(h8, wk, ih, iw[nq:nq + nkv], promoted=False))
    pos = torch.arange(M, device=dev) % 2048
    inv = 1.0 / (500000.0 ** (torch.arange(0, 128, 2, device=dev).float() / 128))
    cos, sin = ops.rope_table(pos, inv)
    qkv_r = ops.gemm_qkv_fwd_fp8_rowwise(h8, wq, wk, wv, ih, iw, rope=(cos, sin))
    ref = qkv.clone()
    ops.rope_apply_(ref[:, :nq], cos, sin, nq // 128, 128)
    ops.rope_apply_(ref[:, nq:nq + nkv], cos, sin, nkv // 128, 128)
    assert torch.equal(qkv_r, ref)
    dq8, wt8, idq, iwt = _operands(M, d, tot, seed=1)
    _check(ops.gemm_qkv_dgrad_fp8_rowwise(dq8, wt8, nq, nkv, idq, iwt), dq8, wt8, idq, iwt, fast=False)
    dqt8, ht8, idt, iht = _operands(tot, d, M, seed=2)
    _check_f32(torch.cat(ops.gemm_qkv_wgrad_fp8_rowwise(dqt8, ht8, True, nq, nkv, idt, iht)), dqt8, ht8, idt, iht)


# ---------------------------------------------------------------------------------------------------------------
# the block and the model
# ---------------------------------------------------------------------------------------------------------------
def _run(p, cfg, x, doc, pos, dout, recipe):
    w = {k: v.clone().requires_grad_(True) for k, v in p.items()}
    inv = 1.0 / (cfg.rope_theta ** (torch.arange(0, cfg.head_dim, 2, device=x.device).float() / cfg.head_dim))
    cos, sin = ops.rope_table(pos, inv)
    xb = x.bfloat16().requires_grad_(True)
    out = ops.decoder_layer(xb, w["input_layernorm.weight"], w["self_attn.q_proj.weight"], w["self_attn.k_proj.weight"],
                            w["self_attn.v_proj.weight"], None, None, None, w["self_attn.o_proj.weight"],
                            w["post_attention_layernorm.weight"], w["mlp.gate_proj.weight"], w["mlp.up_proj.weight"],
                            w["mlp.down_proj.weight"], cos, sin, ops.AttnPlan(doc), cfg.num_attention_heads,
                            cfg.num_key_value_heads, cfg.rms_norm_eps, cfg.head_dim, True, float8_recipe_name=recipe)
    out.backward(dout)
    return out, xb.grad, {k: v.grad for k, v in w.items()}


@pytest.fixture(scope="module")
def bench_block():
    """One Llama-3.2-3B-ASR block, T = 4096 packed, init std 0.02, run twice with the rowwise recipe (the first under
    `set_sync_debug_mode("error")`) and once with tensorwise; relative L2 errors of output, dx and every weight
    gradient against the rowwise restatement and against the unquantised fp32 block, and the forward output errors of
    the two recipes' fp32 restatements against that block (no kernel involved)."""
    from oracle import model_oracle as mo
    cfg = tw._bench_cfg()
    p, x, doc, pos, dout = tw._block_inputs(cfg, 1, 4096, [[1500, 700, 1100, 796]])
    torch.cuda.set_sync_debug_mode("error")
    try:
        out, dx, gr = _run(p, cfg, x, doc, pos, dout, "rowwise")
    finally:
        torch.cuda.set_sync_debug_mode(0)
    out2, dx2, gr2 = _run(p, cfg, x, doc, pos, dout, "rowwise")
    repeatable = torch.equal(out, out2) and torch.equal(dx, dx2) and all(torch.equal(gr[k], gr2[k]) for k in gr)
    del out2, dx2, gr2
    inv = 1.0 / (cfg.rope_theta ** (torch.arange(0, 128, 2, device=x.device).float() / 128))
    cos, sin = mo.rope_cos_sin(pos, inv, 1.0, torch.float32)
    v = doc[0] > 0

    def oracle(layer):
        w = {k: t.clone().requires_grad_(True) for k, t in p.items()}
        xr = x.bfloat16().float().requires_grad_(True)
        y = layer(xr, w, "", cfg, cos, sin, mo.doc_causal_allow(doc))
        y.backward(dout.float())
        return y.detach(), xr.grad, {k: t.grad for k, t in w.items()}

    def errs(run, ref):
        (o, d, g), (y, dxr, wr) = run, ref
        e = {"out": rel_err(o.float()[0, v], y[0, v]), "dx": rel_err(d.float()[0, v], dxr[0, v])}
        e.update({k: rel_err(g[k].float(), wr[k]) for k in g})
        return e

    rw_recipe = oracle(rowwise_recipe_layer)
    res = {"repeatable": repeatable, "vs_recipe": errs((out, dx, gr), rw_recipe)}
    exact = oracle(mo.decoder_layer)
    res["rowwise"] = errs((out, dx, gr), exact)
    res["tensorwise"] = errs(tw._run(p, cfg, x, doc, pos, dout, True), exact)
    res["recipe_out"] = {"rowwise": rel_err(rw_recipe[0][0, v], exact[0][0, v]),
                         "tensorwise": rel_err(oracle(recipe_layer)[0][0, v], exact[0][0, v])}
    for k in ("vs_recipe", "rowwise", "tensorwise", "recipe_out"):
        print(k, {n: round(e, 5) for n, e in res[k].items()})
    return res


def test_block_at_bench_geometry_against_the_recipe_and_bitwise_repeatable(bench_block):
    """Within 0.15 of the rowwise restatement; two runs bitwise identical, no host sync in forward + backward."""
    assert bench_block["repeatable"]
    for k, e in bench_block["vs_recipe"].items():
        assert e < 1.5e-1, (k, e)


def test_block_gradients_closer_to_unquantised_than_tensorwise(bench_block):
    """Against the unquantised fp32 block, dx and every weight gradient at most as far off as tensorwise's: rowwise
    gradients carry 3 mantissa bits instead of 2, on finer scales."""
    rw_, tw_ = bench_block["rowwise"], bench_block["tensorwise"]
    for k in rw_:
        if k != "out":
            assert rw_[k] <= tw_[k], (k, rw_[k], tw_[k])


@pytest.mark.xfail(strict=True, reason=(
    "the power-of-two row scales cost more forward (e4m3) rounding error than tensorwise's exact 448/amax: measured on "
    "an H100, output 5.576e-2 against 5.556e-2, and the fp32 restatements of the two recipes, with no kernel, show the "
    "same order on every seed tried (DESIGN §3.5); whether the output bar changes is the recipe owner's decision"))
def test_block_output_closer_to_unquantised_than_tensorwise(bench_block):
    assert bench_block["rowwise"]["out"] <= bench_block["tensorwise"]["out"]


def test_rowwise_model_against_bf16_checkpointing_and_training(monkeypatch):
    """2-layer model (d 1024): first-step loss within 1e-2 of bf16, weight-gradient cosines printed beside tensorwise's;
    checkpoint_wrapper leaves the rowwise block bit-identical; 30 AdamW steps (lr 3e-5) stay within 1.5x the emulated
    rowwise recipe's gap + 1e-2."""
    from types import SimpleNamespace as NS
    from torch.distributed.algorithms._checkpoint.checkpoint_wrapper import checkpoint_wrapper
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

    def first_step(fp8, recipe):
        m = copy.deepcopy(base)
        m.float8_training, m.float8_recipe_name = fp8, recipe
        l0 = loss_of(m)
        l0.backward()
        return m, float(l0), {n: q.grad.detach().clone() for n, q in m.named_parameters() if q.grad is not None}

    _, lb, gb = first_step(False, "tensorwise")
    _, _, gt = first_step(True, "tensorwise")
    m, lr_, gr = first_step(True, "rowwise")
    print(f"loss bf16 {lb:.5f} rowwise {lr_:.5f} rel {abs(lr_ - lb) / abs(lb):.3e}")
    assert abs(lr_ - lb) / abs(lb) < 1e-2
    cos = lambda a, b: float(torch.nn.functional.cosine_similarity(a.flatten().float(), b.flatten().float(), 0))
    names = [n for n in gb if "layers" in n and gb[n].dim() == 2]
    print("weight-gradient cosine vs bf16 (tensorwise, rowwise):",
          {n.split("layers.")[1]: (round(cos(gb[n], gt[n]), 4), round(cos(gb[n], gr[n]), 4)) for n in names})
    # checkpoint_wrapper recomputes the forward in the backward: the same kernels on the same inputs
    mc = copy.deepcopy(base)
    mc.float8_training, mc.float8_recipe_name = True, "rowwise"
    for i, layer in enumerate(mc.model.layers):
        mc.model.layers[i] = checkpoint_wrapper(layer)
    lc = loss_of(mc)
    lc.backward()
    assert float(lc) == lr_
    for n, q in mc.named_parameters():
        key = n.replace("._checkpoint_wrapped_module", "")
        assert torch.equal(q.grad, gr[key]), n
    del mc

    def train(fp8):
        mm = copy.deepcopy(base)
        mm.float8_training, mm.float8_recipe_name = fp8, "rowwise"
        opt = torch.optim.AdamW(mm.parameters(), lr=3e-5)
        hist = []
        for _ in range(30):
            opt.zero_grad(set_to_none=True)
            ops.invalidate_bf16_cache(mm)
            l = loss_of(mm)
            l.backward()
            opt.step()
            hist.append(float(l))
        return hist

    hb, hr = train(False), train(True)
    dev_max = max(abs(a - b) / b for a, b in zip(hr, hb))
    print(f"30 AdamW steps: bf16 {hb[0]:.4f}->{hb[-1]:.4f} rowwise {hr[0]:.4f}->{hr[-1]:.4f} max rel dev {dev_max:.3e}")
    # the same 30 steps in fp32 torch: the oracle against the rowwise restatement (tw._emulated_training runs the
    # module-level `recipe_layer` for its FP8 arm)
    monkeypatch.setattr(tw, "recipe_layer", rowwise_recipe_layer)
    eb, ef = (tw._emulated_training(base, text, ids, doc, pos, tgt, fp8) for fp8 in (False, True))
    emu_dev = max(abs(a - b) / b for a, b in zip(ef, eb))
    print(f"30 AdamW steps, torch emulation: fp32 {eb[0]:.4f}->{eb[-1]:.4f} rowwise recipe {ef[0]:.4f}->{ef[-1]:.4f} "
          f"max rel dev {emu_dev:.3e}")
    assert hr[-1] < hr[0]
    assert dev_max < 1.5 * emu_dev + 1e-2


def test_rowwise_under_fsdp2_matches_single_gpu():
    """FSDP2 on a one-rank mesh with the rowwise recipe: the loss equals the single-GPU run bit for bit."""
    import os
    import subprocess
    import sys
    require_cuda()
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=1", "--master-addr",
           "127.0.0.1", "--master-port", "29571", os.path.join(root, "tools", "check_fsdp_fp8.py"), "--recipe", "rowwise"]
    r = subprocess.run(cmd, cwd=root, capture_output=True, text=True, timeout=600)
    print(r.stdout[-2000:])
    assert r.returncode == 0 and "FSDP FP8 OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]


def test_generate_is_unchanged_by_rowwise():
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
    m.float8_training, m.float8_recipe_name = True, "rowwise"
    assert torch.equal(a, m.generate(ids, max_new_tokens=8, eos_token_id=1, pad_token_id=0))
