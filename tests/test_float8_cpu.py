"""CPU: FP8 training of the decoder block (config key `float8_training`).

- argument checks of the FP8 entry points (no GPU needed: they fail before any CUDA call);
- the wiring of the FP8 DecoderLayerFn, with the CUDA ops replaced by plain-torch stand-ins (tests/cpu_ops_shim.py plus
  the FP8 stand-ins below, which emulate the kernels with torch float8 casts), against an fp32 autograd restatement of
  the recipe (`recipe_layer`, also the oracle of tests/test_gpu_float8.py);
- the switch: config plumbing, unchanged state-dict keys, TP / CP refusal, cached decoding unaffected.
"""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import model_oracle as mo
from touchnet_b200 import _lib, ops

F8E4M3, F8E5M2 = torch.float8_e4m3fn, torch.float8_e5m2
FMAX = {False: 448.0, True: 57344.0}


# ---------------------------------------------------------------------------------------------------------------
# the recipe in torch (shared with the GPU tests)
# ---------------------------------------------------------------------------------------------------------------
def scale_of(amax: torch.Tensor, e5m2: bool) -> torch.Tensor:
    """s = fmax / max(amax, 1e-12) in fp32 (NaN amax -> NaN scale)."""
    return FMAX[e5m2] / amax.float().clamp(min=1e-12)


def quant(x: torch.Tensor, s: torch.Tensor, e5m2: bool) -> torch.Tensor:
    """sat_rne(x · s): torch's own cast turns out-of-range values into NaN, hence the clamp."""
    f = FMAX[e5m2]
    return (x.float() * s).clamp(-f, f).to(F8E5M2 if e5m2 else F8E4M3)


def fake(x: torch.Tensor, amax: torch.Tensor, e5m2: bool) -> torch.Tensor:
    """x quantised at the scale of `amax` and dequantised, in fp32."""
    s = scale_of(amax, e5m2)
    return quant(x, s, e5m2).float() / s


class _F8Linear(torch.autograd.Function):
    """y = x·Wᵀ with x, W e4m3 (W at the scale of `w_amax`, shared by a weight group); dY e5m2 at its own scale.
    The recipe quantises bf16 tensors (the block's activations and gradients are bf16), so x and dY are rounded to bf16
    first."""

    @staticmethod
    def forward(ctx, x, w, w_amax):
        xb = x.detach().bfloat16()
        xq, wq = fake(xb, xb.abs().max(), False), fake(w.detach().bfloat16(), w_amax, False)
        ctx.save_for_backward(xq, wq)
        return xq @ wq.t()

    @staticmethod
    def backward(ctx, dy):
        xq, wq = ctx.saved_tensors
        db = dy.bfloat16()
        dyq = fake(db, db.abs().max(), True)
        return dyq @ wq, dyq.t() @ xq, None


def f8_linear(x, w, w_amax=None):
    lead = x.shape[:-1]
    w_amax = w.detach().abs().max() if w_amax is None else w_amax
    return _F8Linear.apply(x.reshape(-1, x.shape[-1]), w, w_amax).reshape(*lead, w.shape[0])


def recipe_layer(x, p: dict, prefix: str, cfg, cos, sin, allow):
    """oracle decoder_layer with the seven projections through the FP8 recipe (fp32 arithmetic elsewhere): q/k/v as
    one linear over [Wq;Wk;Wv] (one weight scale, one gradient scale), gate and up with one weight scale."""
    B, T, _ = x.shape
    H, KV, hd = cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim
    g = lambda n: p[prefix + n]
    res = x
    h = mo.rms_norm(x, g("input_layernorm.weight"), cfg.rms_norm_eps)
    wqkv = torch.cat([g("self_attn.q_proj.weight"), g("self_attn.k_proj.weight"), g("self_attn.v_proj.weight")])
    qkv = f8_linear(h, wqkv)
    if prefix + "self_attn.q_proj.bias" in p:
        qkv = qkv + torch.cat([g("self_attn.q_proj.bias"), g("self_attn.k_proj.bias"), g("self_attn.v_proj.bias")])
    q, k, v = qkv.split([H * hd, KV * hd, KV * hd], -1)
    q, k, v = (t.reshape(B, T, n, hd).transpose(1, 2) for t, n in ((q, H), (k, KV), (v, KV)))
    q, k = mo.apply_rope(q, k, cos, sin)
    o, _ = mo.attention(q, k, v, allow, hd ** -0.5)
    x = res + f8_linear(o.reshape(B, T, H * hd), g("self_attn.o_proj.weight"))
    res = x
    h = mo.rms_norm(x, g("post_attention_layernorm.weight"), cfg.rms_norm_eps)
    wg, wu = g("mlp.gate_proj.weight"), g("mlp.up_proj.weight")
    gu_amax = torch.maximum(wg.detach().abs().max(), wu.detach().abs().max())
    hm = F.silu(f8_linear(h, wg, gu_amax)) * f8_linear(h, wu, gu_amax)
    return res + f8_linear(hm, g("mlp.down_proj.weight"))


# ---------------------------------------------------------------------------------------------------------------
# plain-torch stand-ins of the FP8 ops (emulate the kernels; record what they are handed)
# ---------------------------------------------------------------------------------------------------------------
class F8Standins:
    def __init__(self):
        self.casts, self.gemms = [], []

    def fp8_amax(self, x, amax):
        amax.copy_(torch.maximum(amax, x.float().abs().max()))

    def fp8_cast(self, x, amax, e5m2, row=True, t=True, inv=None, out=None, out_t=None):
        s = scale_of(amax, e5m2)
        q = quant(x, s, e5m2)
        self.casts.append((tuple(x.shape), e5m2, row, t))
        if row:
            out = q.clone() if out is None else out.copy_(q)
        if t:
            out_t = q.t().contiguous() if out_t is None else out_t.copy_(q.t())
        if inv is not None:
            inv.copy_(1.0 / s)
        return (out if row else None), (out_t if t else None)

    def _mm(self, a, b, inv_a, inv_b, kind):
        assert b.dtype == F8E4M3 and a.dtype in (F8E4M3, F8E5M2)
        self.gemms.append((kind, a.dtype, tuple(a.shape), tuple(b.shape)))
        return (a.float() @ b.float().t()) * (inv_a * inv_b)

    def gemm_fp8(self, a, b, inv_a, inv_b, *, out_f32=False, residual=None, out=None):
        y = self._mm(a, b, inv_a, inv_b, "gemm")
        if residual is not None:
            y = y + residual.float()
        y = y if out_f32 else y.to(torch.bfloat16)
        return y if out is None else out.copy_(y)

    def gemm_swiglu_fp8(self, x, wg, wu, inv_x, inv_w, need_gu=True):
        g = self._mm(x, wg, inv_x, inv_w, "swiglu").to(torch.bfloat16)
        u = self._mm(x, wu, inv_x, inv_w, "swiglu").to(torch.bfloat16)
        h = (F.silu(g.float()) * u.float()).to(torch.bfloat16)
        return g, u, h

    def gemm_qkv_fwd_fp8(self, x, wq, wk, wv, inv_x, inv_w, rope=None):
        nq, nkv = wq.shape[0], wk.shape[0]
        qkv = self._mm(x, torch.cat([wq, wk, wv]), inv_x, inv_w, "qkv0").to(torch.bfloat16)
        if rope is not None:
            ops.rope_apply_(qkv[:, :nq], rope[0], rope[1], nq // 128, 128)
            ops.rope_apply_(qkv[:, nq:nq + nkv], rope[0], rope[1], nkv // 128, 128)
        return qkv

    def gemm_qkv_dgrad_fp8(self, dqkv, w_t, nq, nkv, inv_a, inv_b):
        return self._mm(dqkv, w_t, inv_a, inv_b, "qkv1").to(torch.bfloat16)

    def gemm_qkv_wgrad_fp8(self, dqkv_t, x_t, f32, nq, nkv, inv_a, inv_b):
        d = self._mm(dqkv_t, x_t, inv_a, inv_b, "qkv2")
        d = d if f32 else d.to(torch.bfloat16)
        return list(d.split([nq, nkv, nkv]))

    NAMES = ["fp8_amax", "fp8_cast", "gemm_fp8", "gemm_swiglu_fp8", "gemm_qkv_fwd_fp8", "gemm_qkv_dgrad_fp8",
             "gemm_qkv_wgrad_fp8"]


@pytest.fixture
def shim(monkeypatch):
    from tests import cpu_ops_shim
    saved = cpu_ops_shim.install()
    st = F8Standins()
    for n in F8Standins.NAMES:
        monkeypatch.setattr(ops, n, getattr(st, n))
    yield st
    cpu_ops_shim.uninstall(saved)


def _cfg(d=256, ffn=512, H=2, KV=1, hd=128, bias=False):
    return mo.OracleConfig(d, ffn, 1, H, KV, hd, 64, rms_norm_eps=1e-5, rope_theta=10000.0, attention_bias=bias)


def _params(cfg, seed=0, std=0.05):
    g = torch.Generator().manual_seed(seed)
    d, f, H, KV, hd = cfg.hidden_size, cfg.intermediate_size, cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim
    r = lambda *s: (torch.randn(*s, generator=g) * std)
    p = {"input_layernorm.weight": 1 + 0.1 * torch.randn(d, generator=g),
         "post_attention_layernorm.weight": 1 + 0.1 * torch.randn(d, generator=g),
         "self_attn.q_proj.weight": r(H * hd, d), "self_attn.k_proj.weight": r(KV * hd, d),
         "self_attn.v_proj.weight": r(KV * hd, d), "self_attn.o_proj.weight": r(d, H * hd),
         "mlp.gate_proj.weight": r(f, d), "mlp.up_proj.weight": r(f, d), "mlp.down_proj.weight": r(d, f)}
    if cfg.attention_bias:
        p.update({"self_attn.q_proj.bias": r(H * hd), "self_attn.k_proj.bias": r(KV * hd), "self_attn.v_proj.bias": r(KV * hd)})
    # weights on the bf16 grid: the block computes on bf16 working copies
    return {k: v.bfloat16().float() for k, v in p.items()}


def _run_block(p, cfg, x, doc, pos, fp8=True):
    """DecoderLayerFn (shimmed ops) on fp32 master weights; returns out, dx, grads."""
    from tests import cpu_ops_shim
    B, T, d = x.shape
    w = {k: v.clone().requires_grad_(True) for k, v in p.items()}
    inv = 1.0 / (cfg.rope_theta ** (torch.arange(0, cfg.head_dim, 2).float() / cfg.head_dim))
    cos, sin = cpu_ops_shim.rope_table(pos, inv)
    plan = ops.AttnPlan(doc)
    xb = x.bfloat16().requires_grad_(True)
    b = lambda n: w.get("self_attn." + n + "_proj.bias")
    out = ops.decoder_layer(xb, w["input_layernorm.weight"], w["self_attn.q_proj.weight"], w["self_attn.k_proj.weight"],
                            w["self_attn.v_proj.weight"], b("q"), b("k"), b("v"), w["self_attn.o_proj.weight"],
                            w["post_attention_layernorm.weight"], w["mlp.gate_proj.weight"], w["mlp.up_proj.weight"],
                            w["mlp.down_proj.weight"], cos, sin, plan, cfg.num_attention_heads, cfg.num_key_value_heads,
                            cfg.rms_norm_eps, cfg.head_dim, fp8)
    return out, xb, w


def _reference(p, cfg, x, doc, pos, dout):
    w = {k: v.clone().requires_grad_(True) for k, v in p.items()}
    xr = x.bfloat16().float().requires_grad_(True)
    inv, sc = 1.0 / (cfg.rope_theta ** (torch.arange(0, cfg.head_dim, 2).float() / cfg.head_dim)), 1.0
    cos, sin = mo.rope_cos_sin(pos, inv, sc, torch.float32)
    y = recipe_layer(xr, w, "", cfg, cos, sin, mo.doc_causal_allow(doc))
    y.backward(dout.float())
    return y, xr, w


def _rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / (b.norm() + 1e-30))


@pytest.mark.parametrize("variant", ["llama", "qwen2_bias", "head_dim_64", "fused_qkv"])
def test_fp8_block_wiring_matches_the_recipe(shim, variant, monkeypatch):
    kw = {"qwen2_bias": dict(bias=True), "head_dim_64": dict(H=4, KV=2, hd=64)}.get(variant, {})
    cfg = _cfg(**kw)
    if variant == "fused_qkv":       # the segmented QKV launches (M >= 256, segments of 256) with the RoPE epilogue
        cfg = _cfg(d=256, H=2, KV=2)
        monkeypatch.setattr(ops, "_FUSE_QKV", True)
    p = _params(cfg)
    B, T = 1, 256
    g = torch.Generator().manual_seed(1)
    x = torch.randn(B, T, cfg.hidden_size, generator=g)
    doc = torch.tensor([[1] * 100 + [2] * 120 + [0] * 36])
    pos = torch.cat([torch.arange(100), torch.arange(120), torch.zeros(36, dtype=torch.long)])[None]
    dout = torch.randn(B, T, cfg.hidden_size, generator=g).bfloat16()

    out, xb, w = _run_block(p, cfg, x, doc, pos)
    # saved for backward: the transposed e4m3 copies of h1, o, h2, hm take the place of the bf16 activations
    saved = out.grad_fn.saved_tensors
    d, f, nq = cfg.hidden_size, cfg.intermediate_size, cfg.num_attention_heads * cfg.head_dim
    f8 = sorted(tuple(t.shape) for t in saved if t.dtype == F8E4M3)
    assert f8 == sorted([(d, T), (nq, T), (d, T), (f, T)]), f8
    out.backward(dout)

    # formats: e4m3 for every forward operand (weights row-major only), e5m2 for every incoming gradient
    fwd = [c for c in shim.casts if not c[1]]
    bwd = [c for c in shim.casts if c[1]]
    kv = cfg.num_key_value_heads * cfg.head_dim
    assert sorted(s for s, _, r, t in fwd if r and t) == sorted([(T, d), (T, nq), (T, d), (T, f)])
    assert sorted(s for s, _, r, t in fwd if r and not t) == sorted([(nq, d), (kv, d), (kv, d), (d, nq), (f, d), (f, d), (d, f)])
    assert sorted(s for s, _, r, t in fwd if t and not r) == sorted([(d, f), (f, d), (f, d), (d, nq), (nq, d), (kv, d), (kv, d)])
    assert sorted(s for s, _, r, t in bwd) == sorted([(T, d), (T, f), (T, f), (T, d), (T, nq), (T, kv), (T, kv)])
    assert all(r and t for _, _, r, t in bwd)
    n_fwd = sum(1 for k, dt, _, _ in shim.gemms if dt == F8E4M3)
    n_bwd = sum(1 for k, dt, _, _ in shim.gemms if dt == F8E5M2)
    assert n_fwd == (1 if variant == "fused_qkv" else 3) + 1 + 2 + 1
    assert n_bwd == (2 if variant == "fused_qkv" else 6) + 2 + 4 + 2

    # against the fp32 restatement: the two quantise bf16 tensors that differ in their last bits (bf16 outputs of
    # the kernels vs fp32 arithmetic), and a 2-3 bit mantissa turns such differences into whole-step rounding flips,
    # so the bar sits above that noise and far below what a wrong scale, format or operand would give (O(1))
    y, xr, wr = _reference(p, cfg, x, doc, pos, dout)
    v = (doc > 0)[0]
    assert _rel(out.float()[0, v], y.detach()[0, v]) < 3e-2
    assert _rel(xb.grad.float()[0, v], xr.grad[0, v]) < 6e-2
    # and closer to it than the bf16 block is: the bars alone would also pass a block that skipped the quantisation
    monkeypatch.setattr(ops, "_FUSE_QKV", False)      # the bf16 QKV launches have no stand-in
    ob, xbb, _ = _run_block(p, cfg, x, doc, pos, fp8=False)
    ob.backward(dout)
    assert _rel(out.float()[0, v], y.detach()[0, v]) < _rel(ob.float()[0, v], y.detach()[0, v])
    assert _rel(xb.grad.float()[0, v], xr.grad[0, v]) < _rel(xbb.grad.float()[0, v], xr.grad[0, v])
    for k in p:
        assert _rel(w[k].grad, wr[k].grad) < 1.5e-1, k


def test_shared_scales_cover_the_weight_groups(shim):
    """q/k/v share one weight scale (the max of their amaxes), gate/up another: a group member with a large amax sets
    the scale of the others."""
    cfg = _cfg()
    p = _params(cfg)
    p["self_attn.v_proj.weight"] = p["self_attn.v_proj.weight"] * 8
    p["mlp.up_proj.weight"] = p["mlp.up_proj.weight"] * 8
    x = torch.randn(1, 256, cfg.hidden_size)
    doc, pos = torch.ones(1, 256, dtype=torch.long), torch.arange(256)[None]
    amaxes = []
    orig = shim.fp8_cast
    shim.fp8_cast = lambda x, amax, *a, **k: (amaxes.append((tuple(x.shape), float(amax))), orig(x, amax, *a, **k))[1]
    ops.fp8_cast = shim.fp8_cast
    _run_block(p, cfg, x, doc, pos)
    by = {}
    for s, a in amaxes:
        by.setdefault(s, set()).add(a)
    wq, wk, wv = (p["self_attn." + n + "_proj.weight"].bfloat16() for n in "qkv")
    qkv_amax = float(torch.stack([wq.abs().max(), wk.abs().max(), wv.abs().max()]).max())
    assert by[(512, 256)] == {float(torch.maximum(p["mlp.gate_proj.weight"].bfloat16().abs().max(),
                                                  p["mlp.up_proj.weight"].bfloat16().abs().max()))}
    assert by[(256, 256)] >= {qkv_amax}
    assert by[(128, 256)] == {qkv_amax}


def test_tensor_and_context_parallelism_raise_with_fp8(shim):
    cfg = _cfg()
    p = _params(cfg)
    x = torch.randn(1, 256, cfg.hidden_size)
    doc, pos = torch.ones(1, 256, dtype=torch.long), torch.arange(256)[None]
    for attr in ("tp", "cp_group"):
        orig = ops.AttnPlan

        class _Plan(orig):
            def __init__(self, *a, **k):
                super().__init__(*a, **k)
                setattr(self, attr, object())
        ops.AttnPlan = _Plan
        try:
            with pytest.raises(_lib.TouchNetB200Error, match="float8_training"):
                _run_block(p, cfg, x, doc, pos)
        finally:
            ops.AttnPlan = orig


def test_dimensions_not_multiple_of_16_raise(shim):
    cfg = _cfg()
    p = _params(cfg)
    x = torch.randn(1, 200, cfg.hidden_size)
    doc, pos = torch.ones(1, 200, dtype=torch.long), torch.arange(200)[None]
    _run_block(p, cfg, torch.randn(1, 192, cfg.hidden_size), doc[:, :192], pos[:, :192])
    with pytest.raises(_lib.TouchNetB200Error, match="multiples of 16"):
        _run_block(p, cfg, x[:, :200 - 4], doc[:, :196], pos[:, :196])


# ---------------------------------------------------------------------------------------------------------------
# entry points: argument checks (before any CUDA call)
# ---------------------------------------------------------------------------------------------------------------
def test_fp8_entry_points_reject_bad_arguments():
    p = ctypes.c_void_p(256)
    q = ctypes.c_void_p(264)       # 8 B aligned only
    bad_calls = [
        ("tn_gemm_fp8", (None, 256, 0, p, 256, p, 256, 0, None, 0, 256, 256, 256, p, p, None), "null"),
        ("tn_gemm_fp8", (p, 256, 0, p, 256, p, 256, 0, None, 0, 256, 256, 256, None, p, None), "null"),
        ("tn_gemm_fp8", (p, 256, 0, p, 256, p, 256, 0, None, 0, 256, 256, 264, p, p, None), "multiples of 16"),
        ("tn_gemm_fp8", (p, 264, 0, p, 256, p, 256, 0, None, 0, 256, 256, 256, p, p, None), "16 B aligned"),
        ("tn_gemm_fp8", (q, 256, 0, p, 256, p, 256, 0, None, 0, 256, 256, 256, p, p, None), "16 B aligned"),
        ("tn_gemm_fp8", (p, 256, 0, p, 256, q, 256, 0, None, 0, 256, 256, 256, p, p, None), "D/R"),
        ("tn_gemm_swiglu_fp8", (p, 256, 0, p, None, 256, p, p, p, 256, 256, 256, 256, p, p, None), "null"),
        ("tn_gemm_swiglu_fp8", (p, 256, 0, p, p, 256, p, p, p, 256, 256, 256, 200, p, p, None), "multiples of 16"),
        ("tn_gemm_dswiglu_fp8", (p, 256, 1, p, 256, p, p, 256, p, p, 256, 256, 256, 8, p, p, None), "multiples of 16"),
        ("tn_gemm_dswiglu_fp8", (p, 256, 1, p, 256, p, p, 256, p, p, 256, 128, 256, 256, p, p, None), ">= 256"),
        ("tn_gemm_qkv_fp8", (1, p, 768, 1, p, p, p, 768, p, None, None, 256, 0, 256, 256, 256, 256, 256, 760, None,
                             None, p, p, None), "multiples of 16"),
        ("tn_gemm_qkv_fp8", (0, p, 256, 0, p, p, p, 256, p, None, None, 768, 0, 256, 128, 256, 256, 640, 256, None,
                             None, p, p, None), "multiples of 256"),
        ("tn_gemm_qkv_fp8", (2, p, 256, 1, p, None, None, 256, p, None, None, 256, 1, 256, 256, 256, 768, 256, 256,
                             None, None, p, p, None), "D1/D2"),
        ("tn_fp8_amax_bf16", (None, 256, 256, 256, p, None), "null"),
        ("tn_fp8_amax_bf16", (p, 256, 256, 200, p, None), "multiples of 16"),
        ("tn_fp8_cast_bf16", (p, 256, 256, 256, 0, p, None, 0, None, 0, None, None), "null"),
        ("tn_fp8_cast_bf16", (p, 256, 250, 256, 0, p, p, 256, None, 0, None, None), "multiples of 16"),
        ("tn_fp8_cast_bf16", (q, 256, 256, 256, 0, p, p, 256, None, 0, None, None), "aligned"),
        ("tn_fp8_cast_bf16", (p, 256, 256, 256, 0, p, p, 248, None, 0, None, None), "ld_out"),
        ("tn_fp8_cast_bf16", (p, 256, 256, 256, 1, p, None, 0, q, 256, None, None), "out_t"),
    ]
    for name, args, needle in bad_calls:
        with pytest.raises(_lib.TouchNetB200Error, match=needle):
            _lib.call(name, *args)


def test_fp8_gemm_wrappers_reject_operand_types():
    a = torch.zeros(16, 16, dtype=F8E4M3)
    inv = torch.ones(())
    with pytest.raises(_lib.TouchNetB200Error, match="e5m2 B"):
        ops.gemm_fp8(a, torch.zeros(16, 16, dtype=F8E5M2), inv, inv)
    with pytest.raises(_lib.TouchNetB200Error, match="A operand"):
        ops.gemm_fp8(torch.zeros(16, 16, dtype=torch.bfloat16), a, inv, inv)
    with pytest.raises(_lib.TouchNetB200Error, match="e5m2 B"):
        ops.gemm_swiglu_fp8(a, torch.zeros(16, 16, dtype=F8E5M2), a, inv, inv)


# ---------------------------------------------------------------------------------------------------------------
# the switch
# ---------------------------------------------------------------------------------------------------------------
class _NS:
    def __init__(self, **kw):
        self.__dict__.update(kw)


def _text(**kw):
    return _NS(hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=2, num_key_value_heads=1,
               head_dim=128, vocab_size=64, rms_norm_eps=1e-5, rope_theta=10000.0, rope_scaling=None,
               attention_bias=False, tie_word_embeddings=False, initializer_range=0.02, model_type="llama",
               pad_token_id=0, **kw)


def test_config_key_is_plumbed_and_state_dict_unchanged():
    from touchnet_b200 import modeling
    off = modeling.B200LlamaForCausalLM(_text())
    on = modeling.B200LlamaForCausalLM(_text(float8_training=True))
    assert off.float8_training is False and on.float8_training is True
    assert list(on.state_dict()) == list(off.state_dict())
    assert [n for n, _ in on.named_buffers()] == [n for n, _ in off.named_buffers()]
    ta = modeling.B200TouchAudioForCausalLM(_NS(audio_config=_NS(input_size=40), text_config=_text(), pad_token_id=0,
                                                float8_training=True))
    assert ta.float8_training and ta.language_model.float8_training and ta.language_model.model.float8_training
    ta.float8_training = False
    assert not ta.language_model.model.float8_training
    ta2 = modeling.B200TouchAudioForCausalLM(_NS(audio_config=_NS(input_size=40), text_config=_text(float8_training=True),
                                                 pad_token_id=0))
    assert ta2.float8_training
    ref = modeling.B200TouchAudioForCausalLM(_NS(audio_config=_NS(input_size=40), text_config=_text(), pad_token_id=0))
    assert list(ta.state_dict()) == list(ref.state_dict())


def test_layers_receive_the_switch(monkeypatch):
    """Every decoder block gets fp8=model.float8_training; cached decoding (generation.py) calls block_forward
    without it."""
    from touchnet_b200 import modeling
    import inspect
    from touchnet_b200 import generation
    seen = []
    monkeypatch.setattr(ops, "decoder_layer", lambda *a, **k: (seen.append(a[-1] if len(a) > 20 else k.get("fp8")), a[0])[1])
    monkeypatch.setattr(ops, "AttnPlan", lambda doc: _NS(tp=None, cp_group=None))
    m = modeling.B200LlamaForCausalLM(_text(float8_training=True))
    m.model.rotary_emb.forward = lambda pos: (None, None)
    m.model.norm.forward = lambda x: x
    m.model(torch.zeros(1, 16, 256, dtype=torch.bfloat16), torch.ones(1, 16, dtype=torch.long), None)
    assert seen == [True, True]
    assert "fp8" not in inspect.getsource(generation)


def test_generate_is_the_same_with_the_switch_on(monkeypatch):
    """Cached decoding never takes the FP8 path: generate returns the same tensor with the switch on and off (the FP8
    stand-ins are not installed, so an FP8 call would fail)."""
    import tests.test_generation_cpu as tg
    from tests import cpu_ops_shim
    saved = cpu_ops_shim.install()
    monkeypatch.setattr(ops, "attn_decode", tg._attn_decode)
    monkeypatch.setattr(ops, "kv_append", tg._kv_append)
    monkeypatch.setattr(ops, "greedy_select", tg._greedy_select)
    try:
        _, ours = tg._models(seed=4)
        ids, mask = tg._prompt()
        off = ours.generate(ids, attention_mask=mask, max_new_tokens=6, eos_token_id=63, **tg._REF_KW)
        ours.float8_training = True
        on = ours.generate(ids, attention_mask=mask, max_new_tokens=6, eos_token_id=63, **tg._REF_KW)
    finally:
        cpu_ops_shim.uninstall(saved)
    assert torch.equal(on, off)
