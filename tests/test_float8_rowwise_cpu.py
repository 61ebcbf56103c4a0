"""CPU: the rowwise FP8 recipe of the decoder block (config key `float8_recipe_name = "rowwise"`).

- the scale rule: s = 448 / max(amax, 1e-12) (fp64 division, fp32 result) rounded down to a power of two;
- `rowwise_recipe_layer`, an fp32 autograd restatement of the recipe (also the oracle of
  tests/test_gpu_float8_rowwise.py), pinned by hand-computed cases and the operand table of DESIGN §3.5;
- the wiring of the rowwise DecoderLayerFn with plain-torch stand-ins of the rowwise kernels, against the restatement;
- the switch: config plumbing, refusals, the tensorwise default, cached decoding unaffected;
- argument checks of the rowwise entry points (no GPU needed: they fail before any CUDA call).
"""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from oracle import model_oracle as mo
from tests.test_float8_cpu import F8E4M3, F8Standins, _cfg, _params, _rel, _text, _NS, quant
from touchnet_b200 import _lib, ops


# ---------------------------------------------------------------------------------------------------------------
# the recipe in torch (shared with the GPU tests)
# ---------------------------------------------------------------------------------------------------------------
def rw_scale(amax: torch.Tensor) -> torch.Tensor:
    """torchao's amax_to_scale for e4m3 (fp64 division, fp32 result) rounded down to a power of two."""
    s = (448.0 / amax.double().clamp(min=1e-12)).float()
    return torch.exp2(torch.floor(torch.log2(s)))


def rw_rows(x: torch.Tensor):
    """(e4m3 copy, scale [rows, 1]) with one scale per row of x."""
    s = rw_scale(x.float().abs().amax(1, keepdim=True))
    return quant(x, s, False), s


def rw_cols(x: torch.Tensor):
    """(e4m3 copy, scale [1, cols]) with one scale per column of x."""
    s = rw_scale(x.float().abs().amax(0, keepdim=True))
    return quant(x, s, False), s


def fake_rows(x):
    q, s = rw_rows(x)
    return q.float() / s


def fake_cols(x):
    q, s = rw_cols(x)
    return q.float() / s


class _RWLinear(torch.autograd.Function):
    """y = x·Wᵀ, dX = dY·W, dW = dYᵀ·X with every operand e4m3 and scaled along that GEMM's reduction axis: x and dY
    per row for y and dX, W per row for y and per column for dX, dY and x per column for dW."""

    @staticmethod
    def forward(ctx, x, w):
        xb, wb = x.detach().bfloat16(), w.detach().bfloat16()
        ctx.save_for_backward(xb, wb)
        return fake_rows(xb) @ fake_rows(wb).t()

    @staticmethod
    def backward(ctx, dy):
        xb, wb = ctx.saved_tensors
        db = dy.bfloat16()
        return fake_rows(db) @ fake_cols(wb), fake_cols(db).t() @ fake_cols(xb)


def rw_linear(x, w):
    lead = x.shape[:-1]
    return _RWLinear.apply(x.reshape(-1, x.shape[-1]), w).reshape(*lead, w.shape[0])


def rowwise_recipe_layer(x, p: dict, prefix: str, cfg, cos, sin, allow):
    """oracle decoder_layer with the seven projections through the rowwise recipe: q/k/v as one linear over [Wq;Wk;Wv]
    (the dq|dk|dv row scale and the Wᵀ column scale span the three, as in the fused QKV dgrad)."""
    B, T, _ = x.shape
    H, KV, hd = cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim
    g = lambda n: p[prefix + n]
    res = x
    h = mo.rms_norm(x, g("input_layernorm.weight"), cfg.rms_norm_eps)
    qkv = rw_linear(h, torch.cat([g("self_attn.q_proj.weight"), g("self_attn.k_proj.weight"),
                                  g("self_attn.v_proj.weight")]))
    if prefix + "self_attn.q_proj.bias" in p:
        qkv = qkv + torch.cat([g("self_attn.q_proj.bias"), g("self_attn.k_proj.bias"), g("self_attn.v_proj.bias")])
    q, k, v = qkv.split([H * hd, KV * hd, KV * hd], -1)
    q, k, v = (t.reshape(B, T, n, hd).transpose(1, 2) for t, n in ((q, H), (k, KV), (v, KV)))
    q, k = mo.apply_rope(q, k, cos, sin)
    o, _ = mo.attention(q, k, v, allow, hd ** -0.5)
    x = res + rw_linear(o.reshape(B, T, H * hd), g("self_attn.o_proj.weight"))
    res = x
    h = mo.rms_norm(x, g("post_attention_layernorm.weight"), cfg.rms_norm_eps)
    hm = F.silu(rw_linear(h, g("mlp.gate_proj.weight"))) * rw_linear(h, g("mlp.up_proj.weight"))
    return res + rw_linear(hm, g("mlp.down_proj.weight"))


def test_scale_rule_hand_computed():
    amax = torch.tensor([1.0, 0.0, 448.0, 3.5, 1.75, 2.0, 3.0, float("nan"), float("inf")])
    s = rw_scale(amax)
    # 448 -> 256; 448e12 -> 2^48; 1 (exact); 128 and 256 exact powers of two stay; 224 -> 128; 149.3 -> 128
    assert s[:7].tolist() == [256.0, 2.0 ** 48, 1.0, 128.0, 256.0, 128.0, 128.0]
    assert torch.isnan(s[7]) and s[8] == 0
    # the kernel's rounding (clear the fp32 mantissa) gives the same scale for every positive finite bf16 amax
    bits = torch.arange(1, 0x7F80, dtype=torch.int32).to(torch.int16).view(torch.bfloat16)
    s = rw_scale(bits.float())
    raw = (448.0 / bits.double().clamp(min=1e-12)).float()
    assert torch.equal((raw.view(torch.int32) & 0x7F800000).view(torch.float32), s)
    # x · s is exact: the quantised value times 1/s is x wherever x is representable at that scale
    x = torch.tensor([[1.5, -0.75, 0.0, 448.0 / 256]]).bfloat16()
    q, s = rw_rows(x)
    assert float(s) == 256.0 and torch.equal(q.float() / s, x.float())


def test_power_of_two_scales_cost_e4m3_rounding_error():
    """The reason the rowwise forward is not closer to the unquantised block than tensorwise (DESIGN §3.5): both
    quantise the forward to e4m3, and rounding a row's scale down to a power of two leaves its amax in [224, 448]
    instead of at 448, so the row's values keep their own binade positions instead of being spread over e4m3's
    range. On unit-RMS rows (RMSNorm outputs) that costs more relative error than the exact row scale, and more than
    one exact scale for the whole tensor, whose rows here are alike."""
    g = torch.Generator().manual_seed(0)
    x = torch.randn(1024, 3072, generator=g).bfloat16()
    amax = x.float().abs().amax(1, keepdim=True)

    def err(s):
        return float((quant(x, s, False).float() / s - x.float()).norm() / x.float().norm())

    e_pow2, e_exact = err(rw_scale(amax)), err((448.0 / amax.double()).float())
    e_tensor = err(448.0 / x.float().abs().max())
    assert e_pow2 > e_exact and e_pow2 > e_tensor, (e_pow2, e_exact, e_tensor)


def test_axiswise_wrappers_check_their_tensors():
    x = torch.zeros(32, 48, dtype=torch.bfloat16)
    with pytest.raises(_lib.TouchNetB200Error, match="unit inner stride"):
        ops.fp8_colwise_amax(x.t(), torch.zeros(32))
    with pytest.raises(_lib.TouchNetB200Error, match="bfloat16"):
        ops.fp8_rowwise_cast(x.float())
    for bad in (torch.zeros(47), torch.zeros(48, dtype=torch.float64), torch.zeros(96)[::2], torch.zeros(1, 48)):
        with pytest.raises(_lib.TouchNetB200Error, match="contiguous float32 vector of 48"):
            ops.fp8_colwise_amax(x, bad)
        with pytest.raises(_lib.TouchNetB200Error, match="contiguous float32 vector of 48"):
            ops.fp8_colwise_cast_t(x, bad)
    with pytest.raises(_lib.TouchNetB200Error, match="inv must be a contiguous float32 vector of 32"):
        ops.fp8_rowwise_cast(x, inv=torch.zeros(48))
    with pytest.raises(_lib.TouchNetB200Error, match="out_t must be float8_e4m3fn"):
        ops.fp8_colwise_cast_t(x, torch.zeros(48), out_t=torch.zeros(32, 48, dtype=F8E4M3))
    with pytest.raises(_lib.TouchNetB200Error, match="CUDA"):
        ops.fp8_colwise_amax(x, torch.zeros(48))


def test_restatement_uses_the_operand_table():
    """dX = dY·W with dY scaled per row and W per column (over out); dW = dYᵀ·X with both per column (over tokens)."""
    g = torch.Generator().manual_seed(0)
    x = torch.randn(32, 48, generator=g).bfloat16().float().requires_grad_(True)
    w = (torch.randn(64, 48, generator=g) * 0.05).bfloat16().float().requires_grad_(True)
    dy = torch.randn(32, 64, generator=g).bfloat16()
    x[3].data.mul_(100)            # one large token row: only its own row scale moves in the forward
    y = rw_linear(x, w)
    y.backward(dy.float())
    xb, wb = x.detach().bfloat16(), w.detach().bfloat16()
    assert torch.equal(y, fake_rows(xb) @ fake_rows(wb).t())
    assert torch.equal(x.grad, fake_rows(dy) @ fake_cols(wb))
    assert torch.equal(w.grad, fake_cols(dy).t() @ fake_cols(xb))
    q, s = rw_rows(xb)
    assert float(s[3]) < float(s[2])


# ---------------------------------------------------------------------------------------------------------------
# plain-torch stand-ins of the rowwise ops (emulate the kernels; record what they are handed)
# ---------------------------------------------------------------------------------------------------------------
class RWStandins:
    def __init__(self):
        self.casts, self.gemms = [], []

    def fp8_rowwise_cast(self, x, out=None, inv=None):
        q, s = rw_rows(x)
        self.casts.append(("row", tuple(x.shape)))
        out = q.clone() if out is None else out.copy_(q)
        inv = (1.0 / s).flatten() if inv is None else inv.copy_((1.0 / s).flatten())
        return out, inv

    def fp8_colwise_amax(self, x, amax):
        amax.copy_(torch.maximum(amax, x.float().abs().amax(0)))

    def fp8_colwise_cast_t(self, x, amax, out_t=None, inv=None):
        s = rw_scale(amax)[None, :]
        q = quant(x, s, False)
        self.casts.append(("col_t", tuple(x.shape)))
        out_t = q.t().contiguous() if out_t is None else out_t.copy_(q.t())
        inv = (1.0 / s).flatten() if inv is None else inv.copy_((1.0 / s).flatten())
        return out_t, inv

    def _mm(self, a, b, inv_a, inv_b, kind, promoted):
        assert a.dtype == F8E4M3 and b.dtype == F8E4M3
        assert inv_a.shape == (a.shape[0],) and inv_b.shape == (b.shape[0],), (inv_a.shape, a.shape, inv_b.shape, b.shape)
        self.gemms.append((kind, promoted, tuple(a.shape), tuple(b.shape), inv_a.clone(), inv_b.clone()))
        return (a.float() @ b.float().t()) * inv_a[:, None] * inv_b[None, :]

    def gemm_fp8_rowwise(self, a, b, inv_a, inv_b, *, promoted, out_f32=False, residual=None, out=None):
        y = self._mm(a, b, inv_a, inv_b, "gemm", promoted)
        if residual is not None:
            y = y + residual.float()
        y = y if out_f32 else y.to(torch.bfloat16)
        return y if out is None else out.copy_(y)

    def gemm_swiglu_fp8_rowwise(self, x, wg, wu, inv_x, inv_w, need_gu=True):
        N = wg.shape[0]
        g = self._mm(x, wg, inv_x, inv_w[:N], "swiglu", False).to(torch.bfloat16)
        u = self._mm(x, wu, inv_x, inv_w[N:], "swiglu", False).to(torch.bfloat16)
        return g, u, (F.silu(g.float()) * u.float()).to(torch.bfloat16)

    def gemm_qkv_fwd_fp8_rowwise(self, x, wq, wk, wv, inv_x, inv_w, rope=None):
        nq, nkv = wq.shape[0], wk.shape[0]
        qkv = self._mm(x, torch.cat([wq, wk, wv]), inv_x, inv_w, "qkv0", False).to(torch.bfloat16)
        if rope is not None:
            ops.rope_apply_(qkv[:, :nq], rope[0], rope[1], nq // 128, 128)
            ops.rope_apply_(qkv[:, nq:nq + nkv], rope[0], rope[1], nkv // 128, 128)
        return qkv

    def gemm_qkv_dgrad_fp8_rowwise(self, dqkv, w_t, nq, nkv, inv_a, inv_b):
        return self._mm(dqkv, w_t, inv_a, inv_b, "qkv1", True).to(torch.bfloat16)

    def gemm_qkv_wgrad_fp8_rowwise(self, dqkv_t, x_t, f32, nq, nkv, inv_a, inv_b):
        d = self._mm(dqkv_t, x_t, inv_a, inv_b, "qkv2", True)
        return list((d if f32 else d.to(torch.bfloat16)).split([nq, nkv, nkv]))

    NAMES = ["fp8_rowwise_cast", "fp8_colwise_amax", "fp8_colwise_cast_t", "gemm_fp8_rowwise", "gemm_swiglu_fp8_rowwise",
             "gemm_qkv_fwd_fp8_rowwise", "gemm_qkv_dgrad_fp8_rowwise", "gemm_qkv_wgrad_fp8_rowwise"]


def _forbid(monkeypatch, names):
    def boom(*a, **k):
        raise AssertionError("called an op of the other recipe")
    for n in names:
        monkeypatch.setattr(ops, n, boom)


@pytest.fixture
def shim(monkeypatch):
    from tests import cpu_ops_shim
    saved = cpu_ops_shim.install()
    st = RWStandins()
    for n in RWStandins.NAMES:
        monkeypatch.setattr(ops, n, getattr(st, n))
    _forbid(monkeypatch, F8Standins.NAMES)          # no tensorwise op may run under the rowwise recipe
    yield st
    cpu_ops_shim.uninstall(saved)


def _run_block(p, cfg, x, doc, pos, fp8=True, recipe="rowwise"):
    from tests import cpu_ops_shim
    w = {k: v.clone().requires_grad_(True) for k, v in p.items()}
    inv = 1.0 / (cfg.rope_theta ** (torch.arange(0, cfg.head_dim, 2).float() / cfg.head_dim))
    cos, sin = cpu_ops_shim.rope_table(pos, inv)
    xb = x.bfloat16().requires_grad_(True)
    b = lambda n: w.get("self_attn." + n + "_proj.bias")
    out = ops.decoder_layer(xb, w["input_layernorm.weight"], w["self_attn.q_proj.weight"], w["self_attn.k_proj.weight"],
                            w["self_attn.v_proj.weight"], b("q"), b("k"), b("v"), w["self_attn.o_proj.weight"],
                            w["post_attention_layernorm.weight"], w["mlp.gate_proj.weight"], w["mlp.up_proj.weight"],
                            w["mlp.down_proj.weight"], cos, sin, ops.AttnPlan(doc), cfg.num_attention_heads,
                            cfg.num_key_value_heads, cfg.rms_norm_eps, cfg.head_dim, fp8, float8_recipe_name=recipe)
    return out, xb, w


def _inputs(cfg, T=256):
    g = torch.Generator().manual_seed(1)
    x = torch.randn(1, T, cfg.hidden_size, generator=g)
    doc = torch.tensor([[1] * 100 + [2] * 120 + [0] * (T - 220)])
    pos = torch.cat([torch.arange(100), torch.arange(120), torch.zeros(T - 220, dtype=torch.long)])[None]
    dout = torch.randn(1, T, cfg.hidden_size, generator=g).bfloat16()
    return x, doc, pos, dout


@pytest.mark.parametrize("variant", ["llama", "qwen2_bias", "head_dim_64", "fused_qkv"])
def test_rowwise_block_wiring_matches_the_recipe(shim, variant, monkeypatch):
    kw = {"qwen2_bias": dict(bias=True), "head_dim_64": dict(H=4, KV=2, hd=64)}.get(variant, {})
    cfg = _cfg(**kw)
    if variant == "fused_qkv":       # the segmented QKV launches (M >= 256, segments of 256) with the RoPE epilogue
        cfg = _cfg(d=256, H=2, KV=2)
        monkeypatch.setattr(ops, "_FUSE_QKV", True)
    p = _params(cfg)
    x, doc, pos, dout = _inputs(cfg)
    T = x.shape[1]
    out, xb, w = _run_block(p, cfg, x, doc, pos)
    # saved for backward: the column-scaled transposed e4m3 copies of h1, o, h2, hm
    d, f, nq = cfg.hidden_size, cfg.intermediate_size, cfg.num_attention_heads * cfg.head_dim
    f8 = sorted(tuple(t.shape) for t in out.grad_fn.saved_tensors if t.dtype == F8E4M3)
    assert f8 == sorted([(d, T), (nq, T), (d, T), (f, T)]), f8
    out.backward(dout)
    # every forward GEMM accumulates fast, every backward GEMM promotes
    fused = variant == "fused_qkv"
    n_fwd = sum(1 for _, pr, *_ in shim.gemms if not pr)
    n_bwd = sum(1 for _, pr, *_ in shim.gemms if pr)
    assert n_fwd == (1 if fused else 3) + 1 + 2 + 1
    assert n_bwd == (2 if fused else 6) + 2 + 4 + 2

    y, xr, wr = _reference(p, cfg, x, doc, pos, dout)
    v = (doc > 0)[0]
    assert _rel(out.float()[0, v], y.detach()[0, v]) < 3e-2
    assert _rel(xb.grad.float()[0, v], xr.grad[0, v]) < 6e-2
    for k in p:
        assert _rel(w[k].grad, wr[k].grad) < 1.5e-1, k


def _reference(p, cfg, x, doc, pos, dout):
    w = {k: v.clone().requires_grad_(True) for k, v in p.items()}
    xr = x.bfloat16().float().requires_grad_(True)
    inv = 1.0 / (cfg.rope_theta ** (torch.arange(0, cfg.head_dim, 2).float() / cfg.head_dim))
    cos, sin = mo.rope_cos_sin(pos, inv, 1.0, torch.float32)
    y = rowwise_recipe_layer(xr, w, "", cfg, cos, sin, mo.doc_causal_allow(doc))
    y.backward(dout.float())
    return y, xr, w


@pytest.mark.parametrize("fused", [False, True])
def test_dqkv_rows_share_one_scale(shim, fused, monkeypatch):
    """The QKV dgrad's A is [dq|dk|dv] with one scale per token row over all three, and Wᵀ one scale per input
    feature over the stacked [Wq;Wk;Wv]; fused and unfused launches hand the same vectors in."""
    cfg = _cfg(d=256, H=2, KV=2)
    monkeypatch.setattr(ops, "_FUSE_QKV", fused)
    p = _params(cfg)
    p["self_attn.v_proj.weight"] = p["self_attn.v_proj.weight"] * 8      # v's columns set Wᵀ's scales
    x, doc, pos, dout = _inputs(cfg)
    out, _, _ = _run_block(p, cfg, x, doc, pos)
    out.backward(dout)
    T = x.shape[1]
    wt = torch.cat([p["self_attn." + n + "_proj.weight"] for n in "qkv"]).bfloat16()
    inv_w = (1.0 / rw_cols(wt)[1]).flatten()
    dgrads = [g for g in shim.gemms if g[1] and g[5].shape == inv_w.shape and torch.equal(g[5], inv_w)]
    assert len(dgrads) == (1 if fused else 3)
    for g in dgrads:
        assert g[4].shape == (T,) and torch.equal(g[4], dgrads[0][4])


def test_default_recipe_is_tensorwise_and_makes_no_rowwise_call(monkeypatch):
    from tests import cpu_ops_shim
    saved = cpu_ops_shim.install()
    try:
        st = F8Standins()
        for n in F8Standins.NAMES:
            monkeypatch.setattr(ops, n, getattr(st, n))
        _forbid(monkeypatch, RWStandins.NAMES)
        cfg = _cfg()
        x, doc, pos, dout = _inputs(cfg)
        from tests.test_float8_cpu import _run_block as run_tw
        out, _, _ = run_tw(_params(cfg), cfg, x, doc, pos)
        out.backward(dout)
        assert st.gemms and st.casts
        out2, _, _ = _run_block(_params(cfg), cfg, x, doc, pos, recipe="tensorwise")
        out2.backward(dout)
        assert torch.equal(out, out2)
    finally:
        cpu_ops_shim.uninstall(saved)


def test_tensor_and_context_parallelism_and_ragged_dimensions_raise(shim):
    cfg = _cfg()
    p = _params(cfg)
    x, doc, pos, _ = _inputs(cfg)
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
    with pytest.raises(_lib.TouchNetB200Error, match="multiples of 16"):
        _run_block(p, cfg, x[:, :196], doc[:, :196], pos[:, :196])


def test_recipe_key_is_plumbed_and_checked():
    from touchnet_b200 import modeling
    off = modeling.B200LlamaForCausalLM(_text(float8_training=True))
    on = modeling.B200LlamaForCausalLM(_text(float8_training=True, float8_recipe_name="rowwise"))
    assert off.float8_recipe_name == "tensorwise" and on.float8_recipe_name == "rowwise"
    assert list(on.state_dict()) == list(off.state_dict())
    assert [n for n, _ in on.named_buffers()] == [n for n, _ in off.named_buffers()]
    on.float8_recipe_name = "tensorwise"
    assert on.model.float8_recipe_name == "tensorwise"
    for bad in ("rowwise_with_gw_hp", "Rowwise", None):
        with pytest.raises(_lib.TouchNetB200Error, match="'tensorwise' or 'rowwise'"):
            on.float8_recipe_name = bad
    with pytest.raises(_lib.TouchNetB200Error, match="'tensorwise' or 'rowwise'"):
        modeling.B200LlamaForCausalLM(_text(float8_recipe_name="delayed"))
    audio = _NS(input_size=40)
    ta = modeling.B200TouchAudioForCausalLM(_NS(audio_config=audio, text_config=_text(float8_recipe_name="tensorwise"),
                                                pad_token_id=0, float8_recipe_name="rowwise"))
    assert ta.float8_recipe_name == "rowwise" and ta.language_model.model.float8_recipe_name == "rowwise"
    ta.float8_recipe_name = "tensorwise"
    assert ta.language_model.float8_recipe_name == "tensorwise"
    ta2 = modeling.B200TouchAudioForCausalLM(_NS(audio_config=audio, text_config=_text(float8_recipe_name="rowwise"),
                                                 pad_token_id=0))
    assert ta2.float8_recipe_name == "rowwise"
    ref = modeling.B200TouchAudioForCausalLM(_NS(audio_config=audio, text_config=_text(), pad_token_id=0))
    assert list(ta.state_dict()) == list(ref.state_dict())


def test_layers_receive_the_recipe(monkeypatch):
    from touchnet_b200 import modeling
    seen = []
    monkeypatch.setattr(ops, "decoder_layer", lambda *a, **k: (seen.append((a[-1], k["float8_recipe_name"])), a[0])[1])
    monkeypatch.setattr(ops, "AttnPlan", lambda doc: _NS(tp=None, cp_group=None))
    m = modeling.B200LlamaForCausalLM(_text(float8_training=True, float8_recipe_name="rowwise"))
    m.model.rotary_emb.forward = lambda pos: (None, None)
    m.model.norm.forward = lambda x: x
    m.model(torch.zeros(1, 16, 256, dtype=torch.bfloat16), torch.ones(1, 16, dtype=torch.long), None)
    assert seen == [(True, "rowwise"), (True, "rowwise")]


def test_generate_is_the_same_with_rowwise_on(monkeypatch):
    """Cached decoding never takes an FP8 path (no FP8 stand-in is installed, so an FP8 call would fail)."""
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
        ours.float8_recipe_name = "rowwise"
        on = ours.generate(ids, attention_mask=mask, max_new_tokens=6, eos_token_id=63, **tg._REF_KW)
    finally:
        cpu_ops_shim.uninstall(saved)
    assert torch.equal(on, off)


# ---------------------------------------------------------------------------------------------------------------
# entry points: argument checks (before any CUDA call)
# ---------------------------------------------------------------------------------------------------------------
def test_rowwise_entry_points_reject_bad_arguments():
    p = ctypes.c_void_p(256)
    q = ctypes.c_void_p(264)       # 8 B aligned only
    r = ctypes.c_void_p(260)       # 4 B aligned only
    bad_calls = [
        ("tn_fp8_rowwise_cast_bf16", (p, 256, 256, 256, p, 256, None, None), "null"),
        ("tn_fp8_rowwise_cast_bf16", (p, 256, 256, 200, p, 256, p, None), "multiples of 16"),
        ("tn_fp8_rowwise_cast_bf16", (q, 256, 256, 256, p, 256, p, None), "aligned"),
        ("tn_fp8_rowwise_cast_bf16", (p, 256, 256, 256, p, 248, p, None), "ld_out"),
        ("tn_fp8_colwise_amax_bf16", (None, 256, 256, 256, p, None), "null"),
        ("tn_fp8_colwise_amax_bf16", (p, 256, 250, 256, p, None), "multiples of 16"),
        ("tn_fp8_colwise_amax_bf16", (p, 200, 256, 256, p, None), "ldx"),
        ("tn_fp8_colwise_amax_bf16", (p, 256, 256, 256, ctypes.c_void_p(258), None), "4 B aligned"),
        ("tn_fp8_colwise_cast_t_bf16", (p, 256, 256, 256, ctypes.c_void_p(258), p, 256, p, None), "4 B aligned"),
        ("tn_fp8_colwise_cast_t_bf16", (p, 256, 256, 256, p, p, 256, ctypes.c_void_p(258), None), "4 B aligned"),
        ("tn_fp8_rowwise_cast_bf16", (p, 256, 256, 256, p, 256, ctypes.c_void_p(258), None), "4 B aligned"),
        ("tn_fp8_colwise_cast_t_bf16", (p, 256, 256, 256, p, None, 256, p, None), "null"),
        ("tn_fp8_colwise_cast_t_bf16", (p, 256, 256, 256, p, q, 256, p, None), "out_t"),
        ("tn_fp8_colwise_cast_t_bf16", (p, 256, 256, 256, p, p, 128, p, None), "out_t"),
        ("tn_gemm_fp8_rowwise", (p, 256, p, 256, p, 256, 0, None, 0, 256, 256, 256, None, p, 0, None), "null"),
        ("tn_gemm_fp8_rowwise", (p, 256, p, 256, p, 256, 0, None, 0, 256, 256, 264, p, p, 1, None), "multiples of 16"),
        ("tn_gemm_fp8_rowwise", (q, 256, p, 256, p, 256, 0, None, 0, 256, 256, 256, p, p, 0, None), "16 B aligned"),
        ("tn_gemm_fp8_rowwise", (p, 256, p, 256, q, 256, 0, None, 0, 256, 256, 256, p, p, 0, None), "D/R"),
        ("tn_gemm_fp8_rowwise", (p, 256, p, 256, p, 256, 0, None, 0, 256, 256, 256, r, p, 0, None), "8 B aligned"),
        ("tn_gemm_swiglu_fp8_rowwise", (p, 256, p, None, 256, p, p, p, 256, 256, 256, 256, p, p, None), "null"),
        ("tn_gemm_swiglu_fp8_rowwise", (p, 256, p, p, 256, p, p, p, 256, 256, 256, 200, p, p, None), "multiples of 16"),
        ("tn_gemm_swiglu_fp8_rowwise", (p, 256, p, p, 256, p, p, p, 256, 256, 256, 256, p, r, None), "8 B aligned"),
        ("tn_gemm_dswiglu_fp8_rowwise", (p, 256, p, 256, p, p, 256, p, p, 256, 256, 256, 8, p, p, None), "multiples of 16"),
        ("tn_gemm_dswiglu_fp8_rowwise", (p, 256, p, 256, p, p, 256, p, p, 256, 128, 256, 256, p, p, None), ">= 256"),
        ("tn_gemm_dswiglu_fp8_rowwise", (p, 256, p, 256, None, p, 256, p, p, 256, 256, 256, 256, p, p, None), "null"),
        ("tn_gemm_qkv_fp8_rowwise", (1, p, 768, p, p, p, 768, p, None, None, 256, 0, 256, 256, 256, 256, 256, 760, None,
                                     None, p, p, None), "multiples of 16"),
        ("tn_gemm_qkv_fp8_rowwise", (0, p, 256, p, p, p, 256, p, None, None, 768, 0, 256, 128, 256, 256, 640, 256, None,
                                     None, p, p, None), "multiples of 256"),
        ("tn_gemm_qkv_fp8_rowwise", (2, p, 256, p, None, None, 256, p, None, None, 256, 1, 256, 256, 256, 768, 256, 256,
                                     None, None, p, p, None), "D1/D2"),
        ("tn_gemm_qkv_fp8_rowwise", (3, p, 256, p, p, p, 256, p, None, None, 768, 0, 256, 256, 256, 256, 768, 256, None,
                                     None, p, p, None), "mode"),
        ("tn_gemm_qkv_fp8_rowwise", (0, p, 256, p, p, p, 256, p, None, None, 768, 0, 256, 256, 256, 256, 768, 256, None,
                                     None, p, r, None), "8 B aligned"),
    ]
    for name, args, needle in bad_calls:
        with pytest.raises(_lib.TouchNetB200Error, match=needle):
            _lib.call(name, *args)


def test_rowwise_gemm_wrappers_reject_operand_types():
    a = torch.zeros(16, 16, dtype=F8E4M3)
    inv = torch.ones(16)
    with pytest.raises(_lib.TouchNetB200Error, match="rowwise FP8 GEMM"):
        ops.gemm_fp8_rowwise(a, torch.zeros(16, 16, dtype=torch.float8_e5m2), inv, inv, promoted=True)
    with pytest.raises(_lib.TouchNetB200Error, match="rowwise FP8 GEMM"):
        ops.gemm_swiglu_fp8_rowwise(torch.zeros(16, 16, dtype=torch.bfloat16), a, a, inv, torch.ones(32))
