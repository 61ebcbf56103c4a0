"""GPU parity: RMSNorm / RoPE / SwiGLU-backward / embedding-add kernels vs the oracle restatement of the HF ops."""
import pytest
import torch

from oracle import model_oracle as mo
from tests.gpu_util import require_cuda, rel_err
from touchnet_b200 import ops

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("rows,d", [(64, 4096), (200, 768), (33, 64), (1024, 2048), (40, 8192), (7, 24)])
@pytest.mark.parametrize("w_f32", [False, True])
def test_rmsnorm_forward_backward(rows, d, w_f32):
    dev = require_cuda()
    torch.manual_seed(rows + d)
    x = torch.randn(rows, d, device=dev).bfloat16()
    w = (1 + 0.1 * torch.randn(d, device=dev)).to(torch.float32 if w_f32 else torch.bfloat16)
    y, s, rstd = ops.rmsnorm_fwd(x, w, 1e-5)
    ref = mo.rms_norm(x, w.bfloat16(), 1e-5)                      # HF op order on the same bf16 data
    assert float((y.float() - ref.float()).abs().max()) <= 2 ** -6 * float(ref.float().abs().max())
    # backward vs autograd of the fp32 formula
    xf = x.float().requires_grad_(True)
    wf = w.bfloat16().float().requires_grad_(True)
    dy = torch.randn(rows, d, device=dev).bfloat16()
    extra = torch.randn(rows, d, device=dev).bfloat16()
    out = wf * (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-5))
    out.backward(dy.float())
    ds, dw = ops.rmsnorm_bwd(x, dy, w, rstd, ds_extra=extra)
    assert rel_err(ds.float(), xf.grad + extra.float()) < 1e-2
    assert rel_err(dw, wf.grad) < 1e-2


def test_rmsnorm_fused_residual():
    dev = require_cuda()
    x = torch.randn(96, 1024, device=dev).bfloat16()
    r = torch.randn(96, 1024, device=dev).bfloat16()
    w = torch.ones(1024, device=dev, dtype=torch.bfloat16)
    y, s, _ = ops.rmsnorm_fwd(x, w, 1e-5, residual=r)
    assert torch.equal(s, x + r)                                  # bf16 add, bit exact
    assert torch.equal(y, ops.rmsnorm_fwd(s, w, 1e-5)[0])


@pytest.mark.parametrize("theta,scaling", [(500000.0, {"rope_type": "llama3", "factor": 32.0, "low_freq_factor": 1.0,
                                                        "high_freq_factor": 4.0, "original_max_position_embeddings": 8192}),
                                           (10000.0, None)])
def test_rope_table_and_apply(theta, scaling):
    dev = require_cuda()
    B, T, H, KV, hd = 2, 640, 4, 2, 128
    cfg = mo.OracleConfig(hidden_size=H * hd, intermediate_size=8, num_hidden_layers=1, num_attention_heads=H,
                          num_key_value_heads=KV, head_dim=hd, vocab_size=8, rope_theta=theta, rope_scaling=scaling)
    inv, sc = mo.rope_inv_freq(cfg)
    pos = torch.cat([torch.arange(300), torch.arange(340)])[None].repeat(B, 1).to(dev)
    pos[1] = torch.arange(T, device=dev) * 13                      # large positions: accurate range reduction
    cos, sin = ops.rope_table(pos, inv.to(dev), sc)
    cos_ref, sin_ref = mo.rope_cos_sin(pos, inv.to(dev), sc, torch.bfloat16)
    # bf16 tables: allow 1 ulp (sincosf vs torch.cos differ by < 1e-6 before rounding)
    assert float((cos.float().view(B, T, -1) - cos_ref[..., :hd // 2].float()).abs().max()) <= 2 ** -8
    assert float((sin.float().view(B, T, -1) - sin_ref[..., :hd // 2].float()).abs().max()) <= 2 ** -8
    q = torch.randn(B * T, H * hd, device=dev).bfloat16()
    k = torch.randn(B * T, KV * hd, device=dev).bfloat16()
    cos_r = torch.cat([cos, cos], -1).view(B, T, hd)               # reference apply on OUR tables: op-order parity
    sin_r = torch.cat([sin, sin], -1).view(B, T, hd)
    q_ref, k_ref = mo.apply_rope(q.view(B, T, H, hd).transpose(1, 2), k.view(B, T, KV, hd).transpose(1, 2), cos_r, sin_r)
    q0 = q.clone()
    ops.rope_apply_(q, cos, sin, H, hd)
    ops.rope_apply_(k, cos, sin, KV, hd)
    assert torch.equal(q.view(B, T, H, hd), q_ref.transpose(1, 2))  # bit exact vs the bf16 HF formula
    assert torch.equal(k.view(B, T, KV, hd), k_ref.transpose(1, 2))
    # inverse rotation = transpose of the rotation: <R q, g> == <q, R^T g> up to the bf16 rounding of R q and R^T g
    # (relative error <= 2^-9 per element with random signs, so the sums differ by ~2^-9 * ||q*g||_2: bound at 4x that)
    g = torch.randn_like(q)
    g2 = g.clone()
    ops.rope_apply_(g2, cos, sin, H, hd, inverse=True)
    lhs = float((q.double() * g.double()).sum())
    rhs = float((q0.double() * g2.double()).sum())
    rounding = 2 ** -9 * float((q.double() * g.double()).square().sum().sqrt())
    assert abs(lhs - rhs) < 2e-2 * abs(lhs) + 4 * rounding
    # and element-wise: R^T (R q) == q up to two bf16 roundings
    back = q.clone()
    ops.rope_apply_(back, cos, sin, H, hd, inverse=True)
    assert float((back.float() - q0.float()).abs().max()) <= 2 ** -6 * float(q0.float().abs().max())


def test_swiglu_backward():
    dev = require_cuda()
    g = torch.randn(300, 1024, device=dev).bfloat16()
    u = torch.randn(300, 1024, device=dev).bfloat16()
    dh = torch.randn(300, 1024, device=dev).bfloat16()
    gf, uf = g.float().requires_grad_(True), u.float().requires_grad_(True)
    (torch.nn.functional.silu(gf) * uf).backward(dh.float())
    dg, du = ops.swiglu_bwd(g, u, dh)
    assert rel_err(dg.float(), gf.grad) < 1e-2 and rel_err(du.float(), uf.grad) < 1e-2


def test_embed_add_and_cast():
    dev = require_cuda()
    V, d, rows = 1000, 512, 777
    emb = torch.randn(V, d, device=dev)
    ids = torch.randint(0, V, (rows,), device=dev)
    proj = torch.randn(rows, d, device=dev).bfloat16()
    flag = torch.zeros(1, dtype=torch.int32, device=dev)
    e = ops.embed_add(ids, emb, proj, rows, d, flag)
    ref = emb[ids].bfloat16() + proj                               # ref: modeling_touch_audio.py:124-131 in bf16
    assert torch.equal(e, ref) and int(flag.item()) == 0
    proj[5, 7] = float("nan")
    ops.embed_add(ids, emb.bfloat16(), proj, rows, d, flag)
    assert int(flag.item()) == 1                                   # ref: :133-134 NaN check
    x = torch.randn(100003, device=dev)
    assert torch.equal(ops.cast_bf16(x), x.bfloat16())


def test_bf16_weight_cache_follows_the_parameter_object():
    """Regression: the bf16 working copy is cached on the parameter object (and keyed by its version counter), so a new
    parameter that happens to reuse a freed parameter's address, or an in-place optimizer update, never sees a stale copy."""
    dev = require_cuda()
    w = torch.nn.Parameter(torch.randn(256, 128, device=dev))
    a = ops.bf16_weight(w)
    assert torch.equal(a, w.detach().bfloat16()) and ops.bf16_weight(w) is a      # cached
    with torch.no_grad():
        w.add_(1.0)                                                                # optimizer-style in-place update
    b = ops.bf16_weight(w)
    assert torch.equal(b, w.detach().bfloat16())
    addr = w.data_ptr()
    del w, a, b
    w2 = torch.nn.Parameter(torch.full((256, 128), 3.0, device=dev))               # very likely the same address
    assert torch.equal(ops.bf16_weight(w2), w2.detach().bfloat16()), (addr, w2.data_ptr())
    m = torch.nn.Linear(128, 256, bias=False).to(dev)
    c = ops.bf16_weight(m.weight)
    ops.invalidate_bf16_cache(m)
    with torch.no_grad():
        m.weight.data.fill_(2.0)                                                   # .data writes do not bump the version
    assert torch.equal(ops.bf16_weight(m.weight), torch.full_like(c, 2.0))
    # side-stream prefetch: same values, consumer waits on the per-parameter event
    ops.invalidate_bf16_cache(m)
    with torch.no_grad():
        m.weight.data.fill_(5.0)
    assert ops.prefetch_bf16_weights(m) == 1 and ops.prefetch_bf16_weights(m) == 0
    assert torch.equal(ops.bf16_weight(m.weight), torch.full_like(c, 5.0))
