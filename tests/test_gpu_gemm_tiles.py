"""GPU: the GEMM's two tile widths (128x256 and 128x128, chosen from the shape's wave count) and its TMA-store epilogue.

With 132 SMs the shapes below select: 2048x4096, 8200x4104, 4096x3072 (fused QKV), 3072x1024 (QKV wgrad), SwiGLU
2048x8192 -> 128x256; 200x264, 3072x3072, and every N <= 256 slice -> 128x128.  Each output element sums its k-blocks in
the same order at either width, so a column slice recomputed at a 128-wide shape must equal the 256-wide result bit for
bit."""
import pytest
import torch

from tests.gpu_util import require_cuda
from touchnet_b200 import ops

pytestmark = pytest.mark.gpu


def _rand(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, device="cuda", generator=g) * scale).bfloat16()


def _close(got, ref, rel, abs_):
    return float((got.float() - ref).abs().max()) < rel * float(ref.abs().max()) + abs_


@pytest.mark.parametrize("M,N,K", [(2048, 4096, 512), (8200, 4104, 256), (200, 264, 1040), (3072, 3072, 256)])
def test_forward_dgrad_wgrad_with_and_without_residual(M, N, K):
    require_cuda()
    a, b = _rand(M, K, scale=0.5, seed=1), _rand(N, K, scale=0.05, seed=2)
    ref = a.float() @ b.float().t()
    assert _close(ops.gemm(a, b), ref, 1e-2, 1e-2)
    r = _rand(M, N, seed=3)
    want = ref.bfloat16().float() + r.float()
    assert float((ops.gemm(a, b, residual=r).float() - want).abs().max()) <= 2 ** -6 * float(want.abs().max())
    dy = _rand(M, N, scale=0.1, seed=4)
    assert _close(ops.gemm(dy, b, b_mn=True), dy.float() @ b.float(), 1e-2, 1e-2)
    ref_dw = dy.float().t() @ a.float()                                         # [N, K]
    dw = ops.gemm(dy, a, a_mn=True, b_mn=True, out_f32=True)
    assert _close(dw, ref_dw, 1e-4, 1e-4)
    assert _close(ops.gemm(dy, a, a_mn=True, b_mn=True), ref_dw, 1e-2, 1e-2)   # bf16 wgrad
    acc = torch.randn(N, K, device="cuda")                                      # fp32 accumulation in place
    want_acc = acc + dw
    ops.gemm(dy, a, a_mn=True, b_mn=True, out_f32=True, residual=acc, out=acc)
    assert torch.equal(acc, want_acc)
    rb = _rand(N, K, seed=5).float()                                            # fp32 +R into a fresh output
    assert torch.equal(ops.gemm(dy, a, a_mn=True, b_mn=True, out_f32=True, residual=rb), dw + rb)


def test_tile_widths_give_identical_bits():
    require_cuda()
    M, N, K = 2048, 4096, 512
    a, b = _rand(M, K, scale=0.5, seed=6), _rand(N, K, scale=0.05, seed=7)
    dy = _rand(M, N, scale=0.1, seed=8)
    bt = b.t().contiguous()                                                      # [K, N]: dgrad a·bt, N = 4096
    y, dx = ops.gemm(a, b), ops.gemm(a, bt, b_mn=True)
    x = _rand(M, N, seed=9)                                                      # wgrad: dyᵀ·x, [N, N] fp32
    dw = ops.gemm(dy, x, a_mn=True, b_mn=True, out_f32=True)
    for c0 in (0, 256, 3840):
        sl = slice(c0, c0 + 256)
        assert torch.equal(ops.gemm(a, b[sl]), y[:, sl])
        assert torch.equal(ops.gemm(a, bt[:, sl], b_mn=True), dx[:, sl])
        assert torch.equal(ops.gemm(dy, x[:, sl], a_mn=True, b_mn=True, out_f32=True), dw[:, sl])


def test_swiglu_wide_tile():
    require_cuda()
    M, N, K = 2048, 8192, 256
    x, wg, wu = _rand(M, K, scale=0.5, seed=10), _rand(N, K, scale=0.05, seed=11), _rand(N, K, scale=0.05, seed=12)
    g, u, h = ops.gemm_swiglu(x, wg, wu)
    assert _close(g, x.float() @ wg.float().t(), 1e-2, 1e-2)
    assert _close(u, x.float() @ wu.float().t(), 1e-2, 1e-2)
    h_ref = (torch.nn.functional.silu(g.float()).bfloat16().float() * u.float()).bfloat16()
    assert float((h != h_ref).float().mean()) < 1e-3
    _, _, h_only = ops.gemm_swiglu(x, wg, wu, need_gu=False)
    assert torch.equal(h_only, h)
    for c0 in (0, 8064):
        sl = slice(c0, c0 + 128)
        gs, us, hs = ops.gemm_swiglu(x, wg[sl], wu[sl])
        assert torch.equal(gs, g[:, sl]) and torch.equal(us, u[:, sl]) and torch.equal(hs, h[:, sl])


def test_qkv_rope_and_segmented_wgrad_wide_tile():
    require_cuda()
    from oracle import model_oracle as mo
    M, d, H, KV = 4096, 1024, 16, 4
    nq, nkv = H * 128, KV * 128
    x = _rand(M, d, scale=0.5, seed=13)
    wq, wk, wv = (_rand(n, d, scale=0.05, seed=14 + i) for i, n in enumerate((nq, nkv, nkv)))
    qkv = ops.gemm_qkv_fwd(x, wq, wk, wv)
    assert torch.equal(qkv, torch.cat([ops.gemm(x, wq), ops.gemm(x, wk), ops.gemm(x, wv)], dim=1))
    pos = (torch.arange(M, device="cuda") % 900)[None]
    inv, sc = mo.rope_inv_freq(mo.OracleConfig(d, 8, 1, H, KV, 128, 8, rope_theta=500000.0))
    cos, sin = ops.rope_table(pos, inv.cuda(), sc)
    fused = ops.gemm_qkv_fwd(x, wq, wk, wv, rope=(cos, sin))
    plain = qkv.clone()
    ops.rope_apply_(plain[:, :nq], cos, sin, H, 128)
    ops.rope_apply_(plain[:, nq:nq + nkv], cos, sin, KV, 128)
    assert torch.equal(fused, plain)
    dqkv = _rand(M, nq + 2 * nkv, scale=0.1, seed=20)
    dx = ops.gemm_qkv_dgrad(dqkv, wq, wk, wv)
    assert _close(dx, dqkv.float() @ torch.cat([wq, wk, wv]).float(), 1e-2, 1e-2)
    offs = [0, nq, nq + nkv, nq + 2 * nkv]
    for f32 in (True, False):
        dws = ops.gemm_qkv_wgrad(dqkv, x, f32, nq, nkv)
        for i, dw in enumerate(dws):
            sep = ops.gemm(dqkv[:, offs[i]:offs[i + 1]], x, a_mn=True, b_mn=True, out_f32=f32)
            assert torch.equal(dw, sep)
            if f32:
                want = dqkv[:, offs[i]:offs[i + 1]].float().t() @ x.float()
                assert _close(dw, want, 1e-4, 1e-4)


def test_fused_dswiglu_wide_tile():
    require_cuda()
    M, N, K = 2048, 4096, 512
    dy, wd = _rand(M, K, scale=0.5, seed=21), _rand(K, N, scale=0.05, seed=22)
    g, u = _rand(M, N, seed=23), _rand(M, N, seed=24)
    dg_ref, du_ref = ops.swiglu_bwd(g, u, ops.gemm(dy, wd, b_mn=True))
    ops._FUSE_DSWIGLU, saved = True, ops._FUSE_DSWIGLU
    try:
        dg, du = ops.gemm_dswiglu(dy, wd, g, u)
        sl = slice(512, 768)
        dgs, dus = ops.gemm_dswiglu(dy, wd[:, sl].contiguous(), g[:, sl].contiguous(), u[:, sl].contiguous())
    finally:
        ops._FUSE_DSWIGLU = saved
    assert torch.equal(dg, dg_ref) and torch.equal(du, du_ref)
    assert torch.equal(dgs, dg[:, sl]) and torch.equal(dus, du[:, sl])
