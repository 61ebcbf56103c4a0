"""Raster-group sweep of the GEMM on every GEMM shape of one training step (tn_set_gemm_group), operands rotated over
more buffers than fit in L2.  Prints TFLOP/s per (shape, group), best of 2 repeats.  The tile width is the one the
library picks for the shape.  Shapes: Llama-3.2-3B (the bench.py workload, default) or Llama-3-8B (`--workload 8b`)."""
import os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from touchnet_b200 import _lib, ops
dev = torch.device("cuda")
if "8b" in sys.argv[1:]:
    M, D, NQ, NKV, FFN, V = 8192, 4096, 4096, 1024, 14336, 128256
else:
    M, D, NQ, NKV, FFN, V = 8192, 3072, 3072, 1024, 8192, 128256
GROUPS = (1, 2, 4, 8, 16, 32, 64)
r = lambda *s: torch.randn(*s, device=dev).bfloat16()
w = lambda *s: (torch.randn(*s, device=dev) * 0.05).bfloat16()
NB = 3
def bench(fn, flop):
    out = []
    for grp in GROUPS:
        _lib.call("tn_set_gemm_group", grp)
        best = 0.0
        for rep in range(2):
            for i in range(2): fn(i)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            it = 9
            e0.record()
            for i in range(it): fn(i)
            e1.record(); torch.cuda.synchronize()
            best = max(best, flop / (e0.elapsed_time(e1) / it) / 1e9)
        out.append(best)
    return out
def show(name, vals):
    b = max(range(len(vals)), key=lambda i: vals[i])
    print(f"{name:34s}" + "".join(f" g{g}:{v:5.0f}{'*' if i == b else ' '}" for i, (g, v) in enumerate(zip(GROUPS, vals))), flush=True)
xs = [r(M, D) for _ in range(NB)]; hs = [r(M, FFN) for _ in range(NB)]
wq, wk, wv, wo = w(NQ, D), w(NKV, D), w(NKV, D), w(D, NQ)
wg, wu, wd = w(FFN, D), w(FFN, D), w(D, FFN)
dqkv = [r(M, NQ + 2 * NKV) for _ in range(NB)]
cases = [
    (f"fwd  qkv fused [{M}x{NQ + 2 * NKV}x{D}]", lambda i: ops.gemm_qkv_fwd(xs[i % NB], wq, wk, wv), 2.0 * M * (NQ + 2 * NKV) * D),
    (f"fwd  o_proj    [{M}x{D}x{NQ}]", lambda i: ops.gemm(xs[i % NB], wo), 2.0 * M * D * NQ),
    (f"fwd  gate/up swiglu [{M}x{2 * FFN}x{D}]", lambda i: ops.gemm_swiglu(xs[i % NB], wg, wu), 2.0 * M * 2 * FFN * D),
    (f"fwd  down      [{M}x{D}x{FFN}]", lambda i: ops.gemm(hs[i % NB], wd), 2.0 * M * D * FFN),
    (f"dgrad down     [{M}x{FFN}x{D}]", lambda i: ops.gemm(xs[i % NB], wd, b_mn=True), 2.0 * M * D * FFN),
    (f"dgrad gate/up  [{M}x{D}x{FFN}]", lambda i: ops.gemm(hs[i % NB], wg, b_mn=True), 2.0 * M * D * FFN),
    (f"dgrad o_proj   [{M}x{D}x{NQ}]", lambda i: ops.gemm(xs[i % NB], wo, b_mn=True), 2.0 * M * D * NQ),
    (f"dgrad qkv fused [{M}x{D}x{NQ + 2 * NKV}]", lambda i: ops.gemm_qkv_dgrad(dqkv[i % NB], wq, wk, wv), 2.0 * M * (NQ + 2 * NKV) * D),
    (f"wgrad down     [{D}x{FFN}x{M}]", lambda i: ops.gemm(xs[i % NB], hs[i % NB], a_mn=True, b_mn=True, out_f32=True), 2.0 * M * D * FFN),
    (f"wgrad gate/up  [{FFN}x{D}x{M}]", lambda i: ops.gemm(hs[i % NB], xs[i % NB], a_mn=True, b_mn=True, out_f32=True), 2.0 * M * D * FFN),
    (f"wgrad o_proj   [{NQ}x{D}x{M}]", lambda i: ops.gemm(xs[i % NB], xs[(i + 1) % NB], a_mn=True, b_mn=True, out_f32=True), 2.0 * M * D * NQ),
    (f"wgrad qkv fused [{NQ + 2 * NKV}x{D}x{M}]", lambda i: ops.gemm_qkv_wgrad(dqkv[i % NB], xs[i % NB], True, NQ, NKV), 2.0 * M * (NQ + 2 * NKV) * D),
]
for name, fn, flop in cases:
    show(name, bench(fn, flop))
del hs, dqkv
wl = w(V, D); lg = r(M, V)
show(f"fwd  lm_head   [{M}x{V}x{D}]", bench(lambda i: ops.gemm(xs[i % NB], wl), 2.0 * M * V * D))
show(f"dgrad lm_head  [{M}x{D}x{V}]", bench(lambda i: ops.gemm(lg, wl, b_mn=True), 2.0 * M * V * D))
show(f"wgrad lm_head  [{V}x{D}x{M}]", bench(lambda i: ops.gemm(lg, xs[i % NB], a_mn=True, b_mn=True, out_f32=True), 2.0 * M * V * D))
_lib.call("tn_set_gemm_group", 8)
