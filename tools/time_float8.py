"""Time FP8 training (config key `float8_training`) against bf16 on the bench.py workload (Llama-3.2-3B-ASR,
TouchAudioForCausalLM, one packed row of T = 8192, fp32 master weights, fused lm_head + pack loss).
    python tools/time_float8.py --out DIR [--steps 10] [--rounds 3]
Writes DIR/time_float8.json and prints it:
  - step time and tokens/s of the bf16, tensorwise FP8 and rowwise FP8 arms (config key `float8_recipe_name`),
    alternated round by round in one process (same model, same batch; CUDA events around `steps` training steps), with
    the peak memory of each arm;
  - per-shape TFLOP/s of the FP8 GEMM entry points at the block's shapes, tensorwise and rowwise, next to
    torch._scaled_mm on the same operands and scales (matching use_fast_accum), the bf16 GEMM at the same shape, and
    the 1,979 TFLOP/s data-sheet FP8 rate (a data-sheet figure, not a measurement);
  - GB/s of the amax and cast kernels, per tensor and per axis, against the 3.35 TB/s data-sheet HBM3 bandwidth;
  - the card name, power limit and SM clocks, read in the same run."""
import argparse
import json
import os
import statistics
import sys
from types import SimpleNamespace as NS

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from tools.time_decode import gpu_info  # noqa: E402
from touchnet_b200 import modeling, ops  # noqa: E402

DATASHEET_FP8_FLOPS = 1979e12
DATASHEET_HBM_BPS = 3.35e12


def _events_ms(fn, iters):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def time_steps(args, dev):
    bench.select_workload(NS(workload="llama32_3b_asr", seq_len=None, batch=None, layers=None))
    B, T = bench._W["batch"], bench._W["seq_len"]
    cfg = bench.asr_config(bench._W["layers"])
    torch.manual_seed(2025)
    with torch.device(dev):
        model = modeling.B200TouchAudioForCausalLM(cfg)
    with torch.no_grad():
        for p in model.parameters():
            if p.dim() == 2:
                p.normal_(0.0, 0.02)
    model.fused_linear_ce = True
    host, meta = bench.make_host_batch(2025, B, T, cfg.text_config.vocab_size)
    d = bench.to_device(host, dev)

    def step():
        model.zero_grad(set_to_none=True)
        ops.invalidate_bf16_cache(model)     # the fp32 -> bf16 cast is part of every step, as in bench.py
        return bench.run_step(model, d, meta, B, T)

    arms = {"bf16": (False, "tensorwise"), "fp8": (True, "tensorwise"), "fp8_rowwise": (True, "rowwise")}
    res = {k: {"ms": [], "loss": None, "peak_gb": 0.0} for k in arms}
    for name, (on, recipe) in arms.items():            # warm-up of every arm
        model.float8_training, model.float8_recipe_name = on, recipe
        for _ in range(args.warmup):
            step()
    torch.cuda.synchronize()
    for _ in range(args.rounds):
        for name, (on, recipe) in arms.items():
            model.float8_training, model.float8_recipe_name = on, recipe
            torch.cuda.reset_peak_memory_stats(dev)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.steps):
                loss = step()
            b.record()
            torch.cuda.synchronize()
            res[name]["ms"].append(a.elapsed_time(b) / args.steps)
            res[name]["loss"] = float(loss)
            res[name]["peak_gb"] = max(res[name]["peak_gb"], torch.cuda.max_memory_allocated(dev) / 1e9)
    for name in arms:
        ms = statistics.median(res[name]["ms"])
        res[name].update(ms_per_step_median=ms, tokens_per_s=B * T / (ms / 1e3))
    res["fp8_over_bf16_tokens_per_s"] = res["fp8"]["tokens_per_s"] / res["bf16"]["tokens_per_s"]
    res["fp8_rowwise_over_bf16_tokens_per_s"] = res["fp8_rowwise"]["tokens_per_s"] / res["bf16"]["tokens_per_s"]
    res["workload"] = f"{bench._W['text']} L={bench._W['layers']} B={B} T={T}"
    del model, d
    torch.cuda.empty_cache()
    return res


def time_gemms(dev, iters):
    """(name, M, N, K, a_e5m2) at the bench block's shapes (T = 8192, d 3072, q 3072, kv 1024, ffn 8192)."""
    shapes = [("qkv fwd", 8192, 5120, 3072, False), ("o fwd", 8192, 3072, 3072, False),
              ("down fwd", 8192, 3072, 8192, False), ("down dgrad", 8192, 8192, 3072, True),
              ("gate/up dgrad", 8192, 3072, 8192, True), ("o dgrad", 8192, 3072, 3072, True),
              ("o wgrad", 3072, 3072, 8192, True), ("gate/up wgrad", 8192, 3072, 8192, True),
              ("down wgrad", 3072, 8192, 8192, True), ("qkv wgrad", 5120, 3072, 8192, True)]
    out = []
    for name, M, N, K, e5 in shapes:
        a = torch.randn(M, K, device=dev).bfloat16()
        b = (torch.randn(N, K, device=dev) * 0.02).bfloat16()
        st = torch.zeros((2, 2), device=dev)
        (a8, _), = ops._fp8_quant([a], st, 0, e5, t=False)
        (b8, _), = ops._fp8_quant([b], st, 1, False, t=False)
        ia, ib = st[0, 1], st[1, 1]
        fl = 2.0 * M * N * K
        ours = _events_ms(lambda: ops.gemm_fp8(a8, b8, ia, ib), iters)
        sa, sb = ia.reshape(1).contiguous(), ib.reshape(1).contiguous()
        sm = _events_ms(lambda: torch._scaled_mm(a8, b8.t(), scale_a=sa, scale_b=sb, out_dtype=torch.bfloat16,
                                                 use_fast_accum=not e5), iters)
        bf = _events_ms(lambda: ops.gemm(a, b), iters)
        # rowwise: e4m3 A and B, per-row scales; the same accumulation as the tensorwise launch at this shape
        ra8, ria = ops.fp8_rowwise_cast(a)
        rb8, rib = ops.fp8_rowwise_cast(b)
        rw = _events_ms(lambda: ops.gemm_fp8_rowwise(ra8, rb8, ria, rib, promoted=e5), iters)
        rsa, rsb = ria[:, None].contiguous(), rib[None, :].contiguous()
        rsm = _events_ms(lambda: torch._scaled_mm(ra8, rb8.t(), scale_a=rsa, scale_b=rsb, out_dtype=torch.bfloat16,
                                                  use_fast_accum=not e5), iters)
        out.append({"shape": f"{name} M={M} N={N} K={K}", "accumulation": "promoted" if e5 else "fast",
                    "fp8_ms": ours, "fp8_tflops": fl / ours / 1e9, "scaled_mm_tflops": fl / sm / 1e9,
                    "rowwise_tflops": fl / rw / 1e9, "scaled_mm_rowwise_tflops": fl / rsm / 1e9,
                    "bf16_tflops": fl / bf / 1e9, "fp8_frac_of_datasheet": fl / (ours / 1e3) / DATASHEET_FP8_FLOPS})
        del a, b, a8, b8, ra8, rb8
    # the two fused entry points at their forward shapes
    x = torch.randn(8192, 3072, device=dev).bfloat16()
    w = (torch.randn(8192, 3072, device=dev) * 0.02).bfloat16()
    st = torch.zeros((2, 2), device=dev)
    (x8, _), = ops._fp8_quant([x], st, 0, False, t=False)
    (w8, _), = ops._fp8_quant([w], st, 1, False, t=False)
    ms = _events_ms(lambda: ops.gemm_swiglu_fp8(x8, w8, w8, st[0, 1], st[1, 1]), iters)
    bf = _events_ms(lambda: ops.gemm_swiglu(x, w, w), iters)
    rx8, rix = ops.fp8_rowwise_cast(x)
    rw8, riw = ops.fp8_rowwise_cast(w)
    riw2 = torch.cat([riw, riw])
    rms = _events_ms(lambda: ops.gemm_swiglu_fp8_rowwise(rx8, rw8, rw8, rix, riw2), iters)
    fl = 2.0 * 8192 * 16384 * 3072
    out.append({"shape": "gate/up fwd (SwiGLU epilogue) M=8192 N=16384 K=3072", "accumulation": "fast", "fp8_ms": ms,
                "fp8_tflops": fl / ms / 1e9, "rowwise_tflops": fl / rms / 1e9, "bf16_tflops": fl / bf / 1e9,
                "fp8_frac_of_datasheet": fl / (ms / 1e3) / DATASHEET_FP8_FLOPS})
    return out


def time_quant(dev, iters):
    out = []
    for rows, cols in ((8192, 3072), (8192, 8192)):
        x = torch.randn(rows, cols, device=dev).bfloat16()
        amax = torch.zeros((), device=dev)
        inv = torch.zeros((), device=dev)
        ops.fp8_amax(x, amax)
        n = rows * cols
        t_amax = _events_ms(lambda: ops.fp8_amax(x, amax), iters)
        t_both = _events_ms(lambda: ops.fp8_cast(x, amax, False, inv=inv), iters)
        t_row = _events_ms(lambda: ops.fp8_cast(x, amax, False, t=False, inv=inv), iters)
        camax = torch.zeros(cols, device=dev)
        t_rowcast = _events_ms(lambda: ops.fp8_rowwise_cast(x), iters)
        t_colamax = _events_ms(lambda: ops.fp8_colwise_amax(x, camax), iters)
        t_colcast = _events_ms(lambda: ops.fp8_colwise_cast_t(x, camax), iters)
        out.append({"shape": f"{rows}x{cols}", "amax_gbps": 2 * n / t_amax / 1e6,
                    "cast_both_layouts_gbps": 4 * n / t_both / 1e6, "cast_row_major_gbps": 3 * n / t_row / 1e6,
                    "rowwise_cast_gbps": 3 * n / t_rowcast / 1e6, "colwise_amax_gbps": 2 * n / t_colamax / 1e6,
                    "colwise_cast_t_gbps": 3 * n / t_colcast / 1e6, "datasheet_hbm_gbps": DATASHEET_HBM_BPS / 1e9})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "time_float8.py measures on the GPU; there is no CPU path"
    dev = torch.device("cuda:0")
    res = {"gpu": gpu_info(), "steps": time_steps(args, dev), "gemm": time_gemms(dev, args.iters),
           "quant": time_quant(dev, args.iters)}
    res["gpu_after"] = gpu_info()
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "time_float8.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
