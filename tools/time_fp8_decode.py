"""Time FP8 cached decoding (model config key `float8_inference`) against bf16 decoding on the DESIGN §6 workload:
Llama-3.2-3B-ASR of bench.py with random bf16 weights, B = 12 left-padded utterance prompts (T = 711), 256 new tokens,
eos unreachable, repetition_penalty 1.5, no_repeat_ngram_size 2.

    python tools/time_fp8_decode.py --out DIR [--reps 3] [--n 96]

The bf16 and FP8 arms alternate --reps times in one process (the same model object, the switch flipped between arms).
Writes DIR/time_fp8_decode.json with, per arm:
  the decode step (median over CUDA-graph replays, CUDA events), generate tokens/s end to end, generate_many tokens/s
  on the 96-utterance workload of tools/time_generate_many.py, the one-off weight quantisation time (FP8) and the peak
  memory of a generate call;
and, at M = 12, the device time of tn_gemm_fp8_decode and of the bf16 GEMM the bf16 step runs on the qkv, o, gate/up
and down shapes (CUDA events around one CUDA graph of 200 launches, so host launch overhead stays out of the window) with
the weight bytes each reads per launch over that time.  The card name, power limit and SM clocks are read in the same
run."""
import argparse
import json
import math
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from tools.time_decode import gpu_info, prompts  # noqa: E402
from tools.time_generate_many import TOKENS_PER_SECOND, median, random_model, utterances  # noqa: E402
from touchnet_b200 import generation, ops  # noqa: E402

# (name, N, K) at d = 3072, q 3072, kv 1024, ffn 8192; gate/up: N = 2 x 8192 weight rows
SHAPES = [("qkv", 5120, 3072), ("o", 3072, 3072), ("gate_up", 16384, 3072), ("down", 3072, 8192)]


def _events(fn, n):
    """Device ms per launch: n launches captured in one CUDA graph, so host launch overhead is not in the window."""
    for _ in range(3):
        fn()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(n):
            fn()
    g.replay()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def kernel_times(M, dev, n=200):
    out = {}
    for name, N, K in SHAPES:
        x = torch.randn(M, K, device=dev).bfloat16()
        w = (torch.randn(N, K, device=dev) * 0.02).bfloat16()
        w8, iw = ops.fp8_rowwise_cast(w)
        if name == "gate_up":
            f8 = lambda: ops.gemm_fp8_decode(x, w8, iw, swiglu=True)  # noqa: E731
            bf = lambda: ops.gemm_swiglu(x, w[:N // 2], w[N // 2:], need_gu=False)  # noqa: E731
        else:
            f8 = lambda: ops.gemm_fp8_decode(x, w8, iw)  # noqa: E731
            bf = lambda: ops.gemm(x, w)  # noqa: E731
        t8, tb = _events(f8, n), _events(bf, n)
        out[name] = {"N": N, "K": K, "fp8_decode_us": 1e3 * t8, "fp8_weight_bytes_per_s": N * K / (t8 * 1e-3),
                     "bf16_us": 1e3 * tb, "bf16_weight_bytes_per_s": 2 * N * K / (tb * 1e-3)}
    return out


def step_ms(model, ids, feats, mask, new, V):
    """Median decode step over graph replays, as tools/time_decode.py measures it."""
    B, T = ids.shape
    with torch.no_grad():
        w = generation._Weights(model.language_model)
        cache = generation.B200KVCache(model, B, T + new)

        def select(lg):
            ops.greedy_select(lg, cache.history, cache.kv_end, cache.positions, cache.next_ids, cache.finished, 1.5, 2,
                              V, 0)

        select(generation.prefill(model, cache, ids, feats, mask, None, weights=w))
        select(generation.decode_step(model, cache, weights=w))
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            select(generation.decode_step(model, cache, weights=w))
        evs = []
        for _ in range(new - 2):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); g.replay(); e1.record()
            evs.append((e0, e1))
        torch.cuda.synchronize()
        del g
    return median([a.elapsed_time(b) for a, b in evs])


def quant_ms(model):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    w = generation._Weights(model.language_model)
    torch.cuda.synchronize()
    assert w.float8 is not None
    return 1e3 * (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--new", type=int, default=256)
    ap.add_argument("--n", type=int, default=96)
    ap.add_argument("--layers", type=int, default=28)
    ap.add_argument("--seed", type=int, default=2025)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_fp8_decode.py measures the GPU: no CUDA device")
    os.makedirs(args.out, exist_ok=True)
    dev = torch.device("cuda")
    res = {"gpu": gpu_info()}
    model = random_model(args.layers, args.seed, dev)
    V = bench.asr_config(args.layers).text_config.vocab_size
    ids, feats, mask, _ = prompts(12, args.seed, V, dev)
    B, T = ids.shape
    secs, utts = utterances(args.n, args.seed, dev)
    budgets = [math.ceil(TOKENS_PER_SECOND * s) for s in secs]
    kw = dict(eos_token_id=V, pad_token_id=0, repetition_penalty=1.5, no_repeat_ngram_size=2)
    res["workload"] = (f"{bench._W['name']} decode: B={B}, T={T}, {args.new} new tokens, eos unreachable, random bf16 "
                       f"weights; generate_many: {args.n} utterances, batch 12, {sum(budgets)} tokens")
    res["kernels_M12"] = kernel_times(12, dev)
    arms = {"bf16": [], "fp8": []}
    for rep in range(args.reps):
        for arm in ("bf16", "fp8"):
            model.float8_inference = arm == "fp8"
            r = {}
            if arm == "fp8":
                r["quantise_ms"] = quant_ms(model)
            r["step_ms"] = step_ms(model, ids, feats, mask, args.new, V)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            t0 = time.perf_counter()
            out = model.generate(ids, feats, mask, max_new_tokens=args.new, bos_token_id=1, **kw)
            torch.cuda.synchronize()
            r["generate_tokens_per_s"] = B * args.new / (time.perf_counter() - t0)
            r["generate_peak_gb"] = torch.cuda.max_memory_allocated() / 1e9
            assert out.shape == (B, T + args.new)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            model.generate_many(utts, batch_size=12, max_new_tokens=budgets, **kw)
            e1.record()
            torch.cuda.synchronize()
            r["generate_many_tokens_per_s"] = sum(budgets) / (e0.elapsed_time(e1) / 1e3)
            arms[arm].append(r)
            print(rep, arm, json.dumps(r), flush=True)
    for arm, rs in arms.items():
        res[arm] = {k: median([r[k] for r in rs]) for k in rs[0]}
        res[arm]["all"] = rs
    res["step_speedup"] = res["bf16"]["step_ms"] / res["fp8"]["step_ms"]
    res["gpu_after"] = gpu_info()
    with open(os.path.join(args.out, "time_fp8_decode.json"), "w") as fh:
        json.dump(res, fh, indent=2)
    print(json.dumps({k: v for k, v in res.items() if k not in ("bf16", "fp8")}, indent=2))
    print(json.dumps({a: {k: v for k, v in res[a].items() if k != "all"} for a in ("bf16", "fp8")}, indent=2))


if __name__ == "__main__":
    main()
