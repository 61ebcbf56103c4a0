"""Time greedy KV-cache decoding (touchnet_b200/generation.py) on the Llama-3.2-3B-ASR configuration of bench.py at the
reference's evaluation batch (B = 12, inference_touch_audio.py --batch_size), against stock HF LlamaForCausalLM.generate
(bf16, sdpa) on the same weights and prompts.

    python tools/time_decode.py --out DIR [--batch 12] [--new 256]

Prompts: seeded 1-30 s utterances at fbank80 stack 5 / stride 4 (<= 750 feature rows) + one `<bos>` row, left-padded;
random bf16 weights; eos unreachable, so every run decodes exactly --new tokens.  Writes DIR/time_decode.json with
  prefill ms, median decode ms per step, decode tokens/s (CUDA events around graph replays),
  per-kernel device time of one decode step (torch.profiler over eager decode steps, in a run of its own),
  decode-attention bytes/s (K+V bytes read / attention kernel time) and decode-GEMM bytes/s (weight bytes / GEMM kernel
  time), each next to the H100 SXM data-sheet HBM3 bandwidth of 3.35 TB/s (a data-sheet figure, not a measurement),
  the same generate through HF LlamaForCausalLM (input_ids + inputs_embeds) as the incumbent,
  and the card name, power limit and SM clocks read in the same run."""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from touchnet_b200 import generation, modeling, ops  # noqa: E402

DATASHEET_HBM_BPS = 3.35e12


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))
    except Exception as e:     # still report what torch knows
        return {"name": torch.cuda.get_device_name(), "error": str(e)}


def prompts(B, seed, vocab, dev):
    g = torch.Generator().manual_seed(seed)
    secs = [1 + 29 * float(torch.rand((), generator=g)) for _ in range(B)]
    rows = [math.ceil((1 + (int(s * 16000) - 400) // 160) / bench.STRIDE) for s in secs]   # fbank frames -> stacked rows
    T = max(rows) + 1
    ids = torch.zeros(B, T, dtype=torch.int64)
    mask = torch.zeros(B, T, dtype=torch.int64)
    feats = torch.zeros(B, T, bench.MEL * bench.STACK)
    for b, r in enumerate(rows):
        feats[b, T - 1 - r:T - 1] = torch.randn(r, feats.shape[-1], generator=g)
        ids[b, T - 1] = 1                         # <bos>
        mask[b, T - 1 - r:] = 1
    return ids.to(dev), feats.to(dev, torch.bfloat16), mask.to(dev), rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--batch", type=int, default=12)
    ap.add_argument("--new", type=int, default=256)
    ap.add_argument("--layers", type=int, default=28)
    ap.add_argument("--seed", type=int, default=2025)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_decode.py measures the GPU: no CUDA device")
    os.makedirs(args.out, exist_ok=True)
    dev = torch.device("cuda")
    cfg = bench.asr_config(args.layers)
    tc = cfg.text_config
    torch.manual_seed(args.seed)
    with torch.device(dev):
        model = modeling.B200TouchAudioForCausalLM(cfg).to(torch.bfloat16)
    with torch.no_grad():
        for p in model.parameters():
            p.normal_(0, 0.02) if p.dim() == 2 else p.fill_(1.0)
    B, V = args.batch, tc.vocab_size
    ids, feats, mask, rows = prompts(B, args.seed, V, dev)
    T = ids.shape[1]
    kw = dict(eos_token_id=V, pad_token_id=0, bos_token_id=1, repetition_penalty=1.5, no_repeat_ngram_size=2,
              do_sample=False, num_beams=1, use_cache=True)
    res = {"workload": f"{bench._W['name']} decode: B={B}, prompt T={T} (left-padded, rows {min(rows)}..{max(rows)} "
                       f"+ <bos>), {args.new} new tokens, eos unreachable, bf16 weights",
           "gpu": gpu_info()}

    # ---- end to end: generate (prefill + eager step + graph replays) ----
    for _ in range(2):
        out = model.generate(ids, feats, mask, max_new_tokens=args.new, **kw)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = model.generate(ids, feats, mask, max_new_tokens=args.new, **kw)
    torch.cuda.synchronize()
    res["generate_s"] = time.perf_counter() - t0
    assert out.shape == (B, T + args.new)

    # ---- prefill and decode step with CUDA events ----
    w = generation._Weights(model.language_model)
    ev = lambda: torch.cuda.Event(enable_timing=True)  # noqa: E731
    pre = []
    with torch.no_grad():
        for _ in range(5):
            cache = generation.B200KVCache(model, B, T + args.new)
            e0, e1 = ev(), ev()
            e0.record()
            logits = generation.prefill(model, cache, ids, feats, mask, None, weights=w)
            e1.record()
            torch.cuda.synchronize()
            pre.append(e0.elapsed_time(e1))

        def select(lg):
            ops.greedy_select(lg, cache.history, cache.kv_end, cache.positions, cache.next_ids, cache.finished, 1.5, 2,
                              V, 0)

        select(logits)
        select(generation.decode_step(model, cache, weights=w))
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            select(generation.decode_step(model, cache, weights=w))
        steps = []
        for _ in range(args.new - 2):
            e0, e1 = ev(), ev()
            e0.record(); g.replay(); e1.record()
            steps.append((e0, e1))
        torch.cuda.synchronize()
        step_ms = sorted(a.elapsed_time(b) for a, b in steps)
        del g
    res["prefill_ms"] = sorted(pre)[len(pre) // 2]
    res["decode_ms_per_step_median"] = step_ms[len(step_ms) // 2]
    res["decode_tokens_per_s"] = B * 1000.0 / res["decode_ms_per_step_median"]
    res["generate_tokens_per_s"] = B * args.new / res["generate_s"]

    # ---- per-kernel times: torch.profiler over eager decode steps, separate run ----
    from torch.profiler import ProfilerActivity, profile
    n_prof = 8
    with torch.no_grad():
        cache = generation.B200KVCache(model, B, T + args.new)
        select(generation.prefill(model, cache, ids, feats, mask, None, weights=w))
        for _ in range(3):
            select(generation.decode_step(model, cache, weights=w))
        torch.cuda.synchronize()
        kv_len = int(cache.kv_end[0]) + 1         # mean attended length over the profiled steps is computed below
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(n_prof):
                select(generation.decode_step(model, cache, weights=w))
            torch.cuda.synchronize()
    kern = {}
    for e in prof.key_averages():
        if e.device_type.name == "CUDA" or getattr(e, "self_device_time_total", 0) > 0:
            t = getattr(e, "self_device_time_total", None)
            if t is None:
                t = e.self_cuda_time_total
            if t > 0:
                kern[e.key] = kern.get(e.key, 0.0) + t / 1000.0 / n_prof      # ms per step
    res["kernel_ms_per_step"] = dict(sorted(kern.items(), key=lambda kv: -kv[1]))
    prof.export_chrome_trace(os.path.join(args.out, "decode_trace.json"))
    attn_ms = sum(v for k, v in kern.items() if "attn_decode" in k)
    gemm_ms = sum(v for k, v in kern.items() if "gemm" in k.lower())
    start = [T - r - 1 for r in rows]
    mean_len = sum(kv_len + n_prof / 2 - s for s in start) / B
    KV, L, d, f = tc.num_key_value_heads, tc.num_hidden_layers, tc.hidden_size, tc.intermediate_size
    H = tc.num_attention_heads
    kv_bytes = L * B * mean_len * KV * 128 * 2 * 2
    w_bytes = (L * (d * H * 128 + 2 * d * KV * 128 + H * 128 * d + 3 * d * f) + V * d) * 2
    res["decode_attention"] = {"ms_per_step": attn_ms, "kv_bytes_per_step": kv_bytes,
                               "bytes_per_s": kv_bytes / (attn_ms / 1e3) if attn_ms else None,
                               "fraction_of_datasheet_3.35TBps": kv_bytes / (attn_ms / 1e3) / DATASHEET_HBM_BPS
                               if attn_ms else None}
    res["decode_gemm"] = {"ms_per_step": gemm_ms, "weight_bytes_per_step": w_bytes,
                          "bytes_per_s": w_bytes / (gemm_ms / 1e3) if gemm_ms else None,
                          "fraction_of_datasheet_3.35TBps": w_bytes / (gemm_ms / 1e3) / DATASHEET_HBM_BPS
                          if gemm_ms else None}
    res["datasheet_floor_ms_per_step"] = (w_bytes + kv_bytes) / DATASHEET_HBM_BPS * 1e3

    # ---- incumbent: stock HF LlamaForCausalLM.generate, bf16, sdpa, input_ids + inputs_embeds ----
    try:
        from transformers import LlamaConfig, LlamaForCausalLM
        hcfg = LlamaConfig(hidden_size=d, intermediate_size=f, num_hidden_layers=L, num_attention_heads=H,
                           num_key_value_heads=KV, head_dim=128, vocab_size=V, rms_norm_eps=tc.rms_norm_eps,
                           rope_theta=tc.rope_theta, rope_scaling=tc.rope_scaling, tie_word_embeddings=False,
                           pad_token_id=0, attn_implementation="sdpa")
        with torch.device(dev):
            hf = LlamaForCausalLM(hcfg).to(torch.bfloat16).eval()
        sd = {k[len("language_model."):]: v for k, v in model.state_dict().items() if k.startswith("language_model.")}
        hf.load_state_dict(sd)
        with torch.no_grad():
            emb = hf.model.embed_tokens(ids) + torch.nn.functional.linear(feats, model.projector.weight)
            hkw = dict(kw, max_new_tokens=args.new)
            hf.generate(input_ids=ids, inputs_embeds=emb, attention_mask=mask, **dict(hkw, max_new_tokens=4))
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            hout = hf.generate(input_ids=ids, inputs_embeds=emb, attention_mask=mask, **hkw)
            torch.cuda.synchronize()
            hs = time.perf_counter() - t0
        n_new = hout.shape[1] - (T if hout.shape[1] > args.new else 0)
        res["incumbent_hf_generate"] = {"s": hs, "new_tokens": n_new, "tokens_per_s": B * n_new / hs}
        res["speedup_vs_hf_generate"] = hs / res["generate_s"] * (args.new / max(n_new, 1))
    except Exception as e:      # the incumbent is a comparison, not the measurement itself
        res["incumbent_hf_generate"] = {"error": repr(e)}
    res["gpu_after"] = gpu_info()
    with open(os.path.join(args.out, "time_decode.json"), "w") as fh:
        json.dump(res, fh, indent=2)
    print(json.dumps({k: v for k, v in res.items() if k != "kernel_ms_per_step"}, indent=2))


if __name__ == "__main__":
    main()
