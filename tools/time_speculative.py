"""Time speculative decoding (generate with assistant_model, touchnet_b200/generation.py) at the workload of
tools/time_decode.py: the Llama-3.2-3B-ASR configuration of bench.py, B = 12 left-padded audio-length prompts, 256 new
tokens, eos unreachable, random bf16 weights; k = 1..4 draft tokens per round.

    python tools/time_speculative.py --out DIR [--batch 12] [--new 256] [--layers 28] [--draft-layers 2] [--runs 5]

Two drafts: the model itself (the same weights: close to the ceiling of the mechanism, but not every proposal is
accepted, since the draft's first step of a round rewrites the prompt's last cache row with the decode path's K/V and
random weights have many near-ties) and an unrelated random --draft-layers model of the same widths (acceptance
measured, not assumed; with random weights it says nothing about a trained pair).  Writes DIR/time_speculative.json
with, per k: the median time of one verify step (B*(k+1) rows: block, lm_head, verify selection) against one decode
step (B rows: block, lm_head, selection), both CUDA events around graph replays; the draft's one-token step time; per
draft, the mean number of tokens a row emits per round it takes part in (counted in a separate eager run that reads the
decoding state around each verify selection), the number of rounds (set by the row that finishes last), end-to-end
tokens/s of generate with and without the draft (median of --runs wall-clock runs each, the spread beside it), and
whether the outputs are identical; the card name, power limit and SM clocks read in the same run."""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from tools.time_decode import gpu_info, prompts  # noqa: E402
from touchnet_b200 import generation, modeling, ops  # noqa: E402


def _model(layers, seed, dev):
    torch.manual_seed(seed)
    with torch.device(dev):
        m = modeling.B200TouchAudioForCausalLM(bench.asr_config(layers)).to(torch.bfloat16)
    with torch.no_grad():
        for p in m.parameters():
            p.normal_(0, 0.02) if p.dim() == 2 else p.fill_(1.0)
    return m


def _replay_ms(fn, n):
    """Median ms of `fn` captured once in a CUDA graph (after one eager call), replayed n times."""
    fn()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(n)]
    for a, b in ev:
        a.record(); g.replay(); b.record()
    torch.cuda.synchronize()
    del g
    t = sorted(a.elapsed_time(b) for a, b in ev)
    return t[len(t) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--batch", type=int, default=12)
    ap.add_argument("--new", type=int, default=256)
    ap.add_argument("--layers", type=int, default=28)
    ap.add_argument("--draft-layers", type=int, default=2)
    ap.add_argument("--seed", type=int, default=2025)
    ap.add_argument("--runs", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_speculative.py measures the GPU: no CUDA device")
    os.makedirs(args.out, exist_ok=True)
    dev = torch.device("cuda")
    model = _model(args.layers, args.seed, dev)
    small = _model(args.draft_layers, args.seed + 1, dev)
    V = model.config.text_config.vocab_size
    B = args.batch
    ids, feats, mask, rows = prompts(B, args.seed, V, dev)
    T = ids.shape[1]
    kw = dict(eos_token_id=V, pad_token_id=0, bos_token_id=1, repetition_penalty=1.5, no_repeat_ngram_size=2,
              do_sample=False, num_beams=1, use_cache=True, max_new_tokens=args.new)
    res = {"workload": f"{bench._W['name']} decode ({args.layers} layers): B={B}, prompt T={T} (left-padded, rows "
                       f"{min(rows)}..{max(rows)} + <bos>), {args.new} new tokens, eos unreachable, random bf16 weights; "
                       f"drafts: the model itself and a random {args.draft_layers}-layer model",
           "gpu": gpu_info(),
           "note": "random weights: the 2-layer draft's acceptance says nothing about a trained model pair; speedups on "
                   "trained pairs are not measured here"}

    def timed(**extra):
        """(output, median s, [min s, max s]) over args.runs calls after one warm-up call."""
        out = model.generate(ids, feats, mask, **kw, **extra)
        ts = []
        for _ in range(args.runs):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            o = model.generate(ids, feats, mask, **kw, **extra)
            torch.cuda.synchronize()
            ts.append(time.perf_counter() - t0)
            assert torch.equal(o, out)
        ts.sort()
        return out, ts[len(ts) // 2], [ts[0], ts[-1]]

    ref, s_plain, spread = timed()
    res["generate_s_median"], res["generate_s_min_max"] = s_plain, spread
    res["generate_tokens_per_s"] = B * args.new / s_plain
    res["runs"] = args.runs

    def acceptance(d, k):
        """Eager rounds; per verify selection, the tokens each row that was not finished emitted.  Returns (mean
        tokens per row-round, rounds)."""
        emitted, rounds = [], [0]
        orig_sel, orig_cap = ops.verify_select, generation._captured

        def sel(logits, draft, history, length, positions, next_ids, finished, *a, **kw_):
            before, live = length.clone(), finished == 0
            out = orig_sel(logits, draft, history, length, positions, next_ids, finished, *a, **kw_)
            emitted.extend((length - before)[live].tolist())
            rounds[0] += 1
            return out

        ops.verify_select = sel
        generation._captured = lambda step, capture: orig_cap(step, False)
        try:
            model.generate(ids, feats, mask, **kw, assistant_model=d, num_assistant_tokens=k)
        finally:
            ops.verify_select, generation._captured = orig_sel, orig_cap
        return sum(emitted) / max(len(emitted), 1), rounds[0]

    w, wd = generation._Weights(model.language_model), generation._Weights(small.language_model)
    with torch.no_grad():
        # one decode step of the model and of the draft (block + lm_head + selection)
        caches = {}
        for name, m, wt in (("model", model, w), ("draft", small, wd)):
            c = generation.B200KVCache(m, B, T + 400)
            lg = generation.prefill(m, c, ids, feats, mask, None, weights=wt)
            sel = lambda lg, c=c: ops.greedy_select(lg, c.history, c.kv_end, c.positions, c.next_ids,  # noqa: E731
                                                    c.finished, 1.5, 2, V, 0)
            sel(lg)
            caches[name] = c
            res[f"{name}_decode_step_ms"] = _replay_ms(lambda m=m, c=c, wt=wt, sel=sel:
                                                       sel(generation.decode_step(m, c, weights=wt)), 50)
    res["per_k"] = {}
    for k in range(1, 5):
        r = {}
        with torch.no_grad():
            c = generation.B200KVCache(model, B, T + 400)
            ops.greedy_select(generation.prefill(model, c, ids, feats, mask, None, weights=w), c.history, c.kv_end,
                              c.positions, c.next_ids, c.finished, 1.5, 2, V, 0)
            drafts = torch.randint(3, V, (B, k), device=dev)
            limit = torch.full((B,), T + 400, dtype=torch.int32, device=dev)
            end = torch.zeros(B, dtype=torch.int32, device=dev)
            ar = torch.arange(k + 1, device=dev)
            ws = generation._multi_ws(c, k + 1, c.S_cap)

            def verify():
                torch.add(c.kv_end, k, out=end)
                x = generation._block_step(model, c, w, torch.cat([c.next_ids[:, None], drafts], 1),
                                           c.positions[:, None] + ar, end, ws, c.S_cap)
                ops.verify_select(generation._logits_last(w, x), drafts, c.history, c.kv_end, c.positions, c.next_ids,
                                  c.finished, limit, 1.5, 2, V, 0)

            r["verify_step_ms"] = _replay_ms(verify, 40 // (k + 1) * 2)
            r["verify_over_decode_step"] = r["verify_step_ms"] / res["model_decode_step_ms"]
        for name, d in (("self", model), (f"{args.draft_layers}_layer", small)):
            out, s, sp = timed(assistant_model=d, num_assistant_tokens=k)
            mean_tok, rounds = acceptance(d, k)
            r[name] = {"identical_to_generate": bool(torch.equal(out, ref)), "s_median": s, "s_min_max": sp,
                       "tokens_per_s": B * args.new / s, "speedup_vs_generate": s_plain / s, "rounds": rounds,
                       "mean_tokens_per_row_round": mean_tok}
        res["per_k"][k] = r
        print(json.dumps({k: r}), flush=True)
    res["gpu_after"] = gpu_info()
    with open(os.path.join(args.out, "time_speculative.json"), "w") as fh:
        json.dump(res, fh, indent=2)
    print(json.dumps(res, indent=2))


if __name__ == "__main__":
    main()
