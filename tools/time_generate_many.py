"""Time continuous batching (`generate_many`) against static batches of `generate` on a test set of utterances, on the
Llama-3.2-3B-ASR configuration of bench.py at the reference's evaluation batch (B = 12).

    python tools/time_generate_many.py --out DIR [--n 96] [--batch 12] [--reps 3]
    python tools/time_generate_many.py --out DIR --assistant {self,small} --num-assistant-tokens K [--do-sample]

Utterances: N seeded 1-30 s durations at fbank80 stack 5 / stride 4 (random feature rows) + one `<bos>` row; random
bf16 weights; `repetition_penalty=1.5, no_repeat_ngram_size=2`.  Random weights never reach eos, so every utterance gets
a token budget standing in for its transcript length: ceil(TOKENS_PER_SECOND * seconds).

  static   `generate` per batch of B consecutive utterances, left-padded, max_new_tokens = the batch's largest budget;
           only each utterance's budgeted tokens count as useful
  many     `generate_many(prompts, batch_size=B, max_new_tokens=budgets)`

Both arms run once to warm every shape (the admission prefill sizes included), then alternate --reps times.  Reported
per arm: decode steps, row-steps spent on finished rows, wall time (CUDA events around the whole call, host work
included), useful tokens/s, time in prefills (static) / admission prefills (many); the per-utterance agreement of the two
token streams; per-kernel device time of `generate_many` over the first 24 utterances with eager steps (torch.profiler,
a run of its own); the card name, power limit and SM clocks read in the same run.  Writes DIR/time_generate_many.json.

With --assistant (speculative decoding in generate_many) the two arms are instead
  many     `generate_many(prompts, batch_size=B, max_new_tokens=budgets)` (greedy, or sampled with --do-sample at the
           reference's knobs 0.7 / 50 / 0.9)
  draft    the same call with assistant_model = the model itself (self) or a random --draft-layers model (small) and
           num_assistant_tokens = K
alternating --reps times after one warm-up each.  Reported: wall time and useful tokens/s of both arms, rounds, live
row-rounds and tokens per live row-round of the draft arm (every token after each utterance's first comes from a
round), whether the greedy outputs equal the no-draft arm's bit for bit, and the device time per launch (CUDA events over
--launches launches, median of --reps) of the round's selection at B slots, V = 128256, a 967-id history: the greedy
verify selection (tn_verify_select_bf16) and the sampled one (tn_spec_sample_verify_bf16) against one
tn_sample_select_slots_bf16.  Writes DIR/time_generate_many_draft.json."""
import argparse
import json
import math
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from tools.time_decode import gpu_info  # noqa: E402
from touchnet_b200 import generation, modeling, ops  # noqa: E402

TOKENS_PER_SECOND = 4


def utterances(n, seed, dev):
    g = torch.Generator().manual_seed(seed)
    secs = [1 + 29 * float(torch.rand((), generator=g)) for _ in range(n)]
    out = []
    for s in secs:
        r = math.ceil((1 + (int(s * 16000) - 400) // 160) / bench.STRIDE)      # fbank frames -> stacked rows
        ids = torch.zeros(r + 1, dtype=torch.int64)
        ids[-1] = 1                                                           # <bos> under a zero feature row
        feats = torch.zeros(r + 1, bench.MEL * bench.STACK)
        feats[:r] = torch.randn(r, feats.shape[1], generator=g)
        out.append({"input_ids": ids.to(dev), "input_features": feats.to(dev, torch.bfloat16)})
    return secs, out


def left_padded(batch, dev):
    T = max(p["input_ids"].numel() for p in batch)
    B, F = len(batch), batch[0]["input_features"].shape[1]
    ids = torch.zeros(B, T, dtype=torch.int64, device=dev)
    mask = torch.zeros(B, T, dtype=torch.int64, device=dev)
    feats = torch.zeros(B, T, F, dtype=torch.bfloat16, device=dev)
    for b, p in enumerate(batch):
        t = p["input_ids"].numel()
        ids[b, T - t:] = p["input_ids"]
        feats[b, T - t:] = p["input_features"]
        mask[b, T - t:] = 1
    return ids, feats, mask


class PrefillTimer:
    """CUDA events around every generation.prefill call (the static arm's prefills)."""

    def __init__(self):
        self.events = []
        self.real = generation.prefill

    def __call__(self, *a, **k):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = self.real(*a, **k)
        e1.record()
        self.events.append((e0, e1))
        return out


def run_static(model, prompts, budgets, B, kw, dev):
    timer = PrefillTimer()
    generation.prefill = timer
    try:
        toks = []
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(0, len(prompts), B):
            chunk, bud = prompts[i:i + B], budgets[i:i + B]
            ids, feats, mask = left_padded(chunk, dev)
            out = model.generate(ids, feats, mask, max_new_tokens=max(bud), **kw)
            T = ids.shape[1]
            toks += [out[b, T:T + n] for b, n in enumerate(bud)]
        e1.record()
        torch.cuda.synchronize()
    finally:
        generation.prefill = timer.real
    steps = sum(max(budgets[i:i + B]) - 1 for i in range(0, len(budgets), B))
    idle = sum(max(budgets[i:i + B]) - n for i in range(0, len(budgets), B) for n in budgets[i:i + B])
    return toks, {"wall_ms": e0.elapsed_time(e1), "decode_steps": steps, "finished_row_steps": idle,
                  "prefill_ms": sum(a.elapsed_time(b) for a, b in timer.events), "prefills": len(timer.events)}


def run_many(model, prompts, budgets, B, kw):
    stats = {}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    toks = model.generate_many(prompts, batch_size=B, max_new_tokens=budgets, stats=stats, **kw)
    e1.record()
    torch.cuda.synchronize()
    steps = stats["decode_steps"]
    idle = B * steps - sum(n - 1 for n in budgets)          # eos is unreachable: utterance i decodes budget_i - 1 steps
    return toks, {"wall_ms": e0.elapsed_time(e1), "decode_steps": steps, "finished_row_steps": idle,
                  "prefill_ms": sum(a.elapsed_time(b) for a, b in stats["admission_events"]),
                  "prefills": stats["admissions"]}


def median(xs):
    return sorted(xs)[len(xs) // 2]


def random_model(layers, seed, dev):
    torch.manual_seed(seed)
    with torch.device(dev):
        model = modeling.B200TouchAudioForCausalLM(bench.asr_config(layers)).to(torch.bfloat16)
    with torch.no_grad():
        for p in model.parameters():
            p.normal_(0, 0.02) if p.dim() == 2 else p.fill_(1.0)
    return model


SAMPLE_KNOBS = dict(do_sample=True, temperature=0.7, top_k=50, top_p=0.9)
HIST = 711 + 256


def time_round_selections(V, B, k, launches, reps, dev):
    """Per-launch device time (us) of the round's selection at B slots: tn_verify_select_bf16 (greedy),
    tn_spec_sample_verify_bf16 (sampled, draft logits = target logits + noise) and one tn_sample_select_slots_bf16."""
    g = torch.Generator().manual_seed(B * 100 + k)
    logits = (torch.randn(B * (k + 1), V, generator=g) * 2.5).to(dev, torch.bfloat16)
    dlogits = (logits.view(B, k + 1, V)[:, :k].float().cpu() + torch.randn(B, k, V, generator=g)).reshape(B * k, V)
    dlogits = dlogits.to(dev, torch.bfloat16)
    drafts = torch.randint(0, V, (B, k), generator=g).to(dev)
    S = HIST + launches * (k + 1) + 8
    state = dict(history=torch.randint(0, V, (B, S), generator=g).to(dev),
                 length=torch.full((B,), HIST, dtype=torch.int32, device=dev),
                 positions=torch.zeros(B, dtype=torch.int64, device=dev),
                 next_ids=torch.zeros(B, dtype=torch.int64, device=dev),
                 finished=torch.zeros(B, dtype=torch.int32, device=dev),
                 limit=torch.full((B,), S, dtype=torch.int32, device=dev))
    key = torch.arange(B, dtype=torch.int64, device=dev)
    picks = torch.zeros((B, k + 1), dtype=torch.int64, device=dev)
    st = [state[n] for n in ("history", "length", "positions", "next_ids", "finished")]
    t, tk, tp = SAMPLE_KNOBS["temperature"], SAMPLE_KNOBS["top_k"], SAMPLE_KNOBS["top_p"]
    arms = {
        "verify_select_greedy": lambda: ops.verify_select(logits, drafts, *st, state["limit"], 1.5, 2, -1, 0,
                                                          picks=picks),
        "spec_sample_verify": lambda: ops.spec_sample_verify(logits, dlogits, drafts, *st, state["limit"], key, 1.5, 2,
                                                             t, tk, tp, 1234, -1, 0, picks=picks),
        "sample_select_slots": lambda: ops.sample_select_slots(logits[:B], *st, state["limit"], key, 1.5, 2, t, tk, tp,
                                                               1234, -1, 0),
    }
    times = {a: [] for a in arms}
    for rep in range(reps + 1):                     # round 0 warms every arm
        for arm, fn in arms.items():
            state["length"].fill_(HIST)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(launches):
                fn()
            e1.record()
            torch.cuda.synchronize()
            assert int(state["finished"].sum()) == 0
            if rep:
                times[arm].append(e0.elapsed_time(e1) * 1e3 / launches)
    return {a: {"us_median": median(v), "us_all": v} for a, v in times.items()}


def run_draft_arm(args, model, prompts, budgets, kw, dev, V):
    draft = model if args.assistant == "self" else random_model(args.draft_layers, args.seed + 1, dev)
    B, k = args.batch, args.num_assistant_tokens
    if args.do_sample:
        kw = dict(kw, **SAMPLE_KNOBS)
    dkw = dict(kw, assistant_model=draft, num_assistant_tokens=k)
    useful = sum(budgets)

    def timed(**extra):
        stats = {}
        torch.manual_seed(args.seed)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        toks = model.generate_many(prompts, batch_size=B, max_new_tokens=budgets, stats=stats, **extra)
        e1.record()
        torch.cuda.synchronize()
        return toks, stats, e0.elapsed_time(e1)

    res = {}
    with torch.no_grad():
        plain, _, _ = timed(**kw)                                          # warm-up of both arms
        spec, stats, _ = timed(**dkw)
        walls = {"many": [], "draft": []}
        for _ in range(args.reps):
            walls["many"].append(timed(**kw)[2])
            toks, _, ms = timed(**dkw)
            walls["draft"].append(ms)
            assert all(torch.equal(a, b) for a, b in zip(toks, spec)), "generate_many with a draft is not reproducible"
    emitted = sum(o.numel() - 1 for o in spec)                               # the first token is the admission's
    res["draft_arm"] = {"assistant": "self" if args.assistant == "self" else f"{args.draft_layers}_layer",
                        "num_assistant_tokens": k, "do_sample": bool(args.do_sample), "rounds": stats["rounds"],
                        "live_row_rounds": stats["live_row_rounds"],
                        "tokens_per_live_row_round": emitted / stats["live_row_rounds"]}
    if not args.do_sample:
        res["draft_arm"]["greedy_outputs_equal_no_draft_arm"] = sum(torch.equal(a, b) for a, b in zip(spec, plain))
        res["draft_arm"]["of"] = len(plain)
    for arm, ws in walls.items():
        res[arm] = {"wall_ms_median": median(ws), "wall_ms_all": ws,
                    "useful_tokens_per_s": useful / (median(ws) / 1e3)}
    res["draft_over_many_tokens_per_s"] = res["draft"]["useful_tokens_per_s"] / res["many"]["useful_tokens_per_s"]
    res["selection_us_per_launch"] = time_round_selections(V, B, k, args.launches, args.reps, dev)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--n", type=int, default=96)
    ap.add_argument("--batch", type=int, default=12)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--layers", type=int, default=28)
    ap.add_argument("--seed", type=int, default=2025)
    ap.add_argument("--assistant", choices=["self", "small"], default=None)
    ap.add_argument("--num-assistant-tokens", type=int, default=3)
    ap.add_argument("--draft-layers", type=int, default=2)
    ap.add_argument("--do-sample", action="store_true")
    ap.add_argument("--launches", type=int, default=100)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_generate_many.py measures the GPU: no CUDA device")
    os.makedirs(args.out, exist_ok=True)
    dev = torch.device("cuda")
    res = {"gpu": gpu_info()}
    V = bench.asr_config(args.layers).text_config.vocab_size
    model = random_model(args.layers, args.seed, dev)
    secs, prompts = utterances(args.n, args.seed, dev)
    budgets = [math.ceil(TOKENS_PER_SECOND * s) for s in secs]
    B = args.batch
    kw = dict(eos_token_id=V, pad_token_id=0, repetition_penalty=1.5, no_repeat_ngram_size=2)
    useful = sum(budgets)
    res["workload"] = (f"{bench._W['name']}: {args.n} utterances of 1-30 s ({min(secs):.1f}..{max(secs):.1f} s, "
                       f"{min(p['input_ids'].numel() for p in prompts)}..{max(p['input_ids'].numel() for p in prompts)} "
                       f"prompt rows incl. <bos>), batch {B}, bf16 random weights, eos unreachable")
    res["budget_rule"] = f"budget = ceil({TOKENS_PER_SECOND} * seconds) tokens per utterance; {useful} useful tokens"
    print(res["budget_rule"], flush=True)
    if args.assistant is not None:
        res.update(run_draft_arm(args, model, prompts, budgets, kw, dev, V))
        res["gpu_after"] = gpu_info()
        with open(os.path.join(args.out, "time_generate_many_draft.json"), "w") as fh:
            json.dump(res, fh, indent=2)
        print(json.dumps(res, indent=2))
        return

    with torch.no_grad():
        s_toks, _ = run_static(model, prompts, budgets, B, kw, dev)            # warm-up: every shape of both arms
        m_toks, _ = run_many(model, prompts, budgets, B, kw)
        runs = {"static": [], "many": []}
        for _ in range(args.reps):
            runs["static"].append(run_static(model, prompts, budgets, B, kw, dev)[1])
            toks, st = run_many(model, prompts, budgets, B, kw)
            runs["many"].append(st)
            assert all(torch.equal(a, b) for a, b in zip(toks, m_toks)), "generate_many is not reproducible"
    for arm, rs in runs.items():
        wall = median([r["wall_ms"] for r in rs])
        res[arm] = {"decode_steps": rs[0]["decode_steps"], "finished_row_steps": rs[0]["finished_row_steps"],
                    "row_steps": B * rs[0]["decode_steps"],
                    "finished_fraction": rs[0]["finished_row_steps"] / (B * rs[0]["decode_steps"]),
                    "wall_ms_median": wall, "wall_ms_all": [r["wall_ms"] for r in rs],
                    "useful_tokens_per_s": useful / (wall / 1e3),
                    "prefill_ms_median": median([r["prefill_ms"] for r in rs]), "prefill_calls": rs[0]["prefills"]}
    res["speedup_many_vs_static"] = res["static"]["wall_ms_median"] / res["many"]["wall_ms_median"]
    same, firsts = 0, []
    for i, (a, b) in enumerate(zip(s_toks, m_toks)):
        if torch.equal(a, b):
            same += 1
        else:
            firsts.append((i, int((a != b).nonzero()[0])))
    # a divergence must be a near-tie: at the first differing token, the uncached forward of the common prefix scores
    # the two picks (after the processors) within the decode tolerance of tests/test_gpu_decode.py
    from transformers.generation.logits_process import NoRepeatNGramLogitsProcessor, RepetitionPenaltyLogitsProcessor
    margins = []
    with torch.no_grad():
        for i, j in firsts:
            p, a, b = prompts[i], s_toks[i], m_toks[i]
            seq = torch.cat([p["input_ids"], a[:j]])[None]
            f = torch.cat([p["input_features"], p["input_features"].new_zeros(j, p["input_features"].shape[1])])[None]
            lg = model(input_ids=seq, input_features=f, attention_mask=torch.ones_like(seq)).logits[:, -1].float()
            sc = NoRepeatNGramLogitsProcessor(2)(seq, RepetitionPenaltyLogitsProcessor(1.5)(seq, lg.clone()))[0]
            margins.append((abs(float(sc[int(a[j])] - sc[int(b[j])])), 3e-2 * float(lg.abs().max()) + 1e-3))
    res["token_agreement"] = {"identical_utterances": same, "of": len(s_toks), "first_divergence (utt, token)": firsts,
                              "divergences_within_tolerance": sum(m <= t for m, t in margins),
                              "largest_margin_over_tolerance": max((m / t for m, t in margins), default=0.0)}

    # ---- per-kernel device time: generate_many on the first 24 utterances with eager decode steps, torch.profiler, a run of its own ----
    from torch.profiler import ProfilerActivity, profile
    with torch.no_grad(), profile(activities=[ProfilerActivity.CUDA]) as prof:
        model.generate_many(prompts[:24], batch_size=B, max_new_tokens=budgets[:24], cuda_graph=False, **kw)
        torch.cuda.synchronize()
    kern = {}
    for e in prof.key_averages():
        t = getattr(e, "self_device_time_total", None)
        if t is None:
            t = e.self_cuda_time_total
        if t > 0:
            kern[e.key] = kern.get(e.key, 0.0) + t / 1000.0
    res["profiled_many_kernel_ms"] = dict(sorted(kern.items(), key=lambda kv: -kv[1])[:25])
    res["gpu_after"] = gpu_info()
    with open(os.path.join(args.out, "time_generate_many.json"), "w") as fh:
        json.dump(res, fh, indent=2)
    print(json.dumps({k: v for k, v in res.items() if k != "profiled_many_kernel_ms"}, indent=2))


if __name__ == "__main__":
    main()
