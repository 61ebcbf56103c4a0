"""Time the sampling selection (`tn_sample_select_slots_bf16`) against the greedy one, per launch and inside
`generate_many`, on the Llama-3.2-3B-ASR configuration of bench.py (V = 128256).

    python tools/time_sample.py --out DIR [--n 96] [--batch 12] [--reps 3] [--launches 200]

  kernel   per-launch time of greedy_select_slots and sample_select_slots at B in {12, 32, 64}: CUDA events over
           --launches warmed launches, repetition_penalty=1.5, no_repeat_ngram_size=2, a history of 711 prompt + 256
           generated ids; logits bf16 N(0, 2.5^2).  Sampling at temperature=0.7, top_k=50, top_p=0.9 (the reference's
           evaluation knobs) and at top_k=0, top_p=0.9 (top-p over the whole vocabulary, the slowest case).  The arms
           alternate --reps times; the median is reported.
  many     generate_many tokens/s, greedy against do_sample=True (0.7, 50, 0.9), on the 96-utterance workload of
           tools/time_generate_many.py, alternating in the same run.

The card name, power limit and SM clocks are read in the same run.  Writes DIR/time_sample.json."""
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
from tools.time_generate_many import TOKENS_PER_SECOND, median, run_many, utterances  # noqa: E402
from touchnet_b200 import modeling, ops  # noqa: E402

HIST = 711 + 256
ARMS = {"greedy": None, "sample_k50_p0.9": (0.7, 50, 0.9), "sample_k0_p0.9": (0.7, 0, 0.9)}


def time_kernels(V, B, launches, reps, dev):
    g = torch.Generator().manual_seed(B)
    logits = (torch.randn(B, V, generator=g) * 2.5).to(dev, torch.bfloat16)
    S = HIST + launches + 8
    hist0 = torch.randint(0, V, (B, S), generator=g).to(dev)
    state = dict(history=hist0.clone(), length=torch.full((B,), HIST, dtype=torch.int32, device=dev),
                 positions=torch.zeros(B, dtype=torch.int64, device=dev),
                 next_ids=torch.zeros(B, dtype=torch.int64, device=dev),
                 finished=torch.zeros(B, dtype=torch.int32, device=dev),
                 limit=torch.full((B,), S, dtype=torch.int32, device=dev))
    key = torch.arange(B, dtype=torch.int64, device=dev)

    def launch(arm):
        s = state
        if ARMS[arm] is None:
            ops.greedy_select_slots(logits, s["history"], s["length"], s["positions"], s["next_ids"], s["finished"],
                                    s["limit"], 1.5, 2, -1, 0)
        else:
            t, k, p = ARMS[arm]
            ops.sample_select_slots(logits, s["history"], s["length"], s["positions"], s["next_ids"], s["finished"],
                                    s["limit"], key, 1.5, 2, t, k, p, 1234, -1, 0)

    times = {a: [] for a in ARMS}
    for rep in range(reps + 1):                     # round 0 warms every arm
        for arm in ARMS:
            state["length"].fill_(HIST)
            for _ in range(5):
                launch(arm)
            state["length"].fill_(HIST)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(launches):
                launch(arm)
            e1.record()
            torch.cuda.synchronize()
            assert int(state["finished"].sum()) == 0
            if rep:
                times[arm].append(e0.elapsed_time(e1) * 1e3 / launches)
    return {a: {"us_median": median(t), "us_all": t} for a, t in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--n", type=int, default=96)
    ap.add_argument("--batch", type=int, default=12)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--layers", type=int, default=28)
    ap.add_argument("--seed", type=int, default=2025)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_sample.py measures the GPU: no CUDA device")
    os.makedirs(args.out, exist_ok=True)
    dev = torch.device("cuda")
    res = {"gpu": gpu_info()}
    cfg = bench.asr_config(args.layers)
    V = cfg.text_config.vocab_size
    res["kernel_us_per_launch"] = {f"B={B}": time_kernels(V, B, args.launches, args.reps, dev) for B in (12, 32, 64)}
    print(json.dumps(res, indent=2), flush=True)

    torch.manual_seed(args.seed)
    with torch.device(dev):
        model = modeling.B200TouchAudioForCausalLM(cfg).to(torch.bfloat16)
    with torch.no_grad():
        for p in model.parameters():
            p.normal_(0, 0.02) if p.dim() == 2 else p.fill_(1.0)
    secs, prompts = utterances(args.n, args.seed, dev)
    budgets = [math.ceil(TOKENS_PER_SECOND * s) for s in secs]
    B = args.batch
    useful = sum(budgets)
    base = dict(eos_token_id=V, pad_token_id=0, repetition_penalty=1.5, no_repeat_ngram_size=2)
    kws = {"greedy": base, "sampled": dict(base, do_sample=True, temperature=0.7, top_k=50, top_p=0.9)}
    res["workload"] = (f"{bench._W['name']}: {args.n} utterances of 1-30 s, batch {B}, bf16 random weights, eos "
                       f"unreachable, {useful} tokens (budget = ceil({TOKENS_PER_SECOND} * seconds))")
    with torch.no_grad():
        for kw in kws.values():                     # warm every shape of both arms
            run_many(model, prompts, budgets, B, kw)
        runs = {a: [] for a in kws}
        for _ in range(args.reps):
            for arm, kw in kws.items():
                runs[arm].append(run_many(model, prompts, budgets, B, kw)[1])
    for arm, rs in runs.items():
        wall = median([r["wall_ms"] for r in rs])
        res[f"many_{arm}"] = {"decode_steps": rs[0]["decode_steps"], "wall_ms_median": wall,
                              "wall_ms_all": [r["wall_ms"] for r in rs], "tokens_per_s": useful / (wall / 1e3),
                              "ms_per_decode_step": wall / rs[0]["decode_steps"]}
    res["sampled_over_greedy_wall"] = res["many_sampled"]["wall_ms_median"] / res["many_greedy"]["wall_ms_median"]
    res["gpu_after"] = gpu_info()
    with open(os.path.join(args.out, "time_sample.json"), "w") as fh:
        json.dump(res, fh, indent=2)
    print(json.dumps(res, indent=2))


if __name__ == "__main__":
    main()
