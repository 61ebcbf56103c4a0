"""GPU: continuous batching (tn_kv_scatter_bf16, tn_slot_admit, tn_greedy_select_slots_bf16 in
touchnet_b200/csrc/decode.cu; generation.generate_many).

  scatter     bit-exact copy into the named slots' rows [0, len); every other cache row unchanged
  admission   slot state and history of the named slots only
  selection   vs HF RepetitionPenaltyLogitsProcessor + NoRepeatNGramLogitsProcessor + torch.argmax at V = 128256, exact;
              finished / idle slots do not move, the limit finishes a slot on its last budgeted token
  invariance  on the Llama-3.2-3B-ASR geometry (2 layers, random weights) a prompt's cache rows, first-token logits
              and generated ids are bit-identical alone or packed with neighbours, in slot 0 or slot B-1, admitted first
              or after other rows finished
  semantics   tokens equal per-prompt `generate` up to near-ties on the reference inference layout (TouchAudio, GPU
              fbank features); a NaN in a prompt's features raises ValueError("NaN in data.")
  replay      graph replay bit-identical to eager steps; kv_end <= S_cap after many refills; two runs bit-identical"""
import math

import pytest
import torch

from tests.gpu_util import require_cuda
from tests.test_gpu_model import small_cfg
from touchnet_b200 import generation, modeling, ops

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16


def test_kv_scatter_is_a_bit_exact_copy_into_the_named_slots():
    dev = require_cuda()
    B, S_cap, KV = 4, 300, 2
    cache = torch.randn(2, B, S_cap, KV * 128, device=dev).to(BF16)
    before = cache.clone()
    qkv = torch.randn(512, 3 * KV * 128, device=dev).to(BF16)               # strided k / v columns of a fused output
    k, v = qkv[:, KV * 128:2 * KV * 128], qkv[:, 2 * KV * 128:]
    docs = [(0, 3, 100, 101), (128, 0, 256, 300), (384, 2, 1, 2)]
    ops.kv_scatter(k, v, cache[0], cache[1], docs)
    expect = before.clone()
    for src, slot, n, _ in docs:
        expect[0, slot, :n] = k[src:src + n]
        expect[1, slot, :n] = v[src:src + n]
    assert torch.equal(cache, expect)


def test_slot_admit_sets_only_the_named_slots():
    dev = require_cuda()
    B, S_cap = 5, 64
    hist = torch.randint(0, 50, (B, S_cap), device=dev)
    state = dict(kv_start=torch.full((B,), 7, dtype=torch.int32, device=dev),
                 kv_end=torch.full((B,), 9, dtype=torch.int32, device=dev),
                 positions=torch.full((B,), 11, dtype=torch.int64, device=dev),
                 finished=torch.ones(B, dtype=torch.int32, device=dev),
                 limit=torch.full((B,), 13, dtype=torch.int32, device=dev))
    old_hist = hist.clone()
    ids = torch.randint(3, 90, (256,), device=dev)
    doc = torch.cat([torch.full((20,), 1), torch.full((108,), 2), torch.full((40,), 130), torch.full((88,), 131)])
    doc = doc.to(dev, torch.int32)
    pos = torch.arange(256, device=dev) % 97
    ops.slot_admit([(0, 3, 60, 63), (128, 1, 40, 64)], ids, doc, pos, hist, state["kv_start"], state["kv_end"],
                   state["positions"], state["finished"], state["limit"])
    assert state["kv_start"].tolist() == [7, 0, 7, 20, 7]       # slot 3: its last document starts at row 20
    assert state["kv_end"].tolist() == [9, 40, 9, 60, 9]
    assert state["positions"].tolist() == [11, int(pos[167]), 11, int(pos[59]), 11]
    assert state["finished"].tolist() == [1, 0, 1, 0, 1]
    assert state["limit"].tolist() == [13, 64, 13, 63, 13]
    assert torch.equal(hist[3, :60], ids[:60]) and torch.equal(hist[3, 60:], old_hist[3, 60:])
    assert torch.equal(hist[1, :40], ids[128:168]) and torch.equal(hist[1, 40:], old_hist[1, 40:])
    for s in (0, 2, 4):
        assert torch.equal(hist[s], old_hist[s])


def test_greedy_select_slots_matches_hf_processors_and_respects_slot_state():
    from transformers.generation.logits_process import NoRepeatNGramLogitsProcessor, RepetitionPenaltyLogitsProcessor
    dev = require_cuda()
    V, B, S_cap = 128256, 6, 64
    g = torch.Generator(device="cpu").manual_seed(V)
    hist = torch.randint(0, 50, (B, S_cap), generator=g).to(dev)
    lens = torch.tensor([37, 20, 45, 30, 12, 50], dtype=torch.int32)
    for b in range(B):
        n = int(lens[b])
        hist[b, n - 2:n] = hist[b, 3:5]                                      # the last bigram occurred before
    logits = (torch.randn(4, V, generator=g) * 3).to(BF16).to(dev)
    logits[0, 7] = logits[0, 9] = logits[0].float().max() + 1               # planted tie: the lower index wins
    row_slot = [4, 0, 5, 2]                                                  # slot 5 finished, 1 and 3 not named
    fin = torch.tensor([0, 0, 0, 1, 0, 1], dtype=torch.int32, device=dev)
    limit = (lens + 10).to(dev, torch.int32)
    limit[2] = int(lens[2]) + 1                                              # slot 2 takes its last budgeted token
    length = lens.to(dev)
    pos = torch.arange(B, dtype=torch.int64, device=dev) + 100
    nxt = torch.full((B,), -5, dtype=torch.int64, device=dev)
    h = hist.clone()
    eos, pad = -1, 0
    ops.greedy_select_slots(logits, h, length, pos, nxt, fin, limit, 1.5, 2, eos, pad, row_slot=row_slot)
    for r, b in enumerate(row_slot):
        n = int(lens[b])
        s = RepetitionPenaltyLogitsProcessor(1.5)(hist[b:b + 1, :n], logits[r:r + 1].float())
        s = NoRepeatNGramLogitsProcessor(2)(hist[b:b + 1, :n], s)
        if b == 5:                                                           # finished: nothing moves, pad fed next
            assert int(nxt[b]) == pad and int(length[b]) == n and int(pos[b]) == 100 + b
            assert torch.equal(h[b], hist[b])
            continue
        tok = int(s.argmax())
        assert int(nxt[b]) == tok and int(h[b, n]) == tok and int(length[b]) == n + 1 and int(pos[b]) == 101 + b
        assert torch.equal(h[b, :n], hist[b, :n]) and torch.equal(h[b, n + 1:], hist[b, n + 1:])
    for b in (1, 3):                                                         # not named: untouched
        assert int(nxt[b]) == -5 and int(length[b]) == int(lens[b]) and torch.equal(h[b], hist[b])
    assert fin.tolist() == [0, 0, 1, 1, 0, 1]                                # the limit finished slot 2
    # the identity map over all B rows (the decode step): idle / finished slots 2, 3, 5 hold still
    logits6 = (torch.randn(B, V, generator=g) * 3).to(BF16).to(dev)
    snap = [t.clone() for t in (h, length, pos)]
    ops.greedy_select_slots(logits6, h, length, pos, nxt, fin, limit, 1.5, 2, eos, pad)
    for b in range(B):
        if fin[b] and b in (2, 3, 5):
            assert int(nxt[b]) == pad and int(length[b]) == int(snap[1][b]) and int(pos[b]) == int(snap[2][b])
            assert torch.equal(h[b], snap[0][b])
        else:
            assert int(length[b]) == int(snap[1][b]) + 1


# ---------------------------------------------------------------------------------------------------------------
# the model-level tests
# ---------------------------------------------------------------------------------------------------------------
def _asr_model(dev, layers=2):
    import bench
    torch.manual_seed(0)
    cfg = bench.asr_config(layers)
    with torch.device(dev):
        model = modeling.B200TouchAudioForCausalLM(cfg).to(BF16)
    with torch.no_grad():
        for p in model.parameters():
            p.normal_(0, 0.02) if p.dim() == 2 else p.fill_(1.0)
    return model, cfg


def _asr_prompt(T, seed, dev, F=400):
    g = torch.Generator().manual_seed(seed)
    ids = torch.zeros(T, dtype=torch.int64)
    ids[-1] = 1                                                              # <bos> under a zero feature row
    feats = torch.randn(T, F, generator=g)
    feats[-1] = 0
    return {"input_ids": ids.to(dev), "input_features": feats.to(dev, BF16)}


@pytest.mark.parametrize("T", [300, 100])        # >= 256 rows and one short prompt (below the fused-QKV threshold alone)
def test_prompt_is_bit_invariant_to_packing_slot_and_admission_time(monkeypatch, T):
    dev = require_cuda()
    model, cfg = _asr_model(dev)
    V = cfg.text_config.vocab_size
    P = _asr_prompt(T, 1, dev)
    others = [_asr_prompt(n, 10 + i, dev) for i, n in enumerate((130, 257, 40, 200))]
    seen = {}
    real = generation._admit

    def spy(model_, cache, limit, w, batch, pad, select):
        def rec(logits, slots):
            for (slot, p), r in zip(batch, range(logits.shape[0])):
                if p.ids.numel() == T and torch.equal(p.feats, P["input_features"]):
                    seen.setdefault("logits", []).append(logits[r].clone())
                    seen.setdefault("rows", []).append(cache.data[:, :, slot, :T].clone())
                    seen.setdefault("slot", []).append(slot)
            select(logits, slots)
        real(model_, cache, limit, w, batch, pad, rec)

    monkeypatch.setattr(generation, "_admit", spy)
    kw = dict(batch_size=3, eos_token_id=V, pad_token_id=0, repetition_penalty=1.5, no_repeat_ngram_size=2,
              max_prompt_length=300)
    runs = [
        ([P], [24]),                                                  # alone, slot 0, first admission
        ([others[0], others[1], P], [5, 24, 24]),                     # packed with two neighbours, slot B-1
        ([others[0], others[1], others[2], P], [3, 24, 24, 24]),      # admitted later, alone, into slot 0
        ([others[2], others[0], others[1], others[3], P], [2, 2, 24, 24, 24]),   # later, packed with a neighbour
    ]
    outs = []
    for prompts, budgets in runs:
        outs.append(model.generate_many(prompts, max_new_tokens=budgets, **kw)[-1])
    assert seen["slot"] == [0, 2, 0, 1]
    for i in range(1, len(runs)):
        assert torch.equal(seen["logits"][i], seen["logits"][0]), i
        assert torch.equal(seen["rows"][i], seen["rows"][0]), i
        assert torch.equal(outs[i], outs[0]), (i, outs[i], outs[0])
    assert outs[0].numel() == 24


def _processed(seq, logits, penalty=1.5, ngram=2):
    from transformers.generation.logits_process import NoRepeatNGramLogitsProcessor, RepetitionPenaltyLogitsProcessor
    s = RepetitionPenaltyLogitsProcessor(penalty)(seq, logits.float().clone())
    return NoRepeatNGramLogitsProcessor(ngram)(seq, s)


def _touch_audio_small(dev):
    from types import SimpleNamespace as NS
    torch.manual_seed(0)
    text = small_cfg(d=256, H=2, KV=1, V=320)
    cfg = NS(audio_config=NS(input_size=400), text_config=text, pad_token_id=0)
    model = modeling.B200TouchAudioForCausalLM(cfg).to(dev)
    model.post_init()
    with torch.no_grad():
        for p in model.parameters():
            if p.dim() == 2:
                p.normal_(0, 0.05)
    return model.to(BF16)


def _fbank_prompts(dev, seconds):
    """GPU fbank -> stack 5 / stride 4 rows + one zero row under <bos> (ref: inference_touch_audio.py:62-76), unpadded."""
    from touchnet_b200 import frontend
    g = torch.Generator().manual_seed(1)
    wavs = [0.3 * (2 * torch.rand(int(16000 * s), generator=g) - 1) for s in seconds]
    flat, lens = frontend._pack(wavs, dev)
    fb, frames = frontend.fbank_batch(flat, lens)
    rows = [int(math.ceil(f / 4)) for f in frames]
    packed = torch.zeros(sum(rows), 400, device=dev)
    frontend.stack_batch(fb, frames, 5, 4, True, into=packed, dst_rows=[sum(rows[:i]) for i in range(len(rows))])
    out = []
    for i, r in enumerate(rows):
        o = sum(rows[:i])
        ids = torch.zeros(r + 1, dtype=torch.int64, device=dev)
        ids[-1] = 1
        feats = torch.zeros(r + 1, 400, device=dev)
        feats[:r] = packed[o:o + r]
        out.append({"input_ids": ids, "input_features": feats, "attention_mask": torch.ones_like(ids)})
    return out


def test_generate_many_matches_per_prompt_generate_up_to_near_ties():
    dev = require_cuda()
    model = _touch_audio_small(dev)
    prompts = _fbank_prompts(dev, [2.0, 1.25, 3.0, 0.8, 2.6, 1.7, 0.5])
    budgets = [12, 5, 16, 3, 9, 14, 7]
    eos, pad = 2, 0
    kw = dict(eos_token_id=eos, pad_token_id=pad, repetition_penalty=1.5, no_repeat_ngram_size=2)
    got = model.generate_many(prompts, batch_size=3, max_new_tokens=budgets, **kw)
    for i, (p, n) in enumerate(zip(prompts, budgets)):
        ids, feats = p["input_ids"][None], p["input_features"][None]
        ref = model.generate(ids, feats, p["attention_mask"][None], max_new_tokens=n, bos_token_id=1, **kw)[0]
        T = ids.shape[1]
        ref = ref[T:]
        if (ref == eos).any():
            ref = ref[:int((ref == eos).nonzero()[0]) + 1]
        m = min(ref.numel(), got[i].numel())
        diff = (got[i][:m] != ref[:m]).nonzero()
        if diff.numel() == 0:
            assert got[i].numel() == ref.numel(), i
            continue
        j = int(diff[0])                   # the first divergence must be a near-tie of the processed scores
        seq = torch.cat([ids[0], ref[:j]])[None]
        f = torch.cat([feats[0], torch.zeros(j, 400, device=dev)])[None]
        with torch.no_grad():
            lg = model(input_ids=seq, input_features=f, attention_mask=torch.ones_like(seq)).logits[0, -1].float()
        s = _processed(seq, lg[None])[0]
        margin = abs(float(s[int(ref[j])] - s[int(got[i][j])]))
        assert margin <= 3e-2 * float(lg.abs().max()) + 1e-3, (i, j, margin)


def test_nan_in_a_prompts_features_raises():
    dev = require_cuda()
    model = _touch_audio_small(dev)
    prompts = _fbank_prompts(dev, [1.0, 1.5, 0.7])
    prompts[2]["input_features"][3, 5] = float("nan")
    with pytest.raises(ValueError, match="NaN in data."):
        model.generate_many(prompts, batch_size=2, max_new_tokens=6, eos_token_id=2, pad_token_id=0)
    assert int(model._nan_flag.item()) == 0


def test_graph_replay_equals_eager_steps_and_runs_are_reproducible(monkeypatch):
    dev = require_cuda()
    model = _touch_audio_small(dev)
    g = torch.Generator().manual_seed(5)
    prompts = []
    for i in range(24):
        T = int(torch.randint(2, 140, (), generator=g))
        ids = torch.randint(3, 320, (T,), generator=g)
        ids[-1] = 1
        prompts.append({"input_ids": ids.to(dev), "input_features": torch.randn(T, 400, generator=g).to(dev, BF16)})
    budgets = [int(torch.randint(1, 40, (), generator=g)) for _ in prompts]
    caches = []

    class Recorded(generation.B200KVCache):
        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            caches.append(self)

    monkeypatch.setattr(generation, "B200KVCache", Recorded)
    kw = dict(batch_size=5, max_new_tokens=budgets, eos_token_id=2, pad_token_id=0, repetition_penalty=1.5,
              no_repeat_ngram_size=2)
    graph = model.generate_many(prompts, **kw)
    graph2 = model.generate_many(prompts, **kw)
    eager = model.generate_many(prompts, cuda_graph=False, **kw)
    for a, b, c, n in zip(graph, graph2, eager, budgets):
        assert torch.equal(a, b) and torch.equal(a, c)
        assert 1 <= a.numel() <= n and (a.numel() == n or int(a[-1]) == 2)
    for cache in caches:
        assert int(cache.kv_end.max()) <= cache.S_cap
