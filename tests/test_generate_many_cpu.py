"""CPU: continuous batching (`generate_many`, touchnet_b200/generation.py) - argument checks of the three slot entry
points, validation of generate_many, and the host loop against transformers' LlamaForCausalLM.generate run on each
prompt alone.

The loop runs on CPU through plain-torch stand-ins: tests/cpu_ops_shim.py for the training ops, the decode stand-ins of
tests/test_generation_cpu.py, and, defined below, the three slot ops (the selection stand-in IS HF's pair of logits
processors + argmax).  What this checks is the loop: packed admission into chosen slots, refills at different steps,
idle slots while the queue drains, budgets, eos, the output order.  The kernels are checked on the GPU
(tests/test_gpu_generate_many.py)."""
import ctypes

import pytest
import torch

from tests.test_generation_cpu import _REF_KW, _attn_decode, _greedy_select, _kv_append, _models
from touchnet_b200 import _lib, generation, ops


# ---------------------------------------------------------------------------------------------------------------
# entry points: argument validation happens before any CUDA call
# ---------------------------------------------------------------------------------------------------------------
def _table(*rows):
    arr = (ctypes.c_int32 * max(1, 4 * len(rows)))(*[x for r in rows for x in r])
    return arr, ctypes.addressof(arr)


def test_slot_entry_points_reject_bad_arguments():
    p = ctypes.c_void_p(256)
    ok_arr, ok = _table((0, 1, 5, 9))
    bad_slot_arr, bad_slot = _table((0, 4, 5, 9))
    twice_arr, twice = _table((0, 1, 5, 9), (128, 1, 5, 9))
    long_arr, too_long = _table((0, 1, 65, 66))
    rows_arr, past_rows = _table((60, 1, 5, 9))
    lim_arr, bad_limit = _table((0, 1, 5, 5))
    map_arr = (ctypes.c_int32 * 2)(0, 7)
    kv = lambda K=p, ldk=128, docs=ok, n=1, ld_batch=128 * 64, rows=64: (    # noqa: E731
        K, ldk, p, 128, rows, p, p, 128, ld_batch, docs, n, 4, 64, 128, None)
    adm = lambda docs=ok, n=1, ids=p, B=4: (docs, n, ids, p, p, 64, p, 64, p, p, p, p, p, B, None)   # noqa: E731
    sel = lambda logits=p, n=4, m=None, B=4, ld=64, V=64, pen=1.5, ng=2: (                            # noqa: E731
        logits, ld, n, m, B, V, p, 16, p, p, p, p, p, pen, ng, 1, 0, None)
    bad_calls = [
        ("tn_kv_scatter_bf16", kv(K=None), "null"),
        ("tn_kv_scatter_bf16", kv(n=0), "bad dims"),
        ("tn_kv_scatter_bf16", kv(n=129), "bad dims"),
        ("tn_kv_scatter_bf16", kv(docs=bad_slot), "out of range"),
        ("tn_kv_scatter_bf16", kv(docs=twice, n=2, rows=256), "named twice"),
        ("tn_kv_scatter_bf16", kv(docs=too_long), "bad dims"),
        ("tn_kv_scatter_bf16", kv(docs=past_rows), "outside"),
        ("tn_kv_scatter_bf16", kv(ldk=64), "strides"),
        ("tn_kv_scatter_bf16", kv(ld_batch=128 * 63), "strides"),
        ("tn_kv_scatter_bf16", kv(K=ctypes.c_void_p(258)), "aligned"),
        ("tn_slot_admit", adm(ids=None), "null"),
        ("tn_slot_admit", adm(B=0), "bad dims"),
        ("tn_slot_admit", adm(docs=bad_slot), "out of range"),
        ("tn_slot_admit", adm(docs=bad_limit), "limit"),
        ("tn_slot_admit", adm(docs=too_long), "bad dims"),
        ("tn_greedy_select_slots_bf16", sel(logits=None), "null"),
        ("tn_greedy_select_slots_bf16", sel(ld=32), "bad dims"),
        ("tn_greedy_select_slots_bf16", sel(n=3), "bad dims"),
        ("tn_greedy_select_slots_bf16", sel(n=2, m=ctypes.addressof(map_arr)), "out of range"),
        ("tn_greedy_select_slots_bf16", sel(n=300, m=ctypes.addressof(map_arr), B=400), "at most"),
        ("tn_greedy_select_slots_bf16", sel(pen=0.0), "repetition_penalty"),
        ("tn_greedy_select_slots_bf16", sel(ng=-1), "no_repeat_ngram_size"),
        ("tn_greedy_select_slots_bf16", sel(ld=1 << 23, V=1 << 23, pen=1.0, ng=0), "too large"),
    ]
    for name, args, needle in bad_calls:
        with pytest.raises(_lib.TouchNetB200Error, match=needle):
            _lib.call(name, *args)
    del ok_arr, bad_slot_arr, twice_arr, long_arr, rows_arr, lim_arr


# ---------------------------------------------------------------------------------------------------------------
# plain-torch stand-ins of the three slot ops
# ---------------------------------------------------------------------------------------------------------------
def _kv_scatter(k, v, kc, vc, docs):
    for src, slot, n, _ in docs:
        kc[slot, :n] = k[src:src + n]
        vc[slot, :n] = v[src:src + n]


def _slot_admit(docs, ids, doc_ids, position_ids, history, kv_start, kv_end, positions, finished, limit):
    for src, slot, n, lim in docs:
        d = doc_ids[src:src + n]
        other = (d != d[-1]).nonzero()
        kv_start[slot] = int(other[-1]) + 1 if other.numel() else 0
        kv_end[slot] = n
        positions[slot] = position_ids[src + n - 1]
        history[slot, :n] = ids[src:src + n]
        finished[slot] = 0
        limit[slot] = lim


def _greedy_select_slots(logits, history, length, positions, next_ids, finished, limit, penalty, ngram, eos, pad,
                         row_slot=None):
    from transformers.generation.logits_process import NoRepeatNGramLogitsProcessor, RepetitionPenaltyLogitsProcessor
    for r in range(logits.shape[0]):
        b = r if row_slot is None else row_slot[r]
        if finished[b]:
            next_ids[b] = pad
            continue
        n = int(length[b])
        seq = history[b:b + 1, :n]
        scores = logits[r:r + 1].float()
        if penalty != 1.0:
            scores = RepetitionPenaltyLogitsProcessor(penalty)(seq, scores)
        if ngram > 0:
            scores = NoRepeatNGramLogitsProcessor(ngram)(seq, scores)
        tok = int(torch.argmax(scores, -1))
        history[b, n] = tok
        next_ids[b] = tok
        length[b] = n + 1
        positions[b] += 1
        if tok == eos or n + 1 == int(limit[b]):
            finished[b] = 1


@pytest.fixture
def stand_ins(monkeypatch):
    from tests import cpu_ops_shim
    saved = cpu_ops_shim.install()
    for name, fn in (("attn_decode", _attn_decode), ("kv_append", _kv_append), ("greedy_select", _greedy_select),
                     ("kv_scatter", _kv_scatter),
                     ("slot_admit", _slot_admit), ("greedy_select_slots", _greedy_select_slots)):
        monkeypatch.setattr(ops, name, fn)
    yield
    cpu_ops_shim.uninstall(saved)


def _prompts(n, seed):
    g = torch.Generator().manual_seed(seed)
    out = []
    for i in range(n):
        T = [3, 9, 5, 14, 2, 7, 11, 6, 4][i % 9]
        ids = torch.randint(3, 64, (T,), generator=g)
        ids[-1] = 1                                          # <bos> closes the prompt, as in the reference layout
        out.append({"input_ids": ids})
    return out


# The stand-ins round to bf16 like the kernels while HF runs in fp32, so a near-tie can legitimately flip a token.  The
# tiny model of test_generation_cpu.py (seed 4) with prompt seed 6 has none: HF's top-2 margin is >= 0.39 at every pick.
def test_generate_many_matches_hf_generate_per_prompt(stand_ins):
    hf, ours = _models(seed=4)
    prompts = _prompts(8, seed=6)
    budgets = [6, 3, 9, 4, 7, 2, 8, 5]
    with torch.no_grad():
        probe = hf.generate(input_ids=prompts[2]["input_ids"][None], max_new_tokens=6, eos_token_id=63, **_REF_KW)
    eos = int(probe[0, prompts[2]["input_ids"].numel() + 1])      # prompt 2 ends on its second token
    refs = []
    with torch.no_grad():
        for p, n in zip(prompts, budgets):
            out = hf.generate(input_ids=p["input_ids"][None], max_new_tokens=n, eos_token_id=eos, **_REF_KW)
            refs.append(out[0, p["input_ids"].numel():])
    assert any(int(r[-1]) == eos and r.numel() < n for r, n in zip(refs, budgets))     # some rows stop early on eos
    steps = {}
    got = ours.generate_many(prompts, batch_size=3, max_new_tokens=budgets, eos_token_id=eos, pad_token_id=0,
                             repetition_penalty=1.5, no_repeat_ngram_size=2, stats=steps)
    assert len(got) == len(prompts)
    for i, (g, r) in enumerate(zip(got, refs)):
        assert g.dtype == torch.int64 and g.dim() == 1
        assert torch.equal(g, r), (i, g, r)
    assert steps["admissions"] > 1 and steps["decode_steps"] < sum(budgets)
    # an iterator of prompts with an explicit max_prompt_length and one int budget gives the same ids
    got2 = ours.generate_many(iter(prompts), batch_size=2, max_new_tokens=4, eos_token_id=eos, pad_token_id=0,
                              repetition_penalty=1.5, no_repeat_ngram_size=2, max_prompt_length=14)
    for g, r in zip(got2, refs):
        n = min(g.numel(), r.numel())
        assert torch.equal(g[:n], r[:n])
        assert g.numel() == 4 or int(g[-1]) == eos


def test_generate_many_multi_document_prompt_attends_to_its_last_document(stand_ins):
    """A prompt whose attention_mask holds several documents (and left padding) decodes as `generate` does."""
    _, ours = _models(seed=4)
    ids = torch.tensor([0, 0, 7, 9, 12, 5, 30, 1])
    mask = torch.tensor([0, 0, 1, 1, 2, 2, 2, 2])
    pos = torch.tensor([1, 1, 0, 1, 0, 1, 2, 3])
    ref = ours.generate(ids[None], attention_mask=mask[None], position_ids=pos[None], max_new_tokens=5, eos_token_id=63,
                        pad_token_id=0, repetition_penalty=1.5, no_repeat_ngram_size=2)[0, 8:]
    other = {"input_ids": torch.tensor([4, 8, 15, 16, 23, 42, 1])}
    got = ours.generate_many([other, {"input_ids": ids, "attention_mask": mask, "position_ids": pos}, other],
                             batch_size=2, max_new_tokens=5, eos_token_id=63, pad_token_id=0, repetition_penalty=1.5,
                             no_repeat_ngram_size=2)
    assert torch.equal(got[1], ref), (got[1], ref)
    assert torch.equal(got[0], got[2])


def test_generate_many_budget_of_one_and_empty_input(stand_ins):
    _, ours = _models(seed=4)
    prompts = _prompts(4, seed=3)
    got = ours.generate_many(prompts, batch_size=2, max_new_tokens=1, eos_token_id=63, pad_token_id=0)
    assert [g.numel() for g in got] == [1, 1, 1, 1]
    assert ours.generate_many([], batch_size=2, max_new_tokens=3, eos_token_id=63, pad_token_id=0) == []


@pytest.mark.parametrize("prompts, kw, needle", [
    ([{"input_ids": torch.ones(6, dtype=torch.int64)}], dict(max_prompt_length=5), "max_prompt_length"),
    ([{"input_ids": torch.ones(0, dtype=torch.int64)}], {}, "non-empty"),
    ([{"input_ids": torch.ones(3, 2, dtype=torch.int64)}], {}, "non-empty 1-D"),
    ([{"input_ids": torch.ones(4, dtype=torch.int64)}], dict(max_new_tokens=[2, 0]), "max_new_tokens"),
    ([{"input_ids": torch.ones(4, dtype=torch.int64)}], dict(max_new_tokens=0), "max_new_tokens"),
    ([{"input_ids": torch.ones(4, dtype=torch.int64)}] * 2, dict(max_new_tokens=[3]), "budgets"),
    ([{"input_ids": torch.ones(4, dtype=torch.int64)}], dict(batch_size=0), "batch_size"),
    (iter([{"input_ids": torch.ones(4, dtype=torch.int64)}]), {}, "max_prompt_length is required"),
    ([{"input_ids": torch.ones(4, dtype=torch.int64), "attention_mask": torch.tensor([1, 1, 1, 0])}], {}, "padding"),
    ([{"input_ids": torch.ones(4, dtype=torch.int64), "input_features": torch.zeros(4, 8)}], {}, "unsupported"),
    ([{"input_ids": torch.ones(4, dtype=torch.int64), "labels": torch.ones(4)}], {}, "unsupported keys"),
    ([{"input_ids": torch.ones(4, dtype=torch.int64)}], dict(eos_token_id=[2, 3]), "single id"),
    ([{"input_ids": torch.ones(4, dtype=torch.int64)}], dict(repetition_penalty=0.0), "repetition_penalty"),
])
def test_generate_many_arguments_are_validated(stand_ins, prompts, kw, needle):
    _, ours = _models()
    args = dict(batch_size=2, max_new_tokens=3, eos_token_id=2, pad_token_id=0)
    args.update(kw)
    with pytest.raises(generation.TouchNetB200Error, match=needle):
        ours.generate_many(prompts, **args)


@pytest.mark.parametrize("kind", ["tp", "cp", "fsdp2"])
def test_generate_many_runs_on_one_unsharded_gpu_model(monkeypatch, kind):
    _, ours = _models()
    if kind == "tp":
        ours.tp_group = object()
    elif kind == "cp":
        ours.model.cp_group = object()
    else:
        monkeypatch.setattr(ops, "_is_dtensor", lambda t: True)
    with pytest.raises(generation.TouchNetB200Error, match={"tp": "tensor parallel", "cp": "context parallel",
                                                            "fsdp2": "unsharded"}[kind]):
        ours.generate_many([{"input_ids": torch.ones(4, dtype=torch.int64)}], batch_size=2, max_new_tokens=3,
                           eos_token_id=2, pad_token_id=0)
