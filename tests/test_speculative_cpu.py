"""CPU: speculative decoding (`generate(assistant_model=...)`, touchnet_b200/generation.py) - the round loop against HF
greedy `generate` and against our own `generate` without a draft, kwargs validation, and the argument checks of the two
new entry points.

The loop runs on CPU through plain-torch stand-ins (tests/cpu_ops_shim.py, the decoding stand-ins of
tests/test_generation_cpu.py, and below: per-row greedy selection, multi-query decode attention and verify selection,
written from HF's logits processors + argmax).  The kernels themselves are checked on the GPU
(tests/test_gpu_speculative.py)."""
import ctypes

import pytest
import torch

from tests.test_generation_cpu import _DIMS, _REF_KW, _Cfg, _attn_decode, _kv_append, _models, _prompt
from touchnet_b200 import _lib, modeling, ops

BF16 = torch.bfloat16


# ---------------------------------------------------------------------------------------------------------------
# entry points: argument validation happens before any CUDA call
# ---------------------------------------------------------------------------------------------------------------
def test_speculative_entry_points_reject_bad_arguments():
    p = ctypes.c_void_p(256)
    bad_calls = [
        ("tn_attn_decode_multi_bf16", (None, 1024, p, p, 128, 128 * 64, p, p, 2, 2, 8, 1, 64, 0.1, p, p, 1024, None, None),
         "null"),
        ("tn_attn_decode_multi_bf16", (p, 1024, p, p, 128, 128 * 64, p, p, 2, 3, 8, 1, 64, 0.1, p, p, 1024, None, None),
         "Tq\\*H/KV"),                                                          # 3 * 8 > 16
        ("tn_attn_decode_multi_bf16", (p, 1024, p, p, 128, 128 * 64, p, p, 2, 0, 8, 1, 64, 0.1, p, p, 1024, None, None),
         "bad dims"),
        ("tn_attn_decode_multi_bf16", (p, 1024, p, p, 128, 128 * 63, p, p, 2, 2, 8, 4, 64, 0.1, p, p, 1024, None, None),
         "stride"),
        ("tn_attn_decode_multi_bf16", (p, 1020, p, p, 128, 128 * 64, p, p, 2, 2, 8, 4, 64, 0.1, p, p, 1024, None, None),
         "multiples of 8"),
        ("tn_verify_select_bf16", (p, 64, 2, 3, 64, None, p, 16, p, p, p, p, p, p, 1.5, 2, 1, 0, None), "null"),
        ("tn_verify_select_bf16", (p, 64, 2, 3, 64, p, p, 16, p, p, p, p, None, p, 1.5, 2, 1, 0, None), "null"),
        ("tn_verify_select_bf16", (p, 64, 2, 0, 64, p, p, 16, p, p, p, p, p, p, 1.5, 2, 1, 0, None), "bad dims"),
        ("tn_verify_select_bf16", (p, 32, 2, 3, 64, p, p, 16, p, p, p, p, p, p, 1.5, 2, 1, 0, None), "bad dims"),
        ("tn_verify_select_bf16", (p, 64, 2, 3, 64, p, p, 16, p, p, p, p, p, p, 0.0, 2, 1, 0, None), "repetition_penalty"),
        ("tn_verify_select_bf16", (p, 64, 2, 3, 64, p, p, 16, p, p, p, p, p, p, 1.0, -1, 1, 0, None),
         "no_repeat_ngram_size"),
        ("tn_verify_select_bf16", (p, 1 << 23, 2, 3, 1 << 23, p, p, 16, p, p, p, p, p, p, 1.0, 0, 1, 0, None), "too large"),
    ]
    for name, args, needle in bad_calls:
        with pytest.raises(_lib.TouchNetB200Error, match=needle):
            _lib.call(name, *args)
    lib = _lib.load()
    assert lib.tn_attn_decode_multi_ws_floats(12, 0, 24, 8, 1007) == 0
    # Tq times the single-query workspace: the same splits for every query row
    assert lib.tn_attn_decode_multi_ws_floats(12, 5, 24, 8, 1007) == 5 * lib.tn_attn_decode_ws_floats(12, 24, 8, 1007)


# ---------------------------------------------------------------------------------------------------------------
# stand-ins of the decoding ops with per-row lengths (the draft's rows advance by different amounts)
# ---------------------------------------------------------------------------------------------------------------
def _pick(scores, seq, penalty, ngram):
    from transformers.generation.logits_process import NoRepeatNGramLogitsProcessor, RepetitionPenaltyLogitsProcessor
    scores = scores.float()[None]
    seq = seq[None]
    if penalty != 1.0:
        scores = RepetitionPenaltyLogitsProcessor(penalty)(seq, scores)
    if ngram > 0:
        scores = NoRepeatNGramLogitsProcessor(ngram)(seq, scores)
    return int(torch.argmax(scores, -1))


def _greedy_select(logits, history, length, positions, next_ids, finished, penalty, ngram, eos, pad):
    for b in range(history.shape[0]):
        n = int(length[b])
        tok = pad if finished[b] else _pick(logits[b], history[b, :n], penalty, ngram)
        history[b, n] = tok
        next_ids[b] = tok
        length[b] += 1
        positions[b] += 1
        finished[b] |= int(tok == eos)


def _attn_decode_multi(q, kc, vc, kv_start, kv_end, Tq, H, KV, scale, workspace=None, lse=False):
    B = kc.shape[0]
    o = torch.empty(B * Tq, H * 128, dtype=BF16)
    for j in range(Tq):
        rows = torch.arange(B) * Tq + j
        end = (kv_end - Tq + j + 1).clamp(max=kc.shape[1])     # the kernel clips a range at the cache length
        o[rows] = _attn_decode(q[rows], kc, vc, kv_start, end, H, KV, scale)
    return o


def _verify_select(logits, draft, history, length, positions, next_ids, finished, limit, penalty, ngram, eos, pad,
                   picks=None):
    B, k = draft.shape
    for b in range(B):
        if finished[b]:
            next_ids[b] = pad
            continue
        n = int(length[b])
        c = 0
        while True:
            tok = _pick(logits[b * (k + 1) + c], torch.cat([history[b, :n], draft[b, :c]]), penalty, ngram)
            history[b, n + c] = tok
            c += 1
            if tok == eos or n + c >= int(limit[b]) or c == k + 1 or int(draft[b, c - 1]) != tok:
                break
        length[b] += c
        positions[b] += c
        next_ids[b] = tok
        finished[b] = int(tok == eos or n + c >= int(limit[b]))


@pytest.fixture
def stand_ins(monkeypatch):
    from tests import cpu_ops_shim
    saved = cpu_ops_shim.install()
    monkeypatch.setattr(ops, "attn_decode", _attn_decode)
    monkeypatch.setattr(ops, "kv_append", _kv_append)
    monkeypatch.setattr(ops, "greedy_select", _greedy_select)
    monkeypatch.setattr(ops, "attn_decode_multi", _attn_decode_multi)
    monkeypatch.setattr(ops, "verify_select", _verify_select)
    yield
    cpu_ops_shim.uninstall(saved)


def _one_layer(seed):
    torch.manual_seed(seed)
    dims = dict(_DIMS, num_hidden_layers=1)
    m = modeling.B200LlamaForCausalLM(_Cfg(**dims, pad_token_id=0, attention_bias=False, initializer_range=0.02,
                                           model_type="llama", rope_scaling=None))
    with torch.no_grad():
        for prm in m.parameters():
            if prm.dim() == 2:
                prm.normal_(0, 0.08)
    return m


def _drafts(ours):
    return {"self": ours, "random": _models(seed=7)[1], "one_layer": _one_layer(9)}


# seed 4: a model without near-ties at any step (see test_generation_cpu.py), so HF's fp32 picks equal the bf16 ones
@pytest.mark.parametrize("k", [1, 2, 3])
@pytest.mark.parametrize("draft_name", ["self", "random", "one_layer"])
def test_speculative_loop_matches_hf_generate(stand_ins, k, draft_name):
    hf, ours = _models(seed=4)
    ids, mask = _prompt()
    T = ids.shape[1]
    with torch.no_grad():
        probe = hf.generate(input_ids=ids, attention_mask=mask, max_new_tokens=10, eos_token_id=63, **_REF_KW)
    eos = int(probe[0, T + 2])               # row 0 stops inside the first round, the others run on
    draft = _drafts(ours)[draft_name]
    with torch.no_grad():
        ref = hf.generate(input_ids=ids, attention_mask=mask, max_new_tokens=10, eos_token_id=eos, **_REF_KW)
    plain = ours.generate(ids, attention_mask=mask, max_new_tokens=10, eos_token_id=eos, **_REF_KW)
    got = ours.generate(ids, attention_mask=mask, max_new_tokens=10, eos_token_id=eos, assistant_model=draft,
                        num_assistant_tokens=k, **_REF_KW)
    assert got.shape == ref.shape and torch.equal(got, ref), (got, ref)
    assert torch.equal(got, plain)


@pytest.mark.parametrize("max_new", [1, 2, 5, 7])
def test_speculative_budget_ends_inside_a_round(stand_ins, max_new):
    hf, ours = _models(seed=4)
    ids, mask = _prompt()
    for name, draft in _drafts(ours).items():
        plain = ours.generate(ids, attention_mask=mask, max_new_tokens=max_new, eos_token_id=63, **_REF_KW)
        got = ours.generate(ids, attention_mask=mask, max_new_tokens=max_new, eos_token_id=63, assistant_model=draft,
                            num_assistant_tokens=3, **_REF_KW)
        assert torch.equal(got, plain), (name, got, plain)
        assert got.shape[1] == ids.shape[1] + max_new


def test_speculative_stops_when_every_row_has_finished(stand_ins):
    hf, ours = _models(seed=4)
    ids, mask = _prompt()
    T = ids.shape[1]
    probe = ours.generate(ids, attention_mask=mask, max_new_tokens=8, eos_token_id=63, **_REF_KW)
    for eos in (int(probe[0, T]), int(probe[0, T + 4])):     # row 0 finishes on its first token / inside a round
        plain = ours.generate(ids[:1], attention_mask=mask[:1], max_new_tokens=8, eos_token_id=eos, **_REF_KW)
        got = ours.generate(ids[:1], attention_mask=mask[:1], max_new_tokens=8, eos_token_id=eos, assistant_model=ours,
                            num_assistant_tokens=2, **_REF_KW)
        assert torch.equal(got, plain) and got.shape[1] < T + 8


@pytest.mark.parametrize("kw, needle", [
    (dict(num_assistant_tokens=0), "num_assistant_tokens"),
    (dict(num_assistant_tokens=2.5), "num_assistant_tokens"),
    (dict(num_assistant_tokens=8), "<= 16"),                          # G = 2: 2 * 9 > 16
    (dict(num_assistant_tokens_schedule="heuristic"), "constant"),
    (dict(assistant_confidence_threshold=0.4), "assistant_confidence_threshold"),
    (dict(prompt_lookup_num_tokens=3), "prompt_lookup_num_tokens"),
    (dict(assistant_early_exit=1), "assistant_early_exit"),
    (dict(assistant_tokenizer=object()), "assistant_tokenizer"),
    (dict(do_sample=True), "greedy"),
    (dict(num_beams=2), "greedy"),
    (dict(output_scores=True), "unsupported"),
])
def test_speculative_kwargs_are_validated(kw, needle):
    _, ours = _models()
    args = dict(max_new_tokens=4, eos_token_id=2, pad_token_id=0, assistant_model=ours)
    args.update(kw)
    with pytest.raises(_lib.TouchNetB200Error, match=needle):
        ours.generate(torch.ones(1, 4, dtype=torch.int64), **args)


def test_speculative_draft_is_checked():
    _, ours = _models()
    other_vocab = modeling.B200LlamaForCausalLM(_Cfg(**dict(_DIMS, vocab_size=128), pad_token_id=0, attention_bias=False,
                                                     initializer_range=0.02, model_type="llama", rope_scaling=None))
    wide_gqa = modeling.B200LlamaForCausalLM(_Cfg(**dict(_DIMS, num_attention_heads=16, num_key_value_heads=1,
                                                         hidden_size=256, head_dim=16), pad_token_id=0,
                                                  attention_bias=False, initializer_range=0.02, model_type="llama",
                                                  rope_scaling=None))
    args = dict(max_new_tokens=4, eos_token_id=2, pad_token_id=0)
    for draft, needle in ((other_vocab, "vocab_size"), (wide_gqa, "2 \\* H/KV"), (torch.nn.Linear(2, 2), "same kind")):
        with pytest.raises(_lib.TouchNetB200Error, match=needle):
            ours.generate(torch.ones(1, 4, dtype=torch.int64), assistant_model=draft, **args)
    # without a draft the assisted-generation knobs stay unsupported arguments, as before
    with pytest.raises(_lib.TouchNetB200Error, match="unsupported"):
        ours.generate(torch.ones(1, 4, dtype=torch.int64), num_assistant_tokens=2, **args)


def test_verify_attention_uses_the_cache_length_of_generate(stand_ins, monkeypatch):
    """The decode attention's split count and chunks are functions of the cache length, so the verify step attends on
    generate's T + max_new_tokens rows (not on its own cache of k more rows) to sum every row in generate's order."""
    _, ours = _models(seed=4)
    ids, mask = _prompt()
    seen = []

    def spy(q, kc, vc, kv_start, kv_end, Tq, H, KV, scale, workspace=None, lse=False):
        seen.append((Tq, kc.shape[1], vc.shape[1]))
        return _attn_decode_multi(q, kc, vc, kv_start, kv_end, Tq, H, KV, scale, workspace, lse)

    monkeypatch.setattr(ops, "attn_decode_multi", spy)
    ours.generate(ids, attention_mask=mask, max_new_tokens=9, eos_token_id=63, assistant_model=_one_layer(9),
                  num_assistant_tokens=3, **_REF_KW)
    T = ids.shape[1]
    verify = {(s, s2) for tq, s, s2 in seen if tq == 4}
    assert verify == {(T + 9, T + 9)}, seen


def test_default_draft_length_needs_room_in_the_tile():
    c = _Cfg(**dict(_DIMS, num_attention_heads=16, num_key_value_heads=1, head_dim=16), pad_token_id=0,
             attention_bias=False, initializer_range=0.02, model_type="llama", rope_scaling=None)
    wide = modeling.B200LlamaForCausalLM(c)
    with pytest.raises(_lib.TouchNetB200Error, match="no room for a draft token"):
        wide.generate(torch.ones(1, 4, dtype=torch.int64), max_new_tokens=4, eos_token_id=2, pad_token_id=0,
                      assistant_model=_models()[1])
