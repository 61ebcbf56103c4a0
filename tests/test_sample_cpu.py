"""CPU: sampling in `generate_many` (do_sample=True) - argument checks of tn_sample_select_slots_bf16, validation and
defaults of the sampling knobs, the host loop with a stand-in sampler, and the fp64 kept-set oracle of
tests/sample_oracle.py against transformers' TopKLogitsWarper / TopPLogitsWarper.

The stand-in sampler is HF's processors and warpers plus torch.multinomial with a generator seeded from
(seed, stream key, length): like the kernel, a draw depends on the prompt's stream and position only, so the loop's key
plumbing (each prompt's index reaching its slot at admission) shows as outputs that do not depend on batch_size.  The
kernel itself is checked on the GPU (tests/test_gpu_sample.py)."""
import ctypes

import pytest
import torch

from tests.sample_oracle import distribution, hf_kept, processed
from tests.test_generate_many_cpu import _prompts, stand_ins  # noqa: F401
from tests.test_generation_cpu import _models
from touchnet_b200 import _lib, generation, ops


def test_sample_entry_point_rejects_bad_arguments():
    p = ctypes.c_void_p(256)
    map_arr = (ctypes.c_int32 * 2)(0, 7)
    key_arr = (ctypes.c_int64 * 2)(0, 1)

    def sel(logits=p, n=4, m=None, keys=None, B=4, ld=64, V=64, pen=1.5, ng=2, sk=p, t=0.7, k=50, tp=0.9):
        return (logits, ld, n, m, keys, B, V, p, 16, p, p, p, p, p, sk, pen, ng, t, k, tp, 123, 1, 0, None)

    bad_calls = [
        (sel(logits=None), "null"),
        (sel(sk=None), "null"),
        (sel(n=2, m=ctypes.addressof(map_arr)), "out of range"),
        (sel(n=1, m=ctypes.addressof(map_arr)), "null"),                          # a map without its keys
        (sel(ld=32), "bad dims"),
        (sel(n=3), "bad dims"),
        (sel(n=300, m=ctypes.addressof(map_arr), keys=ctypes.addressof(key_arr), B=400), "at most"),
        (sel(t=0.0), "temperature"),
        (sel(t=-1.0), "temperature"),
        (sel(t=float("inf")), "temperature"),
        (sel(k=-1), "top_k"),
        (sel(tp=1.5), "top_p"),
        (sel(tp=-0.1), "top_p"),
        (sel(tp=float("nan")), "top_p"),
        (sel(pen=0.0), "repetition_penalty"),
        (sel(ng=-1), "no_repeat_ngram_size"),
        (sel(ld=1 << 23, V=1 << 23, pen=1.0, ng=0), "too large"),
    ]
    for args, needle in bad_calls:
        with pytest.raises(_lib.TouchNetB200Error, match=needle):
            _lib.call("tn_sample_select_slots_bf16", *args)


# ---------------------------------------------------------------------------------------------------------------
# the stand-in sampler
# ---------------------------------------------------------------------------------------------------------------
def _sample_select_slots(logits, history, length, positions, next_ids, finished, limit, stream_key, penalty, ngram,
                         temperature, top_k, top_p, seed, eos, pad, row_slot=None, row_key=None):
    from transformers.generation.logits_process import TopKLogitsWarper, TopPLogitsWarper
    for r in range(logits.shape[0]):
        b = r if row_slot is None else row_slot[r]
        if row_slot is not None:
            stream_key[b] = row_key[r]
        if finished[b]:
            next_ids[b] = pad
            continue
        n = int(length[b])
        seq = history[b:b + 1, :n]
        s = processed(seq, logits[r:r + 1].float(), penalty, ngram, temperature)[None]
        if top_k > 0:
            s = TopKLogitsWarper(top_k)(seq, s)
        if top_p < 1.0:
            s = TopPLogitsWarper(top_p)(seq, s)
        g = torch.Generator().manual_seed((seed * 1000003 + int(stream_key[b]) * 8191 + n) % (2**63))
        tok = int(torch.multinomial(torch.softmax(s, -1), 1, generator=g))
        history[b, n] = tok
        next_ids[b] = tok
        length[b] = n + 1
        positions[b] += 1
        if tok == eos or n + 1 == int(limit[b]):
            finished[b] = 1


@pytest.fixture
def sampler(stand_ins, monkeypatch):  # noqa: F811
    calls = []

    def rec(*a, **k):
        calls.append((k.get("row_slot"), k.get("row_key"), a[10:13]))
        _sample_select_slots(*a, **k)

    monkeypatch.setattr(ops, "sample_select_slots", rec)
    return calls


def test_sampling_host_loop_keys_eos_budgets_and_order(sampler):
    _, ours = _models(seed=4)
    prompts = _prompts(8, seed=6)
    budgets = [6, 3, 9, 4, 7, 2, 8, 5]
    kw = dict(max_new_tokens=budgets, eos_token_id=5, pad_token_id=0, repetition_penalty=1.5, no_repeat_ngram_size=2,
              do_sample=True, temperature=0.8, top_k=20, top_p=0.95)
    runs = []
    for B in (1, 3, 8):
        torch.manual_seed(0)
        runs.append(ours.generate_many(prompts, batch_size=B, **kw))
    first_admission = sampler[:1]
    assert first_admission[0][0] == [0] and first_admission[0][1] == [0]       # prompt 0 into slot 0 carries key 0
    keys = sorted(k for slots, ks, _ in sampler if ks is not None for k in ks)
    assert keys == sorted(list(range(8)) * 3)                                 # every prompt admitted once per run
    assert all(knobs == (0.8, 20, 0.95) for _, _, knobs in sampler)
    for out in runs[1:]:
        for a, b in zip(out, runs[0]):
            assert torch.equal(a, b)
    out = runs[0]
    for o, n in zip(out, budgets):
        assert o.dtype == torch.int64 and o.dim() == 1
        assert o.numel() == n or (int(o[-1]) == 5 and o.numel() < n)
        assert 5 not in o[:-1].tolist()
    torch.manual_seed(1)
    other = ours.generate_many(prompts, batch_size=3, **kw)
    assert any(not torch.equal(a, b) for a, b in zip(other, out))             # the seed comes from torch's generator


def test_none_takes_hf_defaults(sampler):
    _, ours = _models(seed=4)
    ours.generate_many(_prompts(2, seed=1), batch_size=2, max_new_tokens=2, eos_token_id=63, pad_token_id=0,
                       do_sample=True)
    assert sampler and all(knobs == (1.0, 50, 1.0) for _, _, knobs in sampler)


def test_do_sample_false_ignores_the_knobs(stand_ins):  # noqa: F811
    _, ours = _models(seed=4)
    prompts = _prompts(5, seed=2)
    kw = dict(batch_size=2, max_new_tokens=5, eos_token_id=63, pad_token_id=0, repetition_penalty=1.5,
              no_repeat_ngram_size=2)
    base = ours.generate_many(prompts, **kw)
    for knobs in (dict(temperature=0.5, top_k=3, top_p=0.2), dict(temperature=-1.0, top_k=-3, top_p=7.0)):
        got = ours.generate_many(prompts, **kw, **knobs)
        assert all(torch.equal(a, b) for a, b in zip(got, base))


@pytest.mark.parametrize("kw, needle", [
    (dict(temperature=0.0), "temperature"),
    (dict(temperature=-0.5), "temperature"),
    (dict(temperature=float("nan")), "temperature"),
    (dict(top_k=-1), "top_k"),
    (dict(top_k=2.5), "top_k"),
    (dict(top_k=True), "top_k"),
    (dict(top_p=1.01), "top_p"),
    (dict(top_p=-0.01), "top_p"),
])
def test_sampling_knobs_are_validated_before_any_work(monkeypatch, kw, needle):
    _, ours = _models()

    def no_work(*a, **k):
        raise AssertionError("validation must come first")

    monkeypatch.setattr(generation, "_check_scope", no_work)
    with pytest.raises(generation.TouchNetB200Error, match=needle):
        ours.generate_many([{"input_ids": torch.ones(4, dtype=torch.int64)}], batch_size=2, max_new_tokens=3,
                           eos_token_id=2, pad_token_id=0, do_sample=True, **kw)


# ---------------------------------------------------------------------------------------------------------------
# the fp64 oracle of the kept set against HF's warpers on tie-free rows
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("top_k, top_p", [(50, 1.0), (0, 0.9), (50, 0.9), (1, 1.0), (0, 0.0), (7, 0.3), (0, 0.5)])
def test_kept_set_oracle_matches_hf_warpers_without_ties(top_k, top_p):
    g = torch.Generator().manual_seed(top_k * 100 + int(top_p * 10))
    for trial in range(20):
        V = [64, 1000, 5000][trial % 3]
        x = torch.randn(V, generator=g, dtype=torch.float64).float() * 3
        while torch.unique(x).numel() < V:                                  # tie-free rows only
            x = torch.randn(V, generator=g, dtype=torch.float64).float() * 3
        probs, band = distribution(x, top_k, top_p)
        mine, hf = probs > 0, hf_kept(x, top_k, top_p)
        assert torch.equal(mine | band, hf | band), trial
        assert abs(float(probs.sum()) - 1.0) < 1e-12


def test_oracle_keeps_whole_tied_groups():
    x = torch.tensor([3.0, 1.0, 3.0, 2.0, 2.0, 0.0])
    assert (distribution(x, 1, 1.0)[0] > 0).tolist() == [True, False, True, False, False, False]
    assert (distribution(x, 3, 1.0)[0] > 0).tolist() == [True, False, True, True, True, False]
    assert (distribution(x, 0, 0.0)[0] > 0).tolist() == [True, False, True, False, False, False]
    w = torch.exp(x.double() - 3)
    p = float(w[[0, 2]].sum() / w.sum()) + 1e-6                               # just past the two maxima: 2.0 joins
    assert (distribution(x, 0, p)[0] > 0).tolist() == [True, False, True, True, True, False]
