"""CPU: speculative decoding in `generate_many` (assistant_model) - argument checks of tn_spec_sample_verify_bf16, the
draft arguments of generate_many, the host loop through plain-torch stand-ins (greedy: equal to generate_many without
the draft; sampled: the logits, context and state each step hands the verifier), and the fp64 oracle of
tests/spec_sample_oracle.py against the formulas.  The kernels are checked on the GPU (tests/test_gpu_spec_many.py)."""
import ctypes

import pytest
import torch

from tests.sample_oracle import distribution, processed
from tests.spec_sample_oracle import acceptance, emitted, residual
from tests.test_generate_many_cpu import _prompts, stand_ins  # noqa: F401
from tests.test_generation_cpu import _attn_decode, _models
from tests.test_sample_cpu import _sample_select_slots
from tests.test_speculative_cpu import _one_layer, _verify_select
from touchnet_b200 import _lib, generation, ops


def test_spec_sample_verify_rejects_bad_arguments():
    p = ctypes.c_void_p(256)

    def sel(logits=p, dl=p, ld=64, ldd=64, B=4, k=3, V=64, sk=p, pk=p, pen=1.5, ng=2, t=0.7, tk=50, tp=0.9):
        return (logits, ld, dl, ldd, B, k, V, p, p, 16, p, p, p, p, p, sk, pk, pen, ng, t, tk, tp, 123, 1, 0, None)

    for args, needle in [
        (sel(logits=None), "null"), (sel(dl=None), "null"), (sel(sk=None), "null"), (sel(pk=None), "null"),
        (sel(k=0), "bad dims"), (sel(B=0), "bad dims"), (sel(ld=32), "bad dims"), (sel(ldd=32), "bad dims"),
        (sel(B=70000), "too large"), (sel(t=0.0), "temperature"), (sel(t=float("inf")), "temperature"),
        (sel(tk=-1), "top_k"), (sel(tp=1.5), "top_p"), (sel(tp=float("nan")), "top_p"),
        (sel(pen=0.0), "repetition_penalty"), (sel(ng=-1), "no_repeat_ngram_size"),
        (sel(ld=1 << 23, ldd=1 << 23, V=1 << 23, pen=1.0, ng=0), "too large"),
    ]:
        with pytest.raises(_lib.TouchNetB200Error, match=needle):
            _lib.call("tn_spec_sample_verify_bf16", *args)


# ---------------------------------------------------------------------------------------------------------------
# stand-ins with the kernels' range rules (an idle slot has kv_end = 0: its rows below 0 are dropped, its ranges empty)
# ---------------------------------------------------------------------------------------------------------------
def _kv_append(k, v, kc, vc, row_end, T_new):
    for b in range(kc.shape[0]):
        for t in range(T_new):
            row = int(row_end[b]) - T_new + t
            if 0 <= row < kc.shape[1]:
                kc[b, row] = k[b * T_new + t]
                vc[b, row] = v[b * T_new + t]


def _attn_decode_multi(q, kc, vc, kv_start, kv_end, Tq, H, KV, scale, workspace=None, lse=False):
    B = kc.shape[0]
    o = torch.zeros(B * Tq, H * 128, dtype=torch.bfloat16)
    for j in range(Tq):
        rows = torch.arange(B) * Tq + j
        end = (kv_end - Tq + j + 1).clamp(min=0, max=kc.shape[1])
        o[rows] = _attn_decode(q[rows], kc, vc, kv_start, torch.maximum(end, kv_start), H, KV, scale)
    return o


def _hf_speculative_sampling(p, q, x, g):
    """transformers' `_speculative_sampling` for one row: p [k+1, V], q [k, V] probabilities, x [k] candidates."""
    k = x.numel()
    pi, qi = p[torch.arange(k), x], q[torch.arange(k), x]
    ratio = torch.where(qi > 0, pi / qi.clamp(min=1e-300), torch.full_like(pi, float("inf")))
    r = torch.rand(k, generator=g, dtype=torch.float64)
    ok = r <= ratio
    n = k if bool(ok.all()) else int((~ok).int().argmax())
    if n < k:
        d = (p[n] - q[n]).clamp(min=0)
        d = d / d.sum()
    else:
        d = p[k]
    return n, int(torch.multinomial(d, 1, generator=g))


def _spec_sample_verify(logits, dlogits, draft, history, length, positions, next_ids, finished, limit, stream_key,
                        penalty, ngram, temperature, top_k, top_p, seed, eos, pad, picks=None):
    B, k = draft.shape
    for b in range(B):
        if finished[b]:
            next_ids[b] = pad
            continue
        n0 = int(length[b])
        ctx = [torch.cat([history[b, :n0], draft[b, :j]])[None] for j in range(k + 1)]
        dist = lambda row, j: distribution(processed(ctx[j], row[None].float(), penalty, ngram, temperature),  # noqa
                                           top_k, top_p)[0]
        p = torch.stack([dist(logits[b * (k + 1) + j], j) for j in range(k + 1)])
        q = torch.stack([dist(dlogits[b * k + j], j) for j in range(k)])
        g = torch.Generator().manual_seed((seed * 1000003 + int(stream_key[b]) * 8191 + n0 + 7) % (2**63))
        n, last = _hf_speculative_sampling(p, q, draft[b], g)
        toks = draft[b, :n].tolist() + [last]
        c = 0
        for tok in toks:
            history[b, n0 + c] = tok
            c += 1
            if tok == eos or n0 + c >= int(limit[b]):
                break
        length[b] = n0 + c
        positions[b] += c
        next_ids[b] = tok
        finished[b] = int(tok == eos or n0 + c >= int(limit[b]))


def _gemm(a, b, *, a_mn=False, b_mn=False, out_f32=False, residual=None, out=None, M=None, N=None, K=None):
    """The stand-in GEMM in fp64: a CPU fp32 matmul sums in an order that depends on M (the kernels' does not), which
    could make a verify row differ from its decode row in the last bit."""
    A = a.double().t() if a_mn else a.double()
    y = A @ (b.double() if b_mn else b.double().t())
    if residual is not None:
        y = y + residual.double().reshape(y.shape)
    y = y.float() if out_f32 else y.to(torch.bfloat16)
    return out.copy_(y) if out is not None else y


@pytest.fixture
def spec_stand_ins(stand_ins, monkeypatch):  # noqa: F811
    for name, fn in (("gemm", _gemm), ("kv_append", _kv_append), ("attn_decode_multi", _attn_decode_multi),
                     ("verify_select", _verify_select), ("sample_select_slots", _sample_select_slots),
                     ("spec_sample_verify", _spec_sample_verify)):
        monkeypatch.setattr(ops, name, fn)


@pytest.mark.parametrize("k", [1, 3])
def test_greedy_draft_arm_equals_generate_many(spec_stand_ins, k):
    _, ours = _models(seed=4)
    prompts = _prompts(5, seed=6)
    budgets = [6, 3, 9, 1, 7]
    probe = ours.generate_many(prompts[:1], batch_size=1, max_new_tokens=6, eos_token_id=63, pad_token_id=0)
    eos = int(probe[0][2])                                         # prompt 0 stops on its third token
    kw = dict(max_new_tokens=budgets, eos_token_id=eos, pad_token_id=0, repetition_penalty=1.5, no_repeat_ngram_size=2)
    for B in (2, 7):                                               # more prompts than slots; idle slots throughout
        base = ours.generate_many(prompts, batch_size=B, **kw)
        for draft in (ours, _one_layer(9)):
            stats = {}
            got = ours.generate_many(prompts, batch_size=B, assistant_model=draft, num_assistant_tokens=k, stats=stats,
                                     **kw)
            assert all(torch.equal(a, b) for a, b in zip(got, base)), (B, k)
            assert stats["rounds"] == stats["decode_steps"] and stats["live_row_rounds"] >= stats["rounds"]
        if draft is not ours and B == 2:
            assert stats["rounds"] < sum(budgets)


def test_sampled_draft_arm_hands_the_verifier_the_draft_logits_and_context(spec_stand_ins, monkeypatch):
    _, ours = _models(seed=4)
    draft = _one_layer(9)
    prompts = _prompts(5, seed=2)
    seen = {"draft_rows": [], "verify": 0}
    real_sample = _sample_select_slots

    def sample_spy(logits, *a, **kw):
        if kw.get("row_slot") is None and logits.shape[0] == 2:   # the draft's proposals (B = 2, unmapped)
            seen["draft_rows"].append(logits.clone())
        real_sample(logits, *a, **kw)

    def verify_spy(logits, dlogits, draft_ids, history, length, *a, **kw):
        B, k = draft_ids.shape
        assert logits.shape[0] == B * (k + 1) and dlogits.shape[0] == B * k
        # the saved draft logits are the rows the draft sampled its k proposals from, in order
        rows = seen["draft_rows"][-k:]
        for j in range(k):
            assert torch.equal(dlogits.view(B, k, -1)[:, j], rows[j])
        seen["verify"] += 1
        _spec_sample_verify(logits, dlogits, draft_ids, history, length, *a, **kw)

    monkeypatch.setattr(ops, "sample_select_slots", sample_spy)
    monkeypatch.setattr(ops, "spec_sample_verify", verify_spy)
    kw = dict(batch_size=2, max_new_tokens=[5, 3, 7, 4, 6], eos_token_id=63, pad_token_id=0, repetition_penalty=1.5,
              no_repeat_ngram_size=2, do_sample=True, temperature=0.8, top_k=20, top_p=0.95, assistant_model=draft,
              num_assistant_tokens=2)
    torch.manual_seed(0)
    a = ours.generate_many(prompts, **kw)
    assert seen["verify"] > 0
    torch.manual_seed(0)
    b = ours.generate_many(prompts, **kw)
    assert all(torch.equal(x, y) for x, y in zip(a, b))             # both seeds come from torch's generator
    for o, n in zip(a, [5, 3, 7, 4, 6]):                           # each budget, or cut right after an eos
        assert o.dtype == torch.int64 and o.dim() == 1 and 1 <= o.numel() <= n
        assert 63 not in o[:-1].tolist() and (o.numel() == n or int(o[-1]) == 63)
    # the first token is the admission's draw, as without the draft
    monkeypatch.setattr(ops, "sample_select_slots", real_sample)
    torch.manual_seed(0)
    plain = ours.generate_many(prompts, **{n: v for n, v in kw.items() if n not in ("assistant_model",
                                                                                   "num_assistant_tokens")})
    assert all(int(x[0]) == int(y[0]) for x, y in zip(a, plain))


@pytest.mark.parametrize("kw, needle", [
    (dict(num_assistant_tokens=0), "num_assistant_tokens"),
    (dict(num_assistant_tokens=8), "<= 16"),
    (dict(num_assistant_tokens_schedule="heuristic"), "constant"),
    (dict(assistant_confidence_threshold=0.4), "assistant_confidence_threshold"),
    (dict(prompt_lookup_num_tokens=3), "prompt_lookup_num_tokens"),
    (dict(output_scores=True), "unsupported"),
])
def test_draft_arguments_are_validated_before_any_work(monkeypatch, kw, needle):
    _, ours = _models()

    def no_work(*a, **k):
        raise AssertionError("validation must come first")

    monkeypatch.setattr(generation, "_Weights", no_work)
    monkeypatch.setattr(generation, "B200KVCache", no_work)
    with pytest.raises(generation.TouchNetB200Error, match=needle):
        ours.generate_many([{"input_ids": torch.ones(4, dtype=torch.int64)}], batch_size=2, max_new_tokens=3,
                           eos_token_id=2, pad_token_id=0, assistant_model=ours, **kw)


def test_draft_knobs_without_a_draft_and_foreign_drafts():
    _, ours = _models()
    args = dict(batch_size=2, max_new_tokens=3, eos_token_id=2, pad_token_id=0)
    p = [{"input_ids": torch.ones(4, dtype=torch.int64)}]
    with pytest.raises(generation.TouchNetB200Error, match="unsupported"):
        ours.generate_many(p, num_assistant_tokens=2, **args)
    with pytest.raises(TypeError, match="unexpected keyword"):
        ours.generate_many(p, output_scores=True, **args)
    with pytest.raises(generation.TouchNetB200Error, match="same kind"):
        ours.generate_many(p, assistant_model=torch.nn.Linear(2, 2), **args)


# ---------------------------------------------------------------------------------------------------------------
# the fp64 oracle against the formulas
# ---------------------------------------------------------------------------------------------------------------
def test_oracle_acceptance_residual_and_emitted_distribution():
    p = torch.tensor([0.5, 0.3, 0.2, 0.0], dtype=torch.float64)
    q = torch.tensor([0.2, 0.3, 0.1, 0.4], dtype=torch.float64)
    assert acceptance(p, q) == pytest.approx(0.2 + 0.3 + 0.1)
    assert torch.allclose(residual(p, q), torch.tensor([0.75, 0.0, 0.25, 0.0], dtype=torch.float64))
    assert torch.allclose(emitted(p, q), p)                       # speculative sampling emits p exactly
    assert acceptance(p, p) == pytest.approx(1.0) and torch.allclose(emitted(p, p), p)
    disjoint = torch.tensor([0.0, 0.0, 0.0, 1.0], dtype=torch.float64)
    assert acceptance(p, disjoint) == 0.0 and torch.allclose(residual(p, disjoint), p)
    g = torch.Generator().manual_seed(0)
    for _ in range(20):
        a = torch.softmax(torch.randn(50, generator=g, dtype=torch.float64) * 2, 0)
        b = torch.softmax(torch.randn(50, generator=g, dtype=torch.float64) * 2, 0)
        assert torch.allclose(emitted(a, b), a, atol=1e-12)
        assert float(residual(a, b)[a <= b].abs().max()) == 0.0
