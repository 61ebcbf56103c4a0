"""GPU: speculative decoding in `generate_many` (assistant_model) - the speculative-sampling kernel
tn_spec_sample_verify_bf16 against the fp64 oracle of tests/spec_sample_oracle.py, its exact cases and determinism,
and the end-to-end contracts: greedy results bit-identical to generate_many without the draft, sampled results
reproducible, invariant to batching and distributed as sampling without the draft."""
import pytest
import torch

from tests.gpu_util import require_cuda
from tests.sample_oracle import distribution
from tests.spec_sample_oracle import residual
from tests.test_gpu_generate_many import _asr_model, _asr_prompt, _fbank_prompts, _touch_audio_small
from tests.test_gpu_sample import _SAMPLE_KW, _chi2_pvalue
from touchnet_b200 import modeling, ops

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16


def _state(B, S, dev, L=1, limit=None):
    return dict(history=torch.zeros((B, S), dtype=torch.int64, device=dev),
                length=torch.full((B,), L, dtype=torch.int32, device=dev),
                positions=torch.arange(B, dtype=torch.int64, device=dev),
                next_ids=torch.full((B,), -5, dtype=torch.int64, device=dev),
                finished=torch.zeros(B, dtype=torch.int32, device=dev),
                limit=torch.full((B,), S if limit is None else limit, dtype=torch.int32, device=dev))


def _verify(logits, dlogits, drafts, st, keys, t, k, p, seed, eos=-1, pad=0, penalty=1.0, ngram=0):
    return ops.spec_sample_verify(logits, dlogits, drafts, st["history"], st["length"], st["positions"],
                                  st["next_ids"], st["finished"], st["limit"], keys, penalty, ngram, t, k, p, seed,
                                  eos, pad)


def _emitted(picks):
    """(accepted count n, the token emitted at n) per row of picks [B, k+1]."""
    acc = picks >= 0
    n = torch.where(acc.all(1), acc.shape[1], (~acc).int().argmax(1))
    n = n.clamp(max=acc.shape[1] - 1)
    return n, ~picks.gather(1, n[:, None])[:, 0]


def _probs(x, t, k, p):
    return distribution(x.float() / t if t != 1.0 else x.float(), k, p)[0]


# ---------------------------------------------------------------------------------------------------------------
# the kernel's distribution: thousands of rows of the same (p, q), each with its own stream key
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V, t, tk, tp", [(64, 1.0, 0, 1.0), (64, 0.7, 20, 0.9), (128256, 0.7, 50, 0.9),
                                          (128256, 1.0, 40, 1.0)])
def test_acceptance_residual_and_bonus_follow_the_oracle(V, t, tk, tp):
    dev = require_cuda()
    g = torch.Generator().manual_seed(V + tk)
    N = 6000 if V == 64 else 3000
    scale = 2.0 if V == 64 else 4.0
    p0 = (torch.randn(V, generator=g) * scale).to(BF16)
    p1 = (torch.randn(V, generator=g) * scale).to(BF16)
    q0 = (p0.float() + torch.randn(V, generator=g) * scale * 0.7).to(BF16)
    P0, P1, Q0 = _probs(p0, t, tk, tp), _probs(p1, t, tk, tp), _probs(q0, t, tk, tp)
    x = torch.multinomial(Q0.float(), N, replacement=True, generator=g)              # proposals drawn from q
    logits = torch.stack([p0, p1]).repeat(N, 1).to(dev)                               # [N*2, V], k = 1
    dlogits = q0[None].repeat(N, 1).to(dev)
    st = _state(N, 8, dev)
    keys = torch.arange(N, dtype=torch.int64, device=dev) * 7919
    picks = _verify(logits, dlogits, x[:, None].to(dev), st, keys, t, tk, tp, seed=1234).cpu()
    n, last = _emitted(picks)
    accepted = n == 1
    # acceptance rate at position 0: sum_v min(p, q), within 5 binomial standard deviations
    a = float(torch.minimum(P0, Q0).sum())
    rate = float(accepted.double().mean())
    assert abs(rate - a) <= 5 * (a * (1 - a) / N) ** 0.5 + 1e-3, (rate, a)
    # the first emitted token follows p_0
    first = torch.where(accepted, x, last)
    assert _chi2_pvalue(torch.bincount(first, minlength=V).double(), P0 * N) > 1e-4
    # after a rejection at 0: the normalised residual; after the acceptance: p_1
    R = residual(P0, Q0)
    rej = ~accepted
    assert int(rej.sum()) > 100 and int(accepted.sum()) > 100
    assert _chi2_pvalue(torch.bincount(last[rej], minlength=V).double(), R * float(rej.sum())) > 1e-4
    assert float(R[last[rej]].min()) > 0                                              # never a token with p <= q
    assert _chi2_pvalue(torch.bincount(last[accepted], minlength=V).double(), P1 * float(accepted.sum())) > 1e-4
    # the state: one or two tokens appended as the commit of verify_select writes them
    assert torch.equal(st["length"].cpu(), 1 + n.int() + 1)
    assert torch.equal(st["next_ids"].cpu(), last)
    assert torch.equal(st["history"][:, 1].cpu(), first)


@pytest.mark.parametrize("V", [64, 128256])
def test_draft_logits_equal_to_the_target_accept_every_proposal(V):
    dev = require_cuda()
    g = torch.Generator().manual_seed(3)
    B, k = 64, 3
    rows = (torch.randn(B * (k + 1), V, generator=g) * 3).to(BF16).to(dev)
    logits = rows
    dlogits = rows.view(B, k + 1, V)[:, :k].reshape(B * k, V).contiguous()
    st = _state(B, 16, dev)
    keys = torch.arange(B, dtype=torch.int64, device=dev)
    # proposals drawn by the draft's own kernel: sample_select_slots on the draft rows in its context
    dst = {n: v.clone() for n, v in st.items()}
    drafts = torch.zeros((B, k), dtype=torch.int64, device=dev)
    for j in range(k):
        ops.sample_select_slots(dlogits.view(B, k, V)[:, j].contiguous(), dst["history"], dst["length"],
                                dst["positions"], dst["next_ids"], dst["finished"], dst["limit"], keys, 1.3, 2, 0.8,
                                50, 0.95, 99, -1, 0)
        drafts[:, j] = dst["next_ids"]
    picks = _verify(logits, dlogits, drafts, st, keys, 0.8, 50, 0.95, seed=5, penalty=1.3, ngram=2)
    assert bool((picks[:, :k] >= 0).all())
    assert torch.equal(picks[:, :k], drafts)
    assert bool((st["length"] == 1 + k + 1).all())


def test_exact_cases_disjoint_degenerate_eos_limit_and_held_slots():
    dev = require_cuda()
    V, B, k = 64, 8, 2
    g = torch.Generator().manual_seed(5)
    logits = (torch.randn(B * (k + 1), V, generator=g) * 2).to(BF16).to(dev)
    dlogits = (torch.randn(B * k, V, generator=g) * 2).to(BF16).to(dev)
    keys = torch.arange(B, dtype=torch.int64, device=dev)
    # top_k = 1 with different maxima: p(x) = 0 for the draft's pick, rejected at 0, the target's maximum emitted
    dl = logits.view(B, k + 1, V)[:, :k].reshape(B * k, V).clone()
    tmax = logits.float().argmax(1).view(B, k + 1)
    dl.view(B, k, V)[:, 0].scatter_(1, ((tmax[:, 0] + 1) % V)[:, None], 100.0)
    drafts = dl.float().argmax(1).view(B, k)
    st = _state(B, 16, dev)
    picks = _verify(logits, dl, drafts, st, keys, 1.0, 1, 1.0, seed=1)
    assert torch.equal(picks[:, 0], ~tmax[:, 0])
    assert torch.equal(st["next_ids"], tmax[:, 0]) and bool((st["length"] == 2).all())
    # a degenerate target row (NaN) at position 0 emits its greedy pick (the NaN) and stops there
    lg = logits.clone()
    lg[0 * (k + 1), 7] = float("nan")
    st = _state(B, 16, dev)
    drafts = torch.full((B, k), 7, dtype=torch.int64, device=dev)
    picks = _verify(lg, dlogits, drafts, st, keys, 0.7, 0, 0.9, seed=1)
    assert int(picks[0, 0]) == ~7 and int(st["length"][0]) == 2 and int(st["next_ids"][0]) == 7
    # a degenerate draft row: q is a point mass on its pick x; p(x) = 0 under top_k = 1 rejects it
    dg = dlogits.clone()
    dg[0, 5] = float("nan")
    xs = torch.full((B, k), 5, dtype=torch.int64, device=dev)
    st = _state(B, 16, dev)
    picks = _verify(logits, dg, xs, st, keys, 1.0, 1, 1.0, seed=1)
    if int(tmax[0, 0]) != 5:
        assert int(picks[0, 0]) == ~int(tmax[0, 0])
    # eos and limit cut the row; finished and idle slots hold still
    same = logits.view(B, k + 1, V)[:, :k].reshape(B * k, V).contiguous()
    top1 = same.float().argmax(1).view(B, k)
    st = _state(B, 16, dev)
    st["finished"][2] = 1
    st["length"][3] = 0                                          # an idle slot: finished, no tokens
    st["finished"][3] = 1
    st["limit"][4] = 2                                           # room for one token
    before = {n: v.clone() for n, v in st.items()}
    eos = int(top1[1, 0])
    _verify(logits, same, top1, st, keys, 1.0, 1, 1.0, seed=1, eos=eos, pad=0)
    assert int(st["length"][1]) == 2 and int(st["finished"][1]) == 1 and int(st["next_ids"][1]) == eos
    assert int(st["length"][4]) == 2 and int(st["finished"][4]) == 1
    for s in (2, 3):
        assert int(st["next_ids"][s]) == 0
        for n in ("history", "length", "positions", "finished"):
            assert torch.equal(st[n][s], before[n][s]), (s, n)
    # a row that is not cut accepts both top-1 proposals and emits the top-1 bonus token
    if eos not in tmax[0].tolist():
        assert int(st["length"][0]) == 1 + k + 1 and int(st["next_ids"][0]) == int(tmax[0, k])


def test_launches_are_deterministic_and_graph_capture_is_bitwise_equal():
    dev = require_cuda()
    V, B, k = 128256, 12, 3
    g = torch.Generator().manual_seed(9)
    logits = (torch.randn(B * (k + 1), V, generator=g) * 3).to(BF16).to(dev)
    dlogits = (logits[:B * k].float() + torch.randn(B * k, V, generator=g).to(dev)).to(BF16)
    drafts = torch.randint(0, V, (B, k), generator=g).to(dev)
    keys = torch.arange(B, dtype=torch.int64, device=dev)
    outs = []
    for _ in range(2):
        st = _state(B, 32, dev)
        outs.append((_verify(logits, dlogits, drafts, st, keys, 0.7, 50, 0.9, seed=42).clone(), st))
    st = _state(B, 32, dev)
    picks = torch.empty((B, k + 1), dtype=torch.int64, device=dev)
    graph = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.spec_sample_verify(logits, dlogits, drafts, st["history"], st["length"], st["positions"], st["next_ids"],
                               st["finished"], st["limit"], keys, 1.0, 0, 0.7, 50, 0.9, 42, -1, 0, picks=picks)
    torch.cuda.current_stream().wait_stream(s)
    st = _state(B, 32, dev)
    with torch.cuda.graph(graph):
        ops.spec_sample_verify(logits, dlogits, drafts, st["history"], st["length"], st["positions"], st["next_ids"],
                               st["finished"], st["limit"], keys, 1.0, 0, 0.7, 50, 0.9, 42, -1, 0, picks=picks)
    for name, v in _state(B, 32, dev).items():
        st[name].copy_(v)
    graph.replay()
    torch.cuda.synchronize()
    for p, o in ((outs[1][0], outs[1][1]), (picks, st)):
        assert torch.equal(p, outs[0][0])
        for n in ("history", "length", "positions", "next_ids", "finished"):
            assert torch.equal(o[n], outs[0][1][n]), n


# ---------------------------------------------------------------------------------------------------------------
# end to end
# ---------------------------------------------------------------------------------------------------------------
def _random_asr_draft(dev):
    import bench
    torch.manual_seed(11)
    with torch.device(dev):
        d = modeling.B200TouchAudioForCausalLM(bench.asr_config(2)).to(BF16)
    with torch.no_grad():
        for p in d.parameters():
            p.normal_(0, 0.03) if p.dim() == 2 else p.fill_(1.0)
    return d


@pytest.mark.parametrize("k", [1, 3])
def test_greedy_with_a_draft_equals_generate_many_on_the_asr_geometry(k):
    dev = require_cuda()
    model, cfg = _asr_model(dev)
    V = cfg.text_config.vocab_size
    prompts = [_asr_prompt(T, 40 + i, dev) for i, T in enumerate((300, 100, 40, 257, 130, 2, 77))]
    budgets = [12, 7, 16, 5, 9, 14, 1]
    kw = dict(max_new_tokens=budgets, eos_token_id=V, pad_token_id=0, repetition_penalty=1.5, no_repeat_ngram_size=2,
              max_prompt_length=300)
    for B in (3, 12):                                   # more prompts than slots; fewer prompts than batch_size
        base = model.generate_many(prompts, batch_size=B, **kw)
        for draft in (model, _random_asr_draft(dev)):
            stats = {}
            got = model.generate_many(prompts, batch_size=B, assistant_model=draft, num_assistant_tokens=k,
                                      stats=stats, **kw)
            for i, (a, b) in enumerate(zip(got, base)):
                assert torch.equal(a, b), (B, k, i)
            assert stats["rounds"] >= 1 and stats["live_row_rounds"] >= stats["rounds"]


def test_greedy_with_a_draft_equals_generate_many_on_a_touch_audio_model_with_features():
    dev = require_cuda()
    model = _touch_audio_small(dev)
    draft = _touch_audio_small(dev)
    with torch.no_grad():
        for p in draft.parameters():
            if p.dim() == 2:
                p.add_(torch.randn_like(p) * 0.03)
    prompts = _fbank_prompts(dev, [1.0, 0.5, 2.0, 0.3, 1.2])
    kw = dict(batch_size=2, max_new_tokens=[9, 4, 13, 6, 11], eos_token_id=2, pad_token_id=0,
              repetition_penalty=1.5, no_repeat_ngram_size=2)
    base = model.generate_many(prompts, **kw)
    for d in (model, draft):
        for k in (1, 3):
            got = model.generate_many(prompts, assistant_model=d, num_assistant_tokens=k, **kw)
            assert all(torch.equal(a, b) for a, b in zip(got, base)), k


def test_sampled_with_a_draft_is_reproducible_graph_equal_and_invariant_to_batching():
    dev = require_cuda()
    model, cfg = _asr_model(dev)
    V = cfg.text_config.vocab_size
    draft = _random_asr_draft(dev)
    prompts = [_asr_prompt(T, 30 + i, dev) for i, T in enumerate((300, 100, 40, 257, 130, 2))]
    budgets = [12, 7, 16, 5, 9, 14]
    kw = dict(_SAMPLE_KW, eos_token_id=V, max_prompt_length=300, max_new_tokens=budgets, assistant_model=draft,
              num_assistant_tokens=3)

    def run(seed, **extra):
        torch.manual_seed(seed)
        args = dict(kw, batch_size=3)
        args.update(extra)
        return model.generate_many(prompts, **args)

    base = run(0)
    assert [o.numel() for o in base] == budgets
    for r in (run(0), run(0, cuda_graph=False), run(0, batch_size=1), run(0, batch_size=12)):
        for a, b in zip(r, base):
            assert torch.equal(a, b)
    assert any(not torch.equal(a, b) for a, b in zip(run(1), base))
    # the first token of each prompt is the admission's draw: that of sampling without the draft
    torch.manual_seed(0)
    plain = model.generate_many(prompts, **dict(_SAMPLE_KW, eos_token_id=V, max_prompt_length=300,
                                                max_new_tokens=budgets, batch_size=3))
    assert all(int(a[0]) == int(b[0]) for a, b in zip(base, plain))


def test_top_k_1_on_unique_maxima_commits_what_the_greedy_verify_commits():
    """Kernel level: with top_k = 1 and a unique maximum in every target row, p is a point mass on the greedy pick, so
    the sampled verify accepts exactly the draft tokens equal to it and emits it at the first mismatch: the state it
    writes is tn_verify_select_bf16's, bit for bit."""
    dev = require_cuda()
    for V in (64, 128256):
        g = torch.Generator().manual_seed(V)
        B, k = 16, 3
        logits = torch.randn(B * (k + 1), V, generator=g) * 2
        top = torch.randint(0, V, (B * (k + 1),), generator=g)
        logits[torch.arange(B * (k + 1)), top] += 50.0                     # a unique maximum, whatever the penalty
        logits = logits.to(dev, BF16)
        top = top.view(B, k + 1).to(dev)
        drafts = top[:, :k].clone()
        drafts[1::2, 1] = (drafts[1::2, 1] + 1) % V                        # odd slots: rejected at position 1
        drafts[2::4, 0] = (drafts[2::4, 0] + 3) % V                        # every fourth: rejected at position 0
        dlogits = (torch.randn(B * k, V, generator=g) * 2).to(dev, BF16)
        dlogits[torch.arange(B * k, device=dev), drafts.reshape(-1)] = 40.0
        keys = torch.arange(B, dtype=torch.int64, device=dev)
        a, b = _state(B, 32, dev), _state(B, 32, dev)
        a["finished"][5] = b["finished"][5] = 1
        a["limit"][7] = b["limit"][7] = 3
        ops.verify_select(logits, drafts, a["history"], a["length"], a["positions"], a["next_ids"], a["finished"],
                          a["limit"], 1.5, 0, int(top[9, 1]), 0)
        _verify(logits, dlogits, drafts, b, keys, 0.8, 1, 0.9, seed=3, eos=int(top[9, 1]), pad=0, penalty=1.5)
        for n in ("history", "length", "positions", "next_ids", "finished"):
            assert torch.equal(a[n], b[n]), (V, n)
        assert sorted(set(a["length"].tolist())) != [1]


def _top1_generate(monkeypatch, model, prompts, kw, **extra):
    """generate_many(do_sample=True, top_k=1, **extra) and the number of tied maxima among the rows whose draw could
    reach the output: the admission's rows and, per round, the verify rows of live slots."""
    seen = {"ties": 0}
    real_sample, real_verify = ops.sample_select_slots, ops.spec_sample_verify

    def tied(rows):
        lf = rows.float()
        return int(((lf == lf.max(1, keepdim=True).values).sum(1) > 1).sum())

    def sample_spy(logits, history, length, positions, next_ids, finished, *a, row_slot=None, row_key=None):
        if row_slot is not None or "assistant_model" not in extra:
            live = torch.arange(logits.shape[0]) if row_slot is not None else (finished == 0).nonzero()[:, 0]
            seen["ties"] += tied(logits[live.to(logits.device)])
        real_sample(logits, history, length, positions, next_ids, finished, *a, row_slot=row_slot, row_key=row_key)

    def verify_spy(logits, dlogits, drafts, history, length, positions, next_ids, finished, *a, **k):
        live = (finished == 0).nonzero()[:, 0]
        V = logits.shape[1]
        seen["ties"] += tied(logits.view(-1, drafts.shape[1] + 1, V)[live].reshape(-1, V))
        return real_verify(logits, dlogits, drafts, history, length, positions, next_ids, finished, *a, **k)

    with monkeypatch.context() as m:
        m.setattr(ops, "sample_select_slots", sample_spy)
        m.setattr(ops, "spec_sample_verify", verify_spy)
        out = model.generate_many(prompts, do_sample=True, top_k=1, cuda_graph=False, **kw, **extra)   # spies sync
    return out, seen["ties"]


def _wide_touch_audio(dev):
    model = _touch_audio_small(dev)
    with torch.no_grad():
        model.language_model.lm_head.weight.mul_(8)                       # wide logits: few ties at the maximum
    return model


# prompt durations for which no row that can reach the output has a tied maximum on _wide_touch_audio (other durations
# tried, e.g. [1.0, 0.5, 0.7], have one or two tied rows, where top_k = 1 keeps the whole group and draws among it)
@pytest.mark.parametrize("seconds", [[0.8, 0.6, 1.1], [1.3, 0.5, 0.9]])
def test_sampled_top_k_1_with_a_draft_equals_greedy(monkeypatch, seconds):
    """top_k = 1 keeps only the maximum.  On this fixed model and these prompts no row that can reach the output has a
    tied maximum (asserted), so every draw, acceptance and residual is the greedy pick and the result is greedy
    generate_many's, bit for bit."""
    dev = require_cuda()
    model = _wide_touch_audio(dev)
    prompts = _fbank_prompts(dev, seconds)
    kw = dict(batch_size=2, max_new_tokens=[9, 4, 12], eos_token_id=2, pad_token_id=0)
    greedy = model.generate_many(prompts, **kw)
    for k in (1, 3):
        got, ties = _top1_generate(monkeypatch, model, prompts, kw, assistant_model=model, num_assistant_tokens=k)
        assert ties == 0, k
        assert all(torch.equal(a, b) for a, b in zip(got, greedy)), k


def test_sampled_first_generated_tokens_do_not_separate_from_plain_sampling():
    """Many copies of one prompt on a tiny model: the second generated token (the first the verifier emits) has the
    same distribution with and without a draft (two-sample chi-square)."""
    from scipy.stats import chi2_contingency
    dev = require_cuda()
    model = _touch_audio_small(dev)
    draft = _touch_audio_small(dev)
    with torch.no_grad():
        for p in draft.parameters():
            if p.dim() == 2:
                p.add_(torch.randn_like(p) * 0.05)
        model.language_model.lm_head.weight.mul_(3)
    prompt = {"input_ids": torch.tensor([5, 9, 11, 1], device=dev)}
    n = 1500
    kw = dict(batch_size=128, max_new_tokens=3, eos_token_id=-1, pad_token_id=0, do_sample=True, temperature=1.0,
              top_k=0, top_p=1.0)
    torch.manual_seed(0)
    a = torch.stack(model.generate_many([prompt] * n, **kw)).cpu()
    torch.manual_seed(1)
    b = torch.stack(model.generate_many([prompt] * n, assistant_model=draft, num_assistant_tokens=2, **kw)).cpu()
    for pos in (1, 2):
        ca = torch.bincount(a[:, pos], minlength=320).double()
        cb = torch.bincount(b[:, pos], minlength=320).double()
        keep = (ca + cb) >= 10
        table = torch.stack([torch.cat([ca[keep], ca[~keep].sum()[None]]),
                             torch.cat([cb[keep], cb[~keep].sum()[None]])])
        table = table[:, table.sum(0) > 0]
        assert float(chi2_contingency(table.numpy())[1]) > 1e-4, pos
