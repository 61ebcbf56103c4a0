"""GPU: multinomial sampling over cache slots (tn_sample_select_slots_bf16 in touchnet_b200/csrc/decode.cu;
generation.generate_many with do_sample=True).

  distribution  thousands of identical rows, each with its own stream key, over three lengths: the histogram of the
                draws against the fp64 distribution of tests/sample_oracle.py (chi-square, bins merged to an expected
                count >= 5), V in {64, 1000, 128256}, across temperature / top_k / top_p / penalty / ngram; no draw
                outside the oracle's kept set except in its top-p boundary band
  exact         top_k=1 and top_p=0 on a unique maximum give the greedy kernel's token; m tied maxima give only those m;
                all-banned and NaN rows give the greedy pick
  slot state    idle and finished slots hold still, the limit finishes a slot, every write matches greedy_select_slots;
                a mapped row stores its stream key
  determinism   the same launch twice and a graph-captured launch give the same bits
  end to end    on the Llama-3.2-3B-ASR geometry (2 layers, random weights): reproducible under torch.manual_seed, eager
                equals graph replay, a prompt's ids do not depend on batch_size or on another prompt's budget; top_k=1
                on a tiny model selects what the greedy kernel selects"""
import pytest
import torch

from tests.gpu_util import require_cuda
from tests.sample_oracle import distribution, processed
from tests.test_gpu_generate_many import _asr_model, _asr_prompt, _touch_audio_small
from touchnet_b200 import ops

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16


def _state(B, S, hist_row, L, dev, limit=None):
    return dict(history=hist_row.to(dev).repeat(B, 1), length=torch.full((B,), L, dtype=torch.int32, device=dev),
                positions=torch.arange(B, dtype=torch.int64, device=dev),
                next_ids=torch.full((B,), -5, dtype=torch.int64, device=dev),
                finished=torch.zeros(B, dtype=torch.int32, device=dev),
                limit=torch.full((B,), S if limit is None else limit, dtype=torch.int32, device=dev))


def _sample(logits, st, key, penalty, ngram, t, k, p, seed, eos=-1, pad=0, **kw):
    ops.sample_select_slots(logits, st["history"], st["length"], st["positions"], st["next_ids"], st["finished"],
                            st["limit"], key, penalty, ngram, t, k, p, seed, eos, pad, **kw)


def _greedy(logits, st, penalty, ngram, eos=-1, pad=0, **kw):
    ops.greedy_select_slots(logits, st["history"], st["length"], st["positions"], st["next_ids"], st["finished"],
                            st["limit"], penalty, ngram, eos, pad, **kw)


def _chi2_pvalue(counts, expected):
    from scipy.stats import chisquare
    order = torch.argsort(expected, descending=True)
    obs, exp, bins_o, bins_e = 0.0, 0.0, [], []
    for i in order.tolist():
        obs += float(counts[i]); exp += float(expected[i])
        if exp >= 5:
            bins_o.append(obs); bins_e.append(exp)
            obs, exp = 0.0, 0.0
    if bins_e:                                        # the tail joins the last bin
        bins_o[-1] += obs; bins_e[-1] += exp
    if len(bins_e) < 2:
        return 1.0
    return float(chisquare(bins_o, bins_e).pvalue)


@pytest.mark.parametrize("V, t, k, p, pen, ng, scale", [
    (64, 1.0, 0, 1.0, 1.0, 0, 1.5),
    (64, 0.7, 10, 0.9, 1.5, 2, 1.5),
    (1000, 1.3, 50, 1.0, 1.0, 0, 2.0),
    (1000, 0.7, 0, 0.8, 1.5, 2, 2.0),
    (1000, 0.5, 1000, 0.5, 1.5, 1, 2.0),
    (128256, 0.7, 50, 0.9, 1.5, 2, 2.5),
    (128256, 1.0, 0, 0.9, 1.0, 0, 4.0),
])
def test_draws_follow_the_oracle_distribution(V, t, k, p, pen, ng, scale):
    dev = require_cuda()
    B, S = 2048, 64
    g = torch.Generator().manual_seed(V + k)
    row = (torch.randn(V, generator=g) * scale).to(BF16)             # bf16: many tied values
    hist = torch.randint(0, min(V, 200), (S,), generator=g)
    hist[38:40] = hist[10:12]                                          # the last bigram occurred before (length 40)
    logits = row.to(dev)[None].repeat(B, 1)
    key = torch.arange(B, dtype=torch.int64, device=dev) * 3 + 11
    counts = torch.zeros(V, dtype=torch.float64)
    expected = torch.zeros(V, dtype=torch.float64)
    allowed = torch.zeros(V, dtype=torch.bool)
    for L in (40, 41, 42):
        st = _state(B, S, hist, L, dev)
        _sample(logits, st, key, pen, ng, t, k, p, seed=987654321 + V)
        ids = st["next_ids"].cpu()
        counts += torch.bincount(ids, minlength=V).double()
        x = processed(hist[None, :L], row.float()[None], pen, ng, t)
        probs, band = distribution(x, k, p)
        expected += B * probs
        allowed |= (probs > 0) | band
        assert torch.equal(st["length"].cpu(), torch.full((B,), L + 1, dtype=torch.int32))
        assert torch.equal(st["history"][:, L].cpu(), ids)
    outside = counts[~allowed].sum()
    assert outside == 0, f"{int(outside)} draws outside the kept set"
    pv = _chi2_pvalue(counts, expected)
    assert pv > 1e-3, pv


def test_top_k_1_and_top_p_0_on_a_unique_maximum_give_the_greedy_token():
    dev = require_cuda()
    V, B, S = 128256, 64, 64
    g = torch.Generator().manual_seed(7)
    logits = (torch.randn(B, V, generator=g) * 3).to(BF16)
    top = torch.randint(1000, V, (B,), generator=g)
    logits[torch.arange(B), top] = logits.float().max(1).values.to(BF16) + 8   # a unique maximum, outside the history
    logits = logits.to(dev)
    hist = torch.randint(0, 50, (S,), generator=g)
    ref = _state(B, S, hist, 40, dev)
    _greedy(logits, ref, 1.5, 2)
    assert torch.equal(ref["next_ids"].cpu(), top)
    key = torch.arange(B, dtype=torch.int64, device=dev)
    for t, k, p in ((1.0, 1, 1.0), (0.7, 1, 0.9), (1.0, 0, 0.0), (1.3, 50, 0.0)):
        st = _state(B, S, hist, 40, dev)
        _sample(logits, st, key, 1.5, 2, t, k, p, seed=5)
        for name in ref:
            assert torch.equal(st[name], ref[name]), (t, k, p, name)


def test_tied_maxima_are_the_only_draws():
    dev = require_cuda()
    V, B, S = 1000, 2048, 16
    g = torch.Generator().manual_seed(3)
    row = (torch.randn(V, generator=g) * 2).to(BF16)
    ties = [17, 400, 998]
    row[ties] = row.float().max().to(BF16) + 1
    logits = row.to(dev)[None].repeat(B, 1)
    key = torch.arange(B, dtype=torch.int64, device=dev)
    for k, p in ((1, 1.0), (0, 0.0), (2, 0.5)):
        st = _state(B, S, torch.zeros(S, dtype=torch.int64), 8, dev)
        _sample(logits, st, key, 1.0, 0, 1.0, k, p, seed=11)
        assert set(st["next_ids"].tolist()) == set(ties), (k, p)


def test_all_banned_and_nan_rows_take_the_greedy_pick():
    dev = require_cuda()
    V, B, S = 64, 4, 80
    g = torch.Generator().manual_seed(9)
    logits = (torch.randn(B, V, generator=g) * 2).to(BF16)
    logits[1, 30] = float("nan")
    logits[1, 17] = float("nan")
    logits[2, 5] = float("inf")
    logits = logits.to(dev)
    hist = torch.cat([torch.arange(V), torch.arange(V)[:16]])             # every token once: ngram 1 bans them all
    for ngram in (1, 0):
        ref = _state(B, S, hist, V + 4, dev)
        _greedy(logits, ref, 1.0, ngram)
        st = _state(B, S, hist, V + 4, dev)
        _sample(logits, st, torch.arange(B, device=dev), 1.0, ngram, 0.7, 50, 0.9, seed=1)
        picks = st["next_ids"].tolist()
        if ngram == 1:                                                    # banned NaN / inf are -inf too: token 0
            assert picks == [0, 0, 0, 0]
        else:
            assert picks[1] == 17 and picks[2] == 5
        rows = slice(0, B) if ngram == 1 else slice(1, 3)
        for name in ref:
            assert torch.equal(st[name][rows], ref[name][rows]), name


def test_slot_state_matches_greedy_select_slots_and_mapped_rows_store_their_key():
    dev = require_cuda()
    V, B, S = 128256, 6, 64
    g = torch.Generator().manual_seed(V)
    hist = torch.randint(0, 50, (B, S), generator=g)
    lens = torch.tensor([37, 20, 45, 30, 12, 50], dtype=torch.int32)
    logits = (torch.randn(4, V, generator=g) * 3).to(BF16)
    top = torch.randint(1000, V, (4,), generator=g)
    logits[torch.arange(4), top] = logits.float().max(1).values.to(BF16) + 8
    logits = logits.to(dev)

    def fresh():
        st = dict(history=hist.clone().to(dev), length=lens.to(dev),
                  positions=torch.arange(B, dtype=torch.int64, device=dev) + 100,
                  next_ids=torch.full((B,), -5, dtype=torch.int64, device=dev),
                  finished=torch.tensor([0, 0, 0, 1, 0, 1], dtype=torch.int32, device=dev),
                  limit=(lens + 10).to(dev, torch.int32))
        st["limit"][2] = int(lens[2]) + 1                                 # slot 2 takes its last budgeted token
        return st

    row_slot = [4, 0, 5, 2]
    ref, st = fresh(), fresh()
    _greedy(logits, ref, 1.5, 2, eos=-1, pad=0, row_slot=row_slot)
    key = torch.full((B,), -7, dtype=torch.int64, device=dev)
    _sample(logits, st, key, 1.5, 2, 0.7, 1, 0.9, 3, row_slot=row_slot, row_key=[40, 41, 42, 43])
    for name in ref:
        assert torch.equal(st[name], ref[name]), name
    assert st["finished"].tolist() == [0, 0, 1, 1, 0, 1]
    assert key.tolist() == [41, -7, 43, -7, 40, -7]                      # slot 5 is finished: nothing written
    # the identity map over all B rows (a decode step): finished / idle slots hold still, the others read their key
    logits6 = logits[[0, 1, 2, 3, 0, 1]].contiguous()
    ref2 = {n: v.clone() for n, v in ref.items()}
    _greedy(logits6, ref2, 1.5, 2)
    _sample(logits6, st, key, 1.5, 2, 1.0, 1, 1.0, 3)
    for name in ref:
        assert torch.equal(st[name], ref2[name]), name


def test_launches_are_deterministic_and_graph_capture_is_bitwise_equal():
    dev = require_cuda()
    V, B, S = 128256, 12, 1024
    g = torch.Generator().manual_seed(21)
    logits = (torch.randn(B, V, generator=g) * 2.5).to(BF16).to(dev)
    hist = torch.randint(0, V, (S,), generator=g)
    key = torch.arange(B, dtype=torch.int64, device=dev) + 1000
    outs = []
    for mode in ("eager", "eager", "graph"):
        st = _state(B, S, hist, 967, dev)
        run = lambda: _sample(logits, st, key, 1.5, 2, 0.7, 0, 0.9, seed=-42)   # noqa: E731
        if mode == "graph":
            run()                                                       # opt-in and module load outside the capture
            st.update(_state(B, S, hist, 967, dev))
            cg = torch.cuda.CUDAGraph()
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s), torch.cuda.graph(cg, stream=s):
                _sample(logits, st, key, 1.5, 2, 0.7, 0, 0.9, seed=-42)
            torch.cuda.current_stream().wait_stream(s)
            for n, v in _state(B, S, hist, 967, dev).items():
                st[n].copy_(v)
            for _ in range(3):
                cg.replay()
        else:
            for _ in range(3):
                run()
        torch.cuda.synchronize()
        outs.append({n: v.clone() for n, v in st.items()})
    for o in outs[1:]:
        for n in o:
            assert torch.equal(o[n], outs[0][n]), n
    assert len(set(outs[0]["next_ids"].tolist())) > 1                     # the rows drew from their own streams


# ---------------------------------------------------------------------------------------------------------------
# generate_many
# ---------------------------------------------------------------------------------------------------------------
_SAMPLE_KW = dict(pad_token_id=0, repetition_penalty=1.5, no_repeat_ngram_size=2, do_sample=True, temperature=0.7,
                  top_k=50, top_p=0.9)


def test_sampled_generate_many_is_reproducible_and_invariant_to_batching():
    dev = require_cuda()
    model, cfg = _asr_model(dev)
    V = cfg.text_config.vocab_size
    prompts = [_asr_prompt(T, 30 + i, dev) for i, T in enumerate((300, 100, 40, 257, 130, 2))]
    budgets = [12, 7, 16, 5, 9, 14]
    kw = dict(_SAMPLE_KW, eos_token_id=V, max_prompt_length=300)

    def run(seed, **extra):
        torch.manual_seed(seed)
        args = dict(kw, batch_size=3, max_new_tokens=budgets)
        args.update(extra)
        return model.generate_many(prompts, **args)

    base = run(0)
    assert [o.numel() for o in base] == budgets
    assert any(len(set(o.tolist())) > 1 for o in base)
    other = run(1)
    assert any(not torch.equal(a, b) for a, b in zip(base, other))        # a different seed draws differently
    runs = [run(0), run(0, cuda_graph=False), run(0, batch_size=1), run(0, batch_size=4), run(0, batch_size=12)]
    changed = list(budgets)
    changed[0], changed[3] = 3, 10                                        # other prompts' budgets change admissions
    runs.append(run(0, max_new_tokens=changed))
    for r in runs[:-1]:
        for a, b in zip(r, base):
            assert torch.equal(a, b)
    for i, (a, b) in enumerate(zip(runs[-1], base)):
        if i in (0, 3):
            n = min(a.numel(), b.numel())
            assert torch.equal(a[:n], b[:n]), i                            # its own stream, its own positions
        else:
            assert torch.equal(a, b), i


def test_top_k_1_selects_what_the_greedy_kernel_selects(monkeypatch):
    """A tiny model, top_k=1 and no processors: every selection equals the greedy kernel's on the same logits and state
    where the maximum is unique, and without a tie on the way the output is greedy generate_many's, bit for bit."""
    dev = require_cuda()
    model = _touch_audio_small(dev)
    with torch.no_grad():
        model.language_model.lm_head.weight.mul_(8)                       # wide logits: few ties at the maximum
    g = torch.Generator().manual_seed(12)
    prompts = []
    for _ in range(7):
        T = int(torch.randint(2, 60, (), generator=g))
        ids = torch.randint(3, 320, (T,), generator=g)
        prompts.append({"input_ids": ids.to(dev), "input_features": torch.randn(T, 400, generator=g).to(dev, BF16)})
    budgets = [int(torch.randint(2, 12, (), generator=g)) for _ in prompts]
    real = ops.sample_select_slots
    seen = {"rows": 0, "ties": 0}

    def spy(logits, history, length, positions, next_ids, finished, limit, *a, row_slot=None, row_key=None):
        state = [t.clone() for t in (history, length, positions, next_ids, finished)]
        advancing = (finished == 0).tolist()
        ops.greedy_select_slots(logits, *state, limit, 1.0, 0, 2, 0, row_slot=row_slot)
        real(logits, history, length, positions, next_ids, finished, limit, *a, row_slot=row_slot, row_key=row_key)
        slots = list(range(logits.shape[0])) if row_slot is None else row_slot
        lf = logits.float()
        unique = ((lf == lf.max(1, keepdim=True).values).sum(1) == 1).tolist()
        for r, b in enumerate(slots):
            if advancing[b]:
                seen["rows"] += 1
                if unique[r]:
                    assert int(next_ids[b]) == int(state[3][b]), (r, b)
                else:
                    seen["ties"] += 1

    kw = dict(batch_size=3, max_new_tokens=budgets, eos_token_id=2, pad_token_id=0)
    greedy = model.generate_many(prompts, **kw)
    monkeypatch.setattr(ops, "sample_select_slots", spy)
    sampled = model.generate_many(prompts, do_sample=True, top_k=1, cuda_graph=False, **kw)   # the spy syncs
    assert seen["rows"] >= sum(o.numel() for o in sampled)
    if seen["ties"] == 0:
        for a, b in zip(sampled, greedy):
            assert torch.equal(a, b)


def test_do_sample_false_ignores_the_knobs():
    dev = require_cuda()
    model = _touch_audio_small(dev)
    prompts = [{"input_ids": torch.tensor([5, 9, 1], device=dev)}, {"input_ids": torch.tensor([7, 1], device=dev)}]
    kw = dict(batch_size=2, max_new_tokens=6, eos_token_id=2, pad_token_id=0, repetition_penalty=1.5,
              no_repeat_ngram_size=2)
    a = model.generate_many(prompts, **kw)
    b = model.generate_many(prompts, temperature=0.3, top_k=3, top_p=0.5, **kw)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
