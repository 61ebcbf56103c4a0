"""GPU: every draw of the sampling kernels equals the exact CPU replay of tests/sample_replay.py, token for token.

  select        tn_sample_select_slots_bf16 on the cases of tests/sample_replay_cases.py (V from 1 to 156032 across the
                draw_index_order chunk sizes; temperature, top_k, top_p, penalty and ngram; keys >= 2^32 and negative
                seeds; row -> slot maps; edge rows): each drawn token is in the replay's set, and every state write is
                the slot rule's
  spec          tn_spec_sample_verify_bf16 for k in {1, 3, 8}: each position's pick (accepted draft token or emitted
                token) is in the replay's set, and the committed state is commit_row's for those picks
  host wiring   generate_many(do_sample=True), with and without a draft: every selection and verify launch is checked
                against the replay on its own inputs; the seeds are the first (and second) int64 draws of torch's
                default generator after torch.manual_seed, and each slot's stream key is its prompt's index

A test passes only if no draw falls outside its set and the share of draws whose set holds more than one token (the
draw lies within the ex2.approx error of a boundary) stays at or below AMBIGUOUS_MAX."""
import numpy as np
import pytest
import torch

from tests.gpu_util import require_cuda
from tests.sample_replay import select_commit, spec_commit
from tests.sample_replay_cases import SELECT_V, SPEC_V, replay_select, replay_spec, select_cases, spec_cases
from tests.test_gpu_generate_many import _touch_audio_small
from touchnet_b200 import ops

pytestmark = pytest.mark.gpu
AMBIGUOUS_MAX = 0.01                          # over each test's draws
_STATE = ("history", "length", "positions", "next_ids", "finished", "limit", "stream_key")


def _report(name, sizes, total=None):
    """Print a case's draw count and ambiguous share; add both to `total` ([draws, ambiguous])."""
    n = len(sizes)
    amb = sum(s > 1 for s in sizes)
    print(f"{name}: {n} draws compared, ambiguous share {amb / max(n, 1):.4f}")
    assert n > 0, name
    if total is not None:
        total[0] += n
        total[1] += amb


def _check_total(total):
    print(f"in all: {total[0]} draws compared, ambiguous share {total[1] / total[0]:.4f}")
    assert total[1] <= AMBIGUOUS_MAX * total[0], total


def _np_state(case):
    return {n: case[n].numpy().copy() for n in _STATE}


def _check_select(name, case, got, sets):
    """got: the kernel's state (numpy) after the launch of `case`; sets: replay_select(case)."""
    want = _np_state(case)
    slots = case["row_slot"] if case["row_slot"] is not None else list(range(case["logits"].shape[0]))
    sizes = []
    for r, b in enumerate(slots):
        if sets[r] is None:                                          # finished: only next_ids = pad
            want["next_ids"][b] = case["pad"]
            continue
        tok = int(got["next_ids"][b])
        assert tok in sets[r], (name, r, b, tok, sorted(sets[r])[:8])
        sizes.append(len(sets[r]))
        select_commit(want, b, tok, int(case["length"][b]), case["eos"],
                      None if case["row_key"] is None else case["row_key"][r])
    for n in _STATE:
        assert np.array_equal(got[n], want[n]), (name, n)
    return sizes


def _check_spec(name, case, picks, got, sets):
    want = _np_state(case)
    k = case["k"]
    sizes = []
    for b, row in enumerate(sets):
        if row is None:
            want["next_ids"][b] = case["pad"]
            continue
        for j in range(k + 1):
            assert int(picks[b, j]) in row[j], (name, case.get("kind", ["?"] * (b + 1))[b], b, j, int(picks[b, j]),
                                                sorted(row[j])[:8])
            sizes.append(len(row[j]))
        L = int(case["length"][b])
        toks, fin = spec_commit(picks[b], k, L, int(case["limit"][b]), case["eos"])
        n = len(toks)
        hw = max(0, min(n, want["history"].shape[1] - L))
        want["history"][b, L:L + hw] = toks[:hw]
        want["length"][b] += n
        want["positions"][b] += n
        want["next_ids"][b] = toks[-1]
        if fin:
            want["finished"][b] = 1
    for n in _STATE:
        assert np.array_equal(got[n], want[n]), (name, n)
    return sizes


@pytest.mark.parametrize("V", SELECT_V)
def test_select_draws_equal_the_replay(V):
    dev = require_cuda()
    total = [0, 0]
    for name, case in select_cases():
        if case["V"] != V:
            continue
        st = {n: case[n].to(dev) for n in _STATE}
        pen, ng, t, top_k, top_p = case["knobs"]
        ops.sample_select_slots(case["logits"].to(dev), st["history"], st["length"], st["positions"], st["next_ids"],
                                st["finished"], st["limit"], st["stream_key"], pen, ng, t, top_k, top_p, case["seed"],
                                case["eos"], case["pad"], row_slot=case["row_slot"], row_key=case["row_key"])
        got = {n: v.cpu().numpy() for n, v in st.items()}
        _report(name, _check_select(name, case, got, replay_select(case)), total)
    _check_total(total)


@pytest.mark.parametrize("V", SPEC_V)
def test_spec_verify_picks_equal_the_replay(V):
    dev = require_cuda()
    total = [0, 0]
    for name, case in spec_cases():
        if case["V"] != V:
            continue
        st = {n: case[n].to(dev) for n in _STATE}
        pen, ng, t, top_k, top_p = case["knobs"]
        picks = ops.spec_sample_verify(case["logits"].to(dev), case["dlogits"].to(dev), case["draft"].to(dev),
                                       st["history"], st["length"], st["positions"], st["next_ids"], st["finished"],
                                       st["limit"], st["stream_key"], pen, ng, t, top_k, top_p, case["seed"],
                                       case["eos"], case["pad"]).cpu().numpy()
        got = {n: v.cpu().numpy() for n, v in st.items()}
        _report(name, _check_spec(name, case, picks, got, replay_spec(case)), total)
    _check_total(total)


# ---------------------------------------------------------------------------------------------------------------
# host wiring: generate_many's launches against the replay
# ---------------------------------------------------------------------------------------------------------------
_FIRST_ID = 10                                # prompt i starts with token _FIRST_ID + i: a slot's history names it


@pytest.mark.parametrize("with_draft", [False, True])
def test_generate_many_draws_equal_the_replay(monkeypatch, with_draft):
    dev = require_cuda()
    model = _touch_audio_small(dev)
    draft = None
    if with_draft:
        draft = _touch_audio_small(dev)
        with torch.no_grad():
            for p in draft.parameters():
                if p.dim() == 2:
                    p.add_(torch.randn_like(p) * 0.05)
    with torch.no_grad():
        model.language_model.lm_head.weight.mul_(3)
    g = torch.Generator().manual_seed(5)
    prompts = []
    for i in range(7):
        ids = torch.randint(3, 320, (int(torch.randint(2, 30, (), generator=g)),), generator=g)
        ids[0] = _FIRST_ID + i
        prompts.append({"input_ids": ids.to(dev)})
    budgets = [int(torch.randint(3, 14, (), generator=g)) for _ in prompts]
    knobs = dict(repetition_penalty=1.3, no_repeat_ngram_size=2, temperature=0.8, top_k=40, top_p=0.9)
    real_sample, real_verify = ops.sample_select_slots, ops.spec_sample_verify
    seen = {"seeds": set(), "verify_seeds": set(), "sizes": [], "launches": 0}

    def key_ok(key, hist_row):
        return int(key) == int(hist_row[0]) - _FIRST_ID

    def sample_spy(logits, history, length, positions, next_ids, finished, limit, stream_key, pen, ng, t, tk, tp,
                   seed, eos, pad, row_slot=None, row_key=None):
        case = dict(V=logits.shape[1], knobs=(pen, ng, t, tk, tp), seed=seed, eos=eos, pad=pad,
                    logits=logits.cpu(), base=logits.cpu(), row_base=torch.arange(logits.shape[0]),
                    row_slot=row_slot, row_key=row_key, history=history.cpu(), length=length.cpu(),
                    positions=positions.cpu(), next_ids=next_ids.cpu(), finished=finished.cpu(), limit=limit.cpu(),
                    stream_key=stream_key.cpu())
        real_sample(logits, history, length, positions, next_ids, finished, limit, stream_key, pen, ng, t, tk, tp,
                    seed, eos, pad, row_slot=row_slot, row_key=row_key)
        got = dict(history=history.cpu().numpy(), length=length.cpu().numpy(), positions=positions.cpu().numpy(),
                   next_ids=next_ids.cpu().numpy(), finished=finished.cpu().numpy(), limit=limit.cpu().numpy(),
                   stream_key=stream_key.cpu().numpy())
        seen["sizes"] += _check_select("generate_many select", case, got, replay_select(case))
        seen["seeds"].add(seed)
        seen["launches"] += 1
        slots = row_slot if row_slot is not None else range(logits.shape[0])
        for r, b in enumerate(slots):
            if not case["finished"][b]:
                key = row_key[r] if row_key is not None else case["stream_key"][b]
                assert key_ok(key, case["history"][b]), (r, b, key)

    def verify_spy(logits, dlogits, drafts, history, length, positions, next_ids, finished, limit, stream_key, pen,
                   ng, t, tk, tp, seed, eos, pad, picks=None):
        case = dict(V=logits.shape[1], k=drafts.shape[1], knobs=(pen, ng, t, tk, tp), seed=seed, eos=eos, pad=pad,
                    logits=logits.cpu(), dlogits=dlogits.cpu(), draft=drafts.cpu(), history=history.cpu(),
                    length=length.cpu(), positions=positions.cpu(), next_ids=next_ids.cpu(),
                    finished=finished.cpu(), limit=limit.cpu(), stream_key=stream_key.cpu())
        out = real_verify(logits, dlogits, drafts, history, length, positions, next_ids, finished, limit, stream_key,
                          pen, ng, t, tk, tp, seed, eos, pad, picks=picks)
        got = dict(history=history.cpu().numpy(), length=length.cpu().numpy(), positions=positions.cpu().numpy(),
                   next_ids=next_ids.cpu().numpy(), finished=finished.cpu().numpy(), limit=limit.cpu().numpy(),
                   stream_key=stream_key.cpu().numpy())
        seen["sizes"] += _check_spec("generate_many verify", case, out.cpu().numpy(), got, replay_spec(case))
        seen["verify_seeds"].add(seed)
        seen["launches"] += 1
        for b in range(drafts.shape[0]):
            if not case["finished"][b]:
                assert key_ok(case["stream_key"][b], case["history"][b]), b
        return out

    torch.manual_seed(1234)
    seeds = [int(torch.randint(-2 ** 63, 2 ** 63 - 1, (), dtype=torch.int64)) for _ in range(2)]
    extra = dict(assistant_model=draft, num_assistant_tokens=3) if with_draft else {}
    monkeypatch.setattr(ops, "sample_select_slots", sample_spy)
    monkeypatch.setattr(ops, "spec_sample_verify", verify_spy)
    torch.manual_seed(1234)
    out = model.generate_many(prompts, batch_size=3, max_new_tokens=budgets, eos_token_id=2, pad_token_id=0,
                              do_sample=True, cuda_graph=False, **knobs, **extra)
    assert [o.numel() <= b for o, b in zip(out, budgets)] == [True] * len(prompts)
    if with_draft:
        assert seen["seeds"] == set(seeds) and seen["verify_seeds"] == {seeds[0]}
    else:
        assert seen["seeds"] == {seeds[0]} and not seen["verify_seeds"]
    total = [0, 0]
    _report(f"generate_many draft={with_draft} ({seen['launches']} launches)", seen["sizes"], total)
    _check_total(total)
