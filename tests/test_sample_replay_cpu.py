"""CPU: the replay of tests/sample_replay.py checks itself before the GPU tests trust it.

  philox     the Random123 known-answer vectors of philox4x32-10, and the kernels' stream contract around it
  kept sets  the replay's kept sets against the fp64 oracle of tests/sample_oracle.py and transformers' warpers
  spec       the emitted-token frequencies of the replayed speculative sampling against tests/spec_sample_oracle.py
  power      on the GPU tests' own inputs, each defective variant of the replay (sample_replay.MUTATIONS) disagrees
             with the true replay on at least a stated share of the draws both determine: a kernel with that defect
             fails tests/test_gpu_sample_replay.py"""
import numpy as np
import pytest
import torch

from tests.sample_oracle import distribution, hf_kept
from tests.sample_replay import (ACCEPT, LOG2E_F32, PLAIN, RESIDUAL, Dist, draw_bits, philox4x32_10, processed, spec_commit,
                                 spec_position)
from tests.sample_replay_cases import replay_select, replay_spec, select_cases, spec_cases
from tests.spec_sample_oracle import emitted


@pytest.mark.parametrize("ctr, key, out", [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_philox_known_answers(ctr, key, out):
    assert tuple(int(w) for w in philox4x32_10(ctr, key)) == out
    got = philox4x32_10([np.full(3, c) for c in ctr], [np.full(3, k) for k in key])   # vectorised over rows
    assert all((w == o).all() for w, o in zip(got, out))


def test_draw_bits_follow_the_stream_contract():
    """r = (y << 32) | x of Philox at counter (pos, purpose, key lo, key hi) under (seed lo, seed hi), with negative
    seeds and keys as their two's-complement bits."""
    seed, key, pos = -(2 ** 40) - 5, -(2 ** 33) + 1, 41
    s, k = seed % 2 ** 64, key % 2 ** 64
    for purpose in (PLAIN, ACCEPT, RESIDUAL):
        x, y, _, _ = philox4x32_10((pos, purpose, k & 0xFFFFFFFF, k >> 32), (s & 0xFFFFFFFF, s >> 32))
        assert int(draw_bits(seed, pos, purpose, key)) == (int(y) << 32) | int(x)
    r = draw_bits(seed, np.array([pos, pos]), PLAIN, np.array([key, 2 ** 32]))
    assert int(r[0]) == int(draw_bits(seed, pos, PLAIN, key)) != int(r[1])


# ---------------------------------------------------------------------------------------------------------------
# kept sets
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("top_k, top_p", [(50, 1.0), (0, 0.9), (50, 0.9), (1, 1.0), (0, 0.0), (7, 0.3), (2, 0.5)])
def test_kept_sets_match_the_oracle_and_hf(top_k, top_p):
    g = torch.Generator().manual_seed(top_k * 100 + int(top_p * 10))
    for trial in range(12):
        V = [64, 1000, 5000][trial % 3]
        x = (torch.randn(V, generator=g) * 3).to(torch.bfloat16).float()     # bf16: ties
        d = Dist(x.numpy(), top_k, top_p)
        probs, band = distribution(x, top_k, top_p)
        oracle = probs > 0
        for kept in d.cuts:
            kept = torch.from_numpy(kept)
            assert torch.equal(kept | band, oracle | band), trial
        tied_boundary = False
        if 0 < top_k < V:
            tied_boundary = int((x == x.topk(top_k).values[-1]).sum()) > 1
        if not tied_boundary and len(d.cuts) == 1 and not band.any():
            kept = torch.from_numpy(d.cuts[0])
            hf = hf_kept(x, top_k, top_p)
            if top_p < 1.0:                                           # HF cuts inside a tie: compare outside it
                cut_vals = x[kept & ~hf].unique()
                same = ~torch.isin(x, x[kept ^ hf].unique()) if (kept ^ hf).any() else torch.ones(V, dtype=bool)
                assert cut_vals.numel() <= 1, trial
                assert torch.equal(kept[same], hf[same]), trial
            else:
                assert torch.equal(kept, hf), trial


def test_processing_and_degenerate_rows():
    row = np.array([1.0, -2.0, 3.0, 0.5, -0.0, 2.0], dtype=np.float32)
    x = processed(row, [0, 1, 3, 0, 1], penalty=2.0, ngram=2, temperature=0.5)
    # the penalty on 0, 1 and 3 (x / 2 above 0, x * 2 below); the history ends in 1 and (1, 3) occurred: 3 is banned
    assert x.tolist() == [1.0, -8.0, 6.0, -np.inf, -0.0, 4.0]
    assert Dist(np.array([1, np.nan, 2, np.nan], np.float32), 0, 1.0).pick == 1
    assert Dist(np.array([1, np.inf, 2, np.inf], np.float32), 0, 1.0).pick == 1
    d = Dist(np.full(5, -np.inf, np.float32), 2, 0.5)
    assert d.degenerate and d.draw(123) == {0}
    tie = Dist(np.array([3.0, 1.0, 3.0, 2.0, 2.0], np.float32), 3, 1.0)   # top-k keeps the whole tied group
    assert tie.cuts[0].tolist() == [True, False, True, True, True]


def test_weights_near_half_are_zero_or_one():
    half = np.float32(-41 / np.log2(np.e))                         # y = fl(x * log2e) = -41: W = rni(0.5 (1 +- EPS))
    while np.float32(half * LOG2E_F32) != -41:
        half = np.nextafter(half, np.float32(0 if half * LOG2E_F32 < -41 else -100))
    x = np.array([0.0, -28.375, -28.625, half, -200.0], np.float32)
    d = Dist(x, 0, 1.0)
    assert d.lo.tolist()[1:] == [1, 0, 0, 0] and d.hi.tolist()[1:] == [1, 0, 1, 0]
    assert d.lo[0] < 2 ** 40 < d.hi[0] and d.hi[0] - d.lo[0] <= 2 ** 20


def test_spec_commit_rules():
    assert spec_commit([4, 5, ~6], 2, 10, 100, -1) == ([4, 5, 6], False)
    assert spec_commit([4, ~5, 7], 2, 10, 100, -1) == ([4, 5], False)
    assert spec_commit([4, 5, ~6], 2, 10, 100, 4) == ([4], True)             # eos
    assert spec_commit([4, 5, ~6], 2, 10, 12, -1) == ([4, 5], True)          # the limit
    assert spec_commit([~3, 5, ~6], 2, 10, 100, -1) == ([3], False)


# ---------------------------------------------------------------------------------------------------------------
# the replayed speculative sampling emits p's distribution
# ---------------------------------------------------------------------------------------------------------------
def test_spec_replay_emits_the_oracle_distribution():
    from scipy.stats import chisquare
    V, N = 32, 3000
    g = torch.Generator().manual_seed(3)
    p = (torch.randn(V, generator=g) * 2).to(torch.bfloat16).float().numpy()
    q = (torch.randn(V, generator=g) * 2).to(torch.bfloat16).float().numpy()
    knobs = (1.0, 0, 1.0, 0, 1.0)
    Q = Dist(q, 0, 1.0)
    counts = np.zeros(V)
    for key in range(N):
        x = Q.draw(draw_bits(77, 5, PLAIN, key))                     # the draft's proposal, drawn from q
        assert len(x) == 1
        out = spec_position(p, q, [], x.pop(), 11, 0, key, knobs)
        assert len(out) == 1
        pick = out.pop()
        counts[pick if pick >= 0 else ~pick] += 1
    pp = torch.softmax(torch.from_numpy(p).double(), 0)
    qq = torch.softmax(torch.from_numpy(q).double(), 0)
    want = (emitted(pp, qq) * N).numpy()
    keep = want >= 5
    obs = np.r_[counts[keep], counts[~keep].sum()]
    exp = np.r_[want[keep], want[~keep].sum()]
    assert chisquare(obs, exp).pvalue > 1e-3
    assert np.allclose(emitted(pp, qq).numpy(), pp.numpy())


# ---------------------------------------------------------------------------------------------------------------
# power: each defect changes a stated share of the draws of the GPU tests' inputs
# ---------------------------------------------------------------------------------------------------------------
_SELECT_V = (33, 1000, 1025, 32 * 1024 + 1)   # the fast cases of the GPU test
_SPEC_V = (64, 1000)


def _disagreement(true, mutated):
    """(share of the draws both replays determine on which they differ, that count)."""
    pairs = [(a, b) for a, b in zip(true, mutated) if a is not None and len(a) == 1 and len(b) == 1]
    return sum(a != b for a, b in pairs) / max(len(pairs), 1), len(pairs)


def _flat_select(mut, knobs=None):
    out = []
    for name, case in _SELECT:
        if case["V"] in _SELECT_V and (knobs is None or name.endswith(tuple(f"knobs{i}" for i in knobs))):
            out += replay_select(case, mut)
    return out


def _flat_spec(mut):
    return [s for _, case in _SPEC if case["V"] in _SPEC_V for row in replay_spec(case, mut) if row is not None
            for s in row]


_SELECT = select_cases()
_SPEC = spec_cases()


# Shares about half the measured ones.  A select case's degenerate rows (NaN, +inf, all -inf) and its top_k = 1 or
# top_p = 0 knob sets draw one token whatever the stream, so about three quarters of its draws change with the stream.
@pytest.mark.parametrize("mut, knobs, share", [
    ("counter_plus_1", None, 0.12),
    ("swap_seed_words", None, 0.12),
    ("swap_r_words", None, 0.12),
    ("value_order", (0, 2, 6), 0.12),         # the knob sets that keep many tokens
    ("topk_drop_ties", (3,), 0.05),           # top_k = 2: the rows with a tie across the boundary
    ("topp_inclusive", (1, 3, 5, 6), 0.015),  # top_p in (0, 1): draws of the boundary group
])
def test_select_mutations_are_detected(mut, knobs, share):
    got, n = _disagreement(_flat_select((), knobs), _flat_select((mut,), knobs))
    print(f"{mut}: {got:.4f} of {n} draws differ")
    assert n >= 500 and got >= share, (mut, got, n)


@pytest.mark.parametrize("mut, share", [("swap_purposes", 0.1), ("residual_q_minus_p", 0.05),
                                        ("counter_plus_1", 0.1), ("swap_seed_words", 0.1)])
def test_spec_mutations_are_detected(mut, share):
    got, n = _disagreement(_flat_spec(()), _flat_spec((mut,)))
    print(f"{mut}: {got:.4f} of {n} draws differ")
    assert n >= 500 and got >= share, (mut, got, n)
