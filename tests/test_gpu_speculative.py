"""GPU: speculative decoding - the multi-query decode attention (each row bitwise equal to the single-query kernel at
its own length), the verify selection (each position's pick equal to tn_greedy_select_bf16 on the extended history),
and generate(assistant_model=...) bitwise equal to generate() on a small model, on the Llama-3.2-3B-ASR geometry of
bench.py (fewer layers) and on the TouchAudio reference inference layout."""
import math
from types import SimpleNamespace as NS

import pytest
import torch

import bench
from tests.gpu_util import rel_err, require_cuda
from tests.test_gpu_decode import _REF_KW, _ref_decode
from tests.test_gpu_model import small_cfg
from tools import time_decode
from touchnet_b200 import generation, modeling, ops

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16


# ---------------------------------------------------------------------------------------------------------------
# multi-query decode attention
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("G", [1, 2, 3, 4, 8])
@pytest.mark.parametrize("S_cap", [300, 4100])
def test_multi_query_attention_rows_equal_the_single_query_kernel(G, S_cap):
    dev = require_cuda()
    torch.manual_seed(G * 7 + S_cap)
    KV, B = 2, 4
    H = G * KV
    scale = 1 / math.sqrt(128)
    cache = torch.randn(2, B, S_cap, KV * 128, device=dev).to(BF16)
    kc, vc = cache[0], cache[1]
    splits_chunk = S_cap // 3
    for Tq in sorted({1, 2, 16 // G}):
        # ends that put the new block across a 64-key sub-block boundary and across a split boundary; kv_start > 0
        end = torch.tensor([Tq + 5, 64 + Tq // 2 + 1, splits_chunk + Tq // 2, S_cap - 3], dtype=torch.int32, device=dev)
        start = torch.tensor([0, 3, 60, S_cap - 3 - Tq - 70], dtype=torch.int32, device=dev)
        q = torch.randn(B * Tq, H * 128, device=dev).to(BF16)
        o, lse = ops.attn_decode_multi(q, kc, vc, start, end, Tq, H, KV, scale, lse=True)
        o2, lse2 = ops.attn_decode_multi(q, kc, vc, start, end, Tq, H, KV, scale, lse=True)
        assert torch.equal(o, o2) and torch.equal(lse, lse2)                # reproducible
        for j in range(Tq):
            rows = torch.arange(B, device=dev) * Tq + j
            e = end - Tq + j + 1
            ro, rl = ops.attn_decode(q[rows].contiguous(), kc, vc, start, e, H, KV, scale, lse=True)
            assert torch.equal(o[rows], ro), (G, Tq, j)                      # bitwise: the single-query kernel
            assert torch.equal(lse[rows], rl), (G, Tq, j)
            fo, fl = _ref_decode(q[rows], kc, vc, start, e, H, KV, scale)
            for b in range(B):
                assert rel_err(o[rows[b]].float(), fo[b]) < 2e-2 and rel_err(lse[rows[b]], fl[b]) < 2e-3


def test_multi_query_attention_with_padded_heads_in_a_model_step():
    """head_dim 64 (zero-padded 128-wide heads): the verify step's attention rows equal decode_step's."""
    dev = require_cuda()
    c = small_cfg(d=384, H=6, KV=2, V=320)
    c.head_dim = 64
    torch.manual_seed(3)
    m = modeling.B200LlamaForCausalLM(c).to(dev)
    with torch.no_grad():
        for p in m.parameters():
            p.copy_(torch.randn_like(p) * 0.05 if p.dim() == 2 else 1 + 0.1 * torch.randn_like(p))
    m.to(BF16)
    ids = torch.randint(3, 320, (3, 40), device=dev)
    out = m.generate(ids, max_new_tokens=20, eos_token_id=321, pad_token_id=0, **_REF_KW)
    for k in (1, 3):
        got = m.generate(ids, max_new_tokens=20, eos_token_id=321, pad_token_id=0, assistant_model=m,
                         num_assistant_tokens=k, **_REF_KW)
        assert torch.equal(got, out), k


# ---------------------------------------------------------------------------------------------------------------
# verify selection
# ---------------------------------------------------------------------------------------------------------------
def test_verify_select_picks_equal_greedy_select_on_the_extended_history():
    dev = require_cuda()
    g = torch.Generator().manual_seed(5)
    V, B, k, S_cap, n = 128256, 5, 3, 64, 30
    hist = torch.randint(0, 40, (B, S_cap), generator=g).to(dev)              # small id range: repeats and bans
    logits = (torch.randn(B * (k + 1), V, generator=g) * 3).to(BF16).to(dev)
    draft = torch.randint(0, 40, (B, k), generator=g).to(dev)
    length = torch.tensor([n, n, n + 2, n, n], dtype=torch.int32, device=dev)
    fin = torch.tensor([0, 0, 0, 1, 0], dtype=torch.int32, device=dev)
    limit = torch.tensor([S_cap, S_cap, S_cap, S_cap, n + 2], dtype=torch.int32, device=dev)

    def refs(draft):   # each position's pick from tn_greedy_select_bf16 on the extended history
        ref = torch.zeros(B, k + 1, dtype=torch.int64, device=dev)
        for j in range(k + 1):
            h = hist.clone()
            for b in range(B):
                h[b, int(length[b]):int(length[b]) + j] = draft[b, :j]
            z = torch.zeros(B, dtype=torch.int32, device=dev)
            ops.greedy_select(logits.view(B, k + 1, V)[:, j].contiguous(), h, (length + j).clone(),
                              torch.zeros(B, dtype=torch.int64, device=dev), torch.zeros(B, dtype=torch.int64, device=dev),
                              z, 1.5, 2, -1, 0)
            ref[:, j] = h[torch.arange(B, device=dev), (length + j).long()]
        return ref

    # plant acceptances: rows 0 and 4 accept every proposal, row 2 two (then an eos pick), row 1 none
    for j in range(k):
        r = refs(draft)
        draft[0, j], draft[4, j] = r[0, j], r[4, j]
        if j < 2:
            draft[2, j] = r[2, j]
    draft[1, 0] = refs(draft)[1, 0] + 1
    ref = refs(draft)
    eos = int(ref[2, 2])
    h, ln = hist.clone(), length.clone()
    pos = torch.arange(B, dtype=torch.int64, device=dev) * 100
    nxt = torch.full((B,), -5, dtype=torch.int64, device=dev)
    f = fin.clone()
    picks = ops.verify_select(logits, draft, h, ln, pos, nxt, f, limit, 1.5, 2, eos, 0)
    live = fin == 0
    assert torch.equal(picks[live], ref[live])
    emitted = {0: k + 1, 1: 1, 2: 3, 4: 2}                  # row 2 stops on its eos pick, row 4 at limit n + 2
    for b, c in emitted.items():
        n0 = int(length[b])
        assert int(ln[b]) == n0 + c and int(pos[b]) == b * 100 + c, b
        assert torch.equal(h[b, n0:n0 + c], ref[b, :c]) and torch.equal(h[b, :n0], hist[b, :n0])
        assert torch.equal(h[b, n0 + c:], hist[b, n0 + c:])
        assert int(nxt[b]) == int(ref[b, c - 1])
    assert f.tolist() == [int(ref[0, k] == eos), int(ref[1, 0] == eos), 1, 1, 1]
    assert int(nxt[3]) == 0 and int(ln[3]) == n and torch.equal(h[3], hist[3]) and int(pos[3]) == 300


# ---------------------------------------------------------------------------------------------------------------
# end to end
# ---------------------------------------------------------------------------------------------------------------
def _random(cfg, dev, seed, std=0.05):
    torch.manual_seed(seed)
    with torch.device(dev):
        m = modeling.B200LlamaForCausalLM(cfg)
    with torch.no_grad():
        for p in m.parameters():
            p.normal_(0, std) if p.dim() == 2 else p.fill_(1.0)
    return m.to(BF16)


def test_generate_with_a_draft_equals_generate_on_small_cfg():
    dev = require_cuda()
    model = _random(small_cfg(d=256, H=4, KV=2, V=320), dev, 0)
    other = _random(small_cfg(L=2, d=256, H=2, KV=1, V=320), dev, 11)
    g = torch.Generator().manual_seed(2)
    ids = torch.randint(3, 320, (4, 50), generator=g).to(dev)
    mask = torch.ones_like(ids)
    mask[0, :20] = 0
    mask[2, :45] = 0
    ids = ids * mask
    plain = model.generate(ids, attention_mask=mask, max_new_tokens=40, eos_token_id=321, pad_token_id=0, **_REF_KW)
    eos = int(plain[1, 50 + 9])                                  # an eos some rows reach inside a round
    plain = model.generate(ids, attention_mask=mask, max_new_tokens=40, eos_token_id=eos, pad_token_id=0, **_REF_KW)
    for draft in (model, other):
        for k in (1, 2, 3):
            got = model.generate(ids, attention_mask=mask, max_new_tokens=40, eos_token_id=eos, pad_token_id=0,
                                 assistant_model=draft, num_assistant_tokens=k, **_REF_KW)
            assert torch.equal(got, plain), (k, draft is model)


@pytest.mark.parametrize("new", [24, 57])
def test_generate_with_a_draft_on_the_benchmark_geometry(monkeypatch, new):
    """Llama-3.2-3B-ASR text config of bench.py (H/KV = 3: k = 4 fills the m16 tile), 4 layers, B = 12 left-padded
    audio-length prompts (T = 711), eos unreachable; drafts: the model itself and an unrelated 2-layer model.  Graph
    replay equals eager rounds, and runs are reproducible.  At 57 new tokens generate's cache of T + 57 = 768 rows is
    split in chunks of 128 keys while the speculative cache of 768 + k rows would give chunks of 192: the verify step
    must attend with generate's split layout to sum in generate's order."""
    dev = require_cuda()
    cfg = bench.asr_config(4)
    torch.manual_seed(0)
    with torch.device(dev):
        model = modeling.B200TouchAudioForCausalLM(cfg).to(BF16)
        dcfg = bench.asr_config(2)
        draft = modeling.B200TouchAudioForCausalLM(dcfg).to(BF16)
    with torch.no_grad():
        for m in (model, draft):
            for p in m.parameters():
                p.normal_(0, 0.02) if p.dim() == 2 else p.fill_(1.0)
    V = cfg.text_config.vocab_size
    ids, feats, mask, _ = time_decode.prompts(12, 2025, V, dev)
    assert ids.shape == (12, 711)
    kw = dict(eos_token_id=V, pad_token_id=0, bos_token_id=1, max_new_tokens=new, **_REF_KW)
    plain = model.generate(ids, feats, mask, **kw)
    for d in (model, draft):
        got = model.generate(ids, feats, mask, assistant_model=d, **kw)       # default k = 4
        assert torch.equal(got, plain)
        again = model.generate(ids, feats, mask, assistant_model=d, **kw)
        assert torch.equal(again, got)
    orig = generation._captured
    monkeypatch.setattr(generation, "_captured", lambda step, capture: orig(step, False))
    eager = model.generate(ids, feats, mask, assistant_model=draft, **kw)
    assert torch.equal(eager, plain)


def test_touch_audio_with_a_touch_audio_draft_and_nan_features():
    dev = require_cuda()
    torch.manual_seed(0)

    def audio_model(L, seed):
        text = small_cfg(L=L, d=256, H=2, KV=1, V=320)
        m = modeling.B200TouchAudioForCausalLM(NS(audio_config=NS(input_size=400), text_config=text, pad_token_id=0))
        m = m.to(dev)
        torch.manual_seed(seed)
        with torch.no_grad():
            for p in m.parameters():
                if p.dim() == 2:
                    p.normal_(0, 0.05)
        return m.to(BF16)

    model, draft = audio_model(2, 1), audio_model(1, 2)
    B, T = 3, 60
    rows = [40, 25, 59]
    ids = torch.zeros(B, T, dtype=torch.int64, device=dev)
    feats = torch.zeros(B, T, 400, device=dev)
    mask = torch.zeros(B, T, dtype=torch.int64, device=dev)
    for b, r in enumerate(rows):                               # the reference inference layout: features, then <bos>
        feats[b, T - 1 - r:T - 1] = torch.randn(r, 400, device=dev)
        ids[b, T - 1] = 1
        mask[b, T - 1 - r:] = 1
    kw = dict(eos_token_id=2, pad_token_id=0, bos_token_id=1, **_REF_KW)
    plain = model.generate(ids, feats, mask, max_new_tokens=16, **kw)
    for k in (1, 4):
        got = model.generate(ids, feats, mask, max_new_tokens=16, assistant_model=draft, num_assistant_tokens=k, **kw)
        assert torch.equal(got, plain)
    bad = feats.clone()
    bad[1, T - 5, 3] = float("nan")
    with pytest.raises(ValueError, match="NaN in data."):
        model.generate(ids, bad, mask, max_new_tokens=4, assistant_model=draft, **kw)
    # the flags are cleared: the next call runs
    assert torch.equal(model.generate(ids, feats, mask, max_new_tokens=16, assistant_model=draft, **kw), plain)
