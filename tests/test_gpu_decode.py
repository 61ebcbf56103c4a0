"""GPU: KV-cache decoding (touchnet_b200/csrc/decode.cu, touchnet_b200/generation.py).

  decode attention  vs an fp32 softmax in torch (relative L2 < 2e-2 on O, < 2e-3 on lse; the attention tolerances of
                    tests/test_gpu_attention.py), O = 0 / lse = +inf on an empty range, bitwise equal across runs
  cache append      rows bit-identical to their sources
  selection         vs HF RepetitionPenaltyLogitsProcessor + NoRepeatNGramLogitsProcessor + torch.argmax, exact
  cached forward    vs the uncached forward and the fp32 oracle under teacher forcing (logits within 3e-2 * max|ref|,
                    argmax equal where the reference's top-2 margin exceeds twice the error); layer-0 cache rows
                    bit-identical to the K/V of the uncached forward
  graph replay      bit-identical to the eager decode step
  generate          TouchAudio on the reference's inference layout vs the oracle; Llama vs HF generate (bf16, sdpa)"""
import math

import pytest
import torch

from oracle import model_oracle as mo
from tests.gpu_util import rel_err, require_cuda
from tests.test_gpu_model import LLAMA3, oracle_cfg, small_cfg
from touchnet_b200 import generation, modeling, ops

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16


def _ref_decode(q, kc, vc, start, end, H, KV, scale):
    B = q.shape[0]
    G = H // KV
    o = torch.zeros(B, H, 128, device=q.device)
    lse = torch.full((B, H), float("inf"), device=q.device)
    for b in range(B):
        lo, hi = int(start[b]), int(end[b])
        if hi <= lo:
            continue
        k = kc[b, lo:hi].float().view(hi - lo, KV, 128).repeat_interleave(G, 1)
        v = vc[b, lo:hi].float().view(hi - lo, KV, 128).repeat_interleave(G, 1)
        s = torch.einsum("hd,shd->hs", q[b].float().view(H, 128), k) * scale
        lse[b] = torch.logsumexp(s, -1)
        o[b] = torch.einsum("hs,shd->hd", torch.softmax(s, -1), v)
    return o.view(B, H * 128), lse


@pytest.mark.parametrize("H, KV", [(8, 8), (24, 8), (32, 8)])
@pytest.mark.parametrize("S_cap", [1100, 32768])
def test_decode_attention_matches_fp32_softmax(H, KV, S_cap):
    dev = require_cuda()
    torch.manual_seed(H + S_cap)
    B = 5
    lens = [1, 63, 129, 1000, 0]                        # last row: an empty range
    start = torch.tensor([3, 0, S_cap - 129 - 7, S_cap - 1000, 10], dtype=torch.int32, device=dev)
    end = start + torch.tensor(lens, dtype=torch.int32, device=dev)
    cache = torch.randn(2, B, S_cap, KV * 128, device=dev).to(BF16)
    kc, vc = cache[0], cache[1]
    for b in range(B):                                  # rows outside the range must not leak into O, even as NaN
        lo, hi = int(start[b]), int(end[b])
        vc[b, max(lo - 3, 0):lo].fill_(float("nan"))
        vc[b, hi:hi + 3].fill_(float("nan"))
    q = torch.randn(B, H * 128, device=dev).to(BF16)
    scale = 1 / math.sqrt(128)
    o, lse = ops.attn_decode(q, kc, vc, start, end, H, KV, scale, lse=True)
    ro, rlse = _ref_decode(q, kc.nan_to_num(0.0), vc.nan_to_num(0.0), start, end, H, KV, scale)
    for b in range(B - 1):
        assert rel_err(o[b].float(), ro[b]) < 2e-2, (b, rel_err(o[b].float(), ro[b]))
        assert rel_err(lse[b], rlse[b]) < 2e-3
    assert torch.all(o[B - 1] == 0) and torch.all(torch.isinf(lse[B - 1]) & (lse[B - 1] > 0))
    o2, lse2 = ops.attn_decode(q, kc, vc, start, end, H, KV, scale, lse=True)
    assert torch.equal(o, o2) and torch.equal(lse, lse2)


def test_kv_append_is_a_bit_exact_copy():
    dev = require_cuda()
    B, S_cap, KV, T_new = 3, 40, 2, 7
    cache = torch.zeros(2, B, S_cap, KV * 128, dtype=BF16, device=dev)
    qkv = torch.randn(B * T_new, 3 * KV * 128, device=dev).to(BF16)        # strided k / v columns of a fused output
    k, v = qkv[:, KV * 128:2 * KV * 128], qkv[:, 2 * KV * 128:]
    end = torch.tensor([7, 20, 40], dtype=torch.int32, device=dev)
    ops.kv_append(k, v, cache[0], cache[1], end, T_new)
    for b in range(B):
        e = int(end[b])
        assert torch.equal(cache[0, b, e - T_new:e], k[b * T_new:(b + 1) * T_new])
        assert torch.equal(cache[1, b, e - T_new:e], v[b * T_new:(b + 1) * T_new])
        assert torch.all(cache[:, b, :e - T_new] == 0) and torch.all(cache[:, b, e:] == 0)


@pytest.mark.parametrize("V", [320, 128256])
def test_greedy_select_matches_hf_processors(V):
    from transformers.generation.logits_process import NoRepeatNGramLogitsProcessor, RepetitionPenaltyLogitsProcessor
    dev = require_cuda()
    g = torch.Generator(device="cpu").manual_seed(V)
    B, S_cap, n = 6, 64, 37
    hist = torch.randint(0, 50, (B, S_cap), generator=g).to(dev)           # small id range: many repeats and bans
    hist[:, n - 2:n] = hist[:, 10:12]                                       # the last bigram occurred before
    logits = (torch.randn(B, V, generator=g) * 3).to(BF16).to(dev)
    logits[0, 7] = logits[0, 9] = logits[0].float().max() + 1             # planted ties: the lower index wins
    logits[1, :] = -1.0                                                     # all equal (negative, penalised)
    logits[2, 5] = float("inf")
    for penalty, ngram in ((1.5, 2), (1.0, 0), (1.3, 3)):
        h = hist.clone()
        length = torch.full((B,), n, dtype=torch.int32, device=dev)
        pos = torch.arange(B, dtype=torch.int64, device=dev)
        nxt = torch.zeros(B, dtype=torch.int64, device=dev)
        fin = torch.tensor([0, 0, 0, 1, 0, 0], dtype=torch.int32, device=dev)
        eos, pad = int(hist[4, 11]), 0
        ops.greedy_select(logits, h, length, pos, nxt, fin, penalty, ngram, eos, pad)
        scores = logits.float()
        if penalty != 1.0:
            scores = RepetitionPenaltyLogitsProcessor(penalty)(hist[:, :n], scores)
        if ngram:
            scores = NoRepeatNGramLogitsProcessor(ngram)(hist[:, :n], scores)
        ref = torch.argmax(scores, -1)
        ref[3] = pad
        assert torch.equal(nxt, ref), (nxt, ref, penalty, ngram)
        assert torch.equal(h[:, n], ref) and torch.equal(h[:, :n], hist[:, :n])
        assert torch.equal(h[:, n + 1:], hist[:, n + 1:])
        assert torch.all(length == n + 1) and torch.equal(pos, torch.arange(B, device=dev) + 1)
        assert fin.tolist() == [int(ref[b] == eos) or int(b == 3) for b in range(B)]


def _model(hd, bias, dev, seed=0, dtype=torch.float32, rope_scaling=LLAMA3):
    H, KV = (3, 1) if hd == 128 else (6, 2)
    c = small_cfg(d=384, H=H, KV=KV, V=320, rope_scaling=rope_scaling, bias=bias)
    c.head_dim = hd
    if bias:
        c.model_type = "qwen2"
    torch.manual_seed(seed)
    m = modeling.B200LlamaForCausalLM(c).to(dev)
    m.post_init()
    with torch.no_grad():
        for p in m.parameters():
            p.copy_(torch.randn_like(p) * 0.05 if p.dim() == 2 else 1 + 0.1 * torch.randn_like(p))
    return m.to(dtype), c


def _prompts(kind, dev):
    if kind == "left_padded":
        doc = torch.tensor([[0] * 60 + [1] * 140, [1] * 200, [0] * 173 + [1] * 27], device=dev)
        pos = ((doc.cumsum(-1) - 1).clamp(min=0)).to(torch.int64)
    else:   # packed: the new tokens continue each row's last document
        rows = [[90, 110], [20, 50, 30, 100], [199, 1]]
        doc = torch.tensor([sum(([0 if (r == 1 and i == 0) else i + 1 - (r == 1)] * n for i, n in enumerate(lens)), [])
                            for r, lens in enumerate(rows)], device=dev)
        pos = torch.tensor([sum((list(range(n)) for n in lens), []) for lens in rows], device=dev)
    ids = torch.randint(3, 320, doc.shape, device=dev) * (doc > 0)
    return ids, doc, pos


@pytest.mark.parametrize("hd, bias", [(128, False), (128, True), (64, False)])
@pytest.mark.parametrize("kind", ["left_padded", "packed"])
def test_cached_decoding_matches_uncached_forward_and_oracle(hd, bias, kind):
    dev = require_cuda()
    model, c = _model(hd, bias, dev)
    ids, doc, pos = _prompts(kind, dev)
    B, T = ids.shape
    steps = 16
    extra = torch.randint(3, 320, (B, steps), device=dev)
    # the K/V the uncached forward hands to layer 0's attention
    seen = []
    real = ops.attn_fwd

    def spy(q, k, v, plan, H, KV, scale):
        seen.append((k.clone(), v.clone()))
        return real(q, k, v, plan, H, KV, scale)

    ops.attn_fwd = spy
    try:
        with torch.no_grad():
            model(input_ids=ids, attention_mask=doc, position_ids=pos)
    finally:
        ops.attn_fwd = real
    cache = generation.B200KVCache(model, B, T + steps)
    logits = [model(input_ids=ids, attention_mask=doc, position_ids=pos, past_key_values=cache, use_cache=True).logits]
    k0, v0 = seen[0]
    assert torch.equal(cache.data[0, 0, :, :T].reshape(B * T, -1), k0)
    assert torch.equal(cache.data[0, 1, :, :T].reshape(B * T, -1), v0)
    for j in range(steps - 1):
        logits.append(model(input_ids=extra[:, j:j + 1], past_key_values=cache, use_cache=True).logits)
    params = {k: v.detach().bfloat16().float() for k, v in model.state_dict().items()}
    ocfg = oracle_cfg(c)
    ocfg.head_dim = hd
    for j in range(steps):
        full_ids = torch.cat([ids, extra[:, :j]], 1)
        full_doc = torch.cat([doc, doc[:, -1:].expand(B, j)], 1)
        full_pos = torch.cat([pos, pos[:, -1:] + torch.arange(1, j + 1, device=dev)[None]], 1)
        got = logits[j][:, 0].float()
        with torch.no_grad():
            ref = model(input_ids=full_ids, attention_mask=full_doc, position_ids=full_pos).logits[:, -1].float()
            orc = mo.llama_forward(params, ocfg, input_ids=full_ids, attention_mask=full_doc, position_ids=full_pos)[:, -1]
        for r in (ref, orc):
            err = float((got - r).abs().max())
            assert err <= 3e-2 * float(r.abs().max()) + 1e-3, (j, err)
            top2 = r.topk(2, -1).values
            decisive = (top2[:, 0] - top2[:, 1]) > 2 * err
            assert torch.equal(got.argmax(-1)[decisive], r.argmax(-1)[decisive])


def test_graph_replay_is_bit_identical_to_the_eager_step():
    dev = require_cuda()
    model, _ = _model(128, True, dev, dtype=BF16)
    ids, doc, pos = _prompts("packed", dev)
    B, T = ids.shape
    cache = generation.B200KVCache(model, B, T + 8)
    w = generation._Weights(model)

    def step():
        logits = generation.decode_step(model, cache, weights=w)
        ops.greedy_select(logits, cache.history, cache.kv_end, cache.positions, cache.next_ids, cache.finished, 1.5, 2,
                          10 ** 6, 0)
        return logits

    with torch.no_grad():
        first = generation.prefill(model, cache, ids, None, doc, pos, weights=w)
        ops.greedy_select(first, cache.history, cache.kv_end, cache.positions, cache.next_ids, cache.finished, 1.5, 2,
                          10 ** 6, 0)
        step()                                                       # the eager step generate runs before capturing
        state = [t.clone() for t in (cache.data, cache.kv_end, cache.positions, cache.history, cache.next_ids,
                                     cache.finished)]
        eager = [step().clone()]
        eager_state = [t.clone() for t in (cache.data, cache.history, cache.next_ids)]
        eager.append(step().clone())
        for t, s in zip((cache.data, cache.kv_end, cache.positions, cache.history, cache.next_ids, cache.finished), state):
            t.copy_(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            out = step()
        g.replay()
        assert torch.equal(out, eager[0])
        for t, s in zip((cache.data, cache.history, cache.next_ids), eager_state):
            assert torch.equal(t, s)
        g.replay()
        assert torch.equal(out, eager[1])


_REF_KW = dict(use_cache=True, do_sample=False, num_beams=1, repetition_penalty=1.5, no_repeat_ngram_size=2)


def _processed_argmax(scores_row_hist, logits, penalty=1.5, ngram=2):
    from transformers.generation.logits_process import NoRepeatNGramLogitsProcessor, RepetitionPenaltyLogitsProcessor
    s = RepetitionPenaltyLogitsProcessor(penalty)(scores_row_hist, logits.float().clone())
    return NoRepeatNGramLogitsProcessor(ngram)(scores_row_hist, s)


def test_touch_audio_generate_on_the_reference_inference_layout():
    """GPU fbank -> stack -> projector rows, one zero feature row under `<bos>`, left-padded (ref:
    inference_touch_audio.py:51-100), generated with the reference's kwargs; the oracle, teacher-forced on our output,
    must pick each of our tokens or have it within twice the logit error of its pick; finished rows are padded."""
    from types import SimpleNamespace as NS
    from touchnet_b200 import frontend
    dev = require_cuda()
    torch.manual_seed(0)
    text = small_cfg(d=256, H=2, KV=1, V=320)
    cfg = NS(audio_config=NS(input_size=400), text_config=text, pad_token_id=0)
    model = modeling.B200TouchAudioForCausalLM(cfg).to(dev)
    model.post_init()
    with torch.no_grad():
        for p in model.parameters():
            if p.dim() == 2:
                p.normal_(0, 0.05)
    model.to(BF16)
    g = torch.Generator().manual_seed(1)
    wavs = [0.3 * (2 * torch.rand(n, generator=g) - 1) for n in (16000 * 2, 16000 + 4000, 16000 * 3)]
    flat, lens = frontend._pack(wavs, dev)
    fb, frames = frontend.fbank_batch(flat, lens)
    rows = [int(math.ceil(f / 4)) for f in frames]
    feats_packed = torch.zeros(sum(rows), 400, device=dev)
    frontend.stack_batch(fb, frames, 5, 4, True, into=feats_packed, dst_rows=[sum(rows[:i]) for i in range(len(rows))])
    B, T = len(wavs), max(rows) + 1
    bos, eos, pad = 1, 2, 0
    ids = torch.full((B, T), pad, dtype=torch.int64, device=dev)
    feats = torch.zeros(B, T, 400, device=dev)
    mask = torch.zeros(B, T, dtype=torch.int64, device=dev)
    for b, r in enumerate(rows):
        o = sum(rows[:b])
        feats[b, T - 1 - r:T - 1] = feats_packed[o:o + r]
        ids[b, T - 1] = bos
        mask[b, T - 1 - r:] = 1
    new = 12
    out = model.generate(ids, feats, mask, max_new_tokens=new, eos_token_id=eos, pad_token_id=pad, bos_token_id=bos,
                         **_REF_KW)
    n = out.shape[1] - T
    assert 1 <= n <= new and torch.equal(out[:, :T], ids)
    params = {k: v.detach().float() for k, v in model.state_dict().items()}
    ocfg = oracle_cfg(text, audio=400)
    cache = generation.B200KVCache(model, B, T + n)
    ours = [model(input_ids=ids, input_features=feats, attention_mask=mask, past_key_values=cache).logits[:, 0]]
    for j in range(n - 1):
        ours.append(model(input_ids=out[:, T + j:T + j + 1], past_key_values=cache).logits[:, 0])
    for j in range(n):
        seq = out[:, :T + j]
        m = torch.cat([mask, torch.ones(B, j, dtype=mask.dtype, device=dev)], 1)
        p = (m.cumsum(-1) - 1).clamp(min=0)
        f = torch.cat([feats, torch.zeros(B, j, 400, device=dev)], 1).bfloat16().float()
        with torch.no_grad():
            ref = mo.touch_audio_forward(params, ocfg, input_ids=seq, input_features=f, attention_mask=m,
                                         position_ids=p)[:, -1]
        err = float((ours[j].float() - ref).abs().max())
        assert err <= 3e-2 * float(ref.abs().max()) + 1e-3
        s = _processed_argmax(seq, ref)
        for b in range(B):
            if j > 0 and (out[b, T:T + j] == eos).any():
                assert int(out[b, T + j]) == pad
                continue
            tok = int(out[b, T + j])
            assert tok == int(s[b].argmax()) or float(s[b].max() - s[b, tok]) <= 2 * err, (b, j)


def test_llama_generate_matches_hf_generate_up_to_near_ties():
    """Stock HF LlamaForCausalLM.generate (bf16, sdpa) on the same weights: identical tokens up to the first divergence,
    and at a divergence HF's top-2 margin is below twice the measured logit error."""
    from transformers import LlamaConfig, LlamaForCausalLM
    dev = require_cuda()
    model, c = _model(128, False, dev, dtype=BF16, rope_scaling=None)
    hf = LlamaForCausalLM(LlamaConfig(hidden_size=384, intermediate_size=512, num_hidden_layers=2, num_attention_heads=3,
                                      num_key_value_heads=1, head_dim=128, vocab_size=320, rms_norm_eps=1e-5,
                                      rope_theta=500000.0, tie_word_embeddings=False,
                                      pad_token_id=0, attn_implementation="sdpa")).to(dev, BF16).eval()
    hf.load_state_dict(model.state_dict())
    ids, doc, _ = _prompts("left_padded", dev)
    mask = doc
    kw = dict(max_new_tokens=24, eos_token_id=2, pad_token_id=0, bos_token_id=1, **_REF_KW)
    with torch.no_grad():
        ref = hf.generate(input_ids=ids, attention_mask=mask, output_scores=True, return_dict_in_generate=True, **kw)
    got = model.generate(ids, attention_mask=mask, **kw)
    T = ids.shape[1]
    seq = ref.sequences
    for b in range(ids.shape[0]):
        diff = (got[b, T:T + seq.shape[1] - T] != seq[b, T:got.shape[1]]).nonzero()
        if diff.numel() == 0:
            continue
        j = int(diff[0])
        prefix = seq[b:b + 1, :T + j]
        m = torch.cat([mask[b:b + 1], torch.ones(1, j, dtype=mask.dtype, device=dev)], 1)
        p = (m.cumsum(-1) - 1).masked_fill(m == 0, 0)
        with torch.no_grad():
            a = model(input_ids=prefix, attention_mask=m, position_ids=p).logits[0, -1].float()
            h = hf(input_ids=prefix, attention_mask=m, position_ids=p).logits[0, -1].float()
        err = float((a - h).abs().max())
        top2 = ref.scores[j][b].float().topk(2).values
        assert float(top2[0] - top2[1]) <= 2 * err, (b, j, float(top2[0] - top2[1]), err)
