"""CPU: greedy `generate` with a KV cache (touchnet_b200/generation.py) - argument checks of the three decoding entry
points, kwargs validation, and the decoding loop itself against transformers' LlamaForCausalLM.generate.

The loop runs on CPU through plain-torch stand-ins: tests/cpu_ops_shim.py for the training ops and, defined below, for
the three decoding ops (the selection stand-in IS HF's pair of logits processors + argmax, so what this checks is the
loop: prefill / decode wiring, left padding, positions, eos, pad after eos, the output layout).  The kernels themselves
are checked against the same references on the GPU (tests/test_gpu_decode.py)."""
import ctypes

import pytest
import torch

from touchnet_b200 import _lib, generation, modeling, ops

BF16 = torch.bfloat16


# ---------------------------------------------------------------------------------------------------------------
# entry points: argument validation happens before any CUDA call
# ---------------------------------------------------------------------------------------------------------------
def test_decode_entry_points_reject_bad_arguments():
    p = ctypes.c_void_p(256)
    bad_calls = [
        ("tn_attn_decode_bf16", (None, 1024, p, p, 128, 128 * 64, p, p, 2, 8, 1, 64, 0.1, p, p, 1024, None, None), "null"),
        ("tn_attn_decode_bf16", (p, 1024, p, p, 128, 128 * 64, p, p, 2, 8, 3, 64, 0.1, p, p, 1024, None, None), "bad dims"),
        ("tn_attn_decode_bf16", (p, 4096, p, p, 128, 128 * 64, p, p, 2, 32, 1, 64, 0.1, p, p, 4096, None, None), "1..16"),
        ("tn_attn_decode_bf16", (p, 1024, p, p, 128, 128 * 63, p, p, 2, 8, 1, 64, 0.1, p, p, 1024, None, None), "stride"),
        ("tn_attn_decode_bf16", (p, 1020, p, p, 128, 128 * 64, p, p, 2, 8, 1, 64, 0.1, p, p, 1024, None, None),
         "multiples of 8"),
        ("tn_kv_append_bf16", (p, 128, None, 128, p, p, 128, 128 * 8, p, 2, 1, 8, 128, None), "null"),
        ("tn_kv_append_bf16", (p, 128, p, 128, p, p, 128, 128 * 8, p, 2, 9, 8, 128, None), "bad dims"),
        ("tn_kv_append_bf16", (p, 64, p, 128, p, p, 128, 128 * 8, p, 2, 1, 8, 128, None), "strides"),
        ("tn_kv_append_bf16", (ctypes.c_void_p(258), 128, p, 128, p, p, 128, 128 * 8, p, 2, 1, 8, 128, None), "aligned"),
        ("tn_greedy_select_bf16", (p, 64, 2, 64, None, 16, p, p, p, p, 1.5, 2, 1, 0, None), "null"),
        ("tn_greedy_select_bf16", (p, 32, 2, 64, p, 16, p, p, p, p, 1.5, 2, 1, 0, None), "bad dims"),
        ("tn_greedy_select_bf16", (p, 64, 2, 64, p, 16, p, p, p, p, 0.0, 2, 1, 0, None), "repetition_penalty"),
        ("tn_greedy_select_bf16", (p, 64, 2, 64, p, 16, p, p, p, p, 1.0, -1, 1, 0, None), "no_repeat_ngram_size"),
        ("tn_greedy_select_bf16", (p, 1 << 23, 2, 1 << 23, p, 16, p, p, p, p, 1.0, 0, 1, 0, None), "too large"),
    ]
    for name, args, needle in bad_calls:
        with pytest.raises(_lib.TouchNetB200Error, match=needle):
            _lib.call(name, *args)
    lib = _lib.load()
    assert lib.tn_attn_decode_ws_floats(0, 8, 1, 64) == 0
    # the split count depends on the shapes only; workspace = B*H*splits*(128 + 2) floats
    ws = lib.tn_attn_decode_ws_floats(12, 24, 8, 1007)
    assert ws > 0 and ws % (12 * 24 * 130) == 0


# ---------------------------------------------------------------------------------------------------------------
# a tiny model and HF's twin with the same weights
# ---------------------------------------------------------------------------------------------------------------
class _Cfg:
    def __init__(self, **kw):
        self.__dict__.update(kw)


_DIMS = dict(hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=2, num_key_value_heads=1,
             head_dim=128, vocab_size=64, rms_norm_eps=1e-5, rope_theta=10000.0, tie_word_embeddings=False)


def _models(seed=0):
    from transformers import LlamaConfig, LlamaForCausalLM
    torch.manual_seed(seed)
    hf = LlamaForCausalLM(LlamaConfig(**_DIMS, pad_token_id=0, bos_token_id=1, eos_token_id=2,
                                      attn_implementation="eager")).float().eval()
    with torch.no_grad():
        for name, prm in hf.named_parameters():
            if prm.dim() == 2:
                prm.normal_(0, 0.08)
        hf.lm_head.weight.mul_(8.0)        # well separated logits: bf16 stand-ins and fp32 HF pick the same tokens
        hf.model.embed_tokens.weight[0].zero_()
    ours = modeling.B200LlamaForCausalLM(_Cfg(**_DIMS, pad_token_id=0, attention_bias=False, initializer_range=0.02,
                                              model_type="llama", rope_scaling=None))
    ours.load_state_dict(hf.state_dict())
    ours.model.rotary_emb.inv_freq = hf.model.rotary_emb.inv_freq.clone()
    return hf, ours


def _attn_decode(q, kc, vc, kv_start, kv_end, H, KV, scale, workspace=None, lse=False):
    B = q.shape[0]
    G = H // KV
    o = torch.zeros(B, H * 128)
    for b in range(B):
        lo, hi = int(kv_start[b]), int(kv_end[b])
        k = kc[b, lo:hi].float().view(hi - lo, KV, 128).repeat_interleave(G, 1)     # [S, H, 128]
        v = vc[b, lo:hi].float().view(hi - lo, KV, 128).repeat_interleave(G, 1)
        qb = q[b].float().view(H, 128)
        p = torch.softmax(torch.einsum("hd,shd->hs", qb, k) * scale, -1)
        o[b] = torch.einsum("hs,shd->hd", p, v).reshape(-1)
    return o.to(BF16)


def _kv_append(k, v, kc, vc, row_end, T_new):
    for b in range(kc.shape[0]):
        e = int(row_end[b])
        kc[b, e - T_new:e] = k[b * T_new:(b + 1) * T_new]
        vc[b, e - T_new:e] = v[b * T_new:(b + 1) * T_new]


def _greedy_select(logits, history, length, positions, next_ids, finished, penalty, ngram, eos, pad):
    from transformers.generation.logits_process import NoRepeatNGramLogitsProcessor, RepetitionPenaltyLogitsProcessor
    n = int(length[0])
    assert bool((length == n).all())
    seq = history[:, :n]
    scores = logits.float()
    if penalty != 1.0:
        scores = RepetitionPenaltyLogitsProcessor(penalty)(seq, scores)
    if ngram > 0:
        scores = NoRepeatNGramLogitsProcessor(ngram)(seq, scores)
    tok = torch.argmax(scores, -1)
    tok = torch.where(finished.bool(), torch.full_like(tok, pad), tok)
    history[:, n] = tok
    next_ids.copy_(tok)
    length += 1
    positions += 1
    finished |= (tok == eos).to(finished.dtype)


@pytest.fixture
def stand_ins(monkeypatch):
    from tests import cpu_ops_shim
    saved = cpu_ops_shim.install()
    monkeypatch.setattr(ops, "attn_decode", _attn_decode)
    monkeypatch.setattr(ops, "kv_append", _kv_append)
    monkeypatch.setattr(ops, "greedy_select", _greedy_select)
    yield
    cpu_ops_shim.uninstall(saved)


def _prompt():
    ids = torch.tensor([[0, 0, 0, 0, 5, 9, 11, 7, 1],
                        [12, 30, 4, 8, 17, 22, 9, 13, 1],
                        [0, 0, 0, 0, 0, 0, 41, 6, 1]], dtype=torch.int64)
    return ids, (ids != 0).to(torch.int64)


_REF_KW = dict(use_cache=True, do_sample=False, num_beams=1, repetition_penalty=1.5, no_repeat_ngram_size=2,
               bos_token_id=1, pad_token_id=0)


# The stand-ins round to bf16 like the kernels while HF runs in fp32, so a near-tie among the 30 picks of a random tiny
# model can legitimately flip one token; seed 4 is a model without such a tie (HF's top-2 margin >= 0.19 at every step).
def test_generate_loop_matches_hf_generate(stand_ins):
    hf, ours = _models(seed=4)
    ids, mask = _prompt()
    T = ids.shape[1]
    with torch.no_grad():
        probe = hf.generate(input_ids=ids, attention_mask=mask, max_new_tokens=10, eos_token_id=63, **_REF_KW)
    # an eos that row 0 reaches early and the other rows do not reach before it: exercises pad after eos
    eos = int(probe[0, T + 2])
    with torch.no_grad():
        ref = hf.generate(input_ids=ids, attention_mask=mask, max_new_tokens=10, eos_token_id=eos, **_REF_KW)
    got = ours.generate(ids, attention_mask=mask, max_new_tokens=10, eos_token_id=eos, **_REF_KW)
    assert got.shape == ref.shape and torch.equal(got, ref), (got, ref)
    assert (got[0, T + 3:] == 0).all()                      # pad after eos
    assert torch.equal(got[:, :T], ids)
    # every row finishing stops early: HF returns fewer than max_new_tokens columns, and so do we
    if bool((ref[:, T:] == eos).any(1).all()):
        assert got.shape[1] < T + 10


def test_generate_stops_when_every_row_has_finished(stand_ins):
    hf, ours = _models(seed=4)
    ids, mask = _prompt()
    T = ids.shape[1]
    with torch.no_grad():
        probe = hf.generate(input_ids=ids, attention_mask=mask, max_new_tokens=6, eos_token_id=63, **_REF_KW)
    eos = int(probe[0, T])                  # row 0 finishes on its first token
    ids1, mask1 = ids[:1], mask[:1]
    with torch.no_grad():
        ref = hf.generate(input_ids=ids1, attention_mask=mask1, max_new_tokens=6, eos_token_id=eos, **_REF_KW)
    got = ours.generate(ids1, attention_mask=mask1, max_new_tokens=6, eos_token_id=eos, **_REF_KW)
    assert torch.equal(got, ref) and got.shape[1] == T + 1


def test_cached_forward_matches_full_forward_under_teacher_forcing(stand_ins):
    """forward(past_key_values=B200KVCache) - prefill, then one token per call - gives the logits of the uncached
    forward on the extended sequence (multi-document prompt: the new tokens belong to each row's last document)."""
    _, ours = _models(seed=2)
    doc = torch.tensor([[1, 1, 1, 2, 2, 2, 2, 2], [0, 0, 1, 1, 2, 3, 3, 3]], dtype=torch.int64)
    pos = torch.tensor([[0, 1, 2, 0, 1, 2, 3, 4], [0, 0, 0, 1, 0, 0, 1, 2]], dtype=torch.int64)
    ids = torch.randint(3, 64, doc.shape, generator=torch.Generator().manual_seed(3))
    extra = torch.randint(3, 64, (2, 4), generator=torch.Generator().manual_seed(4))
    cache = generation.B200KVCache(ours, 2, 8 + 4)
    steps = [ours(input_ids=ids, attention_mask=doc, position_ids=pos, past_key_values=cache, use_cache=True).logits]
    for j in range(4):
        steps.append(ours(input_ids=extra[:, j:j + 1], past_key_values=cache, use_cache=True).logits)
    for j in range(5):
        n = 8 + j
        full_ids = torch.cat([ids, extra[:, :j]], 1)
        full_doc = torch.cat([doc, doc[:, -1:].expand(2, j)], 1)
        full_pos = torch.cat([pos, pos[:, -1:] + torch.arange(1, j + 1)[None]], 1)
        with torch.no_grad():
            ref = ours(input_ids=full_ids, attention_mask=full_doc, position_ids=full_pos).logits
        assert full_ids.shape[1] == n
        assert steps[j].shape == (2, 1, 64)
        err = (steps[j][:, 0].float() - ref[:, -1].float()).abs().max()
        assert float(err) <= 2e-2 * float(ref[:, -1].float().abs().max()), (j, float(err))


def test_last_document_start_and_padded_last_column():
    m = torch.tensor([[0, 0, 1, 1], [1, 1, 2, 2], [1, 2, 3, 3], [1, 1, 1, 1]])
    assert generation._last_doc_start(m).tolist() == [2, 2, 2, 0]
    _, ours = _models()
    with pytest.raises(_lib.TouchNetB200Error, match="padding"):
        ours.generate(torch.ones(1, 4, dtype=torch.int64), attention_mask=torch.tensor([[1, 1, 1, 0]]),
                      max_new_tokens=2, eos_token_id=2, pad_token_id=0)


@pytest.mark.parametrize("kw, needle", [
    (dict(do_sample=True), "greedy"),
    (dict(num_beams=4), "greedy"),
    (dict(eos_token_id=[2, 3]), "single id"),
    (dict(max_new_tokens=0), "max_new_tokens"),
    (dict(repetition_penalty=0.0), "repetition_penalty"),
    (dict(no_repeat_ngram_size=-1), "no_repeat_ngram_size"),
    (dict(output_scores=True), "unsupported"),
    (dict(input_features=torch.zeros(1, 4, 8)), "unsupported"),      # plain Llama has no audio input
])
def test_generate_kwargs_are_validated(kw, needle):
    _, ours = _models()
    args = dict(max_new_tokens=4, eos_token_id=2, pad_token_id=0)
    args.update(kw)
    with pytest.raises(_lib.TouchNetB200Error, match=needle):
        ours.generate(torch.ones(1, 4, dtype=torch.int64), **args)


def test_generate_ignores_sampling_knobs_of_greedy_search(stand_ins):
    """top_k / top_p / temperature / early_stopping / bos_token_id are accepted and change nothing, as in HF."""
    _, ours = _models()
    ids, mask = _prompt()
    a = ours.generate(ids, attention_mask=mask, max_new_tokens=3, eos_token_id=63, pad_token_id=0)
    b = ours.generate(ids, attention_mask=mask, max_new_tokens=3, eos_token_id=63, pad_token_id=0, top_k=5, top_p=0.5,
                      temperature=0.3, early_stopping=True, bos_token_id=1)
    assert torch.equal(a, b)
