"""Greedy autoregressive decoding with a KV cache for the drop-in models (`model.generate`).

The reference evaluates its ASR models with HF `generate(use_cache=True, do_sample=False, num_beams=1,
repetition_penalty, no_repeat_ngram_size, max_new_tokens, ...)` on left-padded prompts
(ref: touchnet/models/touch_audio/inference_touch_audio.py:51-100, :170-192).  This module reproduces that call:

  prefill  the prompt runs through the training block (ops.block_forward: fused QKV GEMM with the RoPE epilogue, packed
           document attention over the prompt's mask) and every layer's K/V is appended to the cache; lm_head runs on
           the last position only;
  decode   one token per row: the same block at M = B with the attention step replaced by cache append + split-KV decode
           attention (tn_attn_decode_bf16), then lm_head and the greedy selection kernel (tn_greedy_select_bf16:
           repetition penalty, no-repeat-ngram ban, argmax, pad after eos), all lengths and positions on the device;
  generate prefill, one eager decode step, then the decode step captured once in a CUDA graph and replayed per token,
           with one host sync per step to read the finished flags and the NaN flag;
  generate_many
           continuous batching over many prompts: a cache of B slots, finished rows refilled with the next prompts
           (packed prefill into chosen slots: tn_kv_scatter_bf16, tn_slot_admit) while the captured decode step keeps
           replaying (tn_greedy_select_slots_bf16 holds finished and idle slots still); do_sample=True draws the
           tokens instead (tn_sample_select_slots_bf16: temperature, top-k, top-p, a Philox stream per prompt).
  speculative
           generate(assistant_model=draft): per round the draft proposes k tokens, the model scores them in one step of
           B*(k+1) rows (tn_attn_decode_multi_bf16) and keeps the longest prefix equal to its own picks plus its next
           pick (tn_verify_select_bf16); the output is bit-identical to generate without the draft.

The new tokens belong to the last document of each row: the decode query of row b attends to cache rows
[kv_start[b], kv_end[b]) with kv_start[b] the first position of the row's last document in the prompt's attention_mask
(a 0/1 left-padding mask is the one-document case).  Positions continue from each row's last prompt position.
Scope: one GPU, unsharded model.
"""
from __future__ import annotations

import math
from typing import Optional

import torch

from . import _lib, ops
from ._lib import TouchNetB200Error

BF16 = torch.bfloat16


def _parts(model):
    """(B200LlamaForCausalLM, TouchAudio wrapper or None)."""
    lm = getattr(model, "language_model", None)
    return (lm, model) if lm is not None else (model, None)


class B200KVCache:
    """K/V of every layer in one allocation [L, 2, B, S_cap, KV*128] bf16 (heads zero-padded to 128 columns when
    head_dim < 128, as the training attention pads them) plus the device-side decoding state:
      kv_start / kv_end [B] int32  attended cache rows of the next decode query; kv_end is also the token count so far
      positions [B] int64          rope position of the last token in the history
      history [B, S_cap] int64     prompt ids followed by the generated ids (what the repetition processors see)
      next_ids [B] int64           the token the next decode step feeds in
      finished [B] int32           1 once the row has emitted eos
    Pass it as `past_key_values` to the models' forward for step-by-step (teacher-forced) decoding."""

    def __init__(self, model, batch_size: int, max_length: int, device=None):
        lm, _ = _parts(model)
        cfg = lm.config
        a = lm.model.layers[0].self_attn
        dev = torch.device(device) if device is not None else lm.lm_head.weight.device
        self.B, self.S_cap = int(batch_size), int(max_length)
        self.L, self.H, self.KV, self.hd = len(lm.model.layers), a.num_heads, a.num_key_value_heads, a.head_dim
        self.scale = 1.0 / math.sqrt(self.hd)       # softmax scale of the attention
        if self.B <= 0 or self.S_cap <= 0:
            raise TouchNetB200Error(f"B200KVCache: batch_size {batch_size} / max_length {max_length} must be positive")
        self.vocab = cfg.vocab_size
        self.data = torch.zeros((self.L, 2, self.B, self.S_cap, self.KV * 128), dtype=BF16, device=dev)
        self.kv_start = torch.zeros(self.B, dtype=torch.int32, device=dev)
        self.kv_end = torch.zeros(self.B, dtype=torch.int32, device=dev)
        self.positions = torch.zeros(self.B, dtype=torch.int64, device=dev)
        self.history = torch.zeros((self.B, self.S_cap), dtype=torch.int64, device=dev)
        self.next_ids = torch.zeros(self.B, dtype=torch.int64, device=dev)
        self.finished = torch.zeros(self.B, dtype=torch.int32, device=dev)
        self.workspace = torch.empty(int(_lib.load().tn_attn_decode_ws_floats(self.B, self.H, self.KV, self.S_cap)),
                                     dtype=torch.float32, device=dev)
        self.length = 0          # host mirror of kv_end (every row holds the same number of tokens)

    def layer(self, i: int):
        return self.data[i, 0], self.data[i, 1]

    def get_seq_length(self, layer_idx: int = 0) -> int:
        return self.length

    def push(self, ids: torch.Tensor) -> None:
        """Teacher forcing: make `ids` [B] the next token of every row (what tn_greedy_select_bf16 does with its pick)."""
        if self.length >= self.S_cap:
            raise TouchNetB200Error(f"B200KVCache is full ({self.S_cap} tokens)")
        ids = ids.reshape(self.B).to(device=self.history.device, dtype=torch.int64)
        self.history[:, self.length] = ids
        self.next_ids.copy_(ids)
        self.kv_end += 1
        self.positions += 1
        self.length += 1


class _Weights:
    """bf16 working weights resolved once per call (fp32 masters are cast before any graph capture; bf16 models use
    their parameters as they are), so the decode step does no parameter bookkeeping."""

    def __init__(self, lm):
        m = lm.model
        self.layers = []
        for layer in m.layers:
            a, p = layer.self_attn, layer.mlp
            self.layers.append((layer.input_layernorm.weight.detach(), ops.bf16_weight(a.q_proj.weight),
                                ops.bf16_weight(a.k_proj.weight), ops.bf16_weight(a.v_proj.weight),
                                None if a.q_proj.bias is None else a.q_proj.bias.detach(),
                                None if a.k_proj.bias is None else a.k_proj.bias.detach(),
                                None if a.v_proj.bias is None else a.v_proj.bias.detach(),
                                ops.bf16_weight(a.o_proj.weight), layer.post_attention_layernorm.weight.detach(),
                                ops.bf16_weight(p.gate_proj.weight), ops.bf16_weight(p.up_proj.weight),
                                ops.bf16_weight(p.down_proj.weight)))
        self.eps = m.layers[0].input_layernorm.variance_epsilon
        self.embed = m.embed_tokens.weight.detach()
        self.norm = m.norm.weight.detach()
        self.norm_eps = m.norm.variance_epsilon
        self.lm_head = ops.bf16_weight(lm.lm_head.weight)
        rot = m.rotary_emb
        inv = rot.inv_freq
        if inv.dtype != torch.float32:      # see B200RotaryEmbedding.forward
            inv, _ = rot.rope_init_fn(rot.config, device=inv.device)
        self.inv_freq = inv.detach().float().contiguous()
        self.rope_scaling = float(rot.attention_scaling)
        # float8_inference: e4m3 copies of every block's projections (ops.float8_inference_weights), or None
        self.float8 = None
        if lm.float8_inference:
            self.float8 = [ops.float8_inference_weights(lw[1], lw[2], lw[3], lw[7], lw[9], lw[10], lw[11])
                        for lw in self.layers]


def _check_scope(model) -> None:
    lm, _ = _parts(model)
    if getattr(lm, "tp_group", None) is not None or getattr(model, "tp_group", None) is not None:
        raise TouchNetB200Error("generate / cached decoding runs on one GPU: the model is tensor parallel")
    if getattr(lm.model, "cp_group", None) is not None:
        raise TouchNetB200Error("generate / cached decoding runs on one GPU: the model is context parallel")
    try:
        from torch.distributed.fsdp import FSDPModule
    except ImportError:
        FSDPModule = ()
    if any(isinstance(mod, FSDPModule) for mod in model.modules()) or any(ops._is_dtensor(p) for p in model.parameters()):
        raise TouchNetB200Error("generate / cached decoding needs an unsharded model (FSDP2 / DTensor parameters found)")


def _last_doc_start(attention_mask: torch.Tensor) -> torch.Tensor:
    """First position of each row's last document: the rows the new tokens attend to start there."""
    T = attention_mask.shape[1]
    other = attention_mask != attention_mask[:, -1:]
    last_other = T - 1 - other.flip(1).to(torch.int32).argmax(1)          # last position outside the last document
    return torch.where(other.any(1), last_other + 1, torch.zeros_like(last_other)).to(torch.int32)


def _check_mask(attention_mask: torch.Tensor, B: int, T: int) -> None:
    if attention_mask.dim() != 2 or tuple(attention_mask.shape) != (B, T):
        raise TouchNetB200Error("attention_mask must be the [B, T] document-id (or 0/1) mask of the prompt")
    if bool((attention_mask[:, -1] == 0).any()):
        raise TouchNetB200Error("the prompt's last column is padding: generation needs left-padded prompts")


def _logits_last(w: _Weights, x_last: torch.Tensor) -> torch.Tensor:
    h, _, _ = ops.rmsnorm_fwd(x_last, w.norm, w.norm_eps)
    return ops.gemm(h, w.lm_head)


def _default_positions(attention_mask: torch.Tensor) -> torch.Tensor:
    """hf GenerationMixin: cumsum of the mask, 1 at padding."""
    m = (attention_mask != 0).to(torch.int64)
    return (m.cumsum(-1) - 1).masked_fill_(m == 0, 1)


def _prompt_front(model, w: _Weights, input_ids, input_features, doc, pos):
    """Embeddings of the prompt [B, T] (their NaN flag raised here), the AttnPlan of its document ids `doc` and the rope
    tables of its positions `pos`: (x, plan, cos, sin)."""
    _, audio = _parts(model)
    B, T = input_ids.shape
    d = w.embed.shape[1]
    proj, nan_flag = None, None
    if audio is not None:
        nan_flag = audio._nan_flag
        if input_features is not None and T != 1:     # ref: modeling_touch_audio.py:124-131
            feats = input_features if input_features.dtype == BF16 else input_features.to(BF16)
            proj = ops.gemm(ops._rows2d(feats), ops.bf16_weight(audio.projector.weight))
    x = ops.embed_add(input_ids.reshape(-1).contiguous(), w.embed, proj, B * T, d, nan_flag)
    if audio is not None:
        audio.raise_if_nan()
    return (x, ops.AttnPlan(doc), *ops.rope_table(pos, w.inv_freq, w.rope_scaling))


def _pad_rows(t: torch.Tensor, rows: int) -> torch.Tensor:
    return t if t.shape[0] == rows else torch.cat([t, t.new_zeros((rows - t.shape[0], *t.shape[1:]))])


def _layers(cache: B200KVCache, w: _Weights, x, cos, sin, attend, qkv_rows=None, step: bool = False):
    """Every block over the rows x; `attend(q, k, v, k_cache, v_cache) -> (o, lse)` stores the layer's K/V into its
    cache and runs the attention.  `qkv_rows`: see ops.block_forward.  `step`: a cached step (decode, draft or verify)
    rather than a prompt pass; with FP8 weights (w.float8) it selects the kernels (ops.RowwiseInference), and a prompt
    pass runs on its rows zero-padded to a multiple of 16 (row scales keep the padding out of the real rows)."""
    M = x.shape[0]
    Mp = M if w.float8 is None or step else -(-M // 16) * 16
    if Mp != M:
        x, cos, sin = _pad_rows(x, Mp), _pad_rows(cos, Mp), _pad_rows(sin, Mp)
        inner = attend

        def attend(q, k, v, kc, vc):
            o, lse = inner(q[:M], k[:M], v[:M], kc, vc)
            return _pad_rows(o, Mp), lse

    for i, lw in enumerate(w.layers):
        kc, vc = cache.layer(i)
        x, _ = ops.cached_block_forward(x, lw, cos, sin, cache.H, cache.KV, w.eps, cache.hd,
                                        lambda q, k, v, kc=kc, vc=vc: (*attend(q, k, v, kc, vc), k, v),
                                        qkv_rows=qkv_rows, float8=None if w.float8 is None else w.float8[i], step=step)
    return x[:M] if Mp != M else x


def prefill(model, cache: B200KVCache, input_ids, input_features=None, attention_mask=None, position_ids=None,
            weights: Optional[_Weights] = None) -> torch.Tensor:
    """Run the prompt [B, T] through the model, fill cache rows [0, T) of every layer, and return the last position's
    logits [B, V] (bf16).  The cache's device state is set so that the next pick / pushed token is position T."""
    lm, _ = _parts(model)
    w = weights or _Weights(lm)
    B, T = input_ids.shape
    if B != cache.B or T > cache.S_cap or cache.length != 0:
        raise TouchNetB200Error(f"prefill: prompt [{B}, {T}] does not fit an empty cache of [{cache.B}, {cache.S_cap}]")
    dev = input_ids.device
    if attention_mask is None:
        attention_mask = torch.ones((B, T), dtype=torch.int64, device=dev)
    _check_mask(attention_mask, B, T)
    position_ids = (_default_positions(attention_mask) if position_ids is None else position_ids).to(torch.int64)
    x, plan, cos, sin = _prompt_front(model, w, input_ids, input_features, attention_mask, position_ids)
    cache.kv_start.copy_(_last_doc_start(attention_mask))
    cache.kv_end.fill_(T)          # read by kv_append: the state is written before the layers run
    cache.positions.copy_(position_ids[:, -1])
    cache.history[:, :T] = input_ids
    cache.finished.zero_()

    def attend(q, k, v, kc, vc):
        ops.kv_append(k, v, kc, vc, cache.kv_end, T)
        return ops.attn_fwd(q, k, v, plan, cache.H, cache.KV, cache.scale)

    x = _layers(cache, w, x, cos, sin, attend)
    cache.length = T
    return _logits_last(w, x.view(B, T, -1)[:, -1].contiguous())


def decode_step(model, cache: B200KVCache, weights: Optional[_Weights] = None) -> torch.Tensor:
    """One token per row: feed cache.next_ids at cache.positions, append its K/V at row kv_end - 1, attend to
    [kv_start, kv_end); returns the logits [B, V] (bf16).  Reads and writes device state only (graph-capturable)."""
    lm, audio = _parts(model)
    w = weights or _Weights(lm)
    B = cache.B
    x = ops.embed_add(cache.next_ids, w.embed, None, B, w.embed.shape[1], None if audio is None else audio._nan_flag)
    cos, sin = ops.rope_table(cache.positions, w.inv_freq, w.rope_scaling)

    def attend(q, k, v, kc, vc):
        ops.kv_append(k, v, kc, vc, cache.kv_end, 1)
        o = ops.attn_decode(q, kc, vc, cache.kv_start, cache.kv_end, cache.H, cache.KV, cache.scale, cache.workspace)
        return o, None

    return _logits_last(w, _layers(cache, w, x, cos, sin, attend, step=True))


def forward_cached(model, cache: B200KVCache, input_ids, input_features=None, attention_mask=None, position_ids=None):
    """`forward(..., past_key_values=cache)`: prefill on an empty cache, else one decode step per call with input_ids
    [B, 1] (positions continue from the cache; attention_mask / position_ids of later calls are not consulted).
    Returns the last position's logits [B, 1, V]."""
    from .modeling import CausalLMOutputWithPast
    _check_scope(model)
    if input_ids is None:
        raise TouchNetB200Error("cached forward needs input_ids")
    with torch.no_grad():
        if cache.length == 0:
            logits = prefill(model, cache, input_ids, input_features, attention_mask, position_ids)
        else:
            if input_ids.shape != (cache.B, 1):
                raise TouchNetB200Error(f"cached decode takes input_ids [{cache.B}, 1], got {tuple(input_ids.shape)}")
            cache.push(input_ids[:, 0])
            logits = decode_step(model, cache)
            _, audio = _parts(model)
            if audio is not None:
                audio.raise_if_nan()
    return CausalLMOutputWithPast(logits=logits[:, None], past_key_values=cache)


# kwargs of HF `generate` that greedy search ignores (do_sample=False, num_beams=1)
_IGNORED = ("bos_token_id", "top_k", "top_p", "temperature", "early_stopping")


def _validate(max_new_tokens, eos_token_id, pad_token_id, repetition_penalty, no_repeat_ngram_size, do_sample, num_beams,
              kwargs):
    if do_sample:
        raise TouchNetB200Error("generate: only greedy search is implemented (do_sample=True)")
    if num_beams != 1:
        raise TouchNetB200Error(f"generate: only greedy search is implemented (num_beams={num_beams})")
    if isinstance(eos_token_id, (list, tuple)) or (torch.is_tensor(eos_token_id) and eos_token_id.numel() != 1):
        raise TouchNetB200Error("generate: eos_token_id must be a single id")
    if eos_token_id is None or pad_token_id is None:
        raise TouchNetB200Error("generate: eos_token_id and pad_token_id are required")
    if int(max_new_tokens) < 1:
        raise TouchNetB200Error(f"generate: max_new_tokens must be >= 1, got {max_new_tokens}")
    if not float(repetition_penalty) > 0.0:
        raise TouchNetB200Error(f"generate: repetition_penalty must be > 0, got {repetition_penalty}")
    if int(no_repeat_ngram_size) < 0:
        raise TouchNetB200Error(f"generate: no_repeat_ngram_size must be >= 0, got {no_repeat_ngram_size}")
    bad = sorted(k for k, v in kwargs.items() if v is not None)
    if bad:
        raise TouchNetB200Error(f"generate: unsupported arguments {bad}")


def _captured(step, capture: bool):
    """`step` (no arguments, device state only) as a callable that runs it eagerly the first time, then, if `capture`,
    captures it once in a CUDA graph and replays the graph; without `capture` every call runs eagerly."""
    graph, calls = None, 0

    def run():
        nonlocal graph, calls
        if graph is None and calls >= 1 and capture:
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                step()
        if graph is not None:
            graph.replay()
        else:
            step()
        calls += 1

    return run


def _host_sync(flags, *nan_flags) -> list:
    """The one host sync per decode step: the int32 tensors `flags` and the NaN flags (None: no flag) read in one
    `.tolist()`.  A set NaN flag is zeroed and raises ValueError; otherwise returns the values of `flags`, flattened."""
    nan_flags = [f for f in nan_flags if f is not None]
    flags = [f.reshape(-1) for f in flags] + nan_flags
    vals = (flags[0] if len(flags) == 1 else torch.cat(flags)).tolist()
    if nan_flags:
        bad = vals[len(vals) - len(nan_flags):]
        del vals[len(vals) - len(nan_flags):]
        if any(bad):
            for f in nan_flags:
                f.zero_()
            raise ValueError("NaN in data.")
    return vals


def generate(model, input_ids, input_features=None, attention_mask=None, position_ids=None, *, max_new_tokens,
             eos_token_id, pad_token_id, repetition_penalty=1.0, no_repeat_ngram_size=0, do_sample=False, num_beams=1,
             use_cache=True, bos_token_id=None, top_k=None, top_p=None, temperature=None, early_stopping=None, **kwargs):
    """Greedy decoding with HF `generate` semantics: returns [B, T + n] ids (the prompt, then n <= max_new_tokens
    generated ids; rows that emitted eos continue with pad), stopping when every row has emitted eos.
    With `assistant_model` (HF's assisted generation) a draft model proposes `num_assistant_tokens` tokens per round
    and the model verifies them in one step (see generate_speculative): the result is the same tensor, bit for bit."""
    if kwargs.get("assistant_model") is not None:
        return generate_speculative(
            model, input_ids, input_features, attention_mask, position_ids, max_new_tokens=max_new_tokens,
            eos_token_id=eos_token_id, pad_token_id=pad_token_id, repetition_penalty=repetition_penalty,
            no_repeat_ngram_size=no_repeat_ngram_size, do_sample=do_sample, num_beams=num_beams, use_cache=use_cache,
            bos_token_id=bos_token_id, top_k=top_k, top_p=top_p, temperature=temperature, early_stopping=early_stopping,
            **kwargs)
    _validate(max_new_tokens, eos_token_id, pad_token_id, repetition_penalty, no_repeat_ngram_size, do_sample, num_beams,
              kwargs)
    _check_scope(model)
    eos, pad = int(eos_token_id), int(pad_token_id)
    lm, audio = _parts(model)
    B, T = input_ids.shape
    if attention_mask is not None:
        _check_mask(attention_mask, B, T)
    max_new = int(max_new_tokens)
    with torch.no_grad():
        w = _Weights(lm)
        cache = B200KVCache(model, B, T + max_new, device=input_ids.device)
        nan_flag = None if audio is None else audio._nan_flag

        def select(logits):
            ops.greedy_select(logits, cache.history, cache.kv_end, cache.positions, cache.next_ids, cache.finished,
                              float(repetition_penalty), int(no_repeat_ngram_size), eos, pad)

        select(prefill(model, cache, input_ids, input_features, attention_mask, position_ids, weights=w))
        step = _captured(lambda: select(decode_step(model, cache, weights=w)), input_ids.is_cuda)
        n = 1
        while n < max_new and not _host_sync([cache.finished.min()], nan_flag)[0]:
            step()
            n += 1
        if n == max_new and nan_flag is not None:
            _host_sync([], nan_flag)
    return cache.history[:, :T + n].clone()


# ---------------------------------------------------------------------------------------------------------------
# speculative decoding (HF assisted generation): a draft model proposes, the model verifies k + 1 rows in one step
# ---------------------------------------------------------------------------------------------------------------
# assisted-generation knobs of HF `generate` that are not implemented (a fixed number of draft tokens per round only)
_SPEC_UNSUPPORTED = ("assistant_confidence_threshold", "prompt_lookup_num_tokens", "assistant_early_exit",
                     "assistant_tokenizer")


def _gqa(model) -> int:
    a = _parts(model)[0].model.layers[0].self_attn
    return a.num_heads // a.num_key_value_heads


def _spec_args(model, draft, k, schedule, kwargs) -> int:
    """Checks of the draft and of the assisted-generation arguments; returns the number of draft tokens per round."""
    bad = sorted(n for n in _SPEC_UNSUPPORTED if kwargs.pop(n, None) is not None)
    if bad:
        raise TouchNetB200Error(f"generate: unsupported assisted-generation arguments {bad} (a fixed number of draft "
                                "tokens per round only)")
    if schedule is not None and schedule != "constant":
        raise TouchNetB200Error(f"generate: num_assistant_tokens_schedule must be 'constant', got {schedule!r}")
    lm, audio = _parts(model)
    dlm, daudio = _parts(draft)
    if not isinstance(dlm, type(lm)) or (audio is None) != (daudio is None):
        raise TouchNetB200Error("generate: the assistant_model must be a B200 model of the same kind as the model "
                                "(both Llama, or both TouchAudio)")
    if audio is not None and daudio.projector.weight.shape[1] != audio.projector.weight.shape[1]:
        raise TouchNetB200Error("generate: the assistant_model's projector input width differs from the model's")
    if dlm.config.vocab_size != lm.config.vocab_size:
        raise TouchNetB200Error(f"generate: the assistant_model's vocab_size {dlm.config.vocab_size} differs from the "
                                f"model's {lm.config.vocab_size}")
    if dlm.lm_head.weight.device != lm.lm_head.weight.device:
        raise TouchNetB200Error("generate: the assistant_model is on another device")
    _check_scope(draft)
    G, Gd = _gqa(model), _gqa(draft)
    if k is None and G > 8:
        raise TouchNetB200Error(f"generate: the model's H/KV = {G} leaves no room for a draft token: its verify step "
                                "needs H/KV * (num_assistant_tokens + 1) <= 16")
    k = min(4, 16 // G - 1) if k is None else k
    if isinstance(k, bool) or int(k) != k or int(k) < 1:
        raise TouchNetB200Error(f"generate: num_assistant_tokens must be an int >= 1, got {k}")
    k = int(k)
    if G * (k + 1) > 16:
        raise TouchNetB200Error(f"generate: num_assistant_tokens {k} with H/KV = {G}: the verify step needs "
                                "H/KV * (num_assistant_tokens + 1) <= 16")
    if 2 * Gd > 16:
        raise TouchNetB200Error(f"generate: the assistant_model's H/KV = {Gd}: its two-token step needs 2 * H/KV <= 16")
    return k


def _block_step(model, cache: B200KVCache, w: _Weights, ids, pos, end, workspace, s_attn: int):
    """Tq = ids.shape[1] new tokens per row: ids / pos [B, Tq] at cache rows [end - Tq, end) (K/V appended there),
    query j attending to [kv_start, end - Tq + j + 1).  Returns the last hidden state [B*Tq, d].  Every row is computed
    as decode_step computes its token: the QKV path is chosen for B rows, and the attention runs on cache rows
    [0, s_attn) only, so that its split count and chunks (functions of the cache length) are those of a decode step
    on a cache of s_attn rows; a query whose range reaches past s_attn is clipped there."""
    _, audio = _parts(model)
    B, Tq = ids.shape
    x = ops.embed_add(ids.reshape(-1), w.embed, None, B * Tq, w.embed.shape[1], None if audio is None else audio._nan_flag)
    cos, sin = ops.rope_table(pos, w.inv_freq, w.rope_scaling)

    def attend(q, k, v, kc, vc):
        ops.kv_append(k, v, kc, vc, end, Tq)
        return ops.attn_decode_multi(q, kc[:, :s_attn], vc[:, :s_attn], cache.kv_start, end, Tq, cache.H, cache.KV,
                                     cache.scale, workspace), None

    return _layers(cache, w, x, cos, sin, attend, qkv_rows=B, step=True)


def _multi_ws(cache: B200KVCache, Tq: int, s_attn: int) -> torch.Tensor:
    n = _lib.load().tn_attn_decode_multi_ws_floats(cache.B, Tq, cache.H, cache.KV, s_attn)
    return torch.empty(int(n), dtype=torch.float32, device=cache.data.device)


class _SpecRound:
    """One round of speculative decoding over the model's cache tc and the draft's cache dc (both [B, S_gen + k] rows),
    device state only, so that it is captured once as a CUDA graph: bring the draft's state to the model's (and
    `copies`, further (dst, src) pairs), a two-token draft step (the last two accepted tokens: the draft never fed its
    last proposal when all were accepted), k - 1 one-token draft steps, each followed by draft_select(logits, j) and its
    token copied from dc.next_ids into drafts[:, j], then the verify step of B*(k+1) rows and verify(logits).

    The verify step attends to the first S_gen rows of tc only, the cache length of decoding without a draft, so that
    every row sums in that decode step's split order; a query row clipped there lies past its slot's limit, so its pick
    is never emitted.  A slot with no tokens (idle in generate_many) reads history row 0; its draft steps append nothing
    and attend to nothing, its verify step appends rows [0, k) of its own slot and attends to them; every read and write
    stays inside the slot, and its selections hold it still."""

    def __init__(self, model, draft, tc, dc, w, wd, k, S_gen, draft_select, verify, copies=()):
        dev = tc.data.device
        self.model, self.draft, self.tc, self.dc, self.w, self.wd = model, draft, tc, dc, w, wd
        self.k, self.S_gen = k, S_gen
        self.draft_select, self.verify = draft_select, verify
        self.copies = ((dc.history, tc.history), (dc.kv_end, tc.kv_end), (dc.positions, tc.positions),
                       (dc.finished, tc.finished)) + tuple(copies)
        self.drafts = torch.zeros((tc.B, k), dtype=torch.int64, device=dev)
        self.end = torch.zeros(tc.B, dtype=torch.int32, device=dev)
        self.ar = torch.arange(k + 1, dtype=torch.int64, device=dev)
        self.ws, self.dws = _multi_ws(tc, k + 1, S_gen), _multi_ws(dc, 2, dc.S_cap)

    def __call__(self):
        tc, dc, wd, k, ar, B = self.tc, self.dc, self.wd, self.k, self.ar, self.tc.B
        for dst, src in self.copies:
            dst.copy_(src)
        # the last two accepted tokens, at positions - 1 and positions
        ids2 = dc.history.gather(1, (dc.kv_end.to(torch.int64)[:, None] - 2 + ar[None, :2]).clamp_(min=0))
        x = _block_step(self.draft, dc, wd, ids2, dc.positions[:, None] - 1 + ar[None, :2], dc.kv_end, self.dws,
                        dc.S_cap)
        self.draft_select(_logits_last(wd, x.view(B, 2, -1)[:, 1].contiguous()), 0)
        self.drafts[:, 0].copy_(dc.next_ids)
        for j in range(1, k):
            self.draft_select(decode_step(self.draft, dc, weights=wd), j)
            self.drafts[:, j].copy_(dc.next_ids)
        # verify: next_ids and the k proposals at positions + 0..k, appended at rows [kv_end - 1, kv_end + k)
        torch.add(tc.kv_end, k, out=self.end)
        x = _block_step(self.model, tc, self.w, torch.cat([tc.next_ids[:, None], self.drafts], 1),
                        tc.positions[:, None] + ar, self.end, self.ws, self.S_gen)
        self.verify(_logits_last(self.w, x))


def generate_speculative(model, input_ids, input_features=None, attention_mask=None, position_ids=None, *,
                         assistant_model, max_new_tokens, eos_token_id, pad_token_id, num_assistant_tokens=None,
                         num_assistant_tokens_schedule=None, repetition_penalty=1.0, no_repeat_ngram_size=0,
                         do_sample=False, num_beams=1, use_cache=True, bos_token_id=None, top_k=None, top_p=None,
                         temperature=None, early_stopping=None, **kwargs):
    """`generate(..., assistant_model=draft, num_assistant_tokens=k)`: returns exactly what `generate` returns without
    the draft.  Each round the draft proposes k tokens per row (its own greedy picks with the same processors), the
    model scores next_ids and the k proposals in ONE step of B*(k+1) rows (multi-query decode attention) and keeps the
    longest prefix of proposals equal to its own picks plus its next pick (tn_verify_select_bf16).  Since position j of
    that step computes exactly what decode_step computes for the same prefix, the picks are the greedy picks; the draft
    changes how many tokens a round yields, never which.

    The draft receives the same prompt (ids, features, mask, positions).  A round is captured once as a CUDA graph:
    bring the draft's state to the accepted prefix, a two-token draft step (the last two accepted tokens: the draft
    never fed its last proposal when all were accepted), k - 1 one-token draft steps, the verify step; then one host sync
    reads the finished flags and both NaN flags."""
    k = _spec_args(model, assistant_model, num_assistant_tokens, num_assistant_tokens_schedule, kwargs)
    _validate(max_new_tokens, eos_token_id, pad_token_id, repetition_penalty, no_repeat_ngram_size, do_sample, num_beams,
              kwargs)
    _check_scope(model)
    eos, pad = int(eos_token_id), int(pad_token_id)
    penalty, ngram = float(repetition_penalty), int(no_repeat_ngram_size)
    draft = assistant_model
    lm, audio = _parts(model)
    dlm, daudio = _parts(draft)
    B, T = input_ids.shape
    if attention_mask is not None:
        _check_mask(attention_mask, B, T)
    max_new = int(max_new_tokens)
    dev = input_ids.device
    with torch.no_grad():
        w, wd = _Weights(lm), _Weights(dlm)
        S_cap = T + max_new + k              # the verify step writes up to k rows past the final length
        # ... but attends as `generate` does on its cache of T + max_new rows: the same decode splits and chunks.
        # A query row clipped there lies past `limit`, so its pick is never emitted.
        S_gen = T + max_new
        tc = B200KVCache(model, B, S_cap, device=dev)
        dc = B200KVCache(draft, B, S_cap, device=dev)
        flags = (None if audio is None else audio._nan_flag, None if daudio is None else daudio._nan_flag)
        limit = torch.full((B,), T + max_new, dtype=torch.int32, device=dev)
        picks = torch.zeros((B, k + 1), dtype=torch.int64, device=dev)

        ops.greedy_select(prefill(model, tc, input_ids, input_features, attention_mask, position_ids, weights=w),
                          tc.history, tc.kv_end, tc.positions, tc.next_ids, tc.finished, penalty, ngram, eos, pad)
        prefill(draft, dc, input_ids, input_features, attention_mask, position_ids, weights=wd)

        def draft_select(logits, j):
            ops.greedy_select(logits, dc.history, dc.kv_end, dc.positions, dc.next_ids, dc.finished, penalty, ngram,
                              eos, pad)

        def verify(logits):
            ops.verify_select(logits, drafts, tc.history, tc.kv_end, tc.positions, tc.next_ids, tc.finished, limit,
                              penalty, ngram, eos, pad, picks=picks)

        rnd = _SpecRound(model, draft, tc, dc, w, wd, k, S_gen, draft_select, verify)
        drafts = rnd.drafts
        step = _captured(rnd, input_ids.is_cuda)
        if max_new == 1:
            _host_sync([tc.finished.min()], *flags)
        else:
            while not _host_sync([tc.finished.min()], *flags)[0]:
                step()
        count = (tc.kv_end - T).tolist()
        n = min(max_new, max(count))
        out = tc.history[:, :T + n].clone()
        beyond = torch.arange(n, device=dev)[None, :] >= torch.tensor(count, device=dev)[:, None]
        out[:, T:].masked_fill_(beyond, pad)
    return out


# ---------------------------------------------------------------------------------------------------------------
# continuous batching
# ---------------------------------------------------------------------------------------------------------------
_ALIGN = 128            # rows of one attention q block: each admitted prompt starts on a block boundary
_MIN_PACKED_ROWS = 256  # a packed prefill row always takes the fused-QKV path (ops.qkv_fusable), alone or not
_ADMIT_MAX = 128        # documents per admission launch (TN_ADMIT_MAX)


class _Prompt:
    """One utterance of generate_many, validated and on the model's device."""

    def __init__(self, index, p, audio, max_len, budget, dev):
        if not isinstance(p, dict) or "input_ids" not in p:
            raise TouchNetB200Error(f"generate_many: prompt {index} must be a dict with 'input_ids'")
        unknown = sorted(set(p) - {"input_ids", "input_features", "attention_mask", "position_ids"})
        if unknown:
            raise TouchNetB200Error(f"generate_many: prompt {index}: unsupported keys {unknown}")
        ids = torch.as_tensor(p["input_ids"])
        if ids.dim() != 1 or ids.numel() == 0:
            raise TouchNetB200Error(f"generate_many: prompt {index}: input_ids must be a non-empty 1-D tensor")
        T = ids.numel()
        if T > max_len:
            raise TouchNetB200Error(f"generate_many: prompt {index} has {T} tokens, more than max_prompt_length "
                                    f"{max_len}")
        feats = p.get("input_features")
        if feats is not None:
            if audio is None:
                raise TouchNetB200Error("generate_many: unsupported arguments ['input_features'] (a text-only model)")
            if feats.dim() != 2 or feats.shape[0] != T:
                raise TouchNetB200Error(f"generate_many: prompt {index}: input_features must be [T, F] with T = {T}")
        mask = p.get("attention_mask")
        mask = torch.ones(T, dtype=torch.int64, device=dev) if mask is None else mask.to(dev, torch.int64)
        _check_mask(mask.reshape(1, -1), 1, T)
        pos = p.get("position_ids")
        if pos is None:
            pos = _default_positions(mask)
        elif tuple(pos.shape) != (T,):
            raise TouchNetB200Error(f"generate_many: prompt {index}: position_ids must be [{T}]")
        self.index, self.T, self.budget = index, T, budget
        self.ids = ids.to(dev, torch.int64)
        self.feats = None if feats is None else feats.to(dev)
        self.mask, self.pos = mask, pos.to(dev, torch.int64)


def _admit(model, cache: B200KVCache, limit: torch.Tensor, w: _Weights, batch, pad: int, select) -> None:
    """Prefill `batch` [(slot, _Prompt)] into their slots as ONE packed row of documents and select each one's first
    token.  Prompt j occupies rows [o_j, o_j + T_j), o_j a multiple of 128; its documents are its runs of equal
    attention_mask values (padding included: never attended by the new tokens), relabelled o_j + run index so the row's
    ids are non-decreasing and non-zero; the gap rows after it continue its last document (ids pad, features zero),
    so every 128-row q block holds rows of one prompt and sees the K/V blocks it sees when prefilled alone.  Slots not
    in `batch` are not touched.  select=None (a draft model's cache) fills the cache and the state only: no lm_head."""
    lm, audio = _parts(model)
    dev = cache.data.device
    offs, o = [], 0
    for _, p in batch:
        offs.append(o)
        o += -(-p.T // _ALIGN) * _ALIGN
    n = max(o, _MIN_PACKED_ROWS)
    ids = torch.empty(n, dtype=torch.int64, device=dev)
    doc = torch.empty(n, dtype=torch.int64, device=dev)
    pos = torch.zeros(n, dtype=torch.int64, device=dev)
    any_feats = any(p.feats is not None and p.T != 1 for _, p in batch)
    feats = None
    if any_feats:
        width = next(p.feats.shape[1] for _, p in batch if p.feats is not None)
        feats = torch.zeros((n, width), dtype=BF16, device=dev)
    docs = []
    for j, ((slot, p), o0) in enumerate(zip(batch, offs)):
        end = offs[j + 1] if j + 1 < len(batch) else n
        m = p.mask
        runs = torch.cat([m.new_zeros(1), (m[1:] != m[:-1]).to(torch.int64).cumsum(0)]) + (o0 + 1)
        doc[o0:o0 + p.T] = runs
        doc[o0 + p.T:end] = runs[-1]
        ids[o0:o0 + p.T] = p.ids
        ids[o0 + p.T:end] = pad
        pos[o0:o0 + p.T] = p.pos
        if feats is not None and p.feats is not None and p.T != 1:     # as generate: no projector on a 1-token prompt
            feats[o0:o0 + p.T] = p.feats.to(BF16)
        docs.append((o0, slot, p.T, p.T + p.budget))
    x, plan, cos, sin = _prompt_front(model, w, ids.view(1, n), None if feats is None else feats.view(1, n, -1),
                                      doc.view(1, n), pos.view(1, n))
    ops.slot_admit(docs, ids, plan.doc.view(-1), pos, cache.history, cache.kv_start, cache.kv_end, cache.positions,
                   cache.finished, limit)

    def attend(q, k, v, kc, vc):
        ops.kv_scatter(k, v, kc, vc, docs)
        return ops.attn_fwd(q, k, v, plan, cache.H, cache.KV, cache.scale)

    x = _layers(cache, w, x, cos, sin, attend)
    if select is not None:
        last = torch.tensor([o0 + p.T - 1 for (_, p), o0 in zip(batch, offs)], dtype=torch.int64).to(dev)
        select(_logits_last(w, x.index_select(0, last)), [slot for slot, _ in batch])


def _sampling_args(temperature, top_k, top_p):
    """HF's multinomial-sampling knobs, None -> transformers' defaults (temperature 1.0, top_k 50, top_p 1.0)."""
    temperature = 1.0 if temperature is None else temperature
    top_k = 50 if top_k is None else top_k
    top_p = 1.0 if top_p is None else top_p
    if (isinstance(temperature, bool) or not isinstance(temperature, (int, float))
            or not 0.0 < float(temperature) < math.inf):
        raise TouchNetB200Error(f"generate_many: temperature must be a finite number > 0, got {temperature}")
    if isinstance(top_k, bool) or not isinstance(top_k, int) or top_k < 0:
        raise TouchNetB200Error(f"generate_many: top_k must be an int >= 0, got {top_k}")
    if isinstance(top_p, bool) or not isinstance(top_p, (int, float)) or not 0.0 <= float(top_p) <= 1.0:
        raise TouchNetB200Error(f"generate_many: top_p must be in [0, 1], got {top_p}")
    return float(temperature), min(int(top_k), 2**31 - 1), float(top_p)


def generate_many(model, prompts, *, batch_size, max_new_tokens, eos_token_id, pad_token_id, repetition_penalty=1.0,
                  no_repeat_ngram_size=0, max_prompt_length=None, cuda_graph: bool = True, stats: Optional[dict] = None,
                  do_sample: bool = False, temperature=None, top_k=None, top_p=None, assistant_model=None,
                  num_assistant_tokens=None, num_assistant_tokens_schedule=None, **kwargs):
    """Greedy decoding, or multinomial sampling, of many prompts with continuous batching: a cache of `batch_size`
    slots; when a slot's row finishes (eos or its token budget), its generated ids are copied out and the next prompt is
    prefilled into that slot while the other slots keep decoding.  Per prompt, the greedy result is what `generate`
    returns for that prompt alone (HF greedy with the same processors), as a 1-D int64 tensor of the generated ids (eos
    included if reached, no padding); the list is in input order.

    do_sample=True draws each token from HF's sampling distribution (processors, then temperature, top_k, top_p; None
    takes HF's defaults 1.0, 50, 1.0) with tn_sample_select_slots_bf16.  One 64-bit seed is taken from torch's default
    CPU generator, so torch.manual_seed reproduces a call; prompt i draws from its own Philox stream (seed, i) at its
    token positions, so its ids do not depend on batch_size, its slot, its neighbours or when it was admitted.  With
    do_sample=False the three knobs are ignored, as HF ignores them in greedy search.

    prompts          iterable of dicts: input_ids [T], optional input_features [T, F] (TouchAudio), attention_mask [T]
                     (doc ids or 0/1, last document rule of `generate`), position_ids [T]
    max_new_tokens   an int, or one budget per prompt
    max_prompt_length  the longest prompt to expect (default: the longest of `prompts` when it is a sequence)
    cuda_graph       False runs every decode step eagerly (the captured step computes the same bits)
    stats            if a dict, receives decode_steps, admissions and, on CUDA, admission_events (pairs of CUDA events
                     around each admission prefill); with a draft also rounds (= decode_steps) and live_row_rounds
                     (summed over rounds: the slots holding a prompt in that round)

    assistant_model (HF's assisted generation, with num_assistant_tokens k and the checks of `generate`): speculative
    decoding.  Each slot's prompt is prefilled into the same slot of a draft cache; per round the draft proposes k
    tokens per slot and the model scores them in one step of B*(k+1) rows (_SpecRound).  Greedy: the result is the one
    without the draft, bit for bit (tn_verify_select_bf16).  do_sample=True: speculative sampling
    (tn_spec_sample_verify_bf16): the draft draws its proposals with tn_sample_select_slots_bf16 and the same knobs from
    its own Philox streams (a second 64-bit seed, the next draw from torch's default CPU generator), and each prompt's
    ids have exactly the distribution of sampling without the draft; its first token is the same draw."""
    budgets = None
    if isinstance(max_new_tokens, (list, tuple)) or (torch.is_tensor(max_new_tokens) and max_new_tokens.dim() == 1):
        budgets = [int(b) for b in max_new_tokens]
        if not budgets:
            raise TouchNetB200Error("generate_many: max_new_tokens is an empty sequence")
        bad = [b for b in budgets if b < 1]
        if bad:
            raise TouchNetB200Error(f"generate: max_new_tokens must be >= 1, got {bad[0]}")
        max_budget = max(budgets)
    else:
        max_budget = int(max_new_tokens)
    draft, k = assistant_model, None
    if draft is not None:
        k = _spec_args(model, draft, num_assistant_tokens, num_assistant_tokens_schedule, kwargs)
    elif kwargs:        # the keyword arguments of assisted generation only
        raise TypeError(f"generate_many() got an unexpected keyword argument {next(iter(kwargs))!r}")
    else:               # without a draft the assisted-generation knobs are unsupported arguments, as in `generate`
        kwargs = dict(num_assistant_tokens=num_assistant_tokens,
                      num_assistant_tokens_schedule=num_assistant_tokens_schedule)
    _validate(max_budget, eos_token_id, pad_token_id, repetition_penalty, no_repeat_ngram_size, False, 1, kwargs)
    if do_sample:
        temperature, top_k, top_p = _sampling_args(temperature, top_k, top_p)
    _check_scope(model)
    B = int(batch_size)
    if B < 1:
        raise TouchNetB200Error(f"generate_many: batch_size must be >= 1, got {batch_size}")
    if hasattr(prompts, "__len__") and hasattr(prompts, "__getitem__") and not isinstance(prompts, dict):
        prompts = list(prompts)
        if budgets is not None and len(budgets) != len(prompts):
            raise TouchNetB200Error(f"generate_many: {len(budgets)} budgets for {len(prompts)} prompts")
        if not prompts:
            return []
        if max_prompt_length is None:
            max_prompt_length = max(1, max(torch.as_tensor(p["input_ids"]).numel() if isinstance(p, dict) and
                                           "input_ids" in p else 0 for p in prompts))
    elif max_prompt_length is None:
        raise TouchNetB200Error("generate_many: max_prompt_length is required when prompts is not a sequence")
    max_len = int(max_prompt_length)
    if max_len < 1:
        raise TouchNetB200Error(f"generate_many: max_prompt_length must be >= 1, got {max_prompt_length}")
    eos, pad = int(eos_token_id), int(pad_token_id)
    penalty, ngram = float(repetition_penalty), int(no_repeat_ngram_size)
    lm, audio = _parts(model)
    dev = lm.lm_head.weight.device
    it = iter(prompts)
    results: dict = {}
    slot_prompt: list = [None] * B            # the _Prompt decoding in each slot, None = idle
    count = 0
    with torch.no_grad():
        w = _Weights(lm)
        S_gen = max_len + max_budget
        # with a draft the verify step writes up to k rows past a slot's limit
        cache = B200KVCache(model, B, S_gen if draft is None else S_gen + k, device=dev)
        limit = torch.zeros(B, dtype=torch.int32, device=dev)
        stream_key = torch.zeros(B, dtype=torch.int64, device=dev)    # the index of the prompt in each slot
        seed = int(torch.randint(-2**63, 2**63 - 1, (), dtype=torch.int64)) if do_sample else 0
        cache.finished.fill_(1)               # every slot starts idle
        nan_flag = None if audio is None else audio._nan_flag
        admission_events = []
        admissions = 0

        def select(logits, slots=None):
            if do_sample:
                ops.sample_select_slots(logits, cache.history, cache.kv_end, cache.positions, cache.next_ids,
                                        cache.finished, limit, stream_key, float(repetition_penalty),
                                        int(no_repeat_ngram_size), temperature, top_k, top_p, seed, eos, pad,
                                        row_slot=slots,
                                        row_key=None if slots is None else [slot_prompt[s].index for s in slots])
            else:
                ops.greedy_select_slots(logits, cache.history, cache.kv_end, cache.positions, cache.next_ids,
                                        cache.finished, limit, float(repetition_penalty), int(no_repeat_ngram_size),
                                        eos, pad, row_slot=slots)

        if draft is None:
            flags = (nan_flag,)
            step = _captured(lambda: select(decode_step(model, cache, weights=w)), cuda_graph and dev.type == "cuda")
        else:
            dlm, daudio = _parts(draft)
            wd = _Weights(dlm)
            dc = B200KVCache(draft, B, S_gen + k, device=dev)
            flags = (nan_flag, None if daudio is None else daudio._nan_flag)
            dseed = int(torch.randint(-2**63, 2**63 - 1, (), dtype=torch.int64)) if do_sample else 0
            dkey = torch.zeros(B, dtype=torch.int64, device=dev)
            dlogits = torch.empty((B, k, cache.vocab), dtype=BF16, device=dev) if do_sample else None
            picks = torch.zeros((B, k + 1), dtype=torch.int64, device=dev)

            def draft_select(logits, j):
                if do_sample:
                    dlogits[:, j].copy_(logits)
                    ops.sample_select_slots(logits, dc.history, dc.kv_end, dc.positions, dc.next_ids, dc.finished,
                                            limit, dkey, penalty, ngram, temperature, top_k, top_p, dseed, eos, pad)
                else:
                    ops.greedy_select_slots(logits, dc.history, dc.kv_end, dc.positions, dc.next_ids, dc.finished,
                                            limit, penalty, ngram, eos, pad)

            def verify(logits):
                if do_sample:
                    ops.spec_sample_verify(logits, dlogits.view(B * k, -1), rnd.drafts, cache.history, cache.kv_end,
                                           cache.positions, cache.next_ids, cache.finished, limit, stream_key, penalty,
                                           ngram, temperature, top_k, top_p, seed, eos, pad, picks=picks)
                else:
                    ops.verify_select(logits, rnd.drafts, cache.history, cache.kv_end, cache.positions, cache.next_ids,
                                      cache.finished, limit, penalty, ngram, eos, pad, picks=picks)

            rnd = _SpecRound(model, draft, cache, dc, w, wd, k, S_gen, draft_select, verify,
                             copies=((dkey, stream_key),) if do_sample else ())
            step = _captured(rnd, cuda_graph and dev.type == "cuda")

        def admit(free) -> None:
            nonlocal count, admissions
            batch = []
            for slot in free:
                try:
                    p = next(it)
                except StopIteration:
                    break
                if budgets is not None and count >= len(budgets):
                    raise TouchNetB200Error("generate_many: more prompts than budgets")
                budget = budgets[count] if budgets is not None else max_budget
                batch.append((slot, _Prompt(count, p, audio, max_len, budget, dev)))
                count += 1
            for i in range(0, len(batch), _ADMIT_MAX):
                chunk = batch[i:i + _ADMIT_MAX]
                for slot, p in chunk:             # before the admission: its selection reads the prompts' indices
                    slot_prompt[slot] = p
                ev = None
                if stats is not None and dev.type == "cuda":
                    ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
                    ev[0].record()
                _admit(model, cache, limit, w, chunk, pad, select)
                if draft is not None:             # the same slots of the draft's cache, no first-token selection
                    _admit(draft, dc, limit, wd, chunk, pad, None)
                admissions += 1
                if ev is not None:
                    ev[1].record()
                    admission_events.append(ev)

        admit(list(range(B)))
        steps = live_row_rounds = 0
        while any(p is not None for p in slot_prompt):
            live_row_rounds += sum(p is not None for p in slot_prompt)
            step()
            steps += 1
            vals = _host_sync([cache.finished, cache.kv_end], *flags)
            free = []
            for s in range(B):
                p = slot_prompt[s]
                if p is not None and vals[s] != 0:
                    results[p.index] = cache.history[s, p.T:vals[B + s]].clone()
                    slot_prompt[s] = None
                    free.append(s)
            if free:
                admit(free)
        if stats is not None:
            stats.update(decode_steps=steps, admissions=admissions, admission_events=admission_events)
            if draft is not None:
                stats.update(rounds=steps, live_row_rounds=live_row_rounds)
    if budgets is not None and count != len(budgets):
        raise TouchNetB200Error(f"generate_many: {len(budgets)} budgets for {count} prompts")
    return [results[i] for i in range(count)]
