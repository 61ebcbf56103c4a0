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
           with one host sync per step to read the finished flags and the NaN flag.

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


def _prompt_embeds(model, input_ids, input_features, w: _Weights):
    lm, audio = _parts(model)
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
    return x


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
    if position_ids is None:          # hf GenerationMixin: cumsum of the mask, 1 at padding
        m = (attention_mask != 0).to(torch.int64)
        position_ids = (m.cumsum(-1) - 1).masked_fill_(m == 0, 1)
    position_ids = position_ids.to(torch.int64)
    x = _prompt_embeds(model, input_ids, input_features, w)
    plan = ops.AttnPlan(attention_mask)
    cos, sin = ops.rope_table(position_ids, w.inv_freq, w.rope_scaling)
    cache.kv_start.copy_(_last_doc_start(attention_mask))
    cache.kv_end.fill_(T)
    cache.positions.copy_(position_ids[:, -1])
    cache.history[:, :T] = input_ids
    cache.finished.zero_()
    H, KV, hd = cache.H, cache.KV, cache.hd
    scale = 1.0 / math.sqrt(hd)
    for i, lw in enumerate(w.layers):
        kc, vc = cache.layer(i)

        def attend(q, k, v, kc=kc, vc=vc):
            ops.kv_append(k, v, kc, vc, cache.kv_end, T)
            o, lse = ops.attn_fwd(q, k, v, plan, H, KV, scale)
            return o, lse, k, v

        x, _ = ops.block_forward(x, *lw, cos, sin, H, KV, w.eps, hd, attend, need_gu=False)
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
    H, KV, hd = cache.H, cache.KV, cache.hd
    scale = 1.0 / math.sqrt(hd)
    for i, lw in enumerate(w.layers):
        kc, vc = cache.layer(i)

        def attend(q, k, v, kc=kc, vc=vc):
            ops.kv_append(k, v, kc, vc, cache.kv_end, 1)
            o = ops.attn_decode(q, kc, vc, cache.kv_start, cache.kv_end, H, KV, scale, cache.workspace)
            return o, None, k, v

        x, _ = ops.block_forward(x, *lw, cos, sin, H, KV, w.eps, hd, attend, need_gu=False)
    return _logits_last(w, x)


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


def generate(model, input_ids, input_features=None, attention_mask=None, position_ids=None, *, max_new_tokens,
             eos_token_id, pad_token_id, repetition_penalty=1.0, no_repeat_ngram_size=0, do_sample=False, num_beams=1,
             use_cache=True, bos_token_id=None, top_k=None, top_p=None, temperature=None, early_stopping=None, **kwargs):
    """Greedy decoding with HF `generate` semantics: returns [B, T + n] ids (the prompt, then n <= max_new_tokens
    generated ids; rows that emitted eos continue with pad), stopping when every row has emitted eos."""
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

        def done() -> bool:   # the one host sync per step
            flags = cache.finished.min().reshape(1)
            if nan_flag is not None:
                flags = torch.cat([flags, nan_flag.reshape(1).to(flags.dtype)])
            vals = flags.tolist()
            if len(vals) > 1 and vals[1] != 0:
                nan_flag.zero_()
                raise ValueError("NaN in data.")
            return vals[0] != 0

        select(prefill(model, cache, input_ids, input_features, attention_mask, position_ids, weights=w))
        n = 1
        graph = None
        while n < max_new and not done():
            if graph is None and n >= 2 and input_ids.is_cuda:
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph):
                    select(decode_step(model, cache, weights=w))
            if graph is not None:
                graph.replay()
            else:
                select(decode_step(model, cache, weights=w))     # the first decode step runs eagerly
            n += 1
        if n == max_new and nan_flag is not None:
            done()
    return cache.history[:, :T + n].clone()
