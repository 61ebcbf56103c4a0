"""Drop-in modules for the reference's model slot (TrainSpec.model_cls, ref: touchnet/utils/train_spec.py:25-44).

`B200LlamaForCausalLM` mirrors what `TrainSpec("llama")` instantiates (transformers LlamaForCausalLM,
ref: touchnet/__init__.py:35-39) and `B200TouchAudioForCausalLM` mirrors
ref: touchnet/models/touch_audio/modeling_touch_audio.py:19-152 — same constructor contract (config object, meta-device
construction, `post_init()`), same forward signature and output type, and the same parameter FQNs / state-dict keys

    model.embed_tokens.weight, model.layers.N.{input_layernorm,post_attention_layernorm}.weight,
    model.layers.N.self_attn.{q,k,v,o}_proj.weight, model.layers.N.mlp.{gate,up,down}_proj.weight,
    model.norm.weight, lm_head.weight, [language_model.* + projector.weight]

so the reference's parallelize_* (FSDP2 per block, ref: touchnet/models/helper_func.py:134-202), post_init
(ref: touchnet/models/llama/__init__.py:19-36), DCP checkpoints and HF<->DCP converters keep working on them.
All arithmetic runs in libtouchnet_b200.so (see ops.py); there is no eager fallback.
"""
from __future__ import annotations

import math
from typing import Any, Optional

import torch
import torch.nn as nn

from . import ops
from ._lib import TouchNetB200Error

try:  # output container of the reference's forward (transformers is a dependency of the reference itself)
    from transformers.modeling_outputs import CausalLMOutputWithPast
except Exception:  # pragma: no cover - transformers missing: keep the attribute contract
    class CausalLMOutputWithPast(dict):  # type: ignore
        def __init__(self, logits=None, **kw):
            super().__init__(logits=logits, **kw)
            self.logits = logits


# ---------------------------------------------------------------------------------------------------------------
# config helpers (accept HF LlamaConfig / Qwen2Config objects of transformers 4.51 .. 5.x, or any attribute bag)
# ---------------------------------------------------------------------------------------------------------------
def _cfg(config, name, default=None):
    v = getattr(config, name, None)
    return default if v is None else v


def _rope_theta(config) -> float:
    v = getattr(config, "rope_theta", None)
    if v is None:
        rp = getattr(config, "rope_parameters", None) or {}
        v = rp.get("rope_theta", 10000.0)
    return float(v)


def _rope_scaling(config) -> Optional[dict]:
    rs = getattr(config, "rope_scaling", None)
    if rs is None:
        rp = getattr(config, "rope_parameters", None)
        if rp and rp.get("rope_type", "default") != "default":
            rs = dict(rp)
    return rs


def compute_rope_parameters(config, device=None, **_):
    """(inv_freq, attention_scaling) - the `rope_init_fn` the reference's post_init calls
    (ref: touchnet/models/llama/__init__.py:22-27); default and llama3 variants of hf:modeling_rope_utils.py."""
    head_dim = _cfg(config, "head_dim", config.hidden_size // config.num_attention_heads)
    base = _rope_theta(config)
    inv_freq = 1.0 / (base ** (torch.arange(0, head_dim, 2, dtype=torch.int64).to(device=device, dtype=torch.float) / head_dim))
    rs = _rope_scaling(config)
    kind = "default" if rs is None else rs.get("rope_type", rs.get("type", "default"))
    if kind == "default":
        return inv_freq, 1.0
    if kind != "llama3":
        raise TouchNetB200Error(f"rope_type {kind!r} is not supported by touchnet_b200 (default, llama3)")
    factor, lo, hi = rs["factor"], rs["low_freq_factor"], rs["high_freq_factor"]
    old_len = rs["original_max_position_embeddings"]
    low_wl, high_wl = old_len / lo, old_len / hi
    wavelen = 2 * math.pi / inv_freq
    inv_llama = torch.where(wavelen > low_wl, inv_freq / factor, inv_freq)
    smooth = (old_len / wavelen - lo) / (hi - lo)
    smoothed = (1 - smooth) * inv_llama / factor + smooth * inv_llama
    is_medium = ~(wavelen < high_wl) * ~(wavelen > low_wl)
    return torch.where(is_medium, smoothed, inv_llama), 1.0


class B200RotaryEmbedding(nn.Module):
    """Holds exactly the attributes the reference's post_init re-initialises:
    config, rope_init_fn, inv_freq, attention_scaling, original_inv_freq."""

    def __init__(self, config):
        super().__init__()
        self.config = config
        self.rope_init_fn = compute_rope_parameters
        inv_freq, self.attention_scaling = self.rope_init_fn(config, device=None)
        self.register_buffer("inv_freq", inv_freq, persistent=False)
        self.original_inv_freq = self.inv_freq

    def forward(self, position_ids: torch.Tensor):
        """cos/sin tables [B*T, hd/2] (bf16), hf: LlamaRotaryEmbedding.forward modeling_llama.py:124-141."""
        inv = self.inv_freq
        if inv.dtype != torch.float32:
            # `model.to(bfloat16)` also casts buffers; the angles must come from fp32 frequencies (the reference keeps
            # the model in fp32, touchnet/bin/train.py:283, so this only matters for callers that cast the module)
            inv, _ = self.rope_init_fn(self.config, device=inv.device)
        return ops.rope_table(position_ids, inv, float(self.attention_scaling))


class B200RMSNorm(nn.Module):
    def __init__(self, hidden_size: int, eps: float = 1e-6):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(hidden_size))
        self.variance_epsilon = eps

    def forward(self, x):
        w = self.weight
        if ops._is_dtensor(w):      # tensor parallel: replicated weight, sequence-sharded rows (SequenceParallel in the ref plan)
            from . import tensor_parallel
            w = tensor_parallel.replicated_param(w, w.device_mesh.get_group())
        return ops.rms_norm(x, w, self.variance_epsilon)


class B200Attention(nn.Module):
    def __init__(self, config, layer_idx: int):
        super().__init__()
        d = config.hidden_size
        self.layer_idx = layer_idx
        self.num_heads = config.num_attention_heads
        self.num_key_value_heads = _cfg(config, "num_key_value_heads", self.num_heads)
        self.head_dim = _cfg(config, "head_dim", d // self.num_heads)
        bias = bool(_cfg(config, "attention_bias", False)) or getattr(config, "model_type", "") == "qwen2"
        self.q_proj = nn.Linear(d, self.num_heads * self.head_dim, bias=bias)
        self.k_proj = nn.Linear(d, self.num_key_value_heads * self.head_dim, bias=bias)
        self.v_proj = nn.Linear(d, self.num_key_value_heads * self.head_dim, bias=bias)
        self.o_proj = nn.Linear(self.num_heads * self.head_dim, d, bias=False)


class B200MLP(nn.Module):
    def __init__(self, config):
        super().__init__()
        d, f = config.hidden_size, config.intermediate_size
        self.gate_proj = nn.Linear(d, f, bias=False)
        self.up_proj = nn.Linear(d, f, bias=False)
        self.down_proj = nn.Linear(f, d, bias=False)


class B200DecoderLayer(nn.Module):
    def __init__(self, config, layer_idx: int):
        super().__init__()
        self.hidden_size = config.hidden_size
        self.self_attn = B200Attention(config, layer_idx)
        self.mlp = B200MLP(config)
        eps = _cfg(config, "rms_norm_eps", 1e-6)
        self.input_layernorm = B200RMSNorm(config.hidden_size, eps)
        self.post_attention_layernorm = B200RMSNorm(config.hidden_size, eps)

    def forward(self, hidden_states, cos, sin, plan, fp8: bool = False, float8_recipe_name: str = "tensorwise"):
        a, m = self.self_attn, self.mlp
        if plan.tp is None:
            return ops.decoder_layer(
                hidden_states, self.input_layernorm.weight, a.q_proj.weight, a.k_proj.weight, a.v_proj.weight,
                a.q_proj.bias, a.k_proj.bias, a.v_proj.bias, a.o_proj.weight, self.post_attention_layernorm.weight,
                m.gate_proj.weight, m.up_proj.weight, m.down_proj.weight, cos, sin, plan, a.num_heads,
                a.num_key_value_heads, self.input_layernorm.variance_epsilon, a.head_dim, fp8,
                float8_recipe_name=float8_recipe_name)
        # tensor parallel (tensor_parallel.py): this rank's weight shards, H/tp and KV/tp heads
        from .tensor_parallel import local
        wq, wk = local(a.q_proj.weight), local(a.k_proj.weight)
        return ops.decoder_layer(
            hidden_states, local(self.input_layernorm.weight), wq, wk, local(a.v_proj.weight),
            local(a.q_proj.bias), local(a.k_proj.bias), local(a.v_proj.bias), local(a.o_proj.weight),
            local(self.post_attention_layernorm.weight), local(m.gate_proj.weight), local(m.up_proj.weight),
            local(m.down_proj.weight), cos, sin, plan, wq.shape[0] // a.head_dim, wk.shape[0] // a.head_dim,
            self.input_layernorm.variance_epsilon, fp8=fp8, float8_recipe_name=float8_recipe_name)


class B200LlamaModel(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.config = config
        self.padding_idx = _cfg(config, "pad_token_id")
        self.vocab_size = config.vocab_size
        # hf: LlamaModel.__init__ modeling_llama.py: nn.Embedding(vocab, hidden, padding_idx=config.pad_token_id) - the pad
        # row is zero at init and receives no gradient (TouchAudio writes the pad id at every audio-frame position)
        self.embed_tokens = nn.Embedding(config.vocab_size, config.hidden_size, padding_idx=self.padding_idx)
        self.layers = nn.ModuleList([B200DecoderLayer(config, i) for i in range(config.num_hidden_layers)])
        self.norm = B200RMSNorm(config.hidden_size, _cfg(config, "rms_norm_eps", 1e-6))
        self.rotary_emb = B200RotaryEmbedding(config)
        # FP8 projections in every decoder block (ops.block_forward); cached decoding follows float8_inference, not
        # this.  Plain attributes: no parameter or buffer, so state dicts do not change
        self.float8_training = bool(_cfg(config, "float8_training", False))
        # FP8 (rowwise e4m3) projections in cached decoding: prefill, decode, speculative and generate_many steps
        self.float8_inference = bool(_cfg(config, "float8_inference", False))
        # the FP8 recipe when float8_training is on: "tensorwise" (default) or "rowwise"
        self.float8_recipe_name = ops.check_fp8_recipe(_cfg(config, "float8_recipe_name", "tensorwise"))
        hd = _cfg(config, "head_dim", config.hidden_size // config.num_attention_heads)
        if hd > 128 or hd % 8:
            raise TouchNetB200Error(f"touchnet_b200 attention kernels are built for head_dim 128 (smaller multiples of 8 run "
                                    f"through them with zero-padded heads); config has {hd}")

    def forward(self, inputs_embeds: torch.Tensor, attention_mask: Optional[torch.Tensor],
                position_ids: Optional[torch.Tensor]):
        """hf: LlamaModel.forward modeling_llama.py:375-427 (ref restatement touchnet/models/llama/pipeline_llama.py:37-107).
        `attention_mask` carries document ids (ref: touchnet/models/llama/processing_llama.py:37-40)."""
        B, T, _ = inputs_embeds.shape
        dev = inputs_embeds.device
        tp_group = getattr(self, "tp_group", None)
        if tp_group is not None:        # inputs_embeds is this rank's sequence shard; masks / positions are the full [B, T]
            import torch.distributed as dist
            T = T * dist.get_world_size(tp_group)
        if position_ids is None:
            if getattr(self, "cp_group", None) is not None:
                raise TouchNetB200Error("context parallelism needs the (sharded) position_ids of the packed batch")
            position_ids = torch.arange(T, device=dev, dtype=torch.int64)[None].expand(B, T)
        if attention_mask is None:
            attention_mask = torch.ones((B, T), dtype=torch.int32, device=dev)
        if attention_mask.dim() != 2:
            raise TouchNetB200Error("attention_mask must be the [B,T] document-id tensor of the packed batch")
        cp_group = getattr(self, "cp_group", None)
        if cp_group is not None:                            # sequence sharded over the cp mesh: see context_parallel.py
            from . import context_parallel
            plan = context_parallel.make_cp_plan(attention_mask, cp_group, getattr(self, "cp_load_balance", False))
        else:
            plan = ops.AttnPlan(attention_mask)             # once per step, shared by all layers
        if tp_group is not None:
            from . import tensor_parallel
            if attention_mask.shape[1] != T or position_ids.shape[1] != T:
                raise TouchNetB200Error("tensor parallelism: attention_mask / position_ids must cover the whole sequence")
            plan.tp = tensor_parallel.make_context(tp_group, B, dev, cache_on=self)
            plan.tp.begin_step()
        cos, sin = self.rotary_emb(position_ids)            # once per step
        x = inputs_embeds
        if x.dtype != torch.bfloat16:
            x = x.to(torch.bfloat16)
        for layer in self.layers:
            x = layer(x, cos, sin, plan, self.float8_training, self.float8_recipe_name)
        return self.norm(x)


class _EmbedAddFn(torch.autograd.Function):
    """E = embed_tokens(input_ids) + projected audio features (ref: modeling_touch_audio.py:124-131), NaN flag folded in."""

    @staticmethod
    def forward(ctx, input_ids, embed_w, proj, nan_flag, padding_idx=None):
        B, T = input_ids.shape
        ctx.padding_idx = padding_idx
        d = embed_w.shape[1]
        ids = input_ids.reshape(-1).contiguous()
        p2 = None if proj is None else proj.reshape(B * T, d)
        e = ops.embed_add(ids, embed_w, p2, B * T, d, nan_flag)
        ctx.save_for_backward(ids)
        ctx.embed_shape, ctx.embed_dtype, ctx.has_proj = embed_w.shape, embed_w.dtype, proj is not None
        return e.view(B, T, d)

    @staticmethod
    def backward(ctx, de):
        (ids,) = ctx.saved_tensors
        d_embed = None
        if ctx.needs_input_grad[1]:
            d_embed = torch.zeros(ctx.embed_shape, dtype=ctx.embed_dtype, device=de.device)
            d_embed.index_add_(0, ids, de.reshape(-1, de.shape[-1]).to(ctx.embed_dtype))
            if ctx.padding_idx is not None and 0 <= ctx.padding_idx < ctx.embed_shape[0]:
                d_embed[ctx.padding_idx].zero_()          # nn.Embedding(padding_idx=...): no gradient for the pad row
        return None, d_embed, (de if ctx.has_proj else None), None, None


def _root_reshards_after_forward(module: nn.Module) -> bool:
    """True when `module` is an FSDP2 root whose parameter group frees its unsharded parameters when forward returns (the
    reference's default policy, ref: touchnet/models/helper_func.py:196-202): lm_head.weight must then be consumed INSIDE
    forward.  Unknown FSDP internals count as "reshards" (the safe answer)."""
    try:
        from torch.distributed.fsdp import FSDPModule
    except ImportError:
        return False
    if not isinstance(module, FSDPModule):
        return False
    try:
        grp = module._get_fsdp_state()._fsdp_param_group
        if grp is None:
            return False
        info = getattr(grp, "post_forward_mesh_info", None)
        flag = getattr(grp, "_reshard_after_forward", None)
        if flag is not None:
            return bool(flag)
        return info is not None
    except Exception:
        return True


class B200LlamaForCausalLM(nn.Module):
    base_model_prefix = "model"
    _tied_weights_keys = ["lm_head.weight"]
    # fused lm_head + loss (loss.py::FusedLinearCEFn): in training mode `pred.logits` becomes a loss.LazyLogits handle that
    # loss.cross_entropy_loss / loss.accuracy consume without ever materialising [B,T,V].  The "*_b200" TrainSpecs switch it
    # on (train_spec.register: their loss_fn / acc_fn are exactly those two functions); direct users get real logits.
    fused_linear_ce = False
    # tensor parallel only: keep the logits sharded on the vocabulary and let loss.cross_entropy_loss reduce per-row statistics
    # over the tp group (the reference's `loss_parallel`, touchnet/utils/distributed.py:322-323); set by parallelize.py from
    # parallel_dims.loss_parallel_enabled
    loss_parallel = False

    def __init__(self, config):
        super().__init__()
        self.config = config
        self.model = B200LlamaModel(config)       # reads the config keys `float8_training`, `float8_inference`
        self.vocab_size = config.vocab_size
        self.lm_head = nn.Linear(config.hidden_size, config.vocab_size, bias=False)
        if _cfg(config, "tie_word_embeddings", False):
            self.lm_head.weight = self.model.embed_tokens.weight
        else:
            self._tied_weights_keys = None

    @property
    def float8_training(self) -> bool:
        """FP8 (torchao tensorwise recipe) for the q/k/v/o/gate/up/down projections of every decoder block, forward and
        backward; lm_head, attention and norms stay bf16, and cached decoding follows float8_inference.  Set from the config
        key `float8_training`."""
        return self.model.float8_training

    @float8_training.setter
    def float8_training(self, v: bool):
        self.model.float8_training = bool(v)

    @property
    def float8_inference(self) -> bool:
        """FP8 for the q/k/v/o/gate/up/down projections of cached decoding (prefill, decode_step, forward_cached,
        generate, speculative decoding, generate_many), always with the rowwise recipe (one power-of-two scale per row,
        so a row's result does not depend on the other rows): weights quantised once per call, the prompt through the
        rowwise wgmma GEMMs, every cached step through tn_gemm_fp8_decode.  Embedding, norms, biases, the audio
        projector, lm_head and the KV cache stay bf16, as does the uncached forward.  Set from the config key
        `float8_inference`."""
        return self.model.float8_inference

    @float8_inference.setter
    def float8_inference(self, v: bool):
        self.model.float8_inference = bool(v)

    @property
    def float8_recipe_name(self) -> str:
        """The FP8 recipe of float8_training: "tensorwise" (torchao's default: one scale per tensor, e5m2 gradients) or
        "rowwise" (one power-of-two scale per row, e4m3 throughout).  Set from the config key `float8_recipe_name`."""
        return self.model.float8_recipe_name

    @float8_recipe_name.setter
    def float8_recipe_name(self, v: str):
        self.model.float8_recipe_name = ops.check_fp8_recipe(v)

    # -- HF surface the reference touches -------------------------------------------------------------------
    def get_input_embeddings(self):
        return self.model.embed_tokens

    def set_input_embeddings(self, value):
        self.model.embed_tokens = value

    def get_output_embeddings(self):
        return self.lm_head

    def set_output_embeddings(self, new):
        self.lm_head = new

    def get_decoder(self):
        return self.model

    def set_decoder(self, decoder):
        self.model = decoder

    def post_init(self):
        """HF `_init_weights`: normal(0, initializer_range) for Linear / Embedding, ones for norms; then the rope
        buffers (the reference's own post_init repeats the latter, ref: touchnet/models/llama/__init__.py:19-36)."""
        std = float(_cfg(self.config, "initializer_range", 0.02))
        for m in self.modules():
            if isinstance(m, nn.Linear):
                nn.init.normal_(m.weight, 0.0, std)
                if m.bias is not None:
                    nn.init.zeros_(m.bias)
            elif isinstance(m, nn.Embedding):
                nn.init.normal_(m.weight, 0.0, std)
                if m.padding_idx is not None and m.weight.device.type != "meta":
                    with torch.no_grad():
                        m.weight[m.padding_idx].zero_()     # hf `_init_weights`: the padding row stays zero
            elif isinstance(m, B200RMSNorm):
                nn.init.ones_(m.weight)
        rot = self.model.rotary_emb
        dev = rot.inv_freq.device
        if dev.type != "meta":
            inv, scaling = rot.rope_init_fn(rot.config, device=dev)
            rot.inv_freq = inv
            rot.attention_scaling = scaling
            rot.original_inv_freq = inv

    def forward(self, input_ids: Optional[torch.Tensor] = None, attention_mask: Optional[torch.Tensor] = None,
                position_ids: Optional[torch.Tensor] = None, past_key_values=None,
                inputs_embeds: Optional[torch.Tensor] = None, labels=None, use_cache=None, **kwargs: Any):
        assert labels is None, "loss is computed in the train loop (ref: modeling_touch_audio.py:121)"
        if past_key_values is not None and use_cache is not False:
            from . import generation
            if isinstance(past_key_values, generation.B200KVCache):    # prefill or one decode step (generation.py)
                return generation.forward_cached(self, past_key_values, input_ids, None, attention_mask, position_ids)
        ops.begin_forward(self)             # side-stream casts of stale fp32 master weights / new cache epoch under FSDP2
        tp_group = getattr(self, "tp_group", None)
        if inputs_embeds is None:
            if input_ids is None:
                raise TouchNetB200Error("either input_ids or inputs_embeds is required")
            if tp_group is None:
                inputs_embeds = _EmbedAddFn.apply(input_ids, self.model.embed_tokens.weight, None, None,
                                                  self.model.embed_tokens.padding_idx)
            else:
                from . import tensor_parallel
                inputs_embeds = tensor_parallel.embed(input_ids, self.model.embed_tokens.weight,
                                                      tensor_parallel.TPContext(tp_group, input_ids.shape[0]),
                                                      self.model.embed_tokens.padding_idx)
        h = self.model(inputs_embeds, attention_mask, position_ids)
        shift_labels = kwargs.get("shift_labels")
        if shift_labels is not None and tp_group is None and getattr(self.model, "cp_group", None) is None:
            # the reference's Liger route (ref: touchnet/bin/train.py:437-445: `shift_labels` stays in the batch and
            # `pred.loss` is used as is): token-mean cross-entropy of the pre-shifted labels, lm_head fused with the loss
            from . import loss as _loss
            ones = torch.ones(shift_labels.numel(), dtype=torch.int64, device=shift_labels.device)
            tot, _, _ = _loss.fused_linear_cross_entropy(h, self.lm_head.weight, shift_labels, ones, 1.0)
            n_valid = ((shift_labels >= 0) & (shift_labels < self.vocab_size)).sum().clamp(min=1)
            return CausalLMOutputWithPast(loss=tot / n_valid, logits=None)
        if tp_group is None:
            fused = (self.fused_linear_ce and self.training and torch.is_grad_enabled()
                     and not _root_reshards_after_forward(getattr(self, "_tn_fsdp_root", self)))
            if fused:
                from . import loss as _loss
                logits = _loss.LazyLogits(h, self.lm_head.weight)
            else:
                logits = ops.linear(h, self.lm_head.weight)
        else:       # h is the sequence shard
            from . import tensor_parallel
            tpc = tensor_parallel.TPContext(tp_group, h.shape[0])
            if getattr(self, "loss_parallel", False) and self.training and torch.is_grad_enabled():
                # logits stay sharded on the vocabulary; the spec's loss_fn / acc_fn reduce per-row statistics over tp
                logits = tensor_parallel.lm_head_loss_parallel(h, self.lm_head.weight, tpc)
            else:   # replicated [B, T, V] logits
                logits = tensor_parallel.lm_head(h, self.lm_head.weight, tpc)
        out = CausalLMOutputWithPast(logits=logits)
        return out

    def generate(self, input_ids: torch.Tensor, attention_mask: Optional[torch.Tensor] = None,
                 position_ids: Optional[torch.Tensor] = None, **kwargs: Any) -> torch.Tensor:
        """Greedy decoding with a KV cache, HF `generate` semantics (see generation.generate)."""
        from . import generation
        if kwargs.get("input_features") is not None:
            raise TouchNetB200Error("generate: unsupported arguments ['input_features'] (a text-only model)")
        kwargs.pop("input_features", None)
        return generation.generate(self, input_ids, None, attention_mask, position_ids, **kwargs)

    def generate_many(self, prompts, **kwargs: Any):
        """Greedy decoding or sampling of many prompts with continuous batching (see generation.generate_many)."""
        from . import generation
        return generation.generate_many(self, prompts, **kwargs)


class B200TouchAudioForCausalLM(nn.Module):
    """ref: touchnet/models/touch_audio/modeling_touch_audio.py:19-152 (a.k.a. LlamaForASR, docs/TouchAudioForCausalLM.md)."""
    base_model_prefix = "language_model"

    def __init__(self, config):
        super().__init__()
        self.config = config
        self.projector = nn.Linear(config.audio_config.input_size, config.text_config.hidden_size, bias=False)
        self.vocab_size = config.text_config.vocab_size
        self.language_model = B200LlamaForCausalLM(config.text_config)
        self._tied_weights_keys = None
        if self.language_model._tied_weights_keys is not None:
            self._tied_weights_keys = [f"language_model.{k}" for k in self.language_model._tied_weights_keys]
        pad = getattr(config, "pad_token_id", None)
        self.pad_token_id = pad if pad is not None else -1
        self._padding_side = "left"
        self.register_buffer("_nan_flag", torch.zeros(1, dtype=torch.int32), persistent=False)
        # lm_head.weight belongs to the FSDP2 ROOT group when this wrapper is the root: the inner model asks it
        object.__setattr__(self.language_model, "_tn_fsdp_root", self)
        if getattr(config, "float8_training", None) is not None:   # the top-level key of the model JSON wins
            self.float8_training = config.float8_training
        if getattr(config, "float8_recipe_name", None) is not None:
            self.float8_recipe_name = config.float8_recipe_name
        if getattr(config, "float8_inference", None) is not None:
            self.float8_inference = config.float8_inference

    @property
    def fused_linear_ce(self) -> bool:
        return self.language_model.fused_linear_ce

    @fused_linear_ce.setter
    def fused_linear_ce(self, v: bool):
        self.language_model.fused_linear_ce = bool(v)

    @property
    def float8_training(self) -> bool:
        return self.language_model.float8_training

    @float8_training.setter
    def float8_training(self, v: bool):
        self.language_model.float8_training = bool(v)

    @property
    def float8_inference(self) -> bool:
        return self.language_model.float8_inference

    @float8_inference.setter
    def float8_inference(self, v: bool):
        self.language_model.float8_inference = bool(v)

    @property
    def float8_recipe_name(self) -> str:
        return self.language_model.float8_recipe_name

    @float8_recipe_name.setter
    def float8_recipe_name(self, v: str):
        self.language_model.float8_recipe_name = v

    @property
    def model(self):  # the reference's llama post_init / get_num_params reach `model.model.*`
        return self.language_model.model

    @property
    def lm_head(self):
        return self.language_model.lm_head

    def get_input_embeddings(self):
        return self.language_model.get_input_embeddings()

    def set_input_embeddings(self, value):
        self.language_model.set_input_embeddings(value)

    def get_output_embeddings(self):
        return self.language_model.get_output_embeddings()

    def set_output_embeddings(self, new):
        self.language_model.set_output_embeddings(new)

    def get_decoder(self):
        return self.language_model.get_decoder()

    def set_decoder(self, decoder):
        self.language_model.set_decoder(decoder)

    def post_init(self):
        std = float(_cfg(self.config.text_config, "initializer_range", 0.02))
        nn.init.normal_(self.projector.weight, 0.0, std)
        self.language_model.post_init()

    def raise_if_nan(self):
        """The reference syncs every forward to raise ValueError("NaN in data.") (modeling_touch_audio.py:133-134).
        Here the scan is a flag written by the embedding kernel itself (no extra pass over E); reading it is the one
        host sync, done by `forward` every call by default (`check_nan=True`, the reference's behaviour) or by the
        caller at a step boundary when `forward(check_nan=False)` is used to keep the step free of syncs."""
        if int(self._nan_flag.item()) != 0:
            self._nan_flag.zero_()
            raise ValueError("NaN in data.")

    def forward(self, input_ids: Optional[torch.Tensor] = None, input_features: Optional[torch.Tensor] = None,
                attention_mask: Optional[torch.Tensor] = None, position_ids: Optional[torch.Tensor] = None,
                past_key_values=None, inputs_embeds: Optional[torch.Tensor] = None, labels=None, use_cache=None,
                output_attentions=None, output_hidden_states=None, return_dict=None, cache_position=None,
                logits_to_keep=0, check_nan: bool = True, **kwargs: Any):
        assert labels is None  # we calculate loss in train-loop (ref: modeling_touch_audio.py:121)
        if past_key_values is not None and use_cache is not False:
            from . import generation
            if isinstance(past_key_values, generation.B200KVCache):    # prefill or one decode step (generation.py)
                return generation.forward_cached(self, past_key_values, input_ids, input_features, attention_mask,
                                                 position_ids)
        ops.begin_forward(self)             # projector, decoder layers, lm_head: casts overlap the GEMMs in front of them
        tp_group = getattr(self, "tp_group", None)
        if inputs_embeds is None and tp_group is not None:
            # tensor parallel: vocabulary-sharded lookup reduce-scattered onto sequence shards; the (replicated) projector
            # runs on this rank's rows only, so its gradient is a partial sum over tp -> all-reduced
            from . import tensor_parallel
            tp = tensor_parallel.TPContext(tp_group, input_ids.shape[0])
            inputs_embeds = tensor_parallel.embed(input_ids, self.language_model.model.embed_tokens.weight, tp,
                                                  self.language_model.model.embed_tokens.padding_idx)
            if input_features is not None and input_ids.shape[1] != 1:
                feats = tp.seq_slice(input_features)
                feats = feats if feats.dtype == torch.bfloat16 else feats.to(torch.bfloat16)
                wp = tensor_parallel.replicated_param(self.projector.weight, tp_group)
                inputs_embeds = inputs_embeds + ops.linear(feats.contiguous(), wp)
            self._nan_flag.add_(torch.isnan(inputs_embeds).any().to(torch.int32))
        if inputs_embeds is None:
            lm = self.language_model
            proj = None
            if input_features is not None and input_ids.shape[1] != 1:
                feats = input_features if input_features.dtype == torch.bfloat16 else input_features.to(torch.bfloat16)
                proj = ops.linear(feats, self.projector.weight)
            # text-only batches: the reference pushes zeros through the bias-free projector (:128-130) = adds 0
            inputs_embeds = _EmbedAddFn.apply(input_ids, lm.model.embed_tokens.weight, proj, self._nan_flag,
                                              lm.model.embed_tokens.padding_idx)
        if check_nan:
            self.raise_if_nan()
        outputs = self.language_model(input_ids=None, attention_mask=attention_mask, position_ids=position_ids,
                                      inputs_embeds=inputs_embeds, **kwargs)
        outputs.attention_mask = attention_mask
        return outputs

    def generate(self, input_ids: torch.Tensor, input_features: Optional[torch.Tensor] = None,
                 attention_mask: Optional[torch.Tensor] = None, position_ids: Optional[torch.Tensor] = None,
                 **kwargs: Any) -> torch.Tensor:
        """The reference's evaluation call (ref: inference_touch_audio.py:170-192): greedy decoding with a KV cache, HF
        `generate` semantics, the audio features projected into the prompt only (see generation.generate)."""
        from . import generation
        return generation.generate(self, input_ids, input_features, attention_mask, position_ids, **kwargs)

    def generate_many(self, prompts, **kwargs: Any):
        """The evaluation call over a whole test set with continuous batching: finished rows are refilled with the next
        utterances while the others keep decoding (see generation.generate_many)."""
        from . import generation
        return generation.generate_many(self, prompts, **kwargs)


__all__ = ["B200LlamaForCausalLM", "B200TouchAudioForCausalLM", "B200LlamaModel", "B200DecoderLayer", "B200RMSNorm",
           "B200RotaryEmbedding", "compute_rope_parameters"]
