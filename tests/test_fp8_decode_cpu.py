"""CPU: the `float8_inference` switch of cached decoding and the argument checks of tn_gemm_fp8_decode (no GPU needed:
every check below fails before any CUDA call).  The header, the ctypes binding and their arity are covered for the new
symbol by tests/test_capi.py, which walks the whole header."""
import ctypes
from types import SimpleNamespace as NS

import pytest
import torch

from tests.test_float8_cpu import _text
from touchnet_b200 import _lib, generation, modeling, ops

F8 = torch.float8_e4m3fn
BF16 = torch.bfloat16


def _audio(**kw):
    return NS(audio_config=NS(input_size=400), text_config=_text(), pad_token_id=0, **kw)


def test_switch_defaults_to_false_and_is_plumbed():
    m = modeling.B200LlamaForCausalLM(_text())
    assert m.float8_inference is False and m.model.float8_inference is False
    assert modeling.B200LlamaForCausalLM(_text(float8_inference=True)).float8_inference is True
    a = modeling.B200TouchAudioForCausalLM(_audio())
    assert a.float8_inference is False
    a.float8_inference = 1
    assert a.language_model.float8_inference is True
    assert modeling.B200TouchAudioForCausalLM(_audio(float8_inference=True)).float8_inference is True


def test_state_dict_keys_do_not_change():
    torch.manual_seed(0)
    off = modeling.B200TouchAudioForCausalLM(_audio())
    on = modeling.B200TouchAudioForCausalLM(_audio(float8_inference=True))
    assert list(off.state_dict()) == list(on.state_dict())
    assert [n for n, _ in off.named_buffers()] == [n for n, _ in on.named_buffers()]


@pytest.mark.parametrize("fuse", [True, False])
def test_kernel_choice_follows_the_call_not_the_row_count(monkeypatch, fuse):
    """A cached step always runs one QKV launch without RoPE in the epilogue; a prompt pass plans as the rowwise
    training forward does (under either setting of the fused-QKV switch, which other tests' stand-ins turn off)."""
    monkeypatch.setattr(ops, "_FUSE_QKV", fuse)
    step, prompt = ops.RowwiseInference({}, True), ops.RowwiseInference({}, False)
    for M in (16, 48, 256, 4096):
        assert step.qkv_plan(M, 3072, 1024, True) == (True, False)
        assert prompt.qkv_plan(M, 3072, 1024, True) == ops._Rowwise.qkv_plan(M, 3072, 1024, True)
    assert prompt.qkv_plan(4096, 3072, 1024, True) == (fuse, fuse)
    assert prompt.qkv_plan(48, 3072, 1024, True) == (False, False)


def test_weight_dimensions_outside_the_16_rule_raise_before_any_work():
    w = lambda *s: torch.zeros(*s, dtype=BF16)
    with pytest.raises(_lib.TouchNetB200Error, match="float8_inference: GEMM dimensions must be multiples of 16"):
        ops.float8_inference_weights(w(40, 40), w(16, 40), w(16, 40), w(40, 40), w(64, 40), w(64, 40), w(40, 64))


def test_cached_decoding_refuses_sharded_models_with_the_switch_on():
    m = modeling.B200LlamaForCausalLM(_text(float8_inference=True))
    m.tp_group = object()
    with pytest.raises(_lib.TouchNetB200Error, match="tensor parallel"):
        generation._check_scope(m)


def test_wrapper_rejects_bad_operands_before_any_cuda_call():
    x = torch.zeros(3, 64, dtype=BF16)
    w8 = torch.zeros(32, 64, dtype=F8)
    inv = torch.ones(32)
    with pytest.raises(_lib.TouchNetB200Error, match="bfloat16"):
        ops.gemm_fp8_decode(x.float(), w8, inv)
    with pytest.raises(_lib.TouchNetB200Error, match="float8_e4m3fn"):
        ops.gemm_fp8_decode(x, w8.to(BF16), inv)
    with pytest.raises(_lib.TouchNetB200Error, match="differ in K"):
        ops.gemm_fp8_decode(x, torch.zeros(32, 48, dtype=F8), inv)
    with pytest.raises(_lib.TouchNetB200Error, match="multiples of 16"):
        ops.gemm_fp8_decode(torch.zeros(3, 40, dtype=BF16), torch.zeros(32, 40, dtype=F8), inv)
    with pytest.raises(_lib.TouchNetB200Error, match="multiples of 16"):
        ops.gemm_fp8_decode(x, torch.zeros(24, 64, dtype=F8), torch.ones(24))
    with pytest.raises(_lib.TouchNetB200Error, match="inv_w must be a contiguous float32 vector of 32"):
        ops.gemm_fp8_decode(x, w8, torch.ones(16))
    with pytest.raises(_lib.TouchNetB200Error, match="swiglu"):
        ops.gemm_fp8_decode(x, w8, inv, residual=torch.zeros(3, 16, dtype=BF16), swiglu=True)
    with pytest.raises(_lib.TouchNetB200Error, match="residual must be bfloat16"):
        ops.gemm_fp8_decode(x, w8, inv, residual=torch.zeros(3, 16, dtype=BF16))
    with pytest.raises(_lib.TouchNetB200Error, match="CUDA tensor"):
        ops.gemm_fp8_decode(x, w8, inv)


def _entry(*args):
    lib = _lib.load()
    rc = lib.tn_gemm_fp8_decode(*args)
    return rc, lib.tn_last_error().decode()


@pytest.mark.parametrize("args, msg", [
    ((None, 64, 16, 64, 16, 0, None, 0, 16, 16, 1, 16, 64, None), "null pointer"),
    ((16, 64, 16, 64, 16, 3, None, 0, 16, 16, 1, 16, 64, None), "epi=3"),
    ((16, 64, 16, 64, 16, 1, None, 0, 16, 16, 1, 16, 64, None), "R is required with epi 1"),
    ((16, 64, 16, 64, 16, 0, 16, 16, 16, 16, 1, 16, 64, None), "R is required with epi 1"),
    ((16, 64, 16, 64, 16, 0, None, 0, 16, 16, 0, 16, 64, None), "M=0"),
    ((16, 64, 16, 64, 16, 0, None, 0, 16, 16, 1, 24, 64, None), "N=24"),
    ((16, 64, 16, 64, 16, 0, None, 0, 16, 16, 1, 16, 40, None), "K=40"),
    ((16, 1 << 20, 16, 1 << 20, 16, 0, None, 0, 16, 16, 1, 16, 1 << 20, None), "too large"),
    ((16, 60, 16, 64, 16, 0, None, 0, 16, 16, 1, 16, 64, None), "X must be 16 B aligned"),
    ((16, 64, 16, 72, 16, 0, None, 0, 16, 16, 1, 16, 64, None), "W must be 16 B aligned"),
    ((16, 64, 16, 64, 18, 0, None, 0, 16, 16, 1, 16, 64, None), "inv_sw must be 4 B aligned"),
    ((16, 64, 16, 64, 16, 0, None, 0, 16, 8, 1, 16, 64, None), "ldd and ldr"),
])
def test_entry_point_rejects_bad_arguments(args, msg):
    """Pointers are fake small addresses: every check fails before the kernel would dereference them."""
    rc, err = _entry(*args)
    assert rc != 0 and msg in err, err
