"""ctypes binding of the C-ABI library (include/touchnet_b200.h).

The library is the product; there is no fallback.  If ``libtouchnet_b200.so`` is missing or a call fails,
this module raises — loudly — instead of routing anywhere else.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import c_char_p, c_float, c_int, c_int64, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libtouchnet_b200.so")

_lib = None

_vp, _i, _i64, _f = c_void_p, c_int, c_int64, c_float

# name -> argtypes (restype is always int unless listed in _RESTYPES); mirrors include/touchnet_b200.h
_SIGNATURES = {
    "tn_version": [],
    "tn_device_check": [],
    "tn_set_sm_margin": [_i],
    "tn_set_gemm_group": [_i],
    "tn_set_gemm_l2_hints": [_i],
    "tn_set_gemm_split_tail": [_i],
    "tn_gemm_bf16": [_vp, _i64, _i, _vp, _i64, _i, _vp, _i64, _i, _vp, _i64, _i, _i, _i, _vp],
    "tn_gemm_swiglu_bf16": [_vp, _i64, _vp, _vp, _i64, _vp, _vp, _vp, _i64, _i, _i, _i, _vp],
    "tn_gemm_dswiglu_bf16": [_vp, _i64, _vp, _i64, _vp, _vp, _i64, _vp, _vp, _i64, _i, _i, _i, _vp],
    "tn_gemm_qkv_bf16": [_i, _vp, _i64, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _i64, _i, _i, _i, _i, _i, _i, _i, _vp, _vp,
                         _vp],
    "tn_gemm_fp8": [_vp, _i64, _i, _vp, _i64, _vp, _i64, _i, _vp, _i64, _i, _i, _i, _vp, _vp, _vp],
    "tn_gemm_swiglu_fp8": [_vp, _i64, _i, _vp, _vp, _i64, _vp, _vp, _vp, _i64, _i, _i, _i, _vp, _vp, _vp],
    "tn_gemm_dswiglu_fp8": [_vp, _i64, _i, _vp, _i64, _vp, _vp, _i64, _vp, _vp, _i64, _i, _i, _i, _vp, _vp, _vp],
    "tn_gemm_qkv_fp8": [_i, _vp, _i64, _i, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _i64, _i, _i, _i, _i, _i, _i, _i, _vp, _vp,
                        _vp, _vp, _vp],
    "tn_fp8_amax_bf16": [_vp, _i64, _i64, _i64, _vp, _vp],
    "tn_fp8_cast_bf16": [_vp, _i64, _i64, _i64, _i, _vp, _vp, _i64, _vp, _i64, _vp, _vp],
    "tn_fp8_rowwise_cast_bf16": [_vp, _i64, _i64, _i64, _vp, _i64, _vp, _vp],
    "tn_fp8_colwise_amax_bf16": [_vp, _i64, _i64, _i64, _vp, _vp],
    "tn_fp8_colwise_cast_t_bf16": [_vp, _i64, _i64, _i64, _vp, _vp, _i64, _vp, _vp],
    "tn_gemm_fp8_rowwise": [_vp, _i64, _vp, _i64, _vp, _i64, _i, _vp, _i64, _i, _i, _i, _vp, _vp, _i, _vp],
    "tn_gemm_swiglu_fp8_rowwise": [_vp, _i64, _vp, _vp, _i64, _vp, _vp, _vp, _i64, _i, _i, _i, _vp, _vp, _vp],
    "tn_gemm_dswiglu_fp8_rowwise": [_vp, _i64, _vp, _i64, _vp, _vp, _i64, _vp, _vp, _i64, _i, _i, _i, _vp, _vp, _vp],
    "tn_gemm_qkv_fp8_rowwise": [_i, _vp, _i64, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _i64, _i, _i, _i, _i, _i, _i, _i,
                                _vp, _vp, _vp, _vp, _vp],
    "tn_gemm_fp8_decode": [_vp, _i64, _vp, _i64, _vp, _i, _vp, _i64, _vp, _i64, _i, _i, _i, _vp],
    "tn_swiglu_bwd_bf16": [_vp, _vp, _vp, _vp, _vp, _i64, _i64, _i64, _vp],
    "tn_rmsnorm_fwd_bf16": [_vp, _vp, _vp, _i, _vp, _vp, _vp, _i64, _i, _f, _vp],
    "tn_rmsnorm_bwd_bf16": [_vp, _vp, _vp, _vp, _i, _vp, _vp, _vp, _i, _vp, _i64, _i, _vp],
    "tn_rmsnorm_bwd_num_partials": [],
    "tn_rope_table": [_vp, _vp, _f, _vp, _vp, _i64, _i, _vp],
    "tn_rope_apply_bf16": [_vp, _i64, _vp, _vp, _i64, _i, _i, _i, _vp],
    "tn_attn_meta_ints": [_i, _i],
    "tn_attn_prep": [_vp, _vp, _i, _i, _vp],
    "tn_attn_fwd_bf16": [_vp, _i64, _vp, _i64, _vp, _i64, _vp, _i64, _vp, _vp, _vp, _i, _i, _i, _i, _f, _i, _i, _vp],
    "tn_attn_bwd_bf16": [_vp, _i64, _vp, _i64, _vp, _i64, _vp, _i64, _vp, _i64, _vp, _vp, _vp, _i64, _vp, _i64,
                         _vp, _i64, _vp, _vp, _i, _i, _i, _i, _f, _i, _i, _vp, _vp, _vp, _vp, _vp],
    "tn_attn_decode_ws_floats": [_i, _i, _i, _i],
    "tn_attn_decode_bf16": [_vp, _i64, _vp, _vp, _i64, _i64, _vp, _vp, _i, _i, _i, _i, _f, _vp, _vp, _i64, _vp, _vp],
    "tn_attn_decode_multi_ws_floats": [_i, _i, _i, _i, _i],
    "tn_attn_decode_multi_bf16": [_vp, _i64, _vp, _vp, _i64, _i64, _vp, _vp, _i, _i, _i, _i, _i, _f, _vp, _vp, _i64, _vp,
                                  _vp],
    "tn_kv_append_bf16": [_vp, _i64, _vp, _i64, _vp, _vp, _i64, _i64, _vp, _i, _i, _i, _i, _vp],
    "tn_greedy_select_bf16": [_vp, _i64, _i, _i, _vp, _i64, _vp, _vp, _vp, _vp, _f, _i, _i64, _i64, _vp],
    "tn_verify_select_bf16": [_vp, _i64, _i, _i, _i, _vp, _vp, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _f, _i, _i64, _i64,
                              _vp],
    "tn_greedy_select_slots_bf16": [_vp, _i64, _i, _vp, _i, _i, _vp, _i64, _vp, _vp, _vp, _vp, _vp, _f, _i, _i64, _i64,
                                    _vp],
    "tn_sample_select_slots_bf16": [_vp, _i64, _i, _vp, _vp, _i, _i, _vp, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _f, _i,
                                    _f, _i, _f, _i64, _i64, _i64, _vp],
    "tn_spec_sample_verify_bf16": [_vp, _i64, _vp, _i64, _i, _i, _i, _vp, _vp, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                   _f, _i, _f, _i, _f, _i64, _i64, _i64, _vp],
    "tn_kv_scatter_bf16": [_vp, _i64, _vp, _i64, _i64, _vp, _vp, _i64, _i64, _vp, _i, _i, _i, _i, _vp],
    "tn_slot_admit": [_vp, _i, _vp, _vp, _vp, _i64, _vp, _i64, _vp, _vp, _vp, _vp, _vp, _i, _vp],
    "tn_fbank_f32": [_vp, _i, _vp, _vp, _i, _i64, _i, _i, _i, _vp, _vp, _i, _f, _vp, _vp],
    "tn_mfcc_f32": [_vp, _i, _vp, _vp, _i, _i64, _i, _i, _i, _vp, _vp, _i, _f, _vp, _i, _vp, _vp],
    "tn_logmel_power_f32": [_vp, _i, _vp, _vp, _i, _i64, _i, _i, _i, _vp, _vp, _i, _vp, _vp, _vp],
    "tn_logmel_finish_f32": [_vp, _vp, _vp, _i, _i64, _i, _vp],
    "tn_feat_stack_f32": [_vp, _vp, _vp, _i, _i64, _i, _i, _i, _i, _vp, _vp, _i64, _vp],
    "tn_resample_f32": [_vp, _i, _vp, _vp, _vp, _vp, _i, _i64, _i, _vp, _i, _vp, _vp, _vp],
    "tn_spec_augment_f32": [_vp, _vp, _vp, _i, _i64, _i, _vp, _i, _vp, _i, _vp, _i, _vp, _vp],
    "tn_embed_add_bf16": [_vp, _vp, _i, _vp, _vp, _vp, _i64, _i, _i64, _vp],
    "tn_cast_f32_bf16": [_vp, _vp, _i64, _vp],
    "tn_bestrq_tokenize_f32": [_vp, _i64, _vp, _vp, _i64, _i, _i, _i, _vp, _vp],
    "tn_pack_ce_fwd_bf16": [_vp, _i64, _vp, _vp, _vp, _vp, _i64, _i, _vp],
    "tn_pack_ce_bwd_bf16": [_vp, _i64, _vp, _vp, _vp, _vp, _f, _i64, _i, _vp],
    "tn_pack_ce_bwd_vp_bf16": [_vp, _i64, _vp, _vp, _vp, _vp, _f, _i64, _i, _i64, _i64, _vp],
    "tn_pack_layout_i64": [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i64, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp],
    "tn_peer_reduce_scatter_f32": [_vp, _i, _i64, _vp, _i64, _f, _i, _vp],
    "tn_peer_all_gather": [_vp, _i, _i64, _vp, _i, _vp],
    "tn_reduce_bf16_to_f32": [_vp, _i, _vp, _i64, _f, _i, _vp],
    "tn_sumsq_num_partials": [],
    "tn_sumsq_f32": [_vp, _i64, _vp, _vp, _vp],
    "tn_scale_f32": [_vp, _i64, _vp, _vp],
    "tn_scale_bf16": [_vp, _i64, _vp, _vp],
    "tn_pack_ce_fused_bf16": [_vp, _i64, _vp, _vp, _vp, _vp, _vp, _f, _i64, _i, _vp],
    "tn_adamw_f32": [_vp, _vp, _vp, _vp, _vp, _i64, _f, _f, _f, _f, _f, _f, _f, _vp, _vp],
}
_RESTYPES = {"tn_last_error": c_char_p, "tn_attn_meta_ints": c_int64, "tn_attn_decode_ws_floats": c_int64,
             "tn_attn_decode_multi_ws_floats": c_int64}

EXPORTED_SYMBOLS = sorted(list(_SIGNATURES) + ["tn_last_error"])


class TouchNetB200Error(RuntimeError):
    pass


def load(path: str | None = None) -> ctypes.CDLL:
    """Load the native library (once) and attach prototypes.  Raises if it is not built."""
    global _lib
    if _lib is not None:
        return _lib
    path = path or LIB_PATH
    if not os.path.exists(path):
        raise TouchNetB200Error(
            f"{path} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(or `make -C touchnet_b200/csrc`). There is no fallback path.")
    lib = ctypes.CDLL(path)
    lib.tn_last_error.argtypes = []
    lib.tn_last_error.restype = c_char_p
    partial_ok = os.environ.get("TN_DEV_PARTIAL") == "1"  # development only: tolerate a half-built library
    for name, argtypes in _SIGNATURES.items():
        if partial_ok and not hasattr(lib, name):
            continue
        fn = getattr(lib, name)  # AttributeError if the .so does not export what the header declares
        fn.argtypes = argtypes
        fn.restype = _RESTYPES.get(name, c_int)
    _lib = lib
    return lib


# kernels launched per entry point (for bench.py's `gpu_launches` claim)
_LAUNCHES = {"tn_attn_prep": 3, "tn_attn_bwd_bf16": 3, "tn_attn_decode_bf16": 2, "tn_attn_decode_multi_bf16": 2,
             "tn_verify_select_bf16": 2, "tn_spec_sample_verify_bf16": 2, "tn_logmel_power_f32": 2,
             "tn_rmsnorm_bwd_bf16": 2, "tn_pack_layout_i64": 2}
launch_count = 0
_hooks = []   # callables(name, phase) with phase in {"pre", "post"}; bench.py uses them to time kernel classes


def call(name: str, *args) -> None:
    """Invoke an int-returning entry point; non-zero -> TouchNetB200Error(tn_last_error())."""
    global launch_count
    lib = load()
    launch_count += _LAUNCHES.get(name, 1)
    if _hooks:
        for h in _hooks:
            h(name, "pre", args)
        rc = getattr(lib, name)(*args)
        for h in _hooks:
            h(name, "post", args)
        if rc != 0:
            msg = lib.tn_last_error()
            raise TouchNetB200Error(f"{name} failed (rc={rc}): {msg.decode() if msg else '?'}")
        return
    rc = getattr(lib, name)(*args)
    if rc != 0:
        msg = lib.tn_last_error()
        raise TouchNetB200Error(f"{name} failed (rc={rc}): {msg.decode() if msg else '?'}")


def ptr(t) -> int | None:
    """Device pointer of a torch tensor (None -> NULL)."""
    return None if t is None else t.data_ptr()


def stream_handle() -> int:
    import torch

    return torch.cuda.current_stream().cuda_stream
