"""ctypes binding of libb200vlm.so (the C ABI declared in include/b200vlm.h).

The product path has NO fallback: if the CUDA library is missing or fails to
load, importing this module's `lib()` raises, and every model call fails loudly.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb200vlm.so")

OK = 0
EPI_NONE, EPI_GELU_FAST, EPI_GELU_EXACT = 0, 1, 2


class B200Error(RuntimeError):
    pass


class Qwen2VLConfig(C.Structure):
    _fields_ = [
        ("hidden", C.c_int), ("n_layers", C.c_int), ("inter", C.c_int), ("n_heads", C.c_int),
        ("n_kv_heads", C.c_int), ("head_dim", C.c_int), ("vocab", C.c_int),
        ("rms_eps", C.c_float), ("rope_theta", C.c_float), ("mrope_section", C.c_int * 3),
        ("tie_embeddings", C.c_int),
        ("v_depth", C.c_int), ("v_embed", C.c_int), ("v_heads", C.c_int), ("v_mlp", C.c_int),
        ("v_patch_dim", C.c_int), ("v_merge", C.c_int), ("v_out", C.c_int),
        ("v_ln_eps", C.c_float), ("external_vision", C.c_int),
    ]


_P, _I, _L, _F = C.c_void_p, C.c_int, C.c_long, C.c_float

# name -> (restype, argtypes); mirrors include/b200vlm.h one to one
SIGNATURES = {
    "b200_last_error": (C.c_char_p, []),
    "b200_abi_version": (_I, []),
    "b200_device_check": (_I, [_I, C.POINTER(_I)]),
    "b200_cast_f32_bf16": (_I, [_P, _P, _L, _P]),
    "b200_gemm_wt": (_I, [_P, _L, _P, _P, _P, _L, _P, _L, _P, _I, _I, _I, _I, _I, _I, _P, C.c_uint, _P]),
    "b200_gemm_wt_auto_config": (_I, [_I, _I, _I, _I, _I, _P]),
    "b200_gemm_wt_candidates": (_I, [_I, _I, _I, _I, _I, _I, _I, _L, _P, _I, _P]),
    "b200_gemm_wt_tuned": (_I, [_P, _L, _P, _P, _P, _L, _P, _L, _P, _L, _I, _I, _I, _I, _I, _I, _I, _I, _P, _P]),
    "b200_finish_rows": (_I, [_P, _I, _P, _P, _L, _P, _L, _I, _P, _P, _F, _P, _L, _I, _I, _P]),
    "b200_layer_norm": (_I, [_P, _P, _P, _P, _I, _I, _F, _P]),
    "b200_rms_norm": (_I, [_P, _P, _P, _I, _I, _F, _P]),
    "b200_vision_rope": (_I, [_P, _P, _P, _I, _I, _I, _P]),
    "b200_mrope_kv_write": (_I, [_P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _P]),
    "b200_qk_norm": (_I, [_P, _I, _I, _I, _I, _P, _P, _F, _P]),
    "b200_attention": (_I, [_P, _L, _L, _P, _L, _L, _P, _L, _L, _P, _L, _I, _I, _I, _I, _I, _I,
                            _F, _P]),
    "b200_attention_fa": (_I, [_P, _L, _L, _P, _L, _L, _P, _L, _L, _P, _L, _I, _I, _I, _I, _I, _I, _P]),
    "b200_attention_fa_seg": (_I, [_P, _L, _L, _P, _L, _L, _P, _L, _L, _P, _L] + [_I] * 10 + [_P, _I, _P]),
    "b200_vision_qkv_post": (_I, [_P, _P, _P, _I, _I, _I, _F, _P, _I, _P]),
    "b200_swiglu": (_I, [_P, _P, _I, _I, _P]),
    "b200_embed_merge": (_I, [_P, _I, _I, _P, _I, _P, _I, _I, _I, _P, _P, _P]),
    "b200_engine_create": (_I, [C.POINTER(Qwen2VLConfig), _I, C.POINTER(_P)]),
    "b200_engine_destroy": (_I, [_P]),
    "b200_engine_set_weight": (_I, [_P, C.c_char_p, _P, _L]),
    "b200_engine_workspace_bytes": (_L, [_P, _I, _I]),
    "b200_engine_set_workspace": (_I, [_P, _P, _L]),
    "b200_engine_bind_kv": (_I, [_P, _P, _I, _I]),
    "b200_engine_set_rope_tables": (_I, [_P, _P, _P]),
    "b200_engine_set_axis_sel": (_I, [_P, _P]),
    "b200_engine_vision": (_I, [_P, _P, _P, _I, _P, _P]),
    "b200_engine_prefill": (_I, [_P, _P, _P, _I, _I, _I, _P, _P]),
    "b200_engine_prefill_batch": (_I, [_P, _P, _P, _I, _P, _P, _P]),
    "b200_engine_decode": (_I, [_P, _I, _P, _P]),
    "b200_engine_set_next": (_I, [_P, _I, _I, _I, _P]),
    "b200_engine_logits": (_P, [_P]),
    "b200_engine_logprobs": (_P, [_P]),
    "b200_engine_token_log": (_P, [_P]),
    "b200_engine_token_log_capacity": (_I, [_P]),
    "b200_engine_tokens_launched": (_L, [_P]),
    "b200_engine_launch_count": (_L, [_P]),
    "b200_engine_set_graph": (_I, [_P, _I]),
    "b200_engine_set_attn_cluster": (_I, [_P, _I]),
    "b200_engine_set_pdl": (_I, [_P, _I]),
    "b200_engine_set_mega": (_I, [_P, _I]),
    "b200_engine_mega_timeline": (_I, [_P, _P]),
    "b200_engine_debug_buffer": (_I, [_P, C.c_char_p, C.POINTER(C.c_void_p), C.POINTER(C.c_long)]),
    "b200_engine_device_error": (_I, [_P, C.POINTER(_I)]),
    "b200_engine_fetch_tokens": (_I, [_P, _L, _I, _P, _P]),
    "b200_f32_layer_norm": (_I, [_P, _L, _P, _P, _F, _P, _L, _P, _L, _I, _I, _I, _P]),
    "b200_f32_rms_norm": (_I, [_P, _L, _P, _F, _P, _L, _P, _L, _I, _I, _I, _I, _I, _I, _P]),
    "b200_f32_swiglu_split": (_I, [_P, _L, _P, _L, _I, _I, _I, _P]),
    "b200_f32_split": (_I, [_P, _L, _P, _L, _I, _I, _I, _P]),
    "b200_pixel_shuffle_split": (_I, [_P, _I, _I, _I, _I, _I, _P, _L, _I, _P]),
    "b200_clip_patchify": (_I, [_P, _I, _I, _I, _I, _I, _P, _I, _P]),
    "b200_tower_embed": (_I, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _P]),
    "b200_attention_f32": (_I, [_P, _L, _L, _P, _L, _L, _P, _L, _L, _P, _L, _P, _L, _I, _I, _I, _I, _I, _I, _I, _L, _L,
                                _P, _F, _P]),
    "b200_attention_f32_varlen": (_I, [_P, _L, _L, _P, _L, _L, _P, _L, _L, _P, _L, _P, _L, _I, _I, _I, _I, _P, _I, _I, _F, _P]),
    "b200_f32_vision_rope": (_I, [_P, _L, _P, _P, _I, _I, _I, _P]),
    "b200_f32_gather_rows": (_I, [_P, _L, _P, _I, _I, _I, _P, _L, _P]),
    "b200_gemm_wt_f32": (_I, [_P, _L, _P, _L, _P, _P, _L, _P, _L, _P, _L, _I, _I, _I, _I, _I, _I, _I, _P, _P]),
    "b200_engine_set_kv_row": (_I, [_P, _I]),
    "b200_batch_begin": (_I, [_P, _I, _P, _P, _P, _P, _P]),
    "b200_batch_decode": (_I, [_P, _I, _I, _P]),
    "b200_batch_fetch": (_I, [_P, _L, _I, _P, _P, _P]),
    "b200_batch_set_procs": (_I, [_P, _P, _P, _P, _P, _I, _P, _P, _I, _I]),
    "b200_batch_fetch_topk": (_I, [_P, _L, _I, _P, _P, _P]),
    "b200_batch_procs_apply": (_I, [_P, _P, _I, _I, _I] + [_P] * 6 + [_I, _P, _P, _I, _I, _P, _P, _P]),
    "b200_batch_logits": (_P, [_P]),
    "b200_batch_logprobs": (_P, [_P]),
    "b200_batch_token_log": (_P, [_P]),
    "b200_engine_bind_kvq": (_I, [_P, _P, _P, _P, _I, _I, _I]),
    "b200_engine_set_prefill_kvq": (_I, [_P, _P, _P, _P, _I]),
    "b200_engine_bind_batch_kvq": (_I, [_P, _P, _P, _P, _I, _I, _P, _I, _I]),
    "b200_engine_set_prefill_kvq_row": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _I]),
    "b200_batch_kvq_attention": (_I, [_P] * 8 + [_I, _I, _I, _P, _I, _I, _I, _I, _P, _P, _F, _P]),
    "b200_pool_copy_row": (_I, [_P, _I, _I, _I, _P, _I, _I, _I, _I, _I, _I, _I, _P]),
    "b200_kvq_decode_attention": (_I, [_P] * 10 + [_I] * 7 + [_P]),
    "b200_kvq_quantize": (_I, [_P, _I, _P, _P, _P, _I, _L, _I, _I, _I, _P]),
    "b200_kvq_dequantize": (_I, [_P, _P, _P, _I, _P, _I, _L, _I, _I, _I, _P]),
    "b200_memcpy_d2d": (_I, [_P, _P, _L, _P]),
    "b200_engine_last_decode_ms": (_F, [_P]),
}

_lib = None


def lib() -> C.CDLL:
    """Load libb200vlm.so (once).  Raises B200Error if it is not built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise B200Error(
                f"{LIB_PATH} not found: build it with `python -m mlx_vlm_b200.build` "
                "(there is no CPU / PyTorch fallback for the generate path)")
        l = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(l, name)  # AttributeError if the .so lacks a declared symbol
            fn.restype = res
            fn.argtypes = args
        if l.b200_abi_version() != 2:
            raise B200Error("libb200vlm.so ABI version mismatch")
        _lib = l
    return _lib


def check(rc: int, what: str = "") -> None:
    if rc != OK:
        msg = lib().b200_last_error().decode(errors="replace")
        raise B200Error(f"{what or 'b200 call'} failed (code {rc}): {msg}")


def ptr(t) -> int:
    """Device/host address of a torch tensor (None -> NULL)."""
    return 0 if t is None else t.data_ptr()
