"""ctypes binding of libb200nlp.so (the C-ABI declared in include/b200nlp.h).

There is deliberately NO fallback: if the shared library is missing or a kernel launch fails, the call raises.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import c_char_p, c_float, c_int, c_int64, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libb200nlp.so")

_lib = None

P = c_void_p
I64 = c_int64
I = c_int
F = c_float

# name -> argtypes; every function returns int unless listed in _RESTYPE.
_SIGNATURES = {
    "b200_last_error": [],
    "b200_abi_version": [],
    "b200_device_check": [],
    "b200_set_pdl": [I],
    "b200_set_fa_fwd_impl": [I],
    "b200_set_fa_bwd_impl": [I],
    "b200_gemm_bf16": [P, P, P, P, I64, I64, I64, I64, I64, I64, I, I, I, P],
    "b200_gemm_bf16_ex": [P, P, P, P, P, I64, I64, I64, I64, I64, I64, I64, I, I, I, I, P],
    "b200_gemm_bf16_f32": [P, P, P, I64, I64, I64, I64, I64, I64, I, I, I, P],
    "b200_gemm_swiglu_bf16": [P, P, P, P, I64, I64, I64, I64, I64, I64, I64, P],
    "b200_gemm_swiglu_bwd_bf16": [P, P, P, P, I64, I64, I64, I64, I64, I64, I64, P],
    "b200_gemm_splitk_workspace_bytes": [I64, I64],
    "b200_gemm_bf16_splitk": [P, P, P, P, P, I64, I64, I64, I64, I64, I64, I, I, I, P],
    "b200_weight_quantize_int8": [P, P, P, I64, I64, I64, P],
    "b200_weight_only_gemm_bf16": [P, P, P, P, P, P, I64, I64, I64, I64, I64, I, P],
    "b200_weight_only_gemm_f32": [P, P, P, P, I64, I64, I64, I64, I, P],
    "b200_rmsnorm_fwd": [P, P, P, P, I64, I64, F, P],
    "b200_rmsnorm_bwd_workspace_bytes": [I64, I64],
    "b200_rmsnorm_bwd": [P, P, P, P, P, P, P, I, P, I64, I64, P],
    "b200_rmsnorm_bwd_f32": [P, P, P, P, P, P, P, I, P, I64, I64, P],
    "b200_colsum_workspace_bytes": [I64, I64],
    "b200_colsum_bf16": [P, P, I, P, I64, I64, I64, P],
    "b200_colsum_f32": [P, P, I, P, I64, I64, I64, P],
    "b200_rope_inplace": [P, P, P, P, I64, I64, I64, I64, I64, I, P],
    "b200_swiglu_fwd": [P, P, I64, I64, P],
    "b200_swiglu_fwd_f32": [P, P, I64, I64, P],
    "b200_swiglu_bwd": [P, P, P, I64, I64, P],
    "b200_embedding_fwd": [P, P, P, I64, I64, I64, P],
    "b200_embedding_bwd": [P, P, P, I64, I64, I64, P],
    "b200_embedding_bwd_f32": [P, P, P, I64, I64, I64, P],
    "b200_fa_fwd": [P, P, P, P, P, I64, I64, I64, I64, I64, I64, I64, I64, I64, F, P],
    "b200_fa_fwd_flashmask": [P, P, P, P, P, P, I64, I64, I64, I64, I64, I64, I64, I64, I64, F, P],
    "b200_fa_bwd_flashmask": [P, P, P, P, P, P, P, P, P, P, P, I64, I64, I64, I64, I64, I64, I64, I64, I64, I64, I64, I64, I64, F, P],
    "b200_fa_bwd_workspace_bytes": [I64, I64, I64, I64],
    "b200_fa_bwd": [P, P, P, P, P, P, P, P, P, P, I64, I64, I64, I64, I64, I64, I64, I64, I64, I64, I64, I64, I64, F, P],
    "b200_ce_fwd": [P, P, P, P, P, I64, I64, I64, I64, P],
    "b200_ce_bwd": [P, P, P, P, P, F, P, I64, I64, I64, P],
    "b200_ce_rows_fwd": [P, P, P, P, I64, I64, I64, I64, I64, P],
    "b200_ce_reduce": [P, P, I64, P],
    "b200_argmax_bf16": [P, P, I64, I64, I64, P],
    "b200_grad_sqnorm_workspace_bytes": [],
    "b200_grad_sqnorm": [P, P, P, I64, F, P],
    "b200_adamw_step": [P, P, P, P, P, P, I64, I64, F, F, F, F, F, I64, F, F, P],
    "b200_grad_sqnorm_f32": [P, P, P, I64, F, P],
    "b200_adamw_step_f32": [P, P, P, P, P, P, I64, I64, F, F, F, F, F, I64, F, F, P],
    "b200_bf16_to_f32": [P, P, I64, P],
    "b200_add_rmsnorm": [P, P, P, P, P, I64, I64, F, P],
    "b200_add_rmsnorm_f32": [P, P, P, P, P, I64, I64, F, P],
    "b200_decode_rope_append_f32": [P, P, P, P, P, P, P, I64, I64, I64, I64, I64, I64, P],
    "b200_write_cache_kv": [P, P, P, I64, I64, I64, I64, I64, I64, I64, P],
    "b200_decode_rope_append": [P, P, P, P, P, I64, I64, I64, I64, I64, I64, P],
    "b200_decode_attention_workspace_bytes": [I64, I64, I64],
    "b200_decode_attention": [P, P, P, P, P, I64, I64, I64, I64, I64, I64, F, I64, P],
    "b200_write_cache_kv_paged": [P, P, P, P, P, I64, I64, I64, I64, I64, I64, I64, I64, P],
    "b200_decode_rope_append_paged": [P, P, P, P, P, P, P, P, P, I64, I64, I64, I64, I64, I64, I64, P],
    "b200_decode_attention_paged": [P, P, P, P, P, P, P, I64, I64, I64, I64, I64, I64, I64, I64, F, I64, P],
    "b200_softmax_f32": [P, I64, I64, I64, P],
    "b200_top_p_sampling_reject": [P, P, P, P, I64, I64, I64, I64, P],
    "b200_decode_attention_tc": [P, P, P, P, P, I64, I64, I64, I64, I64, I64, F, I64, P],
    "b200_get_padding_offset": [P, P, P, P, P, P, P, P, I64, I64, P],
    "b200_rebuild_padding": [P, P, P, P, P, I64, I64, I64, P],
    "b200_set_value_by_flags_and_idx": [P, P, P, P, I64, I64, P],
    "b200_set_value_by_flags_and_idx_v2": [P, P, P, P, P, P, I64, I64, I64, P],
    "b200_token_penalty_multi_scores": [P, P, P, P, P, P, P, P, P, P, P, I64, I64, I64, I64, I64, P],
    "b200_set_stop_value_multi_ends": [P, P, P, P, P, I64, I64, I, P],
    "b200_fused_get_rotary_embedding": [P, P, I64, I64, I64, I64, I64, F, I, P],
    "b200_step_paddle": [P] * 21 + [I64] * 6 + [P],
    "b200_retire_admit": [P] * 27 + [I64] * 9 + [P],
    "b200_save_output_stream": [P, P, P, I64, I64, P, I64, I64, P],
    "b200_append_attention_workspace_bytes": [I64, I64, I64, I64, I64],
    "b200_append_attention": [P] * 12 + [I64] * 12 + [F, I64, P],
    "b200_write_cache_kv_paged_c8": [P] * 7 + [I64] * 8 + [P],
    "b200_decode_rope_append_paged_c8": [P] * 11 + [I64] * 7 + [P],
    "b200_decode_attention_paged_c8": [P] * 9 + [I64] * 8 + [F, I64, P],
    "b200_append_attention_c8": [P] * 16 + [I64] * 12 + [F, I64, P],
    "b200_update_inputs": [P, P, P, P, P, P, P, P, P, I64, I64, I64, P],
    "b200_generate_step_update": [P, P, P, P, P, P, I64, P, I64, P, I64, I64, P, P, I64, P],
    "b200_argmax_f32": [P, P, I64, I64, I64, P],
    "b200_bf16_rows_to_f32": [P, P, I64, I64, I64, P],
}
_RESTYPE = {
    "b200_last_error": c_char_p,
    "b200_rmsnorm_bwd_workspace_bytes": c_int64,
    "b200_gemm_splitk_workspace_bytes": c_int64,
    "b200_decode_attention_workspace_bytes": c_int64,
    "b200_colsum_workspace_bytes": c_int64,
    "b200_fa_bwd_workspace_bytes": c_int64,
    "b200_append_attention_workspace_bytes": c_int64,
    "b200_grad_sqnorm_workspace_bytes": c_int64,
}


def exported_symbols():
    """Names include/b200nlp.h declares (kept in sync by tests/test_abi.py)."""
    return sorted(_SIGNATURES)


def load():
    """Load the library (building it first if it is absent and nvcc is available)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        from . import build as _build

        _build.build()
    lib = ctypes.CDLL(LIB_PATH)
    for name, argtypes in _SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the .so does not export a declared symbol
        fn.argtypes = argtypes
        fn.restype = _RESTYPE.get(name, c_int)
    _lib = lib
    return lib


class B200Error(RuntimeError):
    pass


# CUDA kernels each entry point launches (used by bench.py to report `gpu_launches`; memsets are not counted).
KERNELS_PER_CALL = {
    "b200_gemm_bf16": 1, "b200_gemm_bf16_ex": 1, "b200_gemm_bf16_splitk": 2, "b200_rmsnorm_fwd": 1, "b200_rmsnorm_bwd": 2, "b200_rmsnorm_bwd_f32": 2, "b200_colsum_bf16": 2, "b200_colsum_f32": 2,
    "b200_rope_inplace": 1, "b200_swiglu_fwd": 1, "b200_swiglu_bwd": 1, "b200_embedding_fwd": 1, "b200_embedding_bwd": 1,
    "b200_fa_fwd": 1, "b200_fa_bwd": 5, "b200_fa_fwd_flashmask": 1, "b200_fa_bwd_flashmask": 5, "b200_ce_fwd": 2, "b200_ce_bwd": 1, "b200_ce_rows_fwd": 1, "b200_ce_reduce": 1, "b200_argmax_bf16": 1, "b200_grad_sqnorm": 2, "b200_grad_sqnorm_f32": 2,
    "b200_adamw_step": 1, "b200_bf16_to_f32": 1, "b200_token_penalty_multi_scores": 2, "b200_generate_step_update": 2, "b200_decode_attention": 2, "b200_decode_attention_tc": 2, "b200_decode_attention_paged": 2, "b200_append_attention": 5,
    "b200_decode_attention_paged_c8": 2, "b200_append_attention_c8": 5,
}
launch_count = 0       # kernels launched through this module since import
call_hook = None       # optional callable(name, args) -> context manager, used by bench.py to time one kernel family


def call(name, *args):
    """Call an int-returning entry point; raise B200Error with the library's message on failure."""
    global launch_count
    lib = load()
    launch_count += KERNELS_PER_CALL.get(name, 1)
    if call_hook is not None:
        with call_hook(name, args):
            rc = getattr(lib, name)(*args)
    else:
        rc = getattr(lib, name)(*args)
    if rc != 0:
        msg = lib.b200_last_error()
        raise B200Error(f"{name} failed (rc={rc}): {msg.decode() if msg else '?'}")
    return rc


def ptr(t):
    """Device pointer of a torch tensor (or None)."""
    if t is None:
        return None
    return c_void_p(t.data_ptr())


def stream_ptr():
    import torch

    return c_void_p(torch.cuda.current_stream().cuda_stream)
