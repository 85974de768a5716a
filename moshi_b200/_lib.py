"""ctypes binding of ``include/moshi_b200.h``.

There is no CPU fallback: if the sm_90a library has not been built, importing a model class raises
with the build command.  ``__graft_entry__.build()`` / ``python -m moshi_b200.build`` produce it
in-tree (``moshi_b200/_C/libmoshi_b200.so``).
"""
from __future__ import annotations

import ctypes as C
import typing as tp
from pathlib import Path

LIB_PATH = Path(__file__).resolve().parent / "_C" / "libmoshi_b200.so"

B200_OK, B200_ERR_INVALID, B200_ERR_SHAPE, B200_ERR_STATE, B200_ERR_CUDA, B200_ERR_MISSING = range(6)
B200_F32, B200_BF16, B200_F16, B200_I64, B200_U8, B200_I8, B200_I32 = range(7)
B200_DEPFORMER_AUTO, B200_DEPFORMER_CHAIN, B200_DEPFORMER_FUSED = range(3)     # b200_lm_set_depformer
ABI_VERSION = 2


class MimiConfigC(C.Structure):
    _fields_ = [
        ("sample_rate", C.c_int), ("frame_rate", C.c_float), ("channels", C.c_int),
        ("dimension", C.c_int), ("n_filters", C.c_int), ("n_residual_layers", C.c_int),
        ("n_ratios", C.c_int), ("ratios", C.c_int * 8),
        ("kernel_size", C.c_int), ("residual_kernel_size", C.c_int), ("last_kernel_size", C.c_int),
        ("dilation_base", C.c_int), ("compress", C.c_int),
        ("tr_d_model", C.c_int), ("tr_num_heads", C.c_int), ("tr_num_layers", C.c_int),
        ("tr_dim_feedforward", C.c_int), ("tr_context", C.c_int), ("tr_max_period", C.c_float),
        ("q_dimension", C.c_int), ("q_bins", C.c_int), ("q_n_q", C.c_int), ("q_n_semantic", C.c_int),
        ("num_codebooks", C.c_int),
    ]


class RowSamplingC(C.Structure):
    """``b200_row_sampling``: one session's sampling settings."""
    _fields_ = [("temp_text", C.c_float), ("temp", C.c_float), ("top_k_text", C.c_int32), ("top_k", C.c_int32),
                ("pad_mult", C.c_float), ("repetition_context", C.c_int32), ("repetition_penalty", C.c_float)]


class LMConfigC(C.Structure):
    _fields_ = [
        ("dim", C.c_int), ("text_card", C.c_int), ("n_q", C.c_int), ("dep_q", C.c_int), ("card", C.c_int),
        ("num_heads", C.c_int), ("num_layers", C.c_int), ("ffn_hidden", C.c_int), ("context", C.c_int),
        ("max_period", C.c_float), ("depformer_dim", C.c_int), ("depformer_num_heads", C.c_int),
        ("depformer_num_layers", C.c_int), ("depformer_ffn_hidden", C.c_int), ("delays", C.c_int * 33),
        ("quantize", C.c_int), ("extra_heads_num_heads", C.c_int), ("extra_heads_dim", C.c_int),
    ]


_P = C.c_void_p
_I = C.c_int
_PROTOTYPES: dict[str, tuple[tp.Any, list]] = {
    "b200_last_error": (C.c_char_p, []),
    "b200_abi_version": (_I, []),
    "b200_launch_count": (C.c_int64, []),
    # Mimi
    "b200_mimi_create": (_I, [C.POINTER(MimiConfigC), C.POINTER(_P)]),
    "b200_mimi_load_tensor": (_I, [_P, C.c_char_p, _P, _I, _I, C.POINTER(C.c_int64)]),
    "b200_mimi_finalize": (_I, [_P]),
    "b200_mimi_destroy": (_I, [_P]),
    "b200_mimi_set_num_codebooks": (_I, [_P, _I]),
    "b200_mimi_streaming_begin": (_I, [_P, _I, _P]),
    "b200_mimi_streaming_end": (_I, [_P]),
    "b200_mimi_reset": (_I, [_P, _P]),
    "b200_mimi_set_exec_mask": (_I, [_P, _P]),
    "b200_mimi_encode": (_I, [_P, _P, _I, _P]),
    "b200_mimi_encode_to_latent": (_I, [_P, _P, _I, _P]),
    "b200_mimi_quantize": (_I, [_P, _P, _I, _P]),
    "b200_mimi_decode": (_I, [_P, _P, _I, _I, _P]),
    "b200_mimi_decode_latent": (_I, [_P, _P, _I, _I, _P]),
    "b200_mimi_encode_host": (_I, [_P, _P, _I, _P]),
    "b200_mimi_decode_host": (_I, [_P, _P, _I, _I, _P]),
    "b200_mimi_set_graph": (_I, [_P, _I]),
    "b200_mimi_state_bytes": (C.c_int64, [_P]),
    "b200_mimi_get_state": (_I, [_P, _P, C.c_int64]),
    "b200_mimi_set_state": (_I, [_P, _P, C.c_int64]),
    "b200_mimi_state_count": (_I, [_P]),
    "b200_mimi_state_entry": (_I, [_P, _I, C.POINTER(C.c_char_p), C.POINTER(_I), C.POINTER(_I), C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "b200_mimi_state_read": (_I, [_P, C.c_char_p, _P, C.c_int64]),
    "b200_mimi_state_write": (_I, [_P, C.c_char_p, _P, C.c_int64]),
    "b200_mimi_session_bytes": (_I, [_P, C.POINTER(C.c_int64)]),
    "b200_mimi_session_export": (_I, [_P, _I, _P, C.c_int64]),
    "b200_mimi_session_import": (_I, [_P, _I, _P, C.c_int64]),
    "b200_mimi_error_flags": (_I, [_P, C.POINTER(_I)]),
    "b200_mimi_read_buffer": (_I, [_P, C.c_char_p, _P, C.c_int64, C.POINTER(C.c_int64)]),
    "b200_mimi_algorithmic_bytes": (C.c_int64, [_P]),
    # LM
    "b200_lm_create": (_I, [C.POINTER(LMConfigC), C.POINTER(_P)]),
    "b200_lm_load_tensor": (_I, [_P, C.c_char_p, _P, _I, _I, C.POINTER(C.c_int64)]),
    "b200_lm_finalize": (_I, [_P]),
    "b200_lm_destroy": (_I, [_P]),
    "b200_lm_set_sampling": (_I, [_P, _I, C.c_float, C.c_float, _I, _I]),
    "b200_lm_set_session_sampling": (_I, [_P, _I]),
    "b200_lm_set_row_sampling": (_I, [_P, _P, _I, _P]),
    "b200_lm_streaming_begin": (_I, [_P, _I, _P]),
    "b200_lm_streaming_end": (_I, [_P]),
    "b200_lm_reset": (_I, [_P, _P]),
    "b200_lm_set_exec_mask": (_I, [_P, _P]),
    "b200_lm_noise_per_row": (_I, [_P]),
    "b200_lm_step": (_I, [_P, _P, _I, _P, _P, _I, C.POINTER(_I)]),
    "b200_lm_step_ex": (_I, [_P, _P, _I, _P, _P, _P, _I, C.POINTER(_I)]),
    "b200_lm_step_host": (_I, [_P, _P, _I, _P, _P, _I, C.POINTER(_I)]),
    "b200_lm_state_bytes": (C.c_int64, [_P]),
    "b200_lm_get_state": (_I, [_P, _P, C.c_int64]),
    "b200_lm_set_state": (_I, [_P, _P, C.c_int64]),
    "b200_lm_read_buffer": (_I, [_P, C.c_char_p, _P, C.c_int64, C.POINTER(C.c_int64)]),
    "b200_lm_set_taps": (_I, [_P, _I]),
    "b200_lm_algorithmic_bytes": (C.c_int64, [_P, _I]),
    "b200_lm_assume_fill": (_I, [_P, _I]),
    "b200_lm_set_graph": (_I, [_P, _I]),
    "b200_lm_set_depformer": (_I, [_P, _I]),
    "b200_lm_set_kv_dtype": (_I, [_P, _I]),
    "b200_lm_set_kv_capacity": (_I, [_P, _I]),
    "b200_lm_set_kv_pool": (_I, [_P, C.c_int64, _I]),
    "b200_lm_kv_pool_usage": (_I, [_P, C.POINTER(_I), C.POINTER(_I)]),
    "b200_lm_session_bytes": (_I, [_P, _I, C.POINTER(C.c_int64)]),
    "b200_lm_session_export": (_I, [_P, _I, _P, C.c_int64]),
    "b200_lm_session_import": (_I, [_P, _I, _P, C.c_int64]),
    "b200_lm_set_cfg": (_I, [_P, C.c_float, _I, _P, _I]),
    "b200_lm_set_condition_sum": (_I, [_P, _P, _I]),
    "b200_lm_set_cross_attention": (_I, [_P, _I]),
    "b200_lm_set_depformer_schedule": (_I, [_P, C.POINTER(_I), _I]),
    "b200_lm_set_depformer_low_rank": (_I, [_P, _I]),
    "b200_lm_set_cross_len": (_I, [_P, _I]),
    "b200_lm_set_condition_cross": (_I, [_P, _P, _P, _I]),
    "b200_lm_seed_noise": (_I, [_P, C.c_uint64]),
    "b200_lm_set_stream": (_I, [_P, _P]),
    "b200_lm_state_count": (_I, [_P]),
    "b200_lm_state_entry": (_I, [_P, _I, C.POINTER(C.c_char_p), C.POINTER(_I), C.POINTER(_I), C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "b200_lm_state_read": (_I, [_P, C.c_char_p, _P, C.c_int64]),
    "b200_lm_state_write": (_I, [_P, C.c_char_p, _P, C.c_int64]),
    "b200_lm_get_offset_cpu": (C.c_int64, [_P]),
    "b200_lm_set_offset_cpu": (_I, [_P, C.c_int64]),
    "b200_lm_error_flags": (_I, [_P, C.POINTER(_I)]),
    # one frame for every session slot, host buffers
    "b200_frame_create": (_I, [_P, _P, _I, _I, _I, _I, _P, C.POINTER(_P)]),
    "b200_frame_destroy": (_I, [_P]),
    "b200_frame_step": (_I, [_P, _P, _P, _P, _P, _P, _P, _P]),
    "b200_frame_read_buffer": (_I, [_P, C.c_char_p, _P, C.c_int64, C.POINTER(C.c_int64)]),
    # batched speech-to-text service
    "b200_asr_create": (_I, [_P, _P, _I, _I, _P, C.POINTER(_P)]),
    "b200_asr_destroy": (_I, [_P]),
    "b200_asr_step": (_I, [_P, _P, _P, _P, _P, _P, C.POINTER(_I)]),
    "b200_asr_read_buffer": (_I, [_P, C.c_char_p, _P, C.c_int64, C.POINTER(C.c_int64)]),
    # kernel-level
    "b200_op_linear_bf16": (_I, [_P, _P, _P, _I, _I, _I, _P]),
    "b200_op_packed_bytes": (C.c_int64, [_I, _I, _I, _I]),
    "b200_op_pack_tiles": (_I, [_P, _P, _I, _I, _I, _I, _P]),
    "b200_op_linear_sk": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _P]),
    "b200_op_linear_ns": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _P]),
    "b200_op_set_gemv_max_rows": (_I, [_I]),
    "b200_op_linear_plan": (_I, [_I, _I, _I, _I, _I, _I, _I, _I, _I, C.POINTER(C.c_int64), _I]),
    "b200_op_depformer_plan": (_I, [_I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, C.POINTER(C.c_int64), _I]),
    "b200_op_mimi_plan": (_I, [C.POINTER(MimiConfigC), _I, _I, _I, C.POINTER(C.c_int64), _I]),
    "b200_op_packed_bytes_i8": (C.c_int64, [_I, _I, _I, _I]),
    "b200_op_quant_pack_tiles": (_I, [_P, _P, _P, _I, _I, _I, _I, _P]),
    "b200_op_quantize_rows": (_I, [_P, _P, _P, _I, _I, _P]),
    "b200_op_linear_i8": (_I, [_P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _P]),
    "b200_op_conv1d": (_I, [_P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _P]),
    "b200_op_tc_linear_f32": (_I, [_P, _P, _P, _I, _I, _I, _P]),
    "b200_op_tc_conv1d": (_I, [_P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _P]),
    "b200_op_attn_step": (_I, [_P, _P, _P, _P, _P, _P, _I, _I, _I, _I, C.c_float, _P]),
    "b200_op_attn_step_paged": (_I, [_P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, C.c_float, _P]),
    "b200_op_attn_step_q8": (_I, [_P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, C.c_float, _I, _P]),
    "b200_op_dep_attn_step": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _P]),
    "b200_op_mimi_ring_attn": (_I, [_P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, C.c_float, _P]),
    "b200_op_rmsnorm": (_I, [_P, _P, _P, _I, _I, _P]),
    "b200_op_layernorm": (_I, [_P, _P, _P, _P, _I, _I, _P]),
    "b200_op_cross_attn_step": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _P]),
    "b200_op_linear_sk_norm": (_I, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _P]),
    "b200_op_sample": (_I, [_P, _P, _P, _I, _I, _I, C.c_float, _I, _P]),
    "b200_op_lm_noise": (_I, [_P, C.c_int64, C.c_uint64, C.c_uint64, _P]),
    "b200_op_sample_text_rows": (_I, [_P, _P, C.c_int64, _P, _I, _I, _I, C.c_float, _I, _P, _P, _P, _I, _P]),
    "b200_op_exp1": (_I, [_P, _P, C.c_int64, _P]),
}

EXPORTED_SYMBOLS = tuple(_PROTOTYPES)

_lib: C.CDLL | None = None


class B200Error(RuntimeError):
    def __init__(self, code: int, message: str):
        super().__init__(f"[b200 rc={code}] {message}")
        self.code = code


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not LIB_PATH.exists():
            raise RuntimeError(
                f"{LIB_PATH} is missing: the GPU path has no CPU fallback. Build it with "
                "`python -m moshi_b200.build` (needs nvcc; cross-compiles for sm_90a).")
        handle = C.CDLL(str(LIB_PATH))
        for name, (res, args) in _PROTOTYPES.items():
            fn = getattr(handle, name)
            fn.restype = res
            fn.argtypes = args
        if handle.b200_abi_version() != ABI_VERSION:
            raise RuntimeError("libmoshi_b200.so ABI version mismatch; rebuild")
        _lib = handle
    return _lib


def check(rc: int) -> None:
    """Maps return codes to the exception types the reference raises on this path."""
    if rc == B200_OK:
        return
    msg = lib().b200_last_error().decode("utf-8", "replace")
    if rc == B200_ERR_SHAPE:
        raise AssertionError(msg)          # reference: shape asserts (lm.py:679-686)
    if rc == B200_ERR_INVALID:
        raise ValueError(msg)
    raise B200Error(rc, msg)               # RuntimeError subclass (lm.py:673-676, compression.py:361-365)


_DTYPES = None


def dtype_code(t) -> int:
    global _DTYPES
    if _DTYPES is None:
        import torch
        _DTYPES = {torch.float32: B200_F32, torch.bfloat16: B200_BF16, torch.float16: B200_F16,
                   torch.int64: B200_I64, torch.uint8: B200_U8, torch.bool: B200_U8, torch.int8: B200_I8,
                   torch.int32: B200_I32}
    return _DTYPES[t]


def ptr(t) -> C.c_void_p:
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def current_stream(device) -> C.c_void_p:
    import torch
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)
