"""ctypes binding of include/tce_b200.h.  Fails loudly when the CUDA library is missing."""
from __future__ import annotations

import ctypes as C
from pathlib import Path

from .build import LIB

_lib = None


class TceError(RuntimeError):
    pass


class W4Tensor(C.Structure):
    _fields_ = [("w", C.c_void_p), ("zeros", C.c_void_p), ("scales", C.c_void_p), ("oc", C.c_int), ("ic", C.c_int)]


class LlamaLayer(C.Structure):
    _fields_ = [(n, W4Tensor) for n in ("q", "k", "v", "o", "gate", "up", "down")] + [("input_norm", C.c_void_p), ("post_norm", C.c_void_p)]


class LlamaConfig(C.Structure):
    _fields_ = [(n, C.c_int) for n in ("num_layers", "num_heads", "num_kv_heads", "head_dim", "embed_dim", "hidden_dim", "vocab_size", "max_ctx")] + [
        ("rms_eps", C.c_float), ("rope_theta", C.c_float), ("qk_alpha", C.c_float), ("tp_rank", C.c_int), ("tp_size", C.c_int)]


class LlamaWeights(C.Structure):
    _fields_ = [("embed_f16", C.c_void_p), ("layers", C.POINTER(LlamaLayer)), ("final_norm", C.c_void_p), ("lm_head", W4Tensor),
                ("rope_cos", C.c_void_p), ("rope_sin", C.c_void_p)]


class Sampling(C.Structure):
    """tce_sampling (include/tce_b200.h): the sampling fields of the reference's opt_params (llm/include/Generate.h:48-72)."""
    _fields_ = [("top_k", C.c_int), ("top_p", C.c_float), ("temp", C.c_float), ("repeat_penalty", C.c_float), ("frequency_penalty", C.c_float),
                ("presence_penalty", C.c_float), ("repeat_last_n", C.c_int), ("seed", C.c_ulonglong)]


class GenRequest(C.Structure):
    """tce_gen_request (include/tce_b200.h): one sequence of tce_llama_generate_batch."""
    _fields_ = [("first_token", C.c_int), ("pos0", C.c_int), ("slot", C.c_int), ("n_predict", C.c_int), ("eos_id", C.c_int),
                ("history", C.POINTER(C.c_int)), ("n_history", C.c_int), ("sampling", Sampling)]


class Lookup(C.Structure):
    """tce_lookup (include/tce_b200.h): the prompt-lookup drafter of tce_llama_generate_lookup."""
    _fields_ = [("max_draft", C.c_int), ("ngram_min", C.c_int), ("ngram_max", C.c_int)]


class LookupStats(C.Structure):
    """tce_lookup_stats (include/tce_b200.h)."""
    _fields_ = [("steps", C.c_int), ("drafted", C.c_int), ("accepted", C.c_int)]


# every symbol include/tce_b200.h declares (tests/test_capi_symbols.py checks header <-> library <-> this table)
SIGNATURES = {
    "tce_version": (C.c_int, []),
    "tce_last_error": (C.c_char_p, []),
    "tce_ctx_create": (C.c_int, [C.c_int, C.POINTER(C.c_void_p)]),
    "tce_ctx_destroy": (C.c_int, [C.c_void_p]),
    "tce_ctx_set_stream": (C.c_int, [C.c_void_p, C.c_void_p]),
    "tce_ctx_synchronize": (C.c_int, [C.c_void_p]),
    "tce_ctx_set_option": (C.c_int, [C.c_void_p, C.c_char_p, C.c_int]),
    "tce_ctx_num_sms": (C.c_int, [C.c_void_p]),
    "tce_ctx_read_gemv_timing": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int]),
    "tce_zeros_width": (C.c_int, [C.c_int, C.c_int]),
    "tce_w4a16_gemv": (C.c_int, [C.c_void_p] * 6 + [C.c_int] * 4),
    "tce_w4a16_gemm": (C.c_int, [C.c_void_p] * 6 + [C.c_int] * 4),
    "tce_naive_fp16_int4": (C.c_int, [C.c_void_p] * 5 + [C.c_int] * 4),
    "tce_f32_matmul_transposed": (C.c_int, [C.c_void_p] * 4 + [C.c_int] * 3),
    "tce_w8a8_matmul": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                  C.c_float, C.c_float, C.c_int, C.c_int]),
    "tce_opt_int8_attention": (C.c_int, [C.c_void_p] * 6 + [C.c_longlong] + [C.c_void_p] * 2 + [C.c_longlong, C.c_void_p, C.c_float, C.c_float] + [C.c_int] * 4 + [C.c_void_p]),
    "tce_attn_prefill": (C.c_int, [C.c_void_p] * 7 + [C.c_float] + [C.c_int] * 6),
    "tce_attn_decode": (C.c_int, [C.c_void_p] * 8 + [C.c_float] + [C.c_int] * 4),
    "tce_attn_span": (C.c_int, [C.c_void_p] * 7 + [C.c_float] + [C.c_int] * 6),
    "tce_rmsnorm_f16": (C.c_int, [C.c_void_p] * 4 + [C.c_int, C.c_int, C.c_float]),
    "tce_argmax_f32": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    "tce_layernorm_q": (C.c_int, [C.c_void_p] * 5 + [C.c_int, C.c_int]),
    "tce_add_f32": (C.c_int, [C.c_void_p] * 4 + [C.c_longlong]),
    "tce_llama_create": (C.c_int, [C.c_void_p, C.POINTER(LlamaConfig), C.POINTER(LlamaWeights), C.POINTER(C.c_void_p)]),
    "tce_llama_destroy": (C.c_int, [C.c_void_p]),
    "tce_llama_load_dir": (C.c_int, [C.c_void_p, C.c_char_p, C.POINTER(LlamaConfig), C.POINTER(C.c_void_p)]),
    "tce_w4_import_x86": (C.c_int, [C.c_void_p] * 2 + [C.c_int] * 2 + [C.c_void_p] * 3),
    "tce_llama_decode": (C.c_int, [C.c_void_p, C.c_void_p]),
    "tce_llama_decode_host": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.POINTER(C.c_int)]),
    "tce_llama_prefill": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "tce_sample": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.POINTER(Sampling), C.c_ulonglong, C.POINTER(C.c_int), C.c_void_p, C.c_void_p,
                             C.POINTER(C.c_int)]),
    "tce_llama_generate": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.POINTER(Sampling), C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.POINTER(C.c_int)]),
    "tce_llama_reserve_slots": (C.c_int, [C.c_void_p, C.c_int]),
    "tce_llama_kv_cache_slot": (C.c_void_p, [C.c_void_p, C.c_int, C.c_int, C.c_int]),
    "tce_llama_prefill_slot": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "tce_llama_decode_batch": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p]),
    "tce_llama_decode_batch_host": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "tce_llama_prefill_batch": (C.c_int, [C.c_void_p, C.c_int] + [C.c_void_p] * 6),
    "tce_llama_score_batch": (C.c_int, [C.c_void_p, C.c_int] + [C.c_void_p] * 9),
    "tce_llama_generate_batch": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(GenRequest), C.c_void_p, C.c_int, C.c_void_p]),
    "tce_llama_kv_copy": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "tce_llama_decode_span_host": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "tce_llama_generate_lookup": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.POINTER(Sampling), C.c_void_p, C.c_int, C.c_void_p, C.c_int,
                                            C.POINTER(Lookup), C.c_int, C.c_void_p, C.POINTER(C.c_int), C.POINTER(LookupStats)]),
    "tce_llama_sample_lookup": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.POINTER(Sampling), C.c_void_p, C.c_int, C.c_void_p, C.c_int,
                                          C.POINTER(Lookup), C.c_int, C.c_void_p, C.POINTER(C.c_int), C.POINTER(LookupStats)]),
    "tce_spec_accept": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_longlong, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.POINTER(Sampling),
                                  C.c_ulonglong, C.c_int, C.c_int, C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_void_p]),
    "tce_llama_batch_logits": (C.c_void_p, [C.c_void_p]),
    "tce_llama_logits": (C.c_void_p, [C.c_void_p]),
    "tce_llama_kv_cache": (C.c_void_p, [C.c_void_p, C.c_int, C.c_int]),
    "tce_llama_kernels_per_step": (C.c_int, [C.c_void_p]),
    "tce_llama_tp_handle": (C.c_int, [C.c_void_p, C.c_void_p]),
    "tce_llama_tp_connect": (C.c_int, [C.c_void_p, C.c_void_p]),
    "tce_llama_debug_buffer": (C.c_void_p, [C.c_void_p, C.c_int]),
    "tce_llama_enqueue_gemvs": (C.c_int, [C.c_void_p]),
}


def lib() -> C.CDLL:
    """Load lib/libtce_b200.so.  No fallback: a missing library is an error, not a slow path."""
    global _lib
    if _lib is None:
        if not Path(LIB).exists():
            raise TceError(f"{LIB} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` (nvcc, sm_90a). "
                           "tinychatengine_b200 has no CPU fallback.")
        L = C.CDLL(str(LIB))
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        raise TceError(f"{what} failed ({rc}): {lib().tce_last_error().decode()}")
