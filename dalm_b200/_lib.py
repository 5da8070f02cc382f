"""ctypes binding of libdalm_b200.so (the C ABI declared in include/dalm_b200.h).

There is no CPU or PyTorch fallback: if the shared library is missing, or a kernel is invoked without an sm_90
device, this module raises.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import c_char_p, c_float, c_int, c_longlong, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libdalm_b200.so")

from ctypes import c_ulonglong

_I, _L, _F, _P, _U = c_int, c_longlong, c_float, c_void_p, c_ulonglong
_DROP = [_F, _U, _U, _P]          # drop_p, drop_seed, drop_stream_id, drop_offset

# name -> argtypes (restype is int unless listed in _RESTYPES). Mirrors include/dalm_b200.h one to one.
SIGNATURES = {
    "dalm_b200_last_error": [],
    "dalm_b200_version": [],
    "dalm_b200_launch_count": [],
    "dalm_b200_reset_launch_count": [],
    "dalm_b200_probe_device": [],
    "dalm_b200_marginal_counts": [_P, _P, _I, _I, _P, _P, _P],
    "dalm_b200_inbatch_loss_fwd_bwd": [_P, _P, _I, _I, _F, _P, _P, _P, _P, _P, _P, _P, _F, _P],
    "dalm_b200_ce_marginal_fwd_bwd": [_P, _P, _I, _P, _P, _P, _P, _I, _I, _I, _L, _F, _P],
    "dalm_b200_ce_marginal_rows": [_P, _P, _I, _P, _P, _P, _P, _I, _I, _I, _L, _F, _I, _I, _P],
    "dalm_b200_finalize_loss": [_P, _P, _I, _I, _P, _P, _P, _P],
    "dalm_b200_bump_counter": [_P, _P],
    "dalm_b200_dropout_scale": [_P, _L, _F, _U, _U, _P, _P],
    "dalm_b200_lora_dx": [_P, _L, _P, _L, _P, _L, _I, _I, _I, _F, _U, _U, _P, _P],
    "dalm_b200_small_matmul_f32": [_P, _P, _P, _I, _I, _I, _I, _I, _F, _P],
    "dalm_b200_gemm_bf16": [_I, _P, _L, _P, _L, _P, _L, _I, _I, _I, _I, _F, _P, _I, _P, _L, _I, _I, _I, *_DROP, _P],
    "dalm_b200_gemm_clear_cache": [],
    "dalm_b200_gemm_set_raster": [_I],
    "dalm_b200_gemm_set_l2_hints": [_I],
    "dalm_b200_attention_fwd": [_P, _L, _P, _L, _P, _L, _P, _P, _L, _P, _I, _I, _I, _I, _I, _F, _I, _I, *_DROP, _P],
    "dalm_b200_attention_tc_fwd": [_P, _L, _P, _L, _P, _L, _P, _P, _L, _P, _I, _I, _I, _I, _I, _F, _I, _I, *_DROP, _P],
    "dalm_b200_attention_tc_bwd": [_P, _L, _P, _L, _P, _L, _P, _P, _L, _P, _P, _L, _P, _P, _L, _P, _L, _P, _L,
                                   _I, _I, _I, _I, _I, _F, _I, _I, *_DROP, _P],
    "dalm_b200_attention_bwd": [_P, _L, _P, _L, _P, _L, _P, _P, _L, _P, _P, _L, _P, _P, _L, _P, _L, _P, _L,
                                _I, _I, _I, _I, _I, _F, _I, _I, *_DROP, _P],
    "dalm_b200_layernorm_fwd": [_P, _P, _P, _P, _P, _L, _P, _P, _I, _I, _F, *_DROP, _P],
    "dalm_b200_layernorm_bwd": [_P, _P, _P, _P, _P, _P, _L, _P, _P, _L, _I, _I, *_DROP, _P],
    "dalm_b200_layernorm_bwd_res": [_P, _P, _P, _P, _P, _P, _L, _P, _P, _P, _L, _I, _I, _P],
    "dalm_b200_rmsnorm_fwd": [_P, _P, _P, _L, _P, _I, _I, _F, _P],
    "dalm_b200_rmsnorm_bwd": [_P, _P, _P, _P, _L, _P, _P, _P, _L, _I, _I, _P],
    "dalm_b200_bert_embed": [_P, _P, _P, _P, _P, _I, _I, _I, _I, _P],
    "dalm_b200_roberta_embed": [_P, _P, _P, _P, _I, _P, _P, _I, _I, _I, _I, _I, _P],
    "dalm_b200_embed_gather": [_P, _P, _P, _I, _I, _I, _P],
    "dalm_b200_rope": [_P, _L, _I, _I, _I, _P, _P, _I, _I, _I, _P],
    "dalm_b200_swiglu_fwd": [_P, _L, _P, _L, _I, _I, _I, _P],
    "dalm_b200_swiglu_bwd": [_P, _L, _P, _L, _I, _I, _I, _P],
    "dalm_b200_geglu_fwd": [_P, _L, _P, _L, _I, _I, _P],
    "dalm_b200_geglu_bwd": [_P, _L, _P, _L, _I, _I, _P],
    "dalm_b200_gemm_bf16_swiglu": [_P, _L, _P, _L, _P, _L, _P, _L, _I, _I, _I, _P],
    "dalm_b200_gemm_bf16_rope": [_P, _L, _P, _L, _P, _L, _I, _I, _I, _P, _P, _P, _I, _I, _P, _P, _I, _F, _P, _L, _P, _L, _P],
    "dalm_b200_gemm_bf16_gelu": [_P, _L, _P, _L, _P, _L, _P, _L, _I, _I, _I, _P, _P],
    "dalm_b200_gelu_fwd": [_P, _L, _P, _L, _I, _I, _P],
    "dalm_b200_gelu_bwd": [_P, _L, _P, _L, _I, _I, _P],
    "dalm_b200_pool_norm_fwd": [_P, _P, _P, _P, _P, _I, _I, _I, _I, _P],
    "dalm_b200_pool_norm_bwd": [_P, _P, _P, _P, _P, _I, _I, _I, _I, _P],
    "dalm_b200_lora_wgrad": [_P, _L, _P, _L, _P, _P, _L, _L, _I, _I, _I, _F, *_DROP, _P],
    "dalm_b200_skinny_gemm": [_P, _L, _P, _L, _P, _L, _I, _I, _I, *_DROP, _P],
    "dalm_b200_pack_scaled_bf16": [_P, _L, _L, _P, _L, _I, _I, _F, _P],
    "dalm_b200_pack_table": [_P, _I, _P],
    "dalm_b200_cast_f32_bf16": [_P, _L, _P, _L, _I, _I, _P],
    "dalm_b200_adam_step": [_P, _P, _P, _P, _L, _F, _F, _F, _F, _I, _F, _P],
    "dalm_b200_col_reduce": [_P, _P, _L, _P, _P, _P, _P, _P, _I, _I, _P],
    "dalm_b200_embed_scatter_add": [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _P],
    "dalm_b200_masked_add": [_P, _P, _L, _P, _I, _I, *_DROP, _P],
    "dalm_b200_adam_step_shadow": [_P, _P, _P, _P, _P, _L, _F, _F, _F, _F, _I, _F, _P],
    "dalm_b200_topk_ip_workspace": [_I, _I],
    "dalm_b200_topk_ip": [_P, _P, _L, _I, _I, _I, _I, _P, _P, _P, _P],
    "dalm_b200_nf4_roundtrip": [_P, _L, _P, _P, _P],
    "dalm_b200_nf4_quantize": [_P, _L, _P, _P, _P],
    "dalm_b200_nf4_dequant_bf16": [_P, _P, _L, _I, _P, _L, _P, _L, _I, _P],
    "dalm_b200_decode_gemm": [_P, _L, _P, _L, _P, _L, _I, _P, _P, _L, _I, _I, _I, _I, _I, _P],
    "dalm_b200_rope_pos": [_P, _L, _I, _I, _I, _P, _P, _P, _I, _I, _P],
    "dalm_b200_qk_norm_rope": [_P, _L, _I, _I, _P, _P, _F, _P, _P, _I, _I, _P, _I, _P, _L, _P, _L, _P],
    "dalm_b200_qk_norm_rope_bwd": [_P, _L, _I, _I, _P, _P, _P, _P, _I, _P, _L, _P, _L, _I, _P, _P, _P],
    "dalm_b200_attention_decode": [_P, _L, _I, _I, _I, _P, _P, _L, _L, _P, _L, _P, _L, _I, _I, _I, _I, _I, _P, _I, _F, _I, _P],
    "dalm_b200_greedy_step": [_P, _L, _I, _I, _P, _I, _L, _P, _P, _L, _P, _L, _I, _P, _I, _P, _P, _P, _P],
    "dalm_b200_sample_step": [_P, _L, _I, _I, _P, _I, _L, _P, _P, _L, _P, _L, _I, _P, _I, _P, _P, _P, _F, _I, _F, _U, _P, _P, _P],
    "dalm_b200_gemm_bf16_grouped": [_I, _I, _P, _L, _P, _I, _P, _L, _P, _L, _I, _I, _I, _P, _P, _I, _P],
    "dalm_b200_moe_router": [_P, _L, _I, _I, _I, _I, _P, _P, _P],
    "dalm_b200_moe_router_bwd": [_P, _L, _P, _P, _P, _I, _I, _I, _I, _P, _L, _P],
    "dalm_b200_moe_permute": [_P, _I, _I, _I, _P, _P, _P, _P, _P, _P, _P, _P],
    "dalm_b200_moe_gather": [_P, _L, _I, _I, _P, _I, _P, _I, _P, _L, _P],
    "dalm_b200_moe_combine": [_P, _L, _P, _P, _I, _I, _I, _P, _L, _P, _L, _I, _P],
    "dalm_b200_moe_down_bwd": [_P, _L, _P, _L, _P, _P, _I, _I, _P, _P, _L, _P],
}
_RESTYPES = {
    "dalm_b200_last_error": c_char_p,
    "dalm_b200_version": c_char_p,
    "dalm_b200_launch_count": c_longlong,
    "dalm_b200_topk_ip_workspace": c_longlong,
    "dalm_b200_reset_launch_count": None,
    "dalm_b200_gemm_clear_cache": None,
    "dalm_b200_gemm_set_raster": None,
    "dalm_b200_gemm_set_l2_hints": None,
}

_lib = None


class DalmB200Error(RuntimeError):
    pass


def load() -> ctypes.CDLL:
    """Load the shared library (once). Raises if it has not been built: there is no fallback path."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise DalmB200Error(
            f"{LIB_PATH} is missing. Build it with `python -m dalm_b200.csrc.build` (needs nvcc); "
            "dalm_b200 has no CPU / PyTorch fallback for its kernels."
        )
    lib = ctypes.CDLL(LIB_PATH)
    for name, argtypes in SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError here == header/library drift
        fn.argtypes = argtypes
        fn.restype = _RESTYPES.get(name, c_int)
    _lib = lib
    return lib


def call(name: str, *args) -> None:
    """Invoke an int-returning entry point; raise with the library's message on failure."""
    lib = load()
    rc = getattr(lib, name)(*args)
    if rc != 0:
        msg = lib.dalm_b200_last_error()
        raise DalmB200Error(f"{name} failed (rc={rc}): {msg.decode() if msg else '?'}")


def launch_count() -> int:
    return int(load().dalm_b200_launch_count())


def reset_launch_count() -> None:
    load().dalm_b200_reset_launch_count()


def version() -> str:
    return load().dalm_b200_version().decode()
