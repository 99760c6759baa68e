"""ctypes binding of the C-ABI CUDA library (include/dolomite_b200.h).

The product path has NO fallback: if the shared library is missing or a kernel returns an error, a
`DolomiteB200Error` is raised.  Nothing here imports or calls the oracle.
"""

from __future__ import annotations

import ctypes
import os
from ctypes import c_char_p, c_float, c_int, c_int64, c_uint32, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libdolomite_b200.so")


class DolomiteB200Error(RuntimeError):
    pass


_P = c_void_p
_I = c_int
_L = c_int64
_F = c_float
_U = c_uint32

# name -> (restype, argtypes).  Must list every symbol include/dolomite_b200.h declares
# (tests/test_abi.py cross-checks this table against the header).
SIGNATURES: dict[str, tuple] = {
    "dolomite_b200_last_error": (c_char_p, []),
    "dolomite_b200_abi_version": (_I, []),
    "dolomite_b200_device_info": (_I, [_P, _P, _P]),
    "dolomite_b200_set_option": (_I, [c_char_p, _I]),
    "dolomite_b200_get_option": (_I, [c_char_p, _P]),
    "dolomite_b200_rmsnorm_fwd": (_I, [_P, _P, _P, _P, _L, _I, _F, _P]),
    "dolomite_b200_rmsnorm_bwd_workspace_bytes": (_L, [_I]),
    "dolomite_b200_rmsnorm_bwd": (_I, [_P, _P, _P, _P, _P, _P, _P, _P, _L, _I, _P]),
    "dolomite_b200_rope_qk_inplace": (_I, [_P, _L, _L, _I, _I, _I, _P, _P, _P, _I, _L, _I, _P]),
    "dolomite_b200_layernorm_fwd": (_I, [_P, _P, _P, _P, _P, _P, _L, _I, _F, _P]),
    "dolomite_b200_layernorm_bwd_workspace_bytes": (_L, [_I]),
    "dolomite_b200_layernorm_bwd": (_I, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _L, _I, _P]),
    "dolomite_b200_act_fwd": (_I, [_I, _I, _P, _P, _L, _L, _P]),
    "dolomite_b200_act_bwd": (_I, [_I, _I, _P, _P, _P, _P, _L, _L, _P]),
    "dolomite_b200_act_bwd_segmented": (_I, [_I, _I, _P, _P, _P, _P, _L, _L, _P, _I, _P]),
    "dolomite_b200_gelu_fwd": (_I, [_P, _P, _L, _P]),
    "dolomite_b200_gelu_bwd": (_I, [_P, _P, _P, _P, _L, _L, _P]),
    "dolomite_b200_swiglu_fwd": (_I, [_P, _P, _L, _L, _P]),
    "dolomite_b200_swiglu_bwd": (_I, [_P, _P, _P, _L, _L, _P]),
    "dolomite_b200_swiglu_bwd_bias": (_I, [_P, _P, _P, _P, _L, _L, _P]),
    "dolomite_b200_embedding_fwd": (_I, [_P, _P, _P, _L, _I, _L, _F, _P]),
    "dolomite_b200_embedding_bwd": (_I, [_P, _P, _P, _L, _I, _L, _F, _P]),
    "dolomite_b200_embedding_fwd_neft": (_I, [_P, _P, _P, _L, _I, _L, _U, _U, _F, _P]),
    "dolomite_b200_cross_entropy_fwd_bwd": (_I, [_P, _L, _P, _P, _P, _P, _P, _L, _L, _L, _F, _F, _P]),
    "dolomite_b200_cross_entropy_count": (_I, [_P, _L, _L, _P, _P]),
    "dolomite_b200_cross_entropy_rows": (_I, [_P, _L, _P, _P, _P, _P, _L, _L, _L, _F, _F, _P]),
    "dolomite_b200_cross_entropy_mean": (_I, [_P, _L, _P, _P, _P]),
    "dolomite_b200_colsum_accum": (_I, [_P, _L, _P, _L, _L, _F, _P]),
    "dolomite_b200_colsum_accum_segmented": (_I, [_P, _L, _P, _L, _L, _P, _I, _F, _P]),
    "dolomite_b200_scale_bf16_by_device_scalar": (_I, [_P, _L, _P, _P]),
    "dolomite_b200_add_scaled": (_I, [_P, _P, _P, _F, _L, _P]),
    "dolomite_b200_dropout_fwd": (_I, [_P, _P, _P, _L, _F, _F, _U, _U, _P]),
    "dolomite_b200_dropout_bwd": (_I, [_P, _P, _L, _F, _F, _U, _U, _P]),
    "dolomite_b200_sumsq_workspace_bytes": (_L, []),
    "dolomite_b200_sumsq_accum": (_I, [_P, _L, _P, _P, _P]),
    "dolomite_b200_clip_coef": (_I, [_P, _F, _P, _P, _P]),
    "dolomite_b200_adamw_step": (_I, [_P, _P, _P, _P, _P, _L, _F, _F, _F, _F, _F, _L, _P, _P]),
    "dolomite_b200_cast_f32_to_bf16": (_I, [_P, _P, _L, _P]),
    "dolomite_b200_accum_bf16_into_f32": (_I, [_P, _P, _F, _L, _P]),
    "dolomite_b200_gemm_bf16": (
        _I,
        [_P, _L, _I, _P, _L, _I, _P, _L, _I, _P, _L, _F, _F, _P, _L, _L, _L, _I, _P],
    ),
    "dolomite_b200_gemm_bf16_wgrad_multi": (_I, [_I, _P, _P, _P, _P, _P, _P, _P, _P, _L, _P, _P, _P]),
    "dolomite_b200_gemm_bf16_tile_n": (_I, [_I, _P, _P, _P, _P]),
    "dolomite_b200_gemm_fp8": (
        _I,
        [_P, _L, _I, _P, _L, _I, _P, _P, _P, _L, _I, _P, _L, _F, _F, _P, _L, _L, _L, _I, _P],
    ),
    "dolomite_b200_gemm_fp8_wgrad_multi": (
        _I,
        [_I, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _L, _P, _P, _I, _I, _I, _P],
    ),
    "dolomite_b200_fp8_cast": (_I, [_P, _L, _L, _L, _I, _P, _P, _P, _P, _P]),
    "dolomite_b200_fp8_scaling_update": (_I, [_P, _I, _L, _P, _P, _F, _P]),
    "dolomite_b200_gemm_bf16_grouped_m": (_I, [_P, _L, _P, _L, _I, _P, _L, _F, _L, _L, _L, _P, _I, _I, _P]),
    "dolomite_b200_gemm_bf16_grouped_k": (_I, [_P, _L, _P, _L, _P, _L, _F, _F, _L, _L, _L, _P, _I, _P]),
    "dolomite_b200_moe_max_rows": (_L, [_L, _I, _I]),
    "dolomite_b200_moe_route": (_I, [_P, _L, _I, _I, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "dolomite_b200_gemm_bf16_grouped_m_gather": (_I, [_P, _L, _L, _P, _P, _L, _P, _L, _F, _L, _L, _L, _P, _I, _I, _P]),
    "dolomite_b200_gemm_bf16_grouped_m_bias": (
        _I,
        [_P, _L, _L, _P, _P, _L, _I, _P, _L, _P, _L, _F, _L, _L, _L, _P, _I, _I, _P],
    ),
    "dolomite_b200_moe_gather": (_I, [_P, _P, _P, _P, _L, _I, _I, _I, _P]),
    "dolomite_b200_moe_combine": (_I, [_P, _P, _P, _P, _P, _L, _I, _I, _F, _P]),
    "dolomite_b200_moe_combine_bwd": (_I, [_P, _P, _P, _P, _P, _P, _P, _L, _I, _I, _I, _F, _P]),
    "dolomite_b200_moe_token_sum": (_I, [_P, _P, _P, _L, _I, _I, _P]),
    "dolomite_b200_moe_router_bwd": (_I, [_P, _P, _P, _P, _L, _I, _I, _P]),
    "dolomite_b200_moe_aux_partial_floats": (_L, [_L, _I]),
    "dolomite_b200_moe_aux_stats": (_I, [_P, _P, _L, _L, _I, _I, _P, _P, _P]),
    "dolomite_b200_moe_aux_finalize": (_I, [_P, _I, _L, _F, _P, _P, _P, _P]),
    "dolomite_b200_moe_router_bwd_aux": (_I, [_P, _P, _P, _P, _P, _P, _P, _L, _L, _I, _I, _P]),
    "dolomite_b200_attn_varlen_fwd": (_I, [_P, _L, _P, _P, _P, _I, _L, _I, _I, _I, _I, _F, _P]),
    "dolomite_b200_attn_decode": (_I, [_P, _L, _P, _P, _P, _P, _I, _L, _I, _I, _I, _F, _P]),
    "dolomite_b200_attn_varlen_bwd_workspace_bytes": (_L, [_L, _I, _I, _I]),
    "dolomite_b200_attn_varlen_bwd": (
        _I,
        [_P, _P, _L, _P, _P, _P, _P, _I, _L, _I, _I, _I, _I, _F, _P, _P],
    ),
    "dolomite_b200_attn_varlen_fwd_dropout": (_I, [_P, _L, _P, _P, _P, _I, _L, _I, _I, _I, _I, _F, _F, _U, _U, _P]),
    "dolomite_b200_attn_varlen_bwd_dropout": (
        _I,
        [_P, _P, _L, _P, _P, _P, _P, _I, _L, _I, _I, _I, _I, _F, _F, _U, _U, _P, _P],
    ),
    "dolomite_b200_attn_varlen_fwd_alibi": (_I, [_P, _L, _P, _P, _P, _I, _L, _I, _I, _I, _I, _F, _F, _U, _U, _P, _P]),
    "dolomite_b200_attn_varlen_bwd_alibi": (
        _I,
        [_P, _P, _L, _P, _P, _P, _P, _I, _L, _I, _I, _I, _I, _F, _F, _U, _U, _P, _P, _P],
    ),
    "dolomite_b200_attn_decode_alibi": (_I, [_P, _L, _P, _P, _P, _P, _I, _L, _I, _I, _I, _F, _P, _P]),
    "dolomite_b200_attn_cache": (_I, [_P, _L, _P, _P, _P, _P, _P, _I, _I, _I, _L, _I, _I, _I, _F, _P]),
    "dolomite_b200_attn_cache_alibi": (_I, [_P, _L, _P, _P, _P, _P, _P, _I, _I, _I, _L, _I, _I, _I, _F, _P, _P]),
}

_lib = None


def lib_available() -> bool:
    return os.path.exists(LIB_PATH)


def load():
    """Load the shared library (once) and attach signatures.  Raises if it is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise DolomiteB200Error(
            f"{LIB_PATH} not found. Build it with `python -m dolomite_engine_b200.build` "
            "(or __graft_entry__.build()); there is no CPU / PyTorch fallback for the hot path."
        )
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    # DOLO_OPTIONS="key=value,key=value": tuning knobs of dolomite_b200_set_option applied at load (A/B runs of bench.py)
    for item in filter(None, os.environ.get("DOLO_OPTIONS", "").split(",")):
        key, _, value = item.partition("=")
        if lib.dolomite_b200_set_option(key.strip().encode(), int(value)) != 0:
            raise DolomiteB200Error(f"DOLO_OPTIONS: {lib.dolomite_b200_last_error().decode()}")
    return lib


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = load().dolomite_b200_last_error()
        raise DolomiteB200Error(f"{what}: rc={rc}: {msg.decode() if msg else '?'}")


# kernels launched per successful call of each entry point (for bench.py's `gpu_launches` accounting)
KERNELS_PER_CALL = {
    "dolomite_b200_rmsnorm_fwd": 1, "dolomite_b200_rmsnorm_bwd": 2, "dolomite_b200_rope_qk_inplace": 1,
    "dolomite_b200_layernorm_fwd": 1, "dolomite_b200_layernorm_bwd": 3, "dolomite_b200_gelu_fwd": 1,
    "dolomite_b200_gelu_bwd": 1, "dolomite_b200_swiglu_fwd": 1, "dolomite_b200_swiglu_bwd": 1, "dolomite_b200_swiglu_bwd_bias": 1,
    "dolomite_b200_act_fwd": 1, "dolomite_b200_act_bwd": 1,
    "dolomite_b200_embedding_fwd": 1, "dolomite_b200_embedding_fwd_neft": 1,
    "dolomite_b200_embedding_bwd": 1, "dolomite_b200_cross_entropy_fwd_bwd": 3, "dolomite_b200_colsum_accum": 1,
    "dolomite_b200_scale_bf16_by_device_scalar": 1, "dolomite_b200_add_scaled": 1, "dolomite_b200_sumsq_accum": 2,
    "dolomite_b200_clip_coef": 1, "dolomite_b200_adamw_step": 1, "dolomite_b200_cast_f32_to_bf16": 1,
    "dolomite_b200_accum_bf16_into_f32": 1, "dolomite_b200_gemm_bf16": 1, "dolomite_b200_attn_varlen_fwd": 1,
    "dolomite_b200_attn_varlen_bwd": 3, "dolomite_b200_attn_varlen_fwd_dropout": 1, "dolomite_b200_attn_varlen_bwd_dropout": 3,
    "dolomite_b200_attn_varlen_fwd_alibi": 1, "dolomite_b200_attn_varlen_bwd_alibi": 3, "dolomite_b200_attn_decode_alibi": 1,
    "dolomite_b200_dropout_fwd": 1, "dolomite_b200_dropout_bwd": 1, "dolomite_b200_gemm_bf16_tile_n": 0,
    "dolomite_b200_moe_aux_stats": 2,
}
launch_counts: dict[str, int] = {}


def reset_launch_counts() -> None:
    launch_counts.clear()


def total_kernel_launches() -> int:
    return sum(KERNELS_PER_CALL.get(k, 1) * v for k, v in launch_counts.items())


def call(name: str, *args):
    """Call an int-status entry point and raise on failure."""
    lib = load()
    launch_counts[name] = launch_counts.get(name, 0) + 1
    rc = getattr(lib, name)(*args)
    if rc != 0:
        msg = lib.dolomite_b200_last_error()
        raise DolomiteB200Error(f"{name} failed (rc={rc}): {msg.decode() if msg else '?'}")
