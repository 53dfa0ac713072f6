"""ctypes binding of the C ABI declared in include/sageattn_b200.h.

The library is mandatory: importing any op without libsageattn_b200.so raises — there is no CPU or
PyTorch fallback (the reference behaves the same way: `from . import _fused`, sageattention/quant.py:20).
"""
import ctypes, os
from ctypes import c_void_p, c_int, c_int64, c_float, c_char_p

_LIB_PATH = os.environ.get("SAB_LIB_PATH") or os.path.join(os.path.dirname(os.path.abspath(__file__)), "lib", "libsageattn_b200.so")

SAB_DTYPE_FP16, SAB_DTYPE_BF16 = 0, 1
SAB_GRAN_PER_BLOCK, SAB_GRAN_PER_WARP, SAB_GRAN_PER_THREAD = 1, 2, 3
SAB_MASK_BOOL, SAB_MASK_BIAS = 1, 2
SAB_SEM_CUDA, SAB_SEM_TRITON = 0, 1

EXPORTS = {
    "sab_last_error": (c_char_p, []),
    "sab_check_device": (c_int, []),
    "sab_version": (c_int, []),
    "sab_k_mean_workspace_bytes": (c_int64, [c_int] * 4),
    "sab_k_mean": (c_int, [c_void_p, c_int, c_void_p] + [c_int] * 4 + [c_int64] * 3 + [c_void_p, c_void_p]),
    "sab_quant_per_block_int8": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p] + [c_int] * 4 + [c_int64] * 6 +
                                 [c_int, c_int, c_int, c_int, c_float, c_void_p]),
    "sab_quant_per_thread_int8": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p] + [c_int] * 4 + [c_int64] * 6 +
                                  [c_int, c_int, c_void_p]),
    "sab_quant_per_block_int8_varlen": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p] +
                                        [c_int] * 4 + [c_int64] * 4 + [c_int, c_int, c_float, c_void_p]),
    "sab_per_channel_fp8_workspace_bytes": (c_int64, [c_int] * 4),
    "sab_per_channel_fp8": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p] + [c_int] * 4 + [c_int64] * 4 +
                            [c_float, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "sab_k_smooth_quant_int8": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p] + [c_int] * 4 + [c_int64] * 6 + [c_int, c_int, c_void_p]),
    "sab_per_channel_fp8_fused": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p] + [c_int] * 4 + [c_int64] * 4 + [c_float, c_void_p]),
    "sab_channel_stats": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p] + [c_int] * 4 + [c_int64] * 3 + [c_void_p, c_void_p]),
    "sab_v_quant_with_amax": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p] + [c_int] * 4 + [c_int64] * 4 +
                              [c_float, c_void_p, c_void_p]),
    "sab_v_transpose_f16": (c_int, [c_void_p, c_int, c_void_p] + [c_int] * 4 + [c_int64] * 4 + [c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "sab_qk_int8_sv_f16_attn": (c_int, [c_void_p] * 7 + [c_int] * 7 + [c_int64] * 10 + [c_int, c_int, c_int, c_float, c_int] +
                                [c_void_p] * 5 + [c_int, c_void_p]),
    "sab_qk_int8_sv_f16_attn_masked": (c_int, [c_void_p] * 7 + [c_int] * 7 + [c_int64] * 10 + [c_int, c_int, c_float, c_int] +
                                       [c_void_p, c_int] + [c_int64] * 4 + [c_void_p]),
    "sab_qk_int8_sv_f8_attn": (c_int, [c_void_p] * 9 + [c_int] * 7 + [c_int64] * 10 + [c_int, c_int, c_int, c_float, c_int] +
                               [c_void_p] * 5 + [c_int, c_int, c_int, c_void_p, c_void_p]),
    "sab_qk_int8_sv_f8_attn_sp": (c_int, [c_void_p] * 8 + [c_int] * 7 + [c_int64] * 10 + [c_int, c_int, c_float, c_int] +
                                  [c_void_p, ctypes.c_uint32, c_int, c_void_p]),
    "sab_qk_int8_sv_f8_attn_blocksparse": (c_int, [c_void_p] * 9 + [c_int] * 7 + [c_int64] * 10 + [c_int, c_int, c_int, c_float, c_int] +
                                           [c_void_p] + [c_int64] * 4 + [c_void_p]),
    "sab_qk_int8_sv_f8_attn_window": (c_int, [c_void_p] * 9 + [c_int] * 7 + [c_int64] * 10 + [c_int, c_int, c_int, c_float, c_int] +
                                      [c_int, c_int, c_void_p]),
    "sab_attn_bwd_workspace_bytes": (c_int64, [c_int] * 3),
    "sab_qk_int8_attn_bwd": (c_int, [c_void_p] * 15 + [c_int] * 7 + [c_int64] * 21 + [c_int, c_int, c_int, c_float, c_int, c_void_p]),
    "sab_qk_int8_attn_bwd_varlen": (c_int, [c_void_p] * 15 + [c_int] * 7 + [c_int64] * 14 + [c_void_p] * 4 +
                                    [c_int, c_int, c_int, c_float, c_int, c_void_p]),
    "sab_qk_int8_attn_bwd_masked": (c_int, [c_void_p] * 15 + [c_int] * 7 + [c_int64] * 21 + [c_int, c_int, c_float, c_int] +
                                    [c_void_p, c_int] + [c_int64] * 4 + [c_void_p, c_void_p]),
    "sab_qk_int8_attn_bwd_blocksparse": (c_int, [c_void_p] * 15 + [c_int] * 7 + [c_int64] * 21 + [c_int, c_int, c_int, c_float, c_int] +
                                         [c_void_p] + [c_int64] * 4 + [c_void_p]),
    "sab_qk_int8_attn_bwd_window": (c_int, [c_void_p] * 15 + [c_int] * 7 + [c_int64] * 21 + [c_int, c_int, c_int, c_float, c_int] +
                                    [c_int, c_int, c_void_p]),
    "sab_k_mean_varlen_workspace_bytes": (c_int64, [c_int] * 4),
    "sab_k_mean_varlen": (c_int, [c_void_p, c_int, c_void_p, c_void_p] + [c_int] * 4 + [c_int64] * 2 + [c_void_p, c_void_p]),
    "sab_quant_int8_varlen": (c_int, [c_void_p, c_int] + [c_void_p] * 5 + [c_int] * 4 + [c_int64] * 4 + [c_int, c_int, c_void_p]),
    "sab_per_channel_fp8_varlen_workspace_bytes": (c_int64, [c_int] * 4),
    "sab_per_channel_fp8_varlen": (c_int, [c_void_p, c_int] + [c_void_p] * 5 + [c_int] * 4 + [c_int64] * 3 +
                                   [c_float, c_void_p, c_void_p]),
    "sab_qk_int8_sv_f8_attn_varlen": (c_int, [c_void_p] * 9 + [c_int] * 7 + [c_int64] * 7 + [c_int, c_int, c_int, c_float] +
                                      [c_void_p] * 5 + [c_int, c_void_p]),
    "sab_qk_int8_attn_bwd_varlen_seq": (c_int, [c_void_p] * 15 + [c_int] * 7 + [c_int64] * 14 + [c_void_p] * 4 +
                                        [c_int] * 5 + [c_float, c_void_p]),
    "sab_qk_int8_sv_f8_attn_varlen_window": (c_int, [c_void_p] * 9 + [c_int] * 7 + [c_int64] * 7 + [c_int, c_int, c_int, c_float] +
                                             [c_void_p] * 5 + [c_int, c_int, c_int, c_void_p]),
    "sab_qk_int8_attn_bwd_varlen_window": (c_int, [c_void_p] * 15 + [c_int] * 7 + [c_int64] * 14 + [c_void_p] * 4 +
                                           [c_int] * 5 + [c_float, c_int, c_int, c_void_p]),
    "sab_qk_int8_sv_f8_attn_varlen_blocksparse": (c_int, [c_void_p] * 9 + [c_int] * 7 + [c_int64] * 7 + [c_int, c_int, c_int, c_float] +
                                                  [c_void_p] * 5 + [c_int, c_int, c_void_p] + [c_int64] * 4 + [c_void_p]),
    "sab_qk_int8_attn_bwd_varlen_blocksparse": (c_int, [c_void_p] * 15 + [c_int] * 7 + [c_int64] * 14 + [c_void_p] * 4 +
                                                [c_int] * 5 + [c_float, c_void_p] + [c_int64] * 4 + [c_void_p]),
    "sab_k_mean_paged": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int64] + [c_int] * 5 + [c_int64] * 3 +
                         [c_void_p, c_void_p]),
    "sab_quant_int8_paged": (c_int, [c_void_p, c_int] + [c_void_p] * 6 + [c_int64] + [c_int] * 5 + [c_int64] * 5 + [c_int, c_void_p]),
    "sab_per_channel_fp8_paged": (c_int, [c_void_p, c_int] + [c_void_p] * 6 + [c_int64] + [c_int] * 5 + [c_int64] * 4 +
                                  [c_float, c_void_p, c_void_p]),
    "sab_qk_int8_sv_f8_attn_varlen_bottom_right": (c_int, [c_void_p] * 9 + [c_int] * 7 + [c_int64] * 7 + [c_int, c_int, c_int, c_float] +
                                                   [c_void_p] * 5 + [c_int, c_void_p]),
    "sab_kvcache8_chunk_keys": (c_int, []),
    "sab_kvcache8_workspace_bytes": (c_int64, [c_int] * 3 + [c_int64]),
    "sab_kvcache8_write": (c_int, [c_void_p] * 2 + [c_int] + [c_void_p] * 2 + [c_int] * 3 + [c_int64] * 4 + [c_void_p] * 4 +
                           [c_int64, c_int, c_void_p]),
    "sab_kvcache8_attn": (c_int, [c_void_p, c_int] + [c_void_p] * 10 + [c_int64] + [c_int] * 7 + [c_int64] * 4 +
                          [c_int, c_int, c_float, c_void_p, c_void_p]),
    "sab_kvcache8_prefill": (c_int, [c_void_p, c_int] + [c_void_p] * 10 + [c_int64] + [c_int] * 7 + [c_int64] * 4 +
                             [c_int, c_int, c_float, c_void_p]),
    "sab_kvcache8_attn_window": (c_int, [c_void_p, c_int] + [c_void_p] * 10 + [c_int64] + [c_int] * 7 + [c_int64] * 4 +
                                 [c_int, c_int, c_float, c_void_p, c_int, c_int, c_void_p]),
    "sab_kvcache8_prefill_window": (c_int, [c_void_p, c_int] + [c_void_p] * 10 + [c_int64] + [c_int] * 7 + [c_int64] * 4 +
                                    [c_int, c_int, c_float, c_int, c_int, c_void_p]),
    "sab_kvcache8_attn_shared": (c_int, [c_void_p, c_int] + [c_void_p] * 10 + [c_int64] + [c_int] * 7 + [c_int64] * 4 +
                                 [c_int, c_int, c_float, c_void_p, c_int, c_void_p]),
    "sab_block_stats": (c_int, [c_void_p, c_int, c_void_p, c_void_p] + [c_int] * 4 + [c_int64] * 3 + [c_int, c_void_p]),
    "sab_predict_block_mask": (c_int, [c_void_p] * 5 + [c_int] * 7 + [c_float] * 3 + [c_void_p]),
    "sab_block_stats_varlen": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p] + [c_int] * 4 + [c_int64] * 2 + [c_int, c_void_p]),
    "sab_predict_block_mask_varlen": (c_int, [c_void_p] * 7 + [c_int] * 7 + [c_float] * 3 + [c_void_p]),
}

_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            raise ImportError(
                f"sageattention_b200: {_LIB_PATH} is missing. Build it with `python -m sageattention_b200.build` "
                "(nvcc, sm_90a). There is no fallback implementation.")
        _lib = ctypes.CDLL(_LIB_PATH)
        for name, (res, args) in EXPORTS.items():
            fn = getattr(_lib, name)
            fn.restype, fn.argtypes = res, args
    return _lib


class SabError(RuntimeError):
    pass


def check(status: int):
    if status != 0:
        msg = lib().sab_last_error().decode("utf-8", "replace")
        if status in (-1,):
            raise ValueError(msg)
        raise SabError(f"sageattn_b200 error {status}: {msg}")
