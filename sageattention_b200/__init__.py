"""sageattention_b200 — H100-native (sm_90a) drop-in for the thu-ml/SageAttention operator API.

Exports the reference's public names (sageattention/__init__.py:1-5)."""
from .core import (sageattn, sageattn_varlen, sageattn_qk_int8_pv_fp16_triton, sageattn_qk_int8_pv_fp16_cuda,
                   sageattn_qk_int8_pv_fp8_cuda, sageattn_qk_int8_pv_fp8_cuda_sm90, sageattn_blocksparse,
                   sageattn_window, sageattn_varlen_qk_int8_pv_fp8_cuda, sageattn_varlen_window,
                   sageattn_varlen_blocksparse, sageattn_varlen_kvcache)
from .quant import per_block_int8, per_warp_int8, per_thread_int8, per_channel_fp8, k_mean, transpose_v_f16
# beyond the reference surface (pre-quantised K/V and the host-buffer end-to-end call)
from .cache import QuantizedKV, quantize_kv, sageattn_prequantized
from .host import sageattn_host
from .predict import predict_block_mask, predict_block_mask_varlen
from .kvcache8 import PagedKVCache8, sageattn_kvcache8, sageattn_kvcache8_prefill

__all__ = ["sageattn", "sageattn_varlen", "sageattn_qk_int8_pv_fp16_triton", "sageattn_qk_int8_pv_fp16_cuda",
           "sageattn_qk_int8_pv_fp8_cuda", "sageattn_qk_int8_pv_fp8_cuda_sm90", "sageattn_blocksparse", "sageattn_window",
           "sageattn_varlen_qk_int8_pv_fp8_cuda", "sageattn_varlen_window", "sageattn_varlen_blocksparse",
           "sageattn_varlen_kvcache",
           "per_block_int8", "per_warp_int8", "per_thread_int8", "per_channel_fp8", "k_mean", "transpose_v_f16",
           "QuantizedKV", "quantize_kv", "sageattn_prequantized", "sageattn_host", "predict_block_mask",
           "predict_block_mask_varlen", "PagedKVCache8", "sageattn_kvcache8", "sageattn_kvcache8_prefill"]
