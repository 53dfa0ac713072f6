"""Pre-quantised K/V for repeated attention calls ("accept pre-quantised/cached K,V across diffusion
steps or decode steps").

`sageattn_qk_int8_pv_fp8_cuda` (sageattention/core.py:636-826) re-derives the K mean, the INT8 K and the FP8 V^T on every
call.  When K and V do not change between calls (cross-attention to a fixed context, several query chunks against one
KV, repeated denoising steps of a cached block) that front-end is 2/3 of the quantisation work and four of the eight
launches.  `quantize_kv` runs it once; `sageattn_prequantized` quantises only Q and launches the attention kernel.
The result is bit-identical to the one-shot call with the same options — same kernels, same order of operations.
"""
from dataclasses import dataclass
from typing import Optional
import warnings
import torch
import torch.nn.functional as F

from . import ops
from ._capi import SAB_GRAN_PER_WARP, SAB_GRAN_PER_THREAD
from .quant import k_mean, quant_q_int8, quant_k_int8, smooth_quant_k, per_channel_fp8

_LOG2E = 1.44269504


def _padded_head_dim(d: int) -> int:
    """sageattention/core.py:752-761."""
    if d > 128:
        raise ValueError(f"Unsupported head_dim: {d}")
    return 64 if d <= 64 else 128


@dataclass
class QuantizedKV:
    """INT8 K (+ scales, + the mean that was subtracted) and FP8 V^T (+ per-channel scales) of one K/V pair."""
    k_int8: torch.Tensor
    k_scale: torch.Tensor
    v_fp8: torch.Tensor
    v_scale: torch.Tensor
    v_mean: Optional[torch.Tensor]
    km: Optional[torch.Tensor]          # [B,Hkv,1,D] / [B,1,Hkv,D] in the input dtype, None without smooth_k
    tensor_layout: str
    qk_quant_gran: str
    pv_accum_dtype: str
    head_dim_og: int
    dtype: torch.dtype

    @property
    def kv_len(self) -> int:
        return self.k_int8.size(1 if self.tensor_layout == "NHD" else 2)

    def nbytes(self) -> int:
        ts = [self.k_int8, self.k_scale, self.v_fp8, self.v_scale, self.v_mean, self.km]
        return sum(t.numel() * t.element_size() for t in ts if t is not None)


def quantize_kv(k: torch.Tensor, v: torch.Tensor, tensor_layout: str = "HND", qk_quant_gran: str = "per_thread",
                pv_accum_dtype: str = "fp32+fp16", smooth_k: bool = True, smooth_v: bool = False) -> QuantizedKV:
    """K/V half of sageattn_qk_int8_pv_fp8_cuda (core.py:745-815): K mean, INT8 K, FP8 V^T — 5 launches, done once."""
    assert k.is_cuda and k.device == v.device, "Input tensors must be on the same cuda device."
    assert k.dtype in [torch.float16, torch.bfloat16] and k.dtype == v.dtype, "k, v must both be fp16 or bf16"
    assert qk_quant_gran in ["per_warp", "per_thread"], "qk_quant_gran must be either 'per_warp' or 'per_thread'."
    if pv_accum_dtype not in ("fp32", "fp32+fp32", "fp32+fp16"):
        raise ValueError(f"Unsupported pv_accum_dtype: {pv_accum_dtype}")
    if tensor_layout not in ("NHD", "HND"):
        raise ValueError(f"Unknown tensor layout: {tensor_layout}")
    head_dim_og = k.size(-1)
    pad = _padded_head_dim(head_dim_og) - head_dim_og
    if pad:
        k, v = F.pad(k, (0, pad)), F.pad(v, (0, pad))
    assert k.stride(-1) == 1 and v.stride(-1) == 1, "Last dim of k, v must be contiguous."
    km = k_mean(k, tensor_layout) if smooth_k else None
    k_int8, k_scale = quant_k_int8(k, km, qk_quant_gran, tensor_layout)
    if pv_accum_dtype in ("fp32+fp32", "fp32+fp16") and smooth_v:
        warnings.warn(f"pv_accum_dtype is '{pv_accum_dtype}', smooth_v will be ignored.")
        smooth_v = False
    scale_max = 2.25 if pv_accum_dtype == "fp32+fp16" else 448.0
    v_fp8, v_scale, vm = per_channel_fp8(v, tensor_layout=tensor_layout, scale_max=scale_max, smooth_v=smooth_v)
    return QuantizedKV(k_int8, k_scale, v_fp8, v_scale, vm, km, tensor_layout, qk_quant_gran, pv_accum_dtype,
                       head_dim_og, k.dtype)


def sageattn_prequantized(q: torch.Tensor, kv: QuantizedKV, is_causal: bool = False, sm_scale: Optional[float] = None,
                          return_lse: bool = False):
    """Attention of `q` against a `QuantizedKV`: quantise Q (1 launch) + the fused kernel.  Same result, bit for bit,
    as sageattn_qk_int8_pv_fp8_cuda(q, k, v, ...) with the options given to quantize_kv."""
    assert q.is_cuda and q.device == kv.k_int8.device, "q must be on the device of the cached K/V."
    assert q.dtype == kv.dtype, "q must have the dtype K/V were quantised from."
    assert q.size(-1) == kv.head_dim_og, "head_dim of q differs from the cached K/V."
    lay = 0 if kv.tensor_layout == "NHD" else 1
    pad = _padded_head_dim(kv.head_dim_og) - kv.head_dim_og
    if pad:
        q = F.pad(q, (0, pad))
    assert q.stride(-1) == 1, "Last dim of q must be contiguous."
    if is_causal:
        assert q.size(1 if lay == 0 else 2) == kv.kv_len, "qo_len and kv_len must be equal for causal attention."
    if sm_scale is None:
        sm_scale = kv.head_dim_og ** -0.5
    q_int8, q_scale = quant_q_int8(q, kv.qk_quant_gran, kv.tensor_layout)
    gran = SAB_GRAN_PER_WARP if kv.qk_quant_gran == "per_warp" else SAB_GRAN_PER_THREAD
    o = torch.empty(q.size(), dtype=q.dtype, device=q.device)
    lse = ops.qk_int8_sv_f8_attn(q_int8, kv.k_int8, kv.v_fp8, o, q_scale, kv.k_scale, kv.v_scale, kv.v_mean, lay,
                                 1 if is_causal else 0, gran, gran, sm_scale, 0, 1 if return_lse else 0)
    o = o[..., :kv.head_dim_og]
    if not return_lse:
        return o
    if kv.km is None:
        return o, lse / _LOG2E
    from .core import _lse_correction
    return o, lse / _LOG2E + _lse_correction(q, kv.km, kv.tensor_layout) * sm_scale
