"""Public API — drop-in for sageattention/core.py of thu-ml/SageAttention, backed by ONE sm_90a backend.

Signatures and behaviour follow the reference (file:line cited per function); the bodies re-state the
host logic (asserts, head-dim padding, K smoothing, LSE correction, output slicing) around the
H100 kernels: fused quantisers (csrc/quant.cu) and the wgmma attention kernel (csrc/attn.cu).
There is no arch dispatch, no Triton, no CPU fallback.
"""
from typing import Any, Optional
import numbers
import warnings
import torch
import torch.nn.functional as F

from . import ops
from ._capi import SAB_GRAN_PER_BLOCK, SAB_GRAN_PER_WARP, SAB_GRAN_PER_THREAD
from .quant import (k_mean, per_block_int8, per_warp_int8, per_thread_int8, per_channel_fp8, quant_q_int8, quant_k_int8, smooth_quant_k,
                    per_block_int8_varlen, per_channel_fp8_varlen, transpose_v_f16, transpose_v_f16_varlen, k_mean_varlen,
                    quant_q_int8_varlen, quant_k_int8_varlen, per_channel_fp8_varlen_seq, k_mean_paged, quant_k_int8_paged,
                    per_channel_fp8_paged)

_LOG2E = 1.44269504
_MAX_BLOCKSPARSE_KV = 1 << 20   # 64 * 16384 key blocks: the longest key range a block-sparse CTA compacts in shared memory


def _check_inputs(q, k, v):
    assert q.is_cuda, "Input tensors must be on cuda."
    assert q.dtype in [torch.float16, torch.bfloat16], "Input tensors must be in dtype of torch.float16 or torch.bfloat16"
    assert q.device == k.device == v.device, "All tensors must be on the same device."
    assert q.dtype == k.dtype == v.dtype, "All tensors must have the same dtype."


def _pad_head_dim(q, k, v):
    """sageattention/core.py:752-761."""
    head_dim_og = q.size(-1)
    if head_dim_og < 64:
        pad = 64 - head_dim_og
    elif 64 < head_dim_og < 128:
        pad = 128 - head_dim_og
    elif head_dim_og > 128:
        raise ValueError(f"Unsupported head_dim: {head_dim_og}")
    else:
        pad = 0
    if pad:
        q, k, v = F.pad(q, (0, pad)), F.pad(k, (0, pad)), F.pad(v, (0, pad))
    return q, k, v, head_dim_og


def _lse_correction(q, km, tensor_layout):
    """q @ km^T in the input dtype (sageattention/core.py:775-786)."""
    nh_dim = 2 if tensor_layout == "NHD" else 1
    g = q.size(nh_dim) // km.size(nh_dim)
    kmb = torch.repeat_interleave(km, g, dim=nh_dim) if g > 1 else km
    if tensor_layout == "NHD":
        return torch.matmul(q.transpose(1, 2), kmb.transpose(1, 2).transpose(2, 3)).squeeze(-1).to(torch.float32)
    return torch.matmul(q, kmb.transpose(2, 3)).squeeze(-1).to(torch.float32)


# ------------------------------------------------------------------------------------------------ dense calls and their gradient
def _quant_qk(q, k, kind, tensor_layout, qk_quant_gran, sm_scale, smooth_k, backend):
    """Q/K front-end of a dense entry point on head-dim-padded q, k: (km, q_int8, q_scale, k_int8, k_scale, q_gran, k_gran,
    fold_sm_scale).  Deterministic, so the backward re-runs it instead of keeping the 8-bit operands alive."""
    km = k_mean(k, tensor_layout) if smooth_k else None
    if kind == "fp16_triton":
        q_int8, q_scale, k_int8, k_scale = per_block_int8(q, k, km=km, sm_scale=sm_scale, tensor_layout=tensor_layout,
                                                          semantics=backend)
        return km, q_int8, q_scale, k_int8, k_scale, SAB_GRAN_PER_BLOCK, SAB_GRAN_PER_BLOCK, 1
    q_int8, q_scale = quant_q_int8(q, qk_quant_gran, tensor_layout)
    k_int8, k_scale = quant_k_int8(k, km, qk_quant_gran, tensor_layout)
    gran = SAB_GRAN_PER_WARP if qk_quant_gran == "per_warp" else SAB_GRAN_PER_THREAD
    return km, q_int8, q_scale, k_int8, k_scale, gran, gran, 0


def _attn_dense(q, k, v, kind, tensor_layout, is_causal, qk_quant_gran, sm_scale, smooth_k, smooth_v, v_range, backend,
                return_lse, block_mask=None, window=None):
    """Quantisers + attention kernel of a dense entry point on head-dim-padded q, k, v.  kind: "fp8" (FP8 PV, V range v_range),
    "fp16_cuda" (FP16 PV, per-warp / per-thread INT8) or "fp16_triton" (FP16 PV, per-block INT8 with sm_scale*log2e folded into
    q).  block_mask ("fp8" only): the [B,Hq,ceil(Sq/128),ceil(Skv/64)] bool view of sageattn_blocksparse; window ("fp8" only):
    the (left, right) of sageattn_window; the quantisers still see every key.  Returns (o, the kernel's log2 lse or an empty
    tensor, km)."""
    km, q_int8, q_scale, k_int8, k_scale, q_gran, k_gran, fold = _quant_qk(q, k, kind, tensor_layout, qk_quant_gran, sm_scale,
                                                                          smooth_k, backend)
    lay = 0 if tensor_layout == "NHD" else 1
    o = torch.empty(q.size(), dtype=q.dtype, device=q.device)
    if kind == "fp8":
        v_fp8, v_scale, vm = per_channel_fp8(v, tensor_layout=tensor_layout, scale_max=v_range, smooth_v=smooth_v)
        if window is not None:
            return o, ops.qk_int8_sv_f8_attn_window(q_int8, k_int8, v_fp8, o, q_scale, k_scale, v_scale, vm, window[0], window[1], lay,
                                                    1 if is_causal else 0, q_gran, k_gran, sm_scale, fold,
                                                    1 if return_lse else 0), km
        if block_mask is not None:
            return o, ops.qk_int8_sv_f8_attn_blocksparse(q_int8, k_int8, v_fp8, o, q_scale, k_scale, v_scale, vm, block_mask, lay,
                                                         1 if is_causal else 0, q_gran, k_gran, sm_scale, fold,
                                                         1 if return_lse else 0), km
        lse = ops.qk_int8_sv_f8_attn(q_int8, k_int8, v_fp8, o, q_scale, k_scale, v_scale, vm, lay, 1 if is_causal else 0,
                                     q_gran, k_gran, sm_scale, fold, 1 if return_lse else 0)
    else:
        v_t = transpose_v_f16(v, tensor_layout=tensor_layout)       # `v.to(torch.float16)`, core.py:297-298, 603
        lse = ops.qk_int8_sv_f16_attn(q_int8, k_int8, v_t, o, q_scale, k_scale, lay, 1 if is_causal else 0, q_gran, k_gran,
                                      sm_scale, fold, 1 if return_lse else 0)
    return o, lse, km


class _SageAttnFunction(torch.autograd.Function):
    """A dense entry point with a gradient: the gradient of attention evaluated at the forward's quantised logits, a
    straight-through estimator through the INT8 Q/K, FP8 V and FP8 P roundings (include/sageattn_b200.h, sab_qk_int8_attn_bwd).
    forward: the unchanged forward with the kernel LSE enabled; saves q, k, v, o and the raw LSE.  backward: re-runs the
    (deterministic) Q/K quantisers instead of saving their 8-bit outputs, then the two gradient kernels.  The LSE and the K mean
    are returned for the LSE correction and carry no gradient.  block_mask (sageattn_blocksparse): P = 0 on the hidden tiles, and
    the block-sparse gradient kernels visit only the visible ones; the mask has no gradient.  window (sageattn_window): P = 0
    outside the window, and the window gradient kernels visit only the tiles inside it."""

    @staticmethod
    def forward(ctx, q, k, v, kind, tensor_layout, is_causal, qk_quant_gran, sm_scale, smooth_k, smooth_v, v_range, backend,
                block_mask=None, window=None):
        o, lse, km = _attn_dense(q, k, v, kind, tensor_layout, is_causal, qk_quant_gran, sm_scale, smooth_k, smooth_v, v_range,
                                 backend, True, block_mask, window)
        ctx.save_for_backward(q, k, v, o, lse, block_mask)
        ctx.cfg = (kind, tensor_layout, is_causal, qk_quant_gran, sm_scale, smooth_k, backend)
        ctx.window = window
        km = km if km is not None else q.new_empty(0)
        ctx.mark_non_differentiable(lse, km)
        return o, lse, km

    @staticmethod
    def backward(ctx, do, _dlse, _dkm):
        kind, tensor_layout, is_causal, qk_quant_gran, sm_scale, smooth_k, backend = ctx.cfg
        q, k, v, o, lse, block_mask = ctx.saved_tensors
        km, q_int8, q_scale, k_int8, k_scale, q_gran, k_gran, fold = _quant_qk(q, k, kind, tensor_layout, qk_quant_gran, sm_scale,
                                                                             smooth_k, backend)
        # the kernels read 16-bit rows with 16-byte loads; dq / dk / dv take the strides of q / k / v
        q, k, v, o, do = (t.contiguous() for t in (q, k, v, o, do))
        dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
        if ctx.window is not None:
            ops.qk_int8_attn_bwd_window(q_int8, k_int8, q_scale, k_scale, q, k, v, o, do, lse, km, dq, dk, dv, ctx.window[0],
                                        ctx.window[1], 0 if tensor_layout == "NHD" else 1, 1 if is_causal else 0, q_gran, k_gran,
                                        sm_scale, fold)
        elif block_mask is not None:
            ops.qk_int8_attn_bwd_blocksparse(q_int8, k_int8, q_scale, k_scale, q, k, v, o, do, lse, km, dq, dk, dv, block_mask,
                                             0 if tensor_layout == "NHD" else 1, 1 if is_causal else 0, q_gran, k_gran, sm_scale,
                                             fold)
        else:
            ops.qk_int8_attn_bwd(q_int8, k_int8, q_scale, k_scale, q, k, v, o, do, lse, km, dq, dk, dv,
                                 0 if tensor_layout == "NHD" else 1, 1 if is_causal else 0, q_gran, k_gran, sm_scale, fold)
        return dq, dk, dv, None, None, None, None, None, None, None, None, None, None, None


def _dense_call(q, k, v, kind, tensor_layout, is_causal, qk_quant_gran, sm_scale, smooth_k, smooth_v, v_range, backend,
                return_lse, head_dim_og, block_mask=None, window=None):
    """Shared tail of the dense entry points (q, k, v already head-dim padded).  The differentiable form runs only when grad mode
    is on and q, k or v requires grad; otherwise the forward's launches and bytes are exactly those of the plain call.  The
    returned lse never carries a gradient.  block_mask, window: see _attn_dense."""
    if torch.is_grad_enabled() and (q.requires_grad or k.requires_grad or v.requires_grad):
        o, lse, km = _SageAttnFunction.apply(q, k, v, kind, tensor_layout, is_causal, qk_quant_gran, sm_scale, smooth_k, smooth_v,
                                             v_range, backend, block_mask, window)
        q = q.detach()
    else:
        o, lse, km = _attn_dense(q, k, v, kind, tensor_layout, is_causal, qk_quant_gran, sm_scale, smooth_k, smooth_v, v_range,
                                 backend, return_lse, block_mask, window)
    o = o[..., :head_dim_og]
    if return_lse:
        if smooth_k:
            return o, lse / _LOG2E + _lse_correction(q, km, tensor_layout) * sm_scale
        return o, lse / _LOG2E
    return o


# ------------------------------------------------------------------------------------------------ masked call and its gradient
def _expand_mask(attn_mask, q, k, tensor_layout):
    """attn_mask as the [B,Hq,Sq,Skv] view the masked kernels read (core.py:314-323): broadcast dimensions get stride 0."""
    if tensor_layout == "HND":
        target_shape = (q.shape[0], q.shape[1], q.shape[2], k.shape[2])
    else:
        target_shape = (q.shape[0], q.shape[2], q.shape[1], k.shape[1])
    try:
        return attn_mask.expand(target_shape)
    except Exception:
        raise AssertionError(f"attn_mask shape {attn_mask.shape} cannot be broadcast to {target_shape}")


class _SageAttnMaskedFunction(torch.autograd.Function):
    """sageattn_qk_int8_pv_fp16_triton with attn_mask and a gradient: the straight-through gradient of _SageAttnFunction at the
    forward's masked logits (include/sageattn_b200.h, sab_qk_int8_attn_bwd_masked), and for a float mask dBias = ln2 * dS.
    forward: the unchanged masked forward with the kernel LSE enabled; saves q, k, v, o, the LSE and the expanded mask view.
    backward: re-runs the K mean and per_block_int8 with the same quantization_backend, then the two gradient kernels.  The mask
    arrives as its expanded [B,Hq,Sq,Skv] view, so the kernels write a dense dBias and autograd's expand backward sums it over the
    broadcast dimensions.  That dBias costs B*Hq*Sq*Skv elements of the bias dtype, allocated during the backward and only when
    the bias requires grad.  The LSE and the K mean are returned for the LSE correction and carry no gradient."""

    @staticmethod
    def forward(ctx, q, k, v, attn_mask, tensor_layout, sm_scale, smooth_k, backend):
        km, q_int8, q_scale, k_int8, k_scale, _, _, _ = _quant_qk(q, k, "fp16_triton", tensor_layout, "per_block", sm_scale, smooth_k,
                                                                  backend)
        v_t = transpose_v_f16(v, tensor_layout=tensor_layout)
        o = torch.empty(q.size(), dtype=q.dtype, device=q.device)
        lse = ops.qk_int8_sv_f16_attn_masked(q_int8, k_int8, v_t, o, q_scale, k_scale, attn_mask, 0 if tensor_layout == "NHD" else 1,
                                             SAB_GRAN_PER_BLOCK, SAB_GRAN_PER_BLOCK, sm_scale, 1, 1)
        ctx.save_for_backward(q, k, v, o, lse, attn_mask)
        ctx.cfg = (tensor_layout, sm_scale, smooth_k, backend)
        km = km if km is not None else q.new_empty(0)
        ctx.mark_non_differentiable(lse, km)
        return o, lse, km

    @staticmethod
    def backward(ctx, do, _dlse, _dkm):
        tensor_layout, sm_scale, smooth_k, backend = ctx.cfg
        q, k, v, o, lse, attn_mask = ctx.saved_tensors
        km, q_int8, q_scale, k_int8, k_scale, q_gran, k_gran, fold = _quant_qk(q, k, "fp16_triton", tensor_layout, "per_block",
                                                                             sm_scale, smooth_k, backend)
        # the kernels read 16-bit rows with 16-byte loads; dq / dk / dv take the strides of q / k / v
        q, k, v, o, do = (t.contiguous() for t in (q, k, v, o, do))
        dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
        dbias = torch.empty(attn_mask.shape, dtype=attn_mask.dtype, device=q.device) if ctx.needs_input_grad[3] else None
        ops.qk_int8_attn_bwd_masked(q_int8, k_int8, q_scale, k_scale, q, k, v, o, do, lse, km, dq, dk, dv, attn_mask, dbias,
                                    0 if tensor_layout == "NHD" else 1, q_gran, k_gran, sm_scale, fold)
        return dq, dk, dv, dbias, None, None, None, None


def sageattn_qk_int8_pv_fp8_cuda(
    q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, tensor_layout: str = "HND", is_causal: bool = False,
    qk_quant_gran: str = "per_thread", sm_scale: Optional[float] = None, pv_accum_dtype: str = "fp32+fp16",
    smooth_k: bool = True, smooth_v: bool = False, return_lse: bool = False, **kwargs: Any,
) -> torch.Tensor:
    """INT8 QK^T + FP8 PV attention (reference: sageattention/core.py:636-826).

    pv_accum_dtype keeps the reference vocabulary.  The PV product always accumulates in fp32
    (per 64-key tile in the tensor core, across tiles on the CUDA cores, so the reference's f16 first-level
    accumulator — a consumer-GPU speed trick — buys nothing); the option still selects the reference's V
    quantisation range: 2.25 for "fp32+fp16", 448 otherwise (core.py:805-807).  smooth_v is honoured
    only for "fp32" (core.py:797-803).  Unknown values raise (the reference silently returns an
    uninitialised tensor)."""
    _check_inputs(q, k, v)
    return _qk_int8_pv_fp8(q, k, v, tensor_layout, is_causal, qk_quant_gran, sm_scale, pv_accum_dtype, smooth_k, smooth_v, return_lse)


def _qk_int8_pv_fp8(q, k, v, tensor_layout, is_causal, qk_quant_gran, sm_scale, pv_accum_dtype, smooth_k, smooth_v, return_lse,
                    block_mask=None, window=None):
    """Body of sageattn_qk_int8_pv_fp8_cuda after _check_inputs; block_mask: that of sageattn_blocksparse, checked and expanded by
    the caller; window: the (left, right) of sageattn_window, checked by the caller."""
    assert qk_quant_gran in ["per_warp", "per_thread"], "qk_quant_gran must be either 'per_warp' or 'per_thread'."
    if pv_accum_dtype not in ("fp32", "fp32+fp32", "fp32+fp16"):
        raise ValueError(f"Unsupported pv_accum_dtype: {pv_accum_dtype}")

    _tensor_layout = 0 if tensor_layout == "NHD" else 1
    if tensor_layout not in ("NHD", "HND"):
        raise ValueError(f"Unknown tensor layout: {tensor_layout}")
    q, k, v, head_dim_og = _pad_head_dim(q, k, v)
    assert q.stride(-1) == 1 and k.stride(-1) == 1 and v.stride(-1) == 1, "Last dim of qkv must be contiguous."
    if is_causal:
        seq_dim = 1 if _tensor_layout == 0 else 2
        assert q.size(seq_dim) == k.size(seq_dim), "qo_len and kv_len must be equal for causal attention."
    if sm_scale is None:
        sm_scale = head_dim_og ** -0.5

    if pv_accum_dtype in ("fp32+fp32", "fp32+fp16") and smooth_v:
        warnings.warn(f"pv_accum_dtype is '{pv_accum_dtype}', smooth_v will be ignored.")
        smooth_v = False
    quant_v_scale_max = 2.25 if pv_accum_dtype == "fp32+fp16" else 448.0
    # front-end: K mean (2 launches), Q / K quantisers, V statistics (2) + FP8 quantiser — 7 launches (reference: 6 + k.mean, core.py:773-809).
    # The single-launch cluster variants (quant.smooth_quant_k, per_channel_fp8(fused=True)) are opt-in.
    return _dense_call(q, k, v, "fp8", tensor_layout, is_causal, qk_quant_gran, sm_scale, smooth_k, smooth_v, quant_v_scale_max,
                       "cuda", return_lse, head_dim_og, block_mask, window)


def sageattn_window(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, window_size=(-1, -1), tensor_layout: str = "HND",
                    is_causal: bool = False, qk_quant_gran: str = "per_thread", sm_scale: Optional[float] = None,
                    pv_accum_dtype: str = "fp32+fp16", smooth_k: bool = True, smooth_v: bool = False,
                    return_lse: bool = False) -> torch.Tensor:
    """Sliding-window (local) sageattn_qk_int8_pv_fp8_cuda (no reference counterpart): the same options, checks, quantisation and
    numerics, but key j is visible to query i only if i - left <= j <= i + right, with (left, right) = window_size (and j <= i
    when is_causal, which needs Sq == Skv).  -1 leaves a side unbounded; alignment is top-left, as the causal rule (query i and
    key i are the same position), and Sq != Skv is allowed when not causal.  The kernels visit only the 128-query x 64-key tiles
    that meet the window and mask the elements on the tiles its edges cross.

    The K mean and the V scales are still taken over every key.  A row with no visible key returns 0 (lse -inf).  window_size
    (-1, -1) gives the bits of sageattn_qk_int8_pv_fp8_cuda, and (-1, 0) those of its causal call.  Differentiable when grad
    mode is on and q, k or v requires grad: the dense straight-through gradient with P = 0 outside the window."""
    window = _check_window_size(window_size)
    _check_inputs(q, k, v)
    return _qk_int8_pv_fp8(q, k, v, tensor_layout, is_causal, qk_quant_gran, sm_scale, pv_accum_dtype, smooth_k, smooth_v,
                           return_lse, window=window)


def _check_window_size(window_size):
    """window_size as a pair of Python ints >= -1, or ValueError."""
    if (not isinstance(window_size, (tuple, list)) or len(window_size) != 2 or
            any(isinstance(w, bool) or not isinstance(w, numbers.Integral) or w < -1 for w in window_size)):
        raise ValueError(f"window_size must be a pair of ints >= -1 (-1: unbounded), got {window_size!r}")
    return int(window_size[0]), int(window_size[1])


def sageattn_blocksparse(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, block_mask: torch.Tensor, tensor_layout: str = "HND",
                         is_causal: bool = False, qk_quant_gran: str = "per_thread", sm_scale: Optional[float] = None,
                         pv_accum_dtype: str = "fp32+fp16", smooth_k: bool = True, smooth_v: bool = False,
                         return_lse: bool = False) -> torch.Tensor:
    """Block-sparse sageattn_qk_int8_pv_fp8_cuda (no reference counterpart): the same options, checks, quantisation and numerics,
    but key j is visible to query i of head h only if block_mask[b, h, i // 128, j // 64] (and j <= i when is_causal), and the
    kernels visit only the visible 128-query x 64-key tiles.

    block_mask: torch.bool on q's device, shape [Bm, Hm, ceil(Sq/128), ceil(Skv/64)] with Bm in {1, B} and Hm in {1, Hq}
    (size-1 dimensions broadcast, any strides); indexed by the Q head under GQA; the block indices do not depend on
    tensor_layout.  The K mean and the V scales are still taken over every key.  A row with no visible key returns 0 (lse -inf).
    With an all-True mask the output is that of sageattn_qk_int8_pv_fp8_cuda to the bit.  Differentiable when grad mode is on
    and q, k or v requires grad: the dense straight-through gradient with P = 0 on hidden tiles; the mask has no gradient."""
    _check_inputs(q, k, v)
    assert isinstance(block_mask, torch.Tensor) and block_mask.dtype == torch.bool, "block_mask must be a torch.bool tensor."
    assert block_mask.device == q.device, "All tensors must be on the same device."
    if tensor_layout not in ("NHD", "HND"):
        raise ValueError(f"Unknown tensor layout: {tensor_layout}")
    if tensor_layout == "HND":
        B, Hq, Sq = q.shape[:3]
        Skv = k.size(2)
    else:
        B, Sq, Hq = q.shape[:3]
        Skv = k.size(1)
    nqb, nkb = (Sq + 127) // 128, (Skv + 63) // 64
    if block_mask.dim() != 4 or tuple(block_mask.shape[2:]) != (nqb, nkb):
        raise ValueError(f"block_mask shape {tuple(block_mask.shape)} must be [B or 1, Hq or 1, {nqb}, {nkb}] "
                         f"(ceil(Sq/128), ceil(Skv/64))")
    if block_mask.size(0) not in (1, B) or block_mask.size(1) not in (1, Hq):
        raise ValueError(f"block_mask shape {tuple(block_mask.shape)} cannot be broadcast to [{B}, {Hq}, {nqb}, {nkb}]")
    return _qk_int8_pv_fp8(q, k, v, tensor_layout, is_causal, qk_quant_gran, sm_scale, pv_accum_dtype, smooth_k, smooth_v,
                           return_lse, block_mask.expand(B, Hq, nqb, nkb))


def sageattn(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, tensor_layout: str = "HND", is_causal: bool = False,
             sm_scale: Optional[float] = None, return_lse: bool = False, **kwargs: Any):
    """sageattention/core.py:79-157.  The reference dispatches on compute capability; on an H100 it calls its sm90 kernel with
    pv_accum_dtype="fp32+fp32" (V range 448).  Here the single backend deliberately keeps the reference's sm89 defaults
    (per-thread INT8, FP8 PV, "fp32+fp16" V range 2.25), so that sageattn() computes the same bytes on every GPU this library
    has targeted; that is a documented difference from the reference's own sageattn() on an H100.  Unknown kwargs (attn_mask=, dropout_p=, scale=, ...) are accepted and ignored
    exactly like the reference so SDPA monkey-patches keep working (example/cogvideox_infer.py:35).

    The 2.25 V range of "fp32+fp16" exists in the reference to keep its fp16 PV accumulator from overflowing; this kernel
    accumulates PV in fp32, so the range buys nothing here and is kept ONLY so that the quantised V bytes (and with them the
    output) match what the reference's default sm89 dispatch produces.  Callers who prefer e4m3's full dynamic range for V call
    sageattn_qk_int8_pv_fp8_cuda(..., pv_accum_dtype="fp32+fp32") (448 range, the reference's sm90 choice) at the same speed."""
    return sageattn_qk_int8_pv_fp8_cuda(q, k, v, tensor_layout=tensor_layout, is_causal=is_causal, sm_scale=sm_scale,
                                        return_lse=return_lse, pv_accum_dtype="fp32+fp16")


def sageattn_qk_int8_pv_fp8_cuda_sm90(q, k, v, tensor_layout: str = "HND", is_causal: bool = False,
                                      qk_quant_gran: str = "per_thread", sm_scale: Optional[float] = None,
                                      pv_accum_dtype: str = "fp32+fp32", smooth_k: bool = True, smooth_v: bool = False,
                                      return_lse: bool = False, **kwargs: Any):
    """API shell for sageattention/core.py:829-996 (Hopper entry point): same numerics contract, served by
    the sm_90a kernel.  Only "fp32+fp32" exists in the reference for this entry (core.py:985-989)."""
    assert pv_accum_dtype == "fp32+fp32", "only 'fp32+fp32' is supported for the sm90 entry point"
    return sageattn_qk_int8_pv_fp8_cuda(q, k, v, tensor_layout=tensor_layout, is_causal=is_causal,
                                        qk_quant_gran=qk_quant_gran, sm_scale=sm_scale, pv_accum_dtype=pv_accum_dtype,
                                        smooth_k=smooth_k, smooth_v=False, return_lse=return_lse)


def sageattn_qk_int8_pv_fp16_triton(q, k, v, tensor_layout: str = "HND", quantization_backend: str = "triton",
                                    is_causal: bool = False, sm_scale: Optional[float] = None, smooth_k: bool = True,
                                    return_lse: bool = False, attn_mask: Optional[torch.Tensor] = None, **kwargs: Any):
    """sageattention/core.py:160-331 on sm_90a: per-block INT8 quantisation with the Triton path's exact rounding
    (bit-exact q/k/scales), sm_scale*log2e folded into q, then the FP16-PV kernel variant (fp16 wgmma, P and
    V in fp16, softmax without exponent offset — the Triton kernel's numerics, triton/attn_qk_int8_per_block.py).
    attn_mask (bool, or the q dtype as an additive bias; broadcast to [B,Hq,Sq,Skv]; non-causal only) follows
    core.py:248-250, 310-325 and attn_qk_int8_per_block.py:33-52 — including the reference's convention that a float
    bias is added AFTER the logits were scaled by sm_scale*log2(e), i.e. it acts as bias*ln(2) in natural-log units.
    Differentiable (no reference counterpart) when grad mode is on and q, k, v or a float attn_mask requires grad, with or without
    a mask; a float mask then gets dBias = ln(2) * dS, summed over its broadcast dimensions (_SageAttnMaskedFunction)."""
    dtype = q.dtype
    _check_inputs(q, k, v)
    if attn_mask is not None:
        assert attn_mask.dtype == torch.bool or attn_mask.dtype == q.dtype, "attn_mask must be of dtype bool or the same dtype as q."
        assert attn_mask.device == q.device, "All tensors must be on the same device."
        assert not is_causal, "Mask should be None for causal attention."
    _tensor_layout = 0 if tensor_layout == "NHD" else 1
    q, k, v, head_dim_og = _pad_head_dim(q, k, v)
    assert q.stride(-1) == 1 and k.stride(-1) == 1 and v.stride(-1) == 1, "Last dim of qkv must be contiguous."
    if sm_scale is None:
        sm_scale = 1.0 / (head_dim_og ** 0.5)
    if quantization_backend not in ("triton", "cuda"):
        raise ValueError(f"Unsupported quantization backend: {quantization_backend}")
    if attn_mask is None:
        return _dense_call(q, k, v, "fp16_triton", tensor_layout, is_causal, "per_block", sm_scale, smooth_k, False, 0.0,
                           quantization_backend, return_lse, head_dim_og)
    if torch.is_grad_enabled() and (q.requires_grad or k.requires_grad or v.requires_grad or attn_mask.requires_grad):
        # the differentiable form (a bool mask cannot require grad); the returned lse carries no gradient
        o, lse, km = _SageAttnMaskedFunction.apply(q, k, v, _expand_mask(attn_mask, q, k, tensor_layout), tensor_layout, sm_scale,
                                                   smooth_k, quantization_backend)
        o = o[..., :head_dim_og]
        if return_lse:
            q = q.detach()
            return o, lse / _LOG2E + _lse_correction(q, km, tensor_layout) * sm_scale if smooth_k else lse / _LOG2E
        return o
    lse_correction = None
    if smooth_k:
        km = k_mean(k, tensor_layout)
        if return_lse:
            lse_correction = _lse_correction(q, km, tensor_layout)
    else:
        km = None
    q_int8, q_scale, k_int8, k_scale = per_block_int8(q, k, km=km, sm_scale=sm_scale, tensor_layout=tensor_layout,
                                                      semantics=quantization_backend)
    v_t = transpose_v_f16(v, tensor_layout=tensor_layout)       # `v.to(torch.float16)`, core.py:297-298
    o = torch.empty(q.size(), dtype=dtype, device=q.device)
    attn_mask = _expand_mask(attn_mask, q, k, tensor_layout)
    lse = ops.qk_int8_sv_f16_attn_masked(q_int8, k_int8, v_t, o, q_scale, k_scale, attn_mask, _tensor_layout,
                                         SAB_GRAN_PER_BLOCK, SAB_GRAN_PER_BLOCK, sm_scale, 1, 1 if return_lse else 0)
    o = o[..., :head_dim_og]
    if return_lse:
        return o, lse / _LOG2E + lse_correction * sm_scale if smooth_k else lse / _LOG2E
    return o


def sageattn_qk_int8_pv_fp16_cuda(q, k, v, tensor_layout: str = "HND", is_causal: bool = False,
                                  qk_quant_gran: str = "per_thread", sm_scale: Optional[float] = None,
                                  pv_accum_dtype: str = "fp32", smooth_k: bool = True, smooth_v: bool = False,
                                  return_lse: bool = False, **kwargs: Any):
    """sageattention/core.py:451-633 (INT8 QK^T + **FP16** PV) on sm_90a: V and P stay in fp16 — callers pick this entry
    over the fp8 ones for accuracy — through the FP16-PV kernel variant (fp16 wgmma, fp32 accumulation).
    Q/K quantisation is the reference's per-warp / per-thread INT8 (core.py:590-593; WARPQ is 32 for every mode here: the
    scale packing is internal to this call).  pv_accum_dtype keeps the reference vocabulary ("fp32", "fp16", "fp16+fp32",
    core.py:601-617): the kernel always accumulates PV in fp32, i.e. every mode gets the accuracy of "fp32".
    smooth_v exists in the reference only to protect the "fp16" accumulator from overflow (core.py:606-610); with fp32
    accumulation it has nothing to do, so it is accepted and ignored with the reference's warning."""
    _check_inputs(q, k, v)
    assert qk_quant_gran in ["per_warp", "per_thread"], "qk_quant_gran must be either 'per_warp' or 'per_thread'."
    if pv_accum_dtype not in ("fp32", "fp16", "fp16+fp32"):
        raise ValueError(f"Unsupported pv_accum_dtype: {pv_accum_dtype}")
    if tensor_layout not in ("NHD", "HND"):
        raise ValueError(f"Unknown tensor layout: {tensor_layout}")
    _tensor_layout = 0 if tensor_layout == "NHD" else 1
    q, k, v, head_dim_og = _pad_head_dim(q, k, v)
    assert q.stride(-1) == 1 and k.stride(-1) == 1 and v.stride(-1) == 1, "Last dim of qkv must be contiguous."
    if is_causal:
        seq_dim = 1 if _tensor_layout == 0 else 2
        assert q.size(seq_dim) == k.size(seq_dim), "qo_len and kv_len must be equal for causal attention."
    if sm_scale is None:
        sm_scale = head_dim_og ** -0.5
    if smooth_v:
        warnings.warn(f"pv_accum_dtype is '{pv_accum_dtype}' (fp32 accumulation on this backend), smooth_v will be ignored.")
    return _dense_call(q, k, v, "fp16_cuda", tensor_layout, is_causal, qk_quant_gran, sm_scale, smooth_k, False, 0.0, "cuda",
                       return_lse, head_dim_og)


def sageattn_varlen(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, cu_seqlens_q: torch.Tensor,
                    cu_seqlens_k: torch.Tensor, max_seqlen_q: int, max_seqlen_k: int, is_causal: bool = False,
                    sm_scale: Optional[float] = None, smooth_k: bool = True, **kwargs: Any) -> torch.Tensor:
    """sageattention/core.py:334-448: packed [T,H,D] tensors, per-block INT8 per sequence (Triton rounding,
    bit-exact), K mean over all tokens of the batch (core.py:433), FP16 P and V (fp16 wgmma) like the
    reference's Triton varlen kernels.  Differentiable (no reference counterpart) when grad mode is on and q, k or v requires
    grad: each sequence gets the dense entry points' straight-through gradient on its own (_SageAttnVarlenFunction)."""
    _check_inputs(q, k, v)
    q, k, v, head_dim_og = _pad_head_dim(q, k, v)
    assert q.stride(-1) == 1 and k.stride(-1) == 1 and v.stride(-1) == 1, "Last dim of qkv must be contiguous."
    assert cu_seqlens_q.is_contiguous() and cu_seqlens_k.is_contiguous(), "cu_seqlens_q and cu_seqlens_k must be contiguous."
    if sm_scale is None:
        sm_scale = 1.0 / (head_dim_og ** 0.5)
    args = (cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k, is_causal, sm_scale, smooth_k)
    if torch.is_grad_enabled() and (q.requires_grad or k.requires_grad or v.requires_grad):
        o = _SageAttnVarlenFunction.apply(q, k, v, *args)
    else:
        o, _ = _attn_varlen(q, k, v, *args, False)
    return o[..., :head_dim_og]


# ------------------------------------------------------------------------------------------------ packed varlen call and its gradient
def _quant_qk_varlen(q, k, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k, sm_scale, smooth_k):
    """Q/K front-end of sageattn_varlen on head-dim-padded packed q, k: (km, q_int8, q_scale, k_int8, k_scale, cu_q_scale,
    cu_k_scale).  Deterministic, so the backward re-runs it."""
    km = None
    if smooth_k:
        km = k_mean(k.unsqueeze(0), "NHD").view(1, k.size(1), k.size(2))   # mean over all tokens
    return (km,) + per_block_int8_varlen(q, k, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k, sm_scale=sm_scale, km=km)


def _attn_varlen(q, k, v, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k, is_causal, sm_scale, smooth_k, return_lse):
    """Quantisers + FP16-PV kernel of sageattn_varlen on head-dim-padded packed q, k, v: (o, the kernel's [Hq,Tq] log2 lse or an
    empty tensor)."""
    _, q_int8, q_scale, k_int8, k_scale, cu_q_scale, cu_k_scale = _quant_qk_varlen(q, k, cu_seqlens_q, cu_seqlens_k, max_seqlen_q,
                                                                                  max_seqlen_k, sm_scale, smooth_k)
    v_t, cu_pad = transpose_v_f16_varlen(v, cu_seqlens_k, max_seqlen_k)
    o = torch.empty(q.shape, dtype=q.dtype, device=q.device)
    lse = ops.qk_int8_sv_f16_attn_varlen(q_int8, k_int8, v_t, o, q_scale, k_scale, cu_seqlens_q.to(torch.int32),
                                         cu_seqlens_k.to(torch.int32), cu_pad, cu_q_scale, cu_k_scale, max_seqlen_q,
                                         1 if is_causal else 0, sm_scale, 1, 1 if return_lse else 0)
    return o, lse


class _SageAttnVarlenFunction(torch.autograd.Function):
    """sageattn_varlen with a gradient: the gradient of _SageAttnFunction applied to each packed sequence on its own
    (include/sageattn_b200.h, sab_qk_int8_attn_bwd_varlen).  forward: the unchanged varlen forward with the kernel LSE enabled;
    saves q, k, v, o, the LSE and the cu_seqlens.  backward: re-runs the K mean and the varlen Q/K quantisers, then the two
    gradient kernels.  Tokens past cu_seqlens[-1] belong to no sequence: their gradient is zero."""

    @staticmethod
    def forward(ctx, q, k, v, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k, is_causal, sm_scale, smooth_k):
        o, lse = _attn_varlen(q, k, v, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k, is_causal, sm_scale, smooth_k, True)
        ctx.save_for_backward(q, k, v, o, lse, cu_seqlens_q, cu_seqlens_k)
        ctx.cfg = (max_seqlen_q, max_seqlen_k, is_causal, sm_scale, smooth_k)
        return o

    @staticmethod
    def backward(ctx, do):
        max_seqlen_q, max_seqlen_k, is_causal, sm_scale, smooth_k = ctx.cfg
        q, k, v, o, lse, cu_seqlens_q, cu_seqlens_k = ctx.saved_tensors
        km, q_int8, q_scale, k_int8, k_scale, cu_q_scale, cu_k_scale = _quant_qk_varlen(q, k, cu_seqlens_q, cu_seqlens_k, max_seqlen_q,
                                                                                      max_seqlen_k, sm_scale, smooth_k)
        # the kernels read 16-bit rows with 16-byte loads; dq / dk / dv take the strides of q / k / v
        q, k, v, o, do = (t.contiguous() for t in (q, k, v, o, do))
        dq, dk, dv = torch.zeros_like(q), torch.zeros_like(k), torch.zeros_like(v)
        ops.qk_int8_attn_bwd_varlen(q_int8, k_int8, q_scale, k_scale, q, k, v, o, do, lse, km, dq, dk, dv,
                                    cu_seqlens_q.to(torch.int32), cu_seqlens_k.to(torch.int32), cu_q_scale, cu_k_scale, max_seqlen_q,
                                    max_seqlen_k, 1 if is_causal else 0, sm_scale, 1)
        return dq, dk, dv, None, None, None, None, None, None, None


# ------------------------------------------------------------------------------------------------ packed INT8+FP8 call and its gradient
def _quant_qk_varlen_f8(q, k, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k, qk_quant_gran, smooth_k):
    """Q/K front-end of sageattn_varlen_qk_int8_pv_fp8_cuda on head-dim-padded packed q, k, every statistic per sequence: (km
    [nseq,Hkv,D] or None, q_int8, q_scale, cu_q_scale, k_int8, k_scale, cu_k_scale).  Deterministic, so the backward re-runs it."""
    km = k_mean_varlen(k, cu_seqlens_k, max_seqlen_k) if smooth_k else None
    q_int8, q_scale, cu_q_scale = quant_q_int8_varlen(q, cu_seqlens_q, max_seqlen_q, qk_quant_gran)
    k_int8, k_scale, cu_k_scale = quant_k_int8_varlen(k, km, cu_seqlens_k, max_seqlen_k, qk_quant_gran)
    return km, q_int8, q_scale, cu_q_scale, k_int8, k_scale, cu_k_scale


def _attn_varlen_f8(q, k, v, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k, is_causal, qk_quant_gran, sm_scale, smooth_k,
                    smooth_v, v_range, return_lse, block_mask=None, window=None):
    """Quantisers + INT8+FP8 kernel of sageattn_varlen_qk_int8_pv_fp8_cuda on head-dim-padded packed q, k, v (cu_seqlens int32):
    (o, the kernel's [Hq,Tq] log2 lse or an empty tensor, km).  window: the (left, right) of sageattn_varlen_window, checked and
    clamped by the caller; block_mask: the [nseq,Hq,.,.] bool view of sageattn_varlen_blocksparse, checked and expanded by the
    caller.  The quantisers still see every key of each sequence."""
    km, q_int8, q_scale, cu_q_scale, k_int8, k_scale, cu_k_scale = _quant_qk_varlen_f8(q, k, cu_seqlens_q, cu_seqlens_k, max_seqlen_q,
                                                                                     max_seqlen_k, qk_quant_gran, smooth_k)
    v_fp8, v_scale, vm, cu_pad = per_channel_fp8_varlen_seq(v, cu_seqlens_k, max_seqlen_k, v_range, smooth_v)
    o = torch.empty(q.shape, dtype=q.dtype, device=q.device)
    gran = SAB_GRAN_PER_WARP if qk_quant_gran == "per_warp" else SAB_GRAN_PER_THREAD
    if window is not None:
        return o, ops.qk_int8_sv_f8_attn_varlen_window(q_int8, k_int8, v_fp8, o, q_scale, k_scale, v_scale, vm, cu_seqlens_q, cu_seqlens_k,
                                                       cu_pad, cu_q_scale, cu_k_scale, max_seqlen_q, window[0], window[1],
                                                       1 if is_causal else 0, gran, gran, sm_scale, 1 if return_lse else 0), km
    if block_mask is not None:
        return o, ops.qk_int8_sv_f8_attn_varlen_blocksparse(q_int8, k_int8, v_fp8, o, q_scale, k_scale, v_scale, vm, cu_seqlens_q,
                                                            cu_seqlens_k, cu_pad, cu_q_scale, cu_k_scale, max_seqlen_q, max_seqlen_k,
                                                            block_mask, 1 if is_causal else 0, gran, gran, sm_scale,
                                                            1 if return_lse else 0), km
    lse = ops.qk_int8_sv_f8_attn_varlen_seq(q_int8, k_int8, v_fp8, o, q_scale, k_scale, v_scale, vm, cu_seqlens_q, cu_seqlens_k, cu_pad,
                                            cu_q_scale, cu_k_scale, max_seqlen_q, 1 if is_causal else 0, gran, gran, sm_scale,
                                            1 if return_lse else 0)
    return o, lse, km


def _lse_correction_varlen(q, km, cu_seqlens_q):
    """[Hq,Tq] fp32: q . km[b] for each token of sequence b, in the input dtype, the correction _lse_correction adds for the dense
    call on that sequence.  The mean is gathered per token on the device (no host sync), [Tq,Hkv,D] (at most the size of q), and
    each token's Hq/Hkv query heads take their dot products with it in one batched product: memory and work grow with Tq, not with
    Tq * nseq.  cuBLAS picks its kernel by shape, so the fp32 sum of an element may be taken in another order than in the dense
    call's product before its rounding to the input dtype: the two can then differ by one unit in the last place, or by more where
    the sum cancels (measured on an H100: 0 of 1.03M elements differ at configs[3]; 47 (bf16) and 662 (fp16) of 0.8M with a
    thousand sequences of 0..200 tokens)."""
    Tq, Hq, D = q.shape
    Hkv = km.size(1)
    seq = torch.searchsorted(cu_seqlens_q[1:], torch.arange(Tq, device=q.device, dtype=cu_seqlens_q.dtype), right=True)
    seq = seq.clamp_(max=km.size(0) - 1)                                                         # rows past cu_seqlens_q[-1]
    kmt = km.index_select(0, seq)                                                                # [Tq,Hkv,D]
    corr = torch.matmul(q.reshape(Tq, Hkv, Hq // Hkv, D), kmt.unsqueeze(-1))                         # [Tq,Hkv,Hq/Hkv,1]
    return corr.view(Tq, Hq).t().to(torch.float32)


class _SageAttnVarlenFp8Function(torch.autograd.Function):
    """sageattn_varlen_qk_int8_pv_fp8_cuda with a gradient: the straight-through gradient of _SageAttnFunction applied to each packed
    sequence on its own (include/sageattn_b200.h, sab_qk_int8_attn_bwd_varlen_seq).  forward: the unchanged forward with the kernel
    LSE enabled; saves q, k, v, o, the LSE and the cu_seqlens.  backward: re-runs the per-sequence K mean and Q/K quantisers, then
    the gradient kernels.  Tokens past cu_seqlens[-1] belong to no sequence: their gradient is zero.  The LSE and the K means are
    returned for the LSE correction and carry no gradient.  window (sageattn_varlen_window): P = 0 outside each sequence's window,
    and the window gradient kernels visit only the tiles inside it.  block_mask (sageattn_varlen_blocksparse): P = 0 on each
    sequence's hidden tiles, and the block-sparse gradient kernels visit only the visible ones; the mask has no gradient."""

    @staticmethod
    def forward(ctx, q, k, v, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k, is_causal, qk_quant_gran, sm_scale, smooth_k,
                smooth_v, v_range, block_mask=None, window=None):
        o, lse, km = _attn_varlen_f8(q, k, v, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k, is_causal, qk_quant_gran, sm_scale,
                                     smooth_k, smooth_v, v_range, True, block_mask, window)
        ctx.save_for_backward(q, k, v, o, lse, cu_seqlens_q, cu_seqlens_k, block_mask)
        ctx.cfg = (max_seqlen_q, max_seqlen_k, is_causal, qk_quant_gran, sm_scale, smooth_k)
        ctx.window = window
        km = km if km is not None else q.new_empty(0)
        ctx.mark_non_differentiable(lse, km)
        return o, lse, km

    @staticmethod
    def backward(ctx, do, _dlse, _dkm):
        max_seqlen_q, max_seqlen_k, is_causal, qk_quant_gran, sm_scale, smooth_k = ctx.cfg
        q, k, v, o, lse, cu_seqlens_q, cu_seqlens_k, block_mask = ctx.saved_tensors
        km, q_int8, q_scale, cu_q_scale, k_int8, k_scale, cu_k_scale = _quant_qk_varlen_f8(q, k, cu_seqlens_q, cu_seqlens_k, max_seqlen_q,
                                                                                         max_seqlen_k, qk_quant_gran, smooth_k)
        # the kernels read 16-bit rows with 16-byte loads; dq / dk / dv take the strides of q / k / v
        q, k, v, o, do = (t.contiguous() for t in (q, k, v, o, do))
        dq, dk, dv = torch.zeros_like(q), torch.zeros_like(k), torch.zeros_like(v)
        gran = SAB_GRAN_PER_WARP if qk_quant_gran == "per_warp" else SAB_GRAN_PER_THREAD
        if ctx.window is not None:
            ops.qk_int8_attn_bwd_varlen_window(q_int8, k_int8, q_scale, k_scale, q, k, v, o, do, lse, km, dq, dk, dv, cu_seqlens_q,
                                               cu_seqlens_k, cu_q_scale, cu_k_scale, max_seqlen_q, max_seqlen_k, ctx.window[0],
                                               ctx.window[1], 1 if is_causal else 0, gran, gran, sm_scale)
        elif block_mask is not None:
            ops.qk_int8_attn_bwd_varlen_blocksparse(q_int8, k_int8, q_scale, k_scale, q, k, v, o, do, lse, km, dq, dk, dv, cu_seqlens_q,
                                                    cu_seqlens_k, cu_q_scale, cu_k_scale, max_seqlen_q, max_seqlen_k, block_mask,
                                                    1 if is_causal else 0, gran, gran, sm_scale)
        else:
            ops.qk_int8_attn_bwd_varlen_seq(q_int8, k_int8, q_scale, k_scale, q, k, v, o, do, lse, km, dq, dk, dv, cu_seqlens_q,
                                            cu_seqlens_k, cu_q_scale, cu_k_scale, max_seqlen_q, max_seqlen_k, 1 if is_causal else 0, gran,
                                            gran, sm_scale)
        return dq, dk, dv, None, None, None, None, None, None, None, None, None, None, None, None


def _check_cu_seqlens(q, k, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k):
    if q.dim() != 3 or k.dim() != 3:
        raise ValueError(f"q, k and v must be packed [T, H, D] tensors (got q {tuple(q.shape)}, k {tuple(k.shape)})")
    for name, cu in (("cu_seqlens_q", cu_seqlens_q), ("cu_seqlens_k", cu_seqlens_k)):
        if not isinstance(cu, torch.Tensor) or cu.dim() != 1 or cu.dtype not in (torch.int32, torch.int64) or cu.numel() < 2:
            raise ValueError(f"{name} must be a 1-D int32 or int64 tensor of nseq + 1 >= 2 offsets")
        if cu.device != q.device:
            raise ValueError(f"{name} must be on q's device")
    if cu_seqlens_q.numel() != cu_seqlens_k.numel():
        raise ValueError(f"cu_seqlens_q and cu_seqlens_k must have the same length ({cu_seqlens_q.numel()} != {cu_seqlens_k.numel()})")
    for name, m in (("max_seqlen_q", max_seqlen_q), ("max_seqlen_k", max_seqlen_k)):
        if isinstance(m, bool) or not isinstance(m, numbers.Integral) or m < 1:
            raise ValueError(f"{name} must be an int >= 1, got {m!r}")
    if q.size(0) == 0 or k.size(0) == 0:
        raise ValueError("the packed batch must hold at least one query and one key")


def sageattn_varlen_qk_int8_pv_fp8_cuda(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, cu_seqlens_q: torch.Tensor,
                                        cu_seqlens_k: torch.Tensor, max_seqlen_q: int, max_seqlen_k: int, is_causal: bool = False,
                                        qk_quant_gran: str = "per_thread", sm_scale: Optional[float] = None,
                                        pv_accum_dtype: str = "fp32+fp16", smooth_k: bool = True, smooth_v: bool = False,
                                        return_lse: bool = False):
    """Packed variable-length sageattn_qk_int8_pv_fp8_cuda (no reference counterpart): q [Tq,Hq,D], k / v [Tk,Hkv,D] (GQA:
    Hq % Hkv == 0), sequence b = q[cu_seqlens_q[b]:cu_seqlens_q[b+1]] against k / v[cu_seqlens_k[b]:cu_seqlens_k[b+1]]
    (cu_seqlens int32 or int64, same length; max_seqlen_* >= every length).  Options, checks and warnings are those of
    sageattn_qk_int8_pv_fp8_cuda.

    Contract: each sequence's output rows (and lse rows) are the bits of sageattn_qk_int8_pv_fp8_cuda(q_b[None], k_b[None],
    v_b[None], tensor_layout="NHD", ...) with the same options; packing changes no sequence's result.  So every statistic is
    per sequence: the K smoothing mean, the Q / K INT8 blocks (which restart at every sequence) and the V FP8 scales and mean.
    This differs from sageattn_varlen, which takes one K mean over all packed tokens, as the reference's varlen call does.

    is_causal: top-left inside each sequence, Lq != Lk allowed.  Empty sequences are allowed: a sequence without keys returns
    zero rows and lse -inf.  Rows past cu_seqlens_q[-1] are not written.  return_lse: also returns the [Hq,Tq] fp32 LSE in
    natural-log units (flash-attn's varlen convention), with each sequence's own K-mean correction (the kernel's LSE is the dense
    call's to the bit; the correction q . km is a per-token product whose fp32 sum can be taken in another order than the dense
    call's before its rounding to the input dtype, see _lse_correction_varlen: so lse, unlike the output, is not bit-identical
    to the dense call's on every element).  Differentiable when grad
    mode is on and q, k or v requires grad: for every sequence, dq / dk / dv are the bits of the dense backward of the
    one-sequence call; tokens past cu_seqlens_*[-1] and keys of a sequence without queries get zero gradients."""
    _check_inputs(q, k, v)
    return _varlen_qk_int8_pv_fp8(q, k, v, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k, is_causal, qk_quant_gran, sm_scale,
                                  pv_accum_dtype, smooth_k, smooth_v, return_lse)


def _varlen_window_arg(window, max_seqlen_q, max_seqlen_k):
    """The (left, right) the packed window kernels receive: a side that reaches past the longest sequence (left >= max_seqlen_q,
    right >= max_seqlen_k) sees as much as -1 in every sequence and becomes -1, so a Python int of any size reaches the C ABI
    as an int32 (ctypes would truncate it silently).  The kernels clamp again at each sequence's own lengths."""
    left, right = window
    return (-1 if left >= max_seqlen_q else left), (-1 if right >= max_seqlen_k else right)


def sageattn_varlen_window(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, cu_seqlens_q: torch.Tensor, cu_seqlens_k: torch.Tensor,
                           max_seqlen_q: int, max_seqlen_k: int, window_size=(-1, -1), is_causal: bool = False,
                           qk_quant_gran: str = "per_thread", sm_scale: Optional[float] = None, pv_accum_dtype: str = "fp32+fp16",
                           smooth_k: bool = True, smooth_v: bool = False, return_lse: bool = False):
    """Sliding-window (local) attention on packed sequences (no reference counterpart): sageattn_varlen_qk_int8_pv_fp8_cuda with the
    window_size of sageattn_window applied inside each sequence.  The options, checks, warnings, V ranges and packed layout are
    those of sageattn_varlen_qk_int8_pv_fp8_cuda; window_size is a pair (left, right) of ints >= -1 (ValueError otherwise, before
    any launch): key j of a sequence is visible to its query i iff i - left <= j <= i + right (-1 leaves a side unbounded), top-left
    inside the sequence, and j <= i when is_causal.  A window never reaches into a neighbouring sequence.

    Contract: "sageattn_window, per sequence".  Sequence b's output rows are the bits of sageattn_window(q_b[None], k_b[None],
    v_b[None], window_size, tensor_layout="NHD", is_causal=..., <same options>); every statistic (K mean, INT8 blocks, V scales and
    mean) is taken per sequence, and each sequence sees the window clamped at its own lengths, as the dense call would.  Causal is
    allowed with Lq != Lk (top-left), which sageattn_window refuses; causal with (left, right) is non-causal with (left, 0), so such
    a sequence gets the bits of sageattn_window(..., (left, 0), is_causal=False) on it.  window_size (-1, -1) gives the bits of
    sageattn_varlen_qk_int8_pv_fp8_cuda, and (-1, 0) non-causal those of its causal call.

    An empty sequence or a row with no visible key gives zero rows and lse -inf; rows past cu_seqlens_q[-1] are not written.
    return_lse gives [Hq,Tq] in natural-log units with sageattn_varlen_qk_int8_pv_fp8_cuda's caveat: the kernel's LSE is the dense
    call's to the bit, the per-token K-mean correction within one unit of it.  Differentiable when grad mode is on and q, k or v
    requires grad: for every sequence, dq / dk / dv are the bits of the dense window backward of the one-sequence call; tokens past
    the end, keys of a sequence without queries and keys no query's window reaches get zero gradients."""
    window = _check_window_size(window_size)
    _check_inputs(q, k, v)
    return _varlen_qk_int8_pv_fp8(q, k, v, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k, is_causal, qk_quant_gran, sm_scale,
                                  pv_accum_dtype, smooth_k, smooth_v, return_lse, window)


def _varlen_block_mask(block_mask, q, cu_seqlens_q, max_seqlen_q, max_seqlen_k):
    """block_mask of sageattn_varlen_blocksparse checked against the packed batch and expanded to [nseq,Hq,nqb,nkb], or
    ValueError (the wording of sageattn_blocksparse).  max_seqlen_k is limited to MAX_KV_LEN: each CTA compacts one mask row of
    ceil(max_seqlen_k/64) blocks in shared memory."""
    nseq, Hq = cu_seqlens_q.numel() - 1, q.size(1)
    nqb, nkb = (max_seqlen_q + 127) // 128, (max_seqlen_k + 63) // 64
    if block_mask.dim() != 4 or tuple(block_mask.shape[2:]) != (nqb, nkb):
        raise ValueError(f"block_mask shape {tuple(block_mask.shape)} must be [nseq or 1, Hq or 1, {nqb}, {nkb}] "
                         f"(ceil(max_seqlen_q/128), ceil(max_seqlen_k/64))")
    if block_mask.size(0) not in (1, nseq) or block_mask.size(1) not in (1, Hq):
        raise ValueError(f"block_mask shape {tuple(block_mask.shape)} cannot be broadcast to [{nseq}, {Hq}, {nqb}, {nkb}]")
    if max_seqlen_k > _MAX_BLOCKSPARSE_KV:
        raise ValueError(f"the block-sparse path supports max_seqlen_k <= {_MAX_BLOCKSPARSE_KV} (got {max_seqlen_k})")
    return block_mask.expand(nseq, Hq, nqb, nkb)


def sageattn_varlen_blocksparse(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, cu_seqlens_q: torch.Tensor,
                                cu_seqlens_k: torch.Tensor, max_seqlen_q: int, max_seqlen_k: int, block_mask: torch.Tensor,
                                is_causal: bool = False, qk_quant_gran: str = "per_thread", sm_scale: Optional[float] = None,
                                pv_accum_dtype: str = "fp32+fp16", smooth_k: bool = True, smooth_v: bool = False,
                                return_lse: bool = False):
    """Block-sparse attention on packed sequences (no reference counterpart): sageattn_varlen_qk_int8_pv_fp8_cuda with the block
    mask of sageattn_blocksparse applied inside each sequence.  The options, checks, warnings, V ranges and packed layout are
    those of sageattn_varlen_qk_int8_pv_fp8_cuda (GQA, int32 / int64 cu_seqlens, empty sequences, max_seqlen_* >= every length).

    block_mask: torch.bool on q's device, shape [nseq or 1, Hq or 1, ceil(max_seqlen_q/128), ceil(max_seqlen_k/64)] (size-1
    dimensions broadcast, any strides), indexed by the Q head under GQA.  Key j of sequence b is visible to its query i iff
    block_mask[b, h, i // 128, j // 64], with the blocks of each sequence starting at its own first token (as its INT8 blocks do),
    and j <= i when is_causal.  Entries past sequence b's own ceil(Lq_b/128) x ceil(Lk_b/64) blocks are ignored.  A wrong shape
    raises ValueError before any launch; max_seqlen_k <= 1048576.  The mask costs nseq * Hq * ceil(max_seqlen_q/128) *
    ceil(max_seqlen_k/64) bytes when not broadcast (about 6 MB for six sequences of up to 16384 tokens and 32 heads).

    Contract: "sageattn_blocksparse, per sequence".  Sequence b's output rows are the bits of sageattn_blocksparse(q_b[None],
    k_b[None], v_b[None], block_mask[b, :, :nq_b, :nk_b][None], tensor_layout="NHD", <same options>) for every sequence the dense
    call accepts (non-causal, or causal with Lq == Lk); every statistic is per sequence.  is_causal is top-left inside each
    sequence, Lq != Lk allowed (no dense counterpart): key j is visible to query i iff the mask allows tile (i // 128, j // 64)
    and j <= i.  With an all-True mask the result (o, lse, dq, dk, dv) is that of sageattn_varlen_qk_int8_pv_fp8_cuda to the bit.

    A row with no visible key gives 0 and lse -inf; rows past cu_seqlens_q[-1] are not written.  return_lse gives [Hq,Tq] in
    natural-log units with sageattn_varlen_qk_int8_pv_fp8_cuda's caveat: the kernel's LSE is exact, the per-token K-mean correction
    within one unit.  Differentiable when grad mode is on and q, k or v requires grad: for every sequence, dq / dk / dv are the bits
    of the dense block-sparse backward of the one-sequence call; tokens past the end, keys of a sequence without queries and keys
    hidden from every row get zero gradients.  The mask has no gradient."""
    _check_inputs(q, k, v)
    assert isinstance(block_mask, torch.Tensor) and block_mask.dtype == torch.bool, "block_mask must be a torch.bool tensor."
    assert block_mask.device == q.device, "All tensors must be on the same device."
    return _varlen_qk_int8_pv_fp8(q, k, v, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k, is_causal, qk_quant_gran, sm_scale,
                                  pv_accum_dtype, smooth_k, smooth_v, return_lse, block_mask=block_mask)


def _varlen_qk_int8_pv_fp8(q, k, v, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k, is_causal, qk_quant_gran, sm_scale,
                           pv_accum_dtype, smooth_k, smooth_v, return_lse, window=None, block_mask=None):
    """Body of sageattn_varlen_qk_int8_pv_fp8_cuda after _check_inputs; window: the (left, right) of sageattn_varlen_window, checked
    by the caller (_check_window_size) and clamped here (_varlen_window_arg); block_mask: the mask of sageattn_varlen_blocksparse,
    checked and expanded here (_varlen_block_mask) once the sequence tables are."""
    assert qk_quant_gran in ["per_warp", "per_thread"], "qk_quant_gran must be either 'per_warp' or 'per_thread'."
    if pv_accum_dtype not in ("fp32", "fp32+fp32", "fp32+fp16"):
        raise ValueError(f"Unsupported pv_accum_dtype: {pv_accum_dtype}")
    _check_cu_seqlens(q, k, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k)
    if k.shape != v.shape:
        raise ValueError(f"k and v must have the same shape (got {tuple(k.shape)} and {tuple(v.shape)})")
    if q.size(1) % k.size(1) != 0:
        raise ValueError(f"num_qo_heads ({q.size(1)}) must be divisible by num_kv_heads ({k.size(1)})")
    if block_mask is not None:
        block_mask = _varlen_block_mask(block_mask, q, cu_seqlens_q, int(max_seqlen_q), int(max_seqlen_k))
    q, k, v, head_dim_og = _pad_head_dim(q, k, v)
    assert q.stride(-1) == 1 and k.stride(-1) == 1 and v.stride(-1) == 1, "Last dim of qkv must be contiguous."
    if sm_scale is None:
        sm_scale = head_dim_og ** -0.5
    if pv_accum_dtype in ("fp32+fp32", "fp32+fp16") and smooth_v:
        warnings.warn(f"pv_accum_dtype is '{pv_accum_dtype}', smooth_v will be ignored.")
        smooth_v = False
    v_range = 2.25 if pv_accum_dtype == "fp32+fp16" else 448.0
    if window is not None:
        window = _varlen_window_arg(window, int(max_seqlen_q), int(max_seqlen_k))
    cu_q, cu_k = cu_seqlens_q.to(torch.int32).contiguous(), cu_seqlens_k.to(torch.int32).contiguous()
    args = (cu_q, cu_k, int(max_seqlen_q), int(max_seqlen_k), is_causal, qk_quant_gran, sm_scale, smooth_k, smooth_v, v_range)
    if torch.is_grad_enabled() and (q.requires_grad or k.requires_grad or v.requires_grad):
        o, lse, km = _SageAttnVarlenFp8Function.apply(q, k, v, *args, block_mask, window)
        q = q.detach()
    else:
        o, lse, km = _attn_varlen_f8(q, k, v, *args, return_lse, block_mask, window)
    o = o[..., :head_dim_og]
    if return_lse:
        if smooth_k:
            return o, lse / _LOG2E + _lse_correction_varlen(q, km, cu_q) * sm_scale
        return o, lse / _LOG2E
    return o


# ------------------------------------------------------------------------------------------------ paged KV cache
def _check_on_cuda(q):
    if not q.is_cuda:
        raise ValueError("q must be a CUDA tensor: there is no CPU implementation")


def _check_kvcache(q, k_cache, v_cache, cu_seqlens_q, seqused_k, block_table, max_seqlen_q):
    """The shape, dtype and device rules of sageattn_varlen_kvcache, or ValueError (the CUDA device itself: _check_on_cuda)."""
    if not isinstance(q, torch.Tensor) or q.dtype not in (torch.float16, torch.bfloat16) or q.dim() != 3:
        raise ValueError("q must be a packed [Tq, Hq, D] fp16 / bf16 tensor")
    _check_on_cuda(q)
    for name, c in (("k_cache", k_cache), ("v_cache", v_cache)):
        if not isinstance(c, torch.Tensor) or c.dim() != 4:
            raise ValueError(f"{name} must be a [num_pages, page_size, Hkv, D] tensor")
        if c.device != q.device or c.dtype != q.dtype:
            raise ValueError(f"{name} must have q's device and dtype ({q.device}, {q.dtype}), got ({c.device}, {c.dtype})")
        if c.stride(-1) != 1 or c.data_ptr() % 16 != 0 or any(s % 8 != 0 for s in c.stride()[:3]):
            raise ValueError(f"{name} needs stride(-1) == 1 and 16-byte aligned rows (other strides multiples of 8 elements)")
    if k_cache.shape != v_cache.shape:
        raise ValueError(f"k_cache and v_cache must have the same shape (got {tuple(k_cache.shape)} and {tuple(v_cache.shape)})")
    num_pages, page_size, Hkv, D = k_cache.shape
    if D not in (64, 128) or q.size(2) != D:
        raise ValueError(f"the head dim must be 64 or 128 and the same for q and the cache (q {q.size(2)}, cache {D})")
    if num_pages < 1 or page_size < 1 or Hkv < 1 or q.size(1) % Hkv != 0:
        raise ValueError(f"num_qo_heads ({q.size(1)}) must be divisible by num_kv_heads ({Hkv}), and the cache must not be empty")
    if not isinstance(cu_seqlens_q, torch.Tensor) or cu_seqlens_q.dim() != 1 or cu_seqlens_q.dtype not in (torch.int32, torch.int64) \
            or cu_seqlens_q.numel() < 2 or cu_seqlens_q.device != q.device:
        raise ValueError("cu_seqlens_q must be a 1-D int32 or int64 tensor of nseq + 1 >= 2 offsets on q's device")
    nseq = cu_seqlens_q.numel() - 1
    if not isinstance(seqused_k, torch.Tensor) or tuple(seqused_k.shape) != (nseq,) or seqused_k.dtype != torch.int32 \
            or seqused_k.device != q.device:
        raise ValueError(f"seqused_k must be an int32 [{nseq}] tensor on q's device")
    if not isinstance(block_table, torch.Tensor) or block_table.dim() != 2 or block_table.size(0) != nseq or block_table.size(1) < 1 \
            or block_table.dtype != torch.int32 or block_table.device != q.device or block_table.stride(1) != 1:
        raise ValueError(f"block_table must be an int32 [{nseq}, max_pages] tensor on q's device with contiguous rows")
    if isinstance(max_seqlen_q, bool) or not isinstance(max_seqlen_q, numbers.Integral) or max_seqlen_q < 1:
        raise ValueError(f"max_seqlen_q must be an int >= 1, got {max_seqlen_q!r}")
    if q.size(0) == 0:
        raise ValueError("the packed batch must hold at least one query")


def sageattn_varlen_kvcache(q: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, cu_seqlens_q: torch.Tensor,
                            seqused_k: torch.Tensor, block_table: torch.Tensor, max_seqlen_q: int, is_causal: bool = False,
                            qk_quant_gran: str = "per_thread", sm_scale: Optional[float] = None, pv_accum_dtype: str = "fp32+fp16",
                            smooth_k: bool = True, smooth_v: bool = False, return_lse: bool = False):
    """Attention of packed queries against a paged KV cache (no reference counterpart): chunked prefill, prefix caching and
    speculative verification, where each sequence's Lq_b new queries attend to Lk_b >= Lq_b keys of which the earlier ones are cached.

    q: packed [Tq,Hq,D] with cu_seqlens_q (int32 or int64, nseq + 1 offsets) and max_seqlen_q, as in
    sageattn_varlen_qk_int8_pv_fp8_cuda.  k_cache / v_cache: [num_pages, page_size, Hkv, D], the same shape, q's dtype, D 64 or 128
    (no head-dim padding: it would copy the cache), Hq % Hkv == 0, stride(-1) == 1 and 16-byte aligned rows; other strides are free,
    so a view such as kv_cache[0] of a [2, num_pages, ...] buffer is accepted.  block_table: int32 [nseq, max_pages]; token t of
    sequence b is k_cache[block_table[b, t // page_size], t % page_size].  Pages may be shared between sequences (prefix sharing).
    Entries past ceil(seqused_k[b] / page_size) are never read, nor are slots past seqused_k[b] in the last page.  Every entry read
    must lie in [0, num_pages): like the cu_seqlens values, the table is trusted.  A padded, unpaged cache [nseq, S_cap, Hkv, D] is
    the case page_size = S_cap, block_table = arange(nseq)[:, None].  seqused_k: int32 [nseq] on the device, Lk_b.

    Synchronisation: the call copies seqused_k to the host once (the other packed entry points do not synchronise).  The host copy
    checks 0 <= Lk_b <= max_pages * page_size (ValueError before any launch) and sizes the packed quantised K / V exactly.  The
    quantisers read the pages directly: there is no gathered 16-bit copy of the cache.  Shape, dtype and device errors raise
    ValueError before any launch; every other option (checks, warnings, V ranges, smooth_v rules) is that of
    sageattn_varlen_qk_int8_pv_fp8_cuda.

    Contract, with K_b / V_b the first Lk_b tokens of sequence b gathered from its pages:
      * non-causal: the bits of sageattn_varlen_qk_int8_pv_fp8_cuda(q, Kp, Vp, cu_seqlens_q, [0, cumsum(seqused_k)], ...) on the
        gathered sequences packed; every statistic (K mean, INT8 blocks, V scale and mean) is per sequence;
      * is_causal: bottom-right, query i of sequence b sees key j iff j <= i + Lk_b - Lq_b.  For Lk_b >= Lq_b, sequence b's rows are
        the bits of sageattn_window(q_b[None], K_b[None], V_b[None], window_size=(-1, Lk_b - Lq_b), tensor_layout="NHD",
        is_causal=False, <same options>).  For Lk_b < Lq_b its first Lq_b - Lk_b rows see no key;
      * a row that sees no key (Lk_b = 0, or the rows above) returns 0 and lse -inf; a sequence with Lq_b = 0 writes nothing, and rows
        past cu_seqlens_q[-1] are not written.
    return_lse: also returns the [Hq,Tq] fp32 LSE in natural-log units, with sageattn_varlen_qk_int8_pv_fp8_cuda's caveat on the
    per-token K-mean correction.  Forward only: the output does not require grad."""
    _check_kvcache(q, k_cache, v_cache, cu_seqlens_q, seqused_k, block_table, max_seqlen_q)
    assert qk_quant_gran in ["per_warp", "per_thread"], "qk_quant_gran must be either 'per_warp' or 'per_thread'."
    if pv_accum_dtype not in ("fp32", "fp32+fp32", "fp32+fp16"):
        raise ValueError(f"Unsupported pv_accum_dtype: {pv_accum_dtype}")
    page_size = k_cache.size(1)
    lk = seqused_k.cpu().tolist()                       # the call's one device -> host copy
    cap = block_table.size(1) * page_size
    if any(n < 0 or n > cap for n in lk):
        raise ValueError(f"seqused_k must lie in [0, max_pages * page_size] = [0, {cap}], got {lk}")
    if sm_scale is None:
        sm_scale = q.size(2) ** -0.5
    if pv_accum_dtype in ("fp32+fp32", "fp32+fp16") and smooth_v:
        warnings.warn(f"pv_accum_dtype is '{pv_accum_dtype}', smooth_v will be ignored.")
        smooth_v = False
    v_range = 2.25 if pv_accum_dtype == "fp32+fp16" else 448.0
    max_seqlen_q = int(max_seqlen_q)
    total_k, max_seqlen_k = sum(lk), max(lk)
    with torch.no_grad():
        if total_k == 0:                                # no sequence has a key: every row sees nothing
            o = torch.zeros_like(q)
            return (o, torch.full((q.size(1), q.size(0)), -float("inf"), dtype=torch.float32, device=q.device)) if return_lse else o
        cu_q = cu_seqlens_q.to(torch.int32).contiguous()
        cu_k = torch.nn.functional.pad(torch.cumsum(seqused_k, 0, dtype=torch.int32), (1, 0))
        k_blocks = sum((n + 63) // 64 for n in lk)
        t_pad = sum((n + 127) // 128 * 128 for n in lk)
        km = k_mean_paged(k_cache, cu_k, block_table, max_seqlen_k) if smooth_k else None
        q_int8, q_scale, cu_q_scale = quant_q_int8_varlen(q, cu_q, max_seqlen_q, qk_quant_gran)
        k_int8, k_scale, cu_k_scale = quant_k_int8_paged(k_cache, km, cu_k, block_table, max_seqlen_k, total_k, k_blocks, qk_quant_gran)
        v_fp8, v_scale, vm, cu_pad = per_channel_fp8_paged(v_cache, cu_k, block_table, max_seqlen_k, t_pad, v_range, smooth_v)
        o = torch.empty(q.shape, dtype=q.dtype, device=q.device)
        gran = SAB_GRAN_PER_WARP if qk_quant_gran == "per_warp" else SAB_GRAN_PER_THREAD
        lse = ops.qk_int8_sv_f8_attn_varlen_bottom_right(q_int8, k_int8, v_fp8, o, q_scale, k_scale, v_scale, vm, cu_q, cu_k, cu_pad,
                                                         cu_q_scale, cu_k_scale, max_seqlen_q, 1 if is_causal else 0, gran, gran,
                                                         sm_scale, 1 if return_lse else 0)
        if return_lse:
            if smooth_k:
                return o, lse / _LOG2E + _lse_correction_varlen(q, km, cu_q) * sm_scale
            return o, lse / _LOG2E
        return o
