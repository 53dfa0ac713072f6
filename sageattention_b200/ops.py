"""torch.library custom-op shims over the C ABI (mirrors sageattention/sm89_compile.py:5-146 of the
reference: ops mutate pre-allocated outputs and have fake impls so they trace under torch.compile).

PyTorch is plumbing here: it owns device memory and the current stream; every op body is a single
call into libsageattn_b200.so through ctypes with raw pointers, sizes and strides.
"""
import math
from typing import Optional
import torch

from . import _capi
from ._capi import check, lib, SAB_MASK_BOOL, SAB_MASK_BIAS


def _stream(t: torch.Tensor) -> int:
    return torch.cuda.current_stream(t.device).cuda_stream


def _dt(t: torch.Tensor) -> int:
    if t.dtype == torch.float16:
        return _capi.SAB_DTYPE_FP16
    if t.dtype == torch.bfloat16:
        return _capi.SAB_DTYPE_BF16
    raise TypeError("Only half and bfloat16 are supported")


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else t.data_ptr()


def _v_pad(value: torch.Tensor) -> int:
    """Token extent of the transposed V operand ([..., D, S_pad]).  The C ABI takes no V strides: the kernel's tensor map
    assumes the packed layout the V quantisers write, so a strided view (e.g. a permuted all-gather buffer) is refused
    instead of read as the wrong keys."""
    if not value.is_contiguous():
        raise ValueError("value (quantised / transposed V) must be contiguous")
    return value.size(-1)


def _bhs_strides(t: torch.Tensor, tensor_layout: int):
    """(stride_b, stride_h, stride_s) in elements; tensor_layout 0 = NHD, 1 = HND (reference encoding)."""
    if tensor_layout == 1:
        return t.stride(0), t.stride(1), t.stride(2)
    return t.stride(0), t.stride(2), t.stride(1)


def _bhsd(t: torch.Tensor, tensor_layout: int):
    if tensor_layout == 1:
        return t.size(0), t.size(1), t.size(2), t.size(3)
    return t.size(0), t.size(2), t.size(1), t.size(3)


def _lse(query: torch.Tensor, rows, return_lse: int) -> torch.Tensor:
    """The lse a forward op returns, real and fake alike: fp32 of shape `rows` ((B, Hq, Sq) dense, (Hq, Tq) packed), or an
    empty tensor when return_lse == 0."""
    return query.new_empty(rows if return_lse else (0,), dtype=torch.float32)


# ----------------------------------------------------------------------------------------------- K mean
@torch.library.custom_op("sageattention_b200::k_mean", mutates_args=("mean",), device_types="cuda")
def k_mean(k: torch.Tensor, mean: torch.Tensor, tensor_layout: int) -> None:
    B, H, S, D = _bhsd(k, tensor_layout)
    sb, sh, ss = _bhs_strides(k, tensor_layout)
    with torch.cuda.device(k.device):
        ws = torch.empty(lib().sab_k_mean_workspace_bytes(B, H, S, D), dtype=torch.uint8, device=k.device)
        check(lib().sab_k_mean(k.data_ptr(), _dt(k), mean.data_ptr(), B, H, S, D, sb, sh, ss, ws.data_ptr(), _stream(k)))


@k_mean.register_fake
def _(k, mean, tensor_layout):
    return None


# ----------------------------------------------------------------------------------------------- fused single-pass front-end
@torch.library.custom_op("sageattention_b200::k_smooth_quant_int8", mutates_args=("mean", "output", "scale"), device_types="cuda")
def k_smooth_quant_int8(k: torch.Tensor, mean: torch.Tensor, output: torch.Tensor, scale: torch.Tensor, tensor_layout: int,
                        granularity: int) -> None:
    """K smoothing mean + INT8 quantisation of K in one launch (cluster per (b,h)); mean [B,H,D] in k.dtype is written too."""
    B, H, S, D = _bhsd(k, tensor_layout)
    xs, os_ = _bhs_strides(k, tensor_layout), _bhs_strides(output, tensor_layout)
    with torch.cuda.device(k.device):
        check(lib().sab_k_smooth_quant_int8(k.data_ptr(), _dt(k), mean.data_ptr(), output.data_ptr(), scale.data_ptr(), B, H, S, D,
                                            *xs, *os_, scale.size(-1), granularity, _stream(k)))


@k_smooth_quant_int8.register_fake
def _(k, mean, output, scale, tensor_layout, granularity):
    return None


@torch.library.custom_op("sageattention_b200::per_channel_fp8_fused", mutates_args=("v_fp8", "v_scale", "v_mean"), device_types="cuda")
def per_channel_fp8_fused(v: torch.Tensor, v_fp8: torch.Tensor, v_scale: torch.Tensor, v_mean: Optional[torch.Tensor],
                          tensor_layout: int, scale_max: float) -> None:
    """per_channel_fp8 (dense form) in one launch: per-channel statistics through a cluster reduction, then quantise + transpose."""
    B, H, S, D = _bhsd(v, tensor_layout)
    sb, sh, ss = _bhs_strides(v, tensor_layout)
    with torch.cuda.device(v.device):
        check(lib().sab_per_channel_fp8_fused(v.data_ptr(), _dt(v), v_fp8.data_ptr(), v_scale.data_ptr(), _ptr(v_mean), B, H, S, D,
                                              sb, sh, ss, v_fp8.size(-1), float(scale_max), _stream(v)))


@per_channel_fp8_fused.register_fake
def _(v, v_fp8, v_scale, v_mean, tensor_layout, scale_max):
    return None


# ----------------------------------------------------------------------------------------------- INT8 quant
@torch.library.custom_op("sageattention_b200::quant_per_block_int8", mutates_args=("output", "scale"), device_types="cuda")
def quant_per_block_int8(input: torch.Tensor, mean: Optional[torch.Tensor], output: torch.Tensor, scale: torch.Tensor,
                         block_size: int, tensor_layout: int, semantics: int, has_sm_scale: bool, sm_scale: float) -> None:
    B, H, S, D = _bhsd(input, tensor_layout)
    xs, os_ = _bhs_strides(input, tensor_layout), _bhs_strides(output, tensor_layout)
    with torch.cuda.device(input.device):
        check(lib().sab_quant_per_block_int8(input.data_ptr(), _dt(input), _ptr(mean), output.data_ptr(), scale.data_ptr(),
                                             B, H, S, D, *xs, *os_, scale.size(-1), block_size, semantics,
                                             1 if has_sm_scale else 0, float(sm_scale), _stream(input)))


@quant_per_block_int8.register_fake
def _(input, mean, output, scale, block_size, tensor_layout, semantics, has_sm_scale, sm_scale):
    return None


@torch.library.custom_op("sageattention_b200::quant_per_thread_int8", mutates_args=("output", "scale"), device_types="cuda")
def quant_per_thread_int8(input: torch.Tensor, mean: Optional[torch.Tensor], output: torch.Tensor, scale: torch.Tensor,
                          tensor_layout: int, is_key: bool) -> None:
    B, H, S, D = _bhsd(input, tensor_layout)
    xs, os_ = _bhs_strides(input, tensor_layout), _bhs_strides(output, tensor_layout)
    with torch.cuda.device(input.device):
        check(lib().sab_quant_per_thread_int8(input.data_ptr(), _dt(input), _ptr(mean), output.data_ptr(), scale.data_ptr(),
                                              B, H, S, D, *xs, *os_, scale.size(-1), 1 if is_key else 0, _stream(input)))


@quant_per_thread_int8.register_fake
def _(input, mean, output, scale, tensor_layout, is_key):
    return None


@torch.library.custom_op("sageattention_b200::quant_per_block_int8_varlen", mutates_args=("output", "scale"), device_types="cuda")
def quant_per_block_int8_varlen(input: torch.Tensor, mean: Optional[torch.Tensor], output: torch.Tensor, scale: torch.Tensor,
                                cu_seqlens: torch.Tensor, cu_scale: torch.Tensor, max_seqlen: int, block_size: int,
                                has_sm_scale: bool, sm_scale: float) -> None:
    T, H, D = input.shape
    with torch.cuda.device(input.device):
        check(lib().sab_quant_per_block_int8_varlen(input.data_ptr(), _dt(input), _ptr(mean), output.data_ptr(), scale.data_ptr(),
                                                    cu_seqlens.data_ptr(), cu_scale.data_ptr(), cu_seqlens.numel() - 1,
                                                    max_seqlen, H, D, input.stride(0), input.stride(1), output.stride(0),
                                                    output.stride(1), block_size, 1 if has_sm_scale else 0, float(sm_scale),
                                                    _stream(input)))


@quant_per_block_int8_varlen.register_fake
def _(input, mean, output, scale, cu_seqlens, cu_scale, max_seqlen, block_size, has_sm_scale, sm_scale):
    return None


# ----------------------------------------------------------------------------------------------- FP8 V
@torch.library.custom_op("sageattention_b200::per_channel_fp8", mutates_args=("v_fp8", "v_scale", "v_mean"), device_types="cuda")
def per_channel_fp8(v: torch.Tensor, v_fp8: torch.Tensor, v_scale: torch.Tensor, v_mean: Optional[torch.Tensor],
                    tensor_layout: int, scale_max: float) -> None:
    B, H, S, D = _bhsd(v, tensor_layout)
    sb, sh, ss = _bhs_strides(v, tensor_layout)
    with torch.cuda.device(v.device):
        ws = torch.empty(lib().sab_per_channel_fp8_workspace_bytes(B, H, S, D), dtype=torch.uint8, device=v.device)
        check(lib().sab_per_channel_fp8(v.data_ptr(), _dt(v), v_fp8.data_ptr(), v_scale.data_ptr(), _ptr(v_mean), B, H, S, D,
                                        sb, sh, ss, v_fp8.size(-1), float(scale_max), None, None, 0, 0, ws.data_ptr(), _stream(v)))


@per_channel_fp8.register_fake
def _(v, v_fp8, v_scale, v_mean, tensor_layout, scale_max):
    return None


@torch.library.custom_op("sageattention_b200::per_channel_fp8_varlen", mutates_args=("v_fp8", "v_scale"), device_types="cuda")
def per_channel_fp8_varlen(v: torch.Tensor, v_fp8: torch.Tensor, v_scale: torch.Tensor, cu_seqlens: torch.Tensor,
                           cu_pad: torch.Tensor, max_seqlen: int, scale_max: float) -> None:
    T, H, D = v.shape
    with torch.cuda.device(v.device):
        ws = torch.empty(lib().sab_per_channel_fp8_workspace_bytes(1, H, T, D), dtype=torch.uint8, device=v.device)
        check(lib().sab_per_channel_fp8(v.data_ptr(), _dt(v), v_fp8.data_ptr(), v_scale.data_ptr(), None, 1, H, T, D,
                                        0, v.stride(1), v.stride(0), v_fp8.size(-1), float(scale_max), cu_seqlens.data_ptr(),
                                        cu_pad.data_ptr(), cu_seqlens.numel() - 1, max_seqlen, ws.data_ptr(), _stream(v)))


@per_channel_fp8_varlen.register_fake
def _(v, v_fp8, v_scale, cu_seqlens, cu_pad, max_seqlen, scale_max):
    return None


# ----------------------------------------------------------------------------------------------- SP building blocks
@torch.library.custom_op("sageattention_b200::channel_stats", mutates_args=("sum_out", "max_out", "min_out"), device_types="cuda")
def channel_stats(x: torch.Tensor, sum_out: torch.Tensor, max_out: torch.Tensor, min_out: torch.Tensor, tensor_layout: int) -> None:
    B, H, S, D = _bhsd(x, tensor_layout)
    sb, sh, ss = _bhs_strides(x, tensor_layout)
    with torch.cuda.device(x.device):
        ws = torch.empty(lib().sab_k_mean_workspace_bytes(B, H, S, D), dtype=torch.uint8, device=x.device)
        check(lib().sab_channel_stats(x.data_ptr(), _dt(x), sum_out.data_ptr(), max_out.data_ptr(), min_out.data_ptr(),
                                      B, H, S, D, sb, sh, ss, ws.data_ptr(), _stream(x)))


@channel_stats.register_fake
def _(x, sum_out, max_out, min_out, tensor_layout):
    return None


@torch.library.custom_op("sageattention_b200::v_quant_with_amax", mutates_args=("v_fp8", "v_scale"), device_types="cuda")
def v_quant_with_amax(v: torch.Tensor, v_fp8: torch.Tensor, amax: torch.Tensor, v_scale: torch.Tensor, tensor_layout: int,
                      scale_max: float) -> None:
    B, H, S, D = _bhsd(v, tensor_layout)
    sb, sh, ss = _bhs_strides(v, tensor_layout)
    with torch.cuda.device(v.device):
        ws = torch.empty(B * H * D * 4, dtype=torch.uint8, device=v.device)
        check(lib().sab_v_quant_with_amax(v.data_ptr(), _dt(v), v_fp8.data_ptr(), amax.data_ptr(), v_scale.data_ptr(), B, H, S, D,
                                          sb, sh, ss, v_fp8.size(-1), float(scale_max), ws.data_ptr(), _stream(v)))


@v_quant_with_amax.register_fake
def _(v, v_fp8, amax, v_scale, tensor_layout, scale_max):
    return None


# ----------------------------------------------------------------------------------------------- attention
@torch.library.custom_op("sageattention_b200::qk_int8_sv_f8_attn", mutates_args=("output",), device_types="cuda")
def qk_int8_sv_f8_attn(query: torch.Tensor, key: torch.Tensor, value: torch.Tensor, output: torch.Tensor,
                       query_scale: torch.Tensor, key_scale: torch.Tensor, value_scale: Optional[torch.Tensor],
                       value_mean: Optional[torch.Tensor], tensor_layout: int, is_causal: int, q_quant_gran: int,
                       k_quant_gran: int, sm_scale: float, fold_sm_scale: int, return_lse: int,
                       causal_q_offset: int = 0, kv_seg_len: int = 0) -> torch.Tensor:
    """Same contract as the reference op (sm89_compile.py:48-66): mutates `output`, returns lse
    ([B,Hq,Sq] fp32 in log2 units, or an empty tensor when return_lse == 0).
    kv_seg_len > 0: key/value are the rank-major all-gather of P shards ([P*B,Hkv,kv_seg_len,D] /
    [P*B,Hkv,D,kv_seg_len]); causal_q_offset is the global index of query row 0."""
    B, Hq, Sq, D = _bhsd(query, tensor_layout)
    _, Hkv, Skv, _ = _bhsd(key, tensor_layout)
    if kv_seg_len > 0:
        Skv = (key.size(0) // B) * kv_seg_len
    qs, ks, os_ = _bhs_strides(query, tensor_layout), _bhs_strides(key, tensor_layout), _bhs_strides(output, tensor_layout)
    lse = _lse(query, (B, Hq, Sq), return_lse)
    with torch.cuda.device(query.device):
        check(lib().sab_qk_int8_sv_f8_attn(query.data_ptr(), key.data_ptr(), value.data_ptr(), output.data_ptr(),
                                           lse.data_ptr() if return_lse else None, query_scale.data_ptr(), key_scale.data_ptr(),
                                           _ptr(value_scale), _ptr(value_mean), _dt(output), B, Hq, Hkv, Sq, Skv, D,
                                           *qs, *ks, _v_pad(value), *os_, is_causal, q_quant_gran, k_quant_gran,
                                           float(sm_scale), fold_sm_scale, None, None, None, None, None, 0,
                                           causal_q_offset, kv_seg_len, None, _stream(query)))
    return lse


@qk_int8_sv_f8_attn.register_fake
def _(query, key, value, output, query_scale, key_scale, value_scale, value_mean, tensor_layout, is_causal,
      q_quant_gran, k_quant_gran, sm_scale, fold_sm_scale, return_lse, causal_q_offset=0, kv_seg_len=0):
    B, Hq, Sq, D = _bhsd(query, tensor_layout)
    return _lse(query, (B, Hq, Sq), return_lse)


def _block_mask_args(block_mask: torch.Tensor, B: int, Hq: int, Sq: int, Skv: int):
    """(pointer, stride_b, stride_h, stride_qb, stride_kb) of a bool [B,Hq,ceil(Sq/128),ceil(Skv/64)] view (strides may be 0)."""
    shape = (B, Hq, (Sq + 127) // 128, (Skv + 63) // 64)
    assert block_mask.dtype == torch.bool and tuple(block_mask.shape) == shape, \
        f"block_mask must be a bool view of shape {shape}"
    return (block_mask.data_ptr(), *block_mask.stride())


@torch.library.custom_op("sageattention_b200::qk_int8_sv_f8_attn_blocksparse", mutates_args=("output",), device_types="cuda")
def qk_int8_sv_f8_attn_blocksparse(query: torch.Tensor, key: torch.Tensor, value: torch.Tensor, output: torch.Tensor,
                                   query_scale: torch.Tensor, key_scale: torch.Tensor, value_scale: Optional[torch.Tensor],
                                   value_mean: Optional[torch.Tensor], block_mask: torch.Tensor, tensor_layout: int,
                                   is_causal: int, q_quant_gran: int, k_quant_gran: int, sm_scale: float, fold_sm_scale: int,
                                   return_lse: int) -> torch.Tensor:
    """qk_int8_sv_f8_attn restricted to the visible tiles of block_mask (include/sageattn_b200.h,
    sab_qk_int8_sv_f8_attn_blocksparse): a bool view [B,Hq,ceil(Sq/128),ceil(Skv/64)], strides may be 0.  Returns lse as
    qk_int8_sv_f8_attn does; a row with no visible key gets 0 and lse -inf."""
    B, Hq, Sq, D = _bhsd(query, tensor_layout)
    _, Hkv, Skv, _ = _bhsd(key, tensor_layout)
    mask = _block_mask_args(block_mask, B, Hq, Sq, Skv)
    qs, ks, os_ = _bhs_strides(query, tensor_layout), _bhs_strides(key, tensor_layout), _bhs_strides(output, tensor_layout)
    lse = _lse(query, (B, Hq, Sq), return_lse)
    with torch.cuda.device(query.device):
        check(lib().sab_qk_int8_sv_f8_attn_blocksparse(query.data_ptr(), key.data_ptr(), value.data_ptr(), output.data_ptr(),
                                                       lse.data_ptr() if return_lse else None, query_scale.data_ptr(),
                                                       key_scale.data_ptr(), _ptr(value_scale), _ptr(value_mean), _dt(output), B, Hq,
                                                       Hkv, Sq, Skv, D, *qs, *ks, _v_pad(value), *os_, is_causal, q_quant_gran,
                                                       k_quant_gran, float(sm_scale), fold_sm_scale, *mask, _stream(query)))
    return lse


@qk_int8_sv_f8_attn_blocksparse.register_fake
def _(query, key, value, output, query_scale, key_scale, value_scale, value_mean, block_mask, tensor_layout, is_causal,
      q_quant_gran, k_quant_gran, sm_scale, fold_sm_scale, return_lse):
    B, Hq, Sq, D = _bhsd(query, tensor_layout)
    return _lse(query, (B, Hq, Sq), return_lse)


@torch.library.custom_op("sageattention_b200::qk_int8_sv_f8_attn_window", mutates_args=("output",), device_types="cuda")
def qk_int8_sv_f8_attn_window(query: torch.Tensor, key: torch.Tensor, value: torch.Tensor, output: torch.Tensor,
                              query_scale: torch.Tensor, key_scale: torch.Tensor, value_scale: Optional[torch.Tensor],
                              value_mean: Optional[torch.Tensor], window_left: int, window_right: int, tensor_layout: int,
                              is_causal: int, q_quant_gran: int, k_quant_gran: int, sm_scale: float, fold_sm_scale: int,
                              return_lse: int) -> torch.Tensor:
    """qk_int8_sv_f8_attn restricted to a sliding window (include/sageattn_b200.h, sab_qk_int8_sv_f8_attn_window): key j is
    visible to query i iff i - window_left <= j <= i + window_right (-1: that side unbounded), and j <= i when causal.  Returns
    lse as qk_int8_sv_f8_attn does; a row with no visible key gets 0 and lse -inf."""
    B, Hq, Sq, D = _bhsd(query, tensor_layout)
    _, Hkv, Skv, _ = _bhsd(key, tensor_layout)
    qs, ks, os_ = _bhs_strides(query, tensor_layout), _bhs_strides(key, tensor_layout), _bhs_strides(output, tensor_layout)
    lse = _lse(query, (B, Hq, Sq), return_lse)
    with torch.cuda.device(query.device):
        check(lib().sab_qk_int8_sv_f8_attn_window(query.data_ptr(), key.data_ptr(), value.data_ptr(), output.data_ptr(),
                                                  lse.data_ptr() if return_lse else None, query_scale.data_ptr(), key_scale.data_ptr(),
                                                  _ptr(value_scale), _ptr(value_mean), _dt(output), B, Hq, Hkv, Sq, Skv, D, *qs, *ks,
                                                  _v_pad(value), *os_, is_causal, q_quant_gran, k_quant_gran, float(sm_scale),
                                                  fold_sm_scale, window_left, window_right, _stream(query)))
    return lse


@qk_int8_sv_f8_attn_window.register_fake
def _(query, key, value, output, query_scale, key_scale, value_scale, value_mean, window_left, window_right, tensor_layout,
      is_causal, q_quant_gran, k_quant_gran, sm_scale, fold_sm_scale, return_lse):
    B, Hq, Sq, D = _bhsd(query, tensor_layout)
    return _lse(query, (B, Hq, Sq), return_lse)


@torch.library.custom_op("sageattention_b200::qk_int8_sv_f8_attn_sp", mutates_args=("output",), device_types="cuda")
def qk_int8_sv_f8_attn_sp(query: torch.Tensor, key: torch.Tensor, value: torch.Tensor, output: torch.Tensor,
                          query_scale: torch.Tensor, key_scale: torch.Tensor, value_scale: torch.Tensor, q_quant_gran: int,
                          k_quant_gran: int, sm_scale: float, kv_seg_len: int, seg_flags: torch.Tensor, seg_epoch: int,
                          heads_per_flag: int) -> None:
    """Sequence-parallel attention whose K/V segments may still be arriving (include/sageattn_b200.h, sab_qk_int8_sv_f8_attn_sp):
    HND tensors, key [P*B,Hkv,kv_seg_len,D] / value [P*B,Hkv,D,kv_seg_len] rank-major, seg_flags uint32 [Hkv/heads_per_flag * P];
    the kernel waits for seg_flags[group * P + segment] == seg_epoch before the first tile of a segment.  Non-causal."""
    B, Hq, Sq, D = query.shape
    Hkv = key.size(1)
    P = key.size(0) // B
    assert seg_flags.dtype in (torch.int32, torch.uint32) and seg_flags.is_contiguous() and seg_flags.numel() >= (Hkv // heads_per_flag) * P
    qs, ks, os_ = _bhs_strides(query, 1), _bhs_strides(key, 1), _bhs_strides(output, 1)
    with torch.cuda.device(query.device):
        check(lib().sab_qk_int8_sv_f8_attn_sp(query.data_ptr(), key.data_ptr(), value.data_ptr(), output.data_ptr(), None,
                                              query_scale.data_ptr(), key_scale.data_ptr(), value_scale.data_ptr(), _dt(output),
                                              B, Hq, Hkv, Sq, P * kv_seg_len, D, *qs, *ks, _v_pad(value), *os_, q_quant_gran,
                                              k_quant_gran, float(sm_scale), kv_seg_len, seg_flags.data_ptr(),
                                              int(seg_epoch) & 0xFFFFFFFF, heads_per_flag, _stream(query)))


@qk_int8_sv_f8_attn_sp.register_fake
def _(query, key, value, output, query_scale, key_scale, value_scale, q_quant_gran, k_quant_gran, sm_scale, kv_seg_len,
      seg_flags, seg_epoch, heads_per_flag):
    return None


@torch.library.custom_op("sageattention_b200::qk_int8_sv_f8_attn_varlen", mutates_args=("output",), device_types="cuda")
def qk_int8_sv_f8_attn_varlen(query: torch.Tensor, key: torch.Tensor, value: torch.Tensor, output: torch.Tensor,
                              query_scale: torch.Tensor, key_scale: torch.Tensor, value_scale: torch.Tensor,
                              cu_seqlens_q: torch.Tensor, cu_seqlens_k: torch.Tensor, cu_pad_v: torch.Tensor,
                              cu_q_scale: torch.Tensor, cu_k_scale: torch.Tensor, max_seqlen_q: int, is_causal: int,
                              sm_scale: float, fold_sm_scale: int) -> None:
    Tq, Hq, D = query.shape
    Tk, Hkv, _ = key.shape
    nseq = cu_seqlens_q.numel() - 1
    with torch.cuda.device(query.device):
        check(lib().sab_qk_int8_sv_f8_attn(query.data_ptr(), key.data_ptr(), value.data_ptr(), output.data_ptr(), None,
                                           query_scale.data_ptr(), key_scale.data_ptr(), value_scale.data_ptr(), None,
                                           _dt(output), nseq, Hq, Hkv, Tq, Tk, D,
                                           0, query.stride(1), query.stride(0), 0, key.stride(1), key.stride(0),
                                           _v_pad(value), 0, output.stride(1), output.stride(0), is_causal,
                                           _capi.SAB_GRAN_PER_BLOCK, _capi.SAB_GRAN_PER_BLOCK, float(sm_scale), fold_sm_scale,
                                           cu_seqlens_q.data_ptr(), cu_seqlens_k.data_ptr(), cu_pad_v.data_ptr(),
                                           cu_q_scale.data_ptr(), cu_k_scale.data_ptr(), max_seqlen_q, 0, 0, None, _stream(query)))


@qk_int8_sv_f8_attn_varlen.register_fake
def _(query, key, value, output, query_scale, key_scale, value_scale, cu_seqlens_q, cu_seqlens_k, cu_pad_v,
      cu_q_scale, cu_k_scale, max_seqlen_q, is_causal, sm_scale, fold_sm_scale):
    return None


# ----------------------------------------------------------------------------------------------- backward
def _bwd_operands(q_int8, k_int8, q, k, v, o, dout, lse, k_mean, dq, dk, dv, tensor_layout, lse_shape, k_mean_shape, k_mean_label):
    """The operand checks of every backward op.  The kernels read o and dout at q's sizes as 16-bit words, and q_int8 / k_int8 at
    q's / k's sizes as bytes: a smaller tensor would be read out of bounds, another dtype as the wrong words.  tensor_layout None:
    packed [T,H,D] tensors and lse_shape (Hq, Tq), else lse_shape (B, Hq, Sq).  k_mean_label: the element count of k_mean_shape
    as the message names it.  Returns the (b, h, s) strides ((t, h) packed) of q_int8, k_int8, q, k, v, o, dout, k_mean reshaped
    to k_mean_shape and the delta workspace."""
    for x, y in ((dq, q), (dk, k), (dv, v)):
        assert x.stride() == y.stride() and x.dtype == y.dtype, "dq / dk / dv must have the strides and dtype of q / k / v"
    for name, t in (("o", o), ("dout", dout)):
        assert t.shape == q.shape and t.dtype == q.dtype, f"{name} must have q's shape and dtype"
    for name, t, ref in (("q_int8", q_int8, q), ("k_int8", k_int8, k)):
        assert t.shape == ref.shape and t.dtype == torch.int8, f"{name} must be int8 with the shape of {name[0]}"
    packed = tensor_layout is None
    assert lse.dtype == torch.float32 and lse.is_contiguous() and tuple(lse.shape) == lse_shape, \
        f"lse must be {'[Hq,Tq]' if packed else '[B,Hq,Sq]'} fp32"
    strides = [s for t in (q_int8, k_int8, q, k, v, o, dout)
               for s in ((t.stride(0), t.stride(1)) if packed else _bhs_strides(t, tensor_layout))]
    if k_mean is not None:
        assert k_mean.numel() == math.prod(k_mean_shape) and k_mean.dtype == k.dtype, \
            f"k_mean must have {k_mean_label} elements of k's dtype"
        k_mean = k_mean.reshape(k_mean_shape).contiguous()
    ws_shape = (1, *lse_shape) if packed else lse_shape
    ws = torch.empty(lib().sab_attn_bwd_workspace_bytes(*ws_shape), dtype=torch.uint8, device=q.device)
    return strides, k_mean, ws


@torch.library.custom_op("sageattention_b200::qk_int8_attn_bwd", mutates_args=("dq", "dk", "dv"), device_types="cuda")
def qk_int8_attn_bwd(q_int8: torch.Tensor, k_int8: torch.Tensor, q_scale: torch.Tensor, k_scale: torch.Tensor, q: torch.Tensor,
                     k: torch.Tensor, v: torch.Tensor, o: torch.Tensor, dout: torch.Tensor, lse: torch.Tensor,
                     k_mean: Optional[torch.Tensor], dq: torch.Tensor, dk: torch.Tensor, dv: torch.Tensor, tensor_layout: int,
                     is_causal: int, q_quant_gran: int, k_quant_gran: int, sm_scale: float, fold_sm_scale: int) -> None:
    """Gradients of the INT8-QK attention (include/sageattn_b200.h, sab_qk_int8_attn_bwd): q_int8 / k_int8 / scales / granularities /
    sm_scale / fold_sm_scale as the forward call received them, q / k / v the unquantised (k unsmoothed) 16-bit inputs, o and dout
    the forward output and its gradient, lse the forward kernel's raw [B,Hq,Sq] log2 LSE, k_mean the K smoothing mean (any shape
    with B*Hkv*D elements, k's dtype; None without smoothing).  dq / dk / dv must have the strides of q / k / v."""
    B, Hq, Sq, D = _bhsd(q, tensor_layout)
    _, Hkv, Skv, _ = _bhsd(k, tensor_layout)
    strides, k_mean, ws = _bwd_operands(q_int8, k_int8, q, k, v, o, dout, lse, k_mean, dq, dk, dv, tensor_layout, (B, Hq, Sq),
                                        (B, Hkv, D), "B*Hkv*D")
    with torch.cuda.device(q.device):
        check(lib().sab_qk_int8_attn_bwd(q_int8.data_ptr(), k_int8.data_ptr(), q_scale.data_ptr(), k_scale.data_ptr(), q.data_ptr(),
                                         k.data_ptr(), v.data_ptr(), o.data_ptr(), dout.data_ptr(), lse.data_ptr(), _ptr(k_mean), dq.data_ptr(),
                                         dk.data_ptr(), dv.data_ptr(), ws.data_ptr(), _dt(q), B, Hq, Hkv, Sq, Skv, D, *strides,
                                         is_causal, q_quant_gran, k_quant_gran, float(sm_scale), fold_sm_scale, _stream(q)))


@qk_int8_attn_bwd.register_fake
def _(q_int8, k_int8, q_scale, k_scale, q, k, v, o, dout, lse, k_mean, dq, dk, dv, tensor_layout, is_causal, q_quant_gran, k_quant_gran,
      sm_scale, fold_sm_scale):
    return None


@torch.library.custom_op("sageattention_b200::qk_int8_attn_bwd_masked", mutates_args=("dq", "dk", "dv", "dbias"), device_types="cuda")
def qk_int8_attn_bwd_masked(q_int8: torch.Tensor, k_int8: torch.Tensor, q_scale: torch.Tensor, k_scale: torch.Tensor, q: torch.Tensor,
                            k: torch.Tensor, v: torch.Tensor, o: torch.Tensor, dout: torch.Tensor, lse: torch.Tensor,
                            k_mean: Optional[torch.Tensor], dq: torch.Tensor, dk: torch.Tensor, dv: torch.Tensor,
                            attn_mask: torch.Tensor, dbias: Optional[torch.Tensor], tensor_layout: int, q_quant_gran: int,
                            k_quant_gran: int, sm_scale: float, fold_sm_scale: int) -> None:
    """Gradients of the masked FP16-PV attention (include/sageattn_b200.h, sab_qk_int8_attn_bwd_masked): the arguments of
    qk_int8_attn_bwd without is_causal, plus the attn_mask view the forward received (qk_int8_sv_f16_attn_masked: [B,Hq,Sq,Skv],
    strides may be 0) and dbias, None or a contiguous [B,Hq,Sq,Skv] tensor of the mask dtype (a float mask only) written with
    ln2 * dS."""
    B, Hq, Sq, D = _bhsd(q, tensor_layout)
    _, Hkv, Skv, _ = _bhsd(k, tensor_layout)
    strides, k_mean, ws = _bwd_operands(q_int8, k_int8, q, k, v, o, dout, lse, k_mean, dq, dk, dv, tensor_layout, (B, Hq, Sq),
                                        (B, Hkv, D), "B*Hkv*D")
    assert attn_mask.dim() == 4 and tuple(attn_mask.shape) == (B, Hq, Sq, Skv), "attn_mask must be expanded to [B,Hq,Sq,Skv]"
    kind = SAB_MASK_BOOL if attn_mask.dtype == torch.bool else SAB_MASK_BIAS
    assert kind == SAB_MASK_BOOL or attn_mask.dtype == q.dtype, "attn_mask must be bool or the q dtype"
    if dbias is not None:
        assert dbias.dtype == attn_mask.dtype and dbias.is_contiguous() and tuple(dbias.shape) == (B, Hq, Sq, Skv), \
            "dbias must be a contiguous [B,Hq,Sq,Skv] tensor of the mask dtype"
    with torch.cuda.device(q.device):
        check(lib().sab_qk_int8_attn_bwd_masked(q_int8.data_ptr(), k_int8.data_ptr(), q_scale.data_ptr(), k_scale.data_ptr(),
                                                q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), dout.data_ptr(), lse.data_ptr(),
                                                _ptr(k_mean), dq.data_ptr(), dk.data_ptr(), dv.data_ptr(), ws.data_ptr(), _dt(q), B, Hq,
                                                Hkv, Sq, Skv, D, *strides, q_quant_gran, k_quant_gran, float(sm_scale), fold_sm_scale,
                                                attn_mask.data_ptr(), kind, *attn_mask.stride(), _ptr(dbias), _stream(q)))


@qk_int8_attn_bwd_masked.register_fake
def _(q_int8, k_int8, q_scale, k_scale, q, k, v, o, dout, lse, k_mean, dq, dk, dv, attn_mask, dbias, tensor_layout, q_quant_gran,
      k_quant_gran, sm_scale, fold_sm_scale):
    return None


@torch.library.custom_op("sageattention_b200::qk_int8_attn_bwd_blocksparse", mutates_args=("dq", "dk", "dv"), device_types="cuda")
def qk_int8_attn_bwd_blocksparse(q_int8: torch.Tensor, k_int8: torch.Tensor, q_scale: torch.Tensor, k_scale: torch.Tensor,
                                 q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, o: torch.Tensor, dout: torch.Tensor,
                                 lse: torch.Tensor, k_mean: Optional[torch.Tensor], dq: torch.Tensor, dk: torch.Tensor,
                                 dv: torch.Tensor, block_mask: torch.Tensor, tensor_layout: int, is_causal: int, q_quant_gran: int,
                                 k_quant_gran: int, sm_scale: float, fold_sm_scale: int) -> None:
    """Gradients of the block-sparse attention (include/sageattn_b200.h, sab_qk_int8_attn_bwd_blocksparse): the arguments of
    qk_int8_attn_bwd plus the block mask view the forward received (qk_int8_sv_f8_attn_blocksparse)."""
    B, Hq, Sq, D = _bhsd(q, tensor_layout)
    _, Hkv, Skv, _ = _bhsd(k, tensor_layout)
    strides, k_mean, ws = _bwd_operands(q_int8, k_int8, q, k, v, o, dout, lse, k_mean, dq, dk, dv, tensor_layout, (B, Hq, Sq),
                                        (B, Hkv, D), "B*Hkv*D")
    mask = _block_mask_args(block_mask, B, Hq, Sq, Skv)
    with torch.cuda.device(q.device):
        check(lib().sab_qk_int8_attn_bwd_blocksparse(q_int8.data_ptr(), k_int8.data_ptr(), q_scale.data_ptr(), k_scale.data_ptr(),
                                                     q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), dout.data_ptr(),
                                                     lse.data_ptr(), _ptr(k_mean), dq.data_ptr(), dk.data_ptr(), dv.data_ptr(),
                                                     ws.data_ptr(), _dt(q), B, Hq, Hkv, Sq, Skv, D, *strides, is_causal, q_quant_gran,
                                                     k_quant_gran, float(sm_scale), fold_sm_scale, *mask, _stream(q)))


@qk_int8_attn_bwd_blocksparse.register_fake
def _(q_int8, k_int8, q_scale, k_scale, q, k, v, o, dout, lse, k_mean, dq, dk, dv, block_mask, tensor_layout, is_causal,
      q_quant_gran, k_quant_gran, sm_scale, fold_sm_scale):
    return None


@torch.library.custom_op("sageattention_b200::qk_int8_attn_bwd_window", mutates_args=("dq", "dk", "dv"), device_types="cuda")
def qk_int8_attn_bwd_window(q_int8: torch.Tensor, k_int8: torch.Tensor, q_scale: torch.Tensor, k_scale: torch.Tensor,
                            q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, o: torch.Tensor, dout: torch.Tensor,
                            lse: torch.Tensor, k_mean: Optional[torch.Tensor], dq: torch.Tensor, dk: torch.Tensor,
                            dv: torch.Tensor, window_left: int, window_right: int, tensor_layout: int, is_causal: int,
                            q_quant_gran: int, k_quant_gran: int, sm_scale: float, fold_sm_scale: int) -> None:
    """Gradients of the sliding-window attention (include/sageattn_b200.h, sab_qk_int8_attn_bwd_window): the arguments of
    qk_int8_attn_bwd plus the window the forward received (qk_int8_sv_f8_attn_window)."""
    B, Hq, Sq, D = _bhsd(q, tensor_layout)
    _, Hkv, Skv, _ = _bhsd(k, tensor_layout)
    strides, k_mean, ws = _bwd_operands(q_int8, k_int8, q, k, v, o, dout, lse, k_mean, dq, dk, dv, tensor_layout, (B, Hq, Sq),
                                        (B, Hkv, D), "B*Hkv*D")
    with torch.cuda.device(q.device):
        check(lib().sab_qk_int8_attn_bwd_window(q_int8.data_ptr(), k_int8.data_ptr(), q_scale.data_ptr(), k_scale.data_ptr(),
                                                q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), dout.data_ptr(),
                                                lse.data_ptr(), _ptr(k_mean), dq.data_ptr(), dk.data_ptr(), dv.data_ptr(),
                                                ws.data_ptr(), _dt(q), B, Hq, Hkv, Sq, Skv, D, *strides, is_causal, q_quant_gran,
                                                k_quant_gran, float(sm_scale), fold_sm_scale, window_left, window_right, _stream(q)))


@qk_int8_attn_bwd_window.register_fake
def _(q_int8, k_int8, q_scale, k_scale, q, k, v, o, dout, lse, k_mean, dq, dk, dv, window_left, window_right, tensor_layout,
      is_causal, q_quant_gran, k_quant_gran, sm_scale, fold_sm_scale):
    return None


@torch.library.custom_op("sageattention_b200::qk_int8_attn_bwd_varlen", mutates_args=("dq", "dk", "dv"), device_types="cuda")
def qk_int8_attn_bwd_varlen(q_int8: torch.Tensor, k_int8: torch.Tensor, q_scale: torch.Tensor, k_scale: torch.Tensor,
                            q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, o: torch.Tensor, dout: torch.Tensor, lse: torch.Tensor,
                            k_mean: Optional[torch.Tensor], dq: torch.Tensor, dk: torch.Tensor, dv: torch.Tensor,
                            cu_seqlens_q: torch.Tensor, cu_seqlens_k: torch.Tensor, cu_q_scale: torch.Tensor,
                            cu_k_scale: torch.Tensor, max_seqlen_q: int, max_seqlen_k: int, is_causal: int, sm_scale: float,
                            fold_sm_scale: int) -> None:
    """Gradients of the packed FP16-PV attention (include/sageattn_b200.h, sab_qk_int8_attn_bwd_varlen): packed [T,H,D] tensors,
    q_int8 / k_int8 / per-block scales / cu_q_scale / cu_k_scale from per_block_int8_varlen, lse the forward's [Hq,Tq] log2 LSE
    (qk_int8_sv_f16_attn_varlen with return_lse=1), k_mean the K mean over all tokens ([Hkv,D] elements, k's dtype; None without
    smoothing).  dq / dk / dv must have the strides of q / k / v; rows past cu_seqlens_*[-1] are not written."""
    Tq, Hq, D = q.shape
    Tk, Hkv, _ = k.shape
    strides, k_mean, ws = _bwd_operands(q_int8, k_int8, q, k, v, o, dout, lse, k_mean, dq, dk, dv, None, (Hq, Tq), (Hkv, D),
                                        "Hkv*D")
    with torch.cuda.device(q.device):
        check(lib().sab_qk_int8_attn_bwd_varlen(q_int8.data_ptr(), k_int8.data_ptr(), q_scale.data_ptr(), k_scale.data_ptr(),
                                                q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), dout.data_ptr(), lse.data_ptr(),
                                                _ptr(k_mean), dq.data_ptr(), dk.data_ptr(), dv.data_ptr(), ws.data_ptr(), _dt(q),
                                                cu_seqlens_q.numel() - 1, Hq, Hkv, Tq, Tk, D, *strides, cu_seqlens_q.data_ptr(),
                                                cu_seqlens_k.data_ptr(), cu_q_scale.data_ptr(), cu_k_scale.data_ptr(), max_seqlen_q,
                                                max_seqlen_k, is_causal, float(sm_scale), fold_sm_scale, _stream(q)))


@qk_int8_attn_bwd_varlen.register_fake
def _(q_int8, k_int8, q_scale, k_scale, q, k, v, o, dout, lse, k_mean, dq, dk, dv, cu_seqlens_q, cu_seqlens_k, cu_q_scale, cu_k_scale,
      max_seqlen_q, max_seqlen_k, is_causal, sm_scale, fold_sm_scale):
    return None


# ----------------------------------------------------------------------------------------------- packed INT8+FP8, per-sequence statistics
@torch.library.custom_op("sageattention_b200::k_mean_varlen", mutates_args=("mean",), device_types="cuda")
def k_mean_varlen(k: torch.Tensor, mean: torch.Tensor, cu_seqlens: torch.Tensor, max_seqlen: int) -> None:
    """Per-sequence K mean (include/sageattn_b200.h, sab_k_mean_varlen): k packed [T,H,D], mean [nseq,H,D] in k's dtype."""
    T, H, D = k.shape
    nseq = cu_seqlens.numel() - 1
    with torch.cuda.device(k.device):
        ws = torch.empty(lib().sab_k_mean_varlen_workspace_bytes(nseq, H, max_seqlen, D), dtype=torch.uint8, device=k.device)
        check(lib().sab_k_mean_varlen(k.data_ptr(), _dt(k), mean.data_ptr(), cu_seqlens.data_ptr(), nseq, max_seqlen, H, D,
                                      k.stride(0), k.stride(1), ws.data_ptr(), _stream(k)))


@k_mean_varlen.register_fake
def _(k, mean, cu_seqlens, max_seqlen):
    return None


@torch.library.custom_op("sageattention_b200::quant_int8_varlen", mutates_args=("output", "scale"), device_types="cuda")
def quant_int8_varlen(input: torch.Tensor, mean: Optional[torch.Tensor], output: torch.Tensor, scale: torch.Tensor,
                      cu_seqlens: torch.Tensor, cu_scale: torch.Tensor, max_seqlen: int, granularity: int, is_key: bool) -> None:
    """Per-sequence per-warp / per-thread INT8 of packed Q or K (include/sageattn_b200.h, sab_quant_int8_varlen)."""
    T, H, D = input.shape
    with torch.cuda.device(input.device):
        check(lib().sab_quant_int8_varlen(input.data_ptr(), _dt(input), _ptr(mean), output.data_ptr(), scale.data_ptr(),
                                          cu_seqlens.data_ptr(), cu_scale.data_ptr(), cu_seqlens.numel() - 1, max_seqlen, H, D,
                                          input.stride(0), input.stride(1), output.stride(0), output.stride(1), granularity,
                                          1 if is_key else 0, _stream(input)))


@quant_int8_varlen.register_fake
def _(input, mean, output, scale, cu_seqlens, cu_scale, max_seqlen, granularity, is_key):
    return None


@torch.library.custom_op("sageattention_b200::per_channel_fp8_varlen_seq", mutates_args=("v_fp8", "v_scale", "v_mean"),
                         device_types="cuda")
def per_channel_fp8_varlen_seq(v: torch.Tensor, v_fp8: torch.Tensor, v_scale: torch.Tensor, v_mean: Optional[torch.Tensor],
                               cu_seqlens: torch.Tensor, cu_pad: torch.Tensor, max_seqlen: int, scale_max: float) -> None:
    """Per-sequence per-channel FP8 of packed V (include/sageattn_b200.h, sab_per_channel_fp8_varlen)."""
    T, H, D = v.shape
    nseq = cu_seqlens.numel() - 1
    with torch.cuda.device(v.device):
        ws = torch.empty(lib().sab_per_channel_fp8_varlen_workspace_bytes(nseq, H, max_seqlen, D), dtype=torch.uint8, device=v.device)
        check(lib().sab_per_channel_fp8_varlen(v.data_ptr(), _dt(v), v_fp8.data_ptr(), v_scale.data_ptr(), _ptr(v_mean),
                                               cu_seqlens.data_ptr(), cu_pad.data_ptr(), nseq, max_seqlen, H, D, v.stride(0), v.stride(1),
                                               v_fp8.size(-1), float(scale_max), ws.data_ptr(), _stream(v)))


@per_channel_fp8_varlen_seq.register_fake
def _(v, v_fp8, v_scale, v_mean, cu_seqlens, cu_pad, max_seqlen, scale_max):
    return None


@torch.library.custom_op("sageattention_b200::qk_int8_sv_f8_attn_varlen_seq", mutates_args=("output",), device_types="cuda")
def qk_int8_sv_f8_attn_varlen_seq(query: torch.Tensor, key: torch.Tensor, value: torch.Tensor, output: torch.Tensor,
                                  query_scale: torch.Tensor, key_scale: torch.Tensor, value_scale: torch.Tensor,
                                  value_mean: Optional[torch.Tensor], cu_seqlens_q: torch.Tensor, cu_seqlens_k: torch.Tensor,
                                  cu_pad_v: torch.Tensor, cu_q_scale: torch.Tensor, cu_k_scale: torch.Tensor, max_seqlen_q: int,
                                  is_causal: int, q_quant_gran: int, k_quant_gran: int, sm_scale: float, return_lse: int) -> torch.Tensor:
    """Packed INT8+FP8 forward with per-sequence V statistics (include/sageattn_b200.h, sab_qk_int8_sv_f8_attn_varlen).  Returns
    the [Hq,Tq] log2 LSE when return_lse, else an empty tensor."""
    Tq, Hq, D = query.shape
    Tk, Hkv, _ = key.shape
    lse = _lse(query, (Hq, Tq), return_lse)
    with torch.cuda.device(query.device):
        check(lib().sab_qk_int8_sv_f8_attn_varlen(query.data_ptr(), key.data_ptr(), value.data_ptr(), output.data_ptr(),
                                                  lse.data_ptr() if return_lse else None, query_scale.data_ptr(), key_scale.data_ptr(),
                                                  value_scale.data_ptr(), _ptr(value_mean), _dt(output), cu_seqlens_q.numel() - 1,
                                                  Hq, Hkv, Tq, Tk, D, query.stride(0), query.stride(1), key.stride(0), key.stride(1),
                                                  _v_pad(value), output.stride(0), output.stride(1), is_causal, q_quant_gran,
                                                  k_quant_gran, float(sm_scale), cu_seqlens_q.data_ptr(), cu_seqlens_k.data_ptr(),
                                                  cu_pad_v.data_ptr(), cu_q_scale.data_ptr(), cu_k_scale.data_ptr(), max_seqlen_q,
                                                  _stream(query)))
    return lse


@qk_int8_sv_f8_attn_varlen_seq.register_fake
def _(query, key, value, output, query_scale, key_scale, value_scale, value_mean, cu_seqlens_q, cu_seqlens_k, cu_pad_v, cu_q_scale,
      cu_k_scale, max_seqlen_q, is_causal, q_quant_gran, k_quant_gran, sm_scale, return_lse):
    Tq, Hq, _ = query.shape
    return _lse(query, (Hq, Tq), return_lse)


# ----------------------------------------------------------------------------------------------- paged KV cache
def _paged(cache: torch.Tensor, block_table: torch.Tensor):
    """(table_stride, page_size, page_stride, stride_t, stride_h) of a [num_pages, page_size, H, D] cache and its block table."""
    return block_table.stride(0), cache.size(1), cache.stride(0), cache.stride(1), cache.stride(2)


@torch.library.custom_op("sageattention_b200::k_mean_paged", mutates_args=("mean",), device_types="cuda")
def k_mean_paged(k_cache: torch.Tensor, mean: torch.Tensor, cu_seqlens: torch.Tensor, block_table: torch.Tensor,
                 max_seqlen: int) -> None:
    """k_mean_varlen reading K from a paged cache (include/sageattn_b200.h, sab_k_mean_paged): mean [nseq,H,D] in the cache's dtype."""
    _, _, H, D = k_cache.shape
    nseq = cu_seqlens.numel() - 1
    tstride, page_size, pstride, st, sh = _paged(k_cache, block_table)
    with torch.cuda.device(k_cache.device):
        ws = torch.empty(lib().sab_k_mean_varlen_workspace_bytes(nseq, H, max_seqlen, D), dtype=torch.uint8, device=k_cache.device)
        check(lib().sab_k_mean_paged(k_cache.data_ptr(), _dt(k_cache), mean.data_ptr(), cu_seqlens.data_ptr(), block_table.data_ptr(),
                                     tstride, page_size, nseq, max_seqlen, H, D, pstride, st, sh, ws.data_ptr(), _stream(k_cache)))


@k_mean_paged.register_fake
def _(k_cache, mean, cu_seqlens, block_table, max_seqlen):
    return None


@torch.library.custom_op("sageattention_b200::quant_int8_paged", mutates_args=("output", "scale"), device_types="cuda")
def quant_int8_paged(k_cache: torch.Tensor, mean: Optional[torch.Tensor], output: torch.Tensor, scale: torch.Tensor,
                     cu_seqlens: torch.Tensor, cu_scale: torch.Tensor, block_table: torch.Tensor, max_seqlen: int,
                     granularity: int) -> None:
    """quant_int8_varlen of K read from a paged cache (include/sageattn_b200.h, sab_quant_int8_paged): output [Tk,H,D] packed."""
    _, _, H, D = k_cache.shape
    tstride, page_size, pstride, st, sh = _paged(k_cache, block_table)
    with torch.cuda.device(k_cache.device):
        check(lib().sab_quant_int8_paged(k_cache.data_ptr(), _dt(k_cache), _ptr(mean), output.data_ptr(), scale.data_ptr(),
                                         cu_seqlens.data_ptr(), cu_scale.data_ptr(), block_table.data_ptr(), tstride, page_size,
                                         cu_seqlens.numel() - 1, max_seqlen, H, D, pstride, st, sh, output.stride(0), output.stride(1),
                                         granularity, _stream(k_cache)))


@quant_int8_paged.register_fake
def _(k_cache, mean, output, scale, cu_seqlens, cu_scale, block_table, max_seqlen, granularity):
    return None


@torch.library.custom_op("sageattention_b200::per_channel_fp8_paged", mutates_args=("v_fp8", "v_scale", "v_mean"), device_types="cuda")
def per_channel_fp8_paged(v_cache: torch.Tensor, v_fp8: torch.Tensor, v_scale: torch.Tensor, v_mean: Optional[torch.Tensor],
                          cu_seqlens: torch.Tensor, cu_pad: torch.Tensor, block_table: torch.Tensor, max_seqlen: int,
                          scale_max: float) -> None:
    """per_channel_fp8_varlen_seq reading V from a paged cache (include/sageattn_b200.h, sab_per_channel_fp8_paged)."""
    _, _, H, D = v_cache.shape
    nseq = cu_seqlens.numel() - 1
    tstride, page_size, pstride, st, sh = _paged(v_cache, block_table)
    with torch.cuda.device(v_cache.device):
        ws = torch.empty(lib().sab_per_channel_fp8_varlen_workspace_bytes(nseq, H, max_seqlen, D), dtype=torch.uint8,
                         device=v_cache.device)
        check(lib().sab_per_channel_fp8_paged(v_cache.data_ptr(), _dt(v_cache), v_fp8.data_ptr(), v_scale.data_ptr(), _ptr(v_mean),
                                              cu_seqlens.data_ptr(), cu_pad.data_ptr(), block_table.data_ptr(), tstride, page_size,
                                              nseq, max_seqlen, H, D, pstride, st, sh, v_fp8.size(-1), float(scale_max), ws.data_ptr(),
                                              _stream(v_cache)))


@per_channel_fp8_paged.register_fake
def _(v_cache, v_fp8, v_scale, v_mean, cu_seqlens, cu_pad, block_table, max_seqlen, scale_max):
    return None


@torch.library.custom_op("sageattention_b200::qk_int8_sv_f8_attn_varlen_bottom_right", mutates_args=("output",), device_types="cuda")
def qk_int8_sv_f8_attn_varlen_bottom_right(query: torch.Tensor, key: torch.Tensor, value: torch.Tensor, output: torch.Tensor,
                                           query_scale: torch.Tensor, key_scale: torch.Tensor, value_scale: torch.Tensor,
                                           value_mean: Optional[torch.Tensor], cu_seqlens_q: torch.Tensor, cu_seqlens_k: torch.Tensor,
                                           cu_pad_v: torch.Tensor, cu_q_scale: torch.Tensor, cu_k_scale: torch.Tensor,
                                           max_seqlen_q: int, is_causal: int, q_quant_gran: int, k_quant_gran: int, sm_scale: float,
                                           return_lse: int) -> torch.Tensor:
    """qk_int8_sv_f8_attn_varlen_seq with causal aligned bottom-right inside each sequence (include/sageattn_b200.h,
    sab_qk_int8_sv_f8_attn_varlen_bottom_right).  Returns the [Hq,Tq] log2 LSE when return_lse, else an empty tensor; a row with
    no visible key gets 0 and lse -inf."""
    Tq, Hq, D = query.shape
    Tk, Hkv, _ = key.shape
    lse = _lse(query, (Hq, Tq), return_lse)
    with torch.cuda.device(query.device):
        check(lib().sab_qk_int8_sv_f8_attn_varlen_bottom_right(query.data_ptr(), key.data_ptr(), value.data_ptr(), output.data_ptr(),
                                                               lse.data_ptr() if return_lse else None, query_scale.data_ptr(),
                                                               key_scale.data_ptr(), value_scale.data_ptr(), _ptr(value_mean),
                                                               _dt(output), cu_seqlens_q.numel() - 1, Hq, Hkv, Tq, Tk, D, query.stride(0),
                                                               query.stride(1), key.stride(0), key.stride(1), _v_pad(value),
                                                               output.stride(0), output.stride(1), is_causal, q_quant_gran, k_quant_gran,
                                                               float(sm_scale), cu_seqlens_q.data_ptr(), cu_seqlens_k.data_ptr(),
                                                               cu_pad_v.data_ptr(), cu_q_scale.data_ptr(), cu_k_scale.data_ptr(),
                                                               max_seqlen_q, _stream(query)))
    return lse


@qk_int8_sv_f8_attn_varlen_bottom_right.register_fake
def _(query, key, value, output, query_scale, key_scale, value_scale, value_mean, cu_seqlens_q, cu_seqlens_k, cu_pad_v, cu_q_scale,
      cu_k_scale, max_seqlen_q, is_causal, q_quant_gran, k_quant_gran, sm_scale, return_lse):
    Tq, Hq, _ = query.shape
    return _lse(query, (Hq, Tq), return_lse)


@torch.library.custom_op("sageattention_b200::qk_int8_attn_bwd_varlen_seq", mutates_args=("dq", "dk", "dv"), device_types="cuda")
def qk_int8_attn_bwd_varlen_seq(q_int8: torch.Tensor, k_int8: torch.Tensor, q_scale: torch.Tensor, k_scale: torch.Tensor,
                                q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, o: torch.Tensor, dout: torch.Tensor,
                                lse: torch.Tensor, k_mean: Optional[torch.Tensor], dq: torch.Tensor, dk: torch.Tensor,
                                dv: torch.Tensor, cu_seqlens_q: torch.Tensor, cu_seqlens_k: torch.Tensor, cu_q_scale: torch.Tensor,
                                cu_k_scale: torch.Tensor, max_seqlen_q: int, max_seqlen_k: int, is_causal: int, q_quant_gran: int,
                                k_quant_gran: int, sm_scale: float) -> None:
    """Gradients of qk_int8_sv_f8_attn_varlen_seq (include/sageattn_b200.h, sab_qk_int8_attn_bwd_varlen_seq): the operands of the
    forward, lse its [Hq,Tq] log2 LSE, k_mean the per-sequence [nseq,Hkv,D] mean (None without smoothing).  dq / dk / dv must
    have the strides of q / k / v; rows past cu_seqlens_*[-1] are not written."""
    Tq, Hq, D = q.shape
    Tk, Hkv, _ = k.shape
    nseq = cu_seqlens_q.numel() - 1
    strides, k_mean, ws = _bwd_operands(q_int8, k_int8, q, k, v, o, dout, lse, k_mean, dq, dk, dv, None, (Hq, Tq), (nseq, Hkv, D),
                                        "nseq*Hkv*D")
    with torch.cuda.device(q.device):
        check(lib().sab_qk_int8_attn_bwd_varlen_seq(q_int8.data_ptr(), k_int8.data_ptr(), q_scale.data_ptr(), k_scale.data_ptr(),
                                                    q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), dout.data_ptr(),
                                                    lse.data_ptr(), _ptr(k_mean), dq.data_ptr(), dk.data_ptr(), dv.data_ptr(),
                                                    ws.data_ptr(), _dt(q), nseq, Hq, Hkv, Tq, Tk, D, *strides, cu_seqlens_q.data_ptr(),
                                                    cu_seqlens_k.data_ptr(), cu_q_scale.data_ptr(), cu_k_scale.data_ptr(), max_seqlen_q,
                                                    max_seqlen_k, is_causal, q_quant_gran, k_quant_gran, float(sm_scale), _stream(q)))


@qk_int8_attn_bwd_varlen_seq.register_fake
def _(q_int8, k_int8, q_scale, k_scale, q, k, v, o, dout, lse, k_mean, dq, dk, dv, cu_seqlens_q, cu_seqlens_k, cu_q_scale, cu_k_scale,
      max_seqlen_q, max_seqlen_k, is_causal, q_quant_gran, k_quant_gran, sm_scale):
    return None


@torch.library.custom_op("sageattention_b200::qk_int8_sv_f8_attn_varlen_window", mutates_args=("output",), device_types="cuda")
def qk_int8_sv_f8_attn_varlen_window(query: torch.Tensor, key: torch.Tensor, value: torch.Tensor, output: torch.Tensor,
                                     query_scale: torch.Tensor, key_scale: torch.Tensor, value_scale: torch.Tensor,
                                     value_mean: Optional[torch.Tensor], cu_seqlens_q: torch.Tensor, cu_seqlens_k: torch.Tensor,
                                     cu_pad_v: torch.Tensor, cu_q_scale: torch.Tensor, cu_k_scale: torch.Tensor, max_seqlen_q: int,
                                     window_left: int, window_right: int, is_causal: int, q_quant_gran: int, k_quant_gran: int,
                                     sm_scale: float, return_lse: int) -> torch.Tensor:
    """qk_int8_sv_f8_attn_varlen_seq restricted to a sliding window inside each sequence (include/sageattn_b200.h,
    sab_qk_int8_sv_f8_attn_varlen_window); window_left / window_right must fit in a C int (the entry point clamps them first).
    Returns the [Hq,Tq] log2 LSE when return_lse, else an empty tensor; a row with no visible key gets 0 and lse -inf."""
    Tq, Hq, D = query.shape
    Tk, Hkv, _ = key.shape
    lse = _lse(query, (Hq, Tq), return_lse)
    with torch.cuda.device(query.device):
        check(lib().sab_qk_int8_sv_f8_attn_varlen_window(query.data_ptr(), key.data_ptr(), value.data_ptr(), output.data_ptr(),
                                                         lse.data_ptr() if return_lse else None, query_scale.data_ptr(),
                                                         key_scale.data_ptr(), value_scale.data_ptr(), _ptr(value_mean), _dt(output),
                                                         cu_seqlens_q.numel() - 1, Hq, Hkv, Tq, Tk, D, query.stride(0), query.stride(1),
                                                         key.stride(0), key.stride(1), _v_pad(value), output.stride(0), output.stride(1),
                                                         is_causal, q_quant_gran, k_quant_gran, float(sm_scale), cu_seqlens_q.data_ptr(),
                                                         cu_seqlens_k.data_ptr(), cu_pad_v.data_ptr(), cu_q_scale.data_ptr(),
                                                         cu_k_scale.data_ptr(), max_seqlen_q, window_left, window_right, _stream(query)))
    return lse


@qk_int8_sv_f8_attn_varlen_window.register_fake
def _(query, key, value, output, query_scale, key_scale, value_scale, value_mean, cu_seqlens_q, cu_seqlens_k, cu_pad_v, cu_q_scale,
      cu_k_scale, max_seqlen_q, window_left, window_right, is_causal, q_quant_gran, k_quant_gran, sm_scale, return_lse):
    Tq, Hq, _ = query.shape
    return _lse(query, (Hq, Tq), return_lse)


@torch.library.custom_op("sageattention_b200::qk_int8_attn_bwd_varlen_window", mutates_args=("dq", "dk", "dv"), device_types="cuda")
def qk_int8_attn_bwd_varlen_window(q_int8: torch.Tensor, k_int8: torch.Tensor, q_scale: torch.Tensor, k_scale: torch.Tensor,
                                   q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, o: torch.Tensor, dout: torch.Tensor,
                                   lse: torch.Tensor, k_mean: Optional[torch.Tensor], dq: torch.Tensor, dk: torch.Tensor,
                                   dv: torch.Tensor, cu_seqlens_q: torch.Tensor, cu_seqlens_k: torch.Tensor, cu_q_scale: torch.Tensor,
                                   cu_k_scale: torch.Tensor, max_seqlen_q: int, max_seqlen_k: int, window_left: int,
                                   window_right: int, is_causal: int, q_quant_gran: int, k_quant_gran: int, sm_scale: float) -> None:
    """Gradients of qk_int8_sv_f8_attn_varlen_window (include/sageattn_b200.h, sab_qk_int8_attn_bwd_varlen_window): the arguments
    of qk_int8_attn_bwd_varlen_seq plus the window the forward received."""
    Tq, Hq, D = q.shape
    Tk, Hkv, _ = k.shape
    nseq = cu_seqlens_q.numel() - 1
    strides, k_mean, ws = _bwd_operands(q_int8, k_int8, q, k, v, o, dout, lse, k_mean, dq, dk, dv, None, (Hq, Tq), (nseq, Hkv, D),
                                        "nseq*Hkv*D")
    with torch.cuda.device(q.device):
        check(lib().sab_qk_int8_attn_bwd_varlen_window(q_int8.data_ptr(), k_int8.data_ptr(), q_scale.data_ptr(), k_scale.data_ptr(),
                                                       q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), dout.data_ptr(),
                                                       lse.data_ptr(), _ptr(k_mean), dq.data_ptr(), dk.data_ptr(), dv.data_ptr(),
                                                       ws.data_ptr(), _dt(q), nseq, Hq, Hkv, Tq, Tk, D, *strides, cu_seqlens_q.data_ptr(),
                                                       cu_seqlens_k.data_ptr(), cu_q_scale.data_ptr(), cu_k_scale.data_ptr(),
                                                       max_seqlen_q, max_seqlen_k, is_causal, q_quant_gran, k_quant_gran,
                                                       float(sm_scale), window_left, window_right, _stream(q)))


@qk_int8_attn_bwd_varlen_window.register_fake
def _(q_int8, k_int8, q_scale, k_scale, q, k, v, o, dout, lse, k_mean, dq, dk, dv, cu_seqlens_q, cu_seqlens_k, cu_q_scale, cu_k_scale,
      max_seqlen_q, max_seqlen_k, window_left, window_right, is_causal, q_quant_gran, k_quant_gran, sm_scale):
    return None


@torch.library.custom_op("sageattention_b200::qk_int8_sv_f8_attn_varlen_blocksparse", mutates_args=("output",), device_types="cuda")
def qk_int8_sv_f8_attn_varlen_blocksparse(query: torch.Tensor, key: torch.Tensor, value: torch.Tensor, output: torch.Tensor,
                                          query_scale: torch.Tensor, key_scale: torch.Tensor, value_scale: torch.Tensor,
                                          value_mean: Optional[torch.Tensor], cu_seqlens_q: torch.Tensor, cu_seqlens_k: torch.Tensor,
                                          cu_pad_v: torch.Tensor, cu_q_scale: torch.Tensor, cu_k_scale: torch.Tensor,
                                          max_seqlen_q: int, max_seqlen_k: int, block_mask: torch.Tensor, is_causal: int,
                                          q_quant_gran: int, k_quant_gran: int, sm_scale: float, return_lse: int) -> torch.Tensor:
    """qk_int8_sv_f8_attn_varlen_seq restricted to the visible tiles of a block mask inside each sequence (include/sageattn_b200.h,
    sab_qk_int8_sv_f8_attn_varlen_blocksparse): a bool view [nseq,Hq,ceil(max_seqlen_q/128),ceil(max_seqlen_k/64)], strides may be
    0.  Returns the [Hq,Tq] log2 LSE when return_lse, else an empty tensor; a row with no visible key gets 0 and lse -inf."""
    Tq, Hq, D = query.shape
    Tk, Hkv, _ = key.shape
    nseq = cu_seqlens_q.numel() - 1
    mask = _block_mask_args(block_mask, nseq, Hq, max_seqlen_q, max_seqlen_k)
    lse = _lse(query, (Hq, Tq), return_lse)
    with torch.cuda.device(query.device):
        check(lib().sab_qk_int8_sv_f8_attn_varlen_blocksparse(query.data_ptr(), key.data_ptr(), value.data_ptr(), output.data_ptr(),
                                                              lse.data_ptr() if return_lse else None, query_scale.data_ptr(),
                                                              key_scale.data_ptr(), value_scale.data_ptr(), _ptr(value_mean),
                                                              _dt(output), nseq, Hq, Hkv, Tq, Tk, D, query.stride(0), query.stride(1),
                                                              key.stride(0), key.stride(1), _v_pad(value), output.stride(0),
                                                              output.stride(1), is_causal, q_quant_gran, k_quant_gran, float(sm_scale),
                                                              cu_seqlens_q.data_ptr(), cu_seqlens_k.data_ptr(), cu_pad_v.data_ptr(),
                                                              cu_q_scale.data_ptr(), cu_k_scale.data_ptr(), max_seqlen_q, max_seqlen_k,
                                                              *mask, _stream(query)))
    return lse


@qk_int8_sv_f8_attn_varlen_blocksparse.register_fake
def _(query, key, value, output, query_scale, key_scale, value_scale, value_mean, cu_seqlens_q, cu_seqlens_k, cu_pad_v, cu_q_scale,
      cu_k_scale, max_seqlen_q, max_seqlen_k, block_mask, is_causal, q_quant_gran, k_quant_gran, sm_scale, return_lse):
    Tq, Hq, _ = query.shape
    return _lse(query, (Hq, Tq), return_lse)


@torch.library.custom_op("sageattention_b200::qk_int8_attn_bwd_varlen_blocksparse", mutates_args=("dq", "dk", "dv"),
                         device_types="cuda")
def qk_int8_attn_bwd_varlen_blocksparse(q_int8: torch.Tensor, k_int8: torch.Tensor, q_scale: torch.Tensor, k_scale: torch.Tensor,
                                        q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, o: torch.Tensor, dout: torch.Tensor,
                                        lse: torch.Tensor, k_mean: Optional[torch.Tensor], dq: torch.Tensor, dk: torch.Tensor,
                                        dv: torch.Tensor, cu_seqlens_q: torch.Tensor, cu_seqlens_k: torch.Tensor,
                                        cu_q_scale: torch.Tensor, cu_k_scale: torch.Tensor, max_seqlen_q: int, max_seqlen_k: int,
                                        block_mask: torch.Tensor, is_causal: int, q_quant_gran: int, k_quant_gran: int,
                                        sm_scale: float) -> None:
    """Gradients of qk_int8_sv_f8_attn_varlen_blocksparse (include/sageattn_b200.h, sab_qk_int8_attn_bwd_varlen_blocksparse): the
    arguments of qk_int8_attn_bwd_varlen_seq plus the block mask view the forward received."""
    Tq, Hq, D = q.shape
    Tk, Hkv, _ = k.shape
    nseq = cu_seqlens_q.numel() - 1
    strides, k_mean, ws = _bwd_operands(q_int8, k_int8, q, k, v, o, dout, lse, k_mean, dq, dk, dv, None, (Hq, Tq), (nseq, Hkv, D),
                                        "nseq*Hkv*D")
    mask = _block_mask_args(block_mask, nseq, Hq, max_seqlen_q, max_seqlen_k)
    with torch.cuda.device(q.device):
        check(lib().sab_qk_int8_attn_bwd_varlen_blocksparse(q_int8.data_ptr(), k_int8.data_ptr(), q_scale.data_ptr(),
                                                            k_scale.data_ptr(), q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(),
                                                            dout.data_ptr(), lse.data_ptr(), _ptr(k_mean), dq.data_ptr(), dk.data_ptr(),
                                                            dv.data_ptr(), ws.data_ptr(), _dt(q), nseq, Hq, Hkv, Tq, Tk, D, *strides,
                                                            cu_seqlens_q.data_ptr(), cu_seqlens_k.data_ptr(), cu_q_scale.data_ptr(),
                                                            cu_k_scale.data_ptr(), max_seqlen_q, max_seqlen_k, is_causal, q_quant_gran,
                                                            k_quant_gran, float(sm_scale), *mask, _stream(q)))


@qk_int8_attn_bwd_varlen_blocksparse.register_fake
def _(q_int8, k_int8, q_scale, k_scale, q, k, v, o, dout, lse, k_mean, dq, dk, dv, cu_seqlens_q, cu_seqlens_k, cu_q_scale, cu_k_scale,
      max_seqlen_q, max_seqlen_k, block_mask, is_causal, q_quant_gran, k_quant_gran, sm_scale):
    return None


# ----------------------------------------------------------------------------------------------- block-mask prediction
@torch.library.custom_op("sageattention_b200::block_stats", mutates_args=("mean", "sim"), device_types="cuda")
def block_stats(x: torch.Tensor, mean: torch.Tensor, sim: torch.Tensor, tensor_layout: int, block_size: int) -> None:
    """Per-block fp32 mean [B,H,ceil(S/block_size),D] and self-similarity [B,H,ceil(S/block_size)] of x (include/sageattn_b200.h,
    sab_block_stats); block_size 128 for q, 64 for k.  A view whose rows are not 16-byte aligned is read from a contiguous copy."""
    B, H, S, D = _bhsd(x, tensor_layout)
    if x.data_ptr() % 16 or any(s % 8 for s in x.stride()[:-1]):
        x = x.contiguous()
    nb = (S + block_size - 1) // block_size
    assert mean.dtype == torch.float32 and mean.is_contiguous() and tuple(mean.shape) == (B, H, nb, D), \
        f"mean must be a contiguous fp32 [{B}, {H}, {nb}, {D}] tensor"
    assert sim.dtype == torch.float32 and sim.is_contiguous() and tuple(sim.shape) == (B, H, nb), \
        f"sim must be a contiguous fp32 [{B}, {H}, {nb}] tensor"
    sb, sh, ss = _bhs_strides(x, tensor_layout)
    with torch.cuda.device(x.device):
        check(lib().sab_block_stats(x.data_ptr(), _dt(x), mean.data_ptr(), sim.data_ptr(), B, H, S, D, sb, sh, ss, block_size,
                                    _stream(x)))


@block_stats.register_fake
def _(x, mean, sim, tensor_layout, block_size):
    return None


@torch.library.custom_op("sageattention_b200::predict_block_mask", mutates_args=("block_mask",), device_types="cuda")
def predict_block_mask(q_mean: torch.Tensor, q_sim: torch.Tensor, k_mean: torch.Tensor, k_sim: torch.Tensor,
                       block_mask: torch.Tensor, Sq: int, Skv: int, is_causal: int, sm_scale: float, cdf_threshold: float,
                       sim_threshold: float) -> None:
    """Writes the bool [B,Hq,ceil(Sq/128),ceil(Skv/64)] block_mask predicted from block_stats of q (block 128) and k (block 64)
    (include/sageattn_b200.h, sab_predict_block_mask)."""
    B, Hq, nq, D = q_mean.shape
    Hkv, nk = k_mean.size(1), k_mean.size(2)
    assert nq == (Sq + 127) // 128 and nk == (Skv + 63) // 64 and k_mean.size(3) == D and k_mean.size(0) == B, \
        "q / k statistics do not match Sq / Skv"
    for t in (q_mean, q_sim, k_mean, k_sim):
        assert t.dtype == torch.float32 and t.is_contiguous(), "block statistics must be contiguous fp32"
    assert tuple(q_sim.shape) == (B, Hq, nq) and tuple(k_sim.shape) == (B, Hkv, nk), "sim shapes do not match the means"
    assert block_mask.dtype == torch.bool and block_mask.is_contiguous() and tuple(block_mask.shape) == (B, Hq, nq, nk), \
        f"block_mask must be a contiguous bool [{B}, {Hq}, {nq}, {nk}] tensor"
    with torch.cuda.device(q_mean.device):
        check(lib().sab_predict_block_mask(q_mean.data_ptr(), q_sim.data_ptr(), k_mean.data_ptr(), k_sim.data_ptr(),
                                           block_mask.data_ptr(), B, Hq, Hkv, Sq, Skv, D, is_causal, float(sm_scale),
                                           float(cdf_threshold), float(sim_threshold), _stream(q_mean)))


@predict_block_mask.register_fake
def _(q_mean, q_sim, k_mean, k_sim, block_mask, Sq, Skv, is_causal, sm_scale, cdf_threshold, sim_threshold):
    return None


@torch.library.custom_op("sageattention_b200::block_stats_varlen", mutates_args=("mean", "sim"), device_types="cuda")
def block_stats_varlen(x: torch.Tensor, mean: torch.Tensor, sim: torch.Tensor, cu_seqlens: torch.Tensor, max_seqlen: int,
                       block_size: int) -> None:
    """block_stats of every sequence of packed x [T,H,D] on its own (include/sageattn_b200.h, sab_block_stats_varlen): mean
    [nseq,H,ceil(max_seqlen/block_size),D] and sim [nseq,H,ceil(max_seqlen/block_size)], blocks past a sequence's end 0."""
    T, H, D = x.shape
    nseq = cu_seqlens.numel() - 1
    if x.data_ptr() % 16 or any(s % 8 for s in x.stride()[:-1]):
        x = x.contiguous()
    nb = (max_seqlen + block_size - 1) // block_size
    assert mean.dtype == torch.float32 and mean.is_contiguous() and tuple(mean.shape) == (nseq, H, nb, D), \
        f"mean must be a contiguous fp32 [{nseq}, {H}, {nb}, {D}] tensor"
    assert sim.dtype == torch.float32 and sim.is_contiguous() and tuple(sim.shape) == (nseq, H, nb), \
        f"sim must be a contiguous fp32 [{nseq}, {H}, {nb}] tensor"
    with torch.cuda.device(x.device):
        check(lib().sab_block_stats_varlen(x.data_ptr(), _dt(x), mean.data_ptr(), sim.data_ptr(), cu_seqlens.data_ptr(), nseq,
                                           max_seqlen, H, D, x.stride(0), x.stride(1), block_size, _stream(x)))


@block_stats_varlen.register_fake
def _(x, mean, sim, cu_seqlens, max_seqlen, block_size):
    return None


@torch.library.custom_op("sageattention_b200::predict_block_mask_varlen", mutates_args=("block_mask",), device_types="cuda")
def predict_block_mask_varlen(q_mean: torch.Tensor, q_sim: torch.Tensor, k_mean: torch.Tensor, k_sim: torch.Tensor,
                              block_mask: torch.Tensor, cu_seqlens_q: torch.Tensor, cu_seqlens_k: torch.Tensor, max_seqlen_q: int,
                              max_seqlen_k: int, is_causal: int, sm_scale: float, cdf_threshold: float, sim_threshold: float) -> None:
    """Writes the bool [nseq,Hq,ceil(max_seqlen_q/128),ceil(max_seqlen_k/64)] block_mask predicted for each sequence from
    block_stats_varlen of q (block 128) and k (block 64) (include/sageattn_b200.h, sab_predict_block_mask_varlen)."""
    nseq, Hq, nq, D = q_mean.shape
    Hkv, nk = k_mean.size(1), k_mean.size(2)
    assert nseq == cu_seqlens_q.numel() - 1 == cu_seqlens_k.numel() - 1, "statistics and cu_seqlens disagree on nseq"
    assert nq == (max_seqlen_q + 127) // 128 and nk == (max_seqlen_k + 63) // 64 and k_mean.size(3) == D and k_mean.size(0) == nseq, \
        "q / k statistics do not match max_seqlen_q / max_seqlen_k"
    for t in (q_mean, q_sim, k_mean, k_sim):
        assert t.dtype == torch.float32 and t.is_contiguous(), "block statistics must be contiguous fp32"
    assert tuple(q_sim.shape) == (nseq, Hq, nq) and tuple(k_sim.shape) == (nseq, Hkv, nk), "sim shapes do not match the means"
    assert block_mask.dtype == torch.bool and block_mask.is_contiguous() and tuple(block_mask.shape) == (nseq, Hq, nq, nk), \
        f"block_mask must be a contiguous bool [{nseq}, {Hq}, {nq}, {nk}] tensor"
    with torch.cuda.device(q_mean.device):
        check(lib().sab_predict_block_mask_varlen(q_mean.data_ptr(), q_sim.data_ptr(), k_mean.data_ptr(), k_sim.data_ptr(),
                                                  block_mask.data_ptr(), cu_seqlens_q.data_ptr(), cu_seqlens_k.data_ptr(), nseq, Hq,
                                                  Hkv, max_seqlen_q, max_seqlen_k, D, is_causal, float(sm_scale), float(cdf_threshold),
                                                  float(sim_threshold), _stream(q_mean)))


@predict_block_mask_varlen.register_fake
def _(q_mean, q_sim, k_mean, k_sim, block_mask, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k, is_causal, sm_scale,
      cdf_threshold, sim_threshold):
    return None


# ----------------------------------------------------------------------------------------------- FP16-PV variant
@torch.library.custom_op("sageattention_b200::v_transpose_f16", mutates_args=("v_f16t",), device_types="cuda")
def v_transpose_f16(v: torch.Tensor, v_f16t: torch.Tensor, tensor_layout: int) -> None:
    B, H, S, D = _bhsd(v, tensor_layout)
    sb, sh, ss = _bhs_strides(v, tensor_layout)
    with torch.cuda.device(v.device):
        check(lib().sab_v_transpose_f16(v.data_ptr(), _dt(v), v_f16t.data_ptr(), B, H, S, D, sb, sh, ss, v_f16t.size(-1),
                                        None, None, 0, 0, _stream(v)))


@v_transpose_f16.register_fake
def _(v, v_f16t, tensor_layout):
    return None


@torch.library.custom_op("sageattention_b200::v_transpose_f16_varlen", mutates_args=("v_f16t",), device_types="cuda")
def v_transpose_f16_varlen(v: torch.Tensor, v_f16t: torch.Tensor, cu_seqlens: torch.Tensor, cu_pad: torch.Tensor,
                           max_seqlen: int) -> None:
    T, H, D = v.shape
    with torch.cuda.device(v.device):
        check(lib().sab_v_transpose_f16(v.data_ptr(), _dt(v), v_f16t.data_ptr(), 1, H, T, D, 0, v.stride(1), v.stride(0),
                                        v_f16t.size(-1), cu_seqlens.data_ptr(), cu_pad.data_ptr(), cu_seqlens.numel() - 1,
                                        max_seqlen, _stream(v)))


@v_transpose_f16_varlen.register_fake
def _(v, v_f16t, cu_seqlens, cu_pad, max_seqlen):
    return None


@torch.library.custom_op("sageattention_b200::qk_int8_sv_f16_attn", mutates_args=("output",), device_types="cuda")
def qk_int8_sv_f16_attn(query: torch.Tensor, key: torch.Tensor, value: torch.Tensor, output: torch.Tensor,
                        query_scale: torch.Tensor, key_scale: torch.Tensor, tensor_layout: int, is_causal: int,
                        q_quant_gran: int, k_quant_gran: int, sm_scale: float, fold_sm_scale: int,
                        return_lse: int) -> torch.Tensor:
    """INT8 QK^T + FP16 PV (the reference Triton kernels' numerics); value = [B,Hkv,D,S_pad] fp16 from v_transpose_f16."""
    B, Hq, Sq, D = _bhsd(query, tensor_layout)
    _, Hkv, Skv, _ = _bhsd(key, tensor_layout)
    qs, ks, os_ = _bhs_strides(query, tensor_layout), _bhs_strides(key, tensor_layout), _bhs_strides(output, tensor_layout)
    lse = _lse(query, (B, Hq, Sq), return_lse)
    with torch.cuda.device(query.device):
        check(lib().sab_qk_int8_sv_f16_attn(query.data_ptr(), key.data_ptr(), value.data_ptr(), output.data_ptr(),
                                            lse.data_ptr() if return_lse else None, query_scale.data_ptr(), key_scale.data_ptr(),
                                            _dt(output), B, Hq, Hkv, Sq, Skv, D, *qs, *ks, _v_pad(value), *os_, is_causal,
                                            q_quant_gran, k_quant_gran, float(sm_scale), fold_sm_scale, None, None, None, None,
                                            None, 0, _stream(query)))
    return lse


@qk_int8_sv_f16_attn.register_fake
def _(query, key, value, output, query_scale, key_scale, tensor_layout, is_causal, q_quant_gran, k_quant_gran, sm_scale,
      fold_sm_scale, return_lse):
    B, Hq, Sq, D = _bhsd(query, tensor_layout)
    return _lse(query, (B, Hq, Sq), return_lse)


@torch.library.custom_op("sageattention_b200::qk_int8_sv_f16_attn_masked", mutates_args=("output",), device_types="cuda")
def qk_int8_sv_f16_attn_masked(query: torch.Tensor, key: torch.Tensor, value: torch.Tensor, output: torch.Tensor,
                               query_scale: torch.Tensor, key_scale: torch.Tensor, attn_mask: torch.Tensor, tensor_layout: int,
                               q_quant_gran: int, k_quant_gran: int, sm_scale: float, fold_sm_scale: int,
                               return_lse: int) -> torch.Tensor:
    """qk_int8_sv_f16_attn with the Triton path's attn_mask: a 4-D view broadcast to [B,Hq,Sq,Skv] (strides may be 0),
    dtype bool (False = masked out) or the q dtype (additive bias).  Non-causal (sageattention/core.py:310)."""
    B, Hq, Sq, D = _bhsd(query, tensor_layout)
    _, Hkv, Skv, _ = _bhsd(key, tensor_layout)
    assert attn_mask.dim() == 4 and tuple(attn_mask.shape) == (B, Hq, Sq, Skv), "attn_mask must be expanded to [B,Hq,Sq,Skv]"
    kind = SAB_MASK_BOOL if attn_mask.dtype == torch.bool else SAB_MASK_BIAS
    assert kind == SAB_MASK_BOOL or attn_mask.dtype == output.dtype, "attn_mask must be bool or the q / output dtype"
    qs, ks, os_ = _bhs_strides(query, tensor_layout), _bhs_strides(key, tensor_layout), _bhs_strides(output, tensor_layout)
    lse = _lse(query, (B, Hq, Sq), return_lse)
    with torch.cuda.device(query.device):
        check(lib().sab_qk_int8_sv_f16_attn_masked(query.data_ptr(), key.data_ptr(), value.data_ptr(), output.data_ptr(),
                                                   lse.data_ptr() if return_lse else None, query_scale.data_ptr(),
                                                   key_scale.data_ptr(), _dt(output), B, Hq, Hkv, Sq, Skv, D, *qs, *ks,
                                                   _v_pad(value), *os_, q_quant_gran, k_quant_gran, float(sm_scale),
                                                   fold_sm_scale, attn_mask.data_ptr(), kind, *attn_mask.stride(),
                                                   _stream(query)))
    return lse


@qk_int8_sv_f16_attn_masked.register_fake
def _(query, key, value, output, query_scale, key_scale, attn_mask, tensor_layout, q_quant_gran, k_quant_gran, sm_scale,
      fold_sm_scale, return_lse):
    B, Hq, Sq, D = _bhsd(query, tensor_layout)
    return _lse(query, (B, Hq, Sq), return_lse)


@torch.library.custom_op("sageattention_b200::qk_int8_sv_f16_attn_varlen", mutates_args=("output",), device_types="cuda")
def qk_int8_sv_f16_attn_varlen(query: torch.Tensor, key: torch.Tensor, value: torch.Tensor, output: torch.Tensor,
                               query_scale: torch.Tensor, key_scale: torch.Tensor, cu_seqlens_q: torch.Tensor,
                               cu_seqlens_k: torch.Tensor, cu_pad_v: torch.Tensor, cu_q_scale: torch.Tensor,
                               cu_k_scale: torch.Tensor, max_seqlen_q: int, is_causal: int, sm_scale: float,
                               fold_sm_scale: int, return_lse: int = 0) -> torch.Tensor:
    """Packed [T,H,D] form of qk_int8_sv_f16_attn: mutates `output`, returns lse ([Hq,Tq] fp32 in log2 units, row
    h*Tq + cu_seqlens_q[b] + i; rows past cu_seqlens_q[-1] are not written), or an empty tensor when return_lse == 0."""
    Tq, Hq, D = query.shape
    Tk, Hkv, _ = key.shape
    nseq = cu_seqlens_q.numel() - 1
    lse = _lse(query, (Hq, Tq), return_lse)
    with torch.cuda.device(query.device):
        check(lib().sab_qk_int8_sv_f16_attn(query.data_ptr(), key.data_ptr(), value.data_ptr(), output.data_ptr(),
                                            lse.data_ptr() if return_lse else None,
                                            query_scale.data_ptr(), key_scale.data_ptr(), _dt(output), nseq, Hq, Hkv, Tq, Tk, D,
                                            0, query.stride(1), query.stride(0), 0, key.stride(1), key.stride(0), _v_pad(value),
                                            0, output.stride(1), output.stride(0), is_causal, _capi.SAB_GRAN_PER_BLOCK,
                                            _capi.SAB_GRAN_PER_BLOCK, float(sm_scale), fold_sm_scale, cu_seqlens_q.data_ptr(),
                                            cu_seqlens_k.data_ptr(), cu_pad_v.data_ptr(), cu_q_scale.data_ptr(),
                                            cu_k_scale.data_ptr(), max_seqlen_q, _stream(query)))
    return lse


@qk_int8_sv_f16_attn_varlen.register_fake
def _(query, key, value, output, query_scale, key_scale, cu_seqlens_q, cu_seqlens_k, cu_pad_v, cu_q_scale, cu_k_scale,
      max_seqlen_q, is_causal, sm_scale, fold_sm_scale, return_lse=0):
    return _lse(query, (query.size(1), query.size(0)), return_lse)


# ----------------------------------------------------------------------------------------------- 8-bit paged KV cache
def kvcache8_chunk_keys() -> int:
    """Keys per split-KV chunk of sageattn_kvcache8 (a compile-time constant of the library)."""
    return lib().sab_kvcache8_chunk_keys()


@torch.library.custom_op("sageattention_b200::kvcache8_write", mutates_args=("k_pages", "k_scale", "v_pages", "v_scale"),
                         device_types="cuda")
def kvcache8_write(k: torch.Tensor, v: torch.Tensor, k_smooth: torch.Tensor, slot_mapping: torch.Tensor, k_pages: torch.Tensor,
                   k_scale: torch.Tensor, v_pages: torch.Tensor, v_scale: torch.Tensor) -> None:
    """Quantise tokens k, v [T,Hkv,D] into the slots slot_mapping [T] of an 8-bit paged cache (include/sageattn_b200.h,
    sab_kvcache8_write)."""
    T, Hkv, D = k.shape
    num_pages, page_size = k_pages.shape[:2]
    with torch.cuda.device(k.device):
        check(lib().sab_kvcache8_write(k.data_ptr(), v.data_ptr(), _dt(k), k_smooth.data_ptr(), slot_mapping.data_ptr(), T, Hkv, D,
                                       k.stride(0), k.stride(1), v.stride(0), v.stride(1), k_pages.data_ptr(), k_scale.data_ptr(),
                                       v_pages.data_ptr(), v_scale.data_ptr(), num_pages, page_size, _stream(k)))


@kvcache8_write.register_fake
def _(k, v, k_smooth, slot_mapping, k_pages, k_scale, v_pages, v_scale):
    return None


@torch.library.custom_op("sageattention_b200::kvcache8_attn", mutates_args=("output",), device_types="cuda")
def kvcache8_attn(q: torch.Tensor, k_pages: torch.Tensor, k_scale: torch.Tensor, v_pages: torch.Tensor, v_scale: torch.Tensor,
                  k_smooth: torch.Tensor, output: torch.Tensor, cu_seqlens_q: torch.Tensor, seqused_k: torch.Tensor,
                  block_table: torch.Tensor, max_seqlen_q: int, is_causal: int, sm_scale: float, return_lse: int) -> torch.Tensor:
    """Split-KV attention of packed q [Tq,Hq,D] against an 8-bit paged cache (include/sageattn_b200.h, sab_kvcache8_attn).  Returns
    the [Hq,Tq] natural-log LSE when return_lse, else an empty tensor."""
    Tq, Hq, D = q.shape
    page_size, Hkv = k_pages.size(1), k_pages.size(2)
    nseq, max_pages = block_table.shape
    lse = torch.empty((Hq, Tq) if return_lse else (0,), dtype=torch.float32, device=q.device)
    with torch.cuda.device(q.device):
        ws = torch.empty(lib().sab_kvcache8_workspace_bytes(Tq, Hq, D, max_pages * page_size), dtype=torch.uint8, device=q.device)
        check(lib().sab_kvcache8_attn(q.data_ptr(), _dt(q), k_pages.data_ptr(), k_scale.data_ptr(), v_pages.data_ptr(),
                                      v_scale.data_ptr(), k_smooth.data_ptr(), output.data_ptr(), lse.data_ptr() if return_lse else None,
                                      cu_seqlens_q.data_ptr(), seqused_k.data_ptr(), block_table.data_ptr(), block_table.stride(0),
                                      max_pages, nseq, Tq, Hq, Hkv, D, page_size, q.stride(0), q.stride(1), output.stride(0),
                                      output.stride(1), max_seqlen_q, is_causal, float(sm_scale), ws.data_ptr(), _stream(q)))
    return lse


@kvcache8_attn.register_fake
def _(q, k_pages, k_scale, v_pages, v_scale, k_smooth, output, cu_seqlens_q, seqused_k, block_table, max_seqlen_q, is_causal,
      sm_scale, return_lse):
    Tq, Hq, _ = q.shape
    return q.new_empty((Hq, Tq) if return_lse else (0,), dtype=torch.float32)


@torch.library.custom_op("sageattention_b200::kvcache8_prefill", mutates_args=("output",), device_types="cuda")
def kvcache8_prefill(q: torch.Tensor, k_pages: torch.Tensor, k_scale: torch.Tensor, v_pages: torch.Tensor, v_scale: torch.Tensor,
                     k_smooth: torch.Tensor, output: torch.Tensor, cu_seqlens_q: torch.Tensor, seqused_k: torch.Tensor,
                     block_table: torch.Tensor, max_seqlen_q: int, is_causal: int, sm_scale: float, return_lse: int) -> torch.Tensor:
    """Attention of packed query chunks q [Tq,Hq,D] of any length against an 8-bit paged cache (include/sageattn_b200.h,
    sab_kvcache8_prefill).  Returns the [Hq,Tq] natural-log LSE when return_lse, else an empty tensor."""
    Tq, Hq, D = q.shape
    page_size, Hkv = k_pages.size(1), k_pages.size(2)
    nseq, max_pages = block_table.shape
    lse = torch.empty((Hq, Tq) if return_lse else (0,), dtype=torch.float32, device=q.device)
    with torch.cuda.device(q.device):
        check(lib().sab_kvcache8_prefill(q.data_ptr(), _dt(q), k_pages.data_ptr(), k_scale.data_ptr(), v_pages.data_ptr(),
                                         v_scale.data_ptr(), k_smooth.data_ptr(), output.data_ptr(),
                                         lse.data_ptr() if return_lse else None, cu_seqlens_q.data_ptr(), seqused_k.data_ptr(),
                                         block_table.data_ptr(), block_table.stride(0), max_pages, nseq, Tq, Hq, Hkv, D, page_size,
                                         q.stride(0), q.stride(1), output.stride(0), output.stride(1), max_seqlen_q, is_causal,
                                         float(sm_scale), _stream(q)))
    return lse


@kvcache8_prefill.register_fake
def _(q, k_pages, k_scale, v_pages, v_scale, k_smooth, output, cu_seqlens_q, seqused_k, block_table, max_seqlen_q, is_causal,
      sm_scale, return_lse):
    Tq, Hq, _ = q.shape
    return q.new_empty((Hq, Tq) if return_lse else (0,), dtype=torch.float32)


@torch.library.custom_op("sageattention_b200::kvcache8_attn_window", mutates_args=("output",), device_types="cuda")
def kvcache8_attn_window(q: torch.Tensor, k_pages: torch.Tensor, k_scale: torch.Tensor, v_pages: torch.Tensor, v_scale: torch.Tensor,
                         k_smooth: torch.Tensor, output: torch.Tensor, cu_seqlens_q: torch.Tensor, seqused_k: torch.Tensor,
                         block_table: torch.Tensor, max_seqlen_q: int, is_causal: int, sm_scale: float, return_lse: int,
                         window_left: int, window_right: int) -> torch.Tensor:
    """kvcache8_attn with a sliding window (include/sageattn_b200.h, sab_kvcache8_attn_window); window_left / window_right int32,
    >= -1.  Returns the [Hq,Tq] natural-log LSE when return_lse, else an empty tensor."""
    Tq, Hq, D = q.shape
    page_size, Hkv = k_pages.size(1), k_pages.size(2)
    nseq, max_pages = block_table.shape
    lse = torch.empty((Hq, Tq) if return_lse else (0,), dtype=torch.float32, device=q.device)
    with torch.cuda.device(q.device):
        ws = torch.empty(lib().sab_kvcache8_workspace_bytes(Tq, Hq, D, max_pages * page_size), dtype=torch.uint8, device=q.device)
        check(lib().sab_kvcache8_attn_window(q.data_ptr(), _dt(q), k_pages.data_ptr(), k_scale.data_ptr(), v_pages.data_ptr(),
                                             v_scale.data_ptr(), k_smooth.data_ptr(), output.data_ptr(),
                                             lse.data_ptr() if return_lse else None, cu_seqlens_q.data_ptr(), seqused_k.data_ptr(),
                                             block_table.data_ptr(), block_table.stride(0), max_pages, nseq, Tq, Hq, Hkv, D, page_size,
                                             q.stride(0), q.stride(1), output.stride(0), output.stride(1), max_seqlen_q, is_causal,
                                             float(sm_scale), ws.data_ptr(), window_left, window_right, _stream(q)))
    return lse


@kvcache8_attn_window.register_fake
def _(q, k_pages, k_scale, v_pages, v_scale, k_smooth, output, cu_seqlens_q, seqused_k, block_table, max_seqlen_q, is_causal,
      sm_scale, return_lse, window_left, window_right):
    Tq, Hq, _ = q.shape
    return q.new_empty((Hq, Tq) if return_lse else (0,), dtype=torch.float32)


@torch.library.custom_op("sageattention_b200::kvcache8_prefill_window", mutates_args=("output",), device_types="cuda")
def kvcache8_prefill_window(q: torch.Tensor, k_pages: torch.Tensor, k_scale: torch.Tensor, v_pages: torch.Tensor,
                            v_scale: torch.Tensor, k_smooth: torch.Tensor, output: torch.Tensor, cu_seqlens_q: torch.Tensor,
                            seqused_k: torch.Tensor, block_table: torch.Tensor, max_seqlen_q: int, is_causal: int, sm_scale: float,
                            return_lse: int, window_left: int, window_right: int) -> torch.Tensor:
    """kvcache8_prefill with a sliding window (include/sageattn_b200.h, sab_kvcache8_prefill_window); window_left / window_right
    int32, >= -1.  Returns the [Hq,Tq] natural-log LSE when return_lse, else an empty tensor."""
    Tq, Hq, D = q.shape
    page_size, Hkv = k_pages.size(1), k_pages.size(2)
    nseq, max_pages = block_table.shape
    lse = torch.empty((Hq, Tq) if return_lse else (0,), dtype=torch.float32, device=q.device)
    with torch.cuda.device(q.device):
        check(lib().sab_kvcache8_prefill_window(q.data_ptr(), _dt(q), k_pages.data_ptr(), k_scale.data_ptr(), v_pages.data_ptr(),
                                                v_scale.data_ptr(), k_smooth.data_ptr(), output.data_ptr(),
                                                lse.data_ptr() if return_lse else None, cu_seqlens_q.data_ptr(), seqused_k.data_ptr(),
                                                block_table.data_ptr(), block_table.stride(0), max_pages, nseq, Tq, Hq, Hkv, D,
                                                page_size, q.stride(0), q.stride(1), output.stride(0), output.stride(1), max_seqlen_q,
                                                is_causal, float(sm_scale), window_left, window_right, _stream(q)))
    return lse


@kvcache8_prefill_window.register_fake
def _(q, k_pages, k_scale, v_pages, v_scale, k_smooth, output, cu_seqlens_q, seqused_k, block_table, max_seqlen_q, is_causal,
      sm_scale, return_lse, window_left, window_right):
    Tq, Hq, _ = q.shape
    return q.new_empty((Hq, Tq) if return_lse else (0,), dtype=torch.float32)


@torch.library.custom_op("sageattention_b200::kvcache8_attn_shared", mutates_args=("output",), device_types="cuda")
def kvcache8_attn_shared(q: torch.Tensor, k_pages: torch.Tensor, k_scale: torch.Tensor, v_pages: torch.Tensor, v_scale: torch.Tensor,
                         k_smooth: torch.Tensor, output: torch.Tensor, cu_seqlens_q: torch.Tensor, seqused_k: torch.Tensor,
                         block_table: torch.Tensor, max_seqlen_q: int, is_causal: int, sm_scale: float, return_lse: int,
                         shared_prefix_len: int) -> torch.Tensor:
    """kvcache8_attn with the first shared_prefix_len keys (whole chunks) shared by every sequence through table row 0
    (include/sageattn_b200.h, sab_kvcache8_attn_shared); shared_prefix_len int32, >= 0.  Returns the [Hq,Tq] natural-log LSE
    when return_lse, else an empty tensor."""
    Tq, Hq, D = q.shape
    page_size, Hkv = k_pages.size(1), k_pages.size(2)
    nseq, max_pages = block_table.shape
    lse = torch.empty((Hq, Tq) if return_lse else (0,), dtype=torch.float32, device=q.device)
    with torch.cuda.device(q.device):
        ws = torch.empty(lib().sab_kvcache8_workspace_bytes(Tq, Hq, D, max_pages * page_size), dtype=torch.uint8, device=q.device)
        check(lib().sab_kvcache8_attn_shared(q.data_ptr(), _dt(q), k_pages.data_ptr(), k_scale.data_ptr(), v_pages.data_ptr(),
                                             v_scale.data_ptr(), k_smooth.data_ptr(), output.data_ptr(),
                                             lse.data_ptr() if return_lse else None, cu_seqlens_q.data_ptr(), seqused_k.data_ptr(),
                                             block_table.data_ptr(), block_table.stride(0), max_pages, nseq, Tq, Hq, Hkv, D, page_size,
                                             q.stride(0), q.stride(1), output.stride(0), output.stride(1), max_seqlen_q, is_causal,
                                             float(sm_scale), ws.data_ptr(), shared_prefix_len, _stream(q)))
    return lse


@kvcache8_attn_shared.register_fake
def _(q, k_pages, k_scale, v_pages, v_scale, k_smooth, output, cu_seqlens_q, seqused_k, block_table, max_seqlen_q, is_causal,
      sm_scale, return_lse, shared_prefix_len):
    Tq, Hq, _ = q.shape
    return q.new_empty((Hq, Tq) if return_lse else (0,), dtype=torch.float32)
