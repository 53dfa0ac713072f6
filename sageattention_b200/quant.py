"""Quantisation front-end with the reference's Python signatures (sageattention/quant.py:22-293,
sageattention/triton/quant_per_thread.py:154-203, quant_per_block.py:49-101,
quant_per_block_varlen.py:60-104) on top of the sm_90a kernels.  Outputs are allocated here and
passed to the C ABI (the reference's ownership convention)."""
from typing import Optional, Tuple
import torch

from . import ops
from ._capi import SAB_SEM_CUDA, SAB_SEM_TRITON

_LOG2E = 1.44269504


def _layout(tensor_layout: str) -> int:
    if tensor_layout == "HND":
        return 1
    if tensor_layout == "NHD":
        return 0
    raise ValueError(f"Unknown tensor layout: {tensor_layout}")


def _dims(t: torch.Tensor, tensor_layout: str):
    if tensor_layout == "HND":
        b, h, s, d = t.shape
    elif tensor_layout == "NHD":
        b, s, h, d = t.shape
    else:
        raise ValueError(f"Unknown tensor layout: {tensor_layout}")
    return b, h, s, d


def _squeeze_mean(km: Optional[torch.Tensor], b: int, h: int, d: int) -> Optional[torch.Tensor]:
    """Accept km as [B,H,D] or with the reference's keepdim seq axis ([B,H,1,D] / [B,1,H,D])."""
    if km is None:
        return None
    km = km.reshape(b, h, d) if km.numel() == b * h * d else km
    assert km.shape == (b, h, d), f"km must have {b * h * d} elements"
    return km.contiguous()


def k_mean(k: torch.Tensor, tensor_layout: str = "HND") -> torch.Tensor:
    """`k.mean(dim=seq, keepdim=True)` (sageattention/core.py:773): fp32 accumulation, result in k.dtype,
    returned with the reference's keepdim shape."""
    b, h, s, d = _dims(k, tensor_layout)
    mean = torch.empty((b, h, d), dtype=k.dtype, device=k.device)
    ops.k_mean(k, mean, _layout(tensor_layout))
    return mean.view(b, h, 1, d) if tensor_layout == "HND" else mean.view(b, 1, h, d)


def per_block_int8(q: torch.Tensor, k: torch.Tensor, km: Optional[torch.Tensor] = None, BLKQ: int = 128,
                   BLKK: int = 64, sm_scale: Optional[float] = None, tensor_layout: str = "HND",
                   semantics: str = "triton") -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
    """Per-block INT8 of q (pre-scaled by sm_scale*log2e) and k (optionally smoothed by km).
    semantics="triton" reproduces sageattention/triton/quant_per_block.py:49-101 bit-exactly;
    semantics="cuda" reproduces sageattention/quant.py:22-103 (csrc/fused/fused.cu)."""
    b, h_qo, qo_len, head_dim = _dims(q, tensor_layout)
    _, h_kv, kv_len, _ = _dims(k, tensor_layout)
    lay = _layout(tensor_layout)
    sem = SAB_SEM_TRITON if semantics == "triton" else SAB_SEM_CUDA
    q_int8 = torch.empty(q.shape, dtype=torch.int8, device=q.device)
    k_int8 = torch.empty(k.shape, dtype=torch.int8, device=k.device)
    q_scale = torch.empty((b, h_qo, (qo_len + BLKQ - 1) // BLKQ), device=q.device, dtype=torch.float32)
    k_scale = torch.empty((b, h_kv, (kv_len + BLKK - 1) // BLKK), device=q.device, dtype=torch.float32)
    if sm_scale is None:
        sm_scale = head_dim ** -0.5
    ops.quant_per_block_int8(q, None, q_int8, q_scale, BLKQ, lay, sem, True, sm_scale * _LOG2E)
    ops.quant_per_block_int8(k, _squeeze_mean(km, b, h_kv, head_dim), k_int8, k_scale, BLKK, lay, sem, False, 1.0)
    return q_int8, q_scale, k_int8, k_scale


def quant_q_int8(q: torch.Tensor, qk_quant_gran: str = "per_thread", tensor_layout: str = "HND"):
    """Q side of per_warp_int8 / per_thread_int8 (BLKQ=128, WARPQ=32): returns (q_int8, q_scale)."""
    b, h_qo, qo_len, _ = _dims(q, tensor_layout)
    lay = _layout(tensor_layout)
    q_int8 = torch.empty(q.shape, dtype=torch.int8, device=q.device)
    nblk = (qo_len + 127) // 128 * 4
    if qk_quant_gran == "per_warp":
        q_scale = torch.empty((b, h_qo, nblk), device=q.device, dtype=torch.float32)
        ops.quant_per_block_int8(q, None, q_int8, q_scale, 32, lay, SAB_SEM_CUDA, False, 1.0)
    else:
        q_scale = torch.empty((b, h_qo, nblk * 8), device=q.device, dtype=torch.float32)
        ops.quant_per_thread_int8(q, None, q_int8, q_scale, lay, False)
    return q_int8, q_scale


def quant_k_int8(k: torch.Tensor, km: Optional[torch.Tensor] = None, qk_quant_gran: str = "per_thread",
                 tensor_layout: str = "HND"):
    """K side of per_warp_int8 / per_thread_int8 (BLKK=64, WARPK=64) with the fused `k - km`: returns (k_int8, k_scale)."""
    b, h_kv, kv_len, head_dim = _dims(k, tensor_layout)
    lay = _layout(tensor_layout)
    k_int8 = torch.empty(k.shape, dtype=torch.int8, device=k.device)
    nblk = (kv_len + 63) // 64
    mean = _squeeze_mean(km, b, h_kv, head_dim)
    if qk_quant_gran == "per_warp":
        k_scale = torch.empty((b, h_kv, nblk), device=k.device, dtype=torch.float32)
        ops.quant_per_block_int8(k, mean, k_int8, k_scale, 64, lay, SAB_SEM_CUDA, False, 1.0)
    else:
        k_scale = torch.empty((b, h_kv, nblk * 4), device=k.device, dtype=torch.float32)
        ops.quant_per_thread_int8(k, mean, k_int8, k_scale, lay, True)
    return k_int8, k_scale


def smooth_quant_k(k: torch.Tensor, qk_quant_gran: str = "per_thread", tensor_layout: str = "HND"):
    """`km = k.mean(dim=seq, keepdim=True)` (sageattention/core.py:773) + the K half of per_thread_int8 / per_warp_int8 in ONE launch
    (csrc/quant.cu k_smooth_quant_kernel: a thread-block cluster per (b,h) reduces the mean through distributed shared memory and
    quantises right away, so K crosses HBM once).  Returns (km, k_int8, k_scale); k_int8 / k_scale are bit-identical to
    quant_k_int8(k, km) with the returned km (km itself is a different fp32 summation order than k_mean(): same value up to one
    ulp on rare channels).  OPT-IN: the default path is k_mean + quant_k_int8."""
    from ._capi import SAB_GRAN_PER_WARP, SAB_GRAN_PER_THREAD
    b, h_kv, kv_len, head_dim = _dims(k, tensor_layout)
    lay = _layout(tensor_layout)
    k_int8 = torch.empty(k.shape, dtype=torch.int8, device=k.device)
    nblk = (kv_len + 63) // 64
    mean = torch.empty((b, h_kv, head_dim), dtype=k.dtype, device=k.device)
    if qk_quant_gran == "per_warp":
        k_scale = torch.empty((b, h_kv, nblk), device=k.device, dtype=torch.float32)
        gran = SAB_GRAN_PER_WARP
    else:
        k_scale = torch.empty((b, h_kv, nblk * 4), device=k.device, dtype=torch.float32)
        gran = SAB_GRAN_PER_THREAD
    ops.k_smooth_quant_int8(k, mean, k_int8, k_scale, lay, gran)
    km = mean.view(b, h_kv, 1, head_dim) if tensor_layout == "HND" else mean.view(b, 1, h_kv, head_dim)
    return km, k_int8, k_scale


def per_warp_int8(q: torch.Tensor, k: torch.Tensor, km: Optional[torch.Tensor] = None, BLKQ: int = 128,
                  WARPQ: int = 32, BLKK: int = 64, tensor_layout: str = "HND"):
    """sageattention/quant.py:105-180: q per WARPQ-row block, k per BLKK block with fused (k - km) in fp32;
    CUDA rounding semantics (cvt.rni, amax floored at 1e-7)."""
    assert BLKQ == 128 and WARPQ == 32 and BLKK == 64, "sm_90a kernel supports the reference defaults"
    q_int8, q_scale = quant_q_int8(q, "per_warp", tensor_layout)
    k_int8, k_scale = quant_k_int8(k, km, "per_warp", tensor_layout)
    return q_int8, q_scale, k_int8, k_scale


def per_thread_int8(q: torch.Tensor, k: torch.Tensor, km: Optional[torch.Tensor] = None, BLKQ: int = 128,
                    WARPQ: int = 32, BLKK: int = 64, WARPK: int = 64, sm_scale: Optional[float] = None,
                    tensor_layout: str = "HND"):
    """sageattention/triton/quant_per_thread.py:154-203 (8 q scales per 32-row block, 4 k scales per
    64-key block; `k - km` rounded to the input dtype first; scale = amax/127 + 1e-7)."""
    assert BLKQ == 128 and WARPQ == 32 and BLKK == 64 and WARPK == 64, "sm_90a kernel supports the reference defaults"
    q_int8, q_scale = quant_q_int8(q, "per_thread", tensor_layout)
    k_int8, k_scale = quant_k_int8(k, km, "per_thread", tensor_layout)
    return q_int8, q_scale, k_int8, k_scale


def per_block_int8_varlen(q, k, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k, BLKQ=128, BLKK=64,
                          sm_scale=None, km: Optional[torch.Tensor] = None):
    """sageattention/triton/quant_per_block_varlen.py:60-104 on packed [T,H,D] tensors.  `km`
    ([1,H,D] or [H,D]) is subtracted inside the kernel (the reference does `k = k - km` in torch first)."""
    h_qo, h_kv, head_dim = q.shape[1], k.shape[1], q.shape[-1]
    q_int8 = torch.empty(q.shape, dtype=torch.int8, device=q.device)
    k_int8 = torch.empty(k.shape, dtype=torch.int8, device=k.device)
    cu_q32, cu_k32 = cu_seqlens_q.to(torch.int32), cu_seqlens_k.to(torch.int32)
    q_batch_len = cu_q32[1:] - cu_q32[:-1]
    k_batch_len = cu_k32[1:] - cu_k32[:-1]
    cu_seqlens_q_scale = torch.nn.functional.pad(torch.cumsum((q_batch_len + BLKQ - 1) // BLKQ, dim=0), (1, 0), value=0).to(torch.int32)
    cu_seqlens_k_scale = torch.nn.functional.pad(torch.cumsum((k_batch_len + BLKK - 1) // BLKK, dim=0), (1, 0), value=0).to(torch.int32)
    nseq = cu_q32.numel() - 1
    # upper bounds avoid a device->host sync (reference: q_scale rows = cu_seqlens_q_scale[-1])
    q_scale = torch.empty((q.shape[0] // BLKQ + nseq, h_qo), device=q.device, dtype=torch.float32)
    k_scale = torch.empty((k.shape[0] // BLKK + nseq, h_kv), device=k.device, dtype=torch.float32)
    if sm_scale is None:
        sm_scale = head_dim ** -0.5
    kmean = None if km is None else km.reshape(h_kv, head_dim).contiguous()
    ops.quant_per_block_int8_varlen(q, None, q_int8, q_scale, cu_q32, cu_seqlens_q_scale, max_seqlen_q, BLKQ, True, sm_scale * _LOG2E)
    ops.quant_per_block_int8_varlen(k, kmean, k_int8, k_scale, cu_k32, cu_seqlens_k_scale, max_seqlen_k, BLKK, False, 1.0)
    return q_int8, q_scale, k_int8, k_scale, cu_seqlens_q_scale, cu_seqlens_k_scale


def per_channel_fp8(v: torch.Tensor, tensor_layout: str = "HND", scale_max: float = 448.0, smooth_v: bool = True, fused: bool = False):
    """Per-channel e4m3 quantisation of V (sageattention/quant.py:224-293).
    Returns (v_fp8, v_scale, vm).  v_fp8 is ``[B, H_kv, D, ceil(kv_len/128)*128]`` float8_e4m3fn
    (token-contiguous "V transposed", zero padded) for BOTH layouts; unlike the reference it is not
    16-token permuted (an mma.sync artefact the wgmma kernel does not need)."""
    b, h_kv, kv_len, head_dim = _dims(v, tensor_layout)
    padded_len = (kv_len + 127) // 128 * 128
    v_fp8 = torch.empty((b, h_kv, head_dim, padded_len), dtype=torch.float8_e4m3fn, device=v.device)
    v_scale = torch.empty((b, h_kv, head_dim), dtype=torch.float32, device=v.device)
    vm = torch.empty((b, h_kv, head_dim), dtype=torch.float32, device=v.device) if smooth_v else None
    if fused:   # statistics + quantisation in one cluster launch (opt-in)
        ops.per_channel_fp8_fused(v, v_fp8, v_scale, vm, _layout(tensor_layout), scale_max)
    else:
        ops.per_channel_fp8(v, v_fp8, v_scale, vm, _layout(tensor_layout), scale_max)
    return v_fp8, v_scale, vm


def per_channel_fp8_varlen(v: torch.Tensor, cu_seqlens_k: torch.Tensor, max_seqlen_k: int, scale_max: float = 448.0):
    """Packed-V form: v [T,H,D] -> v_fp8 [H, D, T_pad] where sequence i occupies token columns
    [cu_pad[i], cu_pad[i] + ceil(L_i/128)*128).  Returns (v_fp8, v_scale [H,D], cu_pad)."""
    T, h_kv, head_dim = v.shape
    cu32 = cu_seqlens_k.to(torch.int32)
    lens = cu32[1:] - cu32[:-1]
    cu_pad = torch.nn.functional.pad(torch.cumsum((lens + 127) // 128 * 128, dim=0), (1, 0), value=0).to(torch.int32)
    nseq = cu32.numel() - 1
    t_pad = (T + 127 * nseq + 127) // 128 * 128          # upper bound, no host sync
    v_fp8 = torch.empty((h_kv, head_dim, t_pad), dtype=torch.float8_e4m3fn, device=v.device)
    v_scale = torch.empty((h_kv, head_dim), dtype=torch.float32, device=v.device)
    ops.per_channel_fp8_varlen(v, v_fp8, v_scale, cu32, cu_pad, max_seqlen_k, scale_max)
    return v_fp8, v_scale, cu_pad


def transpose_v_f16(v: torch.Tensor, tensor_layout: str = "HND") -> torch.Tensor:
    """`v.to(torch.float16)` (sageattention/core.py:297-298) in the layout the kind::f16 PV MMA consumes:
    ``[B, H_kv, D, ceil(kv_len/128)*128]`` fp16, token-contiguous, zero padded."""
    b, h_kv, kv_len, head_dim = _dims(v, tensor_layout)
    padded_len = (kv_len + 127) // 128 * 128
    v_t = torch.empty((b, h_kv, head_dim, padded_len), dtype=torch.float16, device=v.device)
    ops.v_transpose_f16(v, v_t, _layout(tensor_layout))
    return v_t


def transpose_v_f16_varlen(v: torch.Tensor, cu_seqlens_k: torch.Tensor, max_seqlen_k: int):
    """Packed form: v [T,H,D] -> [H, D, T_pad] fp16 with every sequence padded to 128 tokens; returns (v_t, cu_pad)."""
    T, h_kv, head_dim = v.shape
    cu32 = cu_seqlens_k.to(torch.int32)
    lens = cu32[1:] - cu32[:-1]
    cu_pad = torch.nn.functional.pad(torch.cumsum((lens + 127) // 128 * 128, dim=0), (1, 0), value=0).to(torch.int32)
    nseq = cu32.numel() - 1
    t_pad = (T + 127 * nseq + 127) // 128 * 128
    v_t = torch.empty((h_kv, head_dim, t_pad), dtype=torch.float16, device=v.device)
    ops.v_transpose_f16_varlen(v, v_t, cu32, cu_pad, max_seqlen_k)
    return v_t, cu_pad


# ------------------------------------------------------------------------------------------------ packed, per-sequence statistics
def varlen_block_table(cu_seqlens: torch.Tensor, blk: int) -> torch.Tensor:
    """[nseq+1] int32: exclusive cumsum of ceil(L_b / blk) over the sequence lengths of cu_seqlens, on its device (no sync)."""
    cu32 = cu_seqlens.to(torch.int32)
    lens = cu32[1:] - cu32[:-1]
    return torch.nn.functional.pad(torch.cumsum((lens + blk - 1) // blk, dim=0), (1, 0), value=0).to(torch.int32)


def varlen_scale_rows(T: int, nseq: int, blk: int, mult: int) -> int:
    """Rows of a per-sequence scale table without a device->host sync: sum_b ceil(L_b/blk) <= T // blk + nseq blocks."""
    return (T // blk + nseq) * mult


def k_mean_varlen(k: torch.Tensor, cu_seqlens_k: torch.Tensor, max_seqlen_k: int) -> torch.Tensor:
    """Per-sequence `k.mean(dim=seq)` of packed k [T,H,D]: [nseq,H,D] in k.dtype, each sequence bit for bit k_mean() of that
    sequence alone (0 for an empty one)."""
    nseq = cu_seqlens_k.numel() - 1
    mean = torch.empty((nseq, k.size(1), k.size(2)), dtype=k.dtype, device=k.device)
    ops.k_mean_varlen(k, mean, cu_seqlens_k.to(torch.int32), max_seqlen_k)
    return mean


def quant_q_int8_varlen(q: torch.Tensor, cu_seqlens_q: torch.Tensor, max_seqlen_q: int, qk_quant_gran: str = "per_thread"):
    """quant_q_int8 per packed sequence: (q_int8 [T,H,D], q_scale [rows,H], cu_q_scale [nseq+1] in 128-row blocks).  Sequence
    b's scales are rows [cu_q_scale[b] * mult, ...) with mult 4 (per_warp) or 32 (per_thread), in quant_q_int8's order."""
    from ._capi import SAB_GRAN_PER_WARP, SAB_GRAN_PER_THREAD
    nseq = cu_seqlens_q.numel() - 1
    mult = 4 if qk_quant_gran == "per_warp" else 32
    cu_q_scale = varlen_block_table(cu_seqlens_q, 128)
    q_int8 = torch.empty(q.shape, dtype=torch.int8, device=q.device)
    q_scale = torch.empty((varlen_scale_rows(q.size(0), nseq, 128, mult), q.size(1)), dtype=torch.float32, device=q.device)
    ops.quant_int8_varlen(q, None, q_int8, q_scale, cu_seqlens_q.to(torch.int32), cu_q_scale, max_seqlen_q,
                          SAB_GRAN_PER_WARP if qk_quant_gran == "per_warp" else SAB_GRAN_PER_THREAD, False)
    return q_int8, q_scale, cu_q_scale


def quant_k_int8_varlen(k: torch.Tensor, km: Optional[torch.Tensor], cu_seqlens_k: torch.Tensor, max_seqlen_k: int,
                        qk_quant_gran: str = "per_thread"):
    """quant_k_int8 per packed sequence with the fused `k - km[b]` (km [nseq,H,D] or None): (k_int8, k_scale [rows,H],
    cu_k_scale [nseq+1] in 64-key blocks).  Sequence b's scales are rows [cu_k_scale[b] * mult, ...), mult 1 (per_warp) or 4."""
    from ._capi import SAB_GRAN_PER_WARP, SAB_GRAN_PER_THREAD
    nseq = cu_seqlens_k.numel() - 1
    mult = 1 if qk_quant_gran == "per_warp" else 4
    cu_k_scale = varlen_block_table(cu_seqlens_k, 64)
    k_int8 = torch.empty(k.shape, dtype=torch.int8, device=k.device)
    k_scale = torch.empty((varlen_scale_rows(k.size(0), nseq, 64, mult), k.size(1)), dtype=torch.float32, device=k.device)
    ops.quant_int8_varlen(k, None if km is None else km.contiguous(), k_int8, k_scale, cu_seqlens_k.to(torch.int32), cu_k_scale,
                          max_seqlen_k, SAB_GRAN_PER_WARP if qk_quant_gran == "per_warp" else SAB_GRAN_PER_THREAD, True)
    return k_int8, k_scale, cu_k_scale


def per_channel_fp8_varlen_seq(v: torch.Tensor, cu_seqlens_k: torch.Tensor, max_seqlen_k: int, scale_max: float = 448.0,
                               smooth_v: bool = False):
    """per_channel_fp8 per packed sequence: (v_fp8 [H,D,T_pad], v_scale [nseq,H,D], vm [nseq,H,D] or None, cu_pad).  Sequence b
    occupies token columns [cu_pad[b], cu_pad[b] + ceil(L_b/128)*128), zero padded, as in per_channel_fp8_varlen."""
    T, h_kv, head_dim = v.shape
    nseq = cu_seqlens_k.numel() - 1
    cu_pad = varlen_block_table(cu_seqlens_k, 128) * 128
    t_pad = (T + 127 * nseq + 127) // 128 * 128          # upper bound, no host sync
    v_fp8 = torch.empty((h_kv, head_dim, t_pad), dtype=torch.float8_e4m3fn, device=v.device)
    v_scale = torch.empty((nseq, h_kv, head_dim), dtype=torch.float32, device=v.device)
    vm = torch.empty((nseq, h_kv, head_dim), dtype=torch.float32, device=v.device) if smooth_v else None
    ops.per_channel_fp8_varlen_seq(v, v_fp8, v_scale, vm, cu_seqlens_k.to(torch.int32), cu_pad, max_seqlen_k, scale_max)
    return v_fp8, v_scale, vm, cu_pad


# ------------------------------------------------------------------------------------------------ per-sequence statistics, paged K / V
# The inputs are a paged cache [num_pages, page_size, H, D] and a block table [nseq, max_pages] int32: token t of sequence b is
# cache[block_table[b, t // page_size], t % page_size].  cu_seqlens_k holds the exclusive cumsum of the sequence lengths; the
# outputs are those of the packed forms above on the gathered tensor, bit for bit.  The caller passes the exact packed sizes.
def k_mean_paged(k_cache: torch.Tensor, cu_seqlens_k: torch.Tensor, block_table: torch.Tensor, max_seqlen_k: int) -> torch.Tensor:
    """k_mean_varlen of the gathered K: [nseq,H,D] in the cache's dtype."""
    nseq = cu_seqlens_k.numel() - 1
    mean = torch.empty((nseq, k_cache.size(2), k_cache.size(3)), dtype=k_cache.dtype, device=k_cache.device)
    ops.k_mean_paged(k_cache, mean, cu_seqlens_k, block_table, max_seqlen_k)
    return mean


def quant_k_int8_paged(k_cache: torch.Tensor, km: Optional[torch.Tensor], cu_seqlens_k: torch.Tensor, block_table: torch.Tensor,
                       max_seqlen_k: int, total_k: int, k_blocks: int, qk_quant_gran: str = "per_thread"):
    """quant_k_int8_varlen of the gathered K: (k_int8 [total_k,H,D], k_scale [k_blocks*mult,H], cu_k_scale), with total_k the number
    of keys and k_blocks the number of 64-key blocks, sum_b ceil(L_b/64)."""
    from ._capi import SAB_GRAN_PER_WARP, SAB_GRAN_PER_THREAD
    mult = 1 if qk_quant_gran == "per_warp" else 4
    cu_k_scale = varlen_block_table(cu_seqlens_k, 64)
    H, D = k_cache.size(2), k_cache.size(3)
    k_int8 = torch.empty((total_k, H, D), dtype=torch.int8, device=k_cache.device)
    k_scale = torch.empty((k_blocks * mult, H), dtype=torch.float32, device=k_cache.device)
    ops.quant_int8_paged(k_cache, None if km is None else km.contiguous(), k_int8, k_scale, cu_seqlens_k, cu_k_scale, block_table,
                         max_seqlen_k, SAB_GRAN_PER_WARP if qk_quant_gran == "per_warp" else SAB_GRAN_PER_THREAD)
    return k_int8, k_scale, cu_k_scale


def per_channel_fp8_paged(v_cache: torch.Tensor, cu_seqlens_k: torch.Tensor, block_table: torch.Tensor, max_seqlen_k: int,
                          t_pad: int, scale_max: float = 448.0, smooth_v: bool = False):
    """per_channel_fp8_varlen_seq of the gathered V: (v_fp8 [H,D,t_pad], v_scale [nseq,H,D], vm [nseq,H,D] or None, cu_pad), with
    t_pad = sum_b ceil(L_b/128)*128."""
    nseq = cu_seqlens_k.numel() - 1
    H, D = v_cache.size(2), v_cache.size(3)
    cu_pad = varlen_block_table(cu_seqlens_k, 128) * 128
    v_fp8 = torch.empty((H, D, t_pad), dtype=torch.float8_e4m3fn, device=v_cache.device)
    v_scale = torch.empty((nseq, H, D), dtype=torch.float32, device=v_cache.device)
    vm = torch.empty((nseq, H, D), dtype=torch.float32, device=v_cache.device) if smooth_v else None
    ops.per_channel_fp8_paged(v_cache, v_fp8, v_scale, vm, cu_seqlens_k, cu_pad, block_table, max_seqlen_k, scale_max)
    return v_fp8, v_scale, vm, cu_pad
