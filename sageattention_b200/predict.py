"""Block-sparse masks predicted from pooled Q/K statistics (no reference counterpart): predict_block_mask, whose output is the
block_mask that sageattn_blocksparse takes.  Two sm_90a kernels (csrc/predict.cu): one pass over q and k for the per-block
statistics, one that scores, orders and selects key blocks per 128-query block.  The definition is in include/sageattn_b200.h
(sab_block_stats, sab_predict_block_mask).  predict_block_mask_varlen is the same for every packed sequence on its own, through
the packed forms of the two kernels (sab_block_stats_varlen, sab_predict_block_mask_varlen), for sageattn_varlen_blocksparse."""
import math
from typing import Optional

import torch
import torch.nn.functional as F

from . import ops

MAX_KV_LEN = 1 << 20      # the key limit of sageattn_blocksparse (64 * 16384 key blocks)


def _pad8(x: torch.Tensor) -> torch.Tensor:
    """x with its head dim padded to a multiple of 8, as the statistics kernel reads it (zero padding changes no statistic)."""
    return F.pad(x, (0, 8 - x.size(-1) % 8)) if x.size(-1) % 8 else x


def predict_block_mask(q: torch.Tensor, k: torch.Tensor, *, cdf_threshold: float, sim_threshold: float, tensor_layout: str = "HND",
                       is_causal: bool = False, sm_scale: Optional[float] = None) -> torch.Tensor:
    """A block mask for sageattn_blocksparse predicted from block statistics, in the style of SpargeAttn's first stage
    (training-free).  Blocks are the 128-query x 64-key tiles of sageattn_blocksparse.  For each 128-query block i:

    * the candidates are the key blocks whose self-similarity (the mean cosine similarity of the block's keys, diagonal included)
      is >= sim_threshold, and when is_causal those with 64 j <= 128 i + 127;
    * p = softmax over the candidates of sm_scale * (mean query of block i . mean key of block j);
    * in order of descending p (ties: ascending j) a block is kept while the mass of the blocks before it is < cdf_threshold, so
      the kept blocks are the fewest that carry at least cdf_threshold of p (cdf_threshold >= 1 keeps every candidate);
    * a query block whose self-similarity is < sim_threshold sees every key block, a key block whose self-similarity is
      < sim_threshold is seen by every query block (their means do not represent them), and when is_causal the diagonal blocks
      are always visible and every block past the causal horizon is hidden.

    q [B,Hq,Sq,D] / k [B,Hkv,Skv,D] ("HND") or [B,S,H,D] ("NHD"), fp16 / bf16 CUDA tensors, D <= 128, Hq % Hkv == 0, Skv <= 1048576.
    Statistics are fp32 on the original head dim; sm_scale defaults to D ** -0.5.  The inputs carry no gradient here.
    Returns a contiguous torch.bool [B, Hq, ceil(Sq/128), ceil(Skv/64)] tensor on q's device, the same for both layouts, to be
    passed as-is: sageattn_blocksparse(q, k, v, predict_block_mask(q, k, ...), ...).  Deterministic."""
    assert q.is_cuda, "Input tensors must be on cuda."
    assert q.dtype in [torch.float16, torch.bfloat16], "Input tensors must be in dtype of torch.float16 or torch.bfloat16"
    assert q.device == k.device, "All tensors must be on the same device."
    assert q.dtype == k.dtype, "All tensors must have the same dtype."
    if tensor_layout not in ("NHD", "HND"):
        raise ValueError(f"Unknown tensor layout: {tensor_layout}")
    assert q.dim() == 4 and k.dim() == 4, "q and k must be 4-D"
    head_dim_og = q.size(-1)
    if head_dim_og > 128 or k.size(-1) != head_dim_og:
        raise ValueError(f"Unsupported head_dim: {head_dim_og} (q) / {k.size(-1)} (k); at most 128 and equal")
    assert q.stride(-1) == 1 and k.stride(-1) == 1, "Last dim of qkv must be contiguous."
    lay = 0 if tensor_layout == "NHD" else 1
    B, Hq, Sq, _ = ops._bhsd(q, lay)
    Bk, Hkv, Skv, _ = ops._bhsd(k, lay)
    if Bk != B or Hq % Hkv:
        raise ValueError(f"num_qo_heads ({Hq}) must be divisible by num_kv_heads ({Hkv}), and the batch sizes equal")
    if Skv > MAX_KV_LEN or Sq < 1 or Skv < 1:
        raise ValueError(f"predict_block_mask supports 1 <= kv_len <= {MAX_KV_LEN} and qo_len >= 1, got {Skv} / {Sq}")
    if is_causal:
        assert Sq == Skv, "qo_len and kv_len must be equal for causal attention."
    cdf_threshold, sim_threshold = float(cdf_threshold), float(sim_threshold)
    if not cdf_threshold > 0.0:
        raise ValueError(f"cdf_threshold must be > 0, got {cdf_threshold}")
    if math.isnan(sim_threshold):
        raise ValueError("sim_threshold must not be NaN")
    if sm_scale is None:
        sm_scale = head_dim_og ** -0.5
    if not math.isfinite(sm_scale):
        raise ValueError(f"sm_scale must be finite, got {sm_scale}")

    q, k = _pad8(q.detach()), _pad8(k.detach())
    D = q.size(-1)
    nq, nk = (Sq + 127) // 128, (Skv + 63) // 64
    f32 = dict(dtype=torch.float32, device=q.device)
    q_mean, q_sim = torch.empty((B, Hq, nq, D), **f32), torch.empty((B, Hq, nq), **f32)
    k_mean, k_sim = torch.empty((B, Hkv, nk, D), **f32), torch.empty((B, Hkv, nk), **f32)
    block_mask = torch.empty((B, Hq, nq, nk), dtype=torch.bool, device=q.device)
    ops.block_stats(q, q_mean, q_sim, lay, 128)
    ops.block_stats(k, k_mean, k_sim, lay, 64)
    ops.predict_block_mask(q_mean, q_sim, k_mean, k_sim, block_mask, Sq, Skv, 1 if is_causal else 0, sm_scale, cdf_threshold,
                           sim_threshold)
    return block_mask


def predict_block_mask_varlen(q: torch.Tensor, k: torch.Tensor, cu_seqlens_q: torch.Tensor, cu_seqlens_k: torch.Tensor,
                              max_seqlen_q: int, max_seqlen_k: int, *, cdf_threshold: float, sim_threshold: float,
                              is_causal: bool = False, sm_scale: Optional[float] = None) -> torch.Tensor:
    """predict_block_mask of every packed sequence on its own, in three launches whatever the number of sequences: the block mask
    that sageattn_varlen_blocksparse takes.  q [Tq,Hq,D], k [Tk,Hkv,D] packed as for sageattn_varlen_qk_int8_pv_fp8_cuda
    (cu_seqlens int32 or int64 on q's device, the same length; max_seqlen_* >= every length), max_seqlen_k <= 1048576.

    Returns a contiguous torch.bool [nseq, Hq, ceil(max_seqlen_q/128), ceil(max_seqlen_k/64)] tensor on q's device.  Contract: slice
    [b, :, :nq_b, :nk_b] (nq_b = ceil(Lq_b/128), nk_b = ceil(Lk_b/64)) is the bits of predict_block_mask(q_b[None], k_b[None],
    tensor_layout="NHD", <same options>)[0]: the statistics blocks restart at each sequence's first token, and each sequence sorts
    its candidates on its own power-of-two length, so its prefix masses are summed in the dense call's order.  Every entry outside
    the slices is False, and so is every entry of a sequence without queries or keys.  is_causal is top-left inside each sequence,
    with the rules of predict_block_mask, and allows Lq != Lk.  The lengths are read on the device (no host sync).  The inputs carry
    no gradient here.  Deterministic."""
    from .core import _check_cu_seqlens
    assert q.is_cuda, "Input tensors must be on cuda."
    assert q.dtype in [torch.float16, torch.bfloat16], "Input tensors must be in dtype of torch.float16 or torch.bfloat16"
    assert q.device == k.device, "All tensors must be on the same device."
    assert q.dtype == k.dtype, "All tensors must have the same dtype."
    _check_cu_seqlens(q, k, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k)
    head_dim_og = q.size(-1)
    if head_dim_og > 128 or k.size(-1) != head_dim_og:
        raise ValueError(f"Unsupported head_dim: {head_dim_og} (q) / {k.size(-1)} (k); at most 128 and equal")
    assert q.stride(-1) == 1 and k.stride(-1) == 1, "Last dim of qkv must be contiguous."
    Hq, Hkv = q.size(1), k.size(1)
    if Hq % Hkv:
        raise ValueError(f"num_qo_heads ({Hq}) must be divisible by num_kv_heads ({Hkv})")
    max_seqlen_q, max_seqlen_k = int(max_seqlen_q), int(max_seqlen_k)
    if max_seqlen_k > MAX_KV_LEN:
        raise ValueError(f"predict_block_mask_varlen supports max_seqlen_k <= {MAX_KV_LEN}, got {max_seqlen_k}")
    cdf_threshold, sim_threshold = float(cdf_threshold), float(sim_threshold)
    if not cdf_threshold > 0.0:
        raise ValueError(f"cdf_threshold must be > 0, got {cdf_threshold}")
    if math.isnan(sim_threshold):
        raise ValueError("sim_threshold must not be NaN")
    if sm_scale is None:
        sm_scale = head_dim_og ** -0.5
    if not math.isfinite(sm_scale):
        raise ValueError(f"sm_scale must be finite, got {sm_scale}")

    q, k = _pad8(q.detach()), _pad8(k.detach())
    cu_q, cu_k = cu_seqlens_q.to(torch.int32).contiguous(), cu_seqlens_k.to(torch.int32).contiguous()
    nseq, D = cu_q.numel() - 1, q.size(-1)
    nq, nk = (max_seqlen_q + 127) // 128, (max_seqlen_k + 63) // 64
    f32 = dict(dtype=torch.float32, device=q.device)
    q_mean, q_sim = torch.empty((nseq, Hq, nq, D), **f32), torch.empty((nseq, Hq, nq), **f32)
    k_mean, k_sim = torch.empty((nseq, Hkv, nk, D), **f32), torch.empty((nseq, Hkv, nk), **f32)
    block_mask = torch.empty((nseq, Hq, nq, nk), dtype=torch.bool, device=q.device)
    ops.block_stats_varlen(q, q_mean, q_sim, cu_q, max_seqlen_q, 128)
    ops.block_stats_varlen(k, k_mean, k_sim, cu_k, max_seqlen_k, 64)
    ops.predict_block_mask_varlen(q_mean, q_sim, k_mean, k_sim, block_mask, cu_q, cu_k, max_seqlen_q, max_seqlen_k,
                                  1 if is_causal else 0, sm_scale, cdf_threshold, sim_threshold)
    return block_mask
