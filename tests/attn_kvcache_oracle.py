"""CPU restatement of sageattn_varlen_kvcache (attention of packed queries against a paged KV cache): a page gather, then the
existing CPU restatement of the INT8+FP8 call on each sequence (oracle/sage_oracle.py) with the causal mask aligned bottom-right.

Query i of sequence b sees key j iff j <= i + Lk_b - Lq_b when causal; the offset Lk_b - Lq_b may be negative, and then the
first Lq_b - Lk_b rows see no key and give 0 and lse -inf.  Each sequence runs through attn_window_oracle.attn_int8_fp8_tiles, the
kernel's CTA loop (lazy running max, fp32 PV accumulation) with the tiles the kernel visits, and optionally its error bound."""
import torch

from attn_window_oracle import attn_int8_fp8_tiles
from oracle import sage_oracle as O


def gather_pages(cache, block_table, seqused_k):
    """[sum Lk_b, H, D]: the first Lk_b tokens of each sequence, gathered from its pages and packed in sequence order."""
    page_size = cache.size(1)
    parts = []
    for b, n in enumerate(seqused_k.tolist()):
        t = torch.arange(n, device=block_table.device)
        parts.append(cache[block_table[b, t // page_size].long(), t % page_size])
    return torch.cat(parts) if parts else cache.new_empty((0,) + tuple(cache.shape[2:]))


def visible(Lq, Lk, is_causal):
    """[Lq, Lk] bool: the keys each query sees."""
    if not is_causal:
        return torch.ones(Lq, Lk, dtype=torch.bool)
    return torch.arange(Lk)[None, :] <= torch.arange(Lq)[:, None] + (Lk - Lq)


def bottom_right_tiles(Lq, Lk, is_causal):
    """The 64-key tiles each 128-row Q block visits (csrc/attn.cu, the window form with (-1, Lk - Lq)): up to the last key its
    bottom row sees, none when that row sees no key; every tile when not causal."""
    out = []
    for r0 in range(0, Lq, 128):
        k_hi = Lk - 1 if not is_causal else min(Lk - 1, min(r0 + 128, Lq) - 1 + Lk - Lq)
        out.append(range(0, k_hi // 64 + 1) if k_hi >= 0 else range(0))
    return out


def attn_sequence(q, k, v, is_causal=False, qk_quant_gran="per_thread", sm_scale=None, pv_accum_dtype="fp32+fp16", smooth_k=True,
                  smooth_v=False, lazy_tau=4, bound=False, operands=None):
    """One sequence: q [Lq,Hq,D], k / v [Lk,Hkv,D] -> (o [Lq,Hq,D] in q's dtype, lse [Hq,Lq] in natural-log units with the K-mean
    correction of sageattn_qk_int8_pv_fp8_cuda), and with bound=True also the Bound of attn_window_oracle.attn_int8_fp8_tiles
    ([1,Hq,Lq,...], on the raw log2 lse).  operands: (q8, k8, v8, qs, ks, vs, vm), HND with the logical [1,Hkv,Lk,D] v8, in
    place of the restated quantisers (a GPU test passes the library's, to check the attention kernel alone)."""
    Lq, Hq, D = q.shape
    Lk = k.size(0)
    if Lk == 0:
        o, lse = torch.zeros_like(q), torch.full((Hq, Lq), float("-inf"))
        return (o, lse, None) if bound else (o, lse)
    sm_scale = D ** -0.5 if sm_scale is None else sm_scale
    if pv_accum_dtype in ("fp32+fp32", "fp32+fp16"):
        smooth_v = False
    qh, kh, vh = (t.transpose(0, 1)[None] for t in (q, k, v))           # [1,H,L,D]
    km = kh.mean(dim=2, keepdim=True) if smooth_k else None
    if qk_quant_gran == "per_warp":
        q8, qs, k8, ks = O.per_warp_int8_cuda(qh, kh, km)
    else:
        q8, qs, k8, ks = O.quant_per_thread_int8_triton(qh, kh, km)
    v8, vs, vm = O.per_channel_fp8_cuda(vh, "HND", 2.25 if pv_accum_dtype == "fp32+fp16" else 448.0, smooth_v=smooth_v)
    if operands is not None:
        q8, k8, v8, qs, ks, vs, vm = operands
    ranges = bottom_right_tiles(Lq, Lk, is_causal)
    res = attn_int8_fp8_tiles(q8, k8, v8, qs, ks, vs, lambda b, h, i: ranges[i], visible(Lq, Lk, is_causal),
                              qk_quant_gran=qk_quant_gran, sm_scale=sm_scale, lazy_tau=lazy_tau, out_dtype=q.dtype, return_lse=True,
                              v_mean=vm, bound=bound)
    o, lse = res[0], res[1]
    lse = lse[0] / O.LOG2E_PY
    if smooth_k:
        g = Hq // kh.size(1)
        lse = lse + (qh[0] @ km[0].repeat_interleave(g, dim=0).transpose(1, 2)).squeeze(-1).float() * sm_scale
    o = o[0].transpose(0, 1)
    return (o, lse, res[2]) if bound else (o, lse)


def sageattn_varlen_kvcache(q, k_cache, v_cache, cu_seqlens_q, seqused_k, block_table, is_causal=False, **kw):
    """The whole call on CPU tensors: (o [Tq,Hq,D], lse [Hq,Tq]).  Rows past cu_seqlens_q[-1] are 0 and lse -inf here (the
    kernels leave them unwritten)."""
    o = torch.zeros_like(q)
    lse = torch.full((q.size(1), q.size(0)), float("-inf"))
    cu = cu_seqlens_q.tolist()
    cu_k = [0] + torch.cumsum(seqused_k, 0).tolist()
    k, v = gather_pages(k_cache, block_table, seqused_k), gather_pages(v_cache, block_table, seqused_k)
    for b in range(len(cu) - 1):
        s, e = cu[b], cu[b + 1]
        if e == s:
            continue
        o[s:e], lse[:, s:e] = attn_sequence(q[s:e], k[cu_k[b]:cu_k[b + 1]], v[cu_k[b]:cu_k[b + 1]], is_causal, **kw)
    return o, lse
