"""CPU restatement of sliding-window attention on the 8-bit paged KV cache (window_size on sageattn_kvcache8 and
sageattn_kvcache8_prefill), in the kernels' order of operations.

  visible_keys   the keys each row sees: bottom-right, first <= j <= last.
  attend         the decode restatement (attn_kvcache8_oracle.attend) with a window: fixed chunks of `chunk` keys, an exact running
                 max over 64-key tiles from key 0, P = bf16(fp32(p * v_scale)), the chunk combine, and attend's bound.
  attend_folded  the prefill restatement (attn_kvcache8_prefill_oracle.attend_folded) with a window: one chunk, and the bound's
                 accumulation and normalisation terms scaled by row_steps(Lk) / 64 as there.

Both fold every tile, as the restatements without a window do; the kernels skip the tiles left of the window, and a tile in which
a row sees nothing leaves its m, l and O exactly as they were, so skipping it changes nothing.  A windowed row folds no more
accumulation steps than without a window, so row_steps(Lk) still bounds the prefill row.  With window (-1, -1), or any window that
hides no key, both give the results and bounds of the restatements without a window bit for bit (tested).
The quantisers and write are attn_kvcache8_oracle's.
"""
import math

import torch

from attn_kvcache8_oracle import LOG2E, TILE, _bf16_midpoint_distance, quant_rows
from attn_kvcache8_prefill_oracle import DECODE_STEPS, row_steps


def visible_keys(Lq: int, Lk: int, is_causal: bool, window=(-1, -1)):
    """(first, last) [Lq, 1]: row i sees keys first <= j <= last with 0 <= j < Lk.  With off = Lk - Lq: last = i + off when causal,
    else Lk - 1; a window (left, right) also bounds i + off - left <= j <= i + off + right, -1 leaving a side unbounded."""
    rows = torch.arange(Lq)[:, None]
    last = (rows + Lk - Lq) if is_causal else torch.full((Lq, 1), Lk - 1)
    left, right = window
    if right >= 0:
        last = torch.minimum(last, rows + Lk - Lq + right)
    first = rows + Lk - Lq - left if left >= 0 else torch.zeros((Lq, 1), dtype=torch.long)
    return first, last


def _attend(q, k8, ks, v8, vs, k_smooth, is_causal, sm_scale, chunk, window, bound, out_dtype, f):
    """attend's computation with a window; f scales the accumulation (2^-18) and normalisation (2^-15) bound terms."""
    Lq, Hq, D = q.shape
    Lk, Hkv, _ = k8.shape
    G = Hq // Hkv
    o = torch.zeros(Hq, Lq, D, dtype=torch.float64)
    lse = torch.full((Hq, Lq), -math.inf, dtype=torch.float64)
    ob = torch.zeros(Hq, Lq, D, dtype=torch.float64)
    lb = torch.zeros(Hq, Lq, dtype=torch.float64)
    if Lq == 0:
        return (o.transpose(0, 1), lse, ob.transpose(0, 1), lb) if bound else (o.transpose(0, 1), lse)
    q8, qs = quant_rows(q.float(), 127.0, fp8=False)                          # [Lq, Hq, D], [Lq, Hq]
    qh = q8.double().transpose(0, 1)                                          # [Hq, Lq, D]
    c = qs.double().transpose(0, 1) * (sm_scale * LOG2E)                      # [Hq, Lq]
    kh = k8.double().repeat_interleave(G, 1).transpose(0, 1)                  # [Hq, Lk, D]
    vh = v8.double().repeat_interleave(G, 1).transpose(0, 1)
    ksh = ks.double().repeat_interleave(G, 1).transpose(0, 1)                 # [Hq, Lk]
    vsh = vs.double().repeat_interleave(G, 1).transpose(0, 1)
    first, last = visible_keys(Lq, Lk, is_causal, window)
    parts = []                                                                # per chunk: (m, l, O, flips, |P||V|, eta_max)
    for c0 in range(0, Lk, chunk):
        c1 = min(Lk, c0 + chunk)
        m = torch.full((Hq, Lq), -math.inf, dtype=torch.float64)
        l = torch.zeros(Hq, Lq, dtype=torch.float64)
        O = torch.zeros(Hq, Lq, D, dtype=torch.float64)
        F = torch.zeros(Hq, Lq, D, dtype=torch.float64)
        A = torch.zeros(Hq, Lq, D, dtype=torch.float64)
        eta_max = torch.zeros(Hq, Lq, dtype=torch.float64)
        for t0 in range(c0, c1, TILE):
            t1 = min(c1, t0 + TILE)
            keys = torch.arange(t0, t1)[None, :]
            vis = (keys <= last) & (keys >= first)                            # [Lq, n]
            s = (qh @ kh[:, t0:t1].transpose(1, 2)) * c[..., None] * ksh[:, None, t0:t1]
            s = s.masked_fill(~vis, -math.inf)
            m_new = torch.maximum(m, s.amax(-1))
            alpha = torch.where(torch.isinf(m), torch.zeros_like(m), torch.exp2(m - m_new))
            p = torch.where(torch.isinf(s), torch.zeros_like(s), torch.exp2(s - m_new[..., None]))
            x = p * vsh[:, None, t0:t1]
            P = x.float().bfloat16().double()
            l = alpha * l + p.sum(-1)
            O = alpha[..., None] * O + P @ vh[:, t0:t1]
            if bound:
                eta = 2.0 ** -20 * (s.abs().nan_to_num(0.0, posinf=0.0) + m_new.abs().nan_to_num(0.0, posinf=0.0)[..., None] + 1.0)
                ulp, dist = _bf16_midpoint_distance(x)
                flip = torch.where((dist <= eta * x.abs()) & (x > 0), ulp, torch.zeros_like(ulp))
                F = alpha[..., None] * F + flip @ vh[:, t0:t1].abs()
                A = alpha[..., None] * A + P.abs() @ vh[:, t0:t1].abs()
                eta_max = torch.maximum(eta_max, torch.where(vis.expand_as(eta), eta, torch.zeros_like(eta)).amax(-1))
            m = m_new
        parts.append((m, l, O, F, A, eta_max))
    if parts:
        M = torch.stack([pt[0] for pt in parts]).amax(0)
        L = torch.zeros_like(M)
        acc = torch.zeros(Hq, Lq, D, dtype=torch.float64)
        accb = torch.zeros(Hq, Lq, D, dtype=torch.float64)
        eta_all = torch.zeros_like(M)
        for m, l, O, F, A, eta_max in parts:
            w = torch.where(torch.isinf(m), torch.zeros_like(m), torch.exp2(m - M))
            L = L + w * l
            acc = acc + w[..., None] * O
            accb = accb + w[..., None] * (F + 2.0 ** -18 * f * A)
            eta_all = torch.maximum(eta_all, eta_max)
        seen = ~torch.isinf(M)
        Ls = torch.where(seen, L, torch.ones_like(L))
        o = torch.where(seen[..., None], acc / Ls[..., None], torch.zeros_like(acc))
        qk = torch.einsum("thd,hd->ht", q.double(), k_smooth.double().repeat_interleave(G, 0))
        lse = torch.where(seen, (M + torch.log2(Ls)) / LOG2E + qk * sm_scale, lse)
        if bound:
            rho = 2.0 ** -15 * f + eta_all
            half_ulp = 2.0 ** -8 if out_dtype == torch.bfloat16 else 2.0 ** -11
            ob = torch.where(seen[..., None], accb / Ls[..., None] + (rho[..., None] + half_ulp) * o.abs() + 2.0 ** -24,
                             torch.zeros_like(o))
            qk_abs = torch.einsum("thd,hd->ht", q.double().abs(), k_smooth.double().abs().repeat_interleave(G, 0))
            lb = torch.where(seen, (2.0 ** -20 * (M.abs() + 1.0) + 2.0 * rho) / LOG2E + 2.0 ** -22 * lse.abs() +
                             D * 2.0 ** -23 * qk_abs * sm_scale, torch.zeros_like(M))
    if bound:
        return o.transpose(0, 1), lse, ob.transpose(0, 1), lb
    return o.transpose(0, 1), lse


def attend(q: torch.Tensor, k8, ks, v8, vs, k_smooth, is_causal: bool, sm_scale: float, chunk: int, bound: bool = False,
           out_dtype=torch.bfloat16, *, window=(-1, -1)):
    """sageattn_kvcache8 with window_size=window on one sequence.  Arguments, results and bound as attn_kvcache8_oracle.attend."""
    return _attend(q, k8, ks, v8, vs, k_smooth, is_causal, sm_scale, chunk, window, bound, out_dtype, 1.0)


def attend_folded(q: torch.Tensor, k8, ks, v8, vs, k_smooth, is_causal: bool, sm_scale: float, bound: bool = False,
                  out_dtype=torch.bfloat16, acc_steps=None, *, window=(-1, -1)):
    """sageattn_kvcache8_prefill with window_size=window on one sequence.  Arguments, results and bound as
    attn_kvcache8_prefill_oracle.attend_folded: one chunk, the bound's accumulation and normalisation terms scaled by
    acc_steps / 64 (default row_steps(Lk))."""
    Lk = k8.size(0)
    f = (row_steps(Lk) if acc_steps is None else acc_steps) / DECODE_STEPS
    return _attend(q, k8, ks, v8, vs, k_smooth, is_causal, sm_scale, max(Lk, 1), window, bound, out_dtype, f)
