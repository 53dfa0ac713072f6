"""CPU restatement of chunked prefill against the 8-bit paged KV cache (sageattn_kvcache8_prefill), in the kernel's order of
operations.

The numerics are those of the decode kernel restated by attn_kvcache8_oracle.attend with one chunk (chunk >= Lk, so the combine is
the identity): Q quantised per (token, head), logits in log2 units, an exact running max over 64-key tiles from key 0,
P = bf16(fp32(p * v_scale)), O / l.  What differs is the bound.  attend's terms for fp32 accumulation (2^-18 of sum |P| |v8|) and
normalisation (rho = 2^-15 + eta) are set for a row that folds at most one chunk of 1024 keys into its accumulators; a prefill row
folds every key it sees.  attend_folded scales those two terms with the number of fp32 accumulation steps of a row (derivation in
its docstring), and with acc_steps = 64 it is attend with one chunk, bit for bit (tested).

The quantisers, write and gather are attn_kvcache8_oracle's.
"""
import math

import torch

from attn_kvcache8_oracle import LOG2E, TILE, _bf16_midpoint_distance, quant_rows

DECODE_STEPS = 64        # 16-key accumulation steps of one 1024-key chunk: the row attend's bound is set for


def row_steps(Lk: int) -> int:
    """The fp32 accumulation steps a prefill row of a sequence with Lk keys takes: four 16-key MMA steps per 64-key tile, every
    tile up to the row's horizon.  Never below DECODE_STEPS, so the bound is never tighter than the decode restatement's."""
    return max(DECODE_STEPS, 4 * ((Lk + TILE - 1) // TILE))


def attend_folded(q: torch.Tensor, k8, ks, v8, vs, k_smooth, is_causal: bool, sm_scale: float, bound: bool = False,
                  out_dtype=torch.bfloat16, acc_steps=None):
    """One sequence whose rows fold all their keys into one set of accumulators.  Arguments and results as
    attn_kvcache8_oracle.attend without `chunk`; acc_steps defaults to row_steps(Lk).

    Bound: that of attend, with its accumulation and normalisation terms multiplied by f = acc_steps / 64.
      - Accumulation.  Each 16-key MMA step adds one product to fp32 accumulators whose magnitude never exceeds sum |P| |v8|
        (the rescale by alpha <= 1 only shrinks them), so a step adds at most one fp32 rounding of that sum, 2^-24 of it.  attend's
        2^-18 is 64 such steps, one 1024-key chunk; n steps are n 2^-24 = f 2^-18.
      - Normalisation.  Per 64-key tile (4 steps) a lane adds 16 values of p to its part of l and folds it with alpha: at most 17
        fp32 roundings, within 4 x 2^-21 of l.  attend's 2^-15 is 64 x 2^-21, one chunk; n steps are f 2^-15.
    eta (the error of each p), the bf16 rounding flips of P and the output's half ulp are per element and do not grow."""
    Lq, Hq, D = q.shape
    Lk, Hkv, _ = k8.shape
    f = (row_steps(Lk) if acc_steps is None else acc_steps) / DECODE_STEPS
    G = Hq // Hkv
    o = torch.zeros(Hq, Lq, D, dtype=torch.float64)
    lse = torch.full((Hq, Lq), -math.inf, dtype=torch.float64)
    ob = torch.zeros(Hq, Lq, D, dtype=torch.float64)
    lb = torch.zeros(Hq, Lq, dtype=torch.float64)
    if Lq == 0:
        return (o.transpose(0, 1), lse, ob.transpose(0, 1), lb) if bound else (o.transpose(0, 1), lse)
    q8, qs = quant_rows(q.float(), 127.0, fp8=False)
    qh = q8.double().transpose(0, 1)                                          # [Hq, Lq, D]
    c = qs.double().transpose(0, 1) * (sm_scale * LOG2E)                      # [Hq, Lq]
    kh = k8.double().repeat_interleave(G, 1).transpose(0, 1)                  # [Hq, Lk, D]
    vh = v8.double().repeat_interleave(G, 1).transpose(0, 1)
    ksh = ks.double().repeat_interleave(G, 1).transpose(0, 1)                 # [Hq, Lk]
    vsh = vs.double().repeat_interleave(G, 1).transpose(0, 1)
    rows = torch.arange(Lq)[:, None]
    last = (rows + Lk - Lq) if is_causal else torch.full((Lq, 1), Lk - 1)     # the last key row i sees
    m = torch.full((Hq, Lq), -math.inf, dtype=torch.float64)
    l = torch.zeros(Hq, Lq, dtype=torch.float64)
    O = torch.zeros(Hq, Lq, D, dtype=torch.float64)
    F = torch.zeros(Hq, Lq, D, dtype=torch.float64)
    A = torch.zeros(Hq, Lq, D, dtype=torch.float64)
    eta_max = torch.zeros(Hq, Lq, dtype=torch.float64)
    for t0 in range(0, Lk, TILE):
        t1 = min(Lk, t0 + TILE)
        vis = torch.arange(t0, t1)[None, :] <= last                           # [Lq, n]
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
    if Lk > 0:
        # attend's combine of one chunk, in its order of operations (the weight is 1, or 0 for a row that saw nothing)
        M = m
        w = torch.where(torch.isinf(m), torch.zeros_like(m), torch.exp2(m - M))
        L = torch.zeros_like(M) + w * l
        acc = torch.zeros(Hq, Lq, D, dtype=torch.float64) + w[..., None] * O
        accb = torch.zeros(Hq, Lq, D, dtype=torch.float64) + w[..., None] * (F + 2.0 ** -18 * f * A)
        eta_all = torch.maximum(torch.zeros_like(M), eta_max)
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
