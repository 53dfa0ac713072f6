"""CPU restatement of the 8-bit paged KV cache (sageattention_b200/kvcache8.py), in the kernels' order of operations.

  quant_rows     per-row INT8 / e4m3 quantisation in fp32, bit for bit: scale = amax / qmax, x * RN(qmax / amax) (the IEEE quotient
                 x / scale when that overflows), round-to-nearest-even with saturation; an all-zero row gives scale 0 and zeros.
  write          what PagedKVCache8.write stores for tokens k, v: (k8, k_scale, v8 as e4m3 values in fp32, v_scale).
  attend         one sequence against its gathered 8-bit keys: Q quantised per (token, head), logits in log2 units, fixed chunks of
                 `chunk` keys, an exact running max over 64-key tiles, P = bf16(fp32(p * v_scale)), and the chunk combine.  Works in
                 fp64 except the bf16 rounding of P.  With bound=True it also returns a per-element bound on |kernel - restatement|.

The bound (attend's docstring) only allows for what the kernels do differently by design: ex2.approx and fp32 evaluation of the
logits and exponentials, fp32 sums in another order, and the rounding of the output.
"""
import math

import numpy as np
import torch

LOG2E = 1.4426950408889634
TILE = 64


def quant_rows(x: torch.Tensor, qmax: float, fp8: bool):
    """x fp32 [..., D] -> (q fp32 [..., D] holding the int8 / e4m3 values, scale fp32 [...])."""
    x = x.float()
    amax = x.abs().amax(-1)
    qm = torch.tensor(qmax, dtype=torch.float32)
    pos = amax > 0
    scale = torch.where(pos, amax / qm, torch.zeros_like(amax))
    mult = torch.where(pos, qm / amax, torch.zeros_like(amax))
    exact = torch.isinf(mult)
    y = torch.where(exact[..., None], x / scale[..., None], x * mult[..., None])   # fp32, IEEE round-to-nearest
    y = torch.nan_to_num(y, nan=0.0)
    if fp8:
        q = y.clamp(-448.0, 448.0).to(torch.float8_e4m3fn).float()
    else:
        q = torch.round(y).clamp(-128.0, 127.0)
    q = torch.where(pos[..., None], q, torch.zeros_like(q))
    return q, scale


def write(k: torch.Tensor, v: torch.Tensor, k_smooth: torch.Tensor):
    """Tokens k, v [T, Hkv, D] (16-bit), k_smooth fp32 [Hkv, D] -> (k8, k_scale, v8, v_scale)."""
    k8, ks = quant_rows(k.float() - k_smooth.float(), 127.0, fp8=False)
    v8, vs = quant_rows(v.float(), 448.0, fp8=True)
    return k8, ks, v8, vs


def _bf16_midpoint_distance(x: torch.Tensor):
    """(ulp of bf16(x), |x - nearest bf16 rounding boundary|) for fp64 x > 0 (0 where x == 0)."""
    ax = x.abs()
    _, e = torch.frexp(ax)                       # ax = f * 2^e, f in [0.5, 1)
    ulp = torch.ldexp(torch.ones_like(ax), (e - 8).to(torch.int32))
    u = ax / ulp
    dist = (u - (torch.floor(u) + 0.5)).abs() * ulp
    return torch.where(ax > 0, ulp, torch.zeros_like(ax)), torch.where(ax > 0, dist, torch.full_like(ax, math.inf))


def attend(q: torch.Tensor, k8, ks, v8, vs, k_smooth, is_causal: bool, sm_scale: float, chunk: int, bound: bool = False,
           out_dtype=torch.bfloat16):
    """One sequence.  q [Lq, Hq, D] 16-bit; k8 / v8 [Lk, Hkv, D] and ks / vs [Lk, Hkv] from `write`; k_smooth [Hkv, D].
    Returns (o [Lq, Hq, D] fp64, lse [Hq, Lq] fp64 natural log) and, with bound=True, (o_bound [Lq, Hq, D], lse_bound [Hq, Lq]).

    Bound: the kernel evaluates s = float(dot) * c * k_scale in fp32 and p = ex2.approx(s - m), so each p carries a relative error
    eta <= 2^-20 (|s| + |m| + 1) (three fp32 roundings of s and m, 2^-22 of ex2.approx, the fp32 product p * v_scale).  Where
    p * v_scale lies within eta of a bf16 rounding boundary, the kernel's P may be the neighbouring bf16 value: that element adds
    ulp(P) |v8| to the bound.  The rest is continuous: 2^-18 of sum |P| |v8| for fp32 accumulation in the tensor cores' order,
    a relative rho = 2^-15 + max eta on the normalisation (the sums of p and the chunk weights), and half an ulp of the output type."""
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
    rows = torch.arange(Lq)[:, None]
    last = (rows + Lk - Lq) if is_causal else torch.full((Lq, 1), Lk - 1)     # the last key row i sees
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
            keys = torch.arange(t0, t1)
            vis = keys[None, :] <= last                                       # [Lq, n]
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
            accb = accb + w[..., None] * (F + 2.0 ** -18 * A)
            eta_all = torch.maximum(eta_all, eta_max)
        seen = ~torch.isinf(M)
        Ls = torch.where(seen, L, torch.ones_like(L))
        o = torch.where(seen[..., None], acc / Ls[..., None], torch.zeros_like(acc))
        qk = torch.einsum("thd,hd->ht", q.double(), k_smooth.double().repeat_interleave(G, 0))
        lse = torch.where(seen, (M + torch.log2(Ls)) / LOG2E + qk * sm_scale, lse)
        if bound:
            rho = 2.0 ** -15 + eta_all
            half_ulp = 2.0 ** -8 if out_dtype == torch.bfloat16 else 2.0 ** -11
            ob = torch.where(seen[..., None], accb / Ls[..., None] + (rho[..., None] + half_ulp) * o.abs() + 2.0 ** -24,
                             torch.zeros_like(o))
            qk_abs = torch.einsum("thd,hd->ht", q.double().abs(), k_smooth.double().abs().repeat_interleave(G, 0))
            lb = torch.where(seen, (2.0 ** -20 * (M.abs() + 1.0) + 2.0 * rho) / LOG2E + 2.0 ** -22 * lse.abs() +
                             D * 2.0 ** -23 * qk_abs * sm_scale, torch.zeros_like(M))
    if bound:
        return o.transpose(0, 1), lse, ob.transpose(0, 1), lb
    return o.transpose(0, 1), lse


def gather(pages: torch.Tensor, table_row: torch.Tensor, n: int):
    """The first n tokens of one sequence from [num_pages, page_size, ...] pages through its block-table row."""
    page_size = pages.size(1)
    t = torch.arange(n)
    return pages[table_row[t // page_size].long(), t % page_size]


def bytes_read(lens_k, Hkv: int, D: int) -> int:
    """Cache bytes the attention kernel reads: 8-bit K and V plus two fp32 scales per (key, KV head)."""
    return sum(lens_k) * Hkv * (2 * D + 8)
