"""CPU restatement of the sliding-window forward (sab_qk_int8_sv_f8_attn_window, csrc/attn.cu).  TEST INFRASTRUCTURE ONLY:
imported by tests/test_window_cpu.py and tests/test_gpu_window.py, never by the product package.

Key j is visible to query i iff i - left <= j <= i + right (-1: that side unbounded), j < Skv, and j <= i when causal.  The
kernel's CTA for 128-row Q block i runs the loop of the dense restatement (oracle.sage_oracle.attn_int8_fp8_cuda) over the
64-key tiles [j_lo, j_hi) that meet its rows' windows (window_tiles), with the elements outside the window masked.  The per-tile
arithmetic is that restatement's with the kernel's lazy running max, except where a row part sees nothing of a tile: the kernel
then keeps m and d and adds P = 0 (the dense restatement, whose rows always see a key of every tile they reach, would give
P = exp2(0) there).  A row with no visible key gives 0 and lse -inf."""
import torch

from oracle import sage_oracle as O


def window_mask(Sq, Sk, left, right, is_causal=False, device=None):
    """bool [Sq, Sk]: key j visible to query i."""
    i = torch.arange(Sq, device=device)[:, None]
    j = torch.arange(Sk, device=device)[None, :]
    m = torch.ones(Sq, Sk, dtype=torch.bool, device=device)
    if left >= 0:
        m &= j >= i - left
    if right >= 0:
        m &= j <= i + right
    if is_causal:
        m &= j <= i
    return m


def window_tiles(r_lo, r_hi, Sk, left, right, is_causal=False):
    """The 64-key tiles [j_lo, j_hi) holding a key visible to some row of [r_lo, r_hi] (inclusive): csrc/attn_common.cuh."""
    k_lo = 0 if left < 0 else max(0, r_lo - left)
    k_hi = Sk - 1
    if right >= 0:
        k_hi = min(k_hi, r_hi + right)
    if is_causal:
        k_hi = min(k_hi, r_hi)
    return k_lo // 64, (k_hi // 64 + 1 if k_hi >= k_lo else k_lo // 64)


def attn_int8_fp8_window(q8, k8, v8, q_scale, k_scale, v_scale, *, window, qk_quant_gran="per_thread", is_causal=False,
                         sm_scale=1.0, lazy_tau=4, out_dtype=torch.float16, return_lse=False, v_mean=None):
    """The window form of attn_int8_fp8_cuda with fp32 PV accumulation (the kernel's), on [B,H,S,D] tensors; v8 is the LOGICAL
    [B,Hkv,Sk,D] fp8 tensor.  lazy_tau: the kernel's lazy running max (0: the exact max of SAB_ATTN_KERNEL=exact)."""
    left, right = window
    B, Hq, Sq, D = q8.shape
    _, Hk, Sk, _ = k8.shape
    g = Hq // Hk
    tau = float(lazy_tau)
    qs_row = O._expand_q_scale(q_scale, qk_quant_gran, Sq)[:, :, :Sq]
    ks_key = O._expand_k_scale(k_scale, qk_quant_gran, Sk)[:, :, :Sk].repeat_interleave(g, dim=1)
    kf = k8.float().repeat_interleave(g, dim=1)
    vf = v8.float().repeat_interleave(g, dim=1)
    vsc = v_scale.repeat_interleave(g, dim=1)
    sm2 = torch.tensor(sm_scale, dtype=torch.float32) * torch.tensor(O.LOG2E_CU, dtype=torch.float32)
    em_all = window_mask(Sq, Sk, left, right, is_causal)
    out = torch.zeros((B, Hq, Sq, D), dtype=out_dtype)
    lse = torch.full((B, Hq, Sq), -float("inf"), dtype=torch.float32)
    for r0 in range(0, Sq, 128):
        r1 = min(r0 + 128, Sq)
        j_lo, j_hi = window_tiles(r0, r1 - 1, Sk, left, right, is_causal)
        qf = q8[:, :, r0:r1].float()
        m = torch.full((B, Hq, r1 - r0), O.MASK_VALUE, dtype=torch.float32)
        d = torch.zeros((B, Hq, r1 - r0), dtype=torch.float32)
        acc = torch.zeros((B, Hq, r1 - r0, D), dtype=torch.float32)
        for j in range(j_lo, j_hi):
            s0, s1 = 64 * j, min(64 * j + 64, Sk)
            em = em_all[r0:r1, s0:s1]
            S = (qf @ kf[:, :, s0:s1].transpose(-1, -2)) * ((sm2 * qs_row[:, :, r0:r1])[..., None] * ks_key[:, :, None, s0:s1])
            mx = torch.where(em, S, torch.tensor(-float("inf"))).amax(dim=-1)
            mx = torch.where(em.any(-1), mx, torch.tensor(O.MASK_VALUE))
            m_true = torch.maximum(m, mx - (O.S_FP8_OFFSET - tau))
            m_new = torch.where(m_true - m > tau, m_true, m)
            alpha = torch.exp2(m - m_new)
            P = torch.where(em, torch.exp2(S - m_new[..., None]), torch.tensor(0.0))
            d = d * alpha + P.sum(dim=-1)
            acc = acc * alpha[..., None] + P.to(torch.float8_e4m3fn).float() @ vf[:, :, s0:s1]
            m = m_new
        o = (acc / d[..., None]) * vsc[:, :, None, :]
        if v_mean is not None:
            o = o + v_mean.float().repeat_interleave(g, dim=1)[:, :, None, :]
        seen = (d > 0)[..., None]
        out[:, :, r0:r1] = torch.where(seen, o, torch.tensor(0.0)).to(out_dtype)
        lse[:, :, r0:r1] = torch.log2(d) + m
    return (out, lse) if return_lse else out
