"""Restatement of the FP16-PV forward (sage_attn_fwd_kernel with kPV16, csrc/attn.cu), with an elementwise bound on
|kernel - restatement|.  TEST INFRASTRUCTURE ONLY: imported by the FP16-PV tests, never by the product package.

The FP16-PV kernel serves sageattn_qk_int8_pv_fp16_cuda (per-warp / per-thread INT8), sageattn_qk_int8_pv_fp16_triton (per-block
INT8 with sm_scale*log2e folded into the Q scale, and attn_mask in its bool and bias forms) and the packed sageattn_varlen.  One
loop, attn_fp16pv, restates the CTA on [B,H,S,D] tensors; attn_fp16pv_varlen runs it per sequence of a packed [T,H,D] batch.  It
evaluates in fp64 on the device of its inputs, with the kernel's fp32 roundings spelled out where they decide a value (the
logits, the running max, alpha), so full-size cases run on the GPU; q_offset / q_rows evaluate some rows of a call only.

Per 64-key tile j, for each row (log2 units; "fp32(.)" is one fp32 rounding):
  * coef = fp32(k_scale * fp32(q_scale * sm2)), sm2 = fp32(fp32(sm_scale) * log2e), or 1 when folded (fold_sm_scale);
  * visible keys: key < Skv, key <= row when causal (top-left), the bool mask true.  Without a bias the logit is
    S = fp32(float(s) * coef) and the kernel's P argument is x = fmaf(float(s), coef, -m_new); with a bias (mask_kind 2, the mask's
    16-bit values) the logit is y = fmaf(float(s), coef, bias) and x = fp32(y - m_new);
  * m_new = max(m, max over the visible logits), m starting at kMaskValue = -5e6, never -inf: a bool-masked element never enters
    the max (the kernel replaces its integer logit with a sentinel) and gets P = 0 exactly;
  * alpha = exp2(fp32(m - m_new)) (1 when m does not move), P = exp2(x), P16 = fp16(P), d = d * alpha + sum P (un-rounded P);
  * O = O * alpha (a rounding of its own, rescale_o), then O += P16 V16 in the tensor core, V16 = v.to(float16) as
    transpose_v_f16 writes it (a bf16 V becomes fp16 there: values beyond 65504 become inf, values below 2^-24 become fp16
    subnormals or 0, as torch's own conversion does);
  * epilogue: O * rcp(d), then the output dtype; lse = log2(d) + m.
Where the kernel differs from the reference's Triton kernel (oracle.sage_oracle.attn_int8_fp16_triton), this follows the kernel:
  * a row with no visible key gives 0 and lse -inf (the Triton kernel's l starts at 1, and its bool mask is an additive -1e6, so
    a fully masked row averages its keys there);
  * since m starts at -5e6, a row whose every key has a bias below -5e6 (finfo(bf16).min = -3.4e38, or -inf) has P = 0 on every
    key, d = 0, and is treated as fully masked: it returns 0 and lse -inf, where torch SDPA would average over its keys.  A fp16
    finfo.min (-65504) is above -5e6, so such a row attends over its keys as SDPA does;
  * the bias is added by one fmaf in log2 units, not after a separate fp32 product; the per-tile PV is not rounded to fp16 (the
    Triton kernel's dot(..., out_dtype=f16)), it accumulates in place in fp32.

Bound (bound=True), per output element before the output's 16-bit rounding (check_forward in attn_window_oracle adds that
rounding).  Constants of attn_bwd_oracle / attn_window_oracle: U32 = 2^-23, EPS_EXP = 2^-21.
  * ex2 and the logit: the kernel's P is ex2.approx of the same fp32 argument up to the roundings of the logit, so the two P
    differ by at most eps_P P, eps_P = EPS_EXP (1 + |S| + |m|) (S the log2 logit, with the bias when there is one); the same
    relative error, with |m - m_new|, holds for alpha.  The max is a plain running max, so an m one ulp off would only perturb every
    P of the row by that same relative amount: m need not match the kernel bit for bit, and the eps_P term covers it.
    ex2.approx.ftz flushes a P below 2^-126 to 0: TINY32 = 2^-126 per visible element on d (such a P has P16 = 0 on both sides).
  * fp16 rounding of P: fp16 is monotone, so the kernel's P16 lies between fp16(P (1 - eps_P)) and fp16(P (1 + eps_P)).  Where they
    differ the element is ambiguous (P lies within eps_P P of a rounding midpoint, which covers subnormal P below 2^-14 with its
    absolute step of 2^-24 as well): it adds (hi16 - lo16) |v16| to the row's bound.  Elsewhere both sides have the same P16.
  * fp16 wgmma with O carried in as the accumulator: four k16 steps per tile.  Model of a step: its addends (16 exact products
    P16 v16 and O) are aligned to the exponent E of the largest magnitude M among them and cut to U_TC16 2^E <= U_TC16 M each, and
    the sum is rounded to fp32: at most 18 U_TC16 M per step.  The kernel's O before and after the step lies within the bound B_O
    accumulated so far of the restatement's (which takes the step's ambiguous P first), and its products are at most
    max_j hi16_j * max_j |v16_j|, so M <= max(max(|O_before|, |O_after|) + B_O, max hi16 max |v16|) per element.  (A running sum of
    magnitudes would also bound M, but at 32K keys it is some 100 times |O|, and the bound would then miss one wrong tile.)
    U_TC16 = 2^-23, an fp32-wide accumulator, is the first guess; nobody had measured the H100's fp16 wgmma accumulation in this
    project, and the FP8 model's first guess was exceeded by 1.22 times (attn_window_oracle).  The GPU runs of
    tests/test_gpu_fp16pv_forward_edges.py keep it (that file's docstring has the measured ratios); the planted mistakes of
    test_fp16pv_oracle_cpu.py, at 333 keys and at 16K / 32K keys, fail this bound by the margins that file prints.
  * rescale: O * alpha rounds once (U32) and carries alpha's relative error, both of |O| + B_O, the kernel's O at most; d * alpha
    likewise.
  * d: eps_P P per element, its summation at most 82 U32 of the tile's sum (16 terms per thread, two shuffle adds, on either side),
    2 U32 of d per tile (d * alpha + sum), and TINY32 per visible element.
  * epilogue: x = O rcp(d): |e_x| <= B_O / d + |x| B_d / d + 3 U32 |x| (rcp.approx within one ulp and the product).
  * lse = log2(d) + m: (B_d / d) / ln2 + 2^-21 (1 + |log2 d|) + 2^-22 |lse|.
A row that sees no key (d = 0) has bound 0: it must be exactly 0 with lse -inf."""
import collections
import math

import torch

from attn_bwd_oracle import EPS_EXP, U32
from oracle import sage_oracle as O

U_TC16 = 2.0 ** -23    # fp16 wgmma accumulation, per k16 step (see the module docstring)
TINY32 = 2.0 ** -126   # ex2.approx.ftz: a P below this is 0 in the kernel
F16 = torch.float16
BN = 64

Bound = collections.namedtuple("Bound", "o o_bound lse_bound ambiguous visible rows moved mag")
Bound.__doc__ = """o: the restatement's output before its 16-bit rounding (fp64); o_bound / lse_bound: the bounds of the module
docstring; ambiguous / visible: counts of ambiguous and of visible elements with P > 0; rows: rows that see a key; moved: rows whose
running max moves after their first tile with P > 0; mag: sum |P16| |v16| through the alphas over d (the size of the output's
terms)."""


def _r32(x):
    """One fp32 rounding of an fp64 tensor, kept in fp64."""
    return x.float().double()


def attn_fp16pv(q8, k8, v, q_scale, k_scale, *, q_gran="per_block", k_gran=None, is_causal=False, sm_scale=1.0,
                fold_sm_scale=False, out_dtype=F16, mask=None, q_offset=0, q_rows=None, q_len=None, return_lse=False,
                bound=False, emulate=None, mutation=None):
    """The FP16-PV CTA loop.  q8 [B,Hq,n,D] int8 (n rows of the call: q_rows, or q_offset .. q_offset + n), k8 [B,Hkv,Skv,D] int8,
    v [B,Hkv,Skv,D] 16-bit (cast to fp16 here), scales packed as the kernel reads them for the whole call of q_len rows (default
    the last row + 1).  q_gran: "per_block" (the Triton path; with fold_sm_scale), "per_warp" or "per_thread"; k_gran defaults to
    it.  mask: bool (True = visible) or a float bias in log2 units, broadcastable to [B,Hq,n,Skv] (the rows evaluated).
    Returns out (out_dtype) [, lse (fp64, log2)] [, Bound].
    Tests only: emulate (a torch.Generator) replaces the exact arithmetic with a CPU emulation of the kernel's (module docstring
    of test_fp16pv_oracle_cpu); mutation in {"bias_after_max", "skip_alpha", "p_bf16"} plants that mistake."""
    dev = q8.device
    B, Hq, n, D = q8.shape
    _, Hk, Sk, _ = k8.shape
    g = Hq // Hk
    rows = (torch.arange(q_offset, q_offset + n) if q_rows is None else q_rows.cpu().long())
    n_q = q_len if q_len is not None else (int(rows.max()) + 1 if n else 0)
    sm2 = 1.0 if fold_sm_scale else float(torch.tensor(sm_scale, dtype=torch.float32) * torch.tensor(O.LOG2E_CU, dtype=torch.float32))
    qs = O._expand_q_scale(q_scale.cpu(), q_gran, max(n_q, 1))[:, :, rows].to(dev).float()
    qss = (qs * sm2).double()                                                       # fp32 product
    ks = O._expand_k_scale(k_scale.cpu(), k_gran or q_gran, Sk)[:, :, :Sk].to(dev).double().repeat_interleave(g, dim=1)
    rows_d = rows.to(dev)
    bias = mask is not None and mask.dtype != torch.bool
    if mask is not None:
        mask = mask.to(dev).expand(B, Hq, n, Sk)
    m = torch.full((B, Hq, n), O.MASK_VALUE, dtype=torch.float64, device=dev)
    d = torch.zeros((B, Hq, n), dtype=torch.float64, device=dev)
    acc = torch.zeros((B, Hq, n, D), dtype=torch.float64, device=dev)
    qf = q8.double()
    if bound:
        a_abs = torch.zeros_like(acc)
        b_o = torch.zeros_like(acc)
        b_d = torch.zeros_like(d)
        moved = torch.zeros((B, Hq, n), dtype=torch.bool, device=dev)
        n_amb = n_vis = 0
    n_tiles = (Sk + BN - 1) // BN
    if is_causal and n:
        n_tiles = min(n_tiles, int(rows.max()) // BN + 1)
    skip_tile = n_tiles // 2 if mutation == "skip_alpha" else -1
    for j in range(n_tiles):
        s0, s1 = BN * j, min(BN * j + BN, Sk)
        si = qf @ k8[:, :, s0:s1].double().repeat_interleave(g, dim=1).transpose(-1, -2)       # exact integers
        coef = _r32(ks[:, :, None, s0:s1] * qss[..., None])
        vis = torch.ones(si.shape, dtype=torch.bool, device=dev)
        if is_causal:
            vis = vis & (torch.arange(s0, s1, device=dev)[None, :] <= rows_d[:, None])
        if mask is not None and not bias:
            vis = vis & mask[..., s0:s1]
        if bias:
            bt = mask[..., s0:s1].double()
            y = _r32(si * coef + bt)                                                 # fmaf(S, coef, bias)
            ymax = _r32(si * coef) if mutation == "bias_after_max" else y
        else:
            y = ymax = _r32(si * coef)
        mx = torch.where(vis, ymax, -math.inf).amax(dim=-1)
        m_new = torch.maximum(m, mx)
        m_arg = _r32(m - m_new)
        alpha = torch.where(m_new != m, torch.exp2(m_arg), 1.0)
        if bias:
            x = _r32(y - m_new[..., None])
        else:
            x = _r32(si * coef - m_new[..., None])                                   # fmaf(S, coef, -m)
        P = torch.where(vis, torch.exp2(x), 0.0)
        if bound or emulate is not None:
            eps = torch.where(P > 0, EPS_EXP * (1.0 + y.abs() + m_new.abs()[..., None]), 0.0)
            lo16 = (P * (1.0 - eps)).to(F16).double()
            hi16 = (P * (1.0 + eps)).to(F16).double()
        v16 = v[:, :, s0:s1].to(F16).double().repeat_interleave(g, dim=1)
        if emulate is not None:
            P, alpha = _emulate_p(P, eps, alpha, m_new != m, m_arg, lo16, hi16, emulate)
            P16 = P.to(F16).double()
            amb = lo16 != hi16
            pick = torch.rand(P.shape, generator=emulate, dtype=torch.float64).to(dev) < 0.5
            P16 = torch.where(amb, torch.where(pick, lo16, hi16), P16)
            d = _r32(_r32(d * alpha) + _r32(P.sum(dim=-1)))
            acc = _emulate_pv(acc, alpha, P16, v16)
        else:
            P16 = P.to(torch.bfloat16 if mutation == "p_bf16" else F16).double()
            if bound:
                n_amb += int(((lo16 != hi16) & (P > 0)).sum())
                n_vis += int((P > 0).sum())
                moved |= (d > 0) & (m_new != m)
                ch = m_new != m
                e_al = torch.where(ch, U32 + EPS_EXP * (1.0 + m_arg.abs()), 0.0)
                # the kernel's O before the rescale lies within b_o of the restatement's
                o_abs = acc.abs() + b_o
                b_o = ((b_o + (e_al + torch.where(ch, U32, 0.0))[..., None] * o_abs) * alpha[..., None]
                       + torch.where(ch, TINY32, 0.0)[..., None] * o_abs)
                v_abs = v16.abs()
                a_abs = a_abs * alpha[..., None] + P16 @ v_abs
                b_d = ((b_d + e_al * d) * alpha + (eps * P).sum(-1) + 82 * U32 * P.sum(-1)
                       + TINY32 * vis.sum(-1) + torch.where(ch, TINY32, 0.0) * d)
            a_t = alpha if j != skip_tile else torch.ones_like(alpha)
            d = d * alpha + P.sum(dim=-1)
            acc = acc * a_t[..., None]
            for k0 in range(0, s1 - s0, 16):                                          # the four k16 wgmma steps
                k1 = k0 + 16
                new = acc + P16[..., k0:k1] @ v16[..., k0:k1, :]
                if bound:
                    # a flipped fp16 P of this step, then the step's cut addends and rounding: 18 U_TC16 M, M the largest
                    # magnitude among the kernel's addends (its O before and after the step, within b_o of the restatement's,
                    # and the products, at most max P16 max |v16|)
                    b_o = b_o + (hi16[..., k0:k1] - lo16[..., k0:k1]) @ v_abs[..., k0:k1, :]
                    pmax = hi16[..., k0:k1].amax(-1, keepdim=True) * v_abs[..., k0:k1, :].amax(-2, keepdim=True)
                    big = torch.maximum(torch.maximum(acc.abs(), new.abs()) + b_o, pmax)
                    b_o = b_o + 18 * U_TC16 * big
                acc = new
            if bound:
                b_d = b_d + 2 * U32 * d
        m = m_new
    seen = d > 0
    if emulate is not None:
        inv = _r32(1.0 / d) * (1.0 + (2 * torch.rand(d.shape, generator=emulate, dtype=torch.float64).to(dev) - 1) * U32)
        xo = _r32(acc * _r32(inv)[..., None])
        lse_v = torch.log2(d) * (1.0 + 2.0 ** -23) + m
    else:
        xo = acc / d[..., None]
        lse_v = torch.log2(d) + m
    xo = torch.where(seen[..., None], xo, 0.0)
    out = xo.to(out_dtype)
    lse = torch.where(seen, lse_v, -math.inf)
    res = (out, lse) if return_lse else (out,)
    if bound:
        dd = torch.where(seen, d, 1.0)
        bo = b_o / dd[..., None] + xo.abs() * (b_d / dd)[..., None] + 3 * U32 * xo.abs()
        l_r = torch.log2(dd)
        lbd = (b_d / dd) / math.log(2.0) + 2.0 ** -21 * (1.0 + l_r.abs()) + 2.0 ** -22 * (l_r + m).abs()
        res += (Bound(xo, torch.where(seen[..., None], bo, 0.0), torch.where(seen, lbd, 0.0), n_amb, n_vis, int(seen.sum()),
                      int(moved.sum()), torch.where(seen[..., None], a_abs / dd[..., None], 0.0)),)
    return res if len(res) > 1 else res[0]


def _emulate_p(P, eps, alpha, ch, m_arg, lo16, hi16, gen):
    """The kernel's P and alpha as ex2.approx.ftz may give them: a relative perturbation within eps_P (alpha: within its own
    EPS_EXP (1 + |m - m_new|)), P below 2^-126 flushed to 0, rounded to fp32."""
    dev = P.device
    r = (2 * torch.rand(P.shape, generator=gen, dtype=torch.float64) - 1).to(dev)
    P = _r32(P * (1.0 + 0.9 * eps * r))
    P = torch.where(P < TINY32, 0.0, P)
    ra = (2 * torch.rand(alpha.shape, generator=gen, dtype=torch.float64) - 1).to(dev)
    alpha = torch.where(ch, _r32(alpha * (1.0 + 0.9 * EPS_EXP * (1.0 + m_arg.abs()) * ra)), alpha)
    alpha = torch.where(alpha < TINY32, 0.0, alpha)
    return P, alpha


def _emulate_pv(acc, alpha, P16, v16):
    """rescale_o, then four k16 fp16 wgmma steps into O, each with its addends (O and 16 exact products) cut to U_TC16 of the
    binade of the largest magnitude among them (truncation towards zero) and the sum rounded to fp32."""
    acc = _r32(acc * alpha[..., None])
    for k0 in range(0, P16.size(-1), 16):
        prod = P16[..., k0:k0 + 16, None] * v16[..., None, k0:k0 + 16, :]   # [.., R, 16, D], exact
        big = torch.maximum(acc.abs(), prod.abs().amax(dim=-2))
        q = torch.where(big > 0, torch.exp2(torch.floor(torch.log2(torch.where(big > 0, big, 1.0)))) * U_TC16, 1.0)
        cut = lambda t, qq: torch.trunc(t / qq) * qq
        acc = _r32(cut(acc, q) + cut(prod, q[..., None, :]).sum(dim=-2))
    return acc


def varlen_sequences(cu_q, cu_k):
    """[(q start, q end, k start, k end)] of a packed batch."""
    cq, ck = [int(c) for c in cu_q], [int(c) for c in cu_k]
    return [(cq[i], cq[i + 1], ck[i], ck[i + 1]) for i in range(len(cq) - 1)]


def attn_fp16pv_varlen(q8, k8, v, q_scale, k_scale, cu_q, cu_k, cu_qs, cu_ks, *, rows=None, k_shift=0, **kw):
    """The packed form (sab_qk_int8_sv_f16_attn_varlen): q8 [Tq,Hq,D], k8 / v [Tk,Hkv,D], per-block scales [n_blocks, H] with the
    sequences' first blocks cu_qs / cu_ks (per_block_int8_varlen); sm_scale*log2e folded into q_scale.  rows(L) gives the rows
    (a LongTensor) of a sequence of L rows to evaluate (default: all of them).  k_shift (tests only) reads every sequence's K one
    token late.  Returns [(b, rows, out, lse, Bound)] with out [1,Hq,len(rows),D]; kw as attn_fp16pv (bound, out_dtype,
    is_causal)."""
    res = []
    for b, (qa, qb, ka, kb) in enumerate(varlen_sequences(cu_q, cu_k)):
        L = qb - qa
        if L == 0:
            continue
        qsb = q_scale[int(cu_qs[b]):int(cu_qs[b + 1])].transpose(0, 1)[None]
        ksb = k_scale[int(cu_ks[b]):int(cu_ks[b + 1])].transpose(0, 1)[None]
        kk = k8[ka + k_shift:kb + k_shift].transpose(0, 1)[None]
        vv = v[ka:kb].transpose(0, 1)[None]
        r = torch.arange(L) if rows is None else rows(L)
        qq = q8[qa + r.to(q8.device)].transpose(0, 1)[None]
        out = attn_fp16pv(qq, kk, vv, qsb, ksb, q_gran="per_block", fold_sm_scale=True, q_rows=r, q_len=L, return_lse=True, **kw)
        res.append((b, r) + tuple(out))
    return res
