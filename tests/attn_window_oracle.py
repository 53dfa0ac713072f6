"""CPU restatement of the masked forms of the INT8+FP8 forward (sage_attn_fwd_kernel with kWindow or the block mask, csrc/attn.cu),
with an elementwise bound on |kernel - restatement|.  TEST INFRASTRUCTURE ONLY: imported by the window and block-sparse tests,
never by the product package.

One loop, attn_int8_fp8_tiles, restates the kernel's CTA: for each (b, h, 128-row Q block) it visits the ordered list of 64-key
tiles the kernel visits, with the element visibility mask applied inside each tile.  The per-tile arithmetic is that of the dense
restatement (oracle.sage_oracle.attn_int8_fp8_cuda) with the kernel's lazy running max, except where a row part sees nothing of a
tile: the kernel then keeps m and d and adds P = 0 (the dense restatement, whose rows always see a key of every tile they reach,
would give P = exp2(0) there).  A row with no visible key gives 0 and lse -inf.  Two callers:
  * attn_int8_fp8_window: key j is visible to query i iff i - left <= j <= i + right (-1: that side unbounded), j < Skv, and
    j <= i when causal; the tiles are window_tiles (csrc/attn_common.cuh);
  * attn_int8_fp8_blocksparse_causal: the visible tiles of mask row (b, h, i) up to the causal horizon, ascending, with the element
    mask expand_block_mask(...) & tril.  (The non-causal form is also the gathered restatement of attn_blocksparse_oracle.)

The running max m is the kernel's bit for bit: the row max of a tile is float(max int S) * coef with coef = k_scale * (q_scale *
sm_scale*log2e) > 0, so it equals the maximum of the separately rounded products the restatement takes; the offset 8.807 - tau, the
test m_true - m > tau and the mask value are the same fp32 operations.  P, d and O are not: the kernel computes
P = ex2.approx(fmaf(s, coef, -m)), sums d per thread in another order and accumulates P8 V in the tensor core.

Bound (bound=True), per output element, of |kernel - restatement| before the output's 16-bit rounding (check_forward adds that
rounding with attn_bwd_oracle.elementwise_ratio).  Constants as in attn_bwd_oracle: U32 = 2^-23, EPS_EXP = 2^-21.
  * P: both sides evaluate exp2 of the same logit x = S - m (S the log2 logit), the kernel with one FMA rounding of |x| and
    ex2.approx (relative error < 2^-22), the restatement with the roundings of S*coef and of S - m and an exp2 within one ulp.
    So the two P differ by at most eps_P * P with eps_P = EPS_EXP * (1 + |S| + |m|).
  * e4m3: P8 = e4m3(P) is monotone in P, so the kernel's P8 lies between e4m3(P (1 - eps_P)) and e4m3(P (1 + eps_P)).  Where these
    differ the element is ambiguous (P lies within eps_P P of a rounding midpoint) and may take the neighbouring code: it adds
    (hi8 - lo8) |v8[j, c]| to the row's accumulator bound, which the epilogue turns into step * |v8[j, c]| * v_scale[c] / d.
    Everywhere else the two P8 are the same bits.
  * the tile product P8 V8: the restatement sums it in fp32 (64 keys: 64 U32 times sum |P8| |V8|); the kernel in two chained
    k32 FP8 wgmma steps, whose accumulator keeps about 14 bits (DeepSeek-V3 technical report, section 3.3.2, for Hopper FP8
    GEMMs).  Model of a step: its addends (32 exact products and the value carried in) are aligned to the largest exponent E
    among them and cut to U_TC = 2^-13 of 2^E, so each loses less than U_TC 2^E <= U_TC M, M the largest magnitude:
      step 1: 32 U_TC max_j |P8_j v_jc| (j < 32),   step 2: 33 U_TC max(sum_{j<32} |P8_j v_jc|, max_{j>=32} |P8_j v_jc|).
    (A relative 2^-13 of the sum of magnitudes per step, the first model tried, was exceeded by up to 1.22 times on H100 at
    window (63, 64), fp16 output: the cut addends' errors do not cancel.)
  * the fold O += PV in fp32 adds U32 |O|; a rescale O *= alpha, d *= alpha adds U32 plus the relative error of alpha =
    ex2.approx(m - m_new), EPS_EXP (1 + |m - m_new|), of everything accumulated before it (|O| and |d| are tracked as the
    accumulated sums of magnitudes, through the same alphas).
  * d: the sum of un-rounded P, so eps_P P per element, plus the summation: at most 82 U32 of the tile's sum (16 terms per thread
    in the kernel, 64 in torch.sum, two shuffle adds) and 2 U32 of d per tile (d * alpha + sum on either side), 2 U32 at the end.
  * epilogue: x = O / d * v_scale (+ v_mean).  With |e_O| <= B_O and |e_d| <= B_d:
      |e_x| <= v_scale (B_O / d + |O / d| (B_d / d)) + 8 U32 (|x| + |v_mean|)
    (rcp.approx within one ulp, the products, the addition, on both sides).
  * lse = log2(d) + m, the same m: (B_d / d) / ln2 + 2^-21 (1 + |log2 d|) (lg2.approx and log2) + 2^-22 |lse| (the additions),
    a few fp32 ulps of lse.
The bound assumes the kernel's m, which the paragraph above shows is the restatement's; were it not, the lazy max could move on a
different tile, and most of the row's P would change their e4m3 rounding, far outside the bound."""
import collections
import math

import torch

from attn_blocksparse_oracle import expand_block_mask
from attn_bwd_oracle import EPS_EXP, U32, check_elementwise
from oracle import sage_oracle as O

U_TC = 2.0 ** -13     # FP8 wgmma accumulation, per k32 step (see the module docstring)
E4M3 = torch.float8_e4m3fn

Bound = collections.namedtuple("Bound", "o o_bound lse_bound ambiguous visible moved rows")
Bound.__doc__ = """o: the restatement's output before its 16-bit rounding (fp64), o_bound / lse_bound: the bounds of the module
docstring, ambiguous / visible: counts of ambiguous and of visible elements, moved / rows: counts of the rows whose running max
moves on a tile after their first visible one and of the rows that see a key."""


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


def _tc_bound(P8, v_abs):
    """The error bound of the kernel's two k32 FP8 wgmma steps on one tile (module docstring), [.., R, D] from P8 [.., R, n] and
    |V8| [.., n, D] (fp64)."""
    p = P8.double()
    prod = p[..., :, :, None] * v_abs[..., None, :, :]                     # [.., R, n, D], exact
    m1 = prod[..., :32, :].amax(-2)
    if prod.size(-2) <= 32:
        return 32 * U_TC * m1
    m2 = torch.maximum(prod[..., :32, :].sum(-2), prod[..., 32:, :].amax(-2))
    return U_TC * (32 * m1 + 33 * m2)


def attn_int8_fp8_tiles(q8, k8, v8, q_scale, k_scale, v_scale, tiles, mask, *, qk_quant_gran="per_thread", sm_scale=1.0,
                        lazy_tau=4, out_dtype=torch.float16, return_lse=False, v_mean=None, bound=False, p8_fn=None):
    """The kernel's CTA loop on [B,H,S,D] tensors with fp32 PV accumulation; v8 is the LOGICAL [B,Hkv,Sk,D] fp8 tensor.
    tiles(b, h, i): the ordered 64-key tiles CTA (b, h, Q block i) visits.  mask: bool, broadcastable to [B,Hq,Sq,Sk].
    lazy_tau: the kernel's lazy running max (0: the exact max of SAB_ATTN_KERNEL=exact).  v_mean: [B,Hkv,D] (smooth_v).
    bound=True: also return a Bound (module docstring).  p8_fn(P8, lo8, hi8) (tests only) replaces each tile's e4m3 P, given the
    codes of P (1 -+ eps_P)."""
    B, Hq, Sq, D = q8.shape
    _, Hk, Sk, _ = k8.shape
    g = Hq // Hk
    BH = B * Hq
    tau = torch.tensor(float(lazy_tau), dtype=torch.float32)
    off = torch.tensor(O.S_FP8_OFFSET, dtype=torch.float32) - tau          # kFp8Offset - tau, in fp32 as the kernel
    mask_value = torch.tensor(O.MASK_VALUE, dtype=torch.float32)
    qs_row = O._expand_q_scale(q_scale, qk_quant_gran, Sq)[:, :, :Sq].reshape(BH, Sq)
    ks_key = O._expand_k_scale(k_scale, qk_quant_gran, Sk)[:, :, :Sk].repeat_interleave(g, dim=1).reshape(BH, Sk)
    qf = q8.float().reshape(BH, Sq, D)
    kf = k8.float().repeat_interleave(g, dim=1).reshape(BH, Sk, D)
    vf = v8.float().repeat_interleave(g, dim=1).reshape(BH, Sk, D)
    vsc = v_scale.float().repeat_interleave(g, dim=1).reshape(BH, D)
    vm = None if v_mean is None else v_mean.float().repeat_interleave(g, dim=1).reshape(BH, D)
    em4 = mask.expand(B, Hq, Sq, Sk)
    sm2 = torch.tensor(sm_scale, dtype=torch.float32) * torch.tensor(O.LOG2E_CU, dtype=torch.float32)
    out = torch.zeros((BH, Sq, D), dtype=out_dtype)
    lse = torch.full((BH, Sq), -float("inf"), dtype=torch.float32)
    if bound:
        o64 = torch.zeros((BH, Sq, D), dtype=torch.float64)
        ob = torch.zeros((BH, Sq, D), dtype=torch.float64)
        lb = torch.zeros((BH, Sq), dtype=torch.float64)
        n_amb = n_vis = n_moved = n_rows = 0
    for i, r0 in enumerate(range(0, Sq, 128)):
        r1 = min(r0 + 128, Sq)
        groups = collections.defaultdict(list)
        for bh in range(BH):
            groups[tuple(tiles(bh // Hq, bh % Hq, i))].append(bh)
        for tl, idx in groups.items():
            idx = torch.tensor(idx)
            G, R = len(idx), r1 - r0
            q_blk = qf[idx, r0:r1]
            coef_q = (sm2 * qs_row[idx, r0:r1])[..., None]
            m = torch.full((G, R), O.MASK_VALUE, dtype=torch.float32)
            d = torch.zeros((G, R), dtype=torch.float32)
            acc = torch.zeros((G, R, D), dtype=torch.float32)
            if bound:
                a_abs = torch.zeros((G, R, D), dtype=torch.float64)    # sum |P8| |V8| through the alphas
                b_o = torch.zeros((G, R, D), dtype=torch.float64)
                b_d = torch.zeros((G, R), dtype=torch.float64)
                moved = torch.zeros((G, R), dtype=torch.bool)
            for j in tl:
                s0, s1 = 64 * j, min(64 * j + 64, Sk)
                em = em4[idx // Hq, idx % Hq, r0:r1, s0:s1]
                S = (q_blk @ kf[idx, s0:s1].transpose(-1, -2)) * (coef_q * ks_key[idx, None, s0:s1])
                mx = torch.where(em, S, torch.tensor(-float("inf"))).amax(dim=-1)
                mx = torch.where(em.any(-1), mx, mask_value)
                m_true = torch.maximum(m, mx - off)
                m_new = torch.where(m_true - m > tau, m_true, m)
                alpha = torch.exp2(m - m_new)
                P = torch.where(em, torch.exp2(S - m_new[..., None]), torch.tensor(0.0))
                P8 = P.to(E4M3).float()
                if bound or p8_fn is not None:
                    eps = EPS_EXP * (1.0 + S.double().abs() + m_new.double().abs()[..., None])
                    lo8 = (P.double() * (1.0 - eps)).to(E4M3).double()
                    hi8 = (P.double() * (1.0 + eps)).to(E4M3).double()
                if p8_fn is not None:
                    P8 = p8_fn(P8, lo8.float(), hi8.float())
                if bound:
                    n_amb += int((em & (lo8 != hi8)).sum())
                    n_vis += int(em.sum())
                    moved |= (d > 0) & (m_new != m)
                    al = alpha.double()
                    e_al = torch.where(m_new != m, U32 + EPS_EXP * (1.0 + (m - m_new).double().abs()), 0.0)
                    v_abs = vf[idx, s0:s1].double().abs()
                    s_abs = P8.double() @ v_abs
                    b_o = (b_o + e_al[..., None] * a_abs) * al[..., None]
                    a_abs = a_abs * al[..., None] + s_abs
                    b_o = b_o + (hi8 - lo8) @ v_abs + 64 * U32 * s_abs + U32 * a_abs + _tc_bound(P8, v_abs)
                    Pd = P.double()
                    b_d = (b_d + e_al * d.double()) * al + (eps * Pd).sum(-1) + 82 * U32 * Pd.sum(-1)
                d = d * alpha + P.sum(dim=-1)
                acc = acc * alpha[..., None] + P8 @ vf[idx, s0:s1]
                m = m_new
                if bound:
                    b_d = b_d + 2 * U32 * d.double()
            o = (acc / d[..., None]) * vsc[idx, None, :]
            if vm is not None:
                o = o + vm[idx, None, :]
            seen = (d > 0)[..., None]
            out[idx, r0:r1] = torch.where(seen, o, torch.tensor(0.0)).to(out_dtype)
            lse[idx, r0:r1] = torch.log2(d) + m
            if bound:
                dd = d.double()
                n_moved += int(moved.sum())
                n_rows += int((d > 0).sum())
                b_d = b_d + 2 * U32 * dd
                od = acc.double() / dd[..., None]
                x = od * vsc[idx, None, :].double() + (0.0 if vm is None else vm[idx, None, :].double())
                bo = (vsc[idx, None, :].double() * (b_o / dd[..., None] + od.abs() * (b_d / dd)[..., None])
                      + 8 * U32 * (x.abs() + (0.0 if vm is None else vm[idx, None, :].double().abs())))
                o64[idx, r0:r1] = torch.where(seen, x, 0.0)
                ob[idx, r0:r1] = torch.where(seen, bo, 0.0)
                l_r = torch.log2(dd)
                lbd = (b_d / dd) / math.log(2.0) + 2.0 ** -21 * (1.0 + l_r.abs()) + 2.0 ** -22 * (l_r + m.double()).abs()
                lb[idx, r0:r1] = torch.where(d > 0, lbd, 0.0)
    out, lse = out.reshape(B, Hq, Sq, D), lse.reshape(B, Hq, Sq)
    res = (out, lse) if return_lse else (out,)
    if bound:
        res += (Bound(o64.reshape(B, Hq, Sq, D), ob.reshape(B, Hq, Sq, D), lb.reshape(B, Hq, Sq), n_amb, n_vis, n_moved, n_rows),)
    return res if len(res) > 1 else res[0]


def attn_int8_fp8_window(q8, k8, v8, q_scale, k_scale, v_scale, *, window, is_causal=False, **kw):
    """The sliding-window form (sab_qk_int8_sv_f8_attn_window); kw as attn_int8_fp8_tiles."""
    left, right = window
    Sq, Sk = q8.shape[2], k8.shape[2]
    ranges = [range(*window_tiles(r0, min(r0 + 128, Sq) - 1, Sk, left, right, is_causal)) for r0 in range(0, Sq, 128)]
    return attn_int8_fp8_tiles(q8, k8, v8, q_scale, k_scale, v_scale, lambda b, h, i: ranges[i],
                               window_mask(Sq, Sk, left, right, is_causal), **kw)


def blocksparse_causal_tiles(block_mask, Sq, Sk):
    """tiles(b, h, i) of the causal block-sparse kernel: the visible 64-key tiles of mask row (b, h, i) below the causal horizon
    ceil(128 (i + 1) / 64) (csrc/attn.cu build_kv_list), ascending."""
    nk = (Sk + 63) // 64
    bm = block_mask.expand(-1, -1, (Sq + 127) // 128, nk)

    def tiles(b, h, i):
        row = bm[b % bm.size(0), h % bm.size(1), i]
        return [j for j in range(min(nk, 2 * i + 2)) if bool(row[j])]
    return tiles


def attn_int8_fp8_blocksparse_causal(q8, k8, v8, q_scale, k_scale, v_scale, block_mask, **kw):
    """The causal block-sparse form (sab_qk_int8_sv_f8_attn_blocksparse, is_causal=1): block_mask [B or 1, Hq or 1, ceil(Sq/128),
    ceil(Sk/64)] bool indexed by the Q head; kw as attn_int8_fp8_tiles."""
    Sq, Sk = q8.shape[2], k8.shape[2]
    em = expand_block_mask(block_mask, Sq, Sk) & window_mask(Sq, Sk, -1, -1, True)
    return attn_int8_fp8_tiles(q8, k8, v8, q_scale, k_scale, v_scale, blocksparse_causal_tiles(block_mask, Sq, Sk), em, **kw)


def check_forward(name, o, lse, lse_ref, bd, dims=("b", "h", "row", "col")):
    """The kernel's 16-bit output o and raw log2 lse ([B,H,Sq(,D)], any device) against the restatement's lse_ref and Bound bd:
    every element within its bound plus the output rounding (attn_bwd_oracle.check_elementwise; a row that sees no key has bound 0,
    so it must be exactly 0), lse -inf exactly on the rows that see no key and within lse_bound elsewhere.  Returns (worst output
    ratio, worst lse ratio)."""
    o, lse = o.cpu(), lse.cpu().double()
    worst, _ = check_elementwise(name, o, bd.o, bd.o_bound, dims)
    seen = bd.lse_bound > 0
    assert torch.equal(torch.isneginf(lse), ~seen), f"{name}: lse must be -inf exactly on the rows that see no key"
    ratio = ((lse - lse_ref.double()).abs() / bd.lse_bound)[seen]
    worst_l = float(ratio.max()) if ratio.numel() else 0.0
    assert worst_l <= 1.0, f"{name}: lse off by {worst_l:.3g} times its bound"
    return worst, worst_l
