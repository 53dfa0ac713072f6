"""CPU numerics of the opt-in FMA-pipe exponential of the sm_90a attention kernel (csrc/ptx.cuh `ex2_poly2`, builds with
-DSAB_POLY_EXP_PAIRS=n): a float32 restatement of the instruction sequence, its error against exp2, and what replacing
n of every 4 column pairs of P by it does to the attention output of the CPU oracle (far inside the 1e-2 tolerance); the
default build does not use the polynomial."""
import numpy as np
import torch

from oracle import sage_oracle as O

C1, C2, C3 = np.float32(0.6951166391372681), np.float32(0.22764497995376587), np.float32(0.07706724107265472)
MAGIC_BITS = 0x4B400000   # 1.5 * 2^23


def _fma32(a, b, c):
    """fp32 fused multiply-add: the product of two fp32 numbers and the sum are exact in float64 up to one rounding, which is
    then rounded again to fp32 (double rounding can differ from a true FMA by 1 ulp in ~1e-9 of the cases: irrelevant here)."""
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(np.float32)


def ex2_poly_np(y):
    """ex2_poly2 for one lane: clamp, floor via the round-down magic add, degree-3 Horner, exponent insertion."""
    y = np.maximum(np.asarray(y, dtype=np.float32), np.float32(-126.0))
    fl = np.floor(y).astype(np.float32)                      # add.rm(y, 1.5*2^23) - 1.5*2^23 == floor(y), exact
    r_bits = (MAGIC_BITS + fl.astype(np.int64)).astype(np.int64)
    fr = _fma32(fl, np.float32(-1.0) * np.ones_like(y), y)   # y - floor(y) in [0, 1]
    p = _fma32(fr, C3 * np.ones_like(y), C2 * np.ones_like(y))
    p = _fma32(p, fr, C1 * np.ones_like(y))
    p = _fma32(p, fr, np.ones_like(y))
    bits = (p.view(np.uint32).astype(np.int64) + ((r_bits << 23) & 0xFFFFFFFF)) & 0xFFFFFFFF
    return bits.astype(np.uint32).view(np.float32)


def test_polynomial_is_the_minimax_fit_and_accurate():
    y = np.concatenate([np.linspace(-126.0, 9.0, 2_000_001), -np.logspace(-9, 2, 100001), [0.0, -0.0, -1.0, 8.807, -1e-8]]).astype(np.float32)
    got = ex2_poly_np(y).astype(np.float64)
    ref = np.exp2(y.astype(np.float64))
    rel = np.abs(got / ref - 1.0)
    assert rel.max() <= 8.8e-5, rel.max()                   # fitted bound 8.56e-5 + fp32 evaluation
    assert ex2_poly_np(np.float32(0.0)) == np.float32(1.0) and ex2_poly_np(np.float32(-3.0)) == np.float32(0.125)
    assert np.all(np.diff(ex2_poly_np(np.sort(y))) >= -1e-4 * ex2_poly_np(np.sort(y))[1:])   # monotone up to the seam at integers
    # arguments far below the clamp (masked sentinels) give 2^-126, not NaN / inf
    assert ex2_poly_np(np.float32(-5e6)) == np.float32(2.0 ** -126)
    # the coefficients are the minimax fit of 2^x / relative error on [0,1] with p(0) = 1 (refit, compare the bound)
    from scipy.optimize import linprog
    x = np.linspace(0, 1, 2001); f = 2.0 ** x
    A = np.stack([x / f, x ** 2 / f, x ** 3 / f], 1); b = 1 - 1 / f
    n = len(x)
    r = linprog([0, 0, 0, 1], A_ub=np.block([[A, -np.ones((n, 1))], [-A, -np.ones((n, 1))]]), b_ub=np.concatenate([b, -b]),
                bounds=[(None, None)] * 4)
    assert r.status == 0 and abs(r.x[3] - 8.56e-5) < 2e-7
    assert np.allclose(r.x[:3], [float(C1), float(C2), float(C3)], atol=2e-5)


def _mixed_exp2(pairs):
    """exp2 of a [.., 64]-wide tile where `pairs` of every 4 column pairs take the polynomial (attn.cu: ((i >> 1) & 3) < n)."""
    def fn(t):
        ref = torch.exp2(t)
        poly = torch.from_numpy(ex2_poly_np(t.numpy()))
        col = torch.arange(t.shape[-1])
        use = ((col >> 1) & 3) < pairs
        return torch.where(use, poly, ref)
    return fn


def test_effect_on_attention_output():
    """Two regimes.  (1) Benchmark-like inputs (plain randn: flat softmax; at S=512 a key carries at most ~2 % of a row, at
    S=8192 sixteen times less): the output moves by at most (largest key weight) x (one e4m3 step = 2^-4 .. 2^-3) x |v|,
    4e-3 here.  (2) Peaky rows (channel-biased K, causal prefixes with a handful of keys): a P element that
    sits on an e4m3 rounding boundary can land on the other side (flip rate ~2e-3 per emulated element, next test), which
    moves that key's weight by one e4m3 step (6-12 % of it) — visible against the reference's own P bits (up to ~1e-2 on a
    row dominated by one key), but not an accuracy loss: the error against exact attention does not grow, because either
    rounding of a boundary value is equally far from the true P.  This is why the polynomial is opt-in."""
    torch.manual_seed(0)
    B, H, S, D = 1, 2, 512, 128
    worst = {}
    for peaky in (False, True):
        q, k, v = (torch.randn(B, H, S, D).to(torch.float16) for _ in range(3))      # fp16 output grid: 2^-10 relative
        if peaky:
            k = k + 3.0 * torch.randn(B, H, 1, D).to(torch.float16)
            q = q * 3.0
        for causal in (False, True):
            exact = O.sdpa_fp32(q, k, v, is_causal=causal)
            base, base_lse = O.sageattn_qk_int8_pv_fp8_cuda(q, k, v, is_causal=causal, return_lse=True, emulate_f16_accum=False)
            e0 = (base.float() - exact.float()).abs()
            for pairs in (1, 2, 4):
                o, lse = O.sageattn_qk_int8_pv_fp8_cuda(q, k, v, is_causal=causal, return_lse=True, emulate_f16_accum=False,
                                                        exp2_fn=_mixed_exp2(pairs))
                diff = (o.float() - base.float()).abs().max().item()
                e1 = (o.float() - exact.float()).abs()
                worst[(peaky, causal, pairs)] = (round(diff, 5), round(e0.max().item(), 5), round(e1.max().item(), 5))
                assert (lse - base_lse).abs().max().item() <= 2e-4                    # d moves by the 8.6e-5 relative error only
                if not peaky and not causal:
                    assert diff <= 6e-3, (pairs, diff)                                # S=512: a key carries <= ~2 % of a row
                assert diff <= 1.5 * e0.max().item() + 1e-3, (peaky, causal, pairs, diff)   # never beyond the path's own error
                # accuracy against exact attention is unchanged: mean within 2 %, max within 25 % + 1e-3 of the MUFU build's
                assert e1.mean().item() <= 1.02 * e0.mean().item() + 1e-5, (peaky, causal, pairs)
                assert e1.max().item() <= 1.25 * e0.max().item() + 1e-3, (peaky, causal, pairs, e0.max().item(), e1.max().item())
    print("(peaky, causal, pairs): (max |O_poly - O_mufu|, max err MUFU vs exact, max err poly vs exact)")
    for key, val in worst.items():
        print("  ", key, val)


def test_e4m3_flip_rate_of_P():
    """How often the polynomial changes the e4m3 rounding of P in (0, 448]: the relative error is 8.6e-5 against a rounding
    interval of 2^-3 .. 2^-4 relative width, so about 0.1-0.3 % of the emulated elements move by one e4m3 ulp."""
    g = np.random.default_rng(0)
    y = (8.807 - g.exponential(3.0, size=1_000_000)).astype(np.float32)
    a = torch.from_numpy(np.exp2(y.astype(np.float64)).astype(np.float32)).to(torch.float8_e4m3fn).float()
    b = torch.from_numpy(ex2_poly_np(y)).to(torch.float8_e4m3fn).float()
    flips = (a != b).float().mean().item()
    assert flips < 5e-3, flips
    ulp = torch.exp2(torch.floor(torch.log2(torch.maximum(a, b).clamp_min(2.0 ** -6))) - 3)     # e4m3 spacing (2^-9 in the subnormals)
    assert ((a - b).abs() <= ulp).all()                      # never more than one e4m3 step
    print("e4m3 flip rate:", flips)


def test_lazy_rescale_numerics():
    """The lazy running max (csrc/attn.cu, lazy_tau): P is taken against a stale maximum, i.e. scaled by 2^(m_exact - m_stale) with a
    non-integer exponent, so its e4m3 rounding is a different realisation of the same quantisation noise: the output is not
    comparable bit for bit with the reference kernel's, but its error against exact attention is the same (mean within 3 %),
    and the LSE (from un-rounded sums) agrees to 1e-5.  The number of tiles in which ANY of a warp's 32 rows moves its maximum —
    the tiles that pay an O rescale — drops from most to a few."""
    torch.manual_seed(1)
    B, H, S, D = 1, 2, 2048, 128
    q, k, v = (torch.randn(B, H, S, D).to(torch.float16) for _ in range(3))
    k = k + 2.0 * torch.randn(B, H, 1, D).to(torch.float16)
    for causal in (False, True):
        exact = O.sdpa_fp32(q, k, v, is_causal=causal).float()
        base, base_lse = O.sageattn_qk_int8_pv_fp8_cuda(q, k, v, is_causal=causal, return_lse=True, emulate_f16_accum=False)
        e0 = (base.float() - exact).abs()
        for tau in (2, 3, 4):
            o, lse = O.sageattn_qk_int8_pv_fp8_cuda(q, k, v, is_causal=causal, return_lse=True, emulate_f16_accum=False, lazy_tau=tau)
            e1 = (o.float() - exact).abs()
            assert e1.mean().item() <= 1.03 * e0.mean().item() + 1e-5, (causal, tau, e0.mean().item(), e1.mean().item())
            assert e1.max().item() <= 1.3 * e0.max().item() + 1e-3, (causal, tau, e0.max().item(), e1.max().item())
            assert (lse - base_lse).abs().max().item() <= 1e-4
            print(f"causal={causal} tau={tau}: mean err {e0.mean().item():.2e} -> {e1.mean().item():.2e}, max {e0.max().item():.2e} -> {e1.max().item():.2e}, "
                  f"max |O_lazy - O_exact_rule| {(o.float() - base.float()).abs().max().item():.2e}")
    # rescale frequency at warp granularity (32 consecutive rows), S = 2048 -> 32 tiles of 64 keys
    sc = (q[0, 0].float() @ k[0, 0].float().T) * (D ** -0.5) * 1.4426950408889634
    tiles = sc.view(S, S // 64, 64).amax(-1)                         # [rows, tiles] row max per tile, log2 units
    def moved_fraction(tau):
        m = torch.full((S,), -5e6)
        hits = 0
        for j in range(tiles.shape[1]):
            cand = torch.maximum(m, tiles[:, j])
            move = (cand - m > tau) if tau is not None else (cand > m)
            m = torch.where(move, cand, m)
            if j > 0:
                hits += int(move.view(S // 32, 32).any(-1).sum())
        return hits / ((tiles.shape[1] - 1) * (S // 32))
    exact, lazy = moved_fraction(None), moved_fraction(3)
    print(f"warp-tiles that rescale O: exact rule {exact:.2f}, tau=3 {lazy:.3f}")
    assert exact > 0.5 and lazy < 0.15


def test_alternating_tile_row_sums_combine_to_the_sequential_sum():
    """csrc/attn_alt.cu: warpgroup w accumulates d_w = sum over ITS tiles of sum_i P(j)_i relative to the max of its latest
    tile; the epilogue combines d = d_0 2^(m_0 - m_fin) + d_1 2^(m_1 - m_fin).  Against the sequential update_mdo recurrence
    d = d * 2^(m_old - m_new) + sum(P) (attn_utils.cuh:377-458) the result differs by fp32 rounding only — also with the lazy
    max (tau = 3), where m(j) is the maximum IN USE, not the true one."""
    g = np.random.default_rng(3)
    for tau in (0, 3):
        for n_kv in (1, 2, 3, 8, 33):
            S = (g.standard_normal((64, n_kv, 64)) * 1.5 + g.standard_normal((64, n_kv, 1))).astype(np.float32)   # log2-domain logits
            m = np.full(64, -5e6, np.float32)
            d_seq = np.zeros(64, np.float32)
            d_w = [np.zeros(64, np.float32), np.zeros(64, np.float32)]
            m_w = [np.full(64, -5e6, np.float32), np.full(64, -5e6, np.float32)]
            for j in range(n_kv):
                mx = S[:, j].max(-1)
                if tau:
                    m_true = np.maximum(m, mx - np.float32(8.807 - tau))
                    m_new = np.where(m_true - m > tau, m_true, m).astype(np.float32)
                else:
                    m_new = np.maximum(m, mx - np.float32(8.807))
                P = np.exp2(S[:, j] - m_new[:, None]).astype(np.float32)
                assert P.max() <= 448.0 * (1 + 1e-6)
                d_seq = (d_seq * np.exp2(m - m_new) + P.sum(-1)).astype(np.float32)
                w = j & 1
                d_w[w] = (d_w[w] * np.exp2(m_w[w] - m_new) + P.sum(-1)).astype(np.float32)
                m_w[w] = m_new
                m = m_new
            m_fin = np.maximum(m_w[0], m_w[1])
            assert np.array_equal(m_fin, m)
            d_alt = d_w[0] * np.exp2(m_w[0] - m_fin) + d_w[1] * np.exp2(m_w[1] - m_fin)
            assert np.allclose(d_alt, d_seq, rtol=2e-6, atol=0), (tau, n_kv)
