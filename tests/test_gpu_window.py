"""GPU tests (-m gpu) of the sliding-window attention (sageattn_window; sab_qk_int8_sv_f8_attn_window and
sab_qk_int8_attn_bwd_window):
  1. identities, bit for bit on o, lse, dq, dk, dv: (-1, -1) and (>= Skv, >= Skv) are sageattn_qk_int8_pv_fp8_cuda, (-1, 0) is
     its causal call;
  2. windows against the CPU restatement (attn_window_oracle) on the call's own quantised operands and against exact windowed
     attention: narrow and wide windows, causal or not, Sq != Skv with rows that see no key, lengths 1 to 129 and a long case,
     bottom rows of a Q tile whose window starts in a later tile than the top row's;
  3. the gradient kernels elementwise against attn_bwd_masked_oracle fed the window's element mask (the bound of check_elementwise),
     reproducibility, zeros for hidden rows and keys; 4. validation; 5. torch.compile."""
import math
import warnings

import pytest
import torch

import sageattention_b200 as sab
from sageattention_b200 import ops
from attn_window_oracle import attn_int8_fp8_window, check_forward, window_mask
from attn_bwd_masked_oracle import attn_bwd_masked
from attn_bwd_oracle import check_elementwise
from sageattention_b200.core import _quant_qk
from sageattention_b200.quant import per_channel_fp8

pytestmark = pytest.mark.gpu
BF, FP = torch.bfloat16, torch.float16
TOL_EXACT = 6e-2      # max-abs against exact attention (tests/test_gpu_parity.py), rows with >= 128 visible keys
GRAN = {"per_warp": 2, "per_thread": 3}     # SAB_GRAN_*


def _qkv(B, Hq, Hkv, Sq, Sk, D, dt, layout="HND", seed=0, grad=False):
    g = torch.Generator(device="cuda").manual_seed(seed)
    shp = lambda H, S: (B, H, S, D) if layout == "HND" else (B, S, H, D)
    q = torch.randn(shp(Hq, Sq), generator=g, device="cuda").to(dt)
    k = (torch.randn(shp(Hkv, Sk), generator=g, device="cuda") + torch.randn(shp(Hkv, 1), generator=g, device="cuda")).to(dt)
    v = torch.randn(shp(Hkv, Sk), generator=g, device="cuda").to(dt)
    if grad:
        q, k, v = (t.requires_grad_() for t in (q, k, v))
    return q, k, v


def _hnd(x, layout):
    return x if layout == "HND" else x.transpose(1, 2)


def _exact(q, k, v, em, scale):
    g = q.size(1) // k.size(1)
    s = (q.double() @ k.double().repeat_interleave(g, 1).transpose(-1, -2)) * scale
    p = torch.softmax(s.masked_fill(~em, -math.inf), dim=-1).nan_to_num(0.0)
    return p @ v.double().repeat_interleave(g, 1)


# ------------------------------------------------------------------------------------------------ identities
IDENTITY_CASES = [  # B, Hq, Hkv, S, D, dtype, layout, gran, pv_accum, smooth_v
    (1, 2, 2, 512, 128, FP, "HND", "per_thread", "fp32+fp16", False),
    (2, 2, 2, 384, 64, BF, "NHD", "per_warp", "fp32+fp32", False),
    (1, 8, 2, 300, 96, BF, "HND", "per_thread", "fp32", True),
    (1, 4, 1, 257, 128, BF, "NHD", "per_warp", "fp32", True),
    (1, 4, 2, 200, 64, FP, "HND", "per_warp", "fp32+fp16", False),
    (1, 2, 2, 129, 96, FP, "NHD", "per_thread", "fp32+fp32", False),
]


@pytest.mark.parametrize("case", IDENTITY_CASES, ids=lambda c: "-".join(str(x).replace("torch.", "") for x in c))
def test_unbounded_windows_are_the_dense_calls_bitwise(case):
    B, Hq, Hkv, S, D, dt, lay, gran, acc, sv = case
    q, k, v = _qkv(B, Hq, Hkv, S, S, D, dt, lay, seed=S + D)
    kw = dict(tensor_layout=lay, qk_quant_gran=gran, pv_accum_dtype=acc, smooth_v=sv, return_lse=True)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")      # smooth_v with a non-"fp32" pv_accum_dtype warns, in both calls
        o_d, l_d = sab.sageattn_qk_int8_pv_fp8_cuda(q, k, v, **kw)
        o_c, l_c = sab.sageattn_qk_int8_pv_fp8_cuda(q, k, v, is_causal=True, **kw)
        for window in ((-1, -1), (S, S), (S + 1000, S - 1 + 7), (-1, S)):
            o, l = sab.sageattn_window(q, k, v, window, **kw)
            assert torch.equal(o, o_d) and torch.equal(l, l_d), window
            o, l = sab.sageattn_window(q, k, v, window, is_causal=True, **kw)
            assert torch.equal(o, o_c) and torch.equal(l, l_c), window
        for window in ((-1, 0), (S, 0)):
            o, l = sab.sageattn_window(q, k, v, window, **kw)
            assert torch.equal(o, o_c) and torch.equal(l, l_c), window


def test_unbounded_window_with_unequal_lengths_is_the_dense_call_bitwise():
    q, _, _ = _qkv(1, 4, 2, 300, 300, 128, BF, seed=1)
    _, k, v = _qkv(1, 4, 2, 700, 700, 128, BF, seed=2)
    o_d, l_d = sab.sageattn_qk_int8_pv_fp8_cuda(q, k, v, return_lse=True)
    for window in ((-1, -1), (300, 700)):
        o, l = sab.sageattn_window(q, k, v, window, return_lse=True)
        assert torch.equal(o, o_d) and torch.equal(l, l_d)


def _grads(fn, q, k, v, do):
    o = fn(q, k, v)
    return (o,) + torch.autograd.grad(o, (q, k, v), do)


@pytest.mark.parametrize("case", [(128, BF, "HND", "per_thread"), (64, FP, "NHD", "per_warp"), (96, BF, "NHD", "per_thread")])
def test_unbounded_window_gradients_are_the_dense_backward_bitwise(case):
    D, dt, lay, gran = case
    B, Hq, Hkv, S = 1, 4, 2, 320
    q, k, v = _qkv(B, Hq, Hkv, S, S, D, dt, lay, seed=5, grad=True)
    do = torch.randn_like(q)
    kw = dict(tensor_layout=lay, qk_quant_gran=gran)
    for causal, window in ((False, (-1, -1)), (False, (S, S)), (True, (-1, -1)), (True, (-1, 0))):
        a = _grads(lambda q, k, v: sab.sageattn_window(q, k, v, window, is_causal=causal, **kw), q, k, v, do)
        b = _grads(lambda q, k, v: sab.sageattn_qk_int8_pv_fp8_cuda(q, k, v, is_causal=causal, **kw), q, k, v, do)
        for x, y in zip(a, b):
            assert torch.equal(x, y), (causal, window)
    a = _grads(lambda q, k, v: sab.sageattn_window(q, k, v, (-1, 0), **kw), q, k, v, do)
    b = _grads(lambda q, k, v: sab.sageattn_qk_int8_pv_fp8_cuda(q, k, v, is_causal=True, **kw), q, k, v, do)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


# ------------------------------------------------------------------------------------------------ forward vs restatement / exact
def _operands(q, k, v, gran, layout="HND"):
    """The quantised operands sageattn_window computes (pv_accum_dtype "fp32+fp32": V range 448, no smoothing of V)."""
    km, q8, qs, k8, ks, _, _, _ = _quant_qk(q, k, "fp8", layout, gran, q.size(-1) ** -0.5, True, "cuda")
    v8, vs, _ = per_channel_fp8(v, tensor_layout=layout, scale_max=448.0, smooth_v=False)
    return km, q8, qs, k8, ks, v8, vs


WINDOWS = [(0, 0), (1, 0), (63, 64), (127, 0), (200, 37), (1000, -1), (-1, 100)]
SHAPES = [(1, 1), (64, 64), (65, 65), (127, 127), (129, 129), (384, 384), (300, 700), (700, 300), (129, 1), (1, 129)]


def _check_forward(Sq, Sk, window, causal, D, dt, gran, seed):
    B, Hq, Hkv = 1, 4, 2
    q, k, v = _qkv(B, Hq, Hkv, Sq, Sk, D, dt, seed=seed)
    o, lse = sab.sageattn_window(q, k, v, window, is_causal=causal, qk_quant_gran=gran, pv_accum_dtype="fp32+fp32",
                                 return_lse=True)
    em = window_mask(Sq, Sk, *window, is_causal=causal, device="cuda")
    rows = em.any(-1)
    assert torch.isfinite(o).all() and not torch.isnan(lse).any()
    assert torch.all(o[:, :, ~rows] == 0) and torch.all(torch.isneginf(lse[:, :, ~rows])) and torch.isfinite(lse[:, :, rows]).all()
    ref = _exact(q, k, v, em, D ** -0.5)
    wide = em.sum(-1) >= 128
    if wide.any():
        assert (o.double() - ref)[:, :, wide].abs().max().item() < TOL_EXACT
    # the restatement on the call's own quantised operands (the quantisers are deterministic); the op gives the public call's
    # output to the bit and the kernel's raw log2 lse, relative to the smoothed K as the restatement's is
    km, q8, qs, k8, ks, v8, vs = _operands(q, k, v, gran)
    o_op = torch.empty_like(q)
    l_raw = ops.qk_int8_sv_f8_attn_window(q8, k8, v8, o_op, qs, ks, vs, None, window[0], window[1], 1, int(causal), GRAN[gran],
                                          GRAN[gran], D ** -0.5, 0, 1)
    assert torch.equal(o_op, o)
    v8 = v8[..., :Sk].transpose(-1, -2)
    # every element within the restatement's bound (attn_window_oracle), the raw lse within its few fp32 ulps
    oc, lc, bd = attn_int8_fp8_window(*(t.cpu() for t in (q8, k8, v8, qs, ks, vs)), window=window, qk_quant_gran=gran,
                                      is_causal=causal, sm_scale=D ** -0.5, lazy_tau=4, out_dtype=dt, return_lse=True, bound=True)
    check_forward(f"{Sq}x{Sk} window {window} causal {causal}", o, l_raw, lc, bd)
    r = rows.expand_as(lse).cpu()
    assert torch.equal(torch.isneginf(l_raw.cpu()), ~r) and torch.equal(torch.isneginf(lc), ~r)


@pytest.mark.parametrize("window", WINDOWS)
@pytest.mark.parametrize("causal", [False, True])
def test_windows_against_restatement_and_exact(window, causal):
    for i, (Sq, Sk) in enumerate(SHAPES):
        if causal and Sq != Sk:
            continue
        D, dt, gran = ((128, FP, "per_thread"), (64, BF, "per_warp"))[i % 2]
        _check_forward(Sq, Sk, window, causal, D, dt, gran, seed=100 * i + window[0])


def test_rows_with_no_visible_key_get_zeros_and_minus_inf():
    """Sq > Skv: rows i > Skv - 1 + left see no key; with right = 0 and Sq < Skv the keys past the last row are never seen."""
    _check_forward(700, 100, (10, 5), False, 128, BF, "per_thread", seed=7)
    _check_forward(300, 64, (0, 0), False, 64, FP, "per_warp", seed=8)
    _check_forward(100, 700, (-1, 0), False, 128, FP, "per_warp", seed=9)


@pytest.mark.parametrize("window", [(10, 0), (10, 20), (70, 3), (130, 0)])
def test_bottom_rows_whose_window_starts_in_a_later_tile(window):
    """In each 128-row Q tile the bottom rows' windows start up to 127 keys after the top row's: those rows see nothing of the CTA's
    first tile(s) and must leave m and d there; with right = 0 the top rows see nothing of the last tiles either."""
    _check_forward(512, 512, window, False, 128, BF, "per_thread", seed=11)
    _check_forward(512, 512, window, True, 64, FP, "per_warp", seed=12)


def test_long_case_against_exact():
    B, Hq, Hkv, S, D = 1, 2, 1, 8192, 128
    q, k, v = _qkv(B, Hq, Hkv, S, S, D, BF, seed=13)
    for window, causal in (((1024, 0), True), ((300, 300), False), ((1000, -1), False)):
        o, lse = sab.sageattn_window(q, k, v, window, is_causal=causal, return_lse=True)
        assert torch.isfinite(o).all() and torch.isfinite(lse).all()
        for r0 in range(0, S, 2048):   # fp64 reference in row chunks
            em = window_mask(S, S, *window, is_causal=causal, device="cuda")[r0:r0 + 2048]
            ref = _exact(q[:, :, r0:r0 + 2048], k, v, em, D ** -0.5)
            wide = em.sum(-1) >= 128
            assert (o[:, :, r0:r0 + 2048].double() - ref)[:, :, wide].abs().max().item() < TOL_EXACT


# ------------------------------------------------------------------------------------------------ gradient kernels
# (D, dtype, gran, layout, causal, B, Hq, Hkv, Sq, Skv, window): every window dQ / dK/dV instantiation, GQA, ragged lengths
BWD_ORACLE_CASES = [
    (128, BF, "per_thread", "HND", False, 1, 4, 2, 300, 448, (63, 64)),
    (128, FP, "per_thread", "NHD", True, 1, 2, 2, 384, 384, (127, 0)),
    (128, BF, "per_warp", "NHD", True, 1, 4, 1, 333, 333, (10, 0)),
    (128, FP, "per_warp", "HND", False, 2, 2, 2, 200, 517, (0, 0)),
    (64, FP, "per_thread", "HND", True, 1, 4, 2, 320, 320, (200, 37)),
    (64, BF, "per_thread", "NHD", False, 1, 2, 2, 450, 190, (20, 5)),
    (64, BF, "per_warp", "HND", False, 1, 8, 2, 256, 385, (-1, 100)),
    (64, FP, "per_warp", "NHD", False, 2, 2, 1, 257, 257, (1000, -1)),
    (128, BF, "per_thread", "HND", False, 1, 2, 1, 129, 65, (1, 0)),
]


@pytest.mark.parametrize("case", BWD_ORACLE_CASES, ids=lambda c: "-".join(str(x).replace("torch.", "").replace(" ", "") for x in c))
def test_window_gradient_kernels_match_oracle(case):
    """The kernels against tests/attn_bwd_masked_oracle.attn_bwd_masked fed the window's element mask (ANDed with the causal mask),
    the kernels' own quantised operands and the forward kernel's LSE; NaN-filled outputs, so every element must be written."""
    D, dt, gran, layout, causal, B, Hq, Hkv, Sq, Sk, window = case
    lay = 1 if layout == "HND" else 0
    q, k, v = _qkv(B, Hq, Hkv, Sq, Sk, D, dt, layout, seed=Sq + Sk + D)
    do = torch.randn_like(q)
    km, q8, qs, k8, ks, v8, vs = _operands(q, k, v, gran, layout)
    o = torch.empty_like(q)
    lse = ops.qk_int8_sv_f8_attn_window(q8, k8, v8, o, qs, ks, vs, None, window[0], window[1], lay, int(causal), GRAN[gran],
                                        GRAN[gran], D ** -0.5, 0, 1)
    dq, dk, dv = (torch.full_like(t, float("nan")) for t in (q, k, v))
    ops.qk_int8_attn_bwd_window(q8, k8, qs, ks, q, k, v, o, do, lse, km, dq, dk, dv, window[0], window[1], lay, int(causal),
                                GRAN[gran], GRAN[gran], D ** -0.5, 0)
    dq2, dk2, dv2 = (torch.full_like(t, float("nan")) for t in (q, k, v))
    ops.qk_int8_attn_bwd_window(q8, k8, qs, ks, q, k, v, o, do, lse, km, dq2, dk2, dv2, window[0], window[1], lay, int(causal),
                                GRAN[gran], GRAN[gran], D ** -0.5, 0)
    assert torch.equal(dq, dq2) and torch.equal(dk, dk2) and torch.equal(dv, dv2)
    torch.cuda.synchronize()
    em = window_mask(Sq, Sk, *window, is_causal=causal)
    c = lambda x: _hnd(x, layout).cpu()
    *ref, bounds = attn_bwd_masked(c(q8), c(k8), qs.cpu(), ks.cpu(), c(q), c(k), c(v), c(o), c(do), lse.cpu(), em, q_gran=gran,
                                   k_gran=gran, sm_scale=D ** -0.5, k_mean=c(km), bound=True)
    res = {name: check_elementwise(name, x, r, b)
           for name, x, r, b in zip(("dq", "dk", "dv"), (c(dq), c(dk), c(dv)), ref, bounds[:3])}
    print(f"[oracle] {case}: " + ", ".join(f"{n} ratio {w:.3f} normwise {e:.2e}" for n, (w, e) in res.items()))
    assert torch.all(c(dq)[:, :, ~em.any(-1)] == 0)
    unseen = ~em.any(0)
    assert torch.all(c(dk)[:, :, unseen] == 0) and torch.all(c(dv)[:, :, unseen] == 0)


@pytest.mark.parametrize("causal", [False, True])
def test_window_gradients_against_exact_autograd(causal):
    B, Hq, Hkv, S, D = 1, 4, 2, 512, 64
    q, k, v = _qkv(B, Hq, Hkv, S, S, D, BF, seed=6, grad=True)
    do = torch.randn_like(q)
    window = (150, 40)
    o, dq, dk, dv = _grads(lambda q, k, v: sab.sageattn_window(q, k, v, window, is_causal=causal), q, k, v, do)
    em = window_mask(S, S, *window, is_causal=causal, device="cuda")
    qd, kd, vd = (t.detach().double().requires_grad_() for t in (q, k, v))
    ref = _exact(qd, kd, vd, em, D ** -0.5)
    gq, gk, gv = torch.autograd.grad(ref, (qd, kd, vd), do.double())
    for g_, r_ in ((dq, gq), (dk, gk), (dv, gv)):
        assert ((g_.double() - r_).norm() / r_.norm()).item() < 3e-2    # tests/test_gpu_backward.py's normwise gate
    assert not any(torch.isnan(t).any() for t in (o, dq, dk, dv))


# ------------------------------------------------------------------------------------------------ validation and torch.compile
def test_validation_raises_before_any_launch():
    q, k, v = _qkv(1, 2, 2, 256, 256, 64, FP)
    _, k2, v2 = _qkv(1, 2, 2, 384, 384, 64, FP)
    with pytest.raises(ValueError):
        sab.sageattn_window(q, k, v, (-2, 4))
    with pytest.raises(AssertionError):
        sab.sageattn_window(q, k2, v2, (4, 4), is_causal=True)
    with pytest.raises(AssertionError):
        sab.sageattn_window(q, k.float(), v, (4, 4))
    with pytest.raises(ValueError):
        sab.sageattn_window(q, k, v, (4, 4), pv_accum_dtype="fp16")
    o = torch.empty_like(q)
    km, q8, qs, k8, ks, v8, vs = _operands(q, k, v, "per_thread")
    with pytest.raises(ValueError):
        ops.qk_int8_sv_f8_attn_window(q8, k8, v8, o, qs, ks, vs, None, -3, 0, 1, 0, 3, 3, 0.125, 0, 0)


def test_compile_gives_the_eager_bits():
    B, H, S, D = 1, 2, 320, 64
    q, k, v = _qkv(B, H, H, S, S, D, FP, seed=8, grad=True)
    do = torch.randn_like(q)
    fn = lambda q, k, v: sab.sageattn_window(q, k, v, (70, 10))
    eager = _grads(fn, q, k, v, do)
    comp = _grads(torch.compile(fn, fullgraph=True), q, k, v, do)
    for x, y in zip(eager, comp):
        assert torch.equal(x, y)
