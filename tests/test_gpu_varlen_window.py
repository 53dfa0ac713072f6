"""GPU tests (-m gpu) of sageattn_varlen_window, whose contract is "sageattn_window, per sequence":
  1. each sequence's output rows are the bits of sageattn_window on that sequence alone, and its lse rows within the varlen FP8
     test's bound (both granularities, fp16 / bf16, D 64 / 96 / 128, the three pv_accum_dtype with smooth_v, causal and not, GQA
     and MHA, int32 / int64 cu_seqlens, edge lengths with empty sequences and Lq != Lk, windows whose sides fall between a
     sequence's length and max_seqlen); rows with no visible key give 0 and lse -inf; lazy and exact running max;
  2. causal with Lq != Lk gives the bits of sageattn_window(..., (left, 0), is_causal=False), forward and gradients;
  3. identities on o, lse, dq, dk, dv: (-1, -1) is sageattn_varlen_qk_int8_pv_fp8_cuda, (-1, 0) non-causal its causal call;
  4. no leakage: large K / V in the neighbouring sequences change no bit of a sequence; rows past the end keep a sentinel;
  5. dq / dk / dv are the bits of the dense window backward of each one-sequence call; zero past the end, for the keys of a
     sequence without queries and for keys outside every window; reproducible; the forward is unchanged by requires_grad;
     torch.compile(fullgraph=True) gives the eager bits;
  6. the bench lengths (2048 .. 16384, Hq=32, Hkv=8, D=128, bf16) with a causal (4096, 0) window, forward and backward."""
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

from attn_window_oracle import window_mask
from test_gpu_varlen_fp8 import BF, FP, _cu, _packed, _spans

pytestmark = pytest.mark.gpu

WINDOWS = [(0, 0), (1, 0), (63, 64), (127, 0), (200, 37), (1000, -1), (-1, 100)]
# sides between some sequences' lengths and max_seqlen (300): the per-sequence clamp decides their masked tiles
CLAMP_WINDOWS = [(100, 150), (250, 70), (129, 128)]
LENS_Q = [129, 0, 64, 1, 300, 65, 127, 63, 128]
LENS_K = [64, 7, 0, 200, 129, 128, 1, 300, 63]


def _dense(q, k, v, s, e, sk, ek, window, causal, **kw):
    import sageattention_b200 as sab
    return sab.sageattn_window(q[s:e][None], k[sk:ek][None], v[sk:ek][None], window, tensor_layout="NHD", is_causal=causal,
                               return_lse=True, **kw)


def _lse_bound(q, k, s, e, sk, ek, dl, **kw):
    """The varlen FP8 test's bound on lse - dense lse: one unit of the rounded K-mean correction plus its fp32 summation-order
    term, times sm_scale (the kernel LSE itself is exact; see _lse_correction_varlen)."""
    import sageattention_b200 as sab
    if not kw.get("smooth_k", True):
        return torch.zeros_like(dl)
    sm = kw.get("sm_scale") or q.size(-1) ** -0.5
    qb = F.pad(q[s:e], (0, (-q.size(-1)) % 64)).float()
    kmb = sab.k_mean(F.pad(k[sk:ek], (0, (-k.size(-1)) % 64))[None], "NHD")[0, 0].float()
    prod = qb * kmb.repeat_interleave(q.size(1) // k.size(1), dim=0)
    corr, mag = prod.sum(-1).t(), prod.abs().sum(-1).t()
    return (torch.finfo(q.dtype).eps * corr.abs() + 2 * qb.size(-1) * 2.0 ** -24 * mag) * sm * 1.01 + 1e-6 * dl.abs()


def _check_forward(q, k, v, lens_q, lens_k, window, causal, cu_dtype=torch.int32, **kw):
    """The packed call against sageattn_window per sequence: output bits, lse within _lse_bound (-inf where a row sees no key).
    Causal sequences with Lq != Lk are compared with non-causal (left, 0)."""
    import sageattention_b200 as sab
    o, lse = sab.sageattn_varlen_window(q, k, v, _cu(lens_q, cu_dtype), _cu(lens_k, cu_dtype), max(max(lens_q), 1), max(max(lens_k), 1),
                                        window, is_causal=causal, return_lse=True, **kw)
    for b, ((s, e), (sk, ek)) in enumerate(zip(_spans(lens_q), _spans(lens_k))):
        if e == s:
            continue
        rows = window_mask(e - s, ek - sk, *window, is_causal=causal, device="cuda").any(-1)
        assert not o[s:e][~rows].any() and torch.isneginf(lse[:, s:e][:, ~rows]).all(), f"rows of sequence {b} with no visible key"
        if ek == sk:
            continue
        w, c = ((window[0], 0), False) if causal and e - s != ek - sk else (window, causal)
        do, dl = _dense(q, k, v, s, e, sk, ek, w, c, **kw)
        assert torch.equal(o[s:e], do[0]), f"output rows of sequence {b}, window {window}"
        assert torch.equal(torch.isneginf(lse[:, s:e]), torch.isneginf(dl[0])), f"lse -inf of sequence {b}"
        fin = torch.isfinite(dl[0])
        assert ((lse[:, s:e] - dl[0]).abs()[fin] <= _lse_bound(q, k, s, e, sk, ek, dl[0], **kw)[fin]).all(), f"lse rows of sequence {b}"
    return o, lse


FWD_CASES = [  # gran, pv_accum_dtype, smooth_v, causal, Hq, Hkv, D, dtype, cu dtype
    ("per_thread", "fp32+fp16", False, False, 8, 2, 128, BF, torch.int32),
    ("per_warp", "fp32+fp16", False, True, 8, 2, 128, FP, torch.int64),
    ("per_thread", "fp32+fp32", False, True, 4, 4, 64, FP, torch.int32),
    ("per_warp", "fp32+fp32", False, False, 4, 4, 64, BF, torch.int64),
    ("per_thread", "fp32", True, False, 8, 2, 96, BF, torch.int64),
    ("per_warp", "fp32", True, True, 8, 2, 128, FP, torch.int32),
    ("per_thread", "fp32", False, True, 8, 2, 64, BF, torch.int32),
    ("per_warp", "fp32", False, False, 8, 8, 96, FP, torch.int32),
    ("per_warp", "fp32+fp32", False, True, 4, 2, 64, FP, torch.int64),
    ("per_warp", "fp32", True, False, 8, 2, 128, BF, torch.int32),
    ("per_thread", "fp32+fp16", False, True, 4, 4, 128, FP, torch.int64),
]


@pytest.mark.parametrize("case", FWD_CASES, ids=lambda c: "-".join(str(x).replace("torch.", "") for x in c))
def test_forward_bit_for_bit_per_sequence(case):
    gran, acc, smooth_v, causal, Hq, Hkv, D, dt, cu_dtype = case
    lens_k = LENS_Q if causal else LENS_K
    q, k, v, _ = _packed(LENS_Q, lens_k, Hq, Hkv, D, dt, seed=Hq + D, tail=5)
    for window in WINDOWS + CLAMP_WINDOWS:
        _check_forward(q, k, v, LENS_Q, lens_k, window, causal, cu_dtype, qk_quant_gran=gran, pv_accum_dtype=acc, smooth_v=smooth_v)


def test_causal_with_unequal_lengths_is_noncausal_right_0():
    """sageattn_window refuses causal with Lq != Lk; the packed call runs it top-left, which is non-causal (left, 0) to the bit."""
    lens_q, lens_k = [100, 64, 1, 300, 0, 129], [300, 64, 129, 50, 10, 1]
    q, k, v, _ = _packed(lens_q, lens_k, 8, 2, 128, BF, seed=21)
    for window in [(0, 0), (10, 5), (127, -1), (-1, -1), (200, 37), (63, 64)]:
        _check_forward(q, k, v, lens_q, lens_k, window, True)


def test_forward_exact_running_max_bit_for_bit():
    """SAB_ATTN_KERNEL=exact is read once per process: a subprocess runs both granularities, causal and not."""
    code = ("import sys; sys.path[:0] = [%r, %r]\n" % (os.path.dirname(os.path.abspath(__file__)),
                                                       os.path.dirname(os.path.dirname(os.path.abspath(__file__)))) +
            "import test_gpu_varlen_window as T\n"
            "for gran, causal in (('per_thread', False), ('per_warp', True), ('per_thread', True)):\n"
            "    lq = [129, 0, 300, 64]; lk = lq if causal else [64, 200, 0, 129]\n"
            "    q, k, v, _ = T._packed(lq, lk, 8, 2, 128, T.BF, seed=4, tail=3)\n"
            "    q = 6.0 * q\n"
            "    for w in ((70, 3), (200, 37), (-1, 0)):\n"
            "        T._check_forward(q, k, v, lq, lk, w, causal, qk_quant_gran=gran)\n"
            "print('EXACT_OK')\n")
    env = dict(os.environ, SAB_ATTN_KERNEL="exact")
    p = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0 and "EXACT_OK" in p.stdout, p.stdout + p.stderr


# ------------------------------------------------------------------------------------------------ identities, leakage, sentinels
def _grads(fn, q, k, v, do):
    """(o, lse or None, dq, dk, dv) of fn, which returns o or (o, lse)."""
    qg, kg, vg = (t.clone().requires_grad_(True) for t in (q, k, v))
    out = fn(qg, kg, vg)
    o, lse = out if isinstance(out, tuple) else (out, None)
    o.backward(do)
    return o.detach(), lse, qg.grad, kg.grad, vg.grad


@pytest.mark.parametrize("gran, dt, D", [("per_thread", BF, 128), ("per_warp", FP, 64)])
def test_unbounded_windows_are_the_packed_calls_bitwise(gran, dt, D):
    import sageattention_b200 as sab
    lens_q, lens_k = [129, 300, 0, 64, 1], [64, 129, 50, 0, 200]
    q, k, v, do = _packed(lens_q, lens_k, 8, 2, D, dt, seed=D, tail=7)
    cq, ck = _cu(lens_q), _cu(lens_k)
    kw = dict(qk_quant_gran=gran, return_lse=True)
    for causal, window, ref_causal in ((False, (-1, -1), False), (True, (-1, -1), True), (False, (-1, 0), True),
                                       (False, (300, 200), False), (True, (300, -1), True)):
        a = _grads(lambda q, k, v: sab.sageattn_varlen_window(q, k, v, cq, ck, 300, 200, window, is_causal=causal, **kw), q, k, v, do)
        b = _grads(lambda q, k, v: sab.sageattn_varlen_qk_int8_pv_fp8_cuda(q, k, v, cq, ck, 300, 200, is_causal=ref_causal, **kw),
                   q, k, v, do)
        Tq = sum(lens_q)     # o / lse rows past the end are not written
        for name, x, y in zip(("o", "lse", "dq", "dk", "dv"), (a[0][:Tq], a[1][:, :Tq]) + a[2:], (b[0][:Tq], b[1][:, :Tq]) + b[2:]):
            assert torch.equal(x, y), (causal, window, name)


def test_no_leakage_across_sequences():
    import sageattention_b200 as sab
    lens = [200, 129, 300, 64]
    q, k, v, _ = _packed(lens, lens, 8, 2, 128, BF, seed=3)
    cu = _cu(lens)
    spans = _spans(lens)
    for causal, window in ((False, (1000, -1)), (True, (-1, -1)), (False, (63, 64))):
        o, lse = sab.sageattn_varlen_window(q, k, v, cu, cu, 300, 300, window, is_causal=causal, return_lse=True)
        for b, (s, e) in enumerate(spans):
            k2, v2 = k.clone(), v.clone()
            for c, (s2, e2) in enumerate(spans):
                if c != b:
                    k2[s2:e2] = 200.0 * torch.randn_like(k2[s2:e2])
                    v2[s2:e2] = -300.0
            o2, lse2 = sab.sageattn_varlen_window(q, k2, v2, cu, cu, 300, 300, window, is_causal=causal, return_lse=True)
            assert torch.equal(o2[s:e], o[s:e]) and torch.equal(lse2[:, s:e], lse[:, s:e]), (b, window)


def test_rows_past_the_end_keep_a_sentinel():
    from sageattention_b200 import ops, quant as Q
    from sageattention_b200._capi import SAB_GRAN_PER_THREAD as PT
    lens = [100, 0, 200]
    q, k, v, _ = _packed(lens, lens, 4, 2, 128, BF, seed=9, tail=37)
    cu = _cu(lens)
    km = Q.k_mean_varlen(k, cu, 200)
    q8, qs, cqs = Q.quant_q_int8_varlen(q, cu, 200)
    k8, ks, cks = Q.quant_k_int8_varlen(k, km, cu, 200)
    v8, vs, vm, cu_pad = Q.per_channel_fp8_varlen_seq(v, cu, 200, 2.25)
    for window in ((0, 0), (50, 3), (-1, -1)):
        o = torch.full_like(q, 7.0)
        lse = ops.qk_int8_sv_f8_attn_varlen_window(q8, k8, v8, o, qs, ks, vs, vm, cu, cu, cu_pad, cqs, cks, 200, window[0], window[1],
                                                   0, PT, PT, 128 ** -0.5, 1)
        assert (o[300:] == 7.0).all() and not (o[:300] == 7.0).all(-1).any()
        assert lse.shape == (4, q.size(0)) and torch.isfinite(lse[:, :300]).all()


def test_rows_without_a_visible_key_give_zero_and_minus_inf():
    """Lq > Lk with a narrow window: rows i > Lk - 1 + left see nothing; the dense rule, per sequence."""
    import sageattention_b200 as sab
    lens_q, lens_k = [300, 129, 64], [100, 1, 200]
    q, k, v, _ = _packed(lens_q, lens_k, 4, 2, 64, FP, seed=12)
    for window in ((10, 5), (0, 0), (3, -1)):
        o, lse = _check_forward(q, k, v, lens_q, lens_k, window, False)
        assert torch.isneginf(lse).any() and torch.isfinite(lse).any()


# ------------------------------------------------------------------------------------------------ gradients
BWD_CASES = [  # gran, causal, dtype, D, window
    ("per_thread", True, BF, 128, (127, 0)),
    ("per_warp", False, FP, 64, (63, 64)),
    ("per_thread", False, FP, 128, (200, 37)),
    ("per_warp", True, BF, 96, (10, 0)),
    ("per_thread", False, BF, 64, (1000, -1)),
    ("per_warp", False, BF, 128, (-1, 100)),
    ("per_thread", True, FP, 64, (100, 150)),
    ("per_warp", False, BF, 64, (0, 0)),
    ("per_warp", True, FP, 128, (130, 0)),
]


@pytest.mark.parametrize("case", BWD_CASES, ids=lambda c: "-".join(str(x).replace("torch.", "").replace(" ", "") for x in c))
def test_gradients_bit_for_bit_per_sequence(case):
    import sageattention_b200 as sab
    gran, causal, dt, D, window = case
    lens_q = [129, 300, 0, 64, 1, 65]
    lens_k = lens_q if causal else [64, 129, 50, 0, 200, 300]
    q, k, v, do = _packed(lens_q, lens_k, 8, 2, D, dt, seed=D + causal, tail=9)
    cq, ck = _cu(lens_q), _cu(lens_k)
    fn = lambda q, k, v: sab.sageattn_varlen_window(q, k, v, cq, ck, 300, 300, window, is_causal=causal, qk_quant_gran=gran,
                                                    return_lse=True)
    Tq, Tk = sum(lens_q), sum(lens_k)
    o, _, dq, dk, dv = _grads(fn, q, k, v, do)
    again = _grads(fn, q, k, v, do)
    assert all(torch.equal(x, y) for x, y in zip((o[:Tq], dq, dk, dv), (again[0][:Tq],) + again[2:])), "run to run"
    for b, ((s, e), (sk, ek)) in enumerate(zip(_spans(lens_q), _spans(lens_k))):
        if e == s:
            assert not dk[sk:ek].any() and not dv[sk:ek].any(), f"keys of sequence {b} without queries"
            continue
        if ek == sk:
            assert not dq[s:e].any()
            continue
        em = window_mask(e - s, ek - sk, *window, is_causal=causal, device="cuda")
        unseen = ~em.any(0)
        assert not dk[sk:ek][unseen].any() and not dv[sk:ek][unseen].any(), f"keys of sequence {b} outside every window"
        assert not dq[s:e][~em.any(-1)].any()
        qb, kb, vb = (t.clone().requires_grad_(True) for t in (q[s:e][None], k[sk:ek][None], v[sk:ek][None]))
        ob = sab.sageattn_window(qb, kb, vb, window, tensor_layout="NHD", is_causal=causal, qk_quant_gran=gran)
        ob.backward(do[s:e][None])
        assert torch.equal(o[s:e], ob[0].detach()), f"output of sequence {b}"
        for name, got, ref in (("dq", dq[s:e], qb.grad[0]), ("dk", dk[sk:ek], kb.grad[0]), ("dv", dv[sk:ek], vb.grad[0])):
            assert torch.equal(got, ref), f"{name} of sequence {b}"
    assert not dq[Tq:].any() and not dk[Tk:].any() and not dv[Tk:].any()
    # the forward gives the same bits whether or not the inputs require grad (rows past the end are not written)
    o_plain = sab.sageattn_varlen_window(q, k, v, cq, ck, 300, 300, window, is_causal=causal, qk_quant_gran=gran)
    assert torch.equal(o_plain[:Tq], o[:Tq])


def test_causal_gradients_with_unequal_lengths_are_noncausal_right_0():
    import sageattention_b200 as sab
    lens_q, lens_k = [100, 300, 64], [300, 50, 129]
    q, k, v, do = _packed(lens_q, lens_k, 8, 2, 128, BF, seed=17, tail=3)
    cq, ck = _cu(lens_q), _cu(lens_k)
    for window in ((31, 7), (-1, -1)):
        _, _, dq, dk, dv = _grads(lambda q, k, v: sab.sageattn_varlen_window(q, k, v, cq, ck, 300, 300, window, is_causal=True,
                                                                              return_lse=True), q, k, v, do)
        for (s, e), (sk, ek) in zip(_spans(lens_q), _spans(lens_k)):
            qb, kb, vb = (t.clone().requires_grad_(True) for t in (q[s:e][None], k[sk:ek][None], v[sk:ek][None]))
            sab.sageattn_window(qb, kb, vb, (window[0], 0), tensor_layout="NHD").backward(do[s:e][None])
            assert torch.equal(dq[s:e], qb.grad[0]) and torch.equal(dk[sk:ek], kb.grad[0]) and torch.equal(dv[sk:ek], vb.grad[0])


def test_torch_compile_fullgraph_gives_eager_bits():
    import sageattention_b200 as sab
    lens = [300, 64, 129]
    q, k, v, do = _packed(lens, lens, 2, 2, 64, FP, seed=11)
    cu = _cu(lens)

    def f(q, k, v):
        return sab.sageattn_varlen_window(q, k, v, cu, cu, 300, 300, (70, 10), is_causal=True)

    eager = _grads(f, q, k, v, do)
    comp = _grads(torch.compile(f, fullgraph=True), q, k, v, do)
    for i in (0, 2, 3, 4):
        assert torch.equal(eager[i], comp[i])


# ------------------------------------------------------------------------------------------------ long case
def test_bench_lengths_causal_4096_bit_for_bit():
    import sageattention_b200 as sab
    lens = [2048, 16384, 4096, 512, 1024, 8192]
    q, k, v, do = _packed(lens, lens, 32, 8, 128, BF, seed=0)
    cu = _cu(lens)
    window = (4096, 0)
    o, _, dq, dk, dv = _grads(lambda q, k, v: sab.sageattn_varlen_window(q, k, v, cu, cu, 16384, 16384, window, is_causal=True,
                                                                          return_lse=True), q, k, v, do)
    for b, (s, e) in enumerate(_spans(lens)):
        qb, kb, vb = (t.clone().requires_grad_(True) for t in (q[s:e][None], k[s:e][None], v[s:e][None]))
        ob = sab.sageattn_window(qb, kb, vb, window, tensor_layout="NHD", is_causal=True)
        ob.backward(do[s:e][None])
        assert torch.equal(o[s:e], ob[0].detach()), f"output of sequence {b} (L={e - s})"
        for name, got, ref in (("dq", dq[s:e], qb.grad[0]), ("dk", dk[s:e], kb.grad[0]), ("dv", dv[s:e], vb.grad[0])):
            assert torch.equal(got, ref), f"{name} of sequence {b} (L={e - s})"
