"""GPU tests (-m gpu) of sageattn_varlen_qk_int8_pv_fp8_cuda, whose contract is "the dense call, per sequence":
  1. the per-sequence quantisers (K mean, per-thread / per-warp INT8, per-channel FP8 V) equal, bit for bit, the dense quantisers
     run on each sequence alone, at edge lengths, with empty sequences on either side and with tests/quant_cases.py's ties and
     degenerate blocks in a non-first sequence;
  2. the forward's output and lse rows equal the one-sequence dense call bit for bit (both granularities, the three
     pv_accum_dtype, smooth_v, causal with Lq == Lk, Lq != Lk, GQA and MHA, lazy and exact running max); rows past
     cu_seqlens_q[-1] are not written; causal with Lq != Lk against the CPU oracle (tolerance 2e-2, as smoke());
  3. dq / dk / dv equal the dense backward of each one-sequence call bit for bit; against the fp64 gradient oracle; zero past the
     end and for the keys of a sequence without queries; reproducible; unchanged output under requires_grad; torch.compile;
  4. configs[3] (lengths 512..16384 shuffled with seed 0, Hq=32, Hkv=8, D=128, bf16): forward and backward bit for bit."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import quant_cases as QC

pytestmark = pytest.mark.gpu

BF, FP = torch.bfloat16, torch.float16
EDGE = [0, 1, 63, 64, 65, 127, 128, 129, 300]


def _cu(lens, dtype=torch.int32):
    return torch.tensor([0] + list(np.cumsum(lens)), dtype=dtype, device="cuda")


def _packed(lens_q, lens_k, Hq, Hkv, D, dt, seed, tail=0):
    """Packed q / k / v / do with a per-sequence K offset (so the per-sequence means differ) and `tail` extra tokens at the end."""
    g = torch.Generator().manual_seed(seed)
    Tq, Tk = sum(lens_q) + tail, sum(lens_k) + tail
    q = torch.randn(Tq, Hq, D, generator=g)
    k = torch.randn(Tk, Hkv, D, generator=g)
    off = 0
    for L in lens_k:
        k[off:off + L] += 3.0 * torch.randn(1, Hkv, D, generator=g)
        off += L
    v = torch.randn(Tk, Hkv, D, generator=g)
    do = torch.randn(Tq, Hq, D, generator=g)
    return tuple(t.to(dt).cuda() for t in (q, k, v, do))


def _same(a, b):
    """Bitwise equality (NaN included) of two tensors of one dtype."""
    iv = {1: torch.uint8, 2: torch.int16, 4: torch.int32}[a.element_size()]
    return a.shape == b.shape and torch.equal(a.contiguous().view(iv), b.contiguous().view(iv))


def _spans(lens):
    c = [0] + list(np.cumsum(lens))
    return [(int(c[i]), int(c[i + 1])) for i in range(len(lens))]


# ------------------------------------------------------------------------------------------------ 1. quantisers
def _check_quantisers(q, k, v, lens_q, lens_k, gran, smooth_v=True):
    import sageattention_b200 as sab
    from sageattention_b200 import quant as Q
    cu_q, cu_k = _cu(lens_q), _cu(lens_k)
    km = Q.k_mean_varlen(k, cu_k, max(max(lens_k), 1))
    q8, qs, cu_qs = Q.quant_q_int8_varlen(q, cu_q, max(max(lens_q), 1), gran)
    k8, ks, cu_ks = Q.quant_k_int8_varlen(k, km, cu_k, max(max(lens_k), 1), gran)
    for scale_max in (2.25, 448.0):
        v8, vs, vm, cu_pad = Q.per_channel_fp8_varlen_seq(v, cu_k, max(max(lens_k), 1), scale_max, smooth_v)
        for b, (s, e) in enumerate(_spans(lens_k)):
            if e == s:
                assert not vs[b].any() and (vm is None or not vm[b].any())
                continue
            dv8, dvs, dvm = sab.per_channel_fp8(v[s:e][None], "NHD", scale_max, smooth_v)
            c0 = int(cu_pad[b])
            assert torch.equal(v8[:, :, c0:c0 + dv8.size(-1)].view(torch.uint8), dv8[0].view(torch.uint8)), f"v_fp8 of sequence {b}"
            assert _same(vs[b], dvs[0]) and (vm is None or _same(vm[b], dvm[0])), f"v_scale / v_mean of sequence {b}"
    qmult, kmult = (4, 1) if gran == "per_warp" else (32, 4)
    for b, (s, e) in enumerate(_spans(lens_q)):
        if e == s:
            continue
        d8, ds = Q.quant_q_int8(q[s:e][None], gran, "NHD")
        assert torch.equal(q8[s:e], d8[0]), f"q_int8 of sequence {b}"
        r0 = int(cu_qs[b]) * qmult
        assert _same(qs[r0:r0 + ds.size(-1)], ds[0].t()), f"q_scale of sequence {b}"
    for b, (s, e) in enumerate(_spans(lens_k)):
        if e == s:
            assert not km[b].float().any()
            continue
        dkm = sab.k_mean(k[s:e][None], "NHD")
        assert _same(km[b], dkm.view(km[b].shape)), f"k_mean of sequence {b}"
        d8, ds = Q.quant_k_int8(k[s:e][None], dkm, gran, "NHD")
        assert torch.equal(k8[s:e], d8[0]), f"k_int8 of sequence {b}"
        r0 = int(cu_ks[b]) * kmult
        assert _same(ks[r0:r0 + ds.size(-1)], ds[0].t()), f"k_scale of sequence {b}"


@pytest.mark.parametrize("gran", ["per_thread", "per_warp"])
@pytest.mark.parametrize("dt", [FP, BF])
@pytest.mark.parametrize("D", [64, 96, 128])
def test_quantisers_bit_for_bit_per_sequence(gran, dt, D):
    lens_q = EDGE + [4096]
    lens_k = EDGE[::-1] + [4096]            # empty sequences on either side, in other positions
    q, k, v, _ = _packed(lens_q, lens_k, 4, 2, D, dt, seed=D + (dt == BF))
    if D == 96:                             # padded as the entry point pads it (core._pad_head_dim): 128 channels, last 32 zero
        q, k, v = (F.pad(t, (0, 32)) for t in (q, k, v))
    _check_quantisers(q, k, v, lens_q, lens_k, gran)


@pytest.mark.parametrize("gran", ["per_thread", "per_warp"])
@pytest.mark.parametrize("dt", [FP, BF])
def test_quantisers_on_quant_cases_in_a_later_sequence(gran, dt):
    """Rounding ties, degenerate and format-edge blocks (tests/quant_cases.py) as the second sequence of a packed batch."""
    D = 64
    g = torch.Generator().manual_seed(3)
    lead = torch.randn(77, 1, D, generator=g).to(dt)
    for name, (x, _) in QC.degenerate_qk_cases(dt, D).items():
        tie = QC.tie_block(dt, 64, D, k=-2)
        body = torch.cat([x, tie]).unsqueeze(1)                   # [192 + 64, 1, D]
        t = torch.cat([lead, body]).cuda()
        vv = torch.cat([lead, QC.degenerate_v(dt, body.size(0), D).unsqueeze(1)]).cuda()
        lens = [77, body.size(0)]
        _check_quantisers(t, t, vv, lens, lens, gran)


# ------------------------------------------------------------------------------------------------ 2. forward
def _dense_seq(q, k, v, s, e, sk, ek, **kw):
    import sageattention_b200 as sab
    return sab.sageattn_qk_int8_pv_fp8_cuda(q[s:e][None], k[sk:ek][None], v[sk:ek][None], tensor_layout="NHD", return_lse=True, **kw)


def _check_forward(q, k, v, lens_q, lens_k, cu_dtype=torch.int32, **kw):
    import sageattention_b200 as sab
    o, lse = sab.sageattn_varlen_qk_int8_pv_fp8_cuda(q, k, v, _cu(lens_q, cu_dtype), _cu(lens_k, cu_dtype), max(max(lens_q), 1),
                                                     max(max(lens_k), 1), return_lse=True, **kw)
    for b, ((s, e), (sk, ek)) in enumerate(zip(_spans(lens_q), _spans(lens_k))):
        if e == s:
            continue
        if ek == sk:
            assert not o[s:e].any() and torch.isneginf(lse[:, s:e]).all(), f"sequence {b} without keys"
            continue
        do, dl = _dense_seq(q, k, v, s, e, sk, ek, **kw)
        assert torch.equal(o[s:e], do[0]), f"output rows of sequence {b}"
        # the kernel's LSE is the dense call's to the bit; the K-mean correction q . km is another cuBLAS product (core.py,
        # _lse_correction_varlen): its fp32 sum may be taken in another order (each within D * 2^-24 * sum |q_d km_d| of the exact
        # one) before the rounding to the input dtype (one unit, <= eps * |q . km|), times sm_scale
        diff = (lse[:, s:e] - dl[0]).abs()
        if kw.get("smooth_k", True):
            sm = kw.get("sm_scale") or q.size(-1) ** -0.5
            import sageattention_b200 as sab
            qb = F.pad(q[s:e], (0, (-q.size(-1)) % 64)).float()
            kmb = sab.k_mean(F.pad(k[sk:ek], (0, (-k.size(-1)) % 64))[None], "NHD")[0, 0].float()
            prod = qb * kmb.repeat_interleave(q.size(1) // k.size(1), dim=0)
            corr, mag = prod.sum(-1).t(), prod.abs().sum(-1).t()                                 # [Hq, L]
            ulp = (torch.finfo(q.dtype).eps * corr.abs() + 2 * qb.size(-1) * 2.0 ** -24 * mag) * sm * 1.01 + 1e-6 * dl[0].abs()
            assert (diff <= ulp).all(), f"lse rows of sequence {b}"
        else:
            assert torch.equal(lse[:, s:e], dl[0]), f"lse rows of sequence {b}"
    return o, lse


FWD_CASES = [  # gran, pv_accum_dtype, smooth_v, causal, Hq, Hkv, D, dtype
    ("per_thread", "fp32+fp16", False, False, 32, 8, 128, BF),
    ("per_warp", "fp32+fp16", False, True, 32, 8, 128, FP),
    ("per_thread", "fp32+fp32", False, True, 4, 4, 64, FP),
    ("per_warp", "fp32+fp32", False, False, 4, 4, 64, BF),
    ("per_thread", "fp32", True, False, 8, 2, 96, BF),
    ("per_warp", "fp32", True, True, 8, 2, 128, FP),
    ("per_thread", "fp32", False, True, 32, 8, 64, BF),
    ("per_warp", "fp32", False, False, 8, 8, 96, FP),
    ("per_warp", "fp32+fp32", False, True, 4, 2, 64, FP),
    ("per_warp", "fp32", True, False, 8, 2, 128, BF),
    ("per_thread", "fp32+fp16", False, True, 4, 4, 128, FP),
]


@pytest.mark.parametrize("case", FWD_CASES)
def test_forward_bit_for_bit_per_sequence(case):
    gran, acc, smooth_v, causal, Hq, Hkv, D, dt = case
    lens_q = [129, 0, 64, 1, 300, 65, 127]
    lens_k = lens_q if causal else [64, 7, 0, 200, 129, 128, 1]
    q, k, v, _ = _packed(lens_q, lens_k, Hq, Hkv, D, dt, seed=Hq + D, tail=5)
    _check_forward(q, k, v, lens_q, lens_k, cu_dtype=torch.int64 if smooth_v else torch.int32, is_causal=causal, qk_quant_gran=gran,
                   pv_accum_dtype=acc, smooth_v=smooth_v)


@pytest.mark.parametrize("dt", [BF, FP])
def test_many_short_sequences_with_lse(dt):
    """A thousand short packed sequences (lengths 0..200): output rows bit for bit, lse within one unit of the correction per
    sequence.  The call's extra memory stays a small multiple of q (an [Hq,Tq,nseq] correction would be nseq/D = 7.8 times q
    here).  Prints the peak and the share of lse elements that differ from the dense call."""
    g = torch.Generator().manual_seed(5)
    lens_q = torch.randint(0, 201, (1000,), generator=g).tolist()
    lens_k = torch.randint(1, 201, (1000,), generator=g).tolist()
    q, k, v, _ = _packed(lens_q, lens_k, 8, 2, 128, dt, seed=6)
    import sageattention_b200 as sab
    cu_q, cu_k = _cu(lens_q), _cu(lens_k)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    o, lse = sab.sageattn_varlen_qk_int8_pv_fp8_cuda(q, k, v, cu_q, cu_k, 200, 200, qk_quant_gran="per_warp", return_lse=True)
    torch.cuda.synchronize()
    peak = (torch.cuda.max_memory_allocated() - base) / (q.numel() * q.element_size())
    assert peak < 4.0, f"peak extra memory {peak:.2f} x q"
    del o, lse
    o, lse = _check_forward(q, k, v, lens_q, lens_k, qk_quant_gran="per_warp")
    n_diff = 0
    for (s, e), (sk, ek) in zip(_spans(lens_q), _spans(lens_k)):
        if e > s:
            n_diff += int((lse[:, s:e] != _dense_seq(q, k, v, s, e, sk, ek, qk_quant_gran="per_warp")[1][0]).sum())
    print(f"[many short, {dt}] peak extra memory {peak:.2f} x q; lse elements differing from the dense call: {n_diff} of "
          f"{lse.numel()}")


def test_forward_exact_running_max_bit_for_bit():
    """SAB_ATTN_KERNEL=exact is read once per process: a subprocess runs both granularities, causal and not."""
    code = ("import sys; sys.path[:0] = [%r, %r]\n" % (os.path.dirname(os.path.abspath(__file__)),
                                                       os.path.dirname(os.path.dirname(os.path.abspath(__file__)))) +
            "import test_gpu_varlen_fp8 as T\n"
            "for gran, causal in (('per_thread', False), ('per_warp', True), ('per_thread', True)):\n"
            "    lq = [129, 0, 300, 64]; lk = lq if causal else [64, 200, 0, 129]\n"
            "    q, k, v, _ = T._packed(lq, lk, 8, 2, 128, T.BF, seed=4, tail=3)\n"
            "    q = 6.0 * q\n"
            "    T._check_forward(q, k, v, lq, lk, is_causal=causal, qk_quant_gran=gran)\n"
            "print('EXACT_OK')\n")
    env = dict(os.environ, SAB_ATTN_KERNEL="exact")
    p = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0 and "EXACT_OK" in p.stdout, p.stdout + p.stderr


def test_rows_past_the_end_keep_a_sentinel():
    from sageattention_b200 import ops, quant as Q
    from sageattention_b200._capi import SAB_GRAN_PER_THREAD
    lens = [100, 0, 200]
    q, k, v, _ = _packed(lens, lens, 4, 2, 128, BF, seed=9, tail=37)
    cu = _cu(lens)
    km = Q.k_mean_varlen(k, cu, 200)
    q8, qs, cqs = Q.quant_q_int8_varlen(q, cu, 200)
    k8, ks, cks = Q.quant_k_int8_varlen(k, km, cu, 200)
    v8, vs, vm, cu_pad = Q.per_channel_fp8_varlen_seq(v, cu, 200, 2.25)
    o = torch.full_like(q, 7.0)
    lse = ops.qk_int8_sv_f8_attn_varlen_seq(q8, k8, v8, o, qs, ks, vs, vm, cu, cu, cu_pad, cqs, cks, 200, 0, SAB_GRAN_PER_THREAD,
                                            SAB_GRAN_PER_THREAD, 128 ** -0.5, 1)
    assert (o[300:] == 7.0).all() and o[:300].ne(7.0).any()
    assert lse.shape == (4, q.size(0))


def test_causal_lq_ne_lk_against_oracle():
    import sageattention_b200 as sab
    from oracle import sage_oracle as O
    lens_q, lens_k = [100, 64, 1], [300, 64, 129]
    q, k, v, _ = _packed(lens_q, lens_k, 4, 2, 64, FP, seed=21)
    o = sab.sageattn_varlen_qk_int8_pv_fp8_cuda(q, k, v, _cu(lens_q), _cu(lens_k), 100, 300, is_causal=True)
    for (s, e), (sk, ek) in zip(_spans(lens_q), _spans(lens_k)):
        ref = O.sageattn_qk_int8_pv_fp8_cuda(q[s:e][None].cpu(), k[sk:ek][None].cpu(), v[sk:ek][None].cpu(), tensor_layout="NHD",
                                             is_causal=True, lazy_tau=4, emulate_f16_accum=False)
        err = (o[s:e].cpu().float() - ref[0].float()).abs().max().item()
        assert err < 2e-2, err


# ------------------------------------------------------------------------------------------------ 3. gradients
def _grads_varlen(q, k, v, do, lens_q, lens_k, **kw):
    import sageattention_b200 as sab
    qg, kg, vg = (t.clone().requires_grad_(True) for t in (q, k, v))
    o = sab.sageattn_varlen_qk_int8_pv_fp8_cuda(qg, kg, vg, _cu(lens_q), _cu(lens_k), max(lens_q), max(lens_k), **kw)
    o.backward(do)
    return o.detach(), qg.grad, kg.grad, vg.grad


BWD_CASES = [("per_thread", True, BF, 128), ("per_warp", False, FP, 64), ("per_thread", False, FP, 128), ("per_warp", True, BF, 96),
             ("per_warp", False, BF, 64), ("per_thread", True, FP, 64), ("per_thread", False, BF, 64), ("per_warp", True, FP, 128)]


@pytest.mark.parametrize("case", BWD_CASES)
def test_gradients_bit_for_bit_per_sequence(case):
    import sageattention_b200 as sab
    gran, causal, dt, D = case
    lens_q = [129, 300, 0, 64, 1]
    lens_k = lens_q if causal else [64, 129, 50, 0, 200]
    q, k, v, do = _packed(lens_q, lens_k, 8, 2, D, dt, seed=D + causal, tail=9)
    o, dq, dk, dv = _grads_varlen(q, k, v, do, lens_q, lens_k, is_causal=causal, qk_quant_gran=gran)
    for b, ((s, e), (sk, ek)) in enumerate(zip(_spans(lens_q), _spans(lens_k))):
        if e == s:
            assert not dk[sk:ek].any() and not dv[sk:ek].any(), f"keys of sequence {b} without queries"
            continue
        if ek == sk:
            assert not dq[s:e].any()
            continue
        qb, kb, vb = (t.clone().requires_grad_(True) for t in (q[s:e][None], k[sk:ek][None], v[sk:ek][None]))
        ob = sab.sageattn_qk_int8_pv_fp8_cuda(qb, kb, vb, tensor_layout="NHD", is_causal=causal, qk_quant_gran=gran)
        ob.backward(do[s:e][None])
        assert torch.equal(o[s:e], ob[0].detach()), f"output of sequence {b}"
        for name, got, ref in (("dq", dq[s:e], qb.grad[0]), ("dk", dk[sk:ek], kb.grad[0]), ("dv", dv[sk:ek], vb.grad[0])):
            assert torch.equal(got, ref), f"{name} of sequence {b}"
    Tq, Tk = sum(lens_q), sum(lens_k)
    assert not dq[Tq:].any() and not dk[Tk:].any() and not dv[Tk:].any()


def test_gradients_against_fp64_oracle():
    """One sequence of a packed batch against attn_bwd_oracle on the dense quantised operands of that sequence (which the
    quantiser tests show are the packed ones)."""
    import sageattention_b200 as sab
    from sageattention_b200 import ops
    from attn_bwd_oracle import attn_bwd, check_elementwise
    lens = [200, 129, 64]
    q, k, v, do = _packed(lens, lens, 8, 2, 128, BF, seed=33)
    o, dq, dk, dv = _grads_varlen(q, k, v, do, lens, lens, is_causal=True)
    s, e = 200, 329
    hnd = lambda t: t[s:e][None].transpose(1, 2).contiguous()
    km = sab.k_mean(k[s:e][None], "NHD")
    q8, qs, k8, ks = sab.per_thread_int8(q[s:e][None], k[s:e][None], km, tensor_layout="NHD")
    v8, vs, _ = sab.per_channel_fp8(v[s:e][None], "NHD", 2.25, False)
    ob = torch.empty_like(q[s:e][None])
    lse = ops.qk_int8_sv_f8_attn(q8, k8, v8, ob, qs, ks, vs, None, 0, 1, 3, 3, 128 ** -0.5, 0, 1)
    *ref, bounds = attn_bwd(q8.transpose(1, 2), k8.transpose(1, 2), qs, ks, hnd(q), hnd(k), hnd(v), hnd(o), hnd(do), lse,
                            q_gran="per_thread", is_causal=True, sm_scale=128 ** -0.5, k_mean=km.view(1, 2, 1, 128), bound=True)
    for name, got, r, bnd in zip(("dq", "dk", "dv"), (dq, dk, dv), ref, bounds):
        check_elementwise(name, hnd(got), r, bnd)


def test_gradients_reproducible_and_forward_unchanged_by_requires_grad():
    import sageattention_b200 as sab
    lens = [1000, 17, 0, 640]
    q, k, v, do = _packed(lens, lens, 8, 2, 128, BF, seed=7)
    runs = [_grads_varlen(q, k, v, do, lens, lens, is_causal=True) for _ in range(2)]
    for a, b in zip(*runs):
        assert torch.equal(a, b)
    o = sab.sageattn_varlen_qk_int8_pv_fp8_cuda(q, k, v, _cu(lens), _cu(lens), 1000, 1000, is_causal=True)
    assert torch.equal(o, runs[0][0])


def test_torch_compile_fullgraph_gives_eager_gradients():
    import sageattention_b200 as sab
    lens = [300, 64, 129]
    q, k, v, do = _packed(lens, lens, 2, 2, 64, FP, seed=11)
    cu = _cu(lens)

    def f(q, k, v):
        return sab.sageattn_varlen_qk_int8_pv_fp8_cuda(q, k, v, cu, cu, 300, 300, is_causal=True)

    eager = _grads_varlen(q, k, v, do, lens, lens, is_causal=True)
    cf = torch.compile(f, fullgraph=True)
    qg, kg, vg = (t.clone().requires_grad_(True) for t in (q, k, v))
    o = cf(qg, kg, vg)
    o.backward(do)
    for a, b in zip(eager, (o.detach(), qg.grad, kg.grad, vg.grad)):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------ 4. headline shape
def test_headline_shape_bit_for_bit():
    import sageattention_b200 as sab
    lens = [512, 1024, 2048, 4096, 8192, 16384]
    g = torch.Generator().manual_seed(0)
    lens = [lens[i] for i in torch.randperm(len(lens), generator=g).tolist()]
    q, k, v, do = _packed(lens, lens, 32, 8, 128, BF, seed=0)
    for causal in (False, True):
        _check_forward(q, k, v, lens, lens, is_causal=causal)
    o, dq, dk, dv = _grads_varlen(q, k, v, do, lens, lens, is_causal=True)
    for b, (s, e) in enumerate(_spans(lens)):
        qb, kb, vb = (t.clone().requires_grad_(True) for t in (q[s:e][None], k[s:e][None], v[s:e][None]))
        sab.sageattn_qk_int8_pv_fp8_cuda(qb, kb, vb, tensor_layout="NHD", is_causal=True).backward(do[s:e][None])
        for name, got, ref in (("dq", dq[s:e], qb.grad[0]), ("dk", dk[s:e], kb.grad[0]), ("dv", dv[s:e], vb.grad[0])):
            assert torch.equal(got, ref), f"{name} of sequence {b} (L={e - s})"
