"""GPU tests (-m gpu) of sageattn_varlen_blocksparse, whose contract is "sageattn_blocksparse, per sequence", and of
predict_block_mask_varlen, whose contract is "predict_block_mask, per sequence":
  1. each sequence's output rows are the bits of sageattn_blocksparse on its own mask slice, and its lse rows within the varlen
     FP8 test's bound (both granularities, fp16 / bf16, D 64 / 96 / 128, the three pv_accum_dtype with smooth_v, causal with
     Lq == Lk and not, GQA and MHA, int32 / int64 cu_seqlens, edge lengths with empty sequences and Lq != Lk; random masks of
     several densities, all-False rows, broadcast and non-contiguous masks); lazy and exact running max;
  2. mask entries outside every sequence's tiles are never read: random bits there change no output bit;
  3. identities on o, lse, dq, dk, dv: an all-True mask is sageattn_varlen_qk_int8_pv_fp8_cuda, causal with Lq != Lk included;
  4. causal with Lq != Lk under a sparse mask against exact attention with the expanded element mask; rows with no visible key
     give 0 and lse -inf;
  5. no leakage: large K / V in the neighbouring sequences change no bit of a sequence; rows past the end keep a sentinel;
  6. dq / dk / dv are the bits of the dense block-sparse backward of each one-sequence call; zero past the end, for the keys of a
     sequence without queries and for keys hidden from every row; reproducible; the forward is unchanged by requires_grad;
     torch.compile(fullgraph=True) gives the eager bits;
  7. the packed predictor: each slice is the bits of the dense predict_block_mask, entries outside are False; causal with
     Lq != Lk against the fp64 restatement (near-threshold rows counted, not compared); packed prediction plus packed call is the
     dense prediction plus the dense call, per sequence;
  8. the bench lengths (512 .. 16384, Hq=32, Hkv=8, D=128, bf16) with a density-0.25 mask: three sequences, forward and backward."""
import math
import os
import subprocess
import sys
import warnings

import pytest
import torch

from attn_blocksparse_oracle import expand_block_mask
from block_predict_oracle import select
from test_gpu_varlen_fp8 import BF, FP, _cu, _packed, _spans
from test_gpu_varlen_window import _grads, _lse_bound

pytestmark = pytest.mark.gpu

TOL_EXACT = 6e-2      # max-abs against exact attention (tests/test_gpu_blocksparse.py)
EPS = 1e-5            # near-threshold allowance of the predictor (tests/test_gpu_block_predict.py)
LENS_Q = [129, 0, 64, 1, 300, 65, 127, 63, 128]
LENS_K = [64, 7, 0, 200, 129, 128, 1, 300, 63]


def _nb(L, blk):
    return (L + blk - 1) // blk


def _mask(nseq, Hq, max_q, max_k, p, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.rand(nseq, Hq, _nb(max_q, 128), _nb(max_k, 64), generator=g, device="cuda") < p


def _max(lens):
    return max(max(lens), 1)


def _check_forward(q, k, v, lens_q, lens_k, bm, causal, cu_dtype=torch.int32, **kw):
    """The packed call against sageattn_blocksparse per sequence: output bits and lse within _lse_bound.  Sequences the dense
    call refuses (causal with Lq != Lk) are checked against exact attention instead."""
    import sageattention_b200 as sab
    o, lse = sab.sageattn_varlen_blocksparse(q, k, v, _cu(lens_q, cu_dtype), _cu(lens_k, cu_dtype), _max(lens_q), _max(lens_k), bm,
                                             is_causal=causal, return_lse=True, **kw)
    bmx = bm.expand(len(lens_q), q.size(1), *bm.shape[2:])
    for b, ((s, e), (sk, ek)) in enumerate(zip(_spans(lens_q), _spans(lens_k))):
        if e == s:
            continue
        if ek == sk:
            assert not o[s:e].any() and torch.isneginf(lse[:, s:e]).all(), f"sequence {b} without keys"
            continue
        mb = bmx[b, :, :_nb(e - s, 128), :_nb(ek - sk, 64)]
        if causal and e - s != ek - sk:
            _check_exact(q[s:e], k[sk:ek], v[sk:ek], mb, o[s:e], lse[:, s:e], **kw)
            continue
        do, dl = sab.sageattn_blocksparse(q[s:e][None], k[sk:ek][None], v[sk:ek][None], mb[None], tensor_layout="NHD",
                                          is_causal=causal, return_lse=True, **kw)
        assert torch.equal(o[s:e], do[0]), f"output rows of sequence {b}"
        assert torch.equal(torch.isneginf(lse[:, s:e]), torch.isneginf(dl[0])), f"lse -inf of sequence {b}"
        fin = torch.isfinite(dl[0])
        assert ((lse[:, s:e] - dl[0]).abs()[fin] <= _lse_bound(q, k, s, e, sk, ek, dl[0], **kw)[fin]).all(), f"lse rows of sequence {b}"
    return o, lse


def _check_exact(qb, kb, vb, mb, ob, lb, **kw):
    """One sequence, causal top-left with Lq != Lk: exact attention with the expanded element mask and j <= i."""
    Lq, Lk, Hq = qb.size(0), kb.size(0), qb.size(1)
    em = expand_block_mask(mb[None], Lq, Lk)[0] & torch.ones(Lq, Lk, dtype=torch.bool, device="cuda").tril()
    g = Hq // kb.size(1)
    sm = kw.get("sm_scale") or qb.size(-1) ** -0.5
    s = torch.einsum("qhd,khd->hqk", qb.double(), kb.double().repeat_interleave(g, 1)) * sm
    p = torch.softmax(s.masked_fill(~em, -math.inf), -1).nan_to_num(0.0)
    ref = torch.einsum("hqk,khd->qhd", p, vb.double().repeat_interleave(g, 1))
    rows = em.any(-1)                                   # [Hq, Lq]
    wide = (em.sum(-1) >= 64).t()                       # [Lq, Hq]
    if wide.any():   # rows that see a handful of keys carry the e4m3 rounding of single V rows (tests/test_gpu_blocksparse.py)
        assert (ob.double() - ref)[wide].abs().max().item() < TOL_EXACT
    assert not ob.transpose(0, 1)[~rows].any() and torch.isneginf(lb[~rows]).all(), "rows with no visible key"


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
    nseq, mq, mk = len(LENS_Q), _max(LENS_Q), _max(lens_k)
    masks = [_mask(nseq, Hq, mq, mk, p, seed=i) for i, p in enumerate((1.0, 0.5, 0.25, 0.1))]
    rows_off = _mask(nseq, Hq, mq, mk, 0.6, seed=9)
    rows_off[:, :, 1] = False                                              # all-False rows
    masks += [rows_off, _mask(1, 1, mq, mk, 0.5, seed=5), _mask(nseq, 1, mq, mk, 0.4, seed=6)]   # broadcast [1,1] and [nseq,1]
    wide = _mask(nseq, Hq, mq, 2 * mk, 0.5, seed=7)
    masks.append(wide[..., ::2])                                           # non-contiguous
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")      # smooth_v with a non-"fp32" pv_accum_dtype warns, in both calls
        for bm in masks:
            _check_forward(q, k, v, LENS_Q, lens_k, bm, causal, cu_dtype, qk_quant_gran=gran, pv_accum_dtype=acc, smooth_v=smooth_v)


def test_forward_exact_running_max_bit_for_bit():
    """SAB_ATTN_KERNEL=exact is read once per process: a subprocess runs both granularities, causal and not."""
    code = ("import sys; sys.path[:0] = [%r, %r]\n" % (os.path.dirname(os.path.abspath(__file__)),
                                                       os.path.dirname(os.path.dirname(os.path.abspath(__file__)))) +
            "import test_gpu_varlen_blocksparse as T\n"
            "for gran, causal in (('per_thread', False), ('per_warp', True), ('per_thread', True)):\n"
            "    lq = [129, 0, 300, 64]; lk = lq if causal else [64, 200, 0, 129]\n"
            "    q, k, v, _ = T._packed(lq, lk, 8, 2, 128, T.BF, seed=4, tail=3)\n"
            "    q = 6.0 * q\n"
            "    for p in (1.0, 0.3):\n"
            "        T._check_forward(q, k, v, lq, lk, T._mask(4, 8, 300, 300 if causal else 200, p, 1), causal, qk_quant_gran=gran)\n"
            "print('EXACT_OK')\n")
    env = dict(os.environ, SAB_ATTN_KERNEL="exact")
    p = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0 and "EXACT_OK" in p.stdout, p.stdout + p.stderr


def test_padding_entries_are_ignored():
    """Every entry outside the sequences' own tiles set to random bits: no output bit changes, forward or gradient."""
    import sageattention_b200 as sab
    lens_q = [129, 0, 300, 64, 1]
    for causal, lens_k in ((False, [64, 129, 50, 0, 200]), (True, lens_q)):
        q, k, v, do = _packed(lens_q, lens_k, 8, 2, 128, BF, seed=2, tail=4)
        cq, ck, mk = _cu(lens_q), _cu(lens_k), _max(lens_k)
        bm = _mask(5, 8, 300, mk, 0.5, seed=3)
        inside = torch.zeros_like(bm)
        for b, (lq, lk) in enumerate(zip(lens_q, lens_k)):
            inside[b, :, :_nb(lq, 128), :_nb(lk, 64)] = True
        noisy = torch.where(inside, bm, _mask(5, 8, 300, mk, 0.5, seed=4))
        outs = [_grads(lambda q, k, v: sab.sageattn_varlen_blocksparse(q, k, v, cq, ck, 300, mk, m, is_causal=causal, return_lse=True),
                       q, k, v, do) for m in (noisy, bm & inside)]
        Tq = sum(lens_q)
        for name, x, y in zip(("o", "lse", "dq", "dk", "dv"), (outs[0][0][:Tq], outs[0][1][:, :Tq]) + outs[0][2:],
                              (outs[1][0][:Tq], outs[1][1][:, :Tq]) + outs[1][2:]):
            assert torch.equal(x, y), (causal, name)


# ------------------------------------------------------------------------------------------------ identities, causal Lq != Lk
@pytest.mark.parametrize("gran, dt, D", [("per_thread", BF, 128), ("per_warp", FP, 64)])
def test_all_true_mask_is_the_packed_call_bitwise(gran, dt, D):
    import sageattention_b200 as sab
    lens_q, lens_k = [129, 300, 0, 64, 1], [64, 129, 50, 0, 200]
    q, k, v, do = _packed(lens_q, lens_k, 8, 2, D, dt, seed=D, tail=7)
    cq, ck = _cu(lens_q), _cu(lens_k)
    kw = dict(qk_quant_gran=gran, return_lse=True)
    Tq = sum(lens_q)     # o / lse rows past the end are not written
    for causal, bm in ((False, torch.ones(5, 8, 3, 4, dtype=torch.bool, device="cuda")),
                       (True, torch.ones(1, 1, 3, 4, dtype=torch.bool, device="cuda"))):   # causal with Lq != Lk
        a = _grads(lambda q, k, v: sab.sageattn_varlen_blocksparse(q, k, v, cq, ck, 300, 200, bm, is_causal=causal, **kw), q, k, v, do)
        b = _grads(lambda q, k, v: sab.sageattn_varlen_qk_int8_pv_fp8_cuda(q, k, v, cq, ck, 300, 200, is_causal=causal, **kw), q, k, v, do)
        for name, x, y in zip(("o", "lse", "dq", "dk", "dv"), (a[0][:Tq], a[1][:, :Tq]) + a[2:], (b[0][:Tq], b[1][:, :Tq]) + b[2:]):
            assert torch.equal(x, y), (causal, name)


def test_causal_with_unequal_lengths_against_exact():
    lens_q, lens_k = [100, 64, 1, 300, 0, 129, 200], [300, 64, 129, 50, 10, 1, 200]
    q, k, v, _ = _packed(lens_q, lens_k, 8, 2, 128, FP, seed=21)
    for p, seed in ((0.5, 1), (0.25, 2)):
        bm = _mask(7, 8, 300, 300, p, seed)
        bm[:, :, 0, 0] = False                                 # first rows of every sequence see nothing
        o, lse = _check_forward(q, k, v, lens_q, lens_k, bm, True, pv_accum_dtype="fp32+fp32")
        assert torch.isneginf(lse).any() and torch.isfinite(lse).any()


# ------------------------------------------------------------------------------------------------ leakage, sentinels
def test_no_leakage_across_sequences():
    import sageattention_b200 as sab
    lens = [200, 129, 300, 64]
    q, k, v, _ = _packed(lens, lens, 8, 2, 128, BF, seed=3)
    cu = _cu(lens)
    spans = _spans(lens)
    for causal, p in ((False, 0.5), (True, 1.0), (True, 0.3)):
        bm = _mask(4, 8, 300, 300, p, seed=8)
        o, lse = sab.sageattn_varlen_blocksparse(q, k, v, cu, cu, 300, 300, bm, is_causal=causal, return_lse=True)
        for b, (s, e) in enumerate(spans):
            k2, v2 = k.clone(), v.clone()
            for c, (s2, e2) in enumerate(spans):
                if c != b:
                    k2[s2:e2] = 200.0 * torch.randn_like(k2[s2:e2])
                    v2[s2:e2] = -300.0
            o2, lse2 = sab.sageattn_varlen_blocksparse(q, k2, v2, cu, cu, 300, 300, bm, is_causal=causal, return_lse=True)
            assert torch.equal(o2[s:e], o[s:e]) and torch.equal(lse2[:, s:e], lse[:, s:e]), (b, causal, p)


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
    for p in (1.0, 0.5):
        bm = _mask(3, 4, 200, 200, p, seed=1)
        bm[:, :, :, 0] = True                                   # every row sees a key
        o = torch.full_like(q, 7.0)
        lse = ops.qk_int8_sv_f8_attn_varlen_blocksparse(q8, k8, v8, o, qs, ks, vs, vm, cu, cu, cu_pad, cqs, cks, 200, 200, bm, 0, PT, PT,
                                                        128 ** -0.5, 1)
        assert (o[300:] == 7.0).all() and not (o[:300] == 7.0).all(-1).any()
        assert lse.shape == (4, q.size(0)) and torch.isfinite(lse[:, :300]).all()


# ------------------------------------------------------------------------------------------------ gradients
BWD_CASES = [  # gran, causal, dtype, D, density
    ("per_thread", True, BF, 128, 0.5),
    ("per_warp", False, FP, 64, 0.25),
    ("per_thread", False, FP, 128, 0.5),
    ("per_warp", True, BF, 96, 0.3),
    ("per_thread", False, BF, 64, 0.1),
    ("per_warp", True, BF, 64, 0.5),
    ("per_thread", True, FP, 64, 0.3),
    ("per_warp", False, FP, 128, 0.25),
]


@pytest.mark.parametrize("case", BWD_CASES, ids=lambda c: "-".join(str(x).replace("torch.", "") for x in c))
def test_gradients_bit_for_bit_per_sequence(case):
    import sageattention_b200 as sab
    gran, causal, dt, D, p = case
    lens_q = [129, 300, 0, 64, 1, 65]
    lens_k = lens_q if causal else [64, 129, 50, 0, 200, 300]
    q, k, v, do = _packed(lens_q, lens_k, 8, 2, D, dt, seed=D + causal, tail=9)
    cq, ck = _cu(lens_q), _cu(lens_k)
    bm = _mask(6, 8, 300, 300, p, seed=D)
    fn = lambda q, k, v: sab.sageattn_varlen_blocksparse(q, k, v, cq, ck, 300, 300, bm, is_causal=causal, qk_quant_gran=gran,
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
        mb = bm[b, :, :_nb(e - s, 128), :_nb(ek - sk, 64)]
        em = expand_block_mask(mb[None], e - s, ek - sk)[0]                               # [Hq, Lq, Lk]
        if causal:
            em = em & torch.ones(e - s, ek - sk, dtype=torch.bool, device="cuda").tril()
        unseen = ~em.reshape(2, 4, e - s, ek - sk).any(1).any(1).t()                       # [Lk, Hkv]: no Q head of the group sees it
        assert not dk[sk:ek][unseen].any() and not dv[sk:ek][unseen].any(), f"keys of sequence {b} hidden from every row"
        qb, kb, vb = (t.clone().requires_grad_(True) for t in (q[s:e][None], k[sk:ek][None], v[sk:ek][None]))
        ob = sab.sageattn_blocksparse(qb, kb, vb, mb[None], tensor_layout="NHD", is_causal=causal, qk_quant_gran=gran)
        ob.backward(do[s:e][None])
        assert torch.equal(o[s:e], ob[0].detach()), f"output of sequence {b}"
        for name, got, ref in (("dq", dq[s:e], qb.grad[0]), ("dk", dk[sk:ek], kb.grad[0]), ("dv", dv[sk:ek], vb.grad[0])):
            assert torch.equal(got, ref), f"{name} of sequence {b}"
    assert not dq[Tq:].any() and not dk[Tk:].any() and not dv[Tk:].any()
    # the forward gives the same bits whether or not the inputs require grad (rows past the end are not written)
    o_plain = sab.sageattn_varlen_blocksparse(q, k, v, cq, ck, 300, 300, bm, is_causal=causal, qk_quant_gran=gran)
    assert torch.equal(o_plain[:Tq], o[:Tq])


def test_torch_compile_fullgraph_gives_eager_bits():
    import sageattention_b200 as sab
    lens = [300, 64, 129]
    q, k, v, do = _packed(lens, lens, 2, 2, 64, FP, seed=11)
    cu = _cu(lens)
    bm = _mask(3, 2, 300, 300, 0.5, seed=2)

    def f(q, k, v):
        return sab.sageattn_varlen_blocksparse(q, k, v, cu, cu, 300, 300, bm, is_causal=True)

    eager = _grads(f, q, k, v, do)
    comp = _grads(torch.compile(f, fullgraph=True), q, k, v, do)
    for i in (0, 2, 3, 4):
        assert torch.equal(eager[i], comp[i])


# ------------------------------------------------------------------------------------------------ predictor
def _smooth_packed(lens, H, D, dt, seed):
    """Packed tokens that vary smoothly inside each sequence plus noise whose level changes every 64 tokens (the dense predictor
    test's data, one sequence at a time)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    parts = []
    for L in lens:
        pos = torch.arange(L, device="cuda", dtype=torch.float32)[:, None]
        basis = torch.sin(pos * torch.rand(1, 4, generator=g, device="cuda") * 0.02 + torch.rand(1, 4, generator=g, device="cuda") * 6.3)
        coef = torch.randn(H, 4, D, generator=g, device="cuda")
        base = torch.randn(H, 1, D, generator=g, device="cuda")
        level = torch.rand(H, (L + 63) // 64, 1, generator=g, device="cuda").pow(3) * 4.0
        noise = torch.randn(H, L, D, generator=g, device="cuda") * level.repeat_interleave(64, 1)[:, :L]
        parts.append((base + basis @ coef + noise).transpose(0, 1))
    parts.append(torch.randn(3, H, D, generator=g, device="cuda"))           # tokens past the end
    return torch.cat(parts).to(dt).contiguous()


PRED_CASES = [  # lens_q, lens_k, Hq, Hkv, D, dtype, causal
    ([1000, 0, 129, 64, 1, 2048], [777, 50, 0, 65, 64, 2048], 4, 2, 128, BF, False),
    ([300, 1024, 65, 128], [300, 1024, 65, 128], 2, 2, 64, FP, True),
    ([513, 77, 2000], [513, 77, 2000], 8, 2, 96, BF, True),
]


@pytest.mark.parametrize("case", PRED_CASES, ids=lambda c: f"{c[6]}-{c[4]}-{str(c[5]).replace('torch.', '')}")
def test_predictor_slices_are_the_dense_bits(case):
    import sageattention_b200 as sab
    lens_q, lens_k, Hq, Hkv, D, dt, causal = case
    q, k = _smooth_packed(lens_q, Hq, D, dt, seed=D), _smooth_packed(lens_k, Hkv, D, dt, seed=D + 1)
    mq, mk = _max(lens_q), _max(lens_k)
    for cu_dtype in (torch.int32, torch.int64):
        for cdf, sim in ((0.9, 0.5), (0.5, 0.8), (0.99, -1.0), (1.0, 0.3)):
            kw = dict(cdf_threshold=cdf, sim_threshold=sim, is_causal=causal)
            m = sab.predict_block_mask_varlen(q, k, _cu(lens_q, cu_dtype), _cu(lens_k, cu_dtype), mq, mk, **kw)
            assert m.dtype == torch.bool and m.is_contiguous() and tuple(m.shape) == (len(lens_q), Hq, _nb(mq, 128), _nb(mk, 64))
            outside = torch.ones_like(m)
            for b, ((s, e), (sk, ek)) in enumerate(zip(_spans(lens_q), _spans(lens_k))):
                if e == s or ek == sk:
                    continue
                nq, nk = _nb(e - s, 128), _nb(ek - sk, 64)
                outside[b, :, :nq, :nk] = False
                ref = sab.predict_block_mask(q[s:e][None], k[sk:ek][None], tensor_layout="NHD", **kw)[0]
                assert torch.equal(m[b, :, :nq, :nk], ref), (b, cdf, sim)
            assert not m[outside].any()
            assert torch.equal(sab.predict_block_mask_varlen(q, k, _cu(lens_q), _cu(lens_k), mq, mk, **kw), m)   # reproducible


def test_predictor_causal_unequal_lengths_against_restatement():
    """Causal with Lq != Lk (no dense counterpart): each slice against the fp64 restatement on the kernel's own per-sequence
    statistics (sab_block_stats_varlen), rows with a decision within 1e-5 of a threshold counted, not compared."""
    import sageattention_b200 as sab
    from sageattention_b200 import ops
    lens_q, lens_k = [1000, 129, 300, 64], [300, 1024, 65, 2000]
    Hq, Hkv, D = 4, 2, 128
    q, k = _smooth_packed(lens_q, Hq, D, BF, seed=5), _smooth_packed(lens_k, Hkv, D, BF, seed=6)
    cq, ck, mq, mk = _cu(lens_q), _cu(lens_k), _max(lens_q), _max(lens_k)
    f32 = dict(dtype=torch.float32, device="cuda")
    qm, qs = torch.empty(4, Hq, _nb(mq, 128), D, **f32), torch.empty(4, Hq, _nb(mq, 128), **f32)
    km, ks = torch.empty(4, Hkv, _nb(mk, 64), D, **f32), torch.empty(4, Hkv, _nb(mk, 64), **f32)
    ops.block_stats_varlen(q, qm, qs, cq, mq, 128)
    ops.block_stats_varlen(k, km, ks, ck, mk, 64)
    for cdf, sim in ((0.9, 0.5), (0.5, 0.8), (0.99, 0.2)):
        m = sab.predict_block_mask_varlen(q, k, cq, ck, mq, mk, cdf_threshold=cdf, sim_threshold=sim, is_causal=True)
        near_rows = 0
        for b, (lq, lk) in enumerate(zip(lens_q, lens_k)):
            nq, nk = _nb(lq, 128), _nb(lk, 64)
            ref, near = select(qm[b:b + 1, :, :nq].cpu(), qs[b:b + 1, :, :nq].cpu(), km[b:b + 1, :, :nk].cpu(), ks[b:b + 1, :, :nk].cpu(),
                               lq, lk, cdf_threshold=cdf, sim_threshold=sim, is_causal=True, sm_scale=D ** -0.5, eps=EPS)
            far = ~near[0]
            assert torch.equal(m[b, :, :nq, :nk].cpu()[far], ref[0][far]), (b, cdf, sim)
            assert not m[b, :, nq:].any() and not m[b, :, :, nk:].any()
            near_rows += int(near.sum())
        print(f"[predict varlen causal] cdf {cdf} sim {sim}: near-threshold rows {near_rows}")
        assert near_rows <= 0.05 * Hq * sum(_nb(L, 128) for L in lens_q)


def test_packed_prediction_and_call_are_the_dense_ones():
    import sageattention_b200 as sab
    lens = [1000, 0, 129, 2048, 64]
    q, k = _smooth_packed(lens, 8, 128, BF, seed=1), _smooth_packed(lens, 2, 128, BF, seed=2)
    v = _smooth_packed(lens, 2, 128, BF, seed=3)
    cu = _cu(lens)
    for causal in (False, True):
        kw = dict(cdf_threshold=0.9, sim_threshold=0.5, is_causal=causal)
        m = sab.predict_block_mask_varlen(q, k, cu, cu, 2048, 2048, **kw)
        o = sab.sageattn_varlen_blocksparse(q, k, v, cu, cu, 2048, 2048, m, is_causal=causal)
        for b, (s, e) in enumerate(_spans(lens)):
            if e == s:
                continue
            mb = sab.predict_block_mask(q[s:e][None], k[s:e][None], tensor_layout="NHD", **kw)
            ob = sab.sageattn_blocksparse(q[s:e][None], k[s:e][None], v[s:e][None], mb, tensor_layout="NHD", is_causal=causal)
            assert torch.equal(o[s:e], ob[0]), (b, causal)


# ------------------------------------------------------------------------------------------------ long case
def test_bench_lengths_density_quarter_spot_check():
    import sageattention_b200 as sab
    lens = [2048, 16384, 4096, 512, 1024, 8192]
    q, k, v, do = _packed(lens, lens, 32, 8, 128, BF, seed=0)
    cu = _cu(lens)
    bm = _mask(6, 32, 16384, 16384, 0.25, seed=0)
    o, _, dq, dk, dv = _grads(lambda q, k, v: sab.sageattn_varlen_blocksparse(q, k, v, cu, cu, 16384, 16384, bm, return_lse=True),
                              q, k, v, do)
    spans = _spans(lens)
    for b in (3, 0, 2):                                         # 512, 2048 and 4096 tokens
        s, e = spans[b]
        nb_q, nb_k = _nb(e - s, 128), _nb(e - s, 64)
        qb, kb, vb = (t.clone().requires_grad_(True) for t in (q[s:e][None], k[s:e][None], v[s:e][None]))
        ob = sab.sageattn_blocksparse(qb, kb, vb, bm[b:b + 1, :, :nb_q, :nb_k], tensor_layout="NHD")
        ob.backward(do[s:e][None])
        assert torch.equal(o[s:e], ob[0].detach()), f"output of sequence {b} (L={e - s})"
        for name, got, ref in (("dq", dq[s:e], qb.grad[0]), ("dk", dk[s:e], kb.grad[0]), ("dv", dv[s:e], vb.grad[0])):
            assert torch.equal(got, ref), f"{name} of sequence {b} (L={e - s})"
