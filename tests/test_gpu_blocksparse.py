"""GPU tests (-m gpu) of the block-sparse attention (sageattn_blocksparse; sab_qk_int8_sv_f8_attn_blocksparse and
sab_qk_int8_attn_bwd_blocksparse):
  1. an all-True mask gives the bits of sageattn_qk_int8_pv_fp8_cuda (o and lse);
  2. seeded sparse masks against the CPU restatement (attn_blocksparse_oracle) and exact masked attention, causal included;
  3. hidden rows, broadcast masks; 4. the gradient: bit-identity with the dense backward for an all-True mask, fp64 autograd of
  exact block-masked attention, reproducibility, exact zeros; 5. validation; 6. torch.compile."""
import math
import warnings

import pytest
import torch

import sageattention_b200 as sab
from sageattention_b200 import ops
from attn_blocksparse_oracle import attn_int8_fp8_blocksparse, expand_block_mask
from attn_bwd_masked_oracle import attn_bwd_masked
from attn_bwd_oracle import check_elementwise
from sageattention_b200.core import _quant_qk
from sageattention_b200.quant import per_channel_fp8

pytestmark = pytest.mark.gpu
BF, FP = torch.bfloat16, torch.float16
TOL_EXACT = 6e-2      # max-abs against exact attention (tests/test_gpu_parity.py)
TOL_GRAD = 3e-2       # normwise against fp64 autograd of exact attention (tests/test_gpu_backward.py)
# The gradient kernels are checked elementwise against the bound of tests/attn_bwd_oracle.py (check_elementwise) on their own
# operands.  Measured on an H100 80GB HBM3 (400 W power limit) over BWD_ORACLE_CASES: worst ratio of error to bound 0.854;
# normwise relative errors at most 2.4e-3 for bf16 and 3.0e-4 for fp16.
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


def _mask(shape, p, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.rand(shape, generator=g, device="cuda") < p


def _nq_nk(Sq, Sk):
    return (Sq + 127) // 128, (Sk + 63) // 64


CASES = [  # B, Hq, Hkv, Sq, Sk, D, dtype, layout, gran, causal, pv_accum, smooth_v
    (1, 2, 2, 512, 512, 128, FP, "HND", "per_thread", False, "fp32+fp16", False),
    (2, 2, 2, 384, 384, 64, BF, "NHD", "per_warp", True, "fp32+fp32", False),
    (1, 8, 2, 256, 256, 96, BF, "HND", "per_thread", True, "fp32", True),
    (1, 4, 4, 1000, 777, 128, FP, "NHD", "per_warp", False, "fp32+fp32", False),
    (1, 8, 2, 300, 700, 64, FP, "HND", "per_thread", False, "fp32", True),
    (1, 2, 2, 256, 256, 96, BF, "NHD", "per_warp", True, "fp32+fp32", False),
]


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("broadcast", [False, True])
def test_all_true_mask_is_the_dense_call_bitwise(case, broadcast):
    B, Hq, Hkv, Sq, Sk, D, dt, lay, gran, causal, acc, sv = case
    q, k, v = _qkv(B, Hq, Hkv, Sq, Sk, D, dt, lay)
    nq, nk = _nq_nk(Sq, Sk)
    bm = torch.ones((1, 1, nq, nk) if broadcast else (B, Hq, nq, nk), dtype=torch.bool, device="cuda")
    kw = dict(tensor_layout=lay, is_causal=causal, qk_quant_gran=gran, pv_accum_dtype=acc, smooth_v=sv, return_lse=True)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")      # smooth_v with a non-"fp32" pv_accum_dtype warns, in both calls
        o, l = sab.sageattn_blocksparse(q, k, v, bm, **kw)
        o_ref, l_ref = sab.sageattn_qk_int8_pv_fp8_cuda(q, k, v, **kw)
    assert torch.equal(o, o_ref) and torch.equal(l, l_ref)


def _exact(q, k, v, em, scale):
    g = q.size(1) // k.size(1)
    s = (q.double() @ k.double().repeat_interleave(g, 1).transpose(-1, -2)) * scale
    p = torch.softmax(s.masked_fill(~em, -math.inf), dim=-1).nan_to_num(0.0)
    return p @ v.double().repeat_interleave(g, 1)


@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("gran", ["per_thread", "per_warp"])
def test_sparse_mask_against_restatement_and_exact(causal, gran):
    B, Hq, Hkv, Sq, Sk, D = 1, 4, 2, 512, 512, 128
    q, k, v = _qkv(B, Hq, Hkv, Sq, Sk, D, FP, seed=1)
    nq, nk = _nq_nk(Sq, Sk)
    bm = _mask((B, Hq, nq, nk), 0.4, 2)
    bm[0, 0, 1] = False
    bm[0, 1, 2] = True
    o, lse = sab.sageattn_blocksparse(q, k, v, bm, is_causal=causal, qk_quant_gran=gran, pv_accum_dtype="fp32+fp32",
                                      return_lse=True)
    em = expand_block_mask(bm, Sq, Sk)
    if causal:
        em = em & torch.ones(Sq, Sk, dtype=torch.bool, device="cuda").tril()
    ref = _exact(q, k, v, em, D ** -0.5)
    rows = em.any(-1)
    # rows with >= 64 visible keys: a row that sees a handful of keys (causal, near the diagonal) carries the e4m3 rounding of
    # single V rows, as in the dense causal kernel
    wide = em.sum(-1) >= 64
    assert (o.double() - ref)[wide].abs().max().item() < TOL_EXACT
    assert torch.all(o[~rows] == 0) and torch.all(torch.isneginf(lse[~rows])) and not torch.isnan(o).any()
    if not causal:
        # the restatement on the call's own quantised operands (the quantisers are deterministic)
        _, q8, qs, k8, ks, _, _, _ = _quant_qk(q, k, "fp8", "HND", gran, D ** -0.5, True, "cuda")
        v8, vs, _ = per_channel_fp8(v, tensor_layout="HND", scale_max=448.0, smooth_v=False)
        v8 = v8[..., :Sk].transpose(-1, -2)
        oc = attn_int8_fp8_blocksparse(*(t.cpu() for t in (q8, k8, v8, qs, ks, vs, bm)), qk_quant_gran=gran, sm_scale=D ** -0.5,
                                       lazy_tau=4, out_dtype=FP)
        assert (o.cpu().float() - oc.float()).abs().max().item() < 1e-2      # smoke()'s tolerance


def test_broadcast_mask_gives_the_bits_of_its_expanded_copy():
    B, Hq, Hkv, Sq, Sk, D = 2, 4, 4, 384, 448, 64
    q, k, v = _qkv(B, Hq, Hkv, Sq, Sk, D, BF, seed=3)
    bm = _mask((1, Hq, *_nq_nk(Sq, Sk)), 0.5, 4)
    a = sab.sageattn_blocksparse(q, k, v, bm, return_lse=True)
    b = sab.sageattn_blocksparse(q, k, v, bm.expand(B, -1, -1, -1).contiguous(), return_lse=True)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_validation_raises_before_any_launch():
    q, k, v = _qkv(1, 2, 2, 256, 256, 64, FP)
    with pytest.raises(ValueError):
        sab.sageattn_blocksparse(q, k, v, torch.ones(1, 2, 2, 3, dtype=torch.bool, device="cuda"))
    with pytest.raises(ValueError):
        sab.sageattn_blocksparse(q, k, v, torch.ones(3, 2, 2, 4, dtype=torch.bool, device="cuda"))
    with pytest.raises(AssertionError):
        sab.sageattn_blocksparse(q, k, v, torch.ones(1, 2, 2, 4, dtype=torch.uint8, device="cuda"))
    with pytest.raises(AssertionError):
        sab.sageattn_blocksparse(q, k, v, torch.ones(1, 2, 2, 4, dtype=torch.bool))


# ------------------------------------------------------------------------------------------------ gradient
def _grads(fn, q, k, v, do):
    o = fn(q, k, v)
    return (o,) + torch.autograd.grad(o, (q, k, v), do)


@pytest.mark.parametrize("causal", [False, True])
def test_all_true_mask_gradients_are_the_dense_backward_bitwise(causal):
    B, Hq, Hkv, S, D = 1, 4, 2, 384, 128
    q, k, v = _qkv(B, Hq, Hkv, S, S, D, BF, seed=5, grad=True)
    do = torch.randn_like(q)
    bm = torch.ones(1, 1, *_nq_nk(S, S), dtype=torch.bool, device="cuda")
    a = _grads(lambda q, k, v: sab.sageattn_blocksparse(q, k, v, bm, is_causal=causal), q, k, v, do)
    b = _grads(lambda q, k, v: sab.sageattn_qk_int8_pv_fp8_cuda(q, k, v, is_causal=causal), q, k, v, do)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    with torch.no_grad():
        assert torch.equal(sab.sageattn_blocksparse(q, k, v, bm, is_causal=causal), a[0])


@pytest.mark.parametrize("causal", [False, True])
def test_sparse_gradients_against_exact_autograd(causal):
    B, Hq, Hkv, S, D = 1, 4, 2, 512, 64
    q, k, v = _qkv(B, Hq, Hkv, S, S, D, BF, seed=6, grad=True)
    do = torch.randn_like(q)
    nq, nk = _nq_nk(S, S)
    bm = _mask((B, Hq, nq, nk), 0.4, 7)
    bm[0, 0, 0] = False               # hidden rows
    bm[:, :, :, 3] = False            # keys hidden from every row
    fn = lambda q, k, v: sab.sageattn_blocksparse(q, k, v, bm, is_causal=causal)
    o, dq, dk, dv = _grads(fn, q, k, v, do)
    o2, dq2, dk2, dv2 = _grads(fn, q, k, v, do)
    assert all(torch.equal(x, y) for x, y in ((o, o2), (dq, dq2), (dk, dk2), (dv, dv2)))
    em = expand_block_mask(bm, S, S)
    if causal:
        em = em & torch.ones(S, S, dtype=torch.bool, device="cuda").tril()
    qd, kd, vd = (t.detach().double().requires_grad_() for t in (q, k, v))
    ref = _exact(qd, kd, vd, em, D ** -0.5)
    gq, gk, gv = torch.autograd.grad(ref, (qd, kd, vd), do.double())
    for g_, r_ in ((dq, gq), (dk, gk), (dv, gv)):
        assert ((g_.double() - r_).norm() / r_.norm()).item() < TOL_GRAD
    hidden_rows = ~em.any(-1)
    assert torch.all(dq[hidden_rows] == 0) and torch.all(o[hidden_rows] == 0)
    assert torch.all(dk[:, :, 192:256] == 0) and torch.all(dv[:, :, 192:256] == 0)
    assert not any(torch.isnan(t).any() for t in (dq, dk, dv))


def test_compile_gives_the_eager_gradients():
    B, H, S, D = 1, 2, 256, 64
    q, k, v = _qkv(B, H, H, S, S, D, FP, seed=8, grad=True)
    do = torch.randn_like(q)
    bm = _mask((1, 1, *_nq_nk(S, S)), 0.6, 9)
    bm[..., 0] = True
    fn = lambda q, k, v: sab.sageattn_blocksparse(q, k, v, bm)
    eager = _grads(fn, q, k, v, do)
    comp = _grads(torch.compile(fn, fullgraph=True), q, k, v, do)
    for x, y in zip(eager, comp):
        assert torch.equal(x, y)


# ------------------------------------------------------------------------------------------------ exact bits of the sparse index map
def _operands(q, k, v, gran, layout="HND"):
    """The quantised operands sageattn_blocksparse computes (pv_accum_dtype "fp32+fp32": V range 448, no smoothing of V)."""
    km, q8, qs, k8, ks, _, _, _ = _quant_qk(q, k, "fp8", layout, gran, q.size(-1) ** -0.5, True, "cuda")
    v8, vs, _ = per_channel_fp8(v, tensor_layout=layout, scale_max=448.0, smooth_v=False)
    return km, q8, qs, k8, ks, v8, vs


# (D, dtype, gran): every block-sparse forward instantiation; Sq = 300 and Skv = 700 leave a partial last Q block and key tile
GATHER_CASES = [(128, BF, "per_thread"), (128, FP, "per_warp"), (64, FP, "per_thread"), (64, BF, "per_warp"),
                (128, FP, "per_thread"), (128, BF, "per_warp"), (64, BF, "per_thread"), (64, FP, "per_warp")]


@pytest.mark.parametrize("case", GATHER_CASES, ids=lambda c: f"D{c[0]}-{str(c[1])[6:]}-{c[2]}")
def test_sparse_forward_is_the_dense_kernel_on_gathered_blocks_bitwise(case):
    """Non-causal: CTA (b, h, i) of the sparse kernel is the dense kernel op run on Q block i with the visible 64-key blocks of
    k_int8, k_scale and v_fp8 gathered in order, to the bit (o and the kernel's log2 lse)."""
    D, dt, gran = case
    B, Hq, Hkv, Sq, Sk = 1, 4, 2, 300, 700
    q, k, v = _qkv(B, Hq, Hkv, Sq, Sk, D, dt, seed=D + GRAN[gran])
    nq, nk = _nq_nk(Sq, Sk)
    bm = _mask((B, Hq, nq, nk), 0.45, 11)
    bm[0, 0, 1] = False                      # a hidden Q-block row
    bm[0, 1, 0] = True                       # a fully visible one
    bm[0, 2:, :, nk - 1] = True              # the partial last key tile inside the list
    bm[0, 3, 2, nk - 1] = False
    _, q8, qs, k8, ks, v8, vs = _operands(q, k, v, gran)
    o = torch.empty_like(q)
    lse = ops.qk_int8_sv_f8_attn_blocksparse(q8, k8, v8, o, qs, ks, vs, None, bm, 1, 0, GRAN[gran], GRAN[gran], D ** -0.5, 0, 1)
    qm, km_ = {"per_warp": 4, "per_thread": 32}[gran], {"per_warp": 1, "per_thread": 4}[gran]
    for h in range(Hq):
        hk = h // (Hq // Hkv)
        for i in range(nq):
            r0, r1 = 128 * i, min(128 * i + 128, Sq)
            blocks = [j for j in range(nk) if bool(bm[0, h, i, j])]
            if not blocks:
                assert torch.all(o[0, h, r0:r1] == 0) and torch.all(torch.isneginf(lse[0, h, r0:r1]))
                continue
            keys = torch.cat([torch.arange(64 * j, min(64 * j + 64, Sk)) for j in blocks]).cuda()
            cols = torch.cat([torch.arange(j * km_, (j + 1) * km_) for j in blocks]).cuda()
            kg = k8[:, hk:hk + 1, keys].contiguous()
            vg = torch.zeros((1, 1, D, (keys.numel() + 127) // 128 * 128), dtype=torch.uint8, device="cuda")   # e4m3 bytes
            vg[..., :keys.numel()] = v8.view(torch.uint8)[:, hk:hk + 1, :, keys]
            vg = vg.view(v8.dtype)
            og = torch.empty((1, 1, r1 - r0, D), dtype=dt, device="cuda")
            lg = ops.qk_int8_sv_f8_attn(q8[:, h:h + 1, r0:r1].contiguous(), kg, vg, og, qs[:, h:h + 1, i * qm:(i + 1) * qm].contiguous(),
                                        ks[:, hk:hk + 1, cols].contiguous(), vs[:, hk:hk + 1].contiguous(), None, 1, 0, GRAN[gran],
                                        GRAN[gran], D ** -0.5, 0, 1)
            assert torch.equal(o[:, h:h + 1, r0:r1], og), (h, i)
            assert torch.equal(lse[:, h:h + 1, r0:r1], lg), (h, i)


# ------------------------------------------------------------------------------------------------ gradient kernels vs fp64 reference
def _hnd(x, layout):
    return (x if layout == "HND" else x.transpose(1, 2)).cpu()


# (D, dtype, gran, layout, causal, B, Hq, Hkv, Sq, Skv): every block-sparse dQ / dK/dV instantiation, GQA and ragged lengths
BWD_ORACLE_CASES = [
    (128, BF, "per_thread", "HND", False, 1, 4, 2, 300, 448),
    (128, FP, "per_thread", "NHD", True, 1, 2, 2, 384, 384),
    (128, BF, "per_warp", "NHD", True, 1, 4, 1, 333, 333),
    (128, FP, "per_warp", "HND", False, 2, 2, 2, 200, 517),
    (64, FP, "per_thread", "HND", True, 1, 4, 2, 320, 320),
    (64, BF, "per_thread", "NHD", False, 1, 2, 2, 450, 190),
    (64, BF, "per_warp", "HND", False, 1, 8, 2, 256, 385),
    (64, FP, "per_warp", "NHD", True, 2, 2, 1, 257, 257),
]


@pytest.mark.parametrize("case", BWD_ORACLE_CASES, ids=lambda c: "-".join(str(x).replace("torch.", "") for x in c))
def test_sparse_gradient_kernels_match_oracle(case):
    """The kernels against tests/attn_bwd_masked_oracle.attn_bwd_masked fed the element-expanded block mask (ANDed with the
    causal mask), the kernels' own quantised operands and the forward kernel's LSE.  The masks hide whole Q-block rows, hide some
    keys from every row and leave many dK/dV steps with only one of a CTA's two 64-key blocks visible."""
    D, dt, gran, layout, causal, B, Hq, Hkv, Sq, Sk = case
    lay = 1 if layout == "HND" else 0
    q, k, v = _qkv(B, Hq, Hkv, Sq, Sk, D, dt, layout, seed=Sq + Sk + D)
    do = torch.randn_like(q)
    nq, nk = _nq_nk(Sq, Sk)
    bm = _mask((B, Hq, nq, nk), 0.5, Sq + D)
    bm[:, 0, nq - 1] = False                 # hidden rows
    bm[:, :, :, 1] = False                   # keys 64..127 hidden from every row
    bm[:, :, :, 0] = True                    # ... while keys 0..63 of the same 128-key tile are visible
    km, q8, qs, k8, ks, v8, vs = _operands(q, k, v, gran, layout)
    o = torch.empty_like(q)
    lse = ops.qk_int8_sv_f8_attn_blocksparse(q8, k8, v8, o, qs, ks, vs, None, bm, lay, int(causal), GRAN[gran], GRAN[gran],
                                             D ** -0.5, 0, 1)
    dq, dk, dv = (torch.full_like(t, float("nan")) for t in (q, k, v))   # every element must be written
    ops.qk_int8_attn_bwd_blocksparse(q8, k8, qs, ks, q, k, v, o, do, lse, km, dq, dk, dv, bm, lay, int(causal), GRAN[gran],
                                     GRAN[gran], D ** -0.5, 0)
    torch.cuda.synchronize()
    em = expand_block_mask(bm, Sq, Sk).cpu()
    if causal:
        em = em & torch.ones(Sq, Sk, dtype=torch.bool).tril()
    *ref, bounds = attn_bwd_masked(_hnd(q8, layout), _hnd(k8, layout), qs.cpu(), ks.cpu(), _hnd(q, layout), _hnd(k, layout),
                                   _hnd(v, layout), _hnd(o, layout), _hnd(do, layout), lse.cpu(), em, q_gran=gran, k_gran=gran,
                                   sm_scale=D ** -0.5, k_mean=_hnd(km, layout), bound=True)
    res = {name: check_elementwise(name, x, r, b)
           for name, x, r, b in zip(("dq", "dk", "dv"), (_hnd(dq, layout), _hnd(dk, layout), _hnd(dv, layout)), ref, bounds[:3])}
    print(f"[oracle] {case}: " + ", ".join(f"{n} ratio {w:.3f} normwise {e:.2e}" for n, (w, e) in res.items()))
    hidden_rows = ~em.any(-1)
    assert torch.all(_hnd(dq, layout)[hidden_rows] == 0)
    assert torch.all(_hnd(dk, layout)[:, :, 64:128] == 0) and torch.all(_hnd(dv, layout)[:, :, 64:128] == 0)
