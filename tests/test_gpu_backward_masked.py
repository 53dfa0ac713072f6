"""GPU tests (-m gpu) of the masked backward (sab_qk_int8_attn_bwd_masked, the autograd form of sageattn_qk_int8_pv_fp16_triton
with attn_mask):
  1. the masked forward is bit-identical with and without requires_grad inputs;
  2. the gradient kernels, dBias included, against the fp64 CPU oracle (attn_bwd_masked_oracle.attn_bwd_masked) on the kernel's
     own quantised operands and LSE;
  3. public API gradients against fp64 autograd of exact masked attention;
  4. bit-reproducibility; 5. exact zeros on fully masked rows and -inf bias positions; 6. torch.compile.

Tolerances, as for the dense backward (tests/test_gpu_backward.py):
  oracle      every element, dBias included, within the bound of attn_bwd_oracle (check_elementwise; dBias gets ln2 times dS's),
              derived from the kernels' rounding model (input-dtype rounding of P and dS and of dBias, fp32 accumulation,
              ex2.approx).  Measured on an H100 80GB HBM3 (400 W power limit) over ORACLE_CASES: worst ratio of error to bound
              0.947; normwise relative errors at most 2.4e-3 for bf16 and 3.0e-4 for fp16, dBias 1.7e-3 / 2.1e-4;
  TOL_EXACT   3e-2 (normwise ||g - g_ref|| / ||g_ref||): against exact attention the straight-through estimator also carries the
              INT8 quantisation of Q and K.
The oracle and exact-attention tests print their errors (pytest -s)."""
import math
import os
import re

import pytest
import torch

from attn_bwd_masked_oracle import attn_bwd_masked
from attn_bwd_oracle import check_elementwise

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu

TOL_EXACT = 3e-2
BF, FP = torch.bfloat16, torch.float16
LN2 = math.log(2.0)
GRAN = {"per_block": 1, "per_warp": 2}      # SAB_GRAN_*


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / b.norm()).item()


def _shape(B, H, S, D, layout):
    return (B, H, S, D) if layout == "HND" else (B, S, H, D)


def _hnd(x, layout):
    return (x if layout == "HND" else x.transpose(1, 2)).cpu()


def _mask(kind, shape, seed, dt, strided=False):
    """A bool (False = masked out) or bias (dtype dt, -inf entries) mask of `shape` on the GPU.  Query row 0 is fully visible and,
    when there are more rows, row 1 fully masked.  strided: a non-contiguous view (every other key of a wider tensor)."""
    g = torch.Generator().manual_seed(seed)
    wide = shape[:-1] + (2 * shape[-1],) if strided else shape
    keep = torch.rand(wide, generator=g) > 0.3
    keep[..., 0, :] = True
    if shape[-2] > 1:
        keep[..., 1, :] = False
    m = keep if kind == "bool" else torch.where(keep, 2.0 * torch.randn(wide, generator=g), float("-inf")).to(dt)
    m = m.cuda()
    return m[..., ::2] if strided else m


# ------------------------------------------------------------------------------------------- 2. kernels vs oracle
# (D, dtype, layout, kind, Hq, Hkv, gran, Sq, Skv, B, mask shape, strided): per_block = sageattn_qk_int8_pv_fp16_triton's folded
# scales, per_warp through ops.  Mask shapes [Sq,Skv] / [B,1,Sq,Skv] broadcast with stride 0; [1,Hq,Sq,Skv] differs per Q head.
ORACLE_CASES = [
    (128, BF, "HND", "bias", 2, 2, "per_block", 256, 256, 2, "1HSS", False),
    (128, BF, "NHD", "bool", 32, 8, "per_warp", 128, 192, 1, "1HSS", False),    # GQA 32/8, per-head mask
    (128, FP, "HND", "bool", 4, 1, "per_block", 300, 300, 1, "1HSS", True),     # GQA 4/1, strided view
    (128, FP, "NHD", "bias", 2, 2, "per_warp", 200, 333, 1, "SS", False),       # Sq != Skv, odd Skv
    (64, BF, "HND", "bias", 4, 1, "per_block", 257, 190, 1, "1HSS", True),      # GQA 4/1, strided bias
    (64, BF, "NHD", "bool", 2, 2, "per_block", 1, 300, 2, "B1SS", False),       # Sq = 1
    (64, FP, "HND", "bool", 2, 2, "per_warp", 130, 77, 1, "SS", False),
    (64, FP, "NHD", "bias", 8, 2, "per_block", 65, 129, 2, "B1SS", False),
]


def _instantiations():
    src = open(os.path.join(ROOT, "sageattention_b200", "csrc", "attn_bwd.cu")).read()
    return {(int(d), t) for d, t in re.findall(r"launch_bwd_masked<(\d+), (__nv_bfloat16|__half)>\(", src)}


_INST = _instantiations()
_REACHED = {(c[0], "__nv_bfloat16" if c[1] == BF else "__half", c[3]) for c in ORACLE_CASES}
assert len(_INST) == 4 and _REACHED == {(d, t, kind) for d, t in _INST for kind in ("bool", "bias")}, \
    "ORACLE_CASES must reach both mask kinds of every masked dQ and dK/dV kernel of attn_bwd.cu"


def _mask_shape(ms, B, Hq, Sq, Skv):
    return {"SS": (Sq, Skv), "B1SS": (B, 1, Sq, Skv), "1HSS": (1, Hq, Sq, Skv)}[ms]


@pytest.mark.parametrize("case", ORACLE_CASES, ids=lambda c: "-".join(str(x).replace("torch.", "") for x in c))
def test_masked_gradient_kernels_match_oracle(case):
    import sageattention_b200 as sab
    from sageattention_b200 import ops
    D, dt, layout, kind, Hq, Hkv, gran, Sq, Skv, B, ms, strided = case
    lay = 1 if layout == "HND" else 0
    g = torch.Generator().manual_seed(Sq + 3 * Skv + D)
    q = torch.randn(_shape(B, Hq, Sq, D, layout), generator=g).to(dt).cuda()
    k = (torch.randn(_shape(B, Hkv, Skv, D, layout), generator=g) + 2.0 * torch.randn(D, generator=g)).to(dt).cuda()
    v = torch.randn(_shape(B, Hkv, Skv, D, layout), generator=g).to(dt).cuda()
    do = torch.randn(_shape(B, Hq, Sq, D, layout), generator=g).to(dt).cuda()
    mask = _mask(kind, _mask_shape(ms, B, Hq, Sq, Skv), Sq + Skv, dt, strided).expand(B, Hq, Sq, Skv)
    sm = D ** -0.5
    km = sab.k_mean(k, layout)
    if gran == "per_block":
        q8, qs, k8, ks = sab.per_block_int8(q, k, km, sm_scale=sm, tensor_layout=layout)
        fold = 1
    else:
        q8, qs, k8, ks = sab.per_warp_int8(q, k, km, tensor_layout=layout)
        fold = 0
    o = torch.empty_like(q)
    lse = ops.qk_int8_sv_f16_attn_masked(q8, k8, sab.transpose_v_f16(v, layout), o, qs, ks, mask, lay, GRAN[gran], GRAN[gran], sm,
                                         fold, 1)
    # NaN-filled outputs: every element must be written
    dq, dk, dv = (torch.full_like(t, float("nan")) for t in (q, k, v))
    dbias = torch.full((B, Hq, Sq, Skv), float("nan"), dtype=dt, device="cuda") if kind == "bias" else None
    ops.qk_int8_attn_bwd_masked(q8, k8, qs, ks, q, k, v, o, do, lse, km, dq, dk, dv, mask, dbias, lay, GRAN[gran], GRAN[gran], sm,
                                fold)
    torch.cuda.synchronize()
    *ref, bounds = attn_bwd_masked(_hnd(q8, layout), _hnd(k8, layout), qs.cpu(), ks.cpu(), _hnd(q, layout), _hnd(k, layout),
                                   _hnd(v, layout), _hnd(o, layout), _hnd(do, layout), lse.cpu(), mask.cpu(), q_gran=gran,
                                   k_gran="per_block", sm_scale=sm, fold_sm_scale=bool(fold), k_mean=_hnd(km, layout), bound=True)
    got = (_hnd(dq, layout), _hnd(dk, layout), _hnd(dv, layout)) + (() if dbias is None else (dbias.cpu(),))
    res = {name: check_elementwise(name, x, r, b) for name, x, r, b in zip(("dq", "dk", "dv", "dbias"), got, ref, bounds)}
    print(f"[oracle] {case[:11]} {str(dt)[6:]}: " + ", ".join(f"{n} ratio {w:.3f} normwise {e:.2e}" for n, (w, e) in res.items()))
    if Sq > 1:   # query row 1 is fully masked: lse -inf, zero dq (and dBias) rows
        assert torch.isinf(lse[:, :, 1]).all() and not got[0][:, :, 1].any()
        if dbias is not None:
            assert not dbias[:, :, 1].any()
    if dbias is not None:
        assert not dbias[mask.isinf()].any()


def test_masked_backward_refuses_like_the_forward():
    """per-thread K scales: the same status and message from the masked forward and backward."""
    import sageattention_b200 as sab
    from sageattention_b200 import _capi, ops
    q, k, v = (torch.randn(1, 2, 128, 64, device="cuda", dtype=FP) for _ in range(3))
    mask = torch.ones(1, 2, 128, 128, dtype=torch.bool, device="cuda")
    q8, qs, k8, ks = sab.per_thread_int8(q, k, None)
    with pytest.raises(_capi.SabError) as fwd:
        ops.qk_int8_sv_f16_attn_masked(q8, k8, sab.transpose_v_f16(v), torch.empty_like(q), qs, ks, mask, 1, 3, 3, 0.125, 0, 1)
    lse = torch.zeros(1, 2, 128, device="cuda")
    with pytest.raises(_capi.SabError) as bwd:
        ops.qk_int8_attn_bwd_masked(q8, k8, qs, ks, q, k, v, q, q, lse, None, *(torch.empty_like(t) for t in (q, k, v)), mask, None,
                                    1, 3, 3, 0.125, 0)
    assert str(fwd.value) == str(bwd.value) and "per-block / per-warp K scales only" in str(bwd.value)


# ------------------------------------------------------------------------------------------- 1. no behaviour change
@pytest.mark.parametrize("kind", ["bool", "bias"])
@pytest.mark.parametrize("layout", ["HND", "NHD"])
def test_masked_forward_unchanged_by_requires_grad(kind, layout):
    import sageattention_b200 as sab
    B, H, S, D = 2, 2, 320, 96
    g = torch.Generator().manual_seed(1)
    q, k, v = (torch.randn(_shape(B, H, S, D, layout), generator=g).to(BF).cuda() for _ in range(3))
    mask = _mask(kind, (B, 1, S, S) if kind == "bool" else (1, H, S, S), 2, BF)
    with torch.no_grad():
        o0, l0 = sab.sageattn_qk_int8_pv_fp16_triton(q, k, v, tensor_layout=layout, attn_mask=mask, return_lse=True)
    qg, kg, vg = (t.clone().requires_grad_(True) for t in (q, k, v))
    mg = mask.clone().requires_grad_(kind == "bias")
    o1, l1 = sab.sageattn_qk_int8_pv_fp16_triton(qg, kg, vg, tensor_layout=layout, attn_mask=mg, return_lse=True)
    assert o1.requires_grad and o1.grad_fn is not None and not l1.requires_grad
    assert torch.equal(o0, o1.detach()) and torch.equal(l0, l1)
    o1.float().square().sum().backward()
    for t in (qg, kg, vg) + ((mg,) if kind == "bias" else ()):
        assert t.grad is not None and torch.isfinite(t.grad).all()


# ------------------------------------------------------------------------------------------- 3. public API vs exact attention
def _exact_masked(q, k, v, do, mask, layout):
    """fp64 autograd of softmax(q k^T / sqrt(D) + ln2 * bias) v (bool: False = -inf) on the unpadded inputs; a row without a
    visible key outputs zeros.  Returns (dq, dk, dv, dbias reduced to mask.shape or None)."""
    q, k, v = (t.detach().cpu().double().requires_grad_(True) for t in (q, k, v))
    qh, kh, vh = (x if layout == "HND" else x.transpose(1, 2) for x in (q, k, v))
    s = qh @ kh.transpose(-1, -2) * q.shape[-1] ** -0.5
    bias = None
    if mask.dtype == torch.bool:
        s = s.masked_fill(~mask.cpu(), float("-inf"))
    else:
        bias = mask.detach().cpu().double().requires_grad_(True)
        s = s + LN2 * bias
    row_visible = (s != float("-inf")).any(dim=-1, keepdim=True)
    o = (torch.softmax(torch.where(row_visible, s, 0.0), dim=-1) * row_visible) @ vh
    o = o if layout == "HND" else o.transpose(1, 2)
    (o * do.cpu().double()).sum().backward()
    return q.grad, k.grad, v.grad, None if bias is None else bias.grad


def _padding_mask(B, S, pad, device="cuda"):
    """bool [B,1,1,S]: batch entry b masks its last pad[b] keys."""
    m = torch.ones(B, 1, 1, S, dtype=torch.bool)
    for b, n in enumerate(pad):
        if n:
            m[b, ..., S - n:] = False
    return m.to(device)


@pytest.mark.parametrize("kind,B,S,D,dt,layout", [
    ("bias", 1, 1024, 96, BF, "HND"),       # [1,H,S,S] bias requiring grad, head-dim padding
    ("bool", 2, 1024, 96, FP, "NHD"),       # [B,1,1,S] padding mask
    ("bias", 2, 2048, 128, FP, "NHD"),
])
def test_masked_gradients_match_exact_attention(kind, B, S, D, dt, layout):
    import sageattention_b200 as sab
    H = 2
    g = torch.Generator().manual_seed(S + D)
    q = torch.randn(_shape(B, H, S, D, layout), generator=g)
    k = torch.randn(_shape(B, H, S, D, layout), generator=g) + 1.5 * torch.randn(D, generator=g)   # per-channel offset
    v, do = (torch.randn(_shape(B, H, S, D, layout), generator=g) for _ in range(2))
    q, k, v, do = (t.to(dt).cuda() for t in (q, k, v, do))
    q, k, v = (t.requires_grad_(True) for t in (q, k, v))
    if kind == "bias":
        mask = (1.5 * torch.randn(1, H, S, S, generator=g)).to(dt).cuda().requires_grad_(True)
    else:
        mask = _padding_mask(B, S, [0, 300][:B])
    o = sab.sageattn_qk_int8_pv_fp16_triton(q, k, v, tensor_layout=layout, attn_mask=mask)
    o.backward(do)
    ref = _exact_masked(q, k, v, do, mask, layout)
    got = (q.grad, k.grad, v.grad) + ((mask.grad,) if kind == "bias" else ())
    errs = {name: _rel(x, r) for name, x, r in zip(("dq", "dk", "dv", "dbias"), got, ref)}
    print(f"[exact] {kind} B={B} S={S} D={D} {str(dt)[6:]} {layout}: " + ", ".join(f"{n} {e:.2e}" for n, e in errs.items()))
    assert max(errs.values()) <= TOL_EXACT, f"normwise relative errors {errs}"


# ------------------------------------------------------------------------------------------- 4. determinism
def test_masked_backward_is_bit_reproducible():
    import sageattention_b200 as sab
    g = torch.Generator().manual_seed(7)
    q = torch.randn(2, 8, 1000, 128, generator=g).to(BF).cuda()
    k, v = (torch.randn(2, 2, 1000, 128, generator=g).to(BF).cuda() for _ in range(2))
    bias = torch.randn(1, 8, 1000, 1000, generator=g).to(BF).cuda()
    do = torch.randn(q.shape, generator=g).to(BF).cuda()
    grads = []
    for _ in range(2):
        qg, kg, vg, bg = (t.clone().requires_grad_(True) for t in (q, k, v, bias))
        sab.sageattn_qk_int8_pv_fp16_triton(qg, kg, vg, attn_mask=bg).backward(do)
        grads.append((qg.grad, kg.grad, vg.grad, bg.grad))
    for a, b in zip(*grads):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------- 5. exact zeros, no NaN
@pytest.mark.parametrize("kind", ["bool", "bias"])
def test_fully_masked_rows_and_inf_bias_get_exact_zeros(kind):
    import sageattention_b200 as sab
    B, H, S, D = 1, 4, 300, 64
    g = torch.Generator().manual_seed(3)
    q, k, v, do = (torch.randn(B, H, S, D, generator=g).to(FP).cuda() for _ in range(4))
    mask = _mask(kind, (1, H, S, S), 4, FP)               # row 1 fully masked / fully -inf, scattered masked entries
    qg, kg, vg = (t.clone().requires_grad_(True) for t in (q, k, v))
    mg = mask.clone().requires_grad_(kind == "bias")
    o = sab.sageattn_qk_int8_pv_fp16_triton(qg, kg, vg, attn_mask=mg)
    o.backward(do)
    assert not o[:, :, 1].any()
    for t in (qg, kg, vg):
        assert torch.isfinite(t.grad).all()
    assert not qg.grad[:, :, 1].any()
    if kind == "bias":
        assert torch.isfinite(mg.grad).all()
        assert not mg.grad[mask.isinf()].any() and not mg.grad[:, :, 1].any()


# ------------------------------------------------------------------------------------------- 6. torch.compile
def test_masked_torch_compile_fullgraph_gives_eager_gradients():
    import sageattention_b200 as sab
    g = torch.Generator().manual_seed(11)
    q, k, v = (torch.randn(1, 2, 512, 64, generator=g).to(FP).cuda() for _ in range(3))
    bias = torch.randn(1, 2, 512, 512, generator=g).to(FP).cuda()

    def loss(q, k, v, bias):
        return sab.sageattn_qk_int8_pv_fp16_triton(q, k, v, attn_mask=bias).float().square().sum()

    def grads(f):
        ins = [t.clone().requires_grad_(True) for t in (q, k, v, bias)]
        f(*ins).backward()
        return [t.grad for t in ins]

    eager = grads(loss)
    compiled = grads(torch.compile(loss, fullgraph=True))
    for a, b in zip(eager, compiled):
        assert torch.equal(a, b)
