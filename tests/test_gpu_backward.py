"""GPU tests (-m gpu) of the backward (csrc/attn_bwd.cu, the autograd form of the dense entry points in core.py):
  1. the forward of every differentiable entry point is bit-identical with and without requires_grad inputs;
  2. the gradient kernels against the fp64 CPU oracle (attn_bwd_oracle.attn_bwd) on the kernel's own quantised operands and LSE;
  3. sageattn gradients against fp64 autograd of exact attention;
  4. bit-reproducibility; 5. SDPA monkey-patch training; 6. torch.compile.

Tolerances:
  oracle      every element within the bound of attn_bwd_oracle (check_elementwise): on the same quantised operands and LSE the
              kernel differs from the oracle only by the input-dtype rounding of P and dS, fp32 accumulation and ex2.approx, and the
              bound is derived from exactly that rounding model.  Outputs are NaN-filled, so an unwritten element fails.
              Measured on an H100 80GB HBM3 (400 W power limit) over ORACLE_CASES: worst ratio of error to bound 0.957; normwise relative
              errors at most 2.5e-3 for bf16 and 3.0e-4 for fp16, except dq without a K mean (4.3e-3 / 5.6e-4) and dk with one key
              (Skv = 1: dS is a cancellation residue, dk is near zero and its normwise error 1.5e-2, every element inside the bound);
  TOL_EXACT   3e-2 (normwise ||g - g_ref|| / ||g_ref||): against exact attention the straight-through estimator also carries the
              INT8 / FP8 quantisation of the forward.  Measured on an H100 80GB HBM3 (700 W): 1.0-1.9 % for dq / dk / dv over the four
              cases below."""
import os
import re

import pytest
import torch
import torch.nn.functional as F

from attn_bwd_oracle import attn_bwd, check_elementwise

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu

TOL_EXACT = 3e-2
GRAN = {"per_block": 1, "per_warp": 2, "per_thread": 3}      # SAB_GRAN_*


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / b.norm()).item()


# ------------------------------------------------------------------------------------------- 2. kernels vs oracle
# (D, dtype, layout, causal, Hq, Hkv, gran, Sq, Skv, B[, data, smooth_k]): per_block = the folded-scale path of
# sageattn_qk_int8_pv_fp16_triton.  data (default "randn"): "peaked" scales Q by 4 (near one-hot softmax rows), "kchan" offsets
# four K channels by 30 (a large K mean: the K - mean operand of dQ), "voff" offsets V by 20 (dP and delta cancel in dP - delta).
# smooth_k False (default True): no K mean, the kernels' kmean == nullptr branch.
BF, FP = torch.bfloat16, torch.float16
ORACLE_CASES = [
    (128, BF, "HND", False, 2, 2, "per_thread", 256, 256, 2),
    (128, FP, "NHD", True, 2, 2, "per_thread", 384, 384, 1),
    (128, BF, "HND", False, 32, 8, "per_warp", 128, 192, 1),        # GQA 32/8
    (128, FP, "NHD", True, 2, 2, "per_warp", 200, 200, 1),
    (128, BF, "HND", True, 2, 2, "per_block", 320, 320, 1),
    (64, BF, "NHD", False, 2, 2, "per_warp", 200, 333, 1),           # Sq != Skv, tails not multiples of 64 / 128
    (64, FP, "HND", True, 4, 1, "per_thread", 300, 300, 1),          # GQA 4/1
    (64, FP, "HND", False, 2, 2, "per_block", 257, 190, 1),
    (64, BF, "HND", False, 2, 2, "per_thread", 1, 300, 1),           # Sq = 1
    (64, FP, "NHD", False, 2, 2, "per_thread", 17, 100, 2),          # Sq = 17
    (128, BF, "HND", False, 2, 2, "per_thread", 8192, 8192, 1),      # B=1, H=2, S=8192
    # one key tile and its edges: Skv in {1, 17, 64, 65, 128, 129, 4097} against short and long Sq
    (64, BF, "HND", False, 2, 2, "per_thread", 17, 1, 1, "randn", True),
    (128, FP, "NHD", False, 2, 2, "per_warp", 300, 1, 1, "randn", True),
    (128, BF, "NHD", False, 2, 2, "per_block", 17, 17, 1, "randn", True),
    (64, FP, "HND", False, 2, 2, "per_thread", 300, 64, 1, "randn", True),
    (128, FP, "HND", False, 2, 2, "per_thread", 17, 65, 1, "randn", True),
    (64, BF, "NHD", False, 2, 2, "per_warp", 300, 128, 1, "randn", True),
    (64, FP, "NHD", False, 2, 2, "per_block", 17, 129, 1, "randn", True),
    (128, BF, "HND", False, 2, 2, "per_warp", 300, 4097, 1, "randn", True),
    (64, BF, "HND", False, 1, 1, "per_thread", 17, 4097, 1, "randn", True),
    # Q tile edges: Sq in {1, 64, 65, 127, 128, 129}
    (128, FP, "NHD", False, 2, 2, "per_thread", 1, 129, 1, "randn", True),
    (64, FP, "HND", False, 2, 2, "per_warp", 64, 190, 1, "randn", True),
    (128, BF, "NHD", False, 2, 2, "per_thread", 65, 64, 1, "randn", True),
    (64, BF, "NHD", False, 2, 2, "per_block", 127, 300, 1, "randn", True),
    (128, FP, "HND", False, 2, 2, "per_warp", 128, 65, 1, "randn", True),
    (64, FP, "NHD", False, 2, 2, "per_thread", 129, 17, 1, "randn", True),
    # causal S in {1, 63, 64, 65, 128, 129, 255, 257}: the dK/dV loop starts at k0 / 64, the dQ loop ends at the diagonal
    (64, BF, "HND", True, 2, 2, "per_thread", 1, 1, 1, "randn", True),
    (128, FP, "NHD", True, 2, 2, "per_warp", 63, 63, 1, "randn", True),
    (64, FP, "HND", True, 2, 2, "per_block", 64, 64, 1, "randn", True),
    (128, BF, "NHD", True, 2, 2, "per_thread", 65, 65, 1, "randn", True),
    (64, BF, "NHD", True, 2, 2, "per_warp", 128, 128, 1, "randn", True),
    (128, FP, "HND", True, 2, 2, "per_thread", 129, 129, 1, "randn", True),
    (128, BF, "HND", True, 2, 2, "per_block", 255, 255, 1, "randn", True),
    (64, FP, "NHD", True, 2, 2, "per_thread", 257, 257, 1, "randn", True),
    # GQA with B > 1 in NHD
    (128, BF, "NHD", False, 8, 2, "per_thread", 200, 150, 2, "randn", True),
    (64, FP, "NHD", True, 6, 2, "per_warp", 190, 190, 3, "randn", True),
    # no K mean, every instantiation
    (128, BF, "HND", False, 2, 2, "per_thread", 200, 300, 1, "randn", False),
    (128, FP, "NHD", True, 2, 2, "per_thread", 200, 200, 1, "randn", False),
    (128, BF, "NHD", False, 2, 2, "per_warp", 150, 200, 1, "randn", False),
    (128, FP, "HND", False, 2, 2, "per_block", 150, 150, 1, "randn", False),
    (64, BF, "NHD", True, 2, 2, "per_thread", 150, 150, 1, "randn", False),
    (64, FP, "HND", False, 2, 2, "per_thread", 100, 200, 1, "randn", False),
    (64, BF, "HND", False, 2, 2, "per_warp", 100, 200, 1, "randn", False),
    (64, FP, "NHD", True, 2, 2, "per_block", 180, 180, 1, "randn", False),
    # data kinds
    (128, BF, "HND", True, 2, 2, "per_thread", 256, 256, 1, "peaked", True),
    (64, FP, "NHD", False, 2, 2, "per_warp", 200, 300, 1, "peaked", True),
    (128, FP, "HND", False, 2, 2, "per_thread", 200, 260, 1, "kchan", True),
    (64, BF, "NHD", True, 2, 2, "per_block", 300, 300, 1, "kchan", True),
    (128, BF, "NHD", False, 4, 2, "per_warp", 200, 200, 1, "voff", True),
    (64, FP, "HND", True, 2, 2, "per_thread", 256, 256, 1, "voff", True),
]


def _instantiations():
    src = open(os.path.join(ROOT, "sageattention_b200", "csrc", "attn_bwd.cu")).read()
    return {(int(d), kt == "true", t) for d, kt, t in re.findall(r"launch_bwd<(\d+), (true|false), (__nv_bfloat16|__half)>\(", src)}


def _case_instantiation(c):
    D, dt, _, _, _, _, gran = c[:7]
    return D, gran == "per_thread", "__nv_bfloat16" if dt == BF else "__half"


def _case_options(c):
    return tuple(c[10:]) or ("randn", True)


_INST = _instantiations()
assert len(_INST) == 8 and _INST == {_case_instantiation(c) for c in ORACLE_CASES}, \
    f"ORACLE_CASES must reach every instantiation of attn_bwd.cu: missing {_INST - {_case_instantiation(c) for c in ORACLE_CASES}}"
assert {(_case_instantiation(c), c[2]) for c in ORACLE_CASES} == {(i, lay) for i in _INST for lay in ("HND", "NHD")}, \
    "ORACLE_CASES must reach every instantiation in both layouts"
assert {_case_instantiation(c) for c in ORACLE_CASES if not _case_options(c)[1]} == _INST, \
    "ORACLE_CASES must run every instantiation without a K mean"


def _shape(B, H, S, D, layout):
    return (B, H, S, D) if layout == "HND" else (B, S, H, D)


def _hnd(x, layout):
    return (x if layout == "HND" else x.transpose(1, 2)).cpu()


def _dev_hnd(x, layout):
    return x if layout == "HND" else x.transpose(1, 2)


@pytest.mark.parametrize("case", ORACLE_CASES, ids=lambda c: "-".join(str(x).replace("torch.", "") for x in c))
def test_gradient_kernels_match_oracle(case):
    import sageattention_b200 as sab
    from sageattention_b200 import ops
    D, dt, layout, causal, Hq, Hkv, gran, Sq, Skv, B = case[:10]
    data, smooth_k = _case_options(case)
    lay = 1 if layout == "HND" else 0
    g = torch.Generator().manual_seed(Sq + 3 * Skv + D)
    q = torch.randn(_shape(B, Hq, Sq, D, layout), generator=g)
    k = torch.randn(_shape(B, Hkv, Skv, D, layout), generator=g) + 2.0 * torch.randn(D, generator=g)
    v = torch.randn(_shape(B, Hkv, Skv, D, layout), generator=g)
    do = torch.randn(_shape(B, Hq, Sq, D, layout), generator=g)
    if data == "peaked":
        q = 4.0 * q
    elif data == "kchan":
        k[..., :4] += 30.0
    elif data == "voff":
        v = v + 20.0
    q, k, v, do = (t.to(dt).cuda() for t in (q, k, v, do))
    sm = D ** -0.5
    km = sab.k_mean(k, layout) if smooth_k else None
    o = torch.empty_like(q)
    if gran == "per_block":
        q8, qs, k8, ks = sab.per_block_int8(q, k, km, sm_scale=sm, tensor_layout=layout)
        lse = ops.qk_int8_sv_f16_attn(q8, k8, sab.transpose_v_f16(v, layout), o, qs, ks, lay, int(causal), 1, 1, sm, 1, 1)
        qg = kg = 1
        fold = 1
    else:
        q8, qs, k8, ks = (sab.per_thread_int8 if gran == "per_thread" else sab.per_warp_int8)(q, k, km, tensor_layout=layout)
        v8, vs, _ = sab.per_channel_fp8(v, tensor_layout=layout, scale_max=448.0, smooth_v=False)
        lse = ops.qk_int8_sv_f8_attn(q8, k8, v8, o, qs, ks, vs, None, lay, int(causal), GRAN[gran], GRAN[gran], sm, 0, 1)
        qg = kg = GRAN[gran]
        fold = 0
    # NaN-filled outputs: every element must be written
    dq, dk, dv = (torch.full_like(t, float("nan")) for t in (q, k, v))
    ops.qk_int8_attn_bwd(q8, k8, qs, ks, q, k, v, o, do, lse, km, dq, dk, dv, lay, int(causal), qg, kg, sm, fold)
    # the fp64 reference runs on the GPU
    *ref, bounds = attn_bwd(_dev_hnd(q8, layout), _dev_hnd(k8, layout), qs, ks, _dev_hnd(q, layout), _dev_hnd(k, layout),
                            _dev_hnd(v, layout), _dev_hnd(o, layout), _dev_hnd(do, layout), lse, q_gran=gran,
                            k_gran="per_block" if gran == "per_warp" else gran, is_causal=causal, sm_scale=sm,
                            fold_sm_scale=bool(fold), k_mean=None if km is None else _dev_hnd(km, layout), bound=True)
    res = {name: check_elementwise(name, _dev_hnd(got, layout), r, b)
           for name, got, r, b in zip(("dq", "dk", "dv"), (dq, dk, dv), ref, bounds)}
    print(f"[oracle] {case}: " + ", ".join(f"{n} ratio {w:.3f} normwise {e:.2e}" for n, (w, e) in res.items()))


# ------------------------------------------------------------------------------------------- 1. no behaviour change
def _entry_points():
    import sageattention_b200 as sab
    return {
        "sageattn": lambda q, k, v, **kw: sab.sageattn(q, k, v, **kw),
        "fp8_cuda_per_warp": lambda q, k, v, **kw: sab.sageattn_qk_int8_pv_fp8_cuda(q, k, v, qk_quant_gran="per_warp", **kw),
        "fp8_cuda_sm90": lambda q, k, v, **kw: sab.sageattn_qk_int8_pv_fp8_cuda_sm90(q, k, v, **kw),
        "fp16_cuda": lambda q, k, v, **kw: sab.sageattn_qk_int8_pv_fp16_cuda(q, k, v, **kw),
        "fp16_triton": lambda q, k, v, **kw: sab.sageattn_qk_int8_pv_fp16_triton(q, k, v, **kw),
    }


def _inputs(B, H, S, D, dt=BF, layout="HND", seed=0, Hkv=None, Skv=None):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(_shape(B, H, S, D, layout), generator=g)
    k = torch.randn(_shape(B, Hkv or H, Skv or S, D, layout), generator=g) + 1.5 * torch.randn(D, generator=g)   # per-channel offset
    v = torch.randn(_shape(B, Hkv or H, Skv or S, D, layout), generator=g)
    return (t.to(dt).cuda() for t in (q, k, v))


@pytest.mark.parametrize("name", ["sageattn", "fp8_cuda_per_warp", "fp8_cuda_sm90", "fp16_cuda", "fp16_triton"])
@pytest.mark.parametrize("causal", [False, True])
def test_forward_unchanged_by_requires_grad(name, causal):
    fn = _entry_points()[name]
    q, k, v = _inputs(1, 2, 320, 96, seed=1)
    with torch.no_grad():
        o0, l0 = fn(q, k, v, is_causal=causal, return_lse=True)
    qg, kg, vg = (t.clone().requires_grad_(True) for t in (q, k, v))
    o1, l1 = fn(qg, kg, vg, is_causal=causal, return_lse=True)
    assert o1.requires_grad and o1.grad_fn is not None and not l1.requires_grad
    assert torch.equal(o0, o1.detach()) and torch.equal(l0, l1)
    o1.float().square().sum().backward()
    assert all(t.grad is not None and torch.isfinite(t.grad).all() for t in (qg, kg, vg))


# ------------------------------------------------------------------------------------------- 3. public API vs exact attention
def _exact(q, k, v, do, causal, layout="HND"):
    q, k, v = (t.detach().cpu().double().requires_grad_(True) for t in (q, k, v))
    o = F.scaled_dot_product_attention(*(x if layout == "HND" else x.transpose(1, 2) for x in (q, k, v)), is_causal=causal,
                                       enable_gqa=True)
    o = o if layout == "HND" else o.transpose(1, 2)
    (o * do.cpu().double()).sum().backward()
    return q.grad, k.grad, v.grad


@pytest.mark.parametrize("S,D,causal,dt,layout", [
    (1024, 64, False, BF, "HND"), (2048, 128, True, BF, "HND"), (1024, 96, False, FP, "NHD"), (4096, 128, False, FP, "HND"),
])
def test_sageattn_gradients_match_exact_attention(S, D, causal, dt, layout):
    import sageattention_b200 as sab
    q, k, v = (t.requires_grad_(True) for t in _inputs(1, 2, S, D, dt, layout, seed=S + D))
    do = torch.randn(q.shape, generator=torch.Generator().manual_seed(5)).to(dt).cuda()
    o = sab.sageattn(q, k, v, tensor_layout=layout, is_causal=causal)
    o.backward(do)
    errs = {name: _rel(got, r) for name, got, r in zip(("dq", "dk", "dv"), (q.grad, k.grad, v.grad), _exact(q, k, v, do, causal, layout))}
    assert max(errs.values()) <= TOL_EXACT, f"normwise relative errors {errs}"


# ------------------------------------------------------------------------------------------- 4. determinism
def test_backward_is_bit_reproducible():
    import sageattention_b200 as sab
    q, k, v = _inputs(2, 8, 1000, 128, seed=7, Hkv=2)
    do = torch.randn(q.shape, generator=torch.Generator().manual_seed(8)).to(q.dtype).cuda()
    grads = []
    for _ in range(2):
        qg, kg, vg = (t.clone().requires_grad_(True) for t in (q, k, v))
        sab.sageattn(qg, kg, vg, is_causal=True).backward(do)
        grads.append((qg.grad, kg.grad, vg.grad))
    for a, b in zip(*grads):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------- 5. drop-in training
class _Block(torch.nn.Module):
    def __init__(self, dim=256, heads=4):
        super().__init__()
        self.heads = heads
        self.qkv = torch.nn.Linear(dim, 3 * dim)
        self.out = torch.nn.Linear(dim, dim)

    def forward(self, x):
        B, S, C = x.shape
        q, k, v = self.qkv(x).view(B, S, 3, self.heads, C // self.heads).permute(2, 0, 3, 1, 4)
        o = F.scaled_dot_product_attention(q, k, v)
        return self.out(o.transpose(1, 2).reshape(B, S, C))


def test_sdpa_monkey_patch_trains_every_parameter(monkeypatch):
    import sageattention_b200 as sab
    torch.manual_seed(0)
    ref = _Block().cuda().to(BF)
    pat = _Block().cuda().to(BF)
    pat.load_state_dict(ref.state_dict())
    x = torch.randn(2, 512, 256, device="cuda", dtype=BF)
    ref(x).float().square().mean().backward()
    monkeypatch.setattr(F, "scaled_dot_product_attention", sab.sageattn)
    pat(x).float().square().mean().backward()
    for (name, a), b in zip(ref.named_parameters(), pat.parameters()):
        assert b.grad is not None, name
        cos = F.cosine_similarity(a.grad.double().flatten(), b.grad.double().flatten(), dim=0).item()
        assert cos >= 0.999, f"{name}: cosine similarity {cos:.5f}"


# ------------------------------------------------------------------------------------------- 6. torch.compile
def test_torch_compile_fullgraph_gives_eager_gradients():
    import sageattention_b200 as sab
    q, k, v = _inputs(1, 2, 512, 64, seed=11)

    def loss(q, k, v):
        return sab.sageattn(q, k, v, is_causal=True).float().square().sum()

    def grads(f):
        qg, kg, vg = (t.clone().requires_grad_(True) for t in (q, k, v))
        f(qg, kg, vg).backward()
        return qg.grad, kg.grad, vg.grad

    eager = grads(loss)
    compiled = grads(torch.compile(loss, fullgraph=True))
    for a, b in zip(eager, compiled):
        assert torch.equal(a, b)
