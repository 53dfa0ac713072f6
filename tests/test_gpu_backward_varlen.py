"""GPU tests (-m gpu) of the packed varlen backward (sab_qk_int8_attn_bwd_varlen, the autograd form of sageattn_varlen):
  1. the gradient kernels against the fp64 CPU oracle (attn_bwd_varlen_oracle.attn_bwd_varlen) on the kernel's own quantised
     operands and LSE;
  2. the packed backward equals, bit for bit, each sequence run alone;
  3. the forward is bit-identical with and without requires_grad inputs;
  4. sageattn_varlen gradients against fp64 autograd of exact per-sequence attention;
  5. bit-reproducibility and torch.compile; 6. training a packed-sequence block.

Tolerances, as for the dense backward (tests/test_gpu_backward.py):
  oracle      every element within the bound of attn_bwd_oracle (check_elementwise), derived from the kernels' rounding model
              (input-dtype rounding of P and dS, fp32 accumulation, ex2.approx).  Measured on an H100 80GB HBM3 (400 W power limit)
              over VARLEN_ORACLE_CASES: worst ratio of error to bound 0.997 (fp16 dk, in the case with a one-query sequence,
              whose keys' dK is one rounded term); normwise relative errors at most 2.4e-3 for bf16 and 3.0e-4 for fp16;
  TOL_EXACT   3e-2 (normwise ||g - g_ref|| / ||g_ref||): against exact attention the straight-through estimator also carries the
              INT8 quantisation of Q and K.  Measured on an H100 80GB HBM3 (700 W): 1.1-1.3 % for dq / dk / dv over the four cases
              below.
The oracle and exact-attention tests print their errors (pytest -s)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from attn_bwd_oracle import check_elementwise
from attn_bwd_varlen_oracle import attn_bwd_varlen

pytestmark = pytest.mark.gpu

TOL_EXACT = 3e-2
BF, FP = torch.bfloat16, torch.float16


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / b.norm()).item()


def _cu(lens, device="cuda"):
    return torch.tensor([0] + list(np.cumsum(lens)), dtype=torch.int32, device=device)


def _packed(lq, lk, Hq, Hk, D, dt, seed, k_offset=2.0):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(sum(lq), Hq, D, generator=g)
    k = torch.randn(sum(lk), Hk, D, generator=g) + k_offset * torch.randn(1, Hk, D, generator=g)   # per-channel offset
    v = torch.randn(sum(lk), Hk, D, generator=g)
    do = torch.randn(sum(lq), Hq, D, generator=g)
    return (t.to(dt).cuda() for t in (q, k, v, do))


# ------------------------------------------------------------------------------------------- 1. kernels vs oracle
# (lens_q, lens_k, Hq, Hkv, D, dtype).  The first two are the VARLEN_CASES of test_gpu_kernel_edges.py (empty and 1-token
# sequences, Lq != Lk); the last two add GQA 8/1, 17 and 127 / 128 / 129 tokens, sequences with keys but no queries and one of
# more than 1500 tokens.
VARLEN_ORACLE_CASES = [
    ([200, 0, 1, 130, 77], [333, 0, 1, 64, 300], 4, 2, 128, BF),
    ([1, 300, 0, 64, 129], [257, 100, 0, 1, 129], 2, 2, 64, FP),
    ([17, 0, 127, 128, 1600], [17, 90, 128, 129, 1500], 8, 1, 128, FP),
    ([129, 0, 17, 1], [127, 40, 17, 1], 8, 1, 64, BF),
]


@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("case", VARLEN_ORACLE_CASES, ids=lambda c: f"D{c[4]}-H{c[2]}x{c[3]}-{str(c[5])[6:]}")
def test_varlen_gradient_kernels_match_oracle(case, causal):
    import sageattention_b200 as sab
    from sageattention_b200 import ops
    from sageattention_b200.quant import per_block_int8_varlen, transpose_v_f16_varlen
    lq, lk, Hq, Hk, D, dt = case
    q, k, v, do = _packed(lq, lk, Hq, Hk, D, dt, seed=sum(lq) + 3 * sum(lk) + D)
    cq, ck = _cu(lq), _cu(lk)
    sm = D ** -0.5
    km = sab.k_mean(k.unsqueeze(0), "NHD").view(Hk, D)          # the mean over all packed tokens, as sageattn_varlen
    q8, qs, k8, ks, cqs, cks = per_block_int8_varlen(q, k, cq, ck, max(lq), max(lk), sm_scale=sm, km=km)
    v_t, cu_pad = transpose_v_f16_varlen(v, ck, max(lk))
    o = torch.empty_like(q)
    lse = ops.qk_int8_sv_f16_attn_varlen(q8, k8, v_t, o, qs, ks, cq, ck, cu_pad, cqs, cks, max(lq), int(causal), sm, 1, 1)
    # NaN-filled outputs: every row of every sequence must be written, including zero dk / dv of keys without queries
    dq, dk, dv = (torch.full_like(t, float("nan")) for t in (q, k, v))
    ops.qk_int8_attn_bwd_varlen(q8, k8, qs, ks, q, k, v, o, do, lse, km, dq, dk, dv, cq, ck, cqs, cks, max(lq), max(lk), int(causal),
                                sm, 1)
    torch.cuda.synchronize()
    *ref, bounds = attn_bwd_varlen(q8.cpu(), k8.cpu(), qs.cpu(), ks.cpu(), q.cpu(), k.cpu(), v.cpu(), o.cpu(), do.cpu(), lse.cpu(),
                                   cq.cpu(), ck.cpu(), cqs.cpu(), cks.cpu(), is_causal=causal, sm_scale=sm, k_mean=km.cpu(), bound=True)
    res = {name: check_elementwise(name, got.cpu(), r, b, dims=("token", "h", "col"))
           for name, got, r, b in zip(("dq", "dk", "dv"), (dq, dk, dv), ref, bounds)}
    print(f"[oracle] {case[:5]} {str(dt)[6:]} causal={causal}: " + ", ".join(f"{n} ratio {w:.3f} normwise {e:.2e}"
                                                                          for n, (w, e) in res.items()))
    for i in range(len(lq)):
        if lq[i] == 0 and lk[i] > 0:
            s = slice(int(ck[i]), int(ck[i + 1]))
            assert not dk[s].any() and not dv[s].any(), f"sequence {i}: keys without queries must get zero dk / dv"


# ------------------------------------------------------------------------------------------- 2. packed == per sequence
@pytest.mark.parametrize("causal", [False, True])
def test_varlen_backward_equals_each_sequence_alone(causal):
    """smooth_k=False: each sequence's quantised operands do not depend on the others, so the packed backward must give the same
    bits as each sequence alone.  Checks token offsets, scale blocks and LSE rows exactly."""
    import sageattention_b200 as sab
    lens = [512, 130, 77, 1000, 64]
    Hq, Hk, D = 8, 2, 128
    q, k, v, do = _packed(lens, lens, Hq, Hk, D, FP, seed=3)
    cu = _cu(lens)

    def grads(q, k, v, do, cu, L):
        qg, kg, vg = (t.clone().requires_grad_(True) for t in (q, k, v))
        sab.sageattn_varlen(qg, kg, vg, cu, cu, L, L, is_causal=causal, smooth_k=False).backward(do)
        return qg.grad, kg.grad, vg.grad

    packed = grads(q, k, v, do, cu, max(lens))
    for i, L in enumerate(lens):
        s = slice(int(cu[i]), int(cu[i + 1]))
        alone = grads(q[s].contiguous(), k[s].contiguous(), v[s].contiguous(), do[s].contiguous(), _cu([L]), L)
        for name, a, b in zip(("dq", "dk", "dv"), packed, alone):
            assert torch.equal(a[s], b), f"sequence {i}: {name}"


# ------------------------------------------------------------------------------------------- 3. no behaviour change
@pytest.mark.parametrize("causal", [False, True])
def test_varlen_forward_unchanged_by_requires_grad(causal):
    import sageattention_b200 as sab
    lens = [100, 0, 257, 1]
    q, k, v, _ = _packed(lens, lens, 4, 2, 96, BF, seed=1)
    cu = _cu(lens)
    with torch.no_grad():
        o0 = sab.sageattn_varlen(q, k, v, cu, cu, max(lens), max(lens), is_causal=causal)
    qg, kg, vg = (t.clone().requires_grad_(True) for t in (q, k, v))
    o1 = sab.sageattn_varlen(qg, kg, vg, cu, cu, max(lens), max(lens), is_causal=causal)
    assert o1.requires_grad and o1.grad_fn is not None
    assert torch.equal(o0, o1.detach())
    o1.float().square().sum().backward()
    assert all(t.grad is not None and torch.isfinite(t.grad).all() for t in (qg, kg, vg))


# ------------------------------------------------------------------------------------------- 4. public API vs exact attention
def _exact_per_sequence(q, k, v, do, lq, lk, causal):
    """fp64 autograd of exact attention run on each sequence alone (top-left causal), packed."""
    q, k, v = (t.detach().cpu().double().requires_grad_(True) for t in (q, k, v))
    cq, ck = np.cumsum([0] + lq), np.cumsum([0] + lk)
    g = q.shape[1] // k.shape[1]
    outs = []
    for i in range(len(lq)):
        qi = q[cq[i]:cq[i + 1]].transpose(0, 1)
        ki, vi = (t[ck[i]:ck[i + 1]].transpose(0, 1).repeat_interleave(g, 0) for t in (k, v))
        s = qi @ ki.transpose(-1, -2) * q.shape[-1] ** -0.5
        if causal:
            s = s.masked_fill(torch.arange(s.shape[-1])[None, :] > torch.arange(s.shape[-2])[:, None], float("-inf"))
        outs.append((torch.softmax(s, -1) @ vi).transpose(0, 1))
    (torch.cat(outs) * do.cpu().double()).sum().backward()
    return q.grad, k.grad, v.grad


@pytest.mark.parametrize("lq,lk,D,causal,dt", [
    ([1024, 300, 2048], [1024, 300, 2048], 128, False, BF),
    ([1024, 300, 2048], [1024, 300, 2048], 128, True, FP),
    ([700, 64, 1500], [900, 64, 1500], 96, False, FP),        # head-dim padding, Lq != Lk
    ([513, 1200], [513, 1200], 64, True, BF),
])
def test_sageattn_varlen_gradients_match_exact_attention(lq, lk, D, causal, dt):
    import sageattention_b200 as sab
    q, k, v, do = _packed(lq, lk, 4, 2, D, dt, seed=sum(lq) + D, k_offset=1.5)
    q, k, v = (t.requires_grad_(True) for t in (q, k, v))
    o = sab.sageattn_varlen(q, k, v, _cu(lq), _cu(lk), max(lq), max(lk), is_causal=causal)
    o.backward(do)
    ref = _exact_per_sequence(q, k, v, do, lq, lk, causal)
    errs = {name: _rel(got, r) for name, got, r in zip(("dq", "dk", "dv"), (q.grad, k.grad, v.grad), ref)}
    print(f"[exact] lq={lq} lk={lk} D={D} causal={causal} {str(dt)[6:]}: " + ", ".join(f"{n} {e:.2e}" for n, e in errs.items()))
    assert max(errs.values()) <= TOL_EXACT, f"normwise relative errors {errs}"


# ------------------------------------------------------------------------------------------- 5. determinism, torch.compile
def test_varlen_backward_is_bit_reproducible():
    import sageattention_b200 as sab
    lens = [1000, 17, 0, 640]
    q, k, v, do = _packed(lens, lens, 8, 2, 128, BF, seed=7)
    cu = _cu(lens)
    grads = []
    for _ in range(2):
        qg, kg, vg = (t.clone().requires_grad_(True) for t in (q, k, v))
        sab.sageattn_varlen(qg, kg, vg, cu, cu, max(lens), max(lens), is_causal=True).backward(do)
        grads.append((qg.grad, kg.grad, vg.grad))
    for a, b in zip(*grads):
        assert torch.equal(a, b)


def test_varlen_torch_compile_fullgraph_gives_eager_gradients():
    import sageattention_b200 as sab
    lens = [300, 64, 129]
    q, k, v, _ = _packed(lens, lens, 2, 2, 64, FP, seed=11)
    cu = _cu(lens)

    def loss(q, k, v):
        return sab.sageattn_varlen(q, k, v, cu, cu, max(lens), max(lens), is_causal=True).float().square().sum()

    def grads(f):
        qg, kg, vg = (t.clone().requires_grad_(True) for t in (q, k, v))
        f(qg, kg, vg).backward()
        return qg.grad, kg.grad, vg.grad

    eager = grads(loss)
    compiled = grads(torch.compile(loss, fullgraph=True))
    for a, b in zip(eager, compiled):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------- 6. training a packed block
class _PackedBlock(torch.nn.Module):
    def __init__(self, attn, dim=256, heads=4):
        super().__init__()
        self.attn, self.heads = attn, heads
        self.qkv = torch.nn.Linear(dim, 3 * dim)
        self.out = torch.nn.Linear(dim, dim)

    def forward(self, x, cu, lens):
        T, C = x.shape
        q, k, v = self.qkv(x).view(T, 3, self.heads, C // self.heads).unbind(1)      # packed [T,H,Dh] views
        return self.out(self.attn(q, k, v, cu, lens).reshape(T, C))


def _sdpa_per_sequence(q, k, v, cu, lens):
    outs = []
    for i in range(len(lens)):
        s = slice(int(cu[i]), int(cu[i + 1]))
        if lens[i] == 0:
            continue
        outs.append(F.scaled_dot_product_attention(*(t[s].transpose(0, 1) for t in (q, k, v)), is_causal=True).transpose(0, 1))
    return torch.cat(outs)


def test_packed_block_trains_every_parameter():
    import sageattention_b200 as sab
    torch.manual_seed(0)
    lens = [300, 512, 77, 0, 1000]
    cu = _cu(lens)
    ref = _PackedBlock(_sdpa_per_sequence).cuda().to(BF)
    pat = _PackedBlock(lambda q, k, v, cu, lens: sab.sageattn_varlen(q, k, v, cu, cu, max(lens), max(lens), is_causal=True))
    pat = pat.cuda().to(BF)
    pat.load_state_dict(ref.state_dict())
    x = torch.randn(sum(lens), 256, device="cuda", dtype=BF)
    ref(x, cu, lens).float().square().mean().backward()
    pat(x, cu, lens).float().square().mean().backward()
    for (name, a), b in zip(ref.named_parameters(), pat.parameters()):
        assert b.grad is not None, name
        cos = F.cosine_similarity(a.grad.double().flatten(), b.grad.double().flatten(), dim=0).item()
        assert cos >= 0.999, f"{name}: cosine similarity {cos:.5f}"
