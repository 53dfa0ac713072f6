"""CPU checks of the backward's definition and C-ABI boundary (no GPU):
  * attn_bwd_oracle.attn_bwd (the formulas the sm_90a gradient kernels implement, csrc/attn_bwd.cu) equals torch.autograd of fp64 attention
    where the quantised logits are exact: integer-valued q, k in [-127, 127] with unit scales;
  * its row-chunked evaluation equals the whole call, and its elementwise bound holds for a CPU emulation of the kernels'
    arithmetic (fp32 logits and sums, P and dS rounded to the input dtype) but not for that emulation with one planted mistake;
  * sab_qk_int8_attn_bwd validates its arguments like the forward, with the same status codes and messages, before it touches CUDA."""
import math

import pytest
import torch
import torch.nn.functional as F

from attn_bwd_oracle import attn_bwd, check_elementwise, elementwise_ratio
from oracle import sage_oracle as O


def _exact_grads(q, k, v, do, causal, sm):
    """fp64 autograd of softmax(q k^T sm) v (GQA by repeating K/V heads): (o, lse in log2 units, dq, dk, dv)."""
    q, k, v = (t.clone().double().requires_grad_(True) for t in (q, k, v))
    g = q.shape[1] // k.shape[1]
    s = q @ k.repeat_interleave(g, 1).transpose(-1, -2) * sm
    if causal:
        s = s.masked_fill(torch.arange(s.shape[-1])[None, :] > torch.arange(s.shape[-2])[:, None], float("-inf"))
    o = torch.softmax(s, dim=-1) @ v.repeat_interleave(g, 1)
    (o * do.double()).sum().backward()
    lse = torch.logsumexp(s, dim=-1) * O.LOG2E_CU
    return o.detach(), lse.detach(), q.grad, k.grad, v.grad


def _scale_ones(B, H, S, gran, key):
    n = (S + 63) // 64 * (4 if gran == "per_thread" else 1) if key else (S + 127) // 128 * {"per_block": 1, "per_warp": 4, "per_thread": 32}[gran]
    return torch.ones(B, H, n)


@pytest.mark.parametrize("B,Hq,Hk,Sq,Sk,D,causal,gran", [
    (1, 2, 2, 96, 96, 64, False, "per_thread"),
    (1, 2, 2, 130, 130, 64, True, "per_thread"),
    (2, 2, 2, 70, 200, 128, False, "per_warp"),
    (1, 4, 1, 65, 65, 64, True, "per_block"),
    (1, 6, 2, 17, 150, 64, False, "per_thread"),
])
def test_oracle_attn_bwd_is_autograd_where_logits_are_exact(B, Hq, Hk, Sq, Sk, D, causal, gran):
    g = torch.Generator().manual_seed(Sq * 7 + Sk)
    q = torch.randint(-127, 128, (B, Hq, Sq, D), generator=g).float()
    k = torch.randint(-127, 128, (B, Hk, Sk, D), generator=g).float()
    v = torch.randn(B, Hk, Sk, D, generator=g)
    do = torch.randn(B, Hq, Sq, D, generator=g)
    sm = 1.0 / (127.0 * 127.0 * math.sqrt(D))    # keeps the integer logits in a softmax-friendly range
    o, lse, dq, dk, dv = _exact_grads(q, k, v, do, causal, sm)
    kgran = "per_block" if gran != "per_thread" else gran
    got = attn_bwd(q.to(torch.int8), k.to(torch.int8), _scale_ones(B, Hq, Sq, gran, False), _scale_ones(B, Hk, Sk, kgran, True),
                     q, k, v, o, do, lse, q_gran=gran, k_gran=kgran, is_causal=causal, sm_scale=sm)
    for name, a, b in zip(("dq", "dk", "dv"), got, (dq, dk, dv)):
        err = (a - b).abs().max().item() / b.abs().max().item()
        assert err <= 1e-10, f"{name}: relative error {err:.3e}"


def test_oracle_attn_bwd_folded_scale_matches_unfolded():
    """fold_sm_scale: sm_scale*log2e carried by q_scale gives the same gradient."""
    g = torch.Generator().manual_seed(3)
    q = torch.randint(-127, 128, (1, 2, 40, 64), generator=g).float()
    k = torch.randint(-127, 128, (1, 2, 50, 64), generator=g).float()
    v, do = torch.randn(1, 2, 50, 64, generator=g), torch.randn(1, 2, 40, 64, generator=g)
    sm = 1e-5
    o, lse, *_ = _exact_grads(q, k, v, do, False, sm)
    qs, ks = _scale_ones(1, 2, 40, "per_block", False), _scale_ones(1, 2, 50, "per_block", True)
    a = attn_bwd(q.to(torch.int8), k.to(torch.int8), qs, ks, q, k, v, o, do, lse, q_gran="per_block", sm_scale=sm)
    b = attn_bwd(q.to(torch.int8), k.to(torch.int8), qs * sm * O.LOG2E_CU, ks, q, k, v, o, do, lse, q_gran="per_block",
                   sm_scale=sm, fold_sm_scale=True)
    for x, y in zip(a, b):
        assert ((x - y).norm() / y.norm()).item() <= 1e-6   # q_scale is fp32


# ------------------------------------------------------------------------------------------- elementwise bound
def _quantised_case(B, Hq, Hk, S, D, dt, causal, seed, k_offset=2.0):
    """Operands as the kernels receive them: per-block INT8 q (128 rows) and smoothed k (64 keys), the K mean, the forward's
    log2 LSE (fp32) and an O carrying FP8 P / V roundings, as the quantised forward's does.  sm_scale = D^-0.5, not folded."""
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(B, Hq, S, D, generator=g).to(dt)
    k = (torch.randn(B, Hk, S, D, generator=g) + k_offset * torch.randn(D, generator=g)).to(dt)
    v = torch.randn(B, Hk, S, D, generator=g).to(dt)
    do = torch.randn(B, Hq, S, D, generator=g).to(dt)
    km = k.float().mean(dim=2, keepdim=True).to(dt)

    def quant(x, blk):
        n = (S + blk - 1) // blk
        xp = F.pad(x.float(), (0, 0, 0, n * blk - S)).view(B, x.shape[1], n, blk, D)
        sc = (xp.abs().amax(dim=(-1, -2)) / 127.0).clamp_min(1e-8)
        return (xp / sc[..., None, None]).round().clamp(-127, 127).view(B, x.shape[1], n * blk, D)[:, :, :S].to(torch.int8), sc

    q8, qs = quant(q, 128)
    k8, ks = quant(k - km, 64)
    sm = D ** -0.5
    G = Hq // Hk
    qsr = qs.repeat_interleave(128, 2)[:, :, :S, None].double()
    ksr = ks.repeat_interleave(64, 2)[:, :, None, :S].double().repeat_interleave(G, 1)
    s = (q8.double() @ k8.double().repeat_interleave(G, 1).transpose(-1, -2)) * qsr * ksr * sm * O.LOG2E_CU
    if causal:
        s = s.masked_fill(torch.ones(S, S, dtype=torch.bool).triu(1), -math.inf)
    lse = (torch.logsumexp(s * math.log(2.0), dim=-1) / math.log(2.0)).float()
    p8 = torch.exp2(s - lse.double()[..., None]).to(torch.float8_e4m3fn).double()
    o = (p8 @ v.to(torch.float8_e4m3fn).double().repeat_interleave(G, 1)).to(dt)
    return dict(q8=q8, k8=k8, qs=qs, ks=ks, q=q, k=k, v=v, o=o, do=do, lse=lse, km=km, sm=sm, causal=causal)


MISTAKES = ("k_scale", "k_mean", "delta_row", "gqa_head", "tail_tile", "causal_diag")


def _emulate(c, mistake=None):
    """The kernels' arithmetic on the CPU (csrc/attn_bwd.cu): fp32 coefficient, logit and exp2, fp32 dP / delta sums, P and dS
    rounded to the input dtype before fp32-accumulated dV, dQ, dK products, one rounding of each result.  The dQ pass and the
    dK/dV pass compute P separately, as the two kernels do.  mistake (one of MISTAKES) plants one error:
      k_scale     one 64-key block's K scale off by 2^-4 in one 128-row Q tile of the dQ pass;
      k_mean      dQ taken with K instead of K - mean;
      delta_row   delta of the next row;
      gqa_head    the dS of Q head 1 (of KV head 0's group) added to KV head 1's dK;
      tail_tile   the last, partial, 64-key tile dropped (dQ loop and dK / dV stores);
      causal_diag the causal diagonal excluded."""
    q8, k8, q, k, v, o, do = (c[n] for n in ("q8", "k8", "q", "k", "v", "o", "do"))
    T = q.dtype
    B, Hq, S, D = q.shape
    Hk = k.shape[1]
    G = Hq // Hk
    f32 = torch.float32
    sm32 = torch.tensor(c["sm"], dtype=f32)
    qss = c["qs"].repeat_interleave(128, 2)[:, :, :S] * (sm32 * torch.tensor(O.LOG2E_CU, dtype=f32))
    ks = c["ks"].repeat_interleave(64, 2)[:, :, :S].repeat_interleave(G, 1)
    s32 = (q8.double() @ k8.double().repeat_interleave(G, 1).transpose(-1, -2)).float()   # exact integers
    diag = 0 if mistake == "causal_diag" else 1
    visible = torch.ones(S, S, dtype=torch.bool).tril(-1 + diag) if c["causal"] else torch.ones(S, S, dtype=torch.bool)

    def p_of(coef):
        return torch.where(visible, torch.exp2(s32 * coef - c["lse"][..., None]), torch.zeros((), dtype=f32))

    coef = qss[..., None] * ks[:, :, None, :]
    p_kv = p_of(coef)
    coef_q = coef.clone()
    if mistake == "k_scale":
        coef_q[:, :, 128:256, 64:128] = qss[:, :, 128:256, None] * (ks[:, :, None, 64:128] * (1 + 2.0 ** -4))
    p_q = p_of(coef_q)
    tail = S // 64 * 64
    if mistake == "tail_tile":
        p_q[..., tail:] = 0
    dp = do.float() @ v.float().repeat_interleave(G, 1).transpose(-1, -2)
    delta = (do.float() * o.float()).sum(-1, keepdim=True)
    if mistake == "delta_row":
        delta = torch.roll(delta, -1, dims=2)
    ds_q = (p_q * (dp - delta)).to(T).float()
    ds_kv = (p_kv * (dp - delta)).to(T).float()
    kc = k if mistake == "k_mean" else k - c["km"]
    dq = (ds_q @ kc.float().repeat_interleave(G, 1)) * sm32
    dk_h = ds_kv.transpose(-1, -2) @ q.float()
    dv_h = p_kv.to(T).float().transpose(-1, -2) @ do.float()
    if mistake == "gqa_head":
        dk_h = dk_h.clone()
        dk_h[:, 1], dk_h[:, G] = 0, dk_h[:, G] + dk_h[:, 1]   # head 1 belongs to KV head 0, G is KV head 1's first
    dk = dk_h.view(B, Hk, G, S, D).sum(2) * sm32
    dv = dv_h.view(B, Hk, G, S, D).sum(2)
    if mistake == "tail_tile":
        dk[:, :, tail:], dv[:, :, tail:] = 0, 0
    return dq.to(T), dk.to(T), dv.to(T)


def _oracle(c, bound=True, **kw):
    return attn_bwd(c["q8"], c["k8"], c["qs"], c["ks"], c["q"], c["k"], c["v"], c["o"], c["do"], c["lse"], q_gran="per_block",
                    k_gran="per_block", is_causal=c["causal"], sm_scale=c["sm"], k_mean=c["km"], bound=bound, **kw)


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("causal", [False, True])
def test_emulated_kernel_arithmetic_is_inside_the_bound(dt, causal):
    c = _quantised_case(1, 4, 2, 200, 64, dt, causal, seed=11)
    *ref, bounds = _oracle(c)
    for name, got, r, b in zip(("dq", "dk", "dv"), _emulate(c), ref, bounds):
        worst, norm = check_elementwise(name, got, r, b)
        print(f"{name} {str(dt)[6:]} causal={causal}: ratio {worst:.3f}, normwise {norm:.2e}")


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("mistake", MISTAKES)
def test_each_planted_mistake_breaks_the_bound(mistake, dt):
    c = _quantised_case(1, 4, 2, 200, 64, dt, True, seed=11)
    *ref, bounds = _oracle(c)
    worst = max(float(elementwise_ratio(got, r, b).max()) for got, r, b in zip(_emulate(c, mistake), ref, bounds))
    assert worst > 1.0, f"{mistake}: worst ratio {worst:.3f} stays inside the bound"


def test_check_elementwise_reports_the_worst_element():
    ref = torch.zeros(1, 2, 3, 4, dtype=torch.float64)
    bound = torch.full_like(ref, 1e-3)
    got = ref.to(torch.bfloat16)
    got[0, 1, 2, 3] = 0.5
    with pytest.raises(AssertionError, match=r"at \(b=0, h=1, row=2, col=3\)"):
        check_elementwise("dq", got, ref, bound)
    got[0, 1, 2, 3] = float("nan")          # an unwritten (NaN-filled) element fails whatever the bound
    with pytest.raises(AssertionError, match="1 non-finite"):
        check_elementwise("dq", got, ref, torch.full_like(ref, math.inf))


@pytest.mark.parametrize("causal", [False, True])
def test_row_chunks_sum_to_the_whole_call(causal):
    """dQ rows and bounds by chunk equal the whole call's; dK / dV and their bounds are the chunks' sums.  The chunk edges (70,
    128) are not all multiples of the 128-row scale blocks, and causal masking follows the global row."""
    c = _quantised_case(1, 4, 2, 200, 64, torch.bfloat16, causal, seed=5)
    dq, dk, dv, (bq, bk, bv) = _oracle(c)
    parts = []
    for r0, r1 in ((0, 70), (70, 128), (128, 200)):
        sub = dict(c, **{n: c[n][:, :, r0:r1] for n in ("q8", "q", "o", "do", "lse")})
        parts.append(_oracle(sub, q_offset=r0, q_len=200))
    torch.testing.assert_close(torch.cat([p[0] for p in parts], 2), dq, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(torch.cat([p[3][0] for p in parts], 2), bq, rtol=1e-12, atol=0)
    for i, whole, bound in ((1, dk, bk), (2, dv, bv)):
        torch.testing.assert_close(sum(p[i] for p in parts), whole, rtol=1e-10, atol=1e-12)
        torch.testing.assert_close(sum(p[3][i] for p in parts), bound, rtol=1e-10, atol=0)


def _bwd_args(Hq=2, Hkv=2, Sq=128, Skv=128, D=128, causal=0, ptr=1):
    """sab_qk_int8_attn_bwd arguments with non-null dummy pointers: validation must fail before anything is dereferenced."""
    return ([ptr] * 15 + [1, 1, Hq, Hkv, Sq, Skv, D] + [0] * 21 + [causal, 3, 3, 1.0, 0, None])


def test_backward_abi_validates_like_the_forward():
    from sageattention_b200 import _capi
    lib = _capi.lib()
    assert lib.sab_attn_bwd_workspace_bytes(2, 4, 100) >= 2 * 4 * 100 * 4
    # head dim: SAB_ERR_UNSUPPORTED with the forward's message
    st = lib.sab_qk_int8_attn_bwd(*_bwd_args(D=96))
    assert st == -2 and b"head dim" in lib.sab_last_error()
    st_fwd = lib.sab_qk_int8_sv_f8_attn(*([1] * 4), None, 1, 1, None, None, 0, 1, 2, 2, 128, 128, 96, *([0] * 10), 0, 2, 2, 1.0, 0,
                                        *([None] * 5), 0, 0, 0, None, None)
    assert st_fwd == st
    # GQA divisibility: SAB_ERR_INVALID, same message as the forward
    st = lib.sab_qk_int8_attn_bwd(*_bwd_args(Hq=3, Hkv=2))
    msg = lib.sab_last_error()
    assert st == -1 and b"divisible" in msg
    lib.sab_qk_int8_sv_f8_attn(*([1] * 4), None, 1, 1, None, None, 0, 1, 3, 2, 128, 128, 128, *([0] * 10), 0, 2, 2, 1.0, 0,
                               *([None] * 5), 0, 0, 0, None, None)
    assert lib.sab_last_error() == msg
    with pytest.raises(ValueError):
        _capi.check(st)
    # causal needs Sq == Skv (the Python entry points' assertion message)
    st = lib.sab_qk_int8_attn_bwd(*_bwd_args(Sq=128, Skv=256, causal=1))
    assert st == -1 and b"qo_len and kv_len must be equal for causal attention" in lib.sab_last_error()
    # null pointers
    st = lib.sab_qk_int8_attn_bwd(*_bwd_args(ptr=None))
    assert st == -1 and b"null" in lib.sab_last_error()


def test_backward_op_is_registered_with_a_fake_impl():
    import sageattention_b200  # noqa: F401
    op = torch.ops.sageattention_b200.qk_int8_attn_bwd
    assert op.default._schema.arguments[11].alias_info.is_write   # dq mutated
