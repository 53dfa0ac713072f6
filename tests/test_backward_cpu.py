"""CPU checks of the backward's definition and C-ABI boundary (no GPU):
  * attn_bwd_oracle.attn_bwd (the formulas the sm_90a gradient kernels implement, csrc/attn_bwd.cu) equals torch.autograd of fp64 attention
    where the quantised logits are exact: integer-valued q, k in [-127, 127] with unit scales;
  * sab_qk_int8_attn_bwd validates its arguments like the forward, with the same status codes and messages, before it touches CUDA."""
import math

import pytest
import torch

from attn_bwd_oracle import attn_bwd
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
