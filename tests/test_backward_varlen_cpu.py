"""CPU checks of the packed varlen backward's definition and C-ABI boundary (no GPU):
  * attn_bwd_varlen_oracle.attn_bwd_varlen (what sab_qk_int8_attn_bwd_varlen computes) equals torch.autograd of ONE fp64 attention
    over all packed tokens with a block-diagonal mask (top-left causal inside each block), where the quantised logits are exact:
    integer-valued q, k in [-127, 127], a constant Q scale carrying sm_scale*log2e (the folded per-block path) and unit K scales;
  * sab_qk_int8_attn_bwd_varlen validates its arguments like the varlen forward, with the same status codes and messages, before it
    touches CUDA;
  * the new op is registered with a fake impl and mutates dq."""
import math

import numpy as np
import pytest
import torch

from attn_bwd_varlen_oracle import attn_bwd_varlen
from oracle import sage_oracle as O


def _packed_exact(q, k, v, do, lq, lk, causal, sm):
    """fp64 autograd of one attention over the packed tokens, key j visible to row i iff both belong to sequence b and (causal)
    j - cu_k[b] <= i - cu_q[b].  Rows that see no key output zero.  Returns (o, lse in log2 units, dq, dk, dv), packed."""
    q, k, v = (t.clone().double().requires_grad_(True) for t in (q, k, v))
    g = q.shape[1] // k.shape[1]
    seq_q = torch.repeat_interleave(torch.arange(len(lq)), torch.tensor(lq))
    seq_k = torch.repeat_interleave(torch.arange(len(lk)), torch.tensor(lk))
    pos_q = torch.cat([torch.arange(n) for n in lq]) if sum(lq) else torch.zeros(0, dtype=torch.long)
    pos_k = torch.cat([torch.arange(n) for n in lk]) if sum(lk) else torch.zeros(0, dtype=torch.long)
    mask = seq_q[:, None] == seq_k[None, :]
    if causal:
        mask &= pos_k[None, :] <= pos_q[:, None]
    s = torch.einsum("qhd,khd->hqk", q, k.repeat_interleave(g, 1)) * sm              # [Hq,Tq,Tk]
    s = s.masked_fill(~mask, float("-inf"))
    m = s.detach().amax(dim=-1, keepdim=True).nan_to_num(0.0, neginf=0.0)
    e = torch.exp(s - m)
    z = e.sum(dim=-1, keepdim=True)
    p = e / torch.where(z > 0, z, torch.ones_like(z))
    o = torch.einsum("hqk,khd->qhd", p, v.repeat_interleave(g, 1))
    (o * do.double()).sum().backward()
    lse = ((m + torch.log(z)).squeeze(-1) * O.LOG2E_CU).detach()                     # [Hq,Tq]
    return o.detach(), lse, q.grad, k.grad, v.grad


def _cu(lens):
    return torch.tensor([0] + list(np.cumsum(lens)), dtype=torch.int32)


def _cu_blocks(lens, blk):
    return torch.tensor([0] + list(np.cumsum([(n + blk - 1) // blk for n in lens])), dtype=torch.int32)


@pytest.mark.parametrize("lq,lk,Hq,Hk,D,causal", [
    ([5, 0, 1, 40, 17], [5, 0, 1, 40, 17], 2, 2, 64, False),
    ([5, 0, 1, 40, 17], [5, 0, 1, 40, 17], 2, 2, 64, True),
    ([30, 0, 12, 1], [70, 9, 12, 33], 4, 2, 64, False),          # Lq != Lk, a sequence with keys but no queries
    ([30, 0, 12, 1], [70, 9, 12, 33], 4, 1, 64, True),
    ([130, 3], [65, 140], 2, 2, 128, True),                        # more than one 128-row / 64-key scale block
])
def test_varlen_oracle_is_block_diagonal_autograd(lq, lk, Hq, Hk, D, causal):
    g = torch.Generator().manual_seed(sum(lq) * 7 + sum(lk) + Hq)
    Tq, Tk = sum(lq), sum(lk)
    q = torch.randint(-127, 128, (Tq, Hq, D), generator=g).double()
    k = torch.randint(-127, 128, (Tk, Hk, D), generator=g).double()
    v = torch.randn(Tk, Hk, D, generator=g, dtype=torch.float64)
    do = torch.randn(Tq, Hq, D, generator=g, dtype=torch.float64)
    sm = 1.0 / (127.0 * 127.0 * math.sqrt(D))
    o, lse, dq, dk, dv = _packed_exact(q, k, v, do, lq, lk, causal, sm)
    cq, ck, cqs, cks = _cu(lq), _cu(lk), _cu_blocks(lq, 128), _cu_blocks(lk, 64)
    q_scale = torch.full((int(cqs[-1]), Hq), sm * O.LOG2E_CU, dtype=torch.float64)   # sm_scale*log2e folded into the Q scale
    k_scale = torch.ones(int(cks[-1]), Hk, dtype=torch.float64)
    got = attn_bwd_varlen(q.to(torch.int8), k.to(torch.int8), q_scale, k_scale, q, k, v, o, do, lse, cq, ck, cqs, cks,
                          is_causal=causal, sm_scale=sm)
    for name, a, b in zip(("dq", "dk", "dv"), got, (dq, dk, dv)):
        assert a.shape == b.shape
        err = (a - b).abs().max().item() / b.abs().max().item()
        assert err <= 1e-10, f"{name}: relative error {err:.3e}"
    # a sequence with keys but no queries has zero dk / dv
    for i in range(len(lq)):
        if lq[i] == 0 and lk[i] > 0:
            s = slice(int(ck[i]), int(ck[i + 1]))
            assert not got[1][s].any() and not got[2][s].any()


def _fwd_varlen_args(Hq=2, Hkv=2, D=128, cu_k=16, ptr=16):
    """sab_qk_int8_sv_f16_attn, varlen form (2 sequences, 256 tokens), with non-null, 16-byte aligned dummy pointers: validation
    fails before anything is dereferenced."""
    return ([ptr] * 4 + [None, 16, 16] + [1, 2, Hq, Hkv, 256, 256, D] + [0] * 6 + [256] + [0] * 3 +
            [0, 1, 1, 1.0, 1] + [16, cu_k, 16, 16, 16] + [128, None])


def _bwd_varlen_args(Hq=2, Hkv=2, D=128, cu_k=16, ptr=16):
    """sab_qk_int8_attn_bwd_varlen arguments, likewise."""
    return [ptr] * 15 + [1, 2, Hq, Hkv, 256, 256, D] + [0] * 14 + [16, cu_k, 16, 16, 128, 128, 0, 1.0, 1, None]


def test_varlen_backward_abi_validates_like_the_forward():
    from sageattention_b200 import _capi
    lib = _capi.lib()
    cases = [
        (dict(D=96), -2, b"head dim"),                  # SAB_ERR_UNSUPPORTED
        (dict(Hq=3, Hkv=2), -1, b"divisible"),          # SAB_ERR_INVALID
        (dict(cu_k=None), -1, b"varlen needs"),
        (dict(ptr=None), -1, b"null tensor pointer"),
    ]
    for kw, code, text in cases:
        st = lib.sab_qk_int8_attn_bwd_varlen(*_bwd_varlen_args(**kw))
        msg = lib.sab_last_error()
        assert st == code and text in msg, (kw, st, msg)
        st_fwd = lib.sab_qk_int8_sv_f16_attn(*_fwd_varlen_args(**kw))
        msg_fwd = lib.sab_last_error()
        assert st_fwd == st and text in msg_fwd, (kw, st_fwd, msg_fwd)
        if text != b"varlen needs":                     # the backward's list of tables differs (no cu_pad_v, adds max_seqlen_k)
            assert msg == msg_fwd
    with pytest.raises(ValueError):
        _capi.check(lib.sab_qk_int8_attn_bwd_varlen(*_bwd_varlen_args(cu_k=None)))


def test_varlen_backward_op_is_registered_with_a_fake_impl():
    import sageattention_b200  # noqa: F401
    op = torch.ops.sageattention_b200.qk_int8_attn_bwd_varlen
    args = op.default._schema.arguments
    assert args[11].name == "dq" and args[11].alias_info.is_write
    assert all(a.alias_info is not None and a.alias_info.is_write for a in args[11:14])
    # the varlen forward op returns its LSE
    assert torch.ops.sageattention_b200.qk_int8_sv_f16_attn_varlen.default._schema.returns[0].type.kind() == "TensorType"
