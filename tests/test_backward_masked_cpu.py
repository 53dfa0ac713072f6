"""CPU checks of the masked backward's definition and C-ABI boundary (no GPU):
  * attn_bwd_masked_oracle.attn_bwd_masked (the formulas of sab_qk_int8_attn_bwd_masked, csrc/attn_bwd.cu) equals torch.autograd
    of fp64 softmax(q k^T sm + ln2 * bias) v where the quantised logits are exact (integer-valued q, k, unit scales), for dq, dk,
    dv and the bias gradient reduced over its broadcast dimensions, with bool and bias masks of every broadcast shape the entry
    point takes, -inf entries, fully masked rows and GQA;
  * sab_qk_int8_attn_bwd_masked validates its arguments with the masked forward's codes and messages before it touches CUDA;
  * the op mutates dq / dk / dv / dbias and has a fake implementation."""
import math

import pytest
import torch

from attn_bwd_masked_oracle import attn_bwd_masked
from attn_bwd_oracle import attn_bwd
from oracle import sage_oracle as O

LN2 = math.log(2.0)


def _mask(kind, shape, B, Hq, Sq, Sk, seed):
    """A mask of `shape` (broadcastable to [B,Hq,Sq,Sk]) with random masked / -inf entries, query row 1 fully masked (in every
    broadcast copy) and row 0 fully visible."""
    g = torch.Generator().manual_seed(seed)
    keep = torch.rand(shape, generator=g) > 0.3
    keep[..., 0, :] = True
    keep[..., 1, :] = False
    if kind == "bool":
        return keep
    return torch.where(keep, 2.0 * torch.randn(shape, generator=g, dtype=torch.float64), float("-inf"))


def _exact_masked(q, k, v, do, mask, sm):
    """fp64 autograd of softmax(q k^T sm + ln2 * bias) v (bool: False = -inf), GQA by repeating K/V heads; a row without a visible
    key outputs zeros, as the forward kernel does.  Returns (o, lse in log2 units, dq, dk, dv, dbias reduced to mask.shape)."""
    q, k, v = (t.clone().double().requires_grad_(True) for t in (q, k, v))
    g = q.shape[1] // k.shape[1]
    s = q @ k.repeat_interleave(g, 1).transpose(-1, -2) * sm
    bias = None
    if mask.dtype == torch.bool:
        s = s.masked_fill(~mask, float("-inf"))
    else:
        bias = mask.clone().requires_grad_(True)
        s = s + LN2 * bias
    row_visible = (s != float("-inf")).any(dim=-1, keepdim=True)
    p = torch.softmax(torch.where(row_visible, s, 0.0), dim=-1) * row_visible
    o = p @ v.repeat_interleave(g, 1)
    (o * do.double()).sum().backward()
    lse = torch.logsumexp(s, dim=-1) * O.LOG2E_CU
    return o.detach(), lse.detach(), q.grad, k.grad, v.grad, None if bias is None else bias.grad


def _ones(B, H, S, blk):
    return torch.ones(B, H, (S + blk - 1) // blk)


@pytest.mark.parametrize("kind", ["bool", "bias"])
@pytest.mark.parametrize("B,Hq,Hk,Sq,Sk,D,mshape", [
    (1, 2, 2, 70, 96, 64, "SS"),          # [Sq,Skv]
    (2, 4, 1, 33, 130, 64, "B1SS"),       # [B,1,Sq,Skv], GQA 4/1
    (1, 6, 2, 17, 150, 128, "1HSS"),      # [1,Hq,Sq,Skv], GQA 3/1: a mask that differs per Q head
])
def test_masked_oracle_is_autograd_where_logits_are_exact(kind, B, Hq, Hk, Sq, Sk, D, mshape):
    shape = {"SS": (Sq, Sk), "B1SS": (B, 1, Sq, Sk), "1HSS": (1, Hq, Sq, Sk)}[mshape]
    mask = _mask(kind, shape, B, Hq, Sq, Sk, seed=Sq + Sk)
    g = torch.Generator().manual_seed(Sq * 7 + Sk)
    q = torch.randint(-127, 128, (B, Hq, Sq, D), generator=g).float()
    k = torch.randint(-127, 128, (B, Hk, Sk, D), generator=g).float()
    v = torch.randn(B, Hk, Sk, D, generator=g)
    do = torch.randn(B, Hq, Sq, D, generator=g)
    sm = 1.0 / (127.0 * 127.0 * math.sqrt(D))    # keeps the integer logits in a softmax-friendly range
    o, lse, dq, dk, dv, dbias = _exact_masked(q, k, v, do, mask, sm)
    assert torch.isinf(lse[:, :, 1]).all() and torch.isfinite(lse[:, :, 0]).all()
    got = attn_bwd_masked(q.to(torch.int8), k.to(torch.int8), _ones(B, Hq, Sq, 128), _ones(B, Hk, Sk, 64), q, k, v, o, do, lse,
                          mask, q_gran="per_block", k_gran="per_block", sm_scale=sm)
    assert len(got) == 4 and got[3].shape == (B, Hq, Sq, Sk)
    want = (dq, dk, dv) + (() if dbias is None else (dbias,))
    for name, a, b in zip(("dq", "dk", "dv", "dbias"), got[:3] + (got[3].sum_to_size(mask.shape),), want):
        assert torch.isfinite(a).all(), name
        err = (a - b).abs().max().item() / b.abs().max().item()
        assert err <= 1e-10, f"{name}: relative error {err:.3e}"
    # the fully masked row: no gradient at all; masked and -inf positions: exactly 0 in dBias
    assert not got[0][:, :, 1].any() and not got[3][:, :, 1].any()
    hidden = ~mask if kind == "bool" else mask == float("-inf")
    assert not (got[3] * hidden).any()


def test_masked_oracle_without_mask_is_the_dense_oracle():
    """attn_mask of all True / all-zero bias: the dense oracle's gradient (to fp64 rounding: the extended operands sum more,
    zero, terms)."""
    g = torch.Generator().manual_seed(5)
    q = torch.randint(-127, 128, (1, 2, 40, 64), generator=g).float()
    k = torch.randint(-127, 128, (1, 2, 50, 64), generator=g).float()
    v, do = torch.randn(1, 2, 50, 64, generator=g), torch.randn(1, 2, 40, 64, generator=g)
    sm = 1e-5
    o, lse, *_ = _exact_masked(q, k, v, do, torch.ones(40, 50, dtype=torch.bool), sm)
    args = (q.to(torch.int8), k.to(torch.int8), _ones(1, 2, 40, 128), _ones(1, 2, 50, 64), q, k, v, o, do, lse)
    kw = dict(q_gran="per_block", k_gran="per_block", sm_scale=sm)
    dense = attn_bwd(*args, **kw)
    for m in (torch.ones(40, 50, dtype=torch.bool), torch.zeros(40, 50, dtype=torch.float64)):
        masked = attn_bwd_masked(*args, m, **kw)
        for x, y in zip(masked[:3], dense):
            assert ((x - y).abs().max() / y.abs().max()).item() <= 1e-12


# ------------------------------------------------------------------------------------------- C ABI
_FWD_MSG = b"attn_mask is supported by the dense non-causal fp16-PV path with per-block / per-warp K scales only"


def _bwd_masked_args(D=128, Hq=2, Hkv=2, k_gran=1, mask=16, kind=2, dbias=None, ptr=16):
    """sab_qk_int8_attn_bwd_masked arguments with non-null, 16-byte aligned dummy pointers: validation must fail before anything
    is dereferenced."""
    return ([ptr] * 15 + [1, 1, Hq, Hkv, 128, 128, D] + [0] * 21 + [1, k_gran, 1.0, 1] + [mask, kind] + [0] * 4 + [dbias, None])


@pytest.mark.parametrize("kw,code,text", [
    (dict(k_gran=3), -2, _FWD_MSG),                                 # per-thread K scales: the masked forward's refusal
    (dict(mask=None), -1, b"attn_mask: null pointer or unknown kind 2"),
    (dict(kind=3), -1, b"attn_mask: null pointer or unknown kind 3"),
    (dict(kind=1, dbias=32), -1, b"dbias needs an additive bias mask"),
    (dict(dbias=40), -1, b"dbias must be 16-byte aligned"),
    (dict(D=96), -2, b"head dim"),
    (dict(Hq=3), -1, b"divisible"),
    (dict(ptr=None), -1, b"null tensor pointer"),
])
def test_masked_backward_abi_validates_like_the_forward(kw, code, text):
    from sageattention_b200 import _capi
    lib = _capi.lib()
    st = lib.sab_qk_int8_attn_bwd_masked(*_bwd_masked_args(**kw))
    msg = lib.sab_last_error()
    assert st == code and text in msg, (kw, st, msg)
    if code == -1:
        with pytest.raises(ValueError):
            _capi.check(st)


def test_masked_backward_op_is_registered_with_a_fake_impl():
    import sageattention_b200  # noqa: F401
    from torch._library.simple_registry import singleton
    op = torch.ops.sageattention_b200.qk_int8_attn_bwd_masked
    args = op.default._schema.arguments
    names = [a.name for a in args]
    assert names[11:16] == ["dq", "dk", "dv", "attn_mask", "dbias"]
    for i in (11, 12, 13, 15):
        assert args[i].alias_info is not None and args[i].alias_info.is_write, names[i]
    assert args[14].alias_info is None or not args[14].alias_info.is_write   # the mask is read only
    assert singleton.find("sageattention_b200::qk_int8_attn_bwd_masked").fake_impl.kernel is not None
