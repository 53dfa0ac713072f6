"""CPU tests of the oracle's block evaluation (oracle/sage_oracle.py attn_int8_fp8_cuda, `causal_q_offset`) and of its `v_mean`
epilogue.  The GPU tests compare whole 128-row blocks of long sequences, and the sequence-parallel segments, against the oracle
run on one block of Q at a time; that is only sound if a block evaluated on its own is bit-identical to the same rows of the
full evaluation."""
import pytest
import torch

from oracle import sage_oracle as O

BM = 128


def _operands(S, D, gran, seed, Hq=2, Hk=1, B=1):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(B, Hq, S, D, generator=g).half()
    k = (torch.randn(B, Hk, S, D, generator=g) + 4.0 * torch.randn(B, Hk, 1, D, generator=g)).half()
    v = torch.randn(B, Hk, S, D, generator=g).half()
    km = k.mean(dim=2, keepdim=True)
    if gran == "per_warp":
        q8, qs, k8, ks = O.per_warp_int8_cuda(q, k, km)
    else:
        q8, qs, k8, ks = O.quant_per_thread_int8_triton(q, k, km)
    v8, vs, _ = O.per_channel_fp8_cuda(v, "HND", 448.0)
    return q8, qs, k8, ks, v8, vs


def _q_block(q8, qs, gran, r0):
    """Rows r0..r0+127 of Q (fewer at a ragged end) with their Q scales: 4 per 128-row block per warp, 32 per thread."""
    per = 4 if gran == "per_warp" else 32
    b = r0 // BM
    return q8[:, :, r0:r0 + BM], qs[:, :, b * per:(b + 1) * per].contiguous()


@pytest.mark.parametrize("gran", ["per_warp", "per_thread"])
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("tau", [None, 4])
def test_block_evaluation_equals_rows_of_full_evaluation(gran, causal, tau):
    S, D = 600, 64                     # 4 whole blocks + a ragged last block of 88 rows; a partial last K tile
    q8, qs, k8, ks, v8, vs = _operands(S, D, gran, seed=1)
    kw = dict(qk_quant_gran=gran, is_causal=causal, sm_scale=D ** -0.5, out_dtype=torch.float32, return_lse=True, lazy_tau=tau)
    full, full_lse = O.attn_int8_fp8_cuda(q8, k8, v8, qs, ks, vs, **kw)
    for r0 in (0, 256, 512):
        qb, qsb = _q_block(q8, qs, gran, r0)
        o, lse = O.attn_int8_fp8_cuda(qb, k8, v8, qsb, ks, vs, causal_q_offset=r0, **kw)
        assert torch.equal(o, full[:, :, r0:r0 + BM]), (gran, causal, tau, r0)
        assert torch.equal(lse, full_lse[:, :, r0:r0 + BM]), (gran, causal, tau, r0)


def test_causal_q_offset_without_causal_changes_nothing():
    q8, qs, k8, ks, v8, vs = _operands(256, 64, "per_thread", seed=2)
    kw = dict(sm_scale=0.125, out_dtype=torch.float32, lazy_tau=4)
    assert torch.equal(O.attn_int8_fp8_cuda(q8, k8, v8, qs, ks, vs, **kw),
                       O.attn_int8_fp8_cuda(q8, k8, v8, qs, ks, vs, causal_q_offset=128, **kw))


def test_causal_q_offset_hides_only_future_keys():
    """Rows at a global offset r0 see keys 0..r0+row: the result equals non-causal attention over exactly those keys for the
    first row of the block (its visible keys are a prefix) — a check of the mask that does not go through the block identity."""
    S, D = 384, 64
    q8, qs, k8, ks, v8, vs = _operands(S, D, "per_warp", seed=3)
    r0 = 256
    qb, qsb = _q_block(q8, qs, "per_warp", r0)
    kw = dict(qk_quant_gran="per_warp", sm_scale=D ** -0.5, out_dtype=torch.float32)
    o = O.attn_int8_fp8_cuda(qb, k8, v8, qsb, ks, vs, is_causal=True, causal_q_offset=r0, **kw)
    n = r0 + 1                           # row 0 of the block sees keys 0..r0
    ksn = ks[:, :, :(n + 63) // 64]
    o0 = O.attn_int8_fp8_cuda(qb[:, :, :1], k8[:, :, :n], v8[:, :, :n], qsb, ksn, vs, **kw)
    assert torch.equal(o[:, :, :1], o0)


def test_v_mean_is_added_after_the_v_scale():
    q8, qs, k8, ks, v8, vs = _operands(200, 128, "per_thread", seed=4, Hq=4, Hk=2)
    kw = dict(sm_scale=128 ** -0.5, out_dtype=torch.float32, lazy_tau=4)
    base = O.attn_int8_fp8_cuda(q8, k8, v8, qs, ks, vs, **kw)
    assert torch.equal(O.attn_int8_fp8_cuda(q8, k8, v8, qs, ks, vs, v_mean=torch.zeros_like(vs), **kw), base)
    vm = torch.randn(vs.shape, generator=torch.Generator().manual_seed(5))
    got = O.attn_int8_fp8_cuda(q8, k8, v8, qs, ks, vs, v_mean=vm, **kw)
    assert torch.equal(got, base + vm.repeat_interleave(2, dim=1)[:, :, None, :])   # GQA: KV head h // 2 serves Q head h
