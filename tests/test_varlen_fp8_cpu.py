"""CPU tests of sageattn_varlen_qk_int8_pv_fp8_cuda's host side: the per-sequence block tables and scale-table bounds, the
argument checks (Python and C ABI) that answer before any launch, and a CPU restatement of the contract (per-sequence calls of
the dense INT8+FP8 oracle, concatenated)."""
import ctypes
import math

import numpy as np
import pytest
import torch

from oracle import sage_oracle as O

EDGE = [0, 1, 63, 64, 65, 127, 128, 129, 4096]


def test_block_tables_and_bounds():
    from sageattention_b200.quant import varlen_block_table, varlen_scale_rows
    for lens in (EDGE, EDGE[::-1], [0], [4096, 0, 0, 1]):
        cu = torch.tensor([0] + list(np.cumsum(lens)), dtype=torch.int64)
        for blk in (128, 64):
            t = varlen_block_table(cu, blk)
            assert t.dtype == torch.int32
            assert t.tolist() == [0] + list(np.cumsum([math.ceil(L / blk) for L in lens]))
        pad = (varlen_block_table(cu, 128) * 128).tolist()
        assert pad == [0] + list(np.cumsum([math.ceil(L / 128) * 128 for L in lens]))
        T, n = sum(lens), len(lens)
        for blk, mult in ((128, 4), (128, 32), (64, 1), (64, 4)):
            need = sum(math.ceil(L / blk) for L in lens) * mult       # rows the kernels write
            assert varlen_scale_rows(T, n, blk, mult) >= need
        assert (T + 127 * n + 127) // 128 * 128 >= pad[-1]           # V^T columns


def test_python_argument_checks():
    from sageattention_b200.core import _check_cu_seqlens
    q, k = torch.zeros(10, 4, 64), torch.zeros(12, 2, 64)
    cu = torch.tensor([0, 4, 10], dtype=torch.int32)
    cuk = torch.tensor([0, 5, 12], dtype=torch.int64)
    _check_cu_seqlens(q, k, cu, cuk, 6, 7)
    bad = [(q[None], k, cu, cuk, 6, 7), (q, k, cu.float(), cuk, 6, 7), (q, k, cu[None], cuk, 6, 7), (q, k, cu[:1], cuk[:1], 6, 7),
           (q, k, cu, cuk[:2], 6, 7), (q, k, cu, cuk, 0, 7), (q, k, cu, cuk, 6, True), (q[:0], k, cu, cuk, 6, 7)]
    for args in bad:
        with pytest.raises(ValueError):
            _check_cu_seqlens(*args)
    import sageattention_b200 as sab
    with pytest.raises(AssertionError):          # CPU tensors are not computed
        sab.sageattn_varlen_qk_int8_pv_fp8_cuda(q.half(), k.half(), k.half(), cu, cuk, 6, 7)


def test_c_abi_checks_answer_before_the_device():
    from sageattention_b200._capi import lib, SAB_GRAN_PER_BLOCK, SAB_GRAN_PER_THREAD, SAB_DTYPE_BF16
    L = lib()
    buf = ctypes.create_string_buffer(64 + 16)
    p = (ctypes.addressof(buf) + 15) // 16 * 16
    # per-block granularity is not a form of the per-sequence quantiser / forward / backward
    assert L.sab_quant_int8_varlen(p, SAB_DTYPE_BF16, None, p, p, p, p, 1, 64, 1, 64, 64, 64, 64, 64, SAB_GRAN_PER_BLOCK, 0, None) == -1
    assert b"granularity" in L.sab_last_error()
    assert L.sab_quant_int8_varlen(p, SAB_DTYPE_BF16, p, p, p, p, p, 1, 64, 1, 64, 64, 64, 64, 64, SAB_GRAN_PER_THREAD, 0, None) == -1
    assert b"K only" in L.sab_last_error()
    assert L.sab_k_mean_varlen(p, SAB_DTYPE_BF16, None, p, 1, 64, 1, 64, 64, 64, p, None) == -1
    assert L.sab_per_channel_fp8_varlen(p, SAB_DTYPE_BF16, p, p, None, p, p, 1, 64, 1, 64, 64, 64, 100, 2.25, p, None) == -1
    assert L.sab_qk_int8_sv_f8_attn_varlen(p, p, p, p, None, p, p, p, None, SAB_DTYPE_BF16, 1, 2, 2, 64, 64, 64, 64, 64, 64, 64, 128,
                                           64, 64, 0, SAB_GRAN_PER_BLOCK, SAB_GRAN_PER_BLOCK, 1.0, p, p, p, p, p, 64, None) == -1
    assert b"q_gran" in L.sab_last_error()
    assert L.sab_qk_int8_attn_bwd_varlen_seq(*([p] * 15), SAB_DTYPE_BF16, 1, 2, 2, 64, 64, 64, *([64] * 14), *([p] * 4), 64, 64, 0,
                                             SAB_GRAN_PER_BLOCK, SAB_GRAN_PER_THREAD, 1.0, None) == -1
    assert b"q_gran" in L.sab_last_error()


def varlen_oracle(q, k, v, cu_q, cu_k, **kw):
    """The contract on the CPU: O.sageattn_qk_int8_pv_fp8_cuda per sequence (NHD, batch 1), rows concatenated; lse [Hq,Tq]."""
    outs, lses = [], []
    for b in range(len(cu_q) - 1):
        s, e, sk, ek = cu_q[b], cu_q[b + 1], cu_k[b], cu_k[b + 1]
        o, lse = O.sageattn_qk_int8_pv_fp8_cuda(q[s:e][None], k[sk:ek][None], v[sk:ek][None], tensor_layout="NHD", return_lse=True, **kw)
        outs.append(o[0])
        lses.append(lse[0])
    return torch.cat(outs), torch.cat(lses, dim=-1)


@pytest.mark.parametrize("gran", ["per_thread", "per_warp"])
def test_restatement_against_the_dense_oracle(gran):
    g = torch.Generator().manual_seed(1)
    lens_q, lens_k = [5, 130, 64], [70, 9, 64]
    cu_q, cu_k = [0] + list(np.cumsum(lens_q)), [0] + list(np.cumsum(lens_k))
    q = torch.randn(sum(lens_q), 4, 64, generator=g).half()
    k = (torch.randn(sum(lens_k), 2, 64, generator=g) + 2.0).half()
    v = torch.randn(sum(lens_k), 2, 64, generator=g).half()
    kw = dict(qk_quant_gran=gran, lazy_tau=4, emulate_f16_accum=False)
    o, lse = varlen_oracle(q, k, v, cu_q, cu_k, **kw)
    assert o.shape == q.shape and lse.shape == (4, q.size(0))
    for b in range(3):
        s, e, sk, ek = cu_q[b], cu_q[b + 1], cu_k[b], cu_k[b + 1]
        ob, lb = O.sageattn_qk_int8_pv_fp8_cuda(q[s:e][None], k[sk:ek][None], v[sk:ek][None], tensor_layout="NHD", return_lse=True, **kw)
        assert torch.equal(o[s:e], ob[0]) and torch.equal(lse[:, s:e], lb[0])
    # one sequence: the restatement is the dense call itself
    o1, l1 = varlen_oracle(q[:5], k[:70], v[:70], [0, 5], [0, 70], **kw)
    od, ld = O.sageattn_qk_int8_pv_fp8_cuda(q[:5][None], k[:70][None], v[:70][None], tensor_layout="NHD", return_lse=True, **kw)
    assert torch.equal(o1, od[0]) and torch.equal(l1, ld[0])
