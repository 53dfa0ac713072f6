"""CPU tests of chunked prefill against the 8-bit paged KV cache (sageattn_kvcache8_prefill) and of its restatement,
tests/attn_kvcache8_prefill_oracle.attend_folded:
  1. the restatement against fp64 attention on the 16-bit K / V: GQA, bottom-right causal with Lk < Lq, empty sequences, tile and
     page boundaries; at 64 accumulation steps it is the decode restatement with one chunk, bit for bit, and more steps only
     widen its bound;
  2. the host checks raise ValueError before any launch, and query chunks far above the decode call's row limit are accepted;
  3. the C ABI export and its error codes;
  4. bench_kvcache8_prefill.py's FLOP and byte counts."""
import math
import os
import sys

import pytest
import torch

from attn_kvcache8_oracle import attend, bytes_read, write
from attn_kvcache8_prefill_oracle import attend_folded, row_steps

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _fp64(q, k, v, is_causal, sm_scale):
    Lq, Hq, D = q.shape
    Lk = k.size(0)
    g = Hq // k.size(1)
    kh = k.double().repeat_interleave(g, 1).transpose(0, 1)
    vh = v.double().repeat_interleave(g, 1).transpose(0, 1)
    s = (q.double().transpose(0, 1) @ kh.transpose(1, 2)) * sm_scale
    if is_causal:
        vis = torch.arange(Lk)[None, :] <= torch.arange(Lq)[:, None] + Lk - Lq
        s = s.masked_fill(~vis, -math.inf)
    lse = torch.logsumexp(s, -1)
    p = torch.exp(s - lse[..., None]).nan_to_num(0.0)
    return (p @ vh).transpose(0, 1), lse


# ------------------------------------------------------------------------------------------------ 1. the restatement
@pytest.mark.parametrize("is_causal", [False, True])
@pytest.mark.parametrize("Hq,Hkv,D", [(4, 4, 64), (8, 2, 128), (8, 1, 64)])
def test_one_chunk_restatement_against_fp64_attention(is_causal, Hq, Hkv, D):
    g = torch.Generator().manual_seed(Hq * 10 + D + is_causal)
    for Lq, Lk in ((1, 1), (63, 63), (64, 65), (65, 64), (129, 127), (130, 16), (100, 1100), (70, 0), (0, 40), (128, 128 + 37)):
        q = torch.randn(Lq, Hq, D, generator=g).bfloat16()
        k = (torch.randn(Lk, Hkv, D, generator=g) + 2.0 * torch.randn(1, Hkv, D, generator=g)).bfloat16()
        v = torch.randn(Lk, Hkv, D, generator=g).bfloat16()
        ksm = k.float().mean(0) if Lk else torch.zeros(Hkv, D)
        k8, ks, v8, vs = write(k, v, ksm)
        o, lse, ob, lb = attend_folded(q, k8, ks, v8, vs, ksm, is_causal, D ** -0.5, bound=True)
        if Lq == 0:
            assert o.numel() == 0 and lse.numel() == 0
            continue
        oe, le = _fp64(q, k, v, is_causal, D ** -0.5)
        none = torch.isneginf(le)
        assert torch.equal(torch.isneginf(lse), none), (Lq, Lk)
        assert none.any() == (Lk == 0 or (is_causal and Lk < Lq)), (Lq, Lk)
        if is_causal and 0 < Lk < Lq:
            assert none.all(-1).eq(torch.zeros(Hq, dtype=torch.bool)).all()         # every head alike
            assert none[0, :Lq - Lk].all() and not none[0, Lq - Lk:].any()        # exactly the first Lq - Lk rows see nothing
        assert not o.transpose(0, 1)[none].any() and not ob.transpose(0, 1)[none].any()
        if (~none).any():
            err = (o - oe).abs().transpose(0, 1)[~none]
            assert err.max() < 0.15 and err.mean() < 0.025, (Lq, Lk, err.max().item(), err.mean().item())
            assert (lse - le)[~none].abs().max() < 0.05, (Lq, Lk)
            assert (ob.transpose(0, 1)[~none] < 0.05).all()


def test_at_64_steps_it_is_the_decode_restatement_with_one_chunk():
    """acc_steps = 64 gives attend's results and bound with one chunk (chunk >= Lk), to the bit; more steps leave o and lse alone
    and only widen the bound."""
    g = torch.Generator().manual_seed(4)
    for Lq, Lk, causal in ((2, 700, True), (300, 2 * 1024 + 37, True), (1, 1, False), (65, 0, True), (130, 64, True), (5, 200, False)):
        q = torch.randn(Lq, 8, 128, generator=g).half()
        k, v = torch.randn(Lk, 2, 128, generator=g).half(), torch.randn(Lk, 2, 128, generator=g).half()
        ksm = k.float().mean(0) if Lk else torch.zeros(2, 128)
        cached = (*write(k, v, ksm), ksm, causal, 128 ** -0.5)
        for chunk in (max(Lk, 1), 4 * Lk + 64):
            ref = attend(q, *cached, chunk, bound=True, out_dtype=torch.float16)
            got = attend_folded(q, *cached, bound=True, out_dtype=torch.float16, acc_steps=64)
            for a, b in zip(ref, got):
                assert torch.equal(a, b), (Lq, Lk, chunk)
        more = attend_folded(q, *cached, bound=True, out_dtype=torch.float16, acc_steps=640)
        assert torch.equal(more[0], got[0]) and torch.equal(more[1], got[1])
        assert (more[2] >= got[2]).all() and (more[3] >= got[3]).all()
        if Lk and (Lk >= Lq or not causal):
            assert (more[2] > got[2]).any()
    assert row_steps(1) == 64 and row_steps(1024) == 64 and row_steps(1025) == 68 and row_steps(16384 + 5) == 4 * 257


# ------------------------------------------------------------------------------------------------ 2. host checks
class _FakeCache:
    pass


def _cpu_cache():
    from sageattention_b200 import kvcache8
    cache = kvcache8.PagedKVCache8.__new__(kvcache8.PagedKVCache8)
    cache.dtype, cache.device = torch.bfloat16, torch.device("cpu")
    cache.k_pages = torch.zeros(4, 16, 2, 64, dtype=torch.int8)
    cache.v_pages = torch.zeros(4, 16, 2, 64, dtype=torch.float8_e4m3fn)
    cache.k_scale = cache.v_scale = torch.zeros(4, 16, 2)
    cache.k_smooth = torch.zeros(2, 64)
    return cache


def test_host_checks_raise_before_any_launch(monkeypatch):
    import sageattention_b200 as sab
    from sageattention_b200 import kvcache8
    with pytest.raises(ValueError):
        sab.sageattn_kvcache8_prefill(torch.zeros(1, 4, 64), _FakeCache(), None, None, None, 1)
    cache = _cpu_cache()
    launched = []
    monkeypatch.setattr(kvcache8.ops, "kvcache8_prefill", lambda *a: launched.append(a) or torch.empty(0))
    q = torch.zeros(3, 8, 64, dtype=torch.bfloat16)
    cu = torch.tensor([0, 1, 3], dtype=torch.int32)
    used = torch.tensor([5, 20], dtype=torch.int32)
    table = torch.zeros(2, 2, dtype=torch.int32)
    ok = dict(q=q, cache=cache, cu_seqlens_q=cu, seqused_k=used, block_table=table, max_seqlen_q=2)
    bad = [dict(q=q.half()), dict(q=q[..., :32]), dict(q=torch.zeros(3, 5, 64, dtype=torch.bfloat16)),
           dict(q=q[:, :, ::2]), dict(cu_seqlens_q=cu.float()), dict(cu_seqlens_q=cu[:1]), dict(seqused_k=used.long()),
           dict(seqused_k=used[:1]), dict(block_table=table.long()), dict(block_table=table[:1]), dict(block_table=table.t()),
           dict(max_seqlen_q=0), dict(max_seqlen_q=True), dict(max_seqlen_q=2.0),
           dict(q=torch.zeros(0, 8, 64, dtype=torch.bfloat16))]
    for b in bad:
        with pytest.raises(ValueError):
            sab.sageattn_kvcache8_prefill(**{**ok, **b})
    assert not launched
    # no row limit: 4096 query rows per sequence, 16384 per KV head, are accepted
    sab.sageattn_kvcache8_prefill(**{**ok, "max_seqlen_q": 4096})
    sab.sageattn_kvcache8_prefill(**{**ok, "cu_seqlens_q": cu.long(), "max_seqlen_q": 300, "return_lse": True})
    assert len(launched) == 2
    assert launched[0][10] == 4096 and launched[1][7].dtype == torch.int32 and launched[1][13] == 1
    assert launched[0][12] == 64 ** -0.5


def test_the_decode_row_limit_names_the_prefill_call(monkeypatch):
    import sageattention_b200 as sab
    from sageattention_b200 import kvcache8
    monkeypatch.setattr(kvcache8.ops, "kvcache8_attn", lambda *a: pytest.fail("launched"))
    args = dict(q=torch.zeros(3, 8, 64, dtype=torch.bfloat16), cache=_cpu_cache(), cu_seqlens_q=torch.tensor([0, 1, 3], dtype=torch.int32),
                seqused_k=torch.tensor([5, 20], dtype=torch.int32), block_table=torch.zeros(2, 2, dtype=torch.int32), max_seqlen_q=17)
    with pytest.raises(ValueError, match="sageattn_kvcache8_prefill") as e:
        sab.sageattn_kvcache8(**args)
    assert "sageattn_varlen_kvcache" in str(e.value)


# ------------------------------------------------------------------------------------------------ 3. C ABI
def test_c_abi_export_and_error_codes():
    from sageattention_b200 import _capi
    lib = _capi.lib()
    one = 16          # a non-null, 16-byte aligned address: every call below fails its checks before touching it

    def a(**kw):
        p = dict(q=one, dtype=1, ptrs=(one,) * 5, out=one, lse=None, cu=one, used=one, table=one, ts=4, mp=4, nseq=2, Tq=2, Hq=8, Hkv=2,
                 D=128, ps=16, st=(1024, 128, 1024, 128), msq=1, causal=1)
        p.update(kw)
        return lib.sab_kvcache8_prefill(p["q"], p["dtype"], *p["ptrs"], p["out"], p["lse"], p["cu"], p["used"], p["table"],
                                        p["ts"], p["mp"], p["nseq"], p["Tq"], p["Hq"], p["Hkv"], p["D"], p["ps"], *p["st"], p["msq"],
                                        p["causal"], 0.1, None)
    assert a(table=None) == -1 and b"null" in lib.sab_last_error()
    assert a(ptrs=(one, one, one, one, None)) == -1 and b"null" in lib.sab_last_error()     # k_smooth
    assert a(D=80) == -2 and b"head dim" in lib.sab_last_error()
    assert a(dtype=7) == -2
    assert a(Hq=6, Hkv=4) == -1 and b"divisible" in lib.sab_last_error()
    assert a(ts=3) == -1 and b"table_stride" in lib.sab_last_error()
    assert a(ps=24) == -1 and b"multiple of 16" in lib.sab_last_error()
    assert a(msq=0) == -1 and a(nseq=0) == -1 and a(Tq=0) == -1
    assert a(st=(1026, 130, 1024, 128)) == -1 and b"q needs" in lib.sab_last_error()
    assert a(st=(1024, 128, 1024, 127)) == -1 and b"out needs" in lib.sab_last_error()
    assert a(out=one + 2) == -1 and b"out needs" in lib.sab_last_error()
    # grid limits
    assert a(Hq=65536 * 2, Hkv=2) == -1 and b"grid" in lib.sab_last_error()
    assert a(nseq=2 ** 30, msq=1000) == -1 and b"grid" in lib.sab_last_error()
    assert a(mp=2 ** 27, ts=2 ** 27, ps=16) == -1 and b"2^31" in lib.sab_last_error()
    with pytest.raises(ValueError):
        _capi.check(a(D=64, Hq=6, Hkv=4))


def test_public_names_are_exported():
    import sageattention_b200 as sab
    from sageattention_b200 import _capi
    assert hasattr(sab, "sageattn_kvcache8_prefill") and "sageattn_kvcache8_prefill" in sab.__all__
    assert "sab_kvcache8_prefill" in _capi.EXPORTS
    with open(os.path.join(ROOT, "include", "sageattn_b200.h")) as fh:
        assert "int sab_kvcache8_prefill(" in fh.read()


# ------------------------------------------------------------------------------------------------ 4. benchmark counts
def test_bench_counts():
    sys.path.insert(0, ROOT)
    import bench_kvcache as bkv
    import bench_kvcache8_prefill as bp
    w = {x.name: x for x in bp.WORKLOADS}
    assert set(w) == {"chunked_prefill", "prefix_caching"}
    assert w["chunked_prefill"].lens_q == [2048] * 4 and w["chunked_prefill"].lens_k == [4096, 8192, 16384, 32768]
    assert w["prefix_caching"].lens_q == [1024] * 8 and w["prefix_caching"].lens_k == [9216] * 8
    assert w["prefix_caching"].shared_prefix == 8192
    cp = w["chunked_prefill"]
    pairs = bkv.visible_pairs(cp.lens_q, cp.lens_k)
    # rows see Lk - Lq + 1 .. Lk keys: 2048 rows per sequence, sum over a row of Lk - 2048 + i + 1
    assert pairs == sum(2048 * (lk - 2048) + 2048 * 2049 // 2 for lk in cp.lens_k)
    assert bp.flops(cp) == 4 * 32 * 128 * pairs
    # every key of every sequence read once per KV head (the 8-bit cache: 2 D + 8 bytes per key and KV head)
    assert bp.cache_bytes_read(cp) == bytes_read(cp.lens_k, 8, 128) == sum(cp.lens_k) * 8 * 264
    assert bp.cache_bytes_read(cp, bits16=True) == sum(cp.lens_k) * 8 * 128 * 4
    pc = w["prefix_caching"]
    assert bp.cache_bytes_read(pc) == 8 * 9216 * 8 * 264
    # the TFLOP/s a call needs to beat a 4.51 ms call on chunked_prefill: about 430
    assert 400 < bp.flops(cp) / 4.51e-3 / 1e12 < 470
    # the dense bound at D = 128: half the FLOPs INT8 QK^T at 1979, half bf16 PV at 989 TFLOP/s
    assert bp.peak_seconds(cp) == pytest.approx(bp.flops(cp) / 2 / 1979e12 + bp.flops(cp) / 2 / 989e12)
