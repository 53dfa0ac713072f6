"""CPU tests of the 8-bit paged KV cache (sageattention_b200/kvcache8.py) and of its restatement (tests/attn_kvcache8_oracle.py):
  1. the restatement against fp64 attention on the 16-bit K / V: GQA, bottom-right causal with Lk < Lq, empty sequences, chunk
     and page boundaries; the quantisers' edge rules;
  2. the host checks raise ValueError before any launch, including the row limit;
  3. the C ABI exports and its error codes;
  4. bench_kvcache8.py's byte counts."""
import math
import os
import sys

import pytest
import torch

from attn_kvcache8_oracle import attend, bytes_read, quant_rows, write

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


@pytest.mark.parametrize("is_causal", [False, True])
@pytest.mark.parametrize("Hq,Hkv,D", [(4, 4, 64), (8, 2, 128), (8, 1, 64)])
def test_restatement_against_fp64_attention(is_causal, Hq, Hkv, D):
    chunk = 256
    g = torch.Generator().manual_seed(Hq * 10 + D + is_causal)
    for Lq, Lk in ((1, 1), (4, 63), (1, 65), (2, chunk - 1), (3, chunk), (1, chunk + 1), (8, 2 * chunk + 37), (6, 3), (2, 0)):
        q = torch.randn(Lq, Hq, D, generator=g).bfloat16()
        k = (torch.randn(Lk, Hkv, D, generator=g) + 2.0 * torch.randn(1, Hkv, D, generator=g)).bfloat16()
        v = torch.randn(Lk, Hkv, D, generator=g).bfloat16()
        ksm = k.float().mean(0) if Lk else torch.zeros(Hkv, D)
        k8, ks, v8, vs = write(k, v, ksm)
        o, lse, ob, lb = attend(q, k8, ks, v8, vs, ksm, is_causal, D ** -0.5, chunk, bound=True)
        oe, le = _fp64(q, k, v, is_causal, D ** -0.5)
        none = torch.isneginf(le)
        assert torch.equal(torch.isneginf(lse), none), (Lq, Lk)
        assert none.any() == (Lk == 0 or (is_causal and Lk < Lq)), (Lq, Lk)
        assert not o.transpose(0, 1)[none].any() and not ob.transpose(0, 1)[none].any()
        if (~none).any():
            err = (o - oe).abs().transpose(0, 1)[~none]
            assert err.max() < 0.15 and err.mean() < 0.025, (Lq, Lk, err.max().item(), err.mean().item())
            assert (lse - le)[~none].abs().max() < 0.05, (Lq, Lk)
            assert (ob.transpose(0, 1)[~none] < 0.05).all()      # the kernel bound is far below the quantisation error


def test_chunks_do_not_change_the_result_beyond_rounding():
    """The chunk size moves the bf16 rounding of P (the per-tile max changes), never the softmax itself."""
    g = torch.Generator().manual_seed(1)
    q = torch.randn(2, 4, 64, generator=g).half()
    k = torch.randn(700, 2, 64, generator=g).half()
    v = torch.randn(700, 2, 64, generator=g).half()
    k8, ks, v8, vs = write(k, v, torch.zeros(2, 64))
    o1, l1 = attend(q, k8, ks, v8, vs, torch.zeros(2, 64), True, 0.125, 256)
    o2, l2 = attend(q, k8, ks, v8, vs, torch.zeros(2, 64), True, 0.125, 1024)
    assert (o1 - o2).abs().max() < 2e-2 and (l1 - l2).abs().max() < 1e-9


def test_k_smooth_moves_only_the_quantisation_error():
    g = torch.Generator().manual_seed(2)
    q = torch.randn(1, 4, 128, generator=g).bfloat16()
    k = (torch.randn(300, 4, 128, generator=g) + 4.0).bfloat16()
    v = torch.randn(300, 4, 128, generator=g).bfloat16()
    oe, le = _fp64(q, k, v, False, 128 ** -0.5)
    errs = []
    for ksm in (torch.zeros(4, 128), k.float().mean(0)):
        o, lse = attend(q, *write(k, v, ksm), ksm, False, 128 ** -0.5, 512)
        assert (lse - le).abs().max() < 0.05
        errs.append((o - oe).abs().mean().item())
    assert errs[1] < errs[0]                 # smoothing a key offset of 4 cuts the error


def test_quantiser_edge_rules():
    x = torch.tensor([[0.0] * 4, [1.0, -2.0, 0.5, 2.0], [1e-38, -3e-39, 0.0, 2e-39], [0.0, 0.0, 0.0, 1e-45]])
    q, s = quant_rows(x, 127.0, fp8=False)
    assert s[0] == 0 and not q[0].any()
    assert q[1].tolist() == [64.0, -127.0, 32.0, 127.0]       # 63.5 rounds to even
    assert torch.isinf(torch.tensor(127.0) / x[2].abs().max()) and q[2, 0] == 127.0   # denormal amax: the IEEE quotient
    assert q[3, 3] == 127.0
    v, vs = quant_rows(torch.tensor([[448.0, -1.0, 0.3, 0.0]]), 448.0, fp8=True)
    assert vs[0] == 1.0 and v[0, 0] == 448.0 and v[0, 2] == torch.tensor(0.3).to(torch.float8_e4m3fn).float()


# ------------------------------------------------------------------------------------------------ 2. host checks
class _FakeCache:
    pass


def test_host_checks_raise_before_any_launch(monkeypatch):
    import sageattention_b200 as sab
    from sageattention_b200 import kvcache8
    with pytest.raises(ValueError):
        sab.PagedKVCache8(4, 16, 2, 64, device="cpu")
    with pytest.raises(ValueError):
        sab.sageattn_kvcache8(torch.zeros(1, 4, 64), _FakeCache(), None, None, None, 1)
    # a cache object built without a device: every tensor on CPU, reached only through the checks
    cache = kvcache8.PagedKVCache8.__new__(kvcache8.PagedKVCache8)
    cache.dtype, cache.device = torch.bfloat16, torch.device("cpu")
    cache.k_pages = torch.zeros(4, 16, 2, 64, dtype=torch.int8)
    cache.v_pages = torch.zeros(4, 16, 2, 64, dtype=torch.float8_e4m3fn)
    cache.k_scale = cache.v_scale = torch.zeros(4, 16, 2)
    cache.k_smooth = torch.zeros(2, 64)
    launched = []
    monkeypatch.setattr(kvcache8.ops, "kvcache8_attn", lambda *a: launched.append(a) or torch.empty(0))
    q = torch.zeros(3, 8, 64, dtype=torch.bfloat16)
    cu = torch.tensor([0, 1, 3], dtype=torch.int32)
    used = torch.tensor([5, 20], dtype=torch.int32)
    table = torch.zeros(2, 2, dtype=torch.int32)
    ok = dict(q=q, cache=cache, cu_seqlens_q=cu, seqused_k=used, block_table=table, max_seqlen_q=2)
    bad = [dict(q=q.half()), dict(q=q[..., :32]), dict(q=torch.zeros(3, 5, 64, dtype=torch.bfloat16)),
           dict(cu_seqlens_q=cu.float()), dict(cu_seqlens_q=cu[:1]), dict(seqused_k=used.long()), dict(seqused_k=used[:1]),
           dict(block_table=table.long()), dict(block_table=table[:1]), dict(block_table=table.t()), dict(max_seqlen_q=0),
           dict(max_seqlen_q=True), dict(max_seqlen_q=17), dict(q=torch.zeros(0, 8, 64, dtype=torch.bfloat16))]
    for b in bad:
        with pytest.raises(ValueError):
            sab.sageattn_kvcache8(**{**ok, **b})
    with pytest.raises(ValueError, match="sageattn_varlen_kvcache"):
        sab.sageattn_kvcache8(**{**ok, "max_seqlen_q": 17})         # 17 * 8 / 2 = 68 query rows per KV head
    assert not launched
    sab.sageattn_kvcache8(**{**ok, "max_seqlen_q": 16})             # 16 * 4 = 64 rows: the limit itself is allowed
    assert len(launched) == 1


def test_write_checks():
    from sageattention_b200 import kvcache8
    cache = kvcache8.PagedKVCache8.__new__(kvcache8.PagedKVCache8)
    cache.dtype, cache.device = torch.float16, torch.device("cpu")
    cache.k_pages = torch.zeros(4, 16, 2, 64, dtype=torch.int8)
    k = torch.zeros(3, 2, 64, dtype=torch.float16)
    slots = torch.zeros(3, dtype=torch.int64)
    for kk, vv, ss in ((k.bfloat16(), k, slots), (k, k[:2], slots), (k[:, :1], k[:, :1], slots), (k, k, slots.int()),
                       (k, k, slots[:2]), (k[..., ::2], k[..., ::2], slots)):
        with pytest.raises(ValueError):
            cache.write(kk, vv, ss)


# ------------------------------------------------------------------------------------------------ 3. C ABI
def test_c_abi_exports_and_error_codes():
    from sageattention_b200 import _capi
    lib = _capi.lib()
    chunk = lib.sab_kvcache8_chunk_keys()
    assert chunk in (256, 512, 1024)
    assert lib.sab_kvcache8_workspace_bytes(3, 8, 128, 2 * chunk + 1) == 3 * 8 * 3 * 130 * 4
    one = 16          # a non-null, 16-byte aligned address: every call below fails its checks before touching it
    args = dict(k=one, v=one, dtype=0, ksm=one, slots=one, T=4, Hkv=2, D=128, s=(256, 128, 256, 128), pages=(one,) * 4, np=4, ps=16)

    def w(**kw):
        a = {**args, **kw}
        return lib.sab_kvcache8_write(a["k"], a["v"], a["dtype"], a["ksm"], a["slots"], a["T"], a["Hkv"], a["D"], *a["s"], *a["pages"],
                                      a["np"], a["ps"], None)
    assert w(k=None) == -1 and b"null" in lib.sab_last_error()
    assert w(D=96) == -2 and b"head dim" in lib.sab_last_error()
    assert w(dtype=5) == -2
    assert w(ps=8) == -1 and b"multiple of 16" in lib.sab_last_error()
    assert w(s=(256, 130, 256, 128)) == -1 and b"aligned" in lib.sab_last_error()
    assert w(T=0) == 0                       # nothing to write: no launch

    def a(**kw):
        p = dict(q=one, dtype=1, ptrs=(one,) * 5, out=one, lse=None, cu=one, used=one, table=one, ts=4, mp=4, nseq=2, Tq=2, Hq=8, Hkv=2,
                 D=128, ps=16, st=(1024, 128, 1024, 128), msq=1, causal=1, ws=one)
        p.update(kw)
        return lib.sab_kvcache8_attn(p["q"], p["dtype"], *p["ptrs"], p["out"], p["lse"], p["cu"], p["used"], p["table"],
                                     p["ts"], p["mp"], p["nseq"], p["Tq"], p["Hq"], p["Hkv"], p["D"], p["ps"], *p["st"], p["msq"],
                                     p["causal"], 0.1, p["ws"], None)
    assert a(table=None) == -1 and b"null" in lib.sab_last_error()
    assert a(D=80) == -2
    assert a(Hq=6, Hkv=4) == -1 and b"divisible" in lib.sab_last_error()
    assert a(msq=17) == -1 and b"query rows" in lib.sab_last_error()
    assert a(ts=3) == -1
    assert a(ps=24) == -1
    with pytest.raises(ValueError):
        _capi.check(a(msq=17))


def test_public_names_are_exported():
    import sageattention_b200 as sab
    for name in ("PagedKVCache8", "sageattn_kvcache8"):
        assert hasattr(sab, name) and name in sab.__all__


# ------------------------------------------------------------------------------------------------ 4. benchmark counts
def test_bench_byte_counts():
    sys.path.insert(0, ROOT)
    import bench_kvcache8 as bk
    assert bk.cache_bytes_per_token(8, 128) == 8 * (2 * 128 + 8) == 2112
    assert bk.cache_bytes_per_token(8, 128, bits16=True) == 8 * 2 * 128 * 2 == 4096
    w = {x.name: x for x in bk.WORKLOADS}
    dec = w["decode"]
    assert dec.lens_q == [1] * 32 and dec.lens_k == [4096 + 384 * i for i in range(32)]
    assert bk.bytes_read(dec.lens_k) == bytes_read(dec.lens_k, 8, 128) == sum(dec.lens_k) * 2112
    assert w["speculative_verification"].lens_q == [8] * 32 and w["long_context_decode"].lens_k == [131072]
    # at 3.35 TB/s the decode workload's 8-bit read takes about 0.2 ms
    assert 0.15 < bk.bytes_read(dec.lens_k) / 3.35e12 * 1e3 < 0.25
