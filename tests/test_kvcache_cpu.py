"""CPU tests of sageattn_varlen_kvcache's host side and of its restatement (tests/attn_kvcache_oracle.py):
  1. the restatement against an fp64 masked softmax on the gathered pages, bottom-right causal with Lk >= Lq and Lk < Lq, shared
     and shuffled pages, empty sequences; rows that see no key are 0 and lse -inf;
  2. the host checks answer with ValueError before any launch (shapes, dtypes, devices, seqused_k range), and a valid call
     reaches the launches with the exact packed sizes;
  3. bench_kvcache.py's visible-pair counts against the restatement's mask."""
import pytest
import torch

from attn_kvcache_oracle import gather_pages, sageattn_varlen_kvcache, visible


def _cache(lens_q, lens_k, page_size, Hq=4, Hkv=2, D=64, seed=0, shared_prefix=0):
    """Random q, a shuffled paged cache holding lens_k tokens per sequence, its block table and cu_seqlens_q.  shared_prefix:
    every sequence's first shared_prefix // page_size pages are the same pages."""
    g = torch.Generator().manual_seed(seed)
    nseq = len(lens_q)
    max_pages = max((n + page_size - 1) // page_size for n in lens_k) + 1
    npre = shared_prefix // page_size
    num_pages = npre + nseq * max_pages + 3
    k_cache = (torch.randn(num_pages, page_size, Hkv, D, generator=g) + torch.randn(1, 1, Hkv, D, generator=g)).half()
    v_cache = torch.randn(num_pages, page_size, Hkv, D, generator=g).half()
    perm = torch.randperm(num_pages, generator=g)
    table = torch.zeros(nseq, max_pages, dtype=torch.int32)
    nxt = npre
    for b in range(nseq):
        for p in range(max_pages):
            if p < npre:
                table[b, p] = perm[p]
            else:
                table[b, p] = perm[nxt]
                nxt += 1
    q = torch.randn(sum(lens_q), Hq, D, generator=g).half()
    cu = torch.tensor([0] + torch.cumsum(torch.tensor(lens_q), 0).tolist(), dtype=torch.int32)
    return q, k_cache, v_cache, cu, torch.tensor(lens_k, dtype=torch.int32), table


def _fp64(q, k, v, is_causal, sm_scale):
    """Exact attention of one sequence: (o [Lq,Hq,D], lse [Hq,Lq]), zero and -inf on rows that see no key."""
    Lq, Hq, D = q.shape
    g = Hq // k.size(1)
    kh = k.double().repeat_interleave(g, dim=1).transpose(0, 1)
    vh = v.double().repeat_interleave(g, dim=1).transpose(0, 1)
    s = (q.double().transpose(0, 1) @ kh.transpose(1, 2)) * sm_scale
    s = s.masked_fill(~visible(Lq, k.size(0), is_causal), float("-inf"))
    lse = torch.logsumexp(s, -1)
    p = torch.exp(s - lse[..., None]).nan_to_num(0.0)
    return (p @ vh).transpose(0, 1), lse


@pytest.mark.parametrize("is_causal", [False, True])
@pytest.mark.parametrize("page_size", [1, 16, 96])
def test_restatement_against_fp64_attention(is_causal, page_size):
    lens_q = [40, 1, 130, 0, 70, 5]
    lens_k = [300, 1, 200, 9, 30, 0]       # Lk > Lq, Lk = Lq, Lk < Lq (70 vs 30), empty K, empty Q
    q, kc, vc, cu, used, table = _cache(lens_q, lens_k, page_size, seed=page_size, shared_prefix=2 * page_size)
    o, lse = sageattn_varlen_kvcache(q, kc, vc, cu, used, table, is_causal=is_causal, pv_accum_dtype="fp32", smooth_v=True)
    k, v = gather_pages(kc, table, used), gather_pages(vc, table, used)
    cu_k = [0] + torch.cumsum(used, 0).tolist()
    for b, (Lq, Lk) in enumerate(zip(lens_q, lens_k)):
        s = int(cu[b])
        if Lq == 0:
            continue
        ob, lb = o[s:s + Lq], lse[:, s:s + Lq]
        if Lk == 0:
            assert not ob.any() and torch.isneginf(lb).all()
            continue
        oe, le = _fp64(q[s:s + Lq], k[cu_k[b]:cu_k[b + 1]], v[cu_k[b]:cu_k[b + 1]], is_causal, 64 ** -0.5)
        none = torch.isneginf(le)
        assert torch.equal(torch.isneginf(lb), none), f"rows with no visible key, sequence {b}"
        assert none.any() == (is_causal and Lk < Lq)
        assert not ob.transpose(0, 1)[none].any()
        err = (ob.double() - oe).abs()
        assert err.max() < 0.15 and err.mean() < 0.012, (b, err.max().item(), err.mean().item())
        assert (lb - le)[~none].abs().max() < 0.02, b


def test_restatement_rows_follow_the_bottom_right_offset():
    """Row i of a causal sequence sees the first Lk - Lq + i + 1 keys (none when that is <= 0), so with Lk >= Lq the last row
    sees every key."""
    for Lq, Lk in ((5, 12), (64, 64), (1, 300), (130, 129), (7, 3)):
        m = visible(Lq, Lk, True)
        assert torch.equal(m.sum(-1), (torch.arange(Lq) + Lk - Lq + 1).clamp(0, Lk))
        if Lk >= Lq:
            assert m[-1].all()


def test_gather_follows_the_block_table():
    q, kc, vc, cu, used, table = _cache([3, 4], [37, 16], 16, seed=3, shared_prefix=16)
    k = gather_pages(kc, table, used)
    assert k.shape[0] == 53
    assert torch.equal(k[0:16], kc[table[0, 0].long()]) and torch.equal(k[37:53], kc[table[1, 0].long()])
    assert torch.equal(k[0:16], k[37:53])                  # the shared prefix page
    assert torch.equal(k[32:37], kc[table[0, 2].long(), :5])


# ------------------------------------------------------------------------------------------------ 2. host checks
def _reach_the_launches(monkeypatch):
    """Run the host path on CPU tensors: the CUDA check passes, and every launch records its call instead of running."""
    from sageattention_b200 import core
    calls = []
    monkeypatch.setattr(core, "_check_on_cuda", lambda q: None)

    def rec(name, ret):
        def f(*a, **k):
            calls.append((name, a))
            return ret(*a)
        return f
    monkeypatch.setattr(core, "k_mean_paged", rec("k_mean", lambda kc, cu, t, m: torch.zeros(cu.numel() - 1, kc.size(2), kc.size(3),
                                                                                           dtype=kc.dtype)))
    monkeypatch.setattr(core, "quant_q_int8_varlen", rec("q", lambda q, *a: (q, None, None)))
    monkeypatch.setattr(core, "quant_k_int8_paged", rec("k", lambda *a: (None, None, None)))
    monkeypatch.setattr(core, "per_channel_fp8_paged", rec("v", lambda *a: (None, None, None, None)))
    monkeypatch.setattr(core.ops, "qk_int8_sv_f8_attn_varlen_bottom_right", rec("attn", lambda *a: torch.empty(0)))
    return calls


def test_a_valid_call_reaches_the_launches_with_exact_sizes(monkeypatch):
    import sageattention_b200 as sab
    calls = _reach_the_launches(monkeypatch)
    q, kc, vc, cu, used, table = _cache([3, 0, 70], [100, 5, 0], 16)
    sab.sageattn_varlen_kvcache(q, kc, vc, cu, used, table, 70, is_causal=True)
    names = [c[0] for c in calls]
    assert names == ["k_mean", "q", "k", "v", "attn"]
    k_args, v_args = calls[2][1], calls[3][1]
    assert k_args[4:7] == (100, 105, 2 + 1)         # max_seqlen_k, total keys, 64-key blocks
    assert v_args[3:5] == (100, 128 + 128)          # max_seqlen_k, padded V columns
    assert torch.equal(calls[2][1][2], torch.tensor([0, 100, 105, 105], dtype=torch.int32))
    assert calls[4][1][14] == 1                     # is_causal


def test_all_sequences_without_keys_launch_nothing(monkeypatch):
    import sageattention_b200 as sab
    calls = _reach_the_launches(monkeypatch)
    q, kc, vc, cu, used, table = _cache([3, 5], [0, 0], 16)
    o, lse = sab.sageattn_varlen_kvcache(q, kc, vc, cu, used, table, 5, is_causal=True, return_lse=True)
    assert not calls and not o.any() and torch.isneginf(lse).all()


def test_bad_arguments_raise_before_any_launch(monkeypatch):
    import sageattention_b200 as sab
    calls = _reach_the_launches(monkeypatch)
    q, kc, vc, cu, used, table = _cache([3, 4], [20, 30], 16)
    ok = dict(q=q, k_cache=kc, v_cache=vc, cu_seqlens_q=cu, seqused_k=used, block_table=table, max_seqlen_q=4)
    bad = [
        dict(q=q.float()), dict(q=q[None]), dict(q=q[:0]), dict(q=q[..., :32]),
        dict(k_cache=kc.float()), dict(k_cache=kc[0]), dict(v_cache=vc[:-1]), dict(k_cache=kc[..., :32], v_cache=vc[..., :32]),
        dict(k_cache=kc[:, :, :, 1:]), dict(k_cache=kc.transpose(2, 3).contiguous().transpose(2, 3)),
        dict(q=q[:, :3]),                                                   # Hq % Hkv != 0
        dict(cu_seqlens_q=cu.float()), dict(cu_seqlens_q=cu[:1]), dict(cu_seqlens_q=cu[None]),
        dict(seqused_k=used.long()), dict(seqused_k=used[:1]), dict(seqused_k=torch.tensor([20, -1], dtype=torch.int32)),
        dict(seqused_k=torch.tensor([20, table.size(1) * 16 + 1], dtype=torch.int32)),
        dict(block_table=table.long()), dict(block_table=table[:1]), dict(block_table=table[:, :0]), dict(block_table=table.t()),
        dict(max_seqlen_q=0), dict(max_seqlen_q=True), dict(max_seqlen_q=2.0),
        dict(pv_accum_dtype="fp16"),
    ]
    for b in bad:
        with pytest.raises(ValueError):
            sab.sageattn_varlen_kvcache(**{**ok, **b})
    assert not calls
    sab.sageattn_varlen_kvcache(**ok)
    assert len(calls) == 5


def test_cpu_tensors_are_refused():
    import sageattention_b200 as sab
    q, kc, vc, cu, used, table = _cache([3, 4], [20, 30], 16)
    with pytest.raises(ValueError, match="CUDA"):
        sab.sageattn_varlen_kvcache(q, kc, vc, cu, used, table, 4)


def test_the_c_entries_refuse_bad_arguments_without_a_gpu():
    import ctypes
    from sageattention_b200 import _capi
    L = _capi.lib()
    buf = ctypes.create_string_buffer(256)
    p = (ctypes.addressof(buf) + 15) // 16 * 16
    # k_cache, dtype, mean, cu, table, table_stride, page_size, nseq, max_seqlen, H, D, page_stride, stride_t, stride_h, ws, stream
    assert L.sab_k_mean_paged(p, 0, p, p, None, 4, 16, 1, 16, 2, 64, 2048, 128, 64, p, None) == -1
    assert b"block table" in L.sab_last_error()
    assert L.sab_k_mean_paged(p, 0, p, p, p, 4, 0, 1, 16, 2, 64, 2048, 128, 64, p, None) == -1
    assert L.sab_k_mean_paged(p, 0, p, p, p, 4, 16, 1, 16, 2, 96, 2048, 128, 64, p, None) == -2
    assert L.sab_k_mean_paged(p, 0, p, p, p, 4, 16, 1, 16, 2, 64, 2044, 128, 64, p, None) == -1       # page stride % 8
    assert L.sab_quant_int8_paged(p, 0, None, p, p, p, p, None, 4, 16, 1, 16, 2, 64, 2048, 128, 64, 128, 64, 3, None) == -1
    assert L.sab_per_channel_fp8_paged(p, 0, p, p, None, p, p, p, 4, 16, 1, 16, 2, 64, 2048, 128, 64, 100, 448.0, p, None) == -1
    assert b"t_pad" in L.sab_last_error()
    # the attention entry: missing sequence tables
    st = L.sab_qk_int8_sv_f8_attn_varlen_bottom_right(p, p, p, p, None, p, p, p, None, 1, 1, 2, 2, 64, 64, 128, 128, 128, 128, 128,
                                                       128, 128, 128, 1, 3, 3, 1.0, None, None, None, None, None, 64, None)
    assert st == -1 and b"cu_seqlens_q" in L.sab_last_error()


def test_the_new_names_are_exported():
    import inspect
    import sageattention_b200 as sab
    assert "sageattn_varlen_kvcache" in sab.__all__
    params = list(inspect.signature(sab.sageattn_varlen_kvcache).parameters)
    assert params == ["q", "k_cache", "v_cache", "cu_seqlens_q", "seqused_k", "block_table", "max_seqlen_q", "is_causal",
                      "qk_quant_gran", "sm_scale", "pv_accum_dtype", "smooth_k", "smooth_v", "return_lse"]


# ------------------------------------------------------------------------------------------------ 3. bench counts
@pytest.mark.parametrize("is_causal", [False, True])
def test_bench_visible_pairs_agree_with_the_mask(is_causal):
    from bench_kvcache import visible_pairs
    lens_q, lens_k = [2048, 8, 1, 100, 0], [4096, 4000, 1, 50, 7]
    want = sum(int(visible(a, b, is_causal).sum()) for a, b in zip(lens_q, lens_k))
    assert visible_pairs(lens_q, lens_k, is_causal) == want


def test_bench_workloads_have_the_documented_shapes():
    from bench_kvcache import WORKLOADS
    wl = {w.name: w for w in WORKLOADS}
    assert wl["chunked_prefill"].lens_q == [2048] * 4
    assert wl["chunked_prefill"].lens_k == [2048 + 2048, 6144 + 2048, 14336 + 2048, 30720 + 2048]
    assert wl["prefix_caching"].lens_q == [1024] * 8 and wl["prefix_caching"].lens_k == [8192 + 1024] * 8
    assert wl["prefix_caching"].shared_prefix == 8192
    sv = wl["speculative_verification"]
    assert len(sv.lens_q) == 32 and set(sv.lens_q) == {8} and min(sv.lens_k) >= 4096 and max(sv.lens_k) <= 16384
