"""CPU tests of sliding-window attention on the 8-bit paged KV cache (window_size on sageattn_kvcache8 and
sageattn_kvcache8_prefill) and of the windowed restatements, tests/attn_kvcache8_window_oracle.attend / attend_folded:
  1. the windowed restatements against fp64 masked attention on the dequantised cache; at (-1, -1), and with windows that hide
     no key, they give the results and bounds of attn_kvcache8_oracle.attend and attn_kvcache8_prefill_oracle.attend_folded,
     the restatements without a window, bit for bit;
  2. host checks: every malformed window_size raises ValueError before any launch, (-1, -1) calls the op without a window, and
     large sides are clamped to the table's keys;
  3. the C ABI exports and their error codes;
  4. bench_kvcache8_window.py's key, byte and pair counts."""
import math
import os
import sys

import pytest
import torch

import attn_kvcache8_oracle
import attn_kvcache8_prefill_oracle
from attn_kvcache8_oracle import write
from attn_kvcache8_window_oracle import attend, attend_folded

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _dequant_fp64(q, k8, ks, v8, vs, ksm, is_causal, window, sm_scale):
    """fp64 attention of the 16-bit q on the dequantised keys (k8 * k_scale + k_smooth) and values, with the window's mask."""
    Lq, Hq, D = q.shape
    Lk, Hkv, _ = k8.shape
    g = Hq // Hkv
    k = (k8.double() * ks.double()[..., None] + ksm.double()).repeat_interleave(g, 1).transpose(0, 1)
    v = (v8.double() * vs.double()[..., None]).repeat_interleave(g, 1).transpose(0, 1)
    s = (q.double().transpose(0, 1) @ k.transpose(1, 2)) * sm_scale
    i, j = torch.arange(Lq)[:, None], torch.arange(Lk)[None, :]
    off = Lk - Lq
    vis = torch.ones(Lq, Lk, dtype=torch.bool)
    if is_causal:
        vis &= j <= i + off
    if window[0] >= 0:
        vis &= j >= i + off - window[0]
    if window[1] >= 0:
        vis &= j <= i + off + window[1]
    s = s.masked_fill(~vis, -math.inf)
    lse = torch.logsumexp(s, -1)
    p = torch.exp(s - lse[..., None]).nan_to_num(0.0)
    return (p @ v).transpose(0, 1), lse, vis


# ------------------------------------------------------------------------------------------------ 1. the restatements
_WINDOWS = [((0, -1), True), ((1, -1), True), ((63, 0), True), ((64, -1), True), ((65, 7), True), ((200, -1), True),
            ((-1, 0), False), ((5, 5), False), ((-1, 200), False), ((100, -1), False), ((0, 0), False)]


@pytest.mark.parametrize("fold", [False, True])
@pytest.mark.parametrize("window,is_causal", _WINDOWS)
def test_windowed_restatement_against_fp64(fold, window, is_causal):
    g = torch.Generator().manual_seed(7 + window[0] + 3 * window[1] + is_causal)
    Hq, Hkv, D = 8, 2, 64
    for Lq, Lk in ((1, 1), (1, 700), (5, 300), (64, 65), (130, 40), (100, 1100), (3, 0)):
        q = torch.randn(Lq, Hq, D, generator=g).bfloat16()
        k = (torch.randn(Lk, Hkv, D, generator=g) + torch.randn(1, Hkv, D, generator=g)).bfloat16()
        v = torch.randn(Lk, Hkv, D, generator=g).bfloat16()
        ksm = k.float().mean(0) if Lk else torch.zeros(Hkv, D)
        k8, ks, v8, vs = write(k, v, ksm)
        if fold:
            o, lse, ob, lb = attend_folded(q, k8, ks, v8, vs, ksm, is_causal, D ** -0.5, bound=True, window=window)
        else:
            o, lse, ob, lb = attend(q, k8, ks, v8, vs, ksm, is_causal, D ** -0.5, 256, bound=True, window=window)
        oe, le, vis = _dequant_fp64(q, k8, ks, v8, vs, ksm, is_causal, window, D ** -0.5)
        none = ~vis.any(-1)                                             # rows that see no key
        assert torch.equal(torch.isneginf(lse), none[None].expand(Hq, Lq)), (Lq, Lk)
        assert not o[none].any() and not ob[none].any()
        if (~none).any():
            # the restatement differs from fp64 by the quantisation of Q and P only
            err = (o - oe).abs()[~none]
            assert err.max() < 0.08 and err.mean() < 0.01, (Lq, Lk, err.max().item())
            assert (lse - le).abs()[:, ~none].max() < 0.05


def test_no_window_and_wide_windows_give_the_bits_without_a_window():
    """The windowed restatements give the restatements without a window to the bit: at (-1, -1), at left >= Lk (no row's lower
    bound reaches key 0), causal with any right, and non-causal with right >= Lq; also at other accumulation step counts."""
    g = torch.Generator().manual_seed(3)
    for Lq, Lk, causal in ((2, 700, True), (64, 2 * 1024 + 37, True), (1, 1, False), (65, 0, True), (130, 64, True),
                           (5, 200, False), (40, 10, False)):
        q = torch.randn(Lq, 8, 128, generator=g).half()
        k, v = torch.randn(Lk, 2, 128, generator=g).half(), torch.randn(Lk, 2, 128, generator=g).half()
        ksm = k.float().mean(0) if Lk else torch.zeros(2, 128)
        cached = (*write(k, v, ksm), ksm, causal, 128 ** -0.5)
        ref = attn_kvcache8_oracle.attend(q, *cached, 1024, bound=True, out_dtype=torch.float16)
        reff = attn_kvcache8_prefill_oracle.attend_folded(q, *cached, bound=True, out_dtype=torch.float16)
        wides = [(-1, -1), (Lk, -1), (Lk + 5000, -1)] + ([(Lk, 0), (Lk, 3), (-1, 9)] if causal else [(Lk, Lq), (-1, Lq + 7)])
        for w in wides:
            for a, b in zip(ref, attend(q, *cached, 1024, bound=True, out_dtype=torch.float16, window=w)):
                assert torch.equal(a, b), (Lq, Lk, w)
            for a, b in zip(reff, attend_folded(q, *cached, bound=True, out_dtype=torch.float16, window=w)):
                assert torch.equal(a, b), (Lq, Lk, w)
        for steps in (64, 640):
            ref = attn_kvcache8_prefill_oracle.attend_folded(q, *cached, bound=True, out_dtype=torch.float16, acc_steps=steps)
            for a, b in zip(ref, attend_folded(q, *cached, bound=True, out_dtype=torch.float16, acc_steps=steps, window=(Lk, -1))):
                assert torch.equal(a, b), (Lq, Lk, steps)


# ------------------------------------------------------------------------------------------------ 2. host checks
def _cpu_cache():
    from sageattention_b200 import kvcache8
    cache = kvcache8.PagedKVCache8.__new__(kvcache8.PagedKVCache8)
    cache.dtype, cache.device = torch.bfloat16, torch.device("cpu")
    cache.k_pages = torch.zeros(4, 16, 2, 64, dtype=torch.int8)
    cache.v_pages = torch.zeros(4, 16, 2, 64, dtype=torch.float8_e4m3fn)
    cache.k_scale = cache.v_scale = torch.zeros(4, 16, 2)
    cache.k_smooth = torch.zeros(2, 64)
    return cache


def _args():
    return dict(q=torch.zeros(3, 8, 64, dtype=torch.bfloat16), cache=_cpu_cache(), cu_seqlens_q=torch.tensor([0, 1, 3], dtype=torch.int32),
                seqused_k=torch.tensor([5, 20], dtype=torch.int32), block_table=torch.zeros(2, 3, dtype=torch.int32), max_seqlen_q=2)


_CALLS = [("sageattn_kvcache8", "kvcache8_attn"), ("sageattn_kvcache8_prefill", "kvcache8_prefill")]


@pytest.mark.parametrize("call,op", _CALLS)
def test_malformed_window_size_raises_before_any_launch(monkeypatch, call, op):
    import sageattention_b200 as sab
    from sageattention_b200 import kvcache8
    monkeypatch.setattr(kvcache8.ops, op, lambda *a: pytest.fail("launched"))
    monkeypatch.setattr(kvcache8.ops, op + "_window", lambda *a: pytest.fail("launched"))
    for bad in [(-2, 0), (0, -2), (1,), (1, 2, 3), (True, 0), (0, False), (1.0, 0), (0, 2.5), None, 5, "ab", (None, 0)]:
        with pytest.raises(ValueError, match="window_size must be a pair of ints >= -1"):
            getattr(sab, call)(**_args(), window_size=bad)


@pytest.mark.parametrize("call,op", _CALLS)
def test_window_ops_and_clamping(monkeypatch, call, op):
    import sageattention_b200 as sab
    from sageattention_b200 import kvcache8
    plain, windowed = [], []
    monkeypatch.setattr(kvcache8.ops, op, lambda *a: plain.append(a) or torch.empty(0))
    monkeypatch.setattr(kvcache8.ops, op + "_window", lambda *a: windowed.append(a) or torch.empty(0))
    fn = getattr(sab, call)
    fn(**_args())
    fn(**_args(), window_size=(-1, -1))
    fn(**_args(), window_size=[-1, -1])
    assert len(plain) == 3 and not windowed
    assert all(len(a) == 14 for a in plain)                 # the existing op's signature
    fn(**_args(), window_size=(1024, 0))
    fn(**_args(), window_size=(2 ** 40, 2 ** 70))         # clamped at the table's 3 pages x 16 keys
    fn(**_args(), window_size=(-1, 48), is_causal=False)
    fn(**_args(), window_size=(0, -1), return_lse=True)
    assert len(plain) == 3 and len(windowed) == 4
    assert [a[14:] for a in windowed] == [(48, 0), (48, 48), (-1, 48), (0, -1)]
    assert all(type(x) is int for a in windowed for x in a[14:])
    assert windowed[2][11] == 0 and windowed[3][13] == 1 and windowed[0][11] == 1


def test_the_decode_row_limit_holds_with_a_window(monkeypatch):
    import sageattention_b200 as sab
    from sageattention_b200 import kvcache8
    monkeypatch.setattr(kvcache8.ops, "kvcache8_attn_window", lambda *a: pytest.fail("launched"))
    with pytest.raises(ValueError, match="sageattn_kvcache8_prefill"):
        sab.sageattn_kvcache8(**{**_args(), "max_seqlen_q": 17}, window_size=(100, -1))


# ------------------------------------------------------------------------------------------------ 3. C ABI
@pytest.mark.parametrize("name", ["sab_kvcache8_attn_window", "sab_kvcache8_prefill_window"])
def test_c_abi_exports_and_error_codes(name):
    from sageattention_b200 import _capi
    lib = _capi.lib()
    fn = getattr(lib, name)
    one = 16          # a non-null, 16-byte aligned address: every call below fails its checks before touching it
    decode = name == "sab_kvcache8_attn_window"

    def a(**kw):
        p = dict(q=one, dtype=1, ptrs=(one,) * 5, out=one, lse=None, cu=one, used=one, table=one, ts=4, mp=4, nseq=2, Tq=2, Hq=8,
                 Hkv=2, D=128, ps=16, st=(1024, 128, 1024, 128), msq=1, causal=1, wl=4, wr=-1)
        p.update(kw)
        head = (p["q"], p["dtype"], *p["ptrs"], p["out"], p["lse"], p["cu"], p["used"], p["table"], p["ts"], p["mp"], p["nseq"],
                p["Tq"], p["Hq"], p["Hkv"], p["D"], p["ps"], *p["st"], p["msq"], p["causal"], 0.1)
        return fn(*head, *((one,) if decode else ()), p["wl"], p["wr"], None)
    assert a(wl=-2) == -1 and b">= -1" in lib.sab_last_error()
    assert a(wr=-2, causal=0) == -1 and b">= -1" in lib.sab_last_error()
    assert a(wl=-(2 ** 31)) == -1
    assert a(table=None) == -1 and b"null" in lib.sab_last_error()
    assert a(D=80) == -2 and b"head dim" in lib.sab_last_error()
    assert a(Hq=6, Hkv=4) == -1 and b"divisible" in lib.sab_last_error()
    assert a(ps=24) == -1 and b"multiple of 16" in lib.sab_last_error()
    assert a(mp=2 ** 27, ts=2 ** 27, ps=16) == -1
    if decode:
        assert a(msq=17) == -1 and b"query rows" in lib.sab_last_error()
    else:
        assert a(st=(1024, 128, 1024, 127)) == -1 and b"out needs" in lib.sab_last_error()


def test_public_names_are_exported():
    from sageattention_b200 import _capi
    with open(os.path.join(ROOT, "include", "sageattn_b200.h")) as fh:
        header = fh.read()
    for name in ("sab_kvcache8_attn_window", "sab_kvcache8_prefill_window"):
        assert name in _capi.EXPORTS and f"int {name}(" in header


# ------------------------------------------------------------------------------------------------ 4. benchmark counts
def test_bench_counts():
    sys.path.insert(0, ROOT)
    import bench_kvcache8_window as bw
    w = {x.name: x for x in bw.WORKLOADS}
    assert set(w) == {"decode", "long_context_decode", "chunked_prefill"}
    assert w["decode"].lens_q == [1] * 32 and w["decode"].lens_k[0] == 4096 and w["decode"].lens_k[-1] == 16000
    assert w["long_context_decode"].lens_q == [1] and w["long_context_decode"].lens_k == [131072]
    assert w["chunked_prefill"].lens_q == [2048] * 4 and w["chunked_prefill"].lens_k == [4096, 8192, 16384, 32768]
    assert bw.LEFTS == (1024, 4096)
    # keys in the window: decode rows see left + 1 keys (all cache lengths exceed 4096 + 1)
    assert bw.window_keys(w["decode"], 1024) == 32 * 1025
    assert bw.window_keys(w["long_context_decode"], 4096) == 4097
    # prefill: the chunk's 2048 rows reach back left keys from the first row: 2048 + left keys per sequence
    assert bw.window_keys(w["chunked_prefill"], 1024) == 4 * (2048 + 1024)
    assert bw.window_keys(w["chunked_prefill"], 4096) == 4096 + 3 * (2048 + 4096)     # the first sequence holds 4096 keys
    assert bw.bytes_read(w["decode"], 1024) == 32 * 1025 * 8 * (2 * 128 + 8)
    # visible pairs: every row of a chunk sees left + 1 keys when the prefix is at least left long
    assert bw.visible_pairs(w["chunked_prefill"], 1024) == 4 * 2048 * 1025
    # at left = 4096 the first sequence's rows i see min(i + 2048, 4096) + 1 keys
    assert bw.visible_pairs(w["chunked_prefill"], 4096) == sum(min(i + 2048, 4096) + 1 for i in range(2048)) + 3 * 2048 * 4097
    assert bw.flops(w["chunked_prefill"], 1024) == 4 * 32 * 128 * 4 * 2048 * 1025
    # the whole cache (no window): every key per sequence
    assert bw.window_keys(w["decode"], -1) == sum(w["decode"].lens_k)
