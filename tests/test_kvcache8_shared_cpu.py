"""CPU tests of shared-prefix decoding on the 8-bit paged KV cache (shared_prefix_len on sageattn_kvcache8):
  1. host checks: a bool, negative or non-int shared_prefix_len, or one together with a window, raises ValueError before any
     launch; below one chunk the call goes to the op without a shared prefix with its usual arguments, from one chunk up to
     kvcache8_attn_shared with the value clamped at the table's keys;
  2. the C export and its error codes;
  3. bench_kvcache8_shared.py's key and byte counts."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cpu_cache():
    from sageattention_b200 import kvcache8
    cache = kvcache8.PagedKVCache8.__new__(kvcache8.PagedKVCache8)
    cache.dtype, cache.device = torch.bfloat16, torch.device("cpu")
    cache.k_pages = torch.zeros(400, 16, 2, 64, dtype=torch.int8)
    cache.v_pages = torch.zeros(400, 16, 2, 64, dtype=torch.float8_e4m3fn)
    cache.k_scale = cache.v_scale = torch.zeros(400, 16, 2)
    cache.k_smooth = torch.zeros(2, 64)
    return cache


def _args():
    # a table of 300 pages x 16 keys = 4800 keys
    return dict(q=torch.zeros(3, 8, 64, dtype=torch.bfloat16), cache=_cpu_cache(), cu_seqlens_q=torch.tensor([0, 1, 3], dtype=torch.int32),
                seqused_k=torch.tensor([2000, 4000], dtype=torch.int32), block_table=torch.zeros(2, 300, dtype=torch.int32),
                max_seqlen_q=2)


def _chunk():
    from sageattention_b200 import ops
    return ops.kvcache8_chunk_keys()


# ------------------------------------------------------------------------------------------------ 1. host checks
def test_bad_shared_prefix_len_raises_before_any_launch(monkeypatch):
    import sageattention_b200 as sab
    from sageattention_b200 import kvcache8
    for op in ("kvcache8_attn", "kvcache8_attn_window", "kvcache8_attn_shared"):
        monkeypatch.setattr(kvcache8.ops, op, lambda *a: pytest.fail("launched"))
    for bad in (True, False, -1, -(2 ** 40), 1024.0, 2.5, "1024", None, torch.tensor(1024)):
        with pytest.raises(ValueError, match="shared_prefix_len must be an int >= 0"):
            sab.sageattn_kvcache8(**_args(), shared_prefix_len=bad)
    for window in ((100, -1), (-1, 0), (0, 0)):
        for shared in (1, _chunk(), 10 ** 6):
            with pytest.raises(ValueError, match="shared_prefix_len and window_size"):
                sab.sageattn_kvcache8(**_args(), window_size=window, shared_prefix_len=shared)


def test_dispatch_and_clamping(monkeypatch):
    import numpy as np
    import sageattention_b200 as sab
    from sageattention_b200 import kvcache8
    C = _chunk()
    plain, shared, windowed = [], [], []
    monkeypatch.setattr(kvcache8.ops, "kvcache8_attn", lambda *a: plain.append(a) or torch.empty(0))
    monkeypatch.setattr(kvcache8.ops, "kvcache8_attn_shared", lambda *a: shared.append(a) or torch.empty(0))
    monkeypatch.setattr(kvcache8.ops, "kvcache8_attn_window", lambda *a: windowed.append(a) or torch.empty(0))
    for value in (0, 1, C - 1, np.int64(C - 1)):
        sab.sageattn_kvcache8(**_args(), shared_prefix_len=value)
    sab.sageattn_kvcache8(**_args(), window_size=(100, -1), shared_prefix_len=0)
    assert len(plain) == 4 and not shared and len(windowed) == 1
    assert all(len(a) == 14 for a in plain)                  # the existing op's signature
    for value in (C, C + 1, 3 * C + 17, np.int64(2 * C), 4800, 10 ** 6, 2 ** 70):
        sab.sageattn_kvcache8(**_args(), shared_prefix_len=value)
    sab.sageattn_kvcache8(**_args(), shared_prefix_len=C, is_causal=False, return_lse=True)
    assert len(plain) == 4 and len(shared) == 8
    assert [a[14] for a in shared] == [C, C + 1, 3 * C + 17, 2 * C, 4800, 4800, 4800, C]   # clamped at 300 x 16 keys
    assert all(type(a[14]) is int for a in shared)
    assert all(len(a) == 15 for a in shared)
    assert shared[0][11] == 1 and shared[-1][11] == 0 and shared[-1][13] == 1


def test_the_decode_row_limit_holds_with_a_shared_prefix(monkeypatch):
    import sageattention_b200 as sab
    from sageattention_b200 import kvcache8
    monkeypatch.setattr(kvcache8.ops, "kvcache8_attn_shared", lambda *a: pytest.fail("launched"))
    with pytest.raises(ValueError, match="sageattn_kvcache8_prefill"):
        sab.sageattn_kvcache8(**{**_args(), "max_seqlen_q": 17}, shared_prefix_len=2048)


# ------------------------------------------------------------------------------------------------ 2. C ABI
def test_c_abi_export_and_error_codes():
    from sageattention_b200 import _capi
    lib = _capi.lib()
    fn = lib.sab_kvcache8_attn_shared
    one = 16          # a non-null, 16-byte aligned address: every call below fails its checks before touching it

    def a(**kw):
        p = dict(q=one, dtype=1, ptrs=(one,) * 5, out=one, lse=None, cu=one, used=one, table=one, ts=4, mp=4, nseq=2, Tq=2, Hq=8,
                 Hkv=2, D=128, ps=16, st=(1024, 128, 1024, 128), msq=1, causal=1, ws=one, spl=1024)
        p.update(kw)
        return fn(p["q"], p["dtype"], *p["ptrs"], p["out"], p["lse"], p["cu"], p["used"], p["table"], p["ts"], p["mp"], p["nseq"],
                  p["Tq"], p["Hq"], p["Hkv"], p["D"], p["ps"], *p["st"], p["msq"], p["causal"], 0.1, p["ws"], p["spl"], None)
    assert a(spl=-1) == -1 and b"shared_prefix_len must be >= 0" in lib.sab_last_error()
    assert a(spl=-(2 ** 31)) == -1 and b">= 0" in lib.sab_last_error()
    assert a(table=None) == -1 and b"null" in lib.sab_last_error()
    assert a(ws=None) == -1 and b"null" in lib.sab_last_error()
    assert a(q=None, spl=-1) == -1
    assert a(D=80) == -2 and b"head dim" in lib.sab_last_error()
    assert a(Hq=6, Hkv=4) == -1 and b"divisible" in lib.sab_last_error()
    assert a(msq=17) == -1 and b"query rows" in lib.sab_last_error()
    assert a(mp=2 ** 27, ts=2 ** 27, ps=16) == -1


def test_public_name_is_exported():
    from sageattention_b200 import _capi
    with open(os.path.join(ROOT, "include", "sageattn_b200.h")) as fh:
        header = fh.read()
    assert "sab_kvcache8_attn_shared" in _capi.EXPORTS and "int sab_kvcache8_attn_shared(" in header


# ------------------------------------------------------------------------------------------------ 3. benchmark counts
def test_bench_counts():
    sys.path.insert(0, ROOT)
    import bench_kvcache8_shared as bs
    assert bs.CHUNK == _chunk()
    w = {x.name: x for x in bs.WORKLOADS}
    assert set(w) == {"parallel_sampling", "system_prompt", "shared_verification"}
    ps, sp, sv = w["parallel_sampling"], w["system_prompt"], w["shared_verification"]
    assert ps.lens_q == [1] * 32 and ps.lens_k == [8192 + 64 * i for i in range(32)] and ps.shared_prefix == 8192
    assert sp.lens_q == [1] * 64 and sp.lens_k[0] == 4096 + 1024 and sp.lens_k[-1] == 4096 + 8192 and sp.shared_prefix == 4096
    assert sv.lens_q == [4] * 16 and sv.lens_k == [8192 + 512] * 16 and sv.shared_prefix == 8192
    # without sharing: every key of every sequence
    assert bs.keys_read(ps, False) == 32 * 8192 + 64 * sum(range(32))
    # parallel_sampling: 16 sequences per CTA (G = 4, Lq = 1), 2 slices x 8 shared chunks, plus the own keys
    assert bs.keys_read(ps, True) == 2 * 8 * 1024 + 64 * sum(range(32))
    assert 6.0 < bs.keys_read(ps, False) / bs.keys_read(ps, True) < 6.2
    # system_prompt: 4 slices x 4 shared chunks
    assert bs.keys_read(sp, True) == 4 * 4 * 1024 + sum(sp.lens_k) - 64 * 4096
    # shared_verification: 4 sequences per CTA; Lk - Lq + 1 = 8701 >= 8192, so all 8 chunks are shared: 4 slices x 8 chunks
    assert bs.keys_read(sv, True) == 4 * 8 * 1024 + 16 * 512
    assert bs.bytes_read(ps, True) == bs.keys_read(ps, True) * 8 * (2 * 128 + 8)
    # the sharing rule: causal, (c + 1) C <= Lk - Lq + 1
    assert bs.taken_chunks(1, 2047, 8192) == 1 and bs.taken_chunks(1, 2048, 8192) == 2
    assert bs.taken_chunks(4, 2050, 8192) == 1 and bs.taken_chunks(4, 2051, 8192) == 2
    assert bs.taken_chunks(0, 9000, 8192) == 0 and bs.taken_chunks(1, 9000, 2047) == 1
