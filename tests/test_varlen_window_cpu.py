"""CPU tests of sageattn_varlen_window's host side and of the rules its kernels rely on:
  1. the Python checks that answer before any launch (window_size, cu_seqlens) and the clamp that keeps an oversized side out
     of ctypes' silent int32 truncation;
  2. the two C entries' argument checks, which run before anything touches the device (a causal call with Lq != Lk is not
     refused there);
  3. on the CPU restatement of the window forward (attn_window_oracle), per sequence: causal (left, right) is non-causal
     (left, 0) to the bit, and clamping a side at the sequence's own lengths changes neither visibility nor bits;
  4. bench_window.py's packed pair and tile counts against window_mask."""
import ctypes

import numpy as np
import pytest
import torch

from attn_window_oracle import attn_int8_fp8_window, window_mask, window_tiles
from oracle import sage_oracle as O

WINDOWS = [(0, 0), (1, 0), (63, 64), (127, 0), (200, 37), (1000, -1), (-1, 100), (-1, -1), (-1, 0)]
SHAPES = [(100, 300), (300, 100), (1, 129), (129, 1), (64, 65), (200, 200)]


# ------------------------------------------------------------------------------------------------ 1. Python checks
@pytest.mark.parametrize("window", [(-2, 0), (0, -3), (1.5, 2), (1,), (1, 2, 3), (True, 1), (1, False), None, "ab", {0: 1}])
def test_bad_window_size_raises_before_any_launch(window):
    import sageattention_b200 as sab
    q = torch.randn(10, 2, 64, dtype=torch.float16)
    cu = torch.tensor([0, 4, 10], dtype=torch.int32)
    with pytest.raises(ValueError):
        sab.sageattn_varlen_window(q, q, q, cu, cu, 6, 6, window_size=window)


def test_cpu_tensors_are_rejected():
    import sageattention_b200 as sab
    q = torch.randn(10, 2, 64, dtype=torch.float16)
    cu = torch.tensor([0, 4, 10], dtype=torch.int32)
    with pytest.raises(AssertionError):
        sab.sageattn_varlen_window(q, q, q, cu, cu, 6, 6, window_size=(4, 4))


def _reach_the_kernel_call(monkeypatch):
    """Run sageattn_varlen_window's host path on CPU tensors up to the quantisers + kernel call (_attn_varlen_f8), which records
    the window it receives instead of launching."""
    from sageattention_b200 import core
    seen = []
    monkeypatch.setattr(core, "_check_inputs", lambda q, k, v: None)

    def fake(q, k, v, *args):
        seen.append(args[-1])
        return torch.zeros_like(q), torch.empty(0), None
    monkeypatch.setattr(core, "_attn_varlen_f8", fake)
    return seen


def test_bad_cu_seqlens_raise_before_any_launch(monkeypatch):
    import sageattention_b200 as sab
    seen = _reach_the_kernel_call(monkeypatch)
    q, k = torch.zeros(10, 4, 64, dtype=torch.float16), torch.zeros(12, 2, 64, dtype=torch.float16)
    cu, cuk = torch.tensor([0, 4, 10], dtype=torch.int32), torch.tensor([0, 5, 12], dtype=torch.int64)
    sab.sageattn_varlen_window(q, k, k, cu, cuk, 6, 7, (3, 0))
    assert seen == [(3, 0)]
    bad = [(q, k, cu.float(), cuk, 6, 7), (q, k, cu[None], cuk, 6, 7), (q, k, cu[:1], cuk[:1], 6, 7), (q, k, cu, cuk[:2], 6, 7),
           (q, k, cu, cuk, 0, 7), (q, k, cu, cuk, 6, True), (q[:0], k, cu, cuk, 6, 7), (q[None], k, cu, cuk, 6, 7)]
    for q_, k_, cq, ck, mq, mk in bad:
        with pytest.raises(ValueError):
            sab.sageattn_varlen_window(q_, k_, k_, cq, ck, mq, mk, (3, 0))
    with pytest.raises(ValueError):     # k and v of different shapes
        sab.sageattn_varlen_window(q, k, k[:11], cu, cuk, 6, 7, (3, 0))
    assert len(seen) == 1


def test_oversized_sides_are_clamped_before_ctypes(monkeypatch):
    """A side >= max_seqlen (the longest sequence) sees every key in every sequence: it becomes -1, so that no Python int wider
    than a C int reaches the C ABI (ctypes would truncate 2**40 + 5 to 5)."""
    import sageattention_b200 as sab
    from sageattention_b200.core import _varlen_window_arg
    assert _varlen_window_arg((2 ** 40, 2 ** 40 + 5), 300, 200) == (-1, -1)
    assert _varlen_window_arg((299, 199), 300, 200) == (299, 199)
    assert _varlen_window_arg((300, 200), 300, 200) == (-1, -1)
    assert _varlen_window_arg((-1, 0), 300, 200) == (-1, 0)
    seen = _reach_the_kernel_call(monkeypatch)
    q = torch.zeros(10, 2, 64, dtype=torch.float16)
    cu = torch.tensor([0, 4, 10], dtype=torch.int32)
    for window, want in (((2 ** 40, 3), (-1, 3)), ((5, 2 ** 63), (5, -1)), ((np.int64(4), 2), (4, 2)), ((6, 5), (-1, 5))):
        sab.sageattn_varlen_window(q, q, q, cu, cu, 6, 6, window)
        assert seen[-1] == want and all(type(x) is int for x in seen[-1])


# ------------------------------------------------------------------------------------------------ 2. C entries
def _buf():
    buf = ctypes.create_string_buffer(64 + 16)
    return buf, (ctypes.addressof(buf) + 15) // 16 * 16


def _fwd(L, p, left=-1, right=-1, causal=0, D=128, q_gran=3, cu=True, max_q=64, Tq=64, Tk=64):
    c = p if cu else None
    return L.sab_qk_int8_sv_f8_attn_varlen_window(p, p, p, p, None, p, p, p, None, 1, 1, 2, 2, Tq, Tk, D, 128, 128, 128, 128, 128,
                                                  128, 128, causal, q_gran, 3, 1.0, c, c, c, c, c, max_q, left, right, None)


def _bwd(L, p, left=-1, right=-1, causal=0, D=128, q_gran=3, cu=True, max_q=64, max_k=64, Tq=64, Tk=64):
    c = p if cu else None
    return L.sab_qk_int8_attn_bwd_varlen_window(*([p] * 15), 1, 1, 2, 2, Tq, Tk, D, *([128] * 14), c, c, c, c, max_q, max_k, causal,
                                                q_gran, 3, 1.0, left, right, None)


@pytest.mark.parametrize("call", [_fwd, _bwd])
def test_c_entries_reject_bad_arguments_without_a_gpu(call):
    from sageattention_b200 import _capi
    L = _capi.lib()
    _keep, p = _buf()
    assert call(L, p, left=-2) == -1 and b"window_size" in L.sab_last_error()
    assert call(L, p, right=-7) == -1 and b"window_size" in L.sab_last_error()
    assert call(L, p, left=3, cu=False) == -1 and b"cu_seqlens_q" in L.sab_last_error()
    assert call(L, p, left=3, max_q=0) == -1
    assert call(L, p, left=3, q_gran=1) == -1 and b"q_gran" in L.sab_last_error()
    assert call(L, p, left=3, D=96) == -2 and b"head dim" in L.sab_last_error()
    # causal with Lq != Lk is top-left inside each sequence: not refused (the call stops at the head dim, before the device)
    assert call(L, p, left=3, causal=1, Tq=64, Tk=200, D=96) == -2 and b"head dim" in L.sab_last_error()
    with pytest.raises(ValueError):
        _capi.check(call(L, p, left=-2))


def test_every_new_export_is_present():
    import inspect
    import sageattention_b200 as sab
    from sageattention_b200 import _capi, ops
    assert "sageattn_varlen_window" in sab.__all__ and callable(sab.sageattn_varlen_window)
    assert callable(ops.qk_int8_sv_f8_attn_varlen_window) and callable(ops.qk_int8_attn_bwd_varlen_window)
    for name in ("sab_qk_int8_sv_f8_attn_varlen_window", "sab_qk_int8_attn_bwd_varlen_window"):
        assert name in _capi.EXPORTS and hasattr(_capi.lib(), name)
    params = inspect.signature(sab.sageattn_varlen_window).parameters
    assert list(params)[:8] == ["q", "k", "v", "cu_seqlens_q", "cu_seqlens_k", "max_seqlen_q", "max_seqlen_k", "window_size"]
    assert not any(p.kind == p.VAR_KEYWORD for p in params.values())
    assert "window_size" not in inspect.signature(sab.sageattn_varlen_qk_int8_pv_fp8_cuda).parameters


# ------------------------------------------------------------------------------------------------ 3. per-sequence rules
def _operands(Sq, Sk, gran, seed):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(1, 2, Sq, 64, generator=g).half()
    k = (torch.randn(1, 1, Sk, 64, generator=g) + 2.0 * torch.randn(1, 1, 1, 64, generator=g)).half()
    v = torch.randn(1, 1, Sk, 64, generator=g).half()
    km = k.mean(dim=2, keepdim=True)
    q8, qs, k8, ks = (O.per_warp_int8_cuda if gran == "per_warp" else O.quant_per_thread_int8_triton)(q, k, km)
    v8, vs, _ = O.per_channel_fp8_cuda(v, "HND", 448.0)
    return q8, k8, v8, qs, ks, vs


@pytest.mark.parametrize("gran", ["per_thread", "per_warp"])
def test_causal_window_is_noncausal_with_right_0_per_sequence(gran):
    """The rule that lets a packed causal sequence with Lq != Lk (which sageattn_window refuses) be pinned to sageattn_window's
    non-causal (left, 0): same visibility, same tiles, same bits in the restatement."""
    for i, (Sq, Sk) in enumerate(SHAPES):
        q8, k8, v8, qs, ks, vs = _operands(Sq, Sk, gran, seed=i)
        for left, right in WINDOWS:
            assert torch.equal(window_mask(Sq, Sk, left, right, True), window_mask(Sq, Sk, left, 0, False))
            for r0 in range(0, Sq, 128):
                r1 = min(r0 + 128, Sq) - 1
                assert window_tiles(r0, r1, Sk, left, right, True) == window_tiles(r0, r1, Sk, left, 0, False)
            kw = dict(qk_quant_gran=gran, sm_scale=0.125, return_lse=True)
            o_c, l_c = attn_int8_fp8_window(q8, k8, v8, qs, ks, vs, window=(left, right), is_causal=True, **kw)
            o_n, l_n = attn_int8_fp8_window(q8, k8, v8, qs, ks, vs, window=(left, 0), is_causal=False, **kw)
            assert torch.equal(o_c, o_n) and torch.equal(l_c, l_n), (Sq, Sk, left, right)


def test_per_sequence_clamp_keeps_visibility_and_bits():
    """A side >= the sequence's own Lq (left) or Lk (right) becomes -1 in the kernels: the same visible keys, the same tiles and
    the same restated output; that is the clamp sab_qk_int8_sv_f8_attn_window applies to the dense call on that sequence."""
    for i, (Sq, Sk) in enumerate(SHAPES):
        q8, k8, v8, qs, ks, vs = _operands(Sq, Sk, "per_thread", seed=10 + i)
        for left, right in WINDOWS + [(Sq, Sk), (Sq + 50, 3), (4, Sk + 1), (2 ** 31 - 1, 2 ** 31 - 1)]:
            cl = (-1 if left >= Sq else left, -1 if right >= Sk else right)
            for causal in (False, True):
                assert torch.equal(window_mask(Sq, Sk, left, right, causal), window_mask(Sq, Sk, *cl, causal))
                for r0 in range(0, Sq, 128):
                    r1 = min(r0 + 128, Sq) - 1
                    assert window_tiles(r0, r1, Sk, left, right, causal) == window_tiles(r0, r1, Sk, *cl, causal)
            if left < 2 ** 20:
                o, l = attn_int8_fp8_window(q8, k8, v8, qs, ks, vs, window=(left, right), sm_scale=0.125, return_lse=True)
                oc, lc = attn_int8_fp8_window(q8, k8, v8, qs, ks, vs, window=cl, sm_scale=0.125, return_lse=True)
                assert torch.equal(o, oc) and torch.equal(l, lc)


# ------------------------------------------------------------------------------------------------ 4. bench counts
@pytest.mark.parametrize("causal, window", [(True, (1024, 0)), (True, (100, 0)), (False, (300, 200)), (False, (-1, 50))])
def test_bench_packed_counts_agree_with_window_mask(causal, window):
    from bench_window import _visible_varlen
    lens = [300, 1, 129, 700, 64]
    pairs, tiles, masked, dense = _visible_varlen(lens, causal, *window)
    want_pairs = want_tiles = want_masked = want_dense = 0
    for L in lens:
        em = window_mask(L, L, *window, is_causal=causal)
        want_pairs += int(em.sum())
        for r0 in range(0, L, 128):
            blk = em[r0:r0 + 128]
            for j in range((L + 63) // 64):
                t = blk[:, 64 * j:64 * j + 64]
                if t.any():
                    want_tiles += 1
                    # masked: some row of the block does not see every key of the tile that exists
                    want_masked += int(not t.all() or t.size(1) < 64)
            want_dense += (min(r0 + 128, L) - 1) // 64 + 1 if causal else (L + 63) // 64
    assert (pairs, tiles, dense) == (want_pairs, want_tiles, want_dense)
    assert masked == want_masked
