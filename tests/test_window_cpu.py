"""CPU tests of the sliding-window attention: the CPU restatement (attn_window_oracle) against the dense restatement and fp64
exact windowed attention, the C entries' argument checks (no GPU needed: they run before anything touches the device), the
public function's guards and the new exports."""
import math
import os
import re

import pytest
import torch

from attn_bwd_oracle import elementwise_ratio
from attn_window_oracle import E4M3, attn_int8_fp8_window, window_mask, window_tiles
from oracle import sage_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _operands(B, Hq, Hkv, Sq, Sk, D, gran, seed=0):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(B, Hq, Sq, D, generator=g).half()
    k = (torch.randn(B, Hkv, Sk, D, generator=g) + 2.0 * torch.randn(B, Hkv, 1, D, generator=g)).half()
    v = torch.randn(B, Hkv, Sk, D, generator=g).half()
    km = k.mean(dim=2, keepdim=True)
    if gran == "per_warp":
        q8, qs, k8, ks = O.per_warp_int8_cuda(q, k, km)
    else:
        q8, qs, k8, ks = O.quant_per_thread_int8_triton(q, k, km)
    v8, vs, _ = O.per_channel_fp8_cuda(v, "HND", 448.0)
    return q, k, v, q8, qs, k8, ks, v8, vs


@pytest.mark.parametrize("gran", ["per_thread", "per_warp"])
@pytest.mark.parametrize("causal", [False, True])
def test_unbounded_window_is_the_dense_restatement_bitwise(gran, causal):
    """(-1, -1) is the dense call and (-1, 0) its causal call; the restatement gives the dense restatement's bits."""
    B, Hq, Hkv, S, D = 1, 2, 1, 300, 64
    _, _, _, q8, qs, k8, ks, v8, vs = _operands(B, Hq, Hkv, S, S, D, gran)
    kw = dict(qk_quant_gran=gran, sm_scale=D ** -0.5, lazy_tau=4, return_lse=True)
    o_ref, l_ref = O.attn_int8_fp8_cuda(q8, k8, v8, qs, ks, vs, is_causal=causal, **kw)
    for window in ([(-1, -1), (S, S)] if not causal else [(-1, -1), (-1, 0)]):
        o, l = attn_int8_fp8_window(q8, k8, v8, qs, ks, vs, window=window, is_causal=causal, **kw)
        assert torch.equal(o, o_ref) and torch.equal(l, l_ref), window
    if not causal:
        o, l = attn_int8_fp8_window(q8, k8, v8, qs, ks, vs, window=(-1, 0), **kw)
        o_c, l_c = O.attn_int8_fp8_cuda(q8, k8, v8, qs, ks, vs, is_causal=True, **kw)
        assert torch.equal(o, o_c) and torch.equal(l, l_c)


def _exact(q, k, v, em, scale):
    g = q.size(1) // k.size(1)
    s = (q.double() @ k.double().repeat_interleave(g, 1).transpose(-1, -2)) * scale
    p = torch.softmax(s.masked_fill(~em, -math.inf), dim=-1).nan_to_num(0.0)
    return p @ v.double().repeat_interleave(g, 1)


WINDOWS = [(0, 0), (1, 0), (63, 64), (127, 0), (200, 37), (1000, -1), (-1, 100)]


@pytest.mark.parametrize("window", WINDOWS)
@pytest.mark.parametrize("shape", [(320, 320, False), (320, 320, True), (400, 150, False), (150, 400, False)])
def test_restatement_matches_exact_windowed_attention(window, shape):
    Sq, Sk, causal = shape
    B, Hq, Hkv, D = 1, 2, 1, 64
    q, k, v, q8, qs, k8, ks, v8, vs = _operands(B, Hq, Hkv, Sq, Sk, D, "per_thread", seed=Sq + Sk + window[0])
    o, lse = attn_int8_fp8_window(q8, k8, v8, qs, ks, vs, window=window, is_causal=causal, sm_scale=D ** -0.5, return_lse=True)
    em = window_mask(Sq, Sk, *window, is_causal=causal)
    ref = _exact(q, k, v, em, D ** -0.5)
    rows = em.any(-1)
    assert torch.isfinite(o).all() and not torch.isnan(lse).any()
    assert torch.all(o[:, :, ~rows] == 0) and torch.all(torch.isneginf(lse[:, :, ~rows]))
    assert torch.isfinite(lse[:, :, rows]).all()
    # rows with >= 128 visible keys against exact attention at the parity suite's tolerance; every visible row within the e4m3
    # rounding (2^-4 relative) of P and of V's largest element, which a row that sees a handful of keys carries
    wide = em.sum(-1) >= 128
    if wide.any():
        assert (o.double() - ref)[:, :, wide].abs().max().item() < 6e-2
    assert (o.double() - ref)[:, :, rows].abs().max().item() < 0.13 * v.abs().max().item()


def test_window_tiles_cover_exactly_the_visible_tiles():
    for Sq, Sk in ((300, 300), (200, 700), (700, 200), (1, 65), (129, 1)):
        for left, right in WINDOWS + [(-1, -1), (-1, 0), (5, 3)]:
            for causal in ([False, True] if Sq == Sk else [False]):
                em = window_mask(Sq, Sk, left, right, causal)
                for r0 in range(0, Sq, 128):
                    r1 = min(r0 + 128, Sq)
                    j_lo, j_hi = window_tiles(r0, r1 - 1, Sk, left, right, causal)
                    vis = [j for j in range((Sk + 63) // 64) if em[r0:r1, 64 * j:64 * j + 64].any()]
                    assert list(range(j_lo, j_hi)) == vis, (Sq, Sk, left, right, causal, r0)


def test_bottom_rows_start_in_a_later_tile():
    """left = 10: in Q block 1, row 128 sees keys from 118 (tile 1) and row 255 from 245 (tile 3).  The bottom rows see nothing of
    the block's first tiles: their m and d must not move there, and the result must match exact attention."""
    B, Hq, Hkv, S, D = 1, 1, 1, 384, 64
    q, k, v, q8, qs, k8, ks, v8, vs = _operands(B, Hq, Hkv, S, S, D, "per_warp", seed=9)
    assert window_tiles(128, 255, S, 10, 0) == (1, 4)
    for tau in (4, 0):
        o = attn_int8_fp8_window(q8, k8, v8, qs, ks, vs, window=(10, 0), qk_quant_gran="per_warp", sm_scale=D ** -0.5,
                                 lazy_tau=tau)
        ref = _exact(q, k, v, window_mask(S, S, 10, 0), D ** -0.5)
        assert torch.isfinite(o).all() and (o.double() - ref).abs().max().item() < 0.13 * v.abs().max().item()


# ------------------------------------------------------------------------------------------------ the bound of the restatement
def _bound_case(window=(200, 37), dt=torch.float16, gran="per_thread"):
    """The restatement with its bound at 700 x 700, GQA 4:2, D=64, and the keyword arguments to call it again."""
    _, _, _, q8, qs, k8, ks, v8, vs = _operands(1, 4, 2, 700, 700, 64, gran, seed=3)
    kw = dict(qk_quant_gran=gran, sm_scale=0.125, lazy_tau=4, return_lse=True, out_dtype=dt)
    o, lse, bd = attn_int8_fp8_window(q8, k8, v8, qs, ks, vs, window=window, bound=True, **kw)
    return (q8, k8, v8, qs, ks, vs), kw, o, bd


def _worst(o, bd):
    return float(elementwise_ratio(o, bd.o, bd.o_bound).max())


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
def test_bound_accepts_every_ambiguous_p_flipped(dt):
    """A kernel whose P8 takes the other candidate code on every ambiguous element (P within eps_P of an e4m3 rounding midpoint)
    is within the bound; the case has such elements."""
    ops_, kw, o, bd = _bound_case(dt=dt)
    assert bd.ambiguous > 0 and _worst(o, bd) <= 1.0
    flipped = attn_int8_fp8_window(*ops_, window=(200, 37), p8_fn=lambda p8, lo, hi: torch.where(p8 == lo, hi, lo), **kw)[0]
    assert not torch.equal(flipped, o) and _worst(flipped, bd) <= 1.0


@pytest.mark.parametrize("window", [(201, 37), (199, 37), (200, 38), (200, 36)])
def test_bound_rejects_a_window_side_off_by_one(window):
    ops_, kw, o, bd = _bound_case()
    assert _worst(attn_int8_fp8_window(*ops_, window=window, **kw)[0], bd) > 1.0


def test_bound_rejects_one_unambiguous_p_moved_by_one_code():
    """The next e4m3 code on one element of one tile: the largest P below 448 (the last finite code) that is not ambiguous."""
    ops_, kw, o, bd = _bound_case()
    calls = []

    def bump(p8, lo, hi):
        calls.append(1)
        if len(calls) != 3:
            return p8
        cand = torch.where((lo == hi) & (p8 < 448.0), p8, 0.0)
        g, r, j = (int(x) for x in torch.unravel_index(cand.argmax(), cand.shape))
        p8 = p8.clone()
        p8[g, r, j] = (p8[g, r, j].to(E4M3).view(torch.uint8) + 1).view(E4M3).float()
        return p8
    moved = attn_int8_fp8_window(*ops_, window=(200, 37), p8_fn=bump, **kw)[0]
    assert (moved != o).any(-1).sum() == 1 and _worst(moved, bd) > 1.0


def test_bound_rejects_one_row_replaced_by_its_neighbour():
    _, _, o, bd = _bound_case()
    for r in (0, 127, 128, 350, 698):
        bad = o.clone()
        bad[0, 1, r] = o[0, 1, r + 1]
        assert _worst(bad, bd) > 1.0, r


# ------------------------------------------------------------------------------------------------ C entries and Python guards
def _call_fwd(lib, left=-1, right=-1, is_causal=0, Sq=128, Skv=128, D=128, out_dtype=0):
    return lib.sab_qk_int8_sv_f8_attn_window(1, 1, 1, 16, None, 1, 1, None, None, out_dtype, 1, 2, 2, Sq, Skv, D, *([0] * 10),
                                             is_causal, 3, 3, 1.0, 0, left, right, None)


def _call_bwd(lib, left=-1, right=-1, is_causal=0, Sq=128, Skv=128, D=128, out_dtype=0):
    return lib.sab_qk_int8_attn_bwd_window(*([16] * 15), out_dtype, 1, 2, 2, Sq, Skv, D, *([0] * 21), is_causal, 3, 3, 1.0, 0,
                                           left, right, None)


@pytest.mark.parametrize("call", [_call_fwd, _call_bwd])
def test_c_entries_reject_bad_arguments_without_a_gpu(call):
    from sageattention_b200 import _capi
    lib = _capi.lib()
    assert call(lib, left=-2) == -1 and b"window_size" in lib.sab_last_error()
    assert call(lib, right=-5) == -1 and b"window_size" in lib.sab_last_error()
    assert call(lib, left=3, is_causal=1, Skv=256) == -1 and b"must be equal for causal" in lib.sab_last_error()
    assert call(lib, left=3, D=96) == -2 and b"head dim" in lib.sab_last_error()
    assert call(lib, left=3, out_dtype=7) == -2 and b"dtype" in lib.sab_last_error()
    with pytest.raises(ValueError):
        _capi.check(call(lib, left=-2))


@pytest.mark.parametrize("window", [(-2, 0), (0, -3), (1.5, 2), (1,), (1, 2, 3), (True, 1), None, "ab"])
def test_public_function_rejects_bad_windows_before_any_launch(window):
    import sageattention_b200 as sab
    q = torch.randn(1, 2, 128, 64, dtype=torch.float16)
    with pytest.raises(ValueError):
        sab.sageattn_window(q, q, q, window_size=window)


def test_public_function_rejects_cpu_tensors():
    import sageattention_b200 as sab
    q = torch.randn(1, 2, 128, 64, dtype=torch.float16)
    with pytest.raises(AssertionError):
        sab.sageattn_window(q, q, q, window_size=(16, 16))


def test_every_new_export_is_present():
    import sageattention_b200 as sab
    from sageattention_b200 import _capi, ops
    assert "sageattn_window" in sab.__all__ and callable(sab.sageattn_window)
    assert callable(ops.qk_int8_sv_f8_attn_window) and callable(ops.qk_int8_attn_bwd_window)
    hdr = open(os.path.join(ROOT, "include", "sageattn_b200.h")).read()
    for name in ("sab_qk_int8_sv_f8_attn_window", "sab_qk_int8_attn_bwd_window"):
        assert name in _capi.EXPORTS and re.search(rf"\b{name}\s*\(", hdr)
        assert hasattr(_capi.lib(), name)
    # no existing entry point gains a window_size parameter
    import inspect
    for fn in (sab.sageattn, sab.sageattn_qk_int8_pv_fp8_cuda, sab.sageattn_blocksparse):
        assert "window_size" not in inspect.signature(fn).parameters
