"""CPU tests of sageattn_varlen_blocksparse and predict_block_mask_varlen (no GPU needed):
  1. argument and mask-shape checks raise before any launch (the host path runs on CPU tensors up to the kernel call);
  2. the new C entries refuse bad arguments with their error codes before touching the device;
  3. a CPU restatement of the packed predictor's rules (each sequence's blocks, npow and zero padding), causal with Lq != Lk
     included, against tests/block_predict_oracle.py per sequence;
  4. bench_blocksparse.py's packed pair and FLOP counts against the expanded element masks."""
import ctypes
import inspect

import pytest
import torch

from attn_blocksparse_oracle import expand_block_mask
from block_predict_oracle import block_stats, select


# ------------------------------------------------------------------------------------------------ 1. Python checks
def _reach_the_kernel_call(monkeypatch):
    """Run sageattn_varlen_blocksparse's host path on CPU tensors up to the quantisers + kernel call (_attn_varlen_f8), which
    records the block mask it receives instead of launching; F.pad is counted as a launch too."""
    from sageattention_b200 import core
    seen = []
    monkeypatch.setattr(core, "_check_inputs", lambda q, k, v: None)

    def fake(q, k, v, *args):
        seen.append(args[-2])                  # (..., return_lse, block_mask, window)
        return torch.zeros_like(q), torch.empty(0), None
    monkeypatch.setattr(core, "_attn_varlen_f8", fake)
    real_pad = core._pad_head_dim

    def pad(q, k, v):
        seen.append("pad")
        return real_pad(q, k, v)
    monkeypatch.setattr(core, "_pad_head_dim", pad)
    return seen


def test_mask_checks_raise_before_any_launch(monkeypatch):
    import sageattention_b200 as sab
    seen = _reach_the_kernel_call(monkeypatch)
    q, k = torch.zeros(10, 4, 64, dtype=torch.float16), torch.zeros(300, 2, 64, dtype=torch.float16)
    cu, cuk = torch.tensor([0, 4, 10], dtype=torch.int32), torch.tensor([0, 100, 300], dtype=torch.int64)
    good = torch.ones(2, 4, 1, 4, dtype=torch.bool)
    for bm in (good, good[:1], good[:, :1], good[:1, :1], torch.ones(2, 4, 1, 8, dtype=torch.bool)[..., ::2]):
        sab.sageattn_varlen_blocksparse(q, k, k, cu, cuk, 6, 200, bm)
        assert seen[-2] == "pad" and tuple(seen[-1].shape) == (2, 4, 1, 4)        # expanded to [nseq, Hq, nqb, nkb]
    n = len(seen)
    for bm in (torch.ones(2, 4, 1, 3, dtype=torch.bool), torch.ones(2, 4, 2, 4, dtype=torch.bool), torch.ones(3, 4, 1, 4, dtype=torch.bool),
               torch.ones(2, 2, 1, 4, dtype=torch.bool), torch.ones(4, 1, 4, dtype=torch.bool), torch.ones(1, 2, 4, 1, 4, dtype=torch.bool)):
        with pytest.raises(ValueError, match="block_mask shape"):
            sab.sageattn_varlen_blocksparse(q, k, k, cu, cuk, 6, 200, bm)
    with pytest.raises(AssertionError, match="torch.bool"):
        sab.sageattn_varlen_blocksparse(q, k, k, cu, cuk, 6, 200, good.to(torch.uint8))
    with pytest.raises(AssertionError, match="torch.bool"):
        sab.sageattn_varlen_blocksparse(q, k, k, cu, cuk, 6, 200, [[True]])
    with pytest.raises(ValueError, match="max_seqlen_k"):     # the shared-memory list of one mask row
        sab.sageattn_varlen_blocksparse(q, k, k, cu, cuk, 6, (1 << 20) + 1, torch.ones(1, 1, 1, (1 << 14) + 1, dtype=torch.bool))
    # the packed call's own checks come first, still before any launch
    for args in ((q, k, k, cu.float(), cuk, 6, 200), (q, k, k, cu, cuk[:2], 6, 200), (q, k, k, cu, cuk, 0, 200),
                 (q, k, k[:299], cu, cuk, 6, 200)):
        with pytest.raises(ValueError):
            sab.sageattn_varlen_blocksparse(*args, good)
    assert len(seen) == n


def test_cpu_tensors_and_foreign_devices_are_rejected():
    import sageattention_b200 as sab
    q = torch.randn(10, 2, 64, dtype=torch.float16)
    cu = torch.tensor([0, 4, 10], dtype=torch.int32)
    with pytest.raises(AssertionError):
        sab.sageattn_varlen_blocksparse(q, q, q, cu, cu, 6, 6, torch.ones(2, 2, 1, 1, dtype=torch.bool))
    with pytest.raises(AssertionError):
        sab.predict_block_mask_varlen(q, q, cu, cu, 6, 6, cdf_threshold=0.9, sim_threshold=0.5)


def test_every_new_export_is_present():
    import sageattention_b200 as sab
    from sageattention_b200 import _capi, ops
    for name in ("sageattn_varlen_blocksparse", "predict_block_mask_varlen"):
        assert name in sab.__all__ and callable(getattr(sab, name))
    for name in ("qk_int8_sv_f8_attn_varlen_blocksparse", "qk_int8_attn_bwd_varlen_blocksparse", "block_stats_varlen",
                 "predict_block_mask_varlen"):
        assert callable(getattr(ops, name))
    for name in ("sab_qk_int8_sv_f8_attn_varlen_blocksparse", "sab_qk_int8_attn_bwd_varlen_blocksparse", "sab_block_stats_varlen",
                 "sab_predict_block_mask_varlen"):
        assert name in _capi.EXPORTS and hasattr(_capi.lib(), name)
    params = list(inspect.signature(sab.sageattn_varlen_blocksparse).parameters)
    assert params == ["q", "k", "v", "cu_seqlens_q", "cu_seqlens_k", "max_seqlen_q", "max_seqlen_k", "block_mask", "is_causal",
                      "qk_quant_gran", "sm_scale", "pv_accum_dtype", "smooth_k", "smooth_v", "return_lse"]
    params = inspect.signature(sab.predict_block_mask_varlen).parameters
    assert list(params)[:6] == ["q", "k", "cu_seqlens_q", "cu_seqlens_k", "max_seqlen_q", "max_seqlen_k"]
    assert all(params[n].kind == inspect.Parameter.KEYWORD_ONLY for n in ("cdf_threshold", "sim_threshold", "is_causal", "sm_scale"))


# ------------------------------------------------------------------------------------------------ 2. C entries
def _buf():
    buf = ctypes.create_string_buffer(64 + 16)
    return buf, (ctypes.addressof(buf) + 15) // 16 * 16


def _fwd(L, p, mask=True, strides=(0, 0, 0, 1), causal=0, D=128, q_gran=3, cu=True, max_q=64, max_k=64, Tq=64, Tk=64):
    c = p if cu else None
    return L.sab_qk_int8_sv_f8_attn_varlen_blocksparse(p, p, p, p, None, p, p, p, None, 1, 1, 2, 2, Tq, Tk, D, 128, 128, 128, 128, 128,
                                                       128, 128, causal, q_gran, 3, 1.0, c, c, c, c, c, max_q, max_k,
                                                       p if mask else None, *strides, None)


def _bwd(L, p, mask=True, strides=(0, 0, 0, 1), causal=0, D=128, q_gran=3, cu=True, max_q=64, max_k=64, Tq=64, Tk=64):
    c = p if cu else None
    return L.sab_qk_int8_attn_bwd_varlen_blocksparse(*([p] * 15), 1, 1, 2, 2, Tq, Tk, D, *([128] * 14), c, c, c, c, max_q, max_k,
                                                     causal, q_gran, 3, 1.0, p if mask else None, *strides, None)


@pytest.mark.parametrize("call", [_fwd, _bwd])
def test_c_entries_reject_bad_arguments_without_a_gpu(call):
    from sageattention_b200 import _capi
    L = _capi.lib()
    _keep, p = _buf()
    assert call(L, p, mask=False) == -1 and b"block_mask" in L.sab_last_error()
    assert call(L, p, strides=(0, -1, 0, 1)) == -1 and b"strides" in L.sab_last_error()
    assert call(L, p, q_gran=1) == -2 and b"per-warp or per-thread" in L.sab_last_error()
    assert call(L, p, max_k=(1 << 20) + 1) == -2 and b"max_seqlen_k" in L.sab_last_error()
    assert call(L, p, max_k=0) == -1
    assert call(L, p, cu=False) == -1 and b"cu_seqlens" in L.sab_last_error()
    assert call(L, p, D=96) == -2 and b"head dim" in L.sab_last_error()
    # causal with Lq != Lk is top-left inside each sequence: not refused (the call stops at the head dim, before the device)
    assert call(L, p, causal=1, Tq=64, Tk=200, D=96) == -2 and b"head dim" in L.sab_last_error()
    with pytest.raises(ValueError):
        _capi.check(call(L, p, mask=False))


def test_predictor_c_entries_reject_bad_arguments_without_a_gpu():
    from sageattention_b200 import _capi
    L = _capi.lib()
    _keep, p = _buf()

    def stats(x=p, cu=p, nseq=2, max_s=100, D=64, blk=128, st=(64, 8)):
        return L.sab_block_stats_varlen(x, 0, p, p, cu, nseq, max_s, 2, D, *st, blk, None)

    def sel(cu=p, max_q=100, max_k=100, causal=0, cdf=0.9, sim=0.5, D=64, Hkv=2):
        return L.sab_predict_block_mask_varlen(p, p, p, p, p, cu, cu, 2, 2, Hkv, max_q, max_k, D, causal, 0.125, cdf, sim, None)

    assert stats(cu=None) == -1 and b"cu_seqlens" in L.sab_last_error()
    assert stats(x=None) == -1
    assert stats(D=100) == -2 and b"head dim" in L.sab_last_error()
    assert stats(blk=32) == -1 and b"block size" in L.sab_last_error()
    assert stats(max_s=0) == -1 and stats(nseq=0) == -1
    assert stats(st=(12, 8)) == -1 and b"16-byte" in L.sab_last_error()
    assert sel(cu=None) == -1 and b"cu_seqlens" in L.sab_last_error()
    assert sel(cdf=0.0) == -1 and b"cdf_threshold" in L.sab_last_error()
    assert sel(sim=float("nan")) == -1 and b"sim_threshold" in L.sab_last_error()
    assert sel(max_k=(1 << 20) + 1) == -2 and b"kv_len" in L.sab_last_error()
    assert sel(Hkv=3) == -1 and b"divisible" in L.sab_last_error()
    assert sel(D=100) == -2 and b"head dim" in L.sab_last_error()
    # the dense entry refuses causal with Sq != Skv; the packed one does not (it stops at the head dim, before the device)
    assert L.sab_predict_block_mask(p, p, p, p, p, 1, 2, 2, 100, 300, 64, 1, 0.125, 0.9, 0.5, None) == -1
    assert sel(max_q=100, max_k=300, causal=1, D=100) == -2 and b"head dim" in L.sab_last_error()


def test_predictor_argument_checks_raise(monkeypatch):
    import sageattention_b200 as sab
    from sageattention_b200 import ops, predict
    calls = []
    for name in ("block_stats_varlen", "predict_block_mask_varlen"):
        monkeypatch.setattr(ops, name, lambda *a, _n=name: calls.append(_n))
    q = torch.zeros(10, 4, 64, dtype=torch.float16)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    cu = torch.tensor([0, 4, 10], dtype=torch.int32)
    m = predict.predict_block_mask_varlen(q, q[:, :2], cu, cu, 6, 6, cdf_threshold=0.9, sim_threshold=0.5, is_causal=True)
    assert tuple(m.shape) == (2, 4, 1, 1) and calls == ["block_stats_varlen", "block_stats_varlen", "predict_block_mask_varlen"]
    bad = [dict(cdf_threshold=0.0, sim_threshold=0.5), dict(cdf_threshold=0.9, sim_threshold=float("nan")),
           dict(cdf_threshold=0.9, sim_threshold=0.5, sm_scale=float("inf"))]
    for kw in bad:
        with pytest.raises(ValueError):
            sab.predict_block_mask_varlen(q, q, cu, cu, 6, 6, **kw)
    with pytest.raises(ValueError, match="max_seqlen_k"):
        sab.predict_block_mask_varlen(q, q, cu, cu, 6, (1 << 20) + 1, cdf_threshold=0.9, sim_threshold=0.5)
    with pytest.raises(ValueError):
        sab.predict_block_mask_varlen(q, q, cu, cu[:2], 6, 6, cdf_threshold=0.9, sim_threshold=0.5)
    with pytest.raises(ValueError, match="divisible"):
        sab.predict_block_mask_varlen(q, q[:, :3], cu, cu, 6, 6, cdf_threshold=0.9, sim_threshold=0.5)
    assert len(calls) == 3


# ------------------------------------------------------------------------------------------------ 3. packed predictor rules
def _packed_rules(q, k, lens_q, lens_k, **kw):
    """The packed predictor as its kernels define it, in fp64: per sequence b, the statistics of its own blocks and the selection
    over its own nq_b x nk_b blocks (select() sorts on exactly the candidates, so npow_b only fixes the fp32 summation order), then
    zeros everywhere else of the [nseq, Hq, ceil(max_q/128), ceil(max_k/64)] mask."""
    nseq, Hq = len(lens_q), q.size(1)
    mq, mk = max(max(lens_q), 1), max(max(lens_k), 1)
    out = torch.zeros(nseq, Hq, (mq + 127) // 128, (mk + 63) // 64, dtype=torch.bool)
    sq = sk = 0
    for b, (lq, lk) in enumerate(zip(lens_q, lens_k)):
        if lq and lk:
            qm, qs = block_stats(q[sq:sq + lq].transpose(0, 1)[None], 128)
            km, ks = block_stats(k[sk:sk + lk].transpose(0, 1)[None], 64)
            m, _ = select(qm, qs, km, ks, lq, lk, sm_scale=q.size(-1) ** -0.5, **kw)
            out[b, :, :m.size(2), :m.size(3)] = m[0]
        sq, sk = sq + lq, sk + lk
    return out


@pytest.mark.parametrize("causal", [False, True])
def test_packed_predictor_rules_are_the_dense_rules_per_sequence(causal):
    """Each sequence's slice is the oracle's predict_block_mask on that sequence alone (causal top-left inside the sequence,
    Lq != Lk included), entries outside the slices and of empty sequences are False, and no row of a sequence with keys is
    empty when causal (its diagonal blocks are forced)."""
    from block_predict_oracle import predict_block_mask
    lens_q, lens_k = [300, 0, 129, 64, 200, 1], [100, 50, 0, 300, 200, 65]
    g = torch.Generator().manual_seed(0)
    q = torch.randn(sum(lens_q), 4, 64, generator=g, dtype=torch.float64)
    k = torch.randn(sum(lens_k), 2, 64, generator=g, dtype=torch.float64) + torch.randn(1, 2, 64, generator=g, dtype=torch.float64)
    for cdf, sim in ((0.9, 0.05), (0.5, -1.0), (1.0, 0.5)):
        kw = dict(cdf_threshold=cdf, sim_threshold=sim, is_causal=causal)
        got = _packed_rules(q, k, lens_q, lens_k, **kw)
        sq = sk = 0
        for b, (lq, lk) in enumerate(zip(lens_q, lens_k)):
            nq, nk = (lq + 127) // 128, (lk + 63) // 64
            if lq and lk:
                ref, _ = predict_block_mask(q[sq:sq + lq][None], k[sk:sk + lk][None], tensor_layout="NHD", **kw)
                assert torch.equal(got[b, :, :nq, :nk], ref[0])
                if causal:
                    assert got[b, :, :nq, :nk].any(-1).all()
                    j, i = torch.arange(nk)[None, :], torch.arange(nq)[:, None]
                    assert not got[b, :, :nq, :nk][:, 64 * j.expand(nq, nk) > 128 * i.expand(nq, nk) + 127].any()
            else:
                nq = nk = 0
            outside = torch.ones_like(got[b])
            outside[:, :nq, :nk] = False
            assert not got[b][outside].any()
            sq, sk = sq + lq, sk + lk


# ------------------------------------------------------------------------------------------------ 4. bench counts
@pytest.mark.parametrize("causal", [False, True])
def test_bench_pair_and_flop_counts_agree_with_the_element_masks(causal):
    from bench_blocksparse import _varlen_pairs
    lens_q, lens_k = [300, 1, 0, 129, 700, 64], [300, 1, 5, 129, 700, 64]
    if not causal:
        lens_k = [100, 65, 5, 0, 700, 200]
    g = torch.Generator().manual_seed(1)
    mq, mk = max(lens_q), max(lens_k)
    for shape in ((6, 3), (1, 1), (6, 1)):
        bm = torch.rand(*shape, (mq + 127) // 128, (mk + 63) // 64, generator=g) < 0.4
        want = 0
        for b, (lq, lk) in enumerate(zip(lens_q, lens_k)):
            if lq and lk:
                mb = bm[min(b, bm.size(0) - 1), :, :(lq + 127) // 128, :(lk + 63) // 64]
                em = expand_block_mask(mb[None], lq, lk)[0]
                if causal:
                    em = em & torch.ones(lq, lk, dtype=torch.bool).tril()
                want += int(em.sum())
        assert _varlen_pairs(bm, lens_q, lens_k, causal) == want
    # all-True: the dense pair count; FLOPs are 4 * D (forward) or 10 * D (backward) per visible pair and Q head
    ones = torch.ones(1, 2, (mq + 127) // 128, (mk + 63) // 64, dtype=torch.bool)
    dense = sum(lq * (min(lq, lk) * (min(lq, lk) + 1) // 2 + max(lq - lk, 0) * lk) // lq if causal else lq * lk
                for lq, lk in zip(lens_q, lens_k) if lq and lk)
    assert _varlen_pairs(ones, lens_q, lens_k, causal) == 2 * dense
