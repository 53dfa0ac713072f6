"""GPU tests (-m gpu) of sageattn_varlen_kvcache, attention of packed queries against a paged KV cache:
  1. non-causal: o and lse are the bits of sageattn_varlen_qk_int8_pv_fp8_cuda on the gathered, packed K / V;
  2. causal (bottom-right): for Lk_b >= Lq_b, sequence b's rows are the bits of sageattn_window(..., (-1, Lk_b - Lq_b)) on that
     sequence alone, lse within the packed window test's bound; for Lk_b < Lq_b the first Lq_b - Lk_b rows are 0 / -inf and the
     others lie within the per-element bound of the CPU restatement (tests/attn_kvcache_oracle.py);
  3. the paged quantisers give the bits of the packed ones on the gathered tensor;
  4. every cache slot the call must not read (unreferenced pages, slots past Lk_b, table entries past the used pages) holds NaN,
     and the output stays finite and unchanged.
Across D 64 / 128, fp16 / bf16, per_thread / per_warp, smooth_k off, smooth_v with "fp32", GQA, page sizes 1 / 16 / 64 / 96 and a
padded unpaged cache, shuffled tables, shared prefix pages and a strided kv_cache[0] view; lengths crossing 64-key and 128-row
boundaries, Lq = 1, Lk = Lq, Lk < Lq and empty sequences."""
import pytest
import torch

from attn_bwd_oracle import check_elementwise
from attn_kvcache_oracle import attn_sequence, gather_pages
from test_gpu_varlen_window import _lse_bound

pytestmark = pytest.mark.gpu

BF, FP = torch.bfloat16, torch.float16
# Lk > Lq, Lq = 0 with keys, Lk = 0, Lq = Lk = 1, Lk = Lq = 300, Lk < Lq across 128 rows, Lk < Lq short, Lk > Lq by 192
LENS_Q = [129, 0, 64, 1, 300, 200, 8, 63, 65]
LENS_K = [200, 7, 0, 1, 300, 70, 3, 255, 129]


def _cu(lens):
    return torch.tensor([0] + torch.cumsum(torch.tensor(lens), 0).tolist(), dtype=torch.int32, device="cuda")


def make_cache(lens_k, Hkv, D, dt, page_size, layout, seed):
    """(k_cache, v_cache, block_table, seqused_k).  layout: "shuffled" (pages in random order), "shared" (every sequence's first
    two pages are the same two pages), "padded" (an unpaged [nseq, S_cap, Hkv, D] cache: page_size = S_cap, table arange(nseq)),
    "strided" (shuffled pages of k = kv[0], v = kv[1] of one [2, num_pages, page_size, Hkv, D] buffer).  Every slot the call must
    not read is NaN: slots past Lk_b, pages no sequence uses, and one spare page every table entry past the used ones names."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    nseq = len(lens_k)
    if layout == "padded":
        page_size = max(lens_k) + 5
    pages = [(n + page_size - 1) // page_size for n in lens_k]
    npre = 2 if layout == "shared" else 0
    own = [max(0, p - npre) for p in pages]
    num_pages = npre + sum(own) + 3 if layout != "padded" else nseq
    shape = (num_pages, page_size, Hkv, D)
    if layout == "strided":
        kv = torch.randn((2,) + shape, generator=g, device="cuda").to(dt)
        k_cache, v_cache = kv[0], kv[1]
    else:
        k_cache = torch.randn(shape, generator=g, device="cuda").to(dt)
        v_cache = torch.randn(shape, generator=g, device="cuda").to(dt)
    k_cache += (2.0 * torch.randn(Hkv, D, generator=g, device="cuda")).to(dt)
    max_pages = max(pages) + 2
    if layout == "padded":
        table = torch.arange(nseq, dtype=torch.int32, device="cuda")[:, None]
    else:
        perm = torch.randperm(num_pages, generator=g, device="cuda").to(torch.int32)
        spare = perm[-1]                                       # never holds a token
        table = spare.repeat(nseq, max_pages)
        nxt = npre
        for b, p in enumerate(pages):
            table[b, :min(p, npre)] = perm[:min(p, npre)]
            table[b, min(p, npre):p] = perm[nxt:nxt + own[b]]
            nxt += own[b]
    read = torch.zeros(num_pages, page_size, dtype=torch.bool, device="cuda")
    for b, n in enumerate(lens_k):
        t = torch.arange(n, device="cuda")
        read[table[b, t // page_size].long(), t % page_size] = True
    for c in (k_cache, v_cache):
        c[~read] = float("nan")
    return k_cache, v_cache, table, torch.tensor(lens_k, dtype=torch.int32, device="cuda")


def _inputs(lens_q, lens_k, Hq, Hkv, D, dt, page_size, layout, seed):
    g = torch.Generator(device="cuda").manual_seed(seed + 1000)
    q = torch.randn(sum(lens_q) + 3, Hq, D, generator=g, device="cuda").to(dt)[:sum(lens_q)]
    return (q,) + make_cache(lens_k, Hkv, D, dt, page_size, layout, seed)


def _operands(q, k, v, qk_quant_gran="per_thread", pv_accum_dtype="fp32+fp16", smooth_k=True, smooth_v=False):
    """The library's quantised operands of one sequence (the dense quantisers, whose bits the paged ones give): (q8, k8, v8, qs,
    ks, vs, vm), HND on the CPU, v8 logical [1,Hkv,Lk,D]."""
    from sageattention_b200.core import _quant_qk
    from sageattention_b200.quant import per_channel_fp8
    _, q8, qs, k8, ks, _, _, _ = _quant_qk(q[None], k[None], "fp8", "NHD", qk_quant_gran, q.size(-1) ** -0.5, smooth_k, "cuda")
    v8, vs, vm = per_channel_fp8(v[None], tensor_layout="NHD", scale_max=2.25 if pv_accum_dtype == "fp32+fp16" else 448.0,
                                 smooth_v=smooth_v and pv_accum_dtype == "fp32")
    return (q8.transpose(1, 2).cpu(), k8.transpose(1, 2).cpu(), v8[..., :k.size(0)].transpose(-1, -2).cpu(), qs.cpu(), ks.cpu(),
            vs.cpu(), None if vm is None else vm.cpu())


def _check(lens_q, lens_k, Hq, Hkv, D, dt, page_size, layout, causal, seed=0, **kw):
    import sageattention_b200 as sab
    q, kc, vc, table, used = _inputs(lens_q, lens_k, Hq, Hkv, D, dt, page_size, layout, seed)
    cu_q = _cu(lens_q)
    o, lse = sab.sageattn_varlen_kvcache(q, kc, vc, cu_q, used, table, max(max(lens_q), 1), is_causal=causal, return_lse=True, **kw)
    assert torch.isfinite(o).all(), "NaN from a cache slot the call must not read"
    assert not o.requires_grad
    kp, vp = gather_pages(kc, table, used), gather_pages(vc, table, used)
    assert torch.isfinite(kp).all() and torch.isfinite(vp).all()
    cu_k = _cu(lens_k)
    if not causal:
        op, lp = sab.sageattn_varlen_qk_int8_pv_fp8_cuda(q, kp, vp, cu_q, cu_k, max(max(lens_q), 1), max(max(lens_k), 1),
                                                         return_lse=True, **kw)
        assert torch.equal(o, op) and torch.equal(lse, lp), "non-causal: the packed call's bits"
        return o, lse
    spans_q, spans_k = cu_q.tolist(), cu_k.tolist()
    for b, (lq, lk) in enumerate(zip(lens_q, lens_k)):
        s, e, sk, ek = spans_q[b], spans_q[b + 1], spans_k[b], spans_k[b + 1]
        if lq == 0:
            continue
        none = max(0, lq - lk)                                  # rows that see no key
        assert not o[s:s + none].any() and torch.isneginf(lse[:, s:s + none]).all(), f"rows of sequence {b} with no visible key"
        if lk == 0:
            continue
        if lk >= lq:
            od, ld = sab.sageattn_window(q[s:e][None], kp[sk:ek][None], vp[sk:ek][None], (-1, lk - lq), tensor_layout="NHD",
                                         is_causal=False, return_lse=True, **kw)
            assert torch.equal(o[s:e], od[0]), f"output rows of sequence {b} (Lq {lq}, Lk {lk})"
            bound = _lse_bound(q, kp, s, e, sk, ek, ld[0], **kw)
            assert ((lse[:, s:e] - ld[0]).abs() <= bound).all(), f"lse rows of sequence {b}"
        else:
            # no dense call has a negative right side: the restatement with its per-element bound
            _, rl, bd = attn_sequence(q[s:e].cpu(), kp[sk:ek].cpu(), vp[sk:ek].cpu(), True, bound=True,
                                      operands=_operands(q[s:e], kp[sk:ek], vp[sk:ek], **kw), **kw)
            check_elementwise(f"sequence {b} (Lq {lq}, Lk {lk})", o[s:e].transpose(0, 1)[None].cpu(), bd.o, bd.o_bound)
            assert (lse[:, s + none:e].cpu() - rl[:, none:]).abs().max() < 1e-2, f"lse rows of sequence {b}"
    return o, lse


CASES = [  # gran, pv_accum_dtype, smooth_v, smooth_k, Hq, Hkv, D, dtype, page_size, layout
    ("per_thread", "fp32+fp16", False, True, 8, 2, 128, BF, 16, "shuffled"),
    ("per_warp", "fp32+fp16", False, True, 4, 4, 64, FP, 1, "shuffled"),
    ("per_thread", "fp32", True, True, 8, 2, 64, BF, 64, "shared"),
    ("per_warp", "fp32+fp32", False, False, 8, 2, 128, FP, 96, "strided"),
    ("per_thread", "fp32+fp32", False, False, 4, 1, 128, FP, 16, "padded"),
    ("per_warp", "fp32", True, True, 8, 8, 128, BF, 16, "shared"),
    ("per_thread", "fp32+fp16", False, True, 4, 2, 64, FP, 96, "padded"),
    ("per_warp", "fp32+fp16", False, True, 8, 2, 128, BF, 64, "strided"),
]


@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("case", CASES, ids=lambda c: "-".join(str(x).replace("torch.", "") for x in c))
def test_contract_bits(case, causal):
    gran, acc, smooth_v, smooth_k, Hq, Hkv, D, dt, page_size, layout = case
    _check(LENS_Q, LENS_K, Hq, Hkv, D, dt, page_size, layout, causal, seed=Hq + D + page_size, qk_quant_gran=gran,
           pv_accum_dtype=acc, smooth_v=smooth_v, smooth_k=smooth_k)


def test_single_sequences_and_equal_lengths():
    """Lq = 1 (decode-sized), Lk = Lq (the causal call is top-left and bottom-right at once), and one sequence per call."""
    import sageattention_b200 as sab
    for lq, lk in ((1, 1), (1, 513), (128, 128), (64, 64), (129, 4000)):
        _check([lq], [lk], 8, 2, 128, BF, 16, "shuffled", True, seed=lq + lk)
    q, kc, vc, table, used = _inputs([192], [192], 8, 2, 128, BF, 16, "shuffled", 7)
    kp, vp = gather_pages(kc, table, used), gather_pages(vc, table, used)
    o = sab.sageattn_varlen_kvcache(q, kc, vc, _cu([192]), used, table, 192, is_causal=True)
    assert torch.equal(o, sab.sageattn_qk_int8_pv_fp8_cuda(q[None], kp[None], vp[None], tensor_layout="NHD", is_causal=True)[0])


def test_paged_quantisers_are_the_packed_ones_on_the_gathered_tensor():
    from sageattention_b200 import quant as Q
    for D, dt, page_size, layout in ((128, BF, 16, "shuffled"), (64, FP, 1, "shared"), (128, FP, 96, "strided"),
                                     (64, BF, 64, "padded")):
        _, kc, vc, table, used = _inputs([1], LENS_K, 2, 2, D, dt, page_size, layout, seed=D + page_size)
        lk = LENS_K
        cu_k, mk = _cu(lk), max(lk)
        kp, vp = gather_pages(kc, table, used), gather_pages(vc, table, used)
        km = Q.k_mean_paged(kc, cu_k, table, mk)
        assert torch.equal(km, Q.k_mean_varlen(kp, cu_k, mk))
        blocks, t_pad = sum((n + 63) // 64 for n in lk), sum((n + 127) // 128 * 128 for n in lk)
        for gran, mult in (("per_thread", 4), ("per_warp", 1)):
            for mean in (km, None):
                k8, ks, cks = Q.quant_k_int8_paged(kc, mean, cu_k, table, mk, sum(lk), blocks, gran)
                k8r, ksr, cksr = Q.quant_k_int8_varlen(kp, mean, cu_k, mk, gran)
                assert torch.equal(k8, k8r) and torch.equal(cks, cksr)
                assert torch.equal(ks, ksr[:blocks * mult])
        for scale_max, smooth_v in ((448.0, False), (2.25, False), (448.0, True)):
            v8, vs, vm, cp = Q.per_channel_fp8_paged(vc, cu_k, table, mk, t_pad, scale_max, smooth_v)
            v8r, vsr, vmr, cpr = Q.per_channel_fp8_varlen_seq(vp, cu_k, mk, scale_max, smooth_v)
            assert torch.equal(cp, cpr) and torch.equal(vs, vsr) and (vm is None or torch.equal(vm, vmr))
            assert torch.equal(v8.view(torch.uint8), v8r[..., :t_pad].view(torch.uint8))


def test_no_sequence_with_keys_and_rows_past_the_end():
    import sageattention_b200 as sab
    q, kc, vc, table, used = _inputs([5, 3], [0, 0], 4, 2, 64, FP, 16, "shuffled", 3)
    o, lse = sab.sageattn_varlen_kvcache(q, kc, vc, _cu([5, 3]), used, table, 5, is_causal=True, return_lse=True)
    assert not o.any() and torch.isneginf(lse).all()
    # rows past cu_seqlens_q[-1] are not written
    q, kc, vc, table, used = _inputs([70, 10], [100, 10], 4, 2, 64, FP, 16, "shuffled", 4)
    q2 = torch.cat([q, torch.randn(9, 4, 64, device="cuda", dtype=FP)])
    o_ref = sab.sageattn_varlen_kvcache(q, kc, vc, _cu([70, 10]), used, table, 70, is_causal=True)
    o2 = sab.sageattn_varlen_kvcache(q2, kc, vc, _cu([70, 10]), used, table, 70, is_causal=True)
    assert torch.equal(o2[:80], o_ref)


def test_seqused_out_of_range_raises():
    import sageattention_b200 as sab
    q, kc, vc, table, used = _inputs([5, 3], [20, 10], 4, 2, 64, FP, 16, "shuffled", 5)
    with pytest.raises(ValueError):
        sab.sageattn_varlen_kvcache(q, kc, vc, _cu([5, 3]), torch.tensor([20, table.size(1) * 16 + 1], dtype=torch.int32,
                                                                          device="cuda"), table, 5)


def test_bench_workloads_give_the_gather_routes_bits():
    """bench_kvcache.py's chunked-prefill and prefix-caching shapes, shortened to one sequence each, against the gather route."""
    import bench_kvcache as B
    for w in (B.Workload("chunked", [2048], [2048 + 2048], 0), B.Workload("prefix", [1024, 1024], [8192 + 1024] * 2, 8192)):
        q, kc, vc, table, cu, used = B.make_inputs(w)
        fns = B.routes(w, q, kc, vc, table, cu, used)
        assert torch.equal(fns["kvcache"](), fns["gather"]())
        ref = fns["sdpa"]()
        assert (fns["kvcache"]().float() - ref.float()).abs().max() < 0.1
