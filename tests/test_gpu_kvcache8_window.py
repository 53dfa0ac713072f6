"""GPU tests of sliding-window attention on the 8-bit paged KV cache (window_size on sageattn_kvcache8 and
sageattn_kvcache8_prefill) against the windowed restatements (tests/attn_kvcache8_window_oracle.attend and attend_folded):
  1. element by element within the restatement's bound, o and lse: fp16 / bf16, D 64 / 128, GQA 1 / 4 / 8, page_size 16 / 48 /
     256, left in {0, 1, 63, 64, 65, 1023, 1024, 1025, 4096} causal, and non-causal with right in {-1, 0, 5, 200}; decode Lk
     0..5000 (windows across the 1024-key chunk edges), prefill Lq 1..300 against Lk 0..2085, Lk < Lq included;
  2. exact bits: a window covering every key gives the bits of the call without a window, decode and prefill, causal and not;
  3. exact bits: a sequence alone and in a wider-table batch; a 5000-token prompt prefilled with left = 1000 in chunks of 5000,
     2048 and 777 tokens;
  4. keys left of the window are never read: out-of-window table entries point at a valid poison page (K = 127, V = 448, huge
     and NaN scales) and out-of-window slots of the straddling page are poisoned, with the same bits; a window-sized ring of
     pages, overwritten by newer tokens, gives the bits of a linear table over many steps;
  5. a CUDA graph of cache.write + windowed decode on the ring, replayed with seqused_k and the slot mapping advanced in place,
     gives the eager bits;
  6. accuracy at the benchmark's shapes against fp64 attention on the bf16 window."""
import math

import pytest
import torch

from attn_kvcache8_oracle import write
from attn_kvcache8_window_oracle import attend, attend_folded

pytestmark = pytest.mark.gpu
DEV = "cuda"
LEFTS = (0, 1, 63, 64, 65, 1023, 1024, 1025, 4096)
WINDOWS = [((left, -1), True) for left in LEFTS] + [((left, right), False) for left, right in
                                                     ((100, -1), (1024, 0), (7, 5), (-1, 200))]
CONFIGS = [(torch.bfloat16, 128, 8, 2, 16), (torch.float16, 64, 8, 1, 48), (torch.bfloat16, 64, 4, 4, 256),
           (torch.float16, 128, 8, 1, 16)]


def _build(lens_k, Hkv, D, dt, page_size, seed, extra_pages=3, table_extra=0):
    """A PagedKVCache8 holding lens_k tokens per sequence in shuffled pages, the 16-bit tokens, the block table and k_smooth."""
    import sageattention_b200 as sab
    g = torch.Generator().manual_seed(seed)
    pages = [max(1, (n + page_size - 1) // page_size) for n in lens_k]
    num_pages = sum(pages) + extra_pages
    perm = torch.randperm(num_pages, generator=g)
    table = torch.zeros(len(pages), max(pages) + table_extra, dtype=torch.int32)
    nxt = 0
    for b, p in enumerate(pages):
        table[b, :p] = perm[nxt:nxt + p]
        nxt += p
    toks = [((torch.randn(n, Hkv, D, generator=g) + torch.randn(1, Hkv, D, generator=g)).to(dt),
             torch.randn(n, Hkv, D, generator=g).to(dt)) for n in lens_k]
    allk = torch.cat([t[0] for t in toks]) if sum(lens_k) else torch.zeros(1, Hkv, D, dtype=dt)
    ksm = allk.float().mean(0)
    cache = sab.PagedKVCache8(num_pages, page_size, Hkv, D, dt, device=DEV, k_smooth=ksm)
    slots = [table[b][torch.arange(n) // page_size].long() * page_size + torch.arange(n) % page_size for b, n in enumerate(lens_k)]
    if sum(lens_k):
        cache.write(torch.cat([t[0] for t in toks]).to(DEV), torch.cat([t[1] for t in toks]).to(DEV), torch.cat(slots).to(DEV))
    return cache, toks, table.to(DEV), ksm


def _call(prefill, q, cache, lens_q, lens_k, table, window, causal=True, return_lse=True):
    import sageattention_b200 as sab
    cu = torch.tensor([0] + torch.cumsum(torch.tensor(lens_q), 0).tolist(), dtype=torch.int32, device=DEV)
    used = torch.tensor(lens_k, dtype=torch.int32, device=DEV)
    fn = sab.sageattn_kvcache8_prefill if prefill else sab.sageattn_kvcache8
    return fn(q.to(DEV), cache, cu, used, table, max(max(lens_q), 1), is_causal=causal, return_lse=return_lse, window_size=window)


# ------------------------------------------------------------------------------------------------ 1. against the restatement
def _check(prefill, lens_q, lens_k, cfg, window, causal, seed):
    dt, D, Hq, Hkv, ps = cfg
    cache, toks, table, ksm = _build(lens_k, Hkv, D, dt, ps, seed)
    q = torch.randn(sum(lens_q), Hq, D, generator=torch.Generator().manual_seed(seed + 1)).to(dt)
    o, lse = _call(prefill, q, cache, lens_q, lens_k, table, window, causal)
    o, lse = o.cpu(), lse.cpu()
    s = 0
    for b, (Lq, Lk) in enumerate(zip(lens_q, lens_k)):
        k8, ks, v8, vs = write(toks[b][0], toks[b][1], ksm)
        args = (q[s:s + Lq], k8, ks, v8, vs, ksm, causal, D ** -0.5)
        if prefill:
            oe, le, ob, lb = attend_folded(*args, bound=True, out_dtype=dt, window=window)
        else:
            oe, le, ob, lb = attend(*args, 1024, bound=True, out_dtype=dt, window=window)
        ok, lk_ = o[s:s + Lq].double(), lse[:, s:s + Lq].double()
        none = torch.isneginf(le)
        assert torch.equal(torch.isneginf(lk_), none), (b, Lq, Lk)
        assert not ok.transpose(0, 1)[none].any(), (b, Lq, Lk)
        err = (ok - oe).abs()
        assert (err <= ob).all(), (b, Lq, Lk, (err / ob).nan_to_num(0.0).max().item())
        assert ((lk_ - le).abs()[~none] <= lb[~none]).all(), (b, Lq, Lk)
        s += Lq


@pytest.mark.parametrize("i", range(len(WINDOWS)))
def test_decode_against_the_restatement(i):
    window, causal = WINDOWS[i]
    cfg = CONFIGS[i % len(CONFIGS)]
    rows = 64 // (cfg[2] // cfg[3])
    lens_k = [0, 1, 63, 64, 65, 1000, 1024, 1025, 1090, 2048, 2100, 3071, 4097, 5000]
    lens_q = [1, 1, rows, 1, 2, rows, 1, 3, rows, 1, 5, 1, rows, min(rows, 7)]
    _check(False, lens_q, lens_k, cfg, window, causal, seed=100 + i)


@pytest.mark.parametrize("i", range(len(WINDOWS)))
def test_prefill_against_the_restatement(i):
    window, causal = WINDOWS[i]
    cfg = CONFIGS[(i + 1) % len(CONFIGS)]
    lens_q = [1, 63, 65, 129, 300, 300, 128, 200, 1, 0]
    lens_k = [0, 700, 1100, 100, 2085, 300, 1025, 150, 2085, 40]
    _check(True, lens_q, lens_k, cfg, window, causal, seed=200 + i)


# ------------------------------------------------------------------------------------------------ 2. a covering window
@pytest.mark.parametrize("prefill", [False, True])
@pytest.mark.parametrize("causal", [True, False])
def test_a_window_covering_every_key_gives_the_bits_without_a_window(prefill, causal):
    lens_k = [3000, 5, 1024, 2100, 0, 64]
    lens_q = [300, 1, 129, 7, 5, 64] if prefill else [16, 1, 16, 7, 5, 16]
    cache, toks, table, ksm = _build(lens_k, 2, 128, torch.bfloat16, 16, 21)
    q = torch.randn(sum(lens_q), 8, 128, generator=torch.Generator().manual_seed(3)).bfloat16()
    ref = _call(prefill, q, cache, lens_q, lens_k, table, (-1, -1), causal)
    for w in [(3000, -1), (10 ** 9, -1)] + ([(3000, 0), (5000, 7)] if causal else [(3000, 3000), (-1, 300)]):
        got = _call(prefill, q, cache, lens_q, lens_k, table, w, causal)
        assert torch.equal(got[0], ref[0]) and torch.equal(got[1], ref[1]), w


# ------------------------------------------------------------------------------------------------ 3. exact bits across layouts
@pytest.mark.parametrize("prefill", [False, True])
def test_a_sequence_alone_equals_it_in_a_batch(prefill):
    lens_k = [1100, 5, 3000, 900, 5000]
    lens_q = [300, 1, 129, 64, 2] if prefill else [16, 1, 9, 16, 2]
    cache, toks, table, ksm = _build(lens_k, 2, 128, torch.bfloat16, 16, 11, table_extra=17)
    q = torch.randn(sum(lens_q), 8, 128).bfloat16()
    for w in ((1000, 0), (64, -1)):
        o, lse = _call(prefill, q, cache, lens_q, lens_k, table, w)
        s = 0
        for b, (Lq, Lk) in enumerate(zip(lens_q, lens_k)):
            width = (Lk + 15) // 16 or 1
            ob, lb = _call(prefill, q[s:s + Lq], cache, [Lq], [Lk], table[b:b + 1, :width].contiguous(), w)
            assert torch.equal(ob, o[s:s + Lq]) and torch.equal(lb, lse[:, s:s + Lq]), (w, b)
            s += Lq


@pytest.mark.parametrize("dt,D", [(torch.bfloat16, 128), (torch.float16, 64)])
def test_chunked_prefill_with_a_window_is_chunk_size_invariant(dt, D):
    import sageattention_b200 as sab
    n, Hq, Hkv, ps = 5000, 8, 2, 16
    g = torch.Generator().manual_seed(8)
    k = (torch.randn(n, Hkv, D, generator=g) + torch.randn(1, Hkv, D, generator=g)).to(dt).to(DEV)
    v = torch.randn(n, Hkv, D, generator=g).to(dt).to(DEV)
    q = torch.randn(n, Hq, D, generator=g).to(dt).to(DEV)
    pages = (n + ps - 1) // ps
    table = torch.randperm(pages + 4, generator=g)[:pages].int().to(DEV)[None]
    slots = table[0][torch.arange(n, device=DEV) // ps].long() * ps + torch.arange(n, device=DEV) % ps
    outs = []
    for c in (5000, 2048, 777):
        cache = sab.PagedKVCache8(pages + 4, ps, Hkv, D, dt, device=DEV, k_smooth=k[:2048].float().mean(0))
        o, lse = torch.empty_like(q), torch.empty(Hq, n, device=DEV)
        for s in range(0, n, c):
            e = min(n, s + c)
            cache.write(k[s:e], v[s:e], slots[s:e])
            o[s:e], lse[:, s:e] = _call(True, q[s:e], cache, [e - s], [e], table, (1000, 0))
        outs.append((o, lse))
    for o, lse in outs[1:]:
        diff = (o != outs[0][0]).any(-1).any(-1)
        assert not diff.any(), f"rows with other bits: {diff.nonzero().flatten()[:10].tolist()}"
        assert torch.equal(lse, outs[0][1])


# ------------------------------------------------------------------------------------------------ 4. keys left of the window
@pytest.mark.parametrize("prefill", [False, True])
def test_pages_and_slots_left_of_the_window_are_never_read(prefill):
    import sageattention_b200 as sab
    ps, left = 16, 100
    lens_k = [1000, 3000, 150, 2085, 90]
    lens_q = [200, 1, 33, 7, 100] if prefill else [16, 1, 3, 7, 16]
    cache, toks, table, ksm = _build(lens_k, 2, 128, torch.bfloat16, ps, 13, extra_pages=1)
    q = torch.randn(sum(lens_q), 8, 128).bfloat16()
    ref = _call(prefill, q, cache, lens_q, lens_k, table, (left, 0))
    poison = sorted(set(range(cache.num_pages)) - set(table.flatten().tolist()))[0]   # the one page no sequence uses
    bad = sab.PagedKVCache8(cache.num_pages, ps, 2, 128, torch.bfloat16, device=DEV, k_smooth=ksm)
    for a, b in ((bad.k_pages, cache.k_pages), (bad.v_pages.view(torch.uint8), cache.v_pages.view(torch.uint8)),
                 (bad.k_scale, cache.k_scale), (bad.v_scale, cache.v_scale)):
        a.copy_(b)
    bad.k_pages[poison] = 127
    bad.v_pages.view(torch.uint8)[poison] = 0x7E                # e4m3 448
    bad.k_scale[poison] = 3.0e38
    bad.v_scale[poison] = float("nan")
    ptable = table.clone()
    for b, (Lq, Lk) in enumerate(zip(lens_q, lens_k)):
        jmin = max(0, Lk - Lq - left)                           # the first key the call may read
        ptable[b, :jmin // ps] = poison
        if jmin % ps:                                           # the straddling page: poison its slots left of the window
            page = int(table[b, jmin // ps])
            bad.k_pages[page, :jmin % ps] = 127
            bad.v_pages.view(torch.uint8)[page, :jmin % ps] = 0x7F   # e4m3 NaN
            bad.k_scale[page, :jmin % ps] = float("nan")
            bad.v_scale[page, :jmin % ps] = float("inf")
    got = _call(prefill, q, bad, lens_q, lens_k, ptable, (left, 0))
    assert torch.equal(got[0], ref[0]) and torch.equal(got[1], ref[1])


def _ring_setup(left, max_lq, ps, total, seed):
    """Tokens of one sequence, a linear cache holding them all, and a ring cache of R pages (logical page P at P % R)."""
    import sageattention_b200 as sab
    g = torch.Generator().manual_seed(seed)
    k = (torch.randn(total, 2, 128, generator=g) + torch.randn(1, 2, 128, generator=g)).bfloat16().to(DEV)
    v = torch.randn(total, 2, 128, generator=g).bfloat16().to(DEV)
    q = torch.randn(total, 8, 128, generator=g).bfloat16().to(DEV)
    ksm = k[:256].float().mean(0)
    R = (left + max_lq + ps - 1) // ps + 1
    pages = (total + ps - 1) // ps
    lin = sab.PagedKVCache8(pages, ps, 2, 128, torch.bfloat16, device=DEV, k_smooth=ksm)
    ring = sab.PagedKVCache8(R, ps, 2, 128, torch.bfloat16, device=DEV, k_smooth=ksm)
    lin_table = torch.arange(pages, dtype=torch.int32, device=DEV)[None]
    ring_table = (torch.arange(pages, dtype=torch.int32, device=DEV) % R)[None]
    ring_slots = (torch.arange(total, device=DEV) // ps % R) * ps + torch.arange(total, device=DEV) % ps
    return k, v, q, lin, ring, lin_table, ring_table, ring_slots


def test_a_window_sized_ring_of_pages_gives_the_linear_bits():
    left, step, ps, total = 100, 7, 16, 7 * 90
    k, v, q, lin, ring, lin_table, ring_table, ring_slots = _ring_setup(left, step, ps, total, 4)
    lin.write(k, v, torch.arange(total, device=DEV))
    for n in range(step, total + 1, step):
        ring.write(k[n - step:n], v[n - step:n], ring_slots[n - step:n])
        for prefill in (False, True):
            ref = _call(prefill, q[n - step:n], lin, [step], [n], lin_table, (left, 0))
            got = _call(prefill, q[n - step:n], ring, [step], [n], ring_table, (left, 0))
            assert torch.equal(got[0], ref[0]) and torch.equal(got[1], ref[1]), (n, prefill)


# ------------------------------------------------------------------------------------------------ 5. CUDA graph
def test_cuda_graph_of_write_and_windowed_decode_on_a_ring():
    import sageattention_b200 as sab
    left, step, ps, total = 200, 3, 16, 3 * 150
    k, v, q, lin, ring, lin_table, ring_table, ring_slots = _ring_setup(left, step, ps, total, 6)
    eager = sab.PagedKVCache8(ring.num_pages, ps, 2, 128, torch.bfloat16, device=DEV, k_smooth=ring.k_smooth)
    ref = []
    for n in range(step, total + 1, step):
        eager.write(k[n - step:n], v[n - step:n], ring_slots[n - step:n])
        ref.append(_call(False, q[n - step:n], eager, [step], [n], ring_table, (left, 0)))
    k_in, v_in = torch.empty(step, 2, 128, dtype=torch.bfloat16, device=DEV), torch.empty(step, 2, 128, dtype=torch.bfloat16, device=DEV)
    q_in = torch.zeros(step, 8, 128, dtype=torch.bfloat16, device=DEV)
    slot_in = torch.full((step,), -1, dtype=torch.int64, device=DEV)
    used_in = torch.zeros(1, dtype=torch.int32, device=DEV)
    cu = torch.tensor([0, step], dtype=torch.int32, device=DEV)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                               # warm up off the capture (first-launch attributes, allocator)
        ring.write(k_in, v_in, slot_in)
        sab.sageattn_kvcache8(q_in, ring, cu, used_in, ring_table, step, window_size=(left, 0))
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ring.write(k_in, v_in, slot_in)
        out = sab.sageattn_kvcache8(q_in, ring, cu, used_in, ring_table, step, return_lse=True, window_size=(left, 0))
    for i, n in enumerate(range(step, total + 1, step)):
        k_in.copy_(k[n - step:n])
        v_in.copy_(v[n - step:n])
        q_in.copy_(q[n - step:n])
        slot_in.copy_(ring_slots[n - step:n])
        used_in.fill_(n)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out[0], ref[i][0]) and torch.equal(out[1], ref[i][1]), n


# ------------------------------------------------------------------------------------------------ 6. accuracy
@pytest.mark.parametrize("prefill,lk,left", [(False, 16000, 1024), (False, 131072, 4096), (True, 8192, 1024), (True, 4096, 4096)])
def test_accuracy_at_the_benchmark_shapes(prefill, lk, left):
    """One sequence of bench_kvcache8_window.py's workloads (Hq=32, Hkv=8, D=128, bf16, page_size 16, causal, k_smooth the mean
    key): error against fp64 attention on the bf16 window over Q heads 0, 9, 18, 27.  The limits are those the 8-bit cache
    keeps without a window at these shapes (test_gpu_kvcache8_prefill.ACCURACY: max <= 0.0093, mean <= 0.00066), with margin."""
    import sageattention_b200 as sab
    lq, ps = (2048 if prefill else 1), 16
    g = torch.Generator(device=DEV).manual_seed(lk + left)
    k = (torch.randn(lk, 8, 128, generator=g, device=DEV) + torch.randn(1, 8, 128, generator=g, device=DEV)).bfloat16()
    v = torch.randn(lk, 8, 128, generator=g, device=DEV).bfloat16()
    q = torch.randn(lq, 32, 128, generator=g, device=DEV).bfloat16()
    pages = lk // ps
    cache = sab.PagedKVCache8(pages, ps, 8, 128, torch.bfloat16, device=DEV, k_smooth=k.float().mean(0))
    cache.write(k, v, torch.arange(lk, device=DEV))
    table = torch.arange(pages, dtype=torch.int32, device=DEV)[None]
    o = _call(prefill, q, cache, [lq], [lk], table, (left, 0), return_lse=False)
    start = max(0, lk - lq - left)
    i = torch.arange(lq, device=DEV)[:, None] + lk - lq
    j = torch.arange(start, lk, device=DEV)[None, :]
    vis = (j <= i) & (j >= i - left)
    e = []
    for h in (0, 9, 18, 27):
        s = q[:, h].double() @ k[start:, h // 4].double().T * 128 ** -0.5
        ref = torch.softmax(s.masked_fill(~vis, -math.inf), -1) @ v[start:, h // 4].double()
        e.append((o[:, h].double() - ref).abs().flatten().cpu())
    e = torch.cat(e)
    print(f"prefill={prefill} lk={lk} left={left}: max {e.max().item():.4f} mean {e.mean().item():.5f}")
    assert e.max() < 0.02 and e.mean() < 0.0015
