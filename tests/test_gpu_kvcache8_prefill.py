"""GPU tests of sageattn_kvcache8_prefill (chunked prefill against the 8-bit paged KV cache) against its restatement
(tests/attn_kvcache8_prefill_oracle.attend_folded: the decode restatement with one chunk, its bound scaled to a row's steps):
  1. element by element within the restatement's bound: fp16 / bf16, D 64 / 128, GQA 1 / 4 / 8, causal or not, page_size 16 / 48
     / 256, Lq in {1, 63, 64, 65, 127, 128, 129, 300} against Lk in {0, 1, 63, 64, 65, Lq - 3, Lq, Lq + 1000, 2085}, an empty query
     sequence, and one row of 16 K keys; lse too, and rows that see nothing give exact zeros and -inf;
  2. exact bits: a sequence alone and in a batch; relocated pages, a wider table and NaN / garbage in every unreferenced slot and
     page; shared prefix pages; return_lse=False; chunked prefill in chunks of 5000, 2048 and 777 tokens;
  3. a CUDA graph of write + prefill replayed with q, the slot mapping and seqused_k advanced in place gives the eager bits;
  4. accuracy at the benchmark's chunked-prefill shapes against fp64 attention on the 16-bit K / V, next to
     sageattn_varlen_kvcache."""
import math

import pytest
import torch

from attn_kvcache8_oracle import write
from attn_kvcache8_prefill_oracle import attend_folded

pytestmark = pytest.mark.gpu
DEV = "cuda"
LQS = (1, 63, 64, 65, 127, 128, 129, 300)


def _lks(lq):
    return (0, 1, 63, 64, 65, max(lq - 3, 0), lq, lq + 1000, 2 * 1024 + 37)


def _build(lens_k, Hkv, D, dt, page_size, seed, extra_pages=3, shared_prefix_pages=0, g=None):
    """A PagedKVCache8 holding lens_k tokens per sequence in shuffled pages (one write), the 16-bit tokens per sequence, the
    block table and k_smooth (the mean key).  shared_prefix_pages: every sequence's first pages are sequence 0's."""
    import sageattention_b200 as sab
    g = g or torch.Generator().manual_seed(seed)
    pages = [max(1, (n + page_size - 1) // page_size) for n in lens_k]
    npre = shared_prefix_pages
    num_pages = sum(pages) - npre * (len(pages) - 1) + extra_pages
    perm = torch.randperm(num_pages, generator=g)
    table = torch.zeros(len(pages), max(pages), dtype=torch.int32)
    nxt = 0
    for b, p in enumerate(pages):
        for j in range(p):
            if b > 0 and j < npre:
                table[b, j] = table[0, j]
            else:
                table[b, j] = perm[nxt]
                nxt += 1
    toks = []
    for b, n in enumerate(lens_k):
        k = (torch.randn(n, Hkv, D, generator=g) + torch.randn(1, Hkv, D, generator=g)).to(dt)
        v = torch.randn(n, Hkv, D, generator=g).to(dt)
        if b > 0 and npre:
            m = min(n, npre * page_size)
            k[:m], v[:m] = toks[0][0][:m], toks[0][1][:m]
        toks.append((k, v))
    allk = torch.cat([t[0] for t in toks]) if sum(lens_k) else torch.zeros(1, Hkv, D, dtype=dt)
    ksm = allk.float().mean(0)
    cache = sab.PagedKVCache8(num_pages, page_size, Hkv, D, dt, device=DEV, k_smooth=ksm)
    slots = [table[b][torch.arange(n) // page_size].long() * page_size + torch.arange(n) % page_size for b, n in enumerate(lens_k)]
    if sum(lens_k):
        cache.write(torch.cat([t[0] for t in toks]).to(DEV), torch.cat([t[1] for t in toks]).to(DEV), torch.cat(slots).to(DEV))
    return cache, toks, table.to(DEV), ksm


def _call(q, cache, lens_q, lens_k, table, max_seqlen_q, causal=True, return_lse=True):
    import sageattention_b200 as sab
    cu = torch.tensor([0] + torch.cumsum(torch.tensor(lens_q), 0).tolist(), dtype=torch.int32, device=DEV)
    used = torch.tensor(lens_k, dtype=torch.int32, device=DEV)
    return sab.sageattn_kvcache8_prefill(q.to(DEV), cache, cu, used, table, max_seqlen_q, is_causal=causal, return_lse=return_lse)


# ------------------------------------------------------------------------------------------------ 1. against the restatement
def _check(lens_q, lens_k, Hq, Hkv, D, dt, page_size, causal, seed):
    cache, toks, table, ksm = _build(lens_k, Hkv, D, dt, page_size, seed)
    g = torch.Generator().manual_seed(seed + 1)
    q = torch.randn(sum(lens_q), Hq, D, generator=g).to(dt)
    o, lse = _call(q, cache, lens_q, lens_k, table, max(max(lens_q), 1), causal)
    o, lse = o.cpu(), lse.cpu()
    s = 0
    for b, (Lq, Lk) in enumerate(zip(lens_q, lens_k)):
        k8, ks, v8, vs = write(toks[b][0], toks[b][1], ksm)
        oe, le, ob, lb = attend_folded(q[s:s + Lq], k8, ks, v8, vs, ksm, causal, D ** -0.5, bound=True, out_dtype=dt)
        ok, lk_ = o[s:s + Lq].double(), lse[:, s:s + Lq].double()
        none = torch.isneginf(le)
        assert torch.equal(torch.isneginf(lk_), none), (b, Lq, Lk)
        assert not ok.transpose(0, 1)[none].any(), (b, Lq, Lk)                 # exact zeros
        err = (ok - oe).abs()
        assert (err <= ob).all(), (b, Lq, Lk, (err / ob).nan_to_num(0.0).max().item())
        assert ((lk_ - le).abs()[~none] <= lb[~none]).all(), (b, Lq, Lk)
        s += Lq


_CONFIGS = [(dt, D, causal) for dt in (torch.bfloat16, torch.float16) for D in (128, 64) for causal in (True, False)]


@pytest.mark.parametrize("i", range(len(_CONFIGS)))
def test_against_the_restatement(i):
    dt, D, causal = _CONFIGS[i]
    Hq, Hkv = ((2, 2), (8, 2), (8, 1))[i % 3]                 # GQA 1, 4, 8
    page_size = (16, 48, 256)[i % 3]
    lens_q, lens_k = [], []
    for lq in LQS:
        for lk in _lks(lq):
            lens_q.append(lq)
            lens_k.append(lk)
    lens_q.append(0)                                          # an empty query sequence
    lens_k.append(100)
    _check(lens_q, lens_k, Hq, Hkv, D, dt, page_size, causal, seed=10 + i)


def test_one_long_row():
    """16 K keys in one row: the restatement's accumulation term for a whole row."""
    _check([65, 1], [16384 + 5, 16384 + 64], 4, 1, 128, torch.bfloat16, 16, True, seed=3)


# ------------------------------------------------------------------------------------------------ 2. exact bits
def test_a_sequence_alone_equals_it_in_a_batch_and_the_table_does_not_matter():
    import sageattention_b200 as sab
    lens_k, lens_q = [1100, 5, 3000, 900], [300, 1, 129, 64]
    cache, toks, table, ksm = _build(lens_k, 2, 128, torch.bfloat16, 16, 11)
    q = torch.randn(sum(lens_q), 8, 128).bfloat16()
    o, lse = _call(q, cache, lens_q, lens_k, table, 300)
    o2 = _call(q, cache, lens_q, lens_k, table, 300, return_lse=False)
    assert torch.equal(o, o2)
    s = 0
    for b, (Lq, Lk) in enumerate(zip(lens_q, lens_k)):
        ob, lb = _call(q[s:s + Lq], cache, [Lq], [Lk], table[b:b + 1], Lq)
        assert torch.equal(ob, o[s:s + Lq]) and torch.equal(lb, lse[:, s:s + Lq]), b
        s += Lq
    n = cache.num_pages
    perm = torch.randperm(n, generator=torch.Generator().manual_seed(1)).to(DEV)
    moved = sab.PagedKVCache8(n + 5, 16, 2, 128, torch.bfloat16, device=DEV, k_smooth=ksm)
    for src, dst in ((cache.k_pages, moved.k_pages), (cache.v_pages.view(torch.uint8), moved.v_pages.view(torch.uint8)),
                     (cache.k_scale, moved.k_scale), (cache.v_scale, moved.v_scale)):
        dst[perm] = src
    wide = torch.full((table.size(0), table.size(1) + 40), 2 ** 30, dtype=torch.int32, device=DEV)   # garbage past each row
    wide[:, :table.size(1)] = perm.int()[table.long()]
    for b, Lk in enumerate(lens_k):
        wide[b, (Lk + 15) // 16:] = -7
    o2, l2 = _call(q, moved, lens_q, lens_k, wide, 300)
    assert torch.equal(o2, o) and torch.equal(l2, lse)
    used = torch.zeros(n + 5, 16, dtype=torch.bool, device=DEV)
    for b, Lk in enumerate(lens_k):
        t = torch.arange(Lk, device=DEV)
        used[wide[b][t // 16].long(), t % 16] = True
    moved.v_pages.view(torch.uint8)[~used] = 0x7F          # e4m3 NaN
    moved.k_scale[~used] = float("nan")
    moved.v_scale[~used] = float("nan")
    moved.k_pages[~used] = 127
    o3, l3 = _call(q, moved, lens_q, lens_k, wide, 300)
    assert torch.equal(o3, o) and torch.equal(l3, lse)


def test_shared_prefix_pages_give_each_sequence_its_solo_bits():
    lens_k = [1300, 1500, 1064]
    cache, toks, table, ksm = _build(lens_k, 2, 128, torch.float16, 16, 5, shared_prefix_pages=1056 // 16)
    q = torch.randn(3 * 200, 8, 128).half()
    o, lse = _call(q, cache, [200] * 3, lens_k, table, 200)
    for b in range(3):
        ob, lb = _call(q[200 * b:200 * b + 200], cache, [200], [lens_k[b]], table[b:b + 1], 200)
        assert torch.equal(ob, o[200 * b:200 * b + 200]) and torch.equal(lb, lse[:, 200 * b:200 * b + 200])


@pytest.mark.parametrize("dt,D", [(torch.bfloat16, 128), (torch.float16, 64)])
def test_chunked_prefill_is_chunk_size_invariant(dt, D):
    """A 5000-token prompt prefilled in chunks of 5000, 2048 and 777 tokens, each chunk's K / V written first: every row the
    same bits.  A row's q8, keys, tile grid from key 0 and exact max do not depend on the chunk; a tile past a row's horizon adds
    p = 0 with alpha = 1."""
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
            o[s:e], lse[:, s:e] = _call(q[s:e], cache, [e - s], [e], table, e - s)
        outs.append((o, lse))
    for o, lse in outs[1:]:
        diff = (o != outs[0][0]).any(-1).any(-1)
        assert not diff.any(), f"rows with other bits: {diff.nonzero().flatten()[:10].tolist()}"
        assert torch.equal(lse, outs[0][1])


# ------------------------------------------------------------------------------------------------ 3. CUDA graph
def test_cuda_graph_of_write_and_prefill():
    import sageattention_b200 as sab
    ps, Hkv, Hq, D, nseq, c = 16, 2, 8, 128, 2, 256
    lens = [700, 33]
    cache, toks, table, ksm = _build(lens, Hkv, D, torch.bfloat16, ps, 9, extra_pages=0)
    # room for three chunks of c tokens per sequence: widen each sequence's pages
    extra = (3 * c + ps - 1) // ps
    big = sab.PagedKVCache8(cache.num_pages + nseq * extra, ps, Hkv, D, torch.bfloat16, device=DEV, k_smooth=ksm)
    for a, b in ((big.k_pages, cache.k_pages), (big.v_pages.view(torch.uint8), cache.v_pages.view(torch.uint8)),
                 (big.k_scale, cache.k_scale), (big.v_scale, cache.v_scale)):
        a[:cache.num_pages] = b
    tab = torch.zeros(nseq, table.size(1) + extra, dtype=torch.int32, device=DEV)
    for b, n in enumerate(lens):
        np_ = (n + ps - 1) // ps
        tab[b, :np_] = table[b, :np_]
        tab[b, np_:np_ + extra] = torch.arange(extra, dtype=torch.int32, device=DEV) + cache.num_pages + b * extra
    g = torch.Generator().manual_seed(2)
    steps = [(torch.randn(nseq * c, Hkv, D, generator=g).bfloat16(), torch.randn(nseq * c, Hkv, D, generator=g).bfloat16(),
              torch.randn(nseq * c, Hq, D, generator=g).bfloat16()) for _ in range(3)]
    cu = torch.arange(nseq + 1, dtype=torch.int32, device=DEV) * c

    def slots_for(ln):
        return torch.cat([tab[b][(n + torch.arange(c, device=DEV)) // ps].long() * ps + (n + torch.arange(c, device=DEV)) % ps
                          for b, n in enumerate(ln)])
    eager = sab.PagedKVCache8(big.num_pages, ps, Hkv, D, torch.bfloat16, device=DEV, k_smooth=ksm)
    for a, b in ((eager.k_pages, big.k_pages), (eager.v_pages.view(torch.uint8), big.v_pages.view(torch.uint8)),
                 (eager.k_scale, big.k_scale), (eager.v_scale, big.v_scale)):
        a.copy_(b)
    ref, ln = [], list(lens)
    for kn, vn, qn in steps:
        eager.write(kn.to(DEV), vn.to(DEV), slots_for(ln))
        ln = [n + c for n in ln]
        ref.append(sab.sageattn_kvcache8_prefill(qn.to(DEV), eager, cu, torch.tensor(ln, dtype=torch.int32, device=DEV), tab, c,
                                                 return_lse=True))
    k_in = torch.empty(nseq * c, Hkv, D, dtype=torch.bfloat16, device=DEV)
    v_in, q_in = torch.empty_like(k_in), torch.empty(nseq * c, Hq, D, dtype=torch.bfloat16, device=DEV)
    slot_in = torch.empty(nseq * c, dtype=torch.int64, device=DEV)
    used_in = torch.empty(nseq, dtype=torch.int32, device=DEV)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                               # warm up off the capture (first-launch attributes, allocator)
        scratch = sab.PagedKVCache8(1, ps, Hkv, D, torch.bfloat16, device=DEV)
        scratch.write(k_in, v_in, torch.full((nseq * c,), -1, dtype=torch.int64, device=DEV))
        sab.sageattn_kvcache8_prefill(q_in.zero_(), scratch, cu, torch.zeros(nseq, dtype=torch.int32, device=DEV), tab[:, :1] * 0, c)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        big.write(k_in, v_in, slot_in)
        out = sab.sageattn_kvcache8_prefill(q_in, big, cu, used_in, tab, c, return_lse=True)
    ln = list(lens)
    for i, (kn, vn, qn) in enumerate(steps):
        k_in.copy_(kn)
        v_in.copy_(vn)
        q_in.copy_(qn)
        slot_in.copy_(slots_for(ln))
        ln = [n + c for n in ln]
        used_in.copy_(torch.tensor(ln, dtype=torch.int32))
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out[0], ref[i][0]) and torch.equal(out[1], ref[i][1]), i


# ------------------------------------------------------------------------------------------------ 4. accuracy
@pytest.mark.parametrize("lk,seed", [(4096, 31), (8192, 32)])
def test_accuracy_at_the_benchmark_shapes(lk, seed):
    """A 2048-token chunk after a cached prefix (the first two sequences of bench_kvcache8_prefill.py's chunked_prefill): Hq=32,
    Hkv=8, D=128, bf16, page_size 16, causal, k_smooth the mean key; error against fp64 attention on the 16-bit K / V over Q heads
    0, 9, 18, 27.  Bounds: 1.5x the restatement's error at these shapes on the CPU (ACCURACY below).  sageattn_varlen_kvcache on
    the same data is printed, not bounded."""
    import sageattention_b200 as sab
    bmax, bmean = ACCURACY[lk]
    lq, ps = 2048, 16
    g = torch.Generator().manual_seed(seed)
    k = (torch.randn(lk, 8, 128, generator=g) + torch.randn(1, 8, 128, generator=g)).bfloat16()
    v = torch.randn(lk, 8, 128, generator=g).bfloat16()
    q = torch.randn(lq, 32, 128, generator=g).bfloat16()
    pages = lk // ps
    cache = sab.PagedKVCache8(pages, ps, 8, 128, torch.bfloat16, device=DEV, k_smooth=k.float().mean(0))
    cache.write(k.to(DEV), v.to(DEV), torch.arange(lk, device=DEV))
    table = torch.arange(pages, dtype=torch.int32, device=DEV)[None]
    o = _call(q, cache, [lq], [lk], table, lq, return_lse=False).cpu()
    cu = torch.tensor([0, lq], dtype=torch.int32, device=DEV)
    o16 = sab.sageattn_varlen_kvcache(q.to(DEV), k.view(pages, ps, 8, 128).to(DEV), v.view(pages, ps, 8, 128).to(DEV), cu,
                                      torch.tensor([lk], dtype=torch.int32, device=DEV), table, lq, is_causal=True).cpu()
    vis = torch.arange(lk)[None, :] <= torch.arange(lq)[:, None] + lk - lq
    e, e16 = [], []
    for h in (0, 9, 18, 27):
        s = q[:, h].double() @ k[:, h // 4].double().T * 128 ** -0.5
        ref = torch.softmax(s.masked_fill(~vis, -math.inf), -1) @ v[:, h // 4].double()
        e.append((o[:, h].double() - ref).abs().flatten())
        e16.append((o16[:, h].double() - ref).abs().flatten())
    e, e16 = torch.cat(e), torch.cat(e16)
    print(f"lk={lk}: kvcache8_prefill max {e.max().item():.4f} mean {e.mean().item():.5f} | "
          f"varlen_kvcache max {e16.max().item():.4f} mean {e16.mean().item():.5f}")
    assert e.max() < 1.5 * bmax and e.mean() < 1.5 * bmean


# the restatement's max / mean error against fp64 at these shapes and seeds, computed on the CPU (one chunk)
ACCURACY = {4096: (0.00923, 0.000656), 8192: (0.00369, 0.000428)}
