"""GPU tests of shared-prefix decoding on the 8-bit paged KV cache (shared_prefix_len on sageattn_kvcache8):
  1. exact bits against the same call with shared_prefix_len=0: fp16 / bf16, D 64 / 128, GQA 1 / 4 / 8, page_size 16 / 48, causal
     and not, max_seqlen_q 1, 3 and the row limit, shared_prefix_len 0, C - 1, C, C + 1, 3C + 17 and past some Lk_b, Lk_b at
     every threshold of the sharing rule, batches of S - 1, S, S + 1 and 2S + 3 sequences (S sequences per shared CTA), with
     sequences of Lq_b = 0 and Lk_b = 0;
  2. a shared chunk is read through table row 0 only: the entries of rows b >= 1 for the chunks they share point at a valid
     poison page, with the same bits;
  3. a sequence alone gives the bits it has in the batch;
  4. a CUDA graph of cache.write + the shared call, replayed with seqused_k and the slot mapping advanced in place, gives the
     eager bits while sequences start taking a new shared chunk;
  5. one check against tests/attn_kvcache8_oracle.attend, within its bound, at the benchmark's parallel_sampling shape."""
import pytest
import torch

from attn_kvcache8_oracle import attend, write

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROWS = 64           # query rows one CTA holds per KV head


def _chunk():
    from sageattention_b200 import ops
    return ops.kvcache8_chunk_keys()


def _build(lens_k, Hkv, D, dt, ps, prefix_keys, seed, extra_pages=1):
    """A PagedKVCache8 in which every sequence's keys j < prefix_keys are one set of prefix tokens held in shared pages (every
    table row names them), and later keys are the sequence's own tokens in its own shuffled pages.  Returns the cache, the
    16-bit keys / values of each sequence (CPU), the block table and k_smooth; the last extra_pages pages are in no table."""
    import sageattention_b200 as sab
    g = torch.Generator().manual_seed(seed)
    npre = (prefix_keys + ps - 1) // ps
    own = [max(0, (n - npre * ps + ps - 1) // ps) for n in lens_k]
    num_pages = npre + sum(own) + extra_pages
    perm = torch.randperm(num_pages - extra_pages, generator=g).int()
    table = torch.zeros(len(lens_k), npre + max(own), dtype=torch.int32)
    table[:, :npre] = perm[:npre]
    nxt = npre
    for b, p in enumerate(own):
        table[b, npre:npre + p] = perm[nxt:nxt + p]
        nxt += p
    longest = max(max(lens_k), npre * ps)
    pk = torch.randn(npre * ps, Hkv, D, generator=g) + torch.randn(1, Hkv, D, generator=g)
    pv = torch.randn(npre * ps, Hkv, D, generator=g)
    toks, ks, vs, slots = [], [], [], []
    for b, n in enumerate(lens_k):
        m = max(0, n - npre * ps)
        k = torch.cat([pk, torch.randn(m, Hkv, D, generator=g) + pk[:1]]).to(dt)[:n]
        v = torch.cat([pv, torch.randn(m, Hkv, D, generator=g)]).to(dt)[:n]
        toks.append((k, v))
        t = torch.arange(npre * ps, max(n, npre * ps))
        ks.append(k[npre * ps:])
        vs.append(v[npre * ps:])
        slots.append(table[b][t // ps].long() * ps + t % ps)
    t = torch.arange(npre * ps)
    ks.append(pk.to(dt))
    vs.append(pv.to(dt))
    slots.append(table[0][t // ps].long() * ps + t % ps)
    k_smooth = pk.to(dt).float().mean(0)
    cache = sab.PagedKVCache8(num_pages, ps, Hkv, D, dt, device=DEV, k_smooth=k_smooth)
    cache.write(torch.cat(ks).to(DEV), torch.cat(vs).to(DEV), torch.cat(slots).to(DEV))
    assert longest <= table.size(1) * ps
    return cache, toks, table.to(DEV), k_smooth


def _call(q, cache, lens_q, lens_k, table, causal, shared, max_seqlen_q=None):
    import sageattention_b200 as sab
    cu = torch.tensor([0] + torch.cumsum(torch.tensor(lens_q), 0).tolist(), dtype=torch.int32, device=DEV)
    used = torch.tensor(lens_k, dtype=torch.int32, device=DEV)
    msq = max_seqlen_q or max(max(lens_q), 1)
    return sab.sageattn_kvcache8(q, cache, cu, used, table, msq, is_causal=causal, return_lse=True, shared_prefix_len=shared)


def _taken(lq, lk, causal, chunks, C):
    """Chunks c < chunks that a shared CTA computes for a sequence (Lq_b, Lk_b): the sharing rule of the docstring."""
    if lq < 1:
        return 0
    return max(0, min(chunks, ((lk - lq + 1) if causal else lk) // C))


# ------------------------------------------------------------------------------------------------ 1. bits against the plain call
CONFIGS = [(torch.bfloat16, 128, 8, 2, 16), (torch.float16, 64, 8, 1, 48), (torch.float16, 128, 2, 2, 48),
           (torch.bfloat16, 64, 4, 4, 16)]


def _lengths(n, msq, causal, C):
    """n sequences: Lq_b cycling through 1..msq with a 0, Lk_b cycling through 0, 5, the three values around each threshold
    (c + 1) C of the sharing rule for c = 0, 1, 2, and one long sequence with own chunks past the prefix."""
    lens_q, lens_k = [], []
    for b in range(n):
        lq = 0 if b % 7 == 3 else 1 + b % msq
        kind = b % 12
        if kind == 0:
            lk = 4 * C + 300
        elif kind == 1:
            lk = 0
        elif kind == 2:
            lk = 5
        else:
            c, d = (kind - 3) // 3, (kind - 3) % 3 - 1
            lk = (c + 1) * C + d + (max(lq, 1) - 1 if causal else 0)
        lens_q.append(lq)
        lens_k.append(lk)
    return lens_q, lens_k


@pytest.mark.parametrize("msq_mode", ["1", "3", "limit"])
@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("cfg", range(len(CONFIGS)))
def test_bits_equal_the_call_without_a_shared_prefix(cfg, causal, msq_mode):
    dt, D, Hq, Hkv, ps = CONFIGS[cfg]
    C, G = _chunk(), Hq // Hkv
    msq = {"1": 1, "3": min(3, ROWS // G), "limit": ROWS // G}[msq_mode]
    S = ROWS // (G * msq)
    sizes = sorted({max(1, S - 1), S, S + 1, 2 * S + 3})
    lens_q, lens_k = _lengths(max(sizes), msq, causal, C)
    cache, toks, table, ksm = _build(lens_k, Hkv, D, dt, ps, 4 * C + 40, seed=cfg * 10 + causal)
    q = torch.randn(sum(lens_q), Hq, D, generator=torch.Generator().manual_seed(cfg)).to(dt).to(DEV)
    for n in sizes:
        nq = sum(lens_q[:n])
        args = (q[:nq], cache, lens_q[:n], lens_k[:n], table[:n])
        ref = _call(*args, causal, 0, msq)
        assert not ref[0].isnan().any()
        for shared in (C - 1, C, C + 1, 3 * C + 17, 4 * C + 500):
            got = _call(*args, causal, shared, msq)
            assert torch.equal(got[0], ref[0]) and torch.equal(got[1], ref[1]), (n, shared)


# ------------------------------------------------------------------------------------------------ 2. only table row 0 is read
@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("ps", [16, 48])
def test_shared_chunks_read_table_row_0_only(causal, ps):
    C = _chunk()
    lens_k = [3 * C + 100, 3 * C + 2, 2 * C + 3, C, 3 * C + 700, 2 * C - 1, 0, 4 * C]
    lens_q = [1, 4, 2, 1, 3, 4, 1, 0]
    cache, toks, table, ksm = _build(lens_k, 2, 128, torch.bfloat16, ps, 3 * C, seed=ps)
    q = torch.randn(sum(lens_q), 8, 128, generator=torch.Generator().manual_seed(1)).bfloat16().to(DEV)
    shared = 3 * C
    ref = _call(q, cache, lens_q, lens_k, table, causal, 0)
    poison = cache.num_pages - 1                                # in [0, num_pages), named by no table row
    assert poison not in set(table.flatten().tolist())
    cache.k_pages[poison] = 127
    cache.v_pages.view(torch.uint8)[poison] = 0x7F              # e4m3 NaN
    cache.k_scale[poison] = float("nan")
    cache.v_scale[poison] = float("nan")
    ptable = table.clone()
    poisoned = 0
    for b in range(1, len(lens_k)):
        keys = _taken(lens_q[b], lens_k[b], causal, shared // C, C) * C   # keys of b that only shared CTAs read
        ptable[b, :keys // ps] = poison
        poisoned += keys // ps
    assert poisoned > 0
    got = _call(q, cache, lens_q, lens_k, ptable, causal, shared)
    assert torch.equal(got[0], ref[0]) and torch.equal(got[1], ref[1])


# ------------------------------------------------------------------------------------------------ 3. a sequence alone
@pytest.mark.parametrize("causal", [True, False])
def test_a_sequence_alone_equals_it_in_the_batch(causal):
    C = _chunk()
    lens_k = [2 * C + 50, 2 * C + 1, C + 3, 2 * C, 0, 3 * C + 9, 2 * C + 2, 700]
    lens_q = [1, 2, 4, 1, 3, 4, 0, 2]
    cache, toks, table, ksm = _build(lens_k, 2, 128, torch.float16, 16, 2 * C + 20, seed=3)
    q = torch.randn(sum(lens_q), 8, 128, generator=torch.Generator().manual_seed(2)).half().to(DEV)
    o, lse = _call(q, cache, lens_q, lens_k, table, causal, 2 * C + 20, max_seqlen_q=4)
    s = 0
    for b, (lq, lk) in enumerate(zip(lens_q, lens_k)):
        if lq == 0:                                             # a call holds at least one query
            continue
        ob, lb = _call(q[s:s + lq], cache, [lq], [lk], table[b:b + 1].contiguous(), causal, 2 * C + 20, max_seqlen_q=4)
        assert torch.equal(ob, o[s:s + lq]) and torch.equal(lb, lse[:, s:s + lq]), b
        s += lq


# ------------------------------------------------------------------------------------------------ 4. CUDA graph
def test_cuda_graph_of_write_and_shared_decode():
    """Six sequences of Lq = 4 (speculative verification, causal) behind a 2C-key shared prefix, one new token each per step.
    Chunk 1 is shared for b once Lk_b - 3 >= 2C; the sequences start at Lk_b = 2C + b % 3 and reach it at different steps."""
    import sageattention_b200 as sab
    C, n, lq, ps, steps = _chunk(), 6, 4, 16, 6
    start = [2 * C + b % 3 for b in range(n)]
    final = [s + steps for s in start]
    cache, toks, table, ksm = _build(final, 2, 128, torch.bfloat16, ps, 2 * C, seed=9)
    slots = torch.tensor([[int(table[b, (start[b] + i) // ps]) * ps + (start[b] + i) % ps for b in range(n)] for i in range(steps)],
                         dtype=torch.int64, device=DEV)
    for t in (cache.k_pages, cache.v_pages.view(torch.uint8), cache.k_scale, cache.v_scale):   # the steps write these tokens
        t.view(-1, *t.shape[2:])[slots.flatten()] = 0
    eager = sab.PagedKVCache8(cache.num_pages, ps, 2, 128, torch.bfloat16, device=DEV, k_smooth=cache.k_smooth)
    for a, b in ((eager.k_pages, cache.k_pages), (eager.v_pages.view(torch.uint8), cache.v_pages.view(torch.uint8)),
                 (eager.k_scale, cache.k_scale), (eager.v_scale, cache.v_scale)):
        a.copy_(b)
    qs = torch.randn(steps, n * lq, 8, 128, generator=torch.Generator().manual_seed(4)).bfloat16().to(DEV)
    new_k = torch.stack([torch.stack([toks[b][0][start[b] + i] for b in range(n)]) for i in range(steps)]).to(DEV)
    new_v = torch.stack([torch.stack([toks[b][1][start[b] + i] for b in range(n)]) for i in range(steps)]).to(DEV)
    cu = torch.arange(0, n * lq + 1, lq, dtype=torch.int32, device=DEV)
    ref, took = [], []
    for i in range(steps):
        eager.write(new_k[i], new_v[i], slots[i])
        used = torch.tensor([s + i + 1 for s in start], dtype=torch.int32, device=DEV)
        ref.append(sab.sageattn_kvcache8(qs[i], eager, cu, used, table, lq, return_lse=True, shared_prefix_len=2 * C))
        plain = sab.sageattn_kvcache8(qs[i], eager, cu, used, table, lq, return_lse=True)
        assert torch.equal(ref[i][0], plain[0]) and torch.equal(ref[i][1], plain[1]), i
        took.append(sum(_taken(lq, s + i + 1, True, 2, C) for s in start))
    assert len(set(took)) > 2                                   # sequences start taking chunk 1 at different steps
    k_in = torch.zeros(n, 2, 128, dtype=torch.bfloat16, device=DEV)
    v_in = torch.zeros_like(k_in)
    q_in = torch.zeros(n * lq, 8, 128, dtype=torch.bfloat16, device=DEV)
    slot_in = torch.full((n,), -1, dtype=torch.int64, device=DEV)
    used_in = torch.tensor(start, dtype=torch.int32, device=DEV)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                               # warm up off the capture (first-launch attributes, allocator)
        cache.write(k_in, v_in, slot_in)
        sab.sageattn_kvcache8(q_in, cache, cu, used_in, table, lq, return_lse=True, shared_prefix_len=2 * C)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        cache.write(k_in, v_in, slot_in)
        out = sab.sageattn_kvcache8(q_in, cache, cu, used_in, table, lq, return_lse=True, shared_prefix_len=2 * C)
    for i in range(steps):
        k_in.copy_(new_k[i])
        v_in.copy_(new_v[i])
        q_in.copy_(qs[i])
        slot_in.copy_(slots[i])
        used_in.add_(1)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out[0], ref[i][0]) and torch.equal(out[1], ref[i][1]), i


# ------------------------------------------------------------------------------------------------ 5. against the restatement
def test_parallel_sampling_shape_against_the_restatement():
    """bench_kvcache8_shared.py's parallel_sampling setup (Hq=32, Hkv=8, D=128, bf16, page_size 16, causal, Lq = 1, an 8192-key
    shared prompt plus 64 i own keys) for four of its sequences, element by element within the restatement's bound."""
    C = _chunk()
    lens_k = [8192 + 64 * i for i in range(4)]
    cache, toks, table, ksm = _build(lens_k, 8, 128, torch.bfloat16, 16, 8192, seed=5)
    q = torch.randn(4, 32, 128, generator=torch.Generator().manual_seed(6)).bfloat16()
    o, lse = _call(q.to(DEV), cache, [1] * 4, lens_k, table, True, 8192)
    o, lse = o.cpu().double(), lse.cpu().double()
    for b in range(4):
        k8, ks, v8, vs = write(toks[b][0], toks[b][1], ksm)
        oe, le, ob, lb = attend(q[b:b + 1], k8, ks, v8, vs, ksm, True, 128 ** -0.5, C, bound=True, out_dtype=torch.bfloat16)
        assert ((o[b:b + 1] - oe).abs() <= ob).all(), b
        assert ((lse[:, b:b + 1] - le).abs() <= lb).all(), b
