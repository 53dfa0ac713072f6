"""GPU tests of the 8-bit paged KV cache at the inputs serving engines pass it, for sageattn_kvcache8 and sageattn_kvcache8_prefill,
each causal, causal with the window (100, -1) and non-causal with the window (7, 5), against the restatements
(tests/attn_kvcache8_oracle.py, attn_kvcache8_prefill_oracle.py, attn_kvcache8_window_oracle.py) element by element within their
bounds, o and lse, rows that see nothing exactly 0 and -inf:
  1. GQA ratios 3, 5, 7 and 64 ((6, 2), (12, 4), (5, 1), (28, 4), (64, 1)), D 64 / 128, fp16 / bf16, decode row counts
     R = Lq_b * G of 63 and 64 and ones that are not a multiple of 16 (49, 35, 21); prefill at (128, 1), beyond the decode limit;
  2. strided inputs give the bits of contiguous ones: q sliced from a fused QKV tensor, q with a padded head stride, cache.write
     from K / V slices of the fused tensor (the stored pages and scales), a column slice of a wider block table, int64
     cu_seqlens_q;
  3. max_seqlen_q below a sequence's length: the rows written (the first max_seqlen_q) are those of the whole sequence, whose
     length comes from cu_seqlens_q; rows past max_seqlen_q and past cu_seqlens_q[-1] keep the canary the C ABI's output and lse
     were filled with;
  4. long contexts: decode against 131072 keys (128 chunks; with left = 4096, 124 of them write empty partials), prefill of 200
     rows against 65536 keys, pages of 1024 and 2048 keys, and seqused_k above the table's capacity, which gives the bits of
     seqused_k at the capacity;
  5. value distributions of real models: a common K offset of 50 (k_smooth the mean), an attention-sink token, V tokens from 1e-3
     to 1e3, fp16 tokens near 6e4, and sm_scale 1.0 / 0.02 / 0.3; the error against fp64 attention on the 16-bit tokens is
     printed;
  6. quantiser edges, bit for bit in the write kernel (int8 and e4m3 ties, products that round above qmax, amax around and below
     qmax / FLT_MAX, k = 0 with a denormal k_smooth) and, as Q rows, in both Q prologues against the restatement."""
import math

import pytest
import torch

from attn_kvcache8_oracle import attend, write
from attn_kvcache8_prefill_oracle import attend_folded
from attn_kvcache8_window_oracle import attend as attend_w, attend_folded as attend_folded_w, visible_keys

pytestmark = pytest.mark.gpu
DEV = "cuda"
MODES = [(True, (-1, -1)), (True, (100, -1)), (False, (7, 5))]      # (is_causal, window_size)
FLT_MAX = torch.finfo(torch.float32).max


def _chunk():
    from sageattention_b200 import ops
    return ops.kvcache8_chunk_keys()


def _tokens(n, Hkv, D, dt, g, offset=1.0):
    k = (torch.randn(n, Hkv, D, generator=g) + offset * torch.randn(1, Hkv, D, generator=g)).to(dt)
    v = torch.randn(n, Hkv, D, generator=g).to(dt)
    return k, v


def _cache(toks, ksm, page_size, seed, extra_pages=2, table_extra=0):
    """A PagedKVCache8 holding each sequence's (k, v) tokens in shuffled pages, written in one call, and its block table."""
    import sageattention_b200 as sab
    g = torch.Generator().manual_seed(seed)
    Hkv, D = ksm.shape
    dt = toks[0][0].dtype
    pages = [max(1, (k.size(0) + page_size - 1) // page_size) for k, _ in toks]
    num_pages = sum(pages) + extra_pages
    perm = torch.randperm(num_pages, generator=g)
    table = torch.zeros(len(pages), max(pages) + table_extra, dtype=torch.int32)
    nxt = 0
    for b, p in enumerate(pages):
        table[b, :p] = perm[nxt:nxt + p]
        nxt += p
    cache = sab.PagedKVCache8(num_pages, page_size, Hkv, D, dt, device=DEV, k_smooth=ksm)
    slots = [table[b][torch.arange(k.size(0)) // page_size].long() * page_size + torch.arange(k.size(0)) % page_size
             for b, (k, _) in enumerate(toks)]
    if sum(k.size(0) for k, _ in toks):
        cache.write(torch.cat([k for k, _ in toks]).to(DEV), torch.cat([v for _, v in toks]).to(DEV), torch.cat(slots).to(DEV))
    return cache, table.to(DEV)


def _cu(lens_q, dtype=torch.int32):
    return torch.tensor([0] + torch.cumsum(torch.tensor(lens_q), 0).tolist(), dtype=dtype, device=DEV)


def _call(prefill, q, cache, lens_q, lens_k, table, causal, window, msq=None, sm_scale=None, cu=None):
    import sageattention_b200 as sab
    fn = sab.sageattn_kvcache8_prefill if prefill else sab.sageattn_kvcache8
    cu = _cu(lens_q) if cu is None else cu
    used = torch.tensor(lens_k, dtype=torch.int32, device=DEV)
    msq = max(max(lens_q), 1) if msq is None else msq
    return fn(q.to(DEV), cache, cu, used, table, msq, is_causal=causal, sm_scale=sm_scale, return_lse=True, window_size=window)


def _restate(prefill, q_b, k_b, v_b, ksm, causal, window, sm_scale, dt):
    """The restatement of one sequence with its bound: (o, lse, o_bound, lse_bound)."""
    k8, ks, v8, vs = write(k_b, v_b, ksm)
    args = (q_b, k8, ks, v8, vs, ksm, causal, sm_scale)
    if window == (-1, -1):
        return attend_folded(*args, bound=True, out_dtype=dt) if prefill else attend(*args, _chunk(), bound=True, out_dtype=dt)
    if prefill:
        return attend_folded_w(*args, bound=True, out_dtype=dt, window=window)
    return attend_w(*args, _chunk(), bound=True, out_dtype=dt, window=window)


def _compare(o_b, lse_b, ref, what):
    """o_b [Lq, Hq, D] and lse_b [Hq, Lq] of one sequence against the restatement, element by element; returns max err / bound."""
    oe, le, ob, lb = ref
    o_b, lse_b = o_b.cpu().double(), lse_b.cpu().double()
    none = torch.isneginf(le)
    assert torch.equal(torch.isneginf(lse_b), none), what
    assert not o_b.transpose(0, 1)[none].any(), what
    err = (o_b - oe).abs()
    assert (err <= ob).all(), (what, (err / ob).nan_to_num(0.0).max().item())
    assert ((lse_b - le).abs()[~none] <= lb[~none]).all(), (what, (lse_b - le).abs()[~none].max().item())
    return (err / ob.clamp_min(1e-30)).max().item() if err.numel() else 0.0


def _check(prefill, q, toks, ksm, cache, table, lens_q, causal, window, sm_scale=None, what=()):
    lens_k = [k.size(0) for k, _ in toks]
    o, lse = _call(prefill, q, cache, lens_q, lens_k, table, causal, window, sm_scale=sm_scale)
    o, lse = o.cpu(), lse.cpu()
    scale = q.size(-1) ** -0.5 if sm_scale is None else sm_scale
    s = 0
    for b, Lq in enumerate(lens_q):
        ref = _restate(prefill, q[s:s + Lq], toks[b][0], toks[b][1], ksm, causal, window, scale, q.dtype)
        _compare(o[s:s + Lq], lse[:, s:s + Lq], ref, (*what, prefill, causal, window, b))
        s += Lq
    return o, lse


# ------------------------------------------------------------------------------------------------ 1. GQA ratios
GQA = [(6, 2), (12, 4), (28, 4), (5, 1), (64, 1)]
CFGS = [(torch.bfloat16, 128), (torch.float16, 64), (torch.float16, 128), (torch.bfloat16, 64)]


@pytest.mark.parametrize("prefill", [False, True])
@pytest.mark.parametrize("cfg", range(len(CFGS)))
@pytest.mark.parametrize("Hq,Hkv", GQA)
def test_gqa_ratios(Hq, Hkv, cfg, prefill):
    dt, D = CFGS[cfg]
    G = Hq // Hkv
    seed = Hq * 100 + Hkv * 10 + cfg
    g = torch.Generator().manual_seed(seed)
    if prefill:
        lens_q, lens_k = [1, 130, 37, 200], [300, 1100, 0, 150]
    else:
        lim = 64 // G                           # rows R = Lq * G: 63 (G 3, 7), 64 (G 64), 60 / 35 (G 5), 49 (G 7), 21 (G 3)
        lens_q, lens_k = [lim, min(7, lim), 1, max(1, lim - 1)], [1100, 2085, 63, 0]
    toks = [_tokens(n, Hkv, D, dt, g) for n in lens_k]
    allk = torch.cat([k for k, _ in toks])
    ksm = allk.float().mean(0)
    cache, table = _cache(toks, ksm, 16 if D == 128 else 32, seed)
    q = torch.randn(sum(lens_q), Hq, D, generator=g).to(dt)
    for causal, window in MODES:
        _check(prefill, q, toks, ksm, cache, table, lens_q, causal, window, what=(Hq, Hkv, dt, D))


@pytest.mark.parametrize("cfg", range(len(CFGS)))
def test_prefill_at_gqa_128_beyond_the_decode_row_limit(cfg):
    import sageattention_b200 as sab
    dt, D = CFGS[cfg]
    g = torch.Generator().manual_seed(128 + cfg)
    lens_q, lens_k = [1, 70, 2], [300, 1100, 0]
    toks = [_tokens(n, 1, D, dt, g) for n in lens_k]
    ksm = torch.cat([k for k, _ in toks]).float().mean(0)
    cache, table = _cache(toks, ksm, 16, cfg)
    q = torch.randn(sum(lens_q), 128, D, generator=g).to(dt)
    for causal, window in MODES:
        _check(True, q, toks, ksm, cache, table, lens_q, causal, window, what=(dt, D))
    with pytest.raises(ValueError, match="sageattn_kvcache8_prefill"):
        _call(False, q[:1], cache, [1], [300], table[:1], True, (-1, -1))


# ------------------------------------------------------------------------------------------------ 2. strided inputs
@pytest.mark.parametrize("prefill", [False, True])
def test_strided_q_table_views_and_int64_offsets_give_the_contiguous_bits(prefill):
    import sageattention_b200 as sab
    Hq, Hkv, D, dt, ps = 28, 4, 128, torch.bfloat16, 16
    g = torch.Generator().manual_seed(2)
    lens_q = [40, 1, 129] if prefill else [9, 1, 4]
    lens_k = [1500, 77, 2100]
    T = sum(lens_q)
    qkv = torch.randn(T, Hq + 2 * Hkv, D, generator=g).to(dt).to(DEV)
    q_fused = qkv[:, :Hq]
    padded = torch.randn(T, Hq, 2, D, generator=g).to(dt).to(DEV)
    padded[:, :, 0] = q_fused
    q_padded = padded[:, :, 0]                                           # head stride 2D
    assert q_fused.stride() == ((Hq + 2 * Hkv) * D, D, 1) and q_padded.stride() == (2 * Hq * D, 2 * D, 1)
    q = q_fused.contiguous()
    toks = [_tokens(n, Hkv, D, dt, g) for n in lens_k]
    ksm = torch.cat([k for k, _ in toks]).float().mean(0)
    cache, table = _cache(toks, ksm, ps, 3, table_extra=5)
    wide = torch.full((3, table.size(1) + 37), 0, dtype=torch.int32, device=DEV)
    wide[:, 3:3 + table.size(1)] = table
    view = wide[:, 3:3 + table.size(1)]
    assert view.stride(0) > view.size(1) and view.stride(1) == 1
    used = torch.tensor(lens_k, dtype=torch.int32, device=DEV)
    fn = sab.sageattn_kvcache8_prefill if prefill else sab.sageattn_kvcache8
    for causal, window in MODES:
        args = dict(is_causal=causal, return_lse=True, window_size=window)
        ref = fn(q, cache, _cu(lens_q), used, table, max(lens_q), **args)
        for name, qq, tt, cu in (("fused q", q_fused, table, _cu(lens_q)), ("padded q", q_padded, table, _cu(lens_q)),
                                 ("table view", q, view, _cu(lens_q)), ("int64 cu", q, table, _cu(lens_q, torch.int64))):
            got = fn(qq, cache, cu, used, tt, max(lens_q), **args)
            assert torch.equal(got[0], ref[0]) and torch.equal(got[1], ref[1]), (name, causal, window)
        _check(prefill, q.cpu(), toks, ksm, cache, table, lens_q, causal, window)


@pytest.mark.parametrize("dt,D", [(torch.bfloat16, 128), (torch.float16, 64)])
def test_write_from_fused_qkv_slices_stores_the_contiguous_bits(dt, D):
    import sageattention_b200 as sab
    Hq, Hkv, T, ps = 12, 4, 100, 16
    g = torch.Generator().manual_seed(D)
    qkv = (torch.randn(T, Hq + 2 * Hkv, D, generator=g) * 2 + 1).to(dt).to(DEV)
    k, v = qkv[:, Hq:Hq + Hkv], qkv[:, Hq + Hkv:]
    assert k.stride() == v.stride() == ((Hq + 2 * Hkv) * D, D, 1)
    ksm = k.float().mean(0)
    slots = torch.randperm(8 * ps, generator=g)[:T].to(DEV)
    caches = []
    for kk, vv in ((k, v), (k.contiguous(), v.contiguous())):
        c = sab.PagedKVCache8(8, ps, Hkv, D, dt, device=DEV, k_smooth=ksm)
        c.write(kk, vv, slots)
        caches.append(c)
    a, b = caches
    for x, y, what in ((a.k_pages, b.k_pages, "k_pages"), (a.k_scale, b.k_scale, "k_scale"),
                       (a.v_pages.view(torch.uint8), b.v_pages.view(torch.uint8), "v_pages"), (a.v_scale, b.v_scale, "v_scale")):
        assert torch.equal(x, y), what
    k8, ks, v8, vs = write(k.cpu(), v.cpu(), ksm.cpu())
    flat = lambda t: t.reshape(8 * ps, *t.shape[2:]).cpu()[slots.cpu()]
    assert torch.equal(flat(caches[0].k_pages).float(), k8) and torch.equal(flat(caches[0].k_scale), ks)
    assert torch.equal(flat(caches[0].v_pages).float(), v8) and torch.equal(flat(caches[0].v_scale), vs)


# ------------------------------------------------------------------------------------------------ 3. max_seqlen_q < Lq_b
CANARY_O, CANARY_LSE = -640.0, 12345.0           # exact in fp16, bf16 and fp32


def _capi_call(prefill, q, cache, cu, used, table, msq, causal, window, out, lse):
    """The C ABI (sab_kvcache8_attn / _prefill and their _window forms) writing into the given out and lse."""
    from sageattention_b200 import _capi, ops
    lib = _capi.lib()
    Tq, Hq, D = q.shape
    nseq, max_pages = table.shape
    ps, Hkv = cache.page_size, cache.num_kv_heads
    args = [q.data_ptr(), ops._dt(q), cache.k_pages.data_ptr(), cache.k_scale.data_ptr(), cache.v_pages.data_ptr(),
            cache.v_scale.data_ptr(), cache.k_smooth.data_ptr(), out.data_ptr(), lse.data_ptr(), cu.data_ptr(), used.data_ptr(),
            table.data_ptr(), table.stride(0), max_pages, nseq, Tq, Hq, Hkv, D, ps, q.stride(0), q.stride(1), out.stride(0),
            out.stride(1), msq, 1 if causal else 0, D ** -0.5]
    if not prefill:
        ws = torch.empty(lib.sab_kvcache8_workspace_bytes(Tq, Hq, D, max_pages * ps), dtype=torch.uint8, device=DEV)
        args.append(ws.data_ptr())
    fn = ("sab_kvcache8_prefill" if prefill else "sab_kvcache8_attn") + ("" if window == (-1, -1) else "_window")
    win = [] if window == (-1, -1) else list(window)
    _capi.check(getattr(lib, fn)(*args, *win, torch.cuda.current_stream().cuda_stream))


@pytest.mark.parametrize("prefill", [False, True])
@pytest.mark.parametrize("mode", range(len(MODES)))
def test_rows_written_under_a_short_max_seqlen_q_see_what_the_whole_sequence_sees(prefill, mode):
    """Sequences longer than max_seqlen_q: the first max_seqlen_q rows are written, each with the causal and window bounds of the
    whole sequence (j <= i + Lk_b - Lq_b, Lq_b from cu_seqlens_q), and every other row keeps its canary."""
    causal, window = MODES[mode]
    Hq, Hkv, D, dt = 8, 2, 128, torch.bfloat16
    if prefill:
        msq, lens_q, lens_k = 130, [300, 50, 300], [1000, 200, 200]
    else:
        msq, lens_q, lens_k = 4, [9, 16, 3], [500, 12, 2000]
    g = torch.Generator().manual_seed(31 + mode)
    toks = [_tokens(n, Hkv, D, dt, g) for n in lens_k]
    ksm = torch.cat([k for k, _ in toks]).float().mean(0)
    cache, table = _cache(toks, ksm, 16, 5)
    Tq = sum(lens_q) + 5                                          # rows past cu_seqlens_q[-1]
    q = torch.randn(Tq, Hq, D, generator=g).to(dt)
    out = torch.full((Tq, Hq, D), CANARY_O, dtype=dt, device=DEV)
    lse = torch.full((Hq, Tq), CANARY_LSE, dtype=torch.float32, device=DEV)
    _capi_call(prefill, q.to(DEV), cache, _cu(lens_q), torch.tensor(lens_k, dtype=torch.int32, device=DEV), table, msq, causal,
               window, out, lse)
    out, lse = out.cpu(), lse.cpu()
    written = torch.zeros(Tq, dtype=torch.bool)
    s = 0
    for b, (Lq, Lk) in enumerate(zip(lens_q, lens_k)):
        n = min(Lq, msq)
        oe, le, ob, lb = _restate(prefill, q[s:s + Lq], toks[b][0], toks[b][1], ksm, causal, window, D ** -0.5, dt)
        _compare(out[s:s + n], lse[:, s:s + n], (oe[:n], le[:, :n], ob[:n], lb[:, :n]), (prefill, causal, window, b))
        written[s:s + n] = True
        s += Lq
    assert (out[~written] == CANARY_O).all(), (~written).nonzero().flatten()[(out[~written] != CANARY_O).any(-1).any(-1)].tolist()
    assert (lse[:, ~written] == CANARY_LSE).all()


# ------------------------------------------------------------------------------------------------ 4. long contexts
@pytest.mark.parametrize("mode", range(len(MODES)))
def test_decode_against_131072_keys(mode):
    causal, window = MODES[mode]
    if window == (100, -1):
        window = (4096, -1)                                       # 124 of the 128 chunks lie left of the window
    Hq, Hkv, D, dt, n = 8, 2, 128, torch.bfloat16, 131072
    g = torch.Generator(device=DEV).manual_seed(131072 + mode)
    k = (torch.randn(n, Hkv, D, generator=g, device=DEV) + torch.randn(1, Hkv, D, generator=g, device=DEV)).to(dt)
    v = torch.randn(n, Hkv, D, generator=g, device=DEV).to(dt)
    ksm = k.float().mean(0)
    toks = [(k.cpu(), v.cpu())]
    cache, table = _cache(toks, ksm.cpu(), 16, 7)
    q = torch.randn(4, Hq, D, generator=g, device=DEV).to(dt).cpu()
    for lq in (1, 4):
        _check(False, q[:lq], toks, ksm.cpu(), cache, table, [lq], causal, window, what=(n, lq))


@pytest.mark.parametrize("mode", range(len(MODES)))
def test_prefill_of_200_rows_against_65536_keys(mode):
    causal, window = MODES[mode]
    Hq, Hkv, D, dt, n = 4, 1, 128, torch.bfloat16, 65536
    g = torch.Generator().manual_seed(65536 + mode)
    toks = [_tokens(n, Hkv, D, dt, g)]
    ksm = toks[0][0].float().mean(0)
    cache, table = _cache(toks, ksm, 16, 8)
    q = torch.randn(200, Hq, D, generator=g).to(dt)
    _check(True, q, toks, ksm, cache, table, [200], causal, window)


@pytest.mark.parametrize("page_size", [1024, 2048])
@pytest.mark.parametrize("prefill", [False, True])
def test_pages_that_span_whole_chunks(page_size, prefill):
    Hq, Hkv, D, dt = 8, 2, 64, torch.float16
    g = torch.Generator().manual_seed(page_size + prefill)
    lens_k = [5000, 1023, 2049, 4096]
    lens_q = [150, 3, 64, 1] if prefill else [16, 3, 16, 1]
    toks = [_tokens(n, Hkv, D, dt, g) for n in lens_k]
    ksm = torch.cat([k for k, _ in toks]).float().mean(0)
    cache, table = _cache(toks, ksm, page_size, 9)
    q = torch.randn(sum(lens_q), Hq, D, generator=g).to(dt)
    for causal, window in MODES:
        _check(prefill, q, toks, ksm, cache, table, lens_q, causal, window, what=(page_size,))


@pytest.mark.parametrize("prefill", [False, True])
def test_seqused_k_above_the_capacity_gives_the_bits_at_the_capacity(prefill):
    Hq, Hkv, D, dt, ps = 8, 2, 128, torch.bfloat16, 16
    g = torch.Generator().manual_seed(40 + prefill)
    lens_k = [1100, 300, 2048]
    lens_q = [100, 7, 130] if prefill else [8, 1, 5]
    toks = [_tokens(n, Hkv, D, dt, g) for n in lens_k]
    ksm = torch.cat([k for k, _ in toks]).float().mean(0)
    cache, table = _cache(toks, ksm, ps, 10)                    # table width: 128 pages = 2048 keys
    cap = table.size(1) * ps
    assert cap == 2048
    q = torch.randn(sum(lens_q), Hq, D, generator=g).to(dt)
    for causal, window in MODES:
        # every sequence at the capacity (table entries past a sequence's own pages name page 0, a valid page) against
        # seqused_k past it
        ref = _call(prefill, q, cache, lens_q, [cap] * 3, table, causal, window)
        for over in (cap + 1, cap + 1000, 2 ** 31 - 1):
            got = _call(prefill, q, cache, lens_q, [over] * 3, table, causal, window)
            assert torch.equal(got[0], ref[0]) and torch.equal(got[1], ref[1]), (over, causal, window)


# ------------------------------------------------------------------------------------------------ 5. value distributions
def _fp64(q, k, v, causal, window, sm_scale):
    Lq, Hq, D = q.shape
    Lk = k.size(0)
    G = Hq // k.size(1)
    kh = k.double().repeat_interleave(G, 1).transpose(0, 1)
    vh = v.double().repeat_interleave(G, 1).transpose(0, 1)
    s = (q.double().transpose(0, 1) @ kh.transpose(1, 2)) * sm_scale
    first, last = visible_keys(Lq, Lk, causal, window)
    j = torch.arange(Lk)[None, :]
    s = s.masked_fill(~((j <= last) & (j >= first)), -math.inf)
    return (torch.softmax(s, -1).nan_to_num(0.0) @ vh).transpose(0, 1)


def _distribution(name, n, Hkv, D, g):
    """(k, v, q scale) of n tokens."""
    if name == "offset50":
        k = (50.0 + 0.3 * torch.randn(n, Hkv, D, generator=g)).bfloat16()
        return k, torch.randn(n, Hkv, D, generator=g).bfloat16(), 1.0
    if name == "sink":
        k = torch.randn(n, Hkv, D, generator=g)
        k[0] *= 20.0
        return k.bfloat16(), torch.randn(n, Hkv, D, generator=g).bfloat16(), 1.0
    if name == "v_range":
        mag = 10.0 ** (torch.rand(n, Hkv, 1, generator=g) * 6 - 3)              # per-token scales differ by up to 2^20
        return torch.randn(n, Hkv, D, generator=g).bfloat16(), (torch.randn(n, Hkv, D, generator=g) * mag).bfloat16(), 1.0
    if name == "fp16_6e4":
        big = lambda: (torch.randn(n, Hkv, D, generator=g).clamp(-3, 3) * 2.1e4).half()   # |x| up to 6.3e4
        return big(), big(), 1e-4
    raise ValueError(name)


@pytest.mark.parametrize("prefill", [False, True])
@pytest.mark.parametrize("name", ["offset50", "sink", "v_range", "fp16_6e4"])
def test_value_distributions_of_real_models(name, prefill):
    Hq, Hkv, D = 8, 2, 128
    g = torch.Generator().manual_seed(len(name) + prefill)
    lens_k = [1500, 300]
    lens_q = [130, 20] if prefill else [8, 3]
    toks = [_distribution(name, n, Hkv, D, g) for n in lens_k]
    qs = toks[0][2]
    toks = [(k, v) for k, v, _ in toks]
    dt = toks[0][0].dtype
    ksm = torch.cat([k for k, _ in toks]).float().mean(0)
    cache, table = _cache(toks, ksm, 16, 12)
    q = (torch.randn(sum(lens_q), Hq, D, generator=g) * qs).to(dt)
    for causal, window in MODES:
        o, _ = _check(prefill, q, toks, ksm, cache, table, lens_q, causal, window, what=(name,))
        s, errs = 0, []
        for b, Lq in enumerate(lens_q):
            ref = _fp64(q[s:s + Lq], *toks[b], causal, window, D ** -0.5)
            errs.append(((o[s:s + Lq].double() - ref).abs() / toks[b][1].double().abs().max()).flatten())
            s += Lq
        e = torch.cat(errs)
        print(f"{name} prefill={prefill} causal={causal} window={window}: error / max|v| against fp64 max {e.max().item():.2e} "
              f"mean {e.mean().item():.2e}")


@pytest.mark.parametrize("prefill", [False, True])
@pytest.mark.parametrize("sm_scale", [1.0, 0.02, 0.3])
def test_sm_scales(sm_scale, prefill):
    Hq, Hkv, D, dt = 8, 2, 64, torch.float16
    g = torch.Generator().manual_seed(int(sm_scale * 1000) + prefill)
    lens_k = [1200, 70]
    lens_q = [100, 5] if prefill else [8, 5]
    toks = [_tokens(n, Hkv, D, dt, g) for n in lens_k]
    ksm = torch.cat([k for k, _ in toks]).float().mean(0)
    cache, table = _cache(toks, ksm, 32, 13)
    q = torch.randn(sum(lens_q), Hq, D, generator=g).to(dt)
    for causal, window in MODES:
        o, _ = _check(prefill, q, toks, ksm, cache, table, lens_q, causal, window, sm_scale=sm_scale)
        ref = _fp64(q[:lens_q[0]], *toks[0], causal, window, sm_scale)
        print(f"sm_scale={sm_scale} prefill={prefill} causal={causal} window={window}: max error against fp64 "
              f"{(o[:lens_q[0]].double() - ref).abs().max().item():.4f}")


# ------------------------------------------------------------------------------------------------ 6. quantiser edges
def _edge_rows(dt, D):
    """Rows [n, D] (fp32 values exactly representable in dt) at the quantisers' edges, and what each is for."""
    u = 2.0 ** -9
    rows, names = [], []

    def add(name, vals, exact=True):
        r = torch.zeros(D)
        r[:len(vals)] = torch.tensor(vals, dtype=torch.float64).float()
        if exact:
            assert torch.equal(r.to(dt).float(), r), name
        r = r.to(dt).float()
        assert len(vals) == 0 or r.abs().max().item() == max(abs(x) for x in vals), name    # rounding kept the amax
        rows.append(r)
        names.append(name)
    add("int8 ties", [0.5, -0.5, 1.5, -1.5, 2.5, -2.5, 126.5, -126.5, 3.5, 127.0])
    add("e4m3 ties", [448.0, 17.0, 19.0, -17.0, 1.5 * u, 2.5 * u, 0.5 * u, -1.5 * u, 232.0])
    add("zero", [])
    top = 0x7C00 if dt == torch.float16 else 0x7F80
    a = torch.arange(1, top, dtype=torch.int32).to(torch.int16).view(dt).float()
    for qmax in (127.0, 448.0):
        mult = torch.tensor(qmax) / a
        over = a[torch.isfinite(mult) & (a * mult > qmax)]
        for x in over[torch.linspace(0, over.numel() - 1, 3).long()].tolist():
            add(f"above {qmax:.0f}", [x, -x, x / 2, x / 3], exact=False)
        if dt == torch.bfloat16:
            inf = torch.isinf(mult)
            for x in (a[inf].max().item(), a[~inf].min().item(), a[inf].min().item()):   # either side of qmax / FLT_MAX, smallest
                add(f"threshold {qmax:.0f}", [x, -x / 2, x / 7], exact=False)
    if dt == torch.bfloat16:
        add("2^-126", [2.0 ** -126, -(2.0 ** -127), 0.75 * 2.0 ** -126])
    return torch.stack(rows), names


@pytest.mark.parametrize("dt,D", [(torch.bfloat16, 128), (torch.bfloat16, 64), (torch.float16, 128), (torch.float16, 64)])
def test_write_kernel_at_the_quantiser_edges(dt, D):
    import sageattention_b200 as sab
    rows, names = _edge_rows(dt, D)
    n = rows.size(0)
    Hkv = 3
    g = torch.Generator().manual_seed(D)
    # head 0: the edge rows with k_smooth 0; head 1: k = 0 against a k_smooth in the fp32 denormal range; head 2: the edge rows
    # as V and random K
    k = torch.randn(n, Hkv, D, generator=g)
    v = torch.randn(n, Hkv, D, generator=g)
    k[:, 0], v[:, 0] = rows, rows.flip(0)
    k[:, 1] = 0.0
    v[:, 2] = rows
    k, v = k.to(dt), v.to(dt)
    ksm = torch.randn(Hkv, D, generator=g)
    ksm[0] = 0.0
    ksm[1] = torch.randn(D, generator=g) * 2.0 ** -140
    ksm[1, 0] = 3.0 * 2.0 ** -140
    assert (ksm[1].abs() < 2.0 ** -126).all()
    ps = 16
    cache = sab.PagedKVCache8((n + ps - 1) // ps + 1, ps, Hkv, D, dt, device=DEV, k_smooth=ksm)
    slots = torch.randperm(cache.num_pages * ps, generator=g)[:n]
    cache.write(k.to(DEV), v.to(DEV), slots.to(DEV))
    k8, ks, v8, vs = write(k, v, ksm)
    flat = lambda t: t.reshape(cache.num_pages * ps, *t.shape[2:]).cpu()[slots]
    for got, want, what in ((flat(cache.k_pages).float(), k8, "k8"), (flat(cache.k_scale), ks, "k_scale"),
                            (flat(cache.v_pages).float(), v8, "v8"), (flat(cache.v_scale), vs, "v_scale")):
        bad = (got != want).reshape(n, -1).any(-1)
        assert not bad.any(), (what, [names[i] for i in bad.nonzero().flatten().tolist()])
    # anchors worked out by hand (tests/test_kvcache8_edges_cpu.py derives them)
    i = names.index("int8 ties")
    assert k8[i, 0, :10].tolist() == [0.0, 0.0, 2.0, -2.0, 2.0, -2.0, 126.0, -126.0, 4.0, 127.0]
    j = names.index("e4m3 ties")
    assert v8[j, 2, :9].tolist() == [448.0, 16.0, 20.0, -16.0, 2 * 2.0 ** -9, 2 * 2.0 ** -9, 0.0, -2 * 2.0 ** -9, 224.0]
    assert ks[names.index("zero"), 0] == 0 and not k8[names.index("zero"), 0].any()
    for m, name in enumerate(names):
        if name.startswith("above"):
            qmax = float(name.split()[1])
            assert (k8 if qmax == 127.0 else v8)[m, 0 if qmax == 127.0 else 2, :2].tolist() == [qmax, -qmax], name


@pytest.mark.parametrize("prefill", [False, True])
@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
def test_q_prologues_at_the_quantiser_edges(dt, prefill):
    """The edge rows as Q rows (one per Q head and token), against the restatement.  Rows with an amax near FLT_MAX are left out:
    their logits q . k * sm_scale exceed the fp32 range themselves."""
    D, Hkv = 128, 2
    rows, names = _edge_rows(dt, D)
    rows = rows[rows.abs().amax(-1) <= 2.0 ** 16]
    Hq = 8
    n = (rows.size(0) + Hq - 1) // Hq
    g = torch.Generator().manual_seed(6 + prefill)
    q = torch.randn(n * Hq, D, generator=g)
    q[:rows.size(0)] = rows
    q = q.view(n, Hq, D).to(dt)
    lens_k = [700, 1500]
    lens_q = [n, n]
    toks = [_tokens(m, Hkv, D, dt, g) for m in lens_k]
    ksm = torch.cat([k for k, _ in toks]).float().mean(0)
    cache, table = _cache(toks, ksm, 16, 14)
    q2 = torch.cat([q, q.flip(1)])
    for causal, window in MODES:
        _check(prefill, q2, toks, ksm, cache, table, lens_q, causal, window, what=(dt,))
