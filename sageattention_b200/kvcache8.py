"""An 8-bit paged KV cache for decoding: each token is quantised once, when it is written, and attention reads the 8-bit pages.

`sageattn_varlen_kvcache` keeps a 16-bit cache because its K mean and V scales are statistics over each call's keys, so every call
reads and quantises the whole cache again.  Here the statistics belong to the token: K and V get one fp32 scale per (token, head),
and the K smoothing vector belongs to the cache.  A token written once is never touched again, and a decode step reads about 0.52x
the bytes of a bf16 cache at D = 128 with no quantiser pass and no host synchronisation, so write + attention can be captured in
a CUDA graph.  sageattn_kvcache8 serves decode-sized queries; sageattn_kvcache8_prefill serves query chunks of any length
(chunked prefill, prefix caching) from the same cache.
"""
import numbers
from typing import Optional

import torch

from . import ops
from .core import _check_window_size

_ROW_LIMIT = 64     # query rows per (sequence, KV head): max_seqlen_q * Hq / Hkv


def _check_cuda_tensor(name, t, dtype, device, shape=None):
    if not isinstance(t, torch.Tensor) or t.dtype != dtype or t.device != device:
        raise ValueError(f"{name} must be a {dtype} tensor on {device}")
    if shape is not None and tuple(t.shape) != tuple(shape):
        raise ValueError(f"{name} must have shape {tuple(shape)}, got {tuple(t.shape)}")


class PagedKVCache8:
    """A paged KV cache in 8 bits: INT8 K and e4m3 V pages with one fp32 scale per (token, head).

    k_pages int8 / v_pages float8_e4m3fn [num_pages, page_size, Hkv, D] (token-major), k_scale / v_scale fp32
    [num_pages, page_size, Hkv], k_smooth fp32 [Hkv, D].  Slot s is token s % page_size of page s // page_size.

    k_smooth is subtracted from every key before quantisation and is fixed for the cache's life (for example the mean of a
    prefill's keys, `k.float().mean(0)`; zeros by default).  Every logit of a row moves by the same q . k_smooth, so it changes the
    quantisation error and never the softmax, and one vector per cache keeps shared prefix pages valid for every sequence.
    D is 64 or 128, page_size a multiple of 16; `dtype` (fp16 / bf16) is that of the tokens written, of q and of the output."""

    def __init__(self, num_pages: int, page_size: int, num_kv_heads: int, head_dim: int, dtype: torch.dtype = torch.bfloat16,
                 device="cuda", k_smooth: Optional[torch.Tensor] = None):
        device = torch.device(device)
        if device.type != "cuda":
            raise ValueError("the cache lives on a CUDA device: there is no CPU implementation")
        if device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        if head_dim not in (64, 128):
            raise ValueError(f"head_dim must be 64 or 128, got {head_dim}")
        if page_size < 16 or page_size % 16 != 0:
            raise ValueError(f"page_size must be a positive multiple of 16, got {page_size}")
        if num_pages < 1 or num_kv_heads < 1:
            raise ValueError("the cache needs at least one page and one KV head")
        if dtype not in (torch.float16, torch.bfloat16):
            raise ValueError(f"dtype must be torch.float16 or torch.bfloat16, got {dtype}")
        shape = (num_pages, page_size, num_kv_heads, head_dim)
        self.dtype, self.device = dtype, device
        self.k_pages = torch.zeros(shape, dtype=torch.int8, device=device)
        self.v_pages = torch.zeros(shape, dtype=torch.float8_e4m3fn, device=device)
        self.k_scale = torch.zeros(shape[:3], dtype=torch.float32, device=device)
        self.v_scale = torch.zeros(shape[:3], dtype=torch.float32, device=device)
        if k_smooth is None:
            self.k_smooth = torch.zeros(num_kv_heads, head_dim, dtype=torch.float32, device=device)
        else:
            if not isinstance(k_smooth, torch.Tensor) or tuple(k_smooth.shape) != (num_kv_heads, head_dim):
                raise ValueError(f"k_smooth must be a [{num_kv_heads}, {head_dim}] tensor")
            self.k_smooth = k_smooth.to(device=device, dtype=torch.float32).contiguous().clone()

    @property
    def num_pages(self) -> int:
        return self.k_pages.size(0)

    @property
    def page_size(self) -> int:
        return self.k_pages.size(1)

    @property
    def num_kv_heads(self) -> int:
        return self.k_pages.size(2)

    @property
    def head_dim(self) -> int:
        return self.k_pages.size(3)

    @property
    def bytes_per_token(self) -> int:
        """Cache bytes one token takes: 8-bit K and V plus two fp32 scales per KV head."""
        return self.num_kv_heads * (2 * self.head_dim + 8)

    def nbytes(self) -> int:
        ts = (self.k_pages, self.v_pages, self.k_scale, self.v_scale, self.k_smooth)
        return sum(t.numel() * t.element_size() for t in ts)

    def write(self, k: torch.Tensor, v: torch.Tensor, slot_mapping: torch.Tensor) -> None:
        """Quantise and store tokens k, v [T, Hkv, D] (the cache's dtype, last dim contiguous) in place, one launch.  slot_mapping is
        int64 [T] on the device holding page * page_size + slot; -1 (any negative value) skips the token.  Per (token, head), in fp32:
        K x = k - k_smooth, k_scale = max|x| / 127, k8 = round-to-nearest-even, saturated, of x * (127 / max|x|); V v_scale =
        max|v| / 448, v8 = e4m3(v * (448 / max|v|)), round-to-nearest, saturated; an all-zero row stores scale 0 and zeros.  The bits
        stored depend on the token alone, so writing tokens one at a time or all at once is the same; unmapped slots are not
        touched.  Slots are trusted: two tokens mapped to one slot leave either."""
        Hkv, D = self.num_kv_heads, self.head_dim
        for name, t in (("k", k), ("v", v)):
            if not isinstance(t, torch.Tensor) or t.dim() != 3 or t.shape[1:] != (Hkv, D):
                raise ValueError(f"{name} must be a [T, {Hkv}, {D}] tensor")
            if t.dtype != self.dtype or t.device != self.device:
                raise ValueError(f"{name} must have the cache's dtype and device ({self.dtype}, {self.device})")
            if t.stride(-1) != 1 or t.data_ptr() % 8 != 0 or t.stride(0) % 4 != 0 or t.stride(1) % 4 != 0:
                raise ValueError(f"{name} needs stride(-1) == 1 and 8-byte aligned rows")
        if k.size(0) != v.size(0):
            raise ValueError(f"k and v must hold the same number of tokens ({k.size(0)} and {v.size(0)})")
        _check_cuda_tensor("slot_mapping", slot_mapping, torch.int64, self.device, (k.size(0),))
        if k.size(0) == 0:
            return
        ops.kvcache8_write(k, v, self.k_smooth, slot_mapping.contiguous(), self.k_pages, self.k_scale,
                           self.v_pages.view(torch.uint8), self.v_scale)


def _attn_args(q, cache, cu_seqlens_q, seqused_k, block_table, max_seqlen_q):
    """The argument checks both cache calls share; returns (Hq, D, cu_seqlens_q as int32)."""
    if not isinstance(cache, PagedKVCache8):
        raise ValueError("cache must be a PagedKVCache8")
    dev = cache.device
    if not isinstance(q, torch.Tensor) or q.dim() != 3 or q.dtype != cache.dtype or q.device != dev:
        raise ValueError(f"q must be a packed [Tq, Hq, D] tensor with the cache's dtype and device ({cache.dtype}, {dev})")
    Tq, Hq, D = q.shape
    Hkv = cache.num_kv_heads
    if D != cache.head_dim:
        raise ValueError(f"q's head dim ({D}) differs from the cache's ({cache.head_dim})")
    if Hq < 1 or Hq % Hkv != 0:
        raise ValueError(f"num_qo_heads ({Hq}) must be divisible by num_kv_heads ({Hkv})")
    if Tq < 1:
        raise ValueError("the packed batch must hold at least one query")
    if q.stride(-1) != 1 or q.data_ptr() % 8 != 0 or q.stride(0) % 4 != 0 or q.stride(1) % 4 != 0:
        raise ValueError("q needs stride(-1) == 1 and 8-byte aligned rows")
    if not isinstance(cu_seqlens_q, torch.Tensor) or cu_seqlens_q.dim() != 1 or cu_seqlens_q.dtype not in (torch.int32, torch.int64) \
            or cu_seqlens_q.numel() < 2 or cu_seqlens_q.device != dev:
        raise ValueError("cu_seqlens_q must be a 1-D int32 or int64 tensor of nseq + 1 >= 2 offsets on q's device")
    nseq = cu_seqlens_q.numel() - 1
    _check_cuda_tensor("seqused_k", seqused_k, torch.int32, dev, (nseq,))
    if not isinstance(block_table, torch.Tensor) or block_table.dim() != 2 or block_table.size(0) != nseq or block_table.size(1) < 1 \
            or block_table.dtype != torch.int32 or block_table.device != dev or block_table.stride(1) != 1:
        raise ValueError(f"block_table must be an int32 [{nseq}, max_pages] tensor on q's device with contiguous rows")
    if isinstance(max_seqlen_q, bool) or not isinstance(max_seqlen_q, numbers.Integral) or max_seqlen_q < 1:
        raise ValueError(f"max_seqlen_q must be an int >= 1, got {max_seqlen_q!r}")
    cu_q = cu_seqlens_q if cu_seqlens_q.dtype == torch.int32 else cu_seqlens_q.to(torch.int32)
    return Hq, D, cu_q


def _window_arg(window_size, block_table, cache):
    """window_size checked as sageattn_window's, each side clamped at the table's max_pages * page_size keys (no row sees more),
    so a Python int of any size reaches the C ABI as an int32."""
    left, right = _check_window_size(window_size)
    max_keys = block_table.size(1) * cache.page_size
    return min(left, max_keys), min(right, max_keys)


def sageattn_kvcache8(q: torch.Tensor, cache: PagedKVCache8, cu_seqlens_q: torch.Tensor, seqused_k: torch.Tensor,
                      block_table: torch.Tensor, max_seqlen_q: int, is_causal: bool = True, sm_scale: Optional[float] = None,
                      return_lse: bool = False, window_size=(-1, -1), shared_prefix_len: int = 0):
    """Attention of packed queries against a PagedKVCache8, for decoding and speculative verification.

    q: packed [Tq, Hq, D] in the cache's dtype with cu_seqlens_q (int32 or int64, nseq + 1 offsets) and max_seqlen_q, as in
    sageattn_varlen_kvcache; Hq % Hkv == 0.  seqused_k: int32 [nseq], Lk_b.  block_table: int32 [nseq, max_pages]; key j of
    sequence b is slot j % page_size of page block_table[b, j // page_size].  Table entries are trusted: each one read must lie in
    [0, num_pages).  Pages may be shared between sequences.  Lk_b is read on the device only and clamped to max_pages * page_size;
    the call never synchronises with the host, so cache.write + this call can be captured in a CUDA graph and replayed with
    seqused_k and the slot mapping advanced in place.

    Limits: max_seqlen_q * Hq / Hkv <= 64 (decode and speculative verification; one CTA holds every query row of a KV head), else
    ValueError: use sageattn_kvcache8_prefill for longer query chunks.  Rows of a sequence past max_seqlen_q, and rows past
    cu_seqlens_q[-1], are not written.  Forward only.

    Causal is bottom-right: query i of sequence b sees key j iff j <= i + Lk_b - Lq_b, Lq_b = cu_seqlens_q[b + 1] - cu_seqlens_q[b]
    even when it exceeds max_seqlen_q: the rows written then see what they see in the whole sequence, with and without a window.
    A row that sees no key returns 0 and lse -inf.  Numerics: Q is quantised per (token, head) to INT8 as K is (without smoothing); logits in log2 units are
    float(dot(q8, k8)) * (q_scale * sm_scale * log2e) * k_scale.  Keys are cut into fixed chunks of ops.kvcache8_chunk_keys() keys;
    within a chunk an exact running max over 64-key tiles, p = 2^(s - m), P = bf16(p * v_scale) times the e4m3 V with fp32
    accumulation; a second kernel merges a row's chunks in ascending order with no atomics.  A sequence's bits depend only on its
    own q, keys and values, not on the rest of the batch or on the table width.  return_lse also returns the [Hq, Tq] fp32 LSE in
    natural-log units of the logits q . k * sm_scale.

    window_size = (left, right), a pair of ints >= -1 (ValueError otherwise, before any launch), makes a sliding window aligned as
    the causal rule: with off_b = Lk_b - Lq_b, query i sees key j iff i + off_b - left <= j <= i + off_b + right (-1 leaves a side
    unbounded), and j <= i + off_b as well when is_causal.  Only keys j >= max(0, Lk_b - Lq_b - left) are ever loaded: their
    table entries, K / V bytes and scales are the only ones read, so the entries below that bound may name any page in
    [0, num_pages) (a shared null page, or pages reused for newer tokens).  Skipping keys left of the window changes no bit of what
    a row computes, and (-1, -1) is the call without a window.

    shared_prefix_len = P, an int >= 0 (ValueError otherwise, and together with a window, before any launch), reads a prefix
    that every sequence shares once for many sequences instead of once per sequence: parallel sampling, beam search, requests
    behind one system prompt.  P is clamped at max_pages * page_size, and only whole chunks are shared: P' = (P // C) * C with
    C = ops.kvcache8_chunk_keys(); P < C is the call without a shared prefix.  The caller promises that keys j < P' of every
    sequence are the same tokens, stored in the pages that block_table[0, :P' // page_size] names: row 0 is the only table row
    read for a shared chunk, and the promise is trusted as table entries are.  Chunk c < P' / C of sequence b is computed for
    up to 64 / (max_seqlen_q * Hq / Hkv) sequences at once when Lq_b >= 1 and (c + 1) * C <= Lk_b (causal: <= Lk_b - Lq_b + 1),
    so no row of b has a masked key in it; its other chunks run as without a shared prefix.  Which chunks are shared is decided
    on the device, so the call stays free of host synchronisation.  Where the promise holds, o and lse are bit for bit those of
    the call with shared_prefix_len=0.  A batch with several shared prefixes can be split into one call per prefix group: a
    sequence's bits do not depend on the batch."""
    Hq, D, cu_q = _attn_args(q, cache, cu_seqlens_q, seqused_k, block_table, max_seqlen_q)
    window = _window_arg(window_size, block_table, cache)
    if isinstance(shared_prefix_len, bool) or not isinstance(shared_prefix_len, numbers.Integral) or shared_prefix_len < 0:
        raise ValueError(f"shared_prefix_len must be an int >= 0, got {shared_prefix_len!r}")
    if shared_prefix_len > 0 and window != (-1, -1):
        raise ValueError("shared_prefix_len and window_size cannot be combined: use one or the other")
    shared = min(int(shared_prefix_len), block_table.size(1) * cache.page_size)
    Hkv = cache.num_kv_heads
    if max_seqlen_q * (Hq // Hkv) > _ROW_LIMIT:
        raise ValueError(f"max_seqlen_q * Hq / Hkv = {max_seqlen_q * (Hq // Hkv)} exceeds the {_ROW_LIMIT} query rows the split-KV "
                         "kernel holds per KV head; use sageattn_kvcache8_prefill for longer query chunks on this cache (or "
                         "sageattn_varlen_kvcache on a 16-bit cache)")
    if sm_scale is None:
        sm_scale = D ** -0.5
    with torch.no_grad():
        o = torch.empty(q.shape, dtype=q.dtype, device=cache.device)
        args = (q, cache.k_pages, cache.k_scale, cache.v_pages.view(torch.uint8), cache.v_scale, cache.k_smooth, o, cu_q.contiguous(),
                seqused_k.contiguous(), block_table, int(max_seqlen_q), 1 if is_causal else 0, float(sm_scale), 1 if return_lse else 0)
        if window != (-1, -1):
            lse = ops.kvcache8_attn_window(*args, *window)
        elif shared >= ops.kvcache8_chunk_keys():
            lse = ops.kvcache8_attn_shared(*args, shared)
        else:
            lse = ops.kvcache8_attn(*args)
    return (o, lse) if return_lse else o


def sageattn_kvcache8_prefill(q: torch.Tensor, cache: PagedKVCache8, cu_seqlens_q: torch.Tensor, seqused_k: torch.Tensor,
                              block_table: torch.Tensor, max_seqlen_q: int, is_causal: bool = True, sm_scale: Optional[float] = None,
                              return_lse: bool = False, window_size=(-1, -1)):
    """Attention of packed query chunks of any length against a PagedKVCache8: chunked prefill, prefix caching and long
    speculative verification on the 8-bit cache alone.

    Arguments, checks and the causal rule are those of sageattn_kvcache8, without its row limit: q packed [Tq, Hq, D] in the cache's
    dtype, cu_seqlens_q int32 or int64, seqused_k int32 [nseq] (read on the device only), block_table int32 [nseq, max_pages] with
    contiguous rows and trusted entries.  The call never synchronises with the host and allocates nothing but o (and lse), so
    cache.write + this call can be captured in a CUDA graph.  Causal is bottom-right: query i of sequence b sees key j iff
    j <= i + Lk_b - Lq_b; a row that sees no key returns 0 and lse -inf.  Rows of a sequence past max_seqlen_q, and rows past
    cu_seqlens_q[-1], are not written; the rows written take Lq_b from cu_seqlens_q, as in sageattn_kvcache8.  Forward only.

    Numerics: those of sageattn_kvcache8 without chunks.  Q is quantised per (token, head) to INT8; logits in log2 units are
    float(dot(q8, k8)) * (q_scale * sm_scale * log2e) * k_scale; one exact running max per row over 64-key tiles from key 0,
    p = 2^(s - m), P = bf16(p * v_scale) times the e4m3 V with fp32 accumulation, O / l.  A row's bits depend only on its own
    q, keys and values: not on the batch, the table width, or the size of the chunk it was prefilled in.  return_lse also returns
    the [Hq, Tq] fp32 LSE in natural-log units of the logits q . k * sm_scale.

    window_size: the sliding window of sageattn_kvcache8, with the same rule and the same promise: only keys
    j >= max(0, Lk_b - Lq_b - left) are ever loaded, and a row's bits do not change with the chunk size."""
    Hq, D, cu_q = _attn_args(q, cache, cu_seqlens_q, seqused_k, block_table, max_seqlen_q)
    window = _window_arg(window_size, block_table, cache)
    if sm_scale is None:
        sm_scale = D ** -0.5
    with torch.no_grad():
        o = torch.empty(q.shape, dtype=q.dtype, device=cache.device)
        args = (q, cache.k_pages, cache.k_scale, cache.v_pages.view(torch.uint8), cache.v_scale, cache.k_smooth, o, cu_q.contiguous(),
                seqused_k.contiguous(), block_table, int(max_seqlen_q), 1 if is_causal else 0, float(sm_scale), 1 if return_lse else 0)
        lse = ops.kvcache8_prefill(*args) if window == (-1, -1) else ops.kvcache8_prefill_window(*args, *window)
    return (o, lse) if return_lse else o
