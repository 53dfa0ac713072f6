"""Sequence-parallel SageAttention over NCCL (BASELINE.json configs[4]).

One process per GPU.  Rank r holds the r-th contiguous slice of the sequence of Q, K and V
(``[B,H,S/P,D]`` / ``[B,S/P,H,D]``); the output stays sharded like Q.  The reference library has no
such code (its example delegates to xfuser, example/parallel_sageattn_cogvideo.py:39-51); the design
follows from the numerics:
  * K smoothing must use ONE mean for all keys of a row (softmax is invariant to a common shift of all
    keys, not to a per-shard shift): fp32 per-channel sums are all-reduced (B*Hkv*D floats).
  * per-channel V scales need the global |max|: all-reduce(MAX) of B*Hkv*D floats.
  * what crosses NVLink is the QUANTISED K (int8) and V (fp8) plus the K scales — half the bytes of
    bf16 K/V.  The all-gather output is consumed in place by the attention kernel (rank-major segment
    addressing in its TMA coordinates, kv_seg_len), no re-layout pass.
With S/P a multiple of 128 the per-rank quantisation blocks coincide with the single-GPU blocks, so the
gathered INT8/FP8 tensors equal the single-GPU ones whenever the all-reduced mean rounds identically.
"""
from typing import Any, Optional
import torch
import torch.distributed as dist

from . import ops
from ._capi import SAB_GRAN_PER_WARP, SAB_GRAN_PER_THREAD, SAB_SEM_CUDA
from .core import _check_inputs, _pad_head_dim, _LOG2E


# ------------------------------------------------------------------ device-agnostic collective helpers (gloo-testable)
def global_k_mean(k_sum_local: torch.Tensor, total_len: int, dtype: torch.dtype, group=None) -> torch.Tensor:
    """[B,H,D] fp32 local per-channel sums -> global mean rounded to `dtype` (k.mean semantics, core.py:773)."""
    s = k_sum_local.clone()
    dist.all_reduce(s, op=dist.ReduceOp.SUM, group=group)
    return (s / float(total_len)).to(dtype)


def global_abs_max(max_local: torch.Tensor, min_local: torch.Tensor, group=None) -> torch.Tensor:
    """per-channel max(|max|, |min|) over all ranks (fused.cu:386)."""
    a = torch.maximum(max_local.abs(), min_local.abs())
    dist.all_reduce(a, op=dist.ReduceOp.MAX, group=group)
    return a


def gather_rank_major(x: torch.Tensor, group=None) -> torch.Tensor:
    """all-gather along a new leading rank axis folded into dim 0: [n, ...] -> [P*n, ...]."""
    world = dist.get_world_size(group)
    out = torch.empty((world * x.size(0),) + tuple(x.shape[1:]), dtype=x.dtype, device=x.device)
    dist.all_gather_into_tensor(out.view(torch.uint8) if x.dtype == torch.float8_e4m3fn else out,
                                x.contiguous().view(torch.uint8) if x.dtype == torch.float8_e4m3fn else x.contiguous(),
                                group=group)
    return out


def gather_scales(scale_local: torch.Tensor, group=None) -> torch.Tensor:
    """[B,H,n] per-rank block scales -> [B,H,P*n] in global block order."""
    world = dist.get_world_size(group)
    B, H, n = scale_local.shape
    g = gather_rank_major(scale_local, group).view(world, B, H, n)
    return g.permute(1, 2, 0, 3).reshape(B, H, world * n).contiguous()


def _chunk_count(n_heads: int, want: int) -> int:
    """Number of KV-head chunks for the pipelined exchange: the divisor of n_heads closest to `want` (>= 1; e.g. 30 heads, want 4 -> 5... 3)."""
    if not want or want <= 1:
        return 1
    divs = [d for d in range(1, n_heads + 1) if n_heads % d == 0]
    return min(divs, key=lambda d: (abs(d - want), -d))


_COMM_STREAMS = {}


def _comm_stream(dev):
    key = (dev.type, dev.index)
    if key not in _COMM_STREAMS:
        _COMM_STREAMS[key] = torch.cuda.Stream(dev)
    return _COMM_STREAMS[key]


# ------------------------------------------------------------------ gather fused into the attention launch (opt-in)
def pull_schedule(world: int, rank: int, n_chunks: int):
    """Issue order of the peer copies: KV-head chunk by chunk (the attention grid runs the heads in order), within a chunk
    the own shard first and then the peers in ring order starting after this rank, so that at any time every rank pulls
    from a different peer.  Element = (chunk, source rank); the flag of that element is index chunk * world + source."""
    return [(c, (rank + step) % world) for c in range(n_chunks) for step in range(world)]


class _FusedGatherWorkspace:
    """The gathered K / V buffers the attention kernel reads, allocated as SYMMETRIC (peer-mapped) memory: rank r quantises its
    shard straight into segment r of its own buffers, where the peers read it; so the own segment needs no copy at all and every
    transfer is a peer-to-peer copy (DMA engines).  Plus the arrival flags and the call epoch.  One per (group, shapes)."""

    def __init__(self, group, dev, B, Hk, Sl, D, world, n_chunks, rank):
        import torch.distributed._symmetric_memory as symm_mem
        self.nk = B * Hk * Sl * D                       # bytes of one INT8 K shard (== one FP8 V shard)
        self.world, self.rank, self.B = world, rank, B
        self.buf = symm_mem.empty(2 * world * self.nk, dtype=torch.uint8, device=dev)
        self.hdl = symm_mem.rendezvous(self.buf, group if group is not None else dist.group.WORLD)
        self.shape_k, self.shape_v = (world * B, Hk, Sl, D), (world * B, Hk, D, Sl)
        self.k_all = self.buf[:world * self.nk].view(torch.int8).view(self.shape_k)
        self.v_all = self.buf[world * self.nk:].view(torch.float8_e4m3fn).view(self.shape_v)
        self.k_local = self.k_all[rank * B:(rank + 1) * B]
        self.v_local = self.v_all[rank * B:(rank + 1) * B]
        self.flags = torch.zeros((n_chunks * world,), dtype=torch.uint32, device=dev)   # stream_write_value32 wants a flat uint32 tensor
        self.epoch = 0

    def peer_shard(self, src):
        """Views of rank `src`'s OWN segment inside rank `src`'s buffers (peer-mapped)."""
        k = self.hdl.get_buffer(src, self.shape_k, torch.int8, 0)
        v = self.hdl.get_buffer(src, self.shape_v, torch.uint8, self.world * self.nk).view(torch.float8_e4m3fn)
        return k[src * self.B:(src + 1) * self.B], v[src * self.B:(src + 1) * self.B]


_FUSED_WS = {}


def _fused_workspace(group, dev, B, Hk, Sl, D, world, n_chunks, rank):
    key = (id(group), dev.index, B, Hk, Sl, D, world, n_chunks)
    if key not in _FUSED_WS:
        _FUSED_WS[key] = _FusedGatherWorkspace(group, dev, B, Hk, Sl, D, world, n_chunks, rank)
    return _FUSED_WS[key]


# ------------------------------------------------------------------ the SP operator
def sageattn_sp(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, tensor_layout: str = "HND", is_causal: bool = False,
                qk_quant_gran: str = "per_thread", sm_scale: Optional[float] = None, pv_accum_dtype: str = "fp32+fp16",
                smooth_k: bool = True, group=None, overlap_chunks: int = 1, fused_gather: bool = False,
                gather_chunks: int = 4, **kwargs: Any) -> torch.Tensor:
    """Sequence-parallel `sageattn_qk_int8_pv_fp8_cuda`: local shards in, local output shard out.

    fused_gather=True (non-causal; bit-identical to the collective path): the K/V exchange
    is not an NCCL collective before the attention launch but peer copies that run WHILE the one attention launch computes:
    every rank quantises its shard into a symmetric (peer-mapped) buffer, a side stream pulls the peers' shards KV-head chunk
    by chunk with the copy engines (no SMs) and raises one flag per (chunk, segment) in stream order, and the kernel's TMA
    producer waits for the flag of a segment before its first tile (csrc/attn.cu kSeg).  Same data in the same order as the
    collective path, hence the same bits out."""
    if group is None and not dist.is_initialized():
        raise RuntimeError("sageattn_sp needs an initialised torch.distributed process group (NCCL)")
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    dtype = q.dtype
    _check_inputs(q, k, v)
    assert qk_quant_gran in ["per_warp", "per_thread"]
    if pv_accum_dtype not in ("fp32", "fp32+fp32", "fp32+fp16"):
        raise ValueError(f"Unsupported pv_accum_dtype: {pv_accum_dtype}")
    lay = 0 if tensor_layout == "NHD" else 1
    q, k, v, head_dim_og = _pad_head_dim(q, k, v)
    if sm_scale is None:
        sm_scale = head_dim_og ** -0.5
    if lay == 1:
        B, Hq, Sl, D = q.shape
        Hk = k.size(1)
    else:
        B, Sl, Hq, D = q.shape
        Hk = k.size(2)
    assert Sl % 128 == 0, "per-rank sequence length must be a multiple of 128 (quantisation blocks must not straddle ranks)"
    S = Sl * world
    dev = q.device

    # 1. global K mean (tiny all-reduce)
    kmean = None
    if smooth_k:
        ksum = torch.empty((B, Hk, D), dtype=torch.float32, device=dev)
        kmax, kmin = torch.empty_like(ksum), torch.empty_like(ksum)
        ops.channel_stats(k, ksum, kmax, kmin, lay)
        kmean = global_k_mean(ksum, S, dtype, group)
    # 2. global per-channel |V| max (tiny all-reduce)
    vsum = torch.empty((B, Hk, D), dtype=torch.float32, device=dev)
    vmax, vmin = torch.empty_like(vsum), torch.empty_like(vsum)
    ops.channel_stats(v, vsum, vmax, vmin, lay)
    v_amax = global_abs_max(vmax, vmin, group)

    # 3. quantise the local shards (HND int8 buffers so the all-gather output is [P*B,H,Sl,D])
    fused = bool(fused_gather) and world > 1
    if fused:
        assert not is_causal, "fused_gather supports non-causal attention only"
        n_fc = _chunk_count(Hk, gather_chunks)
        ws = _fused_workspace(group, dev, B, Hk, Sl, D, world, n_fc, rank)
    q_int8 = torch.empty((B, Hq, Sl, D), dtype=torch.int8, device=dev)
    k_int8 = ws.k_local if fused else torch.empty((B, Hk, Sl, D), dtype=torch.int8, device=dev)
    qv = q if lay == 1 else q.transpose(1, 2)
    kv_ = k if lay == 1 else k.transpose(1, 2)
    vv = v if lay == 1 else v.transpose(1, 2)
    if qk_quant_gran == "per_warp":
        gran = SAB_GRAN_PER_WARP
        q_scale = torch.empty((B, Hq, Sl // 128 * 4), dtype=torch.float32, device=dev)
        k_scale = torch.empty((B, Hk, Sl // 64), dtype=torch.float32, device=dev)
        ops.quant_per_block_int8(qv, None, q_int8, q_scale, 32, 1, SAB_SEM_CUDA, False, 1.0)
        ops.quant_per_block_int8(kv_, kmean, k_int8, k_scale, 64, 1, SAB_SEM_CUDA, False, 1.0)
    else:
        gran = SAB_GRAN_PER_THREAD
        q_scale = torch.empty((B, Hq, Sl // 128 * 32), dtype=torch.float32, device=dev)
        k_scale = torch.empty((B, Hk, Sl // 64 * 4), dtype=torch.float32, device=dev)
        ops.quant_per_thread_int8(qv, None, q_int8, q_scale, 1, False)
        ops.quant_per_thread_int8(kv_, kmean, k_int8, k_scale, 1, True)
    scale_max = 2.25 if pv_accum_dtype == "fp32+fp16" else 448.0
    v_fp8 = ws.v_local if fused else torch.empty((B, Hk, D, Sl), dtype=torch.float8_e4m3fn, device=dev)
    v_scale = torch.empty((B, Hk, D), dtype=torch.float32, device=dev)
    ops.v_quant_with_amax(vv, v_fp8, v_amax, v_scale, 1, scale_max)

    if fused:
        from torch._C._distributed_c10d import _SymmetricMemory
        o = torch.empty((B, Hq, Sl, D), dtype=dtype, device=dev)
        ks_all = gather_scales(k_scale, group)               # tiny (B*Hk*S/64*{1,4} floats): ordinary collective, before the launch
        cur = torch.cuda.current_stream(dev)
        comm = _comm_stream(dev)
        ws.hdl.barrier(channel=0)                            # every rank's quantised shard is in segment `rank` of its buffers
        ws.epoch += 1
        hc = Hk // n_fc
        for c in range(n_fc):                                # the own segment is in place: its flags go up before the launch
            _SymmetricMemory.stream_write_value32(ws.flags, c * world + rank, ws.epoch)
        comm.wait_stream(cur)
        with torch.cuda.stream(comm):
            for c, src in pull_schedule(world, rank, n_fc):
                if src == rank:
                    continue
                pk, pv = ws.peer_shard(src)
                for b in range(B):                           # a head range of one batch entry is contiguous: one peer memcpy
                    ws.k_all[src * B + b, c * hc:(c + 1) * hc].copy_(pk[b, c * hc:(c + 1) * hc], non_blocking=True)
                    ws.v_all[src * B + b, c * hc:(c + 1) * hc].copy_(pv[b, c * hc:(c + 1) * hc], non_blocking=True)
                _SymmetricMemory.stream_write_value32(ws.flags, c * world + src, ws.epoch)
            ws.hdl.barrier(channel=1)                        # all ranks finished pulling: segment `rank` may be rewritten
        # the ONE attention launch, on the compute stream, not ordered after the copies: the kernel itself waits per segment
        ops.qk_int8_sv_f8_attn_sp(q_int8, ws.k_all, ws.v_all, o, q_scale, ks_all, v_scale, gran, gran, sm_scale, Sl,
                                  ws.flags, ws.epoch, hc)
        cur.wait_stream(comm)                                # the next call's quantisation overwrites the staging buffers
        o = o[..., :head_dim_og]
        return o if lay == 1 else o.transpose(1, 2)

    # 4+5. all-gather the quantised K / V (+ K scales) over NVLink and attend.  Heads are independent, so the work is
    #      pipelined over KV-head chunks: NCCL gathers chunk c+1 on a side stream while the attention kernel runs on
    #      chunk c (the gather of an 8-bit K/V chunk is ~5x shorter than its attention at S=32K, so all but the first
    #      gather is hidden).  Each chunk's gather output is consumed in place (rank-major segments, kv_seg_len).
    #      Each chunk is its own launch with its own tail wave, so the default is overlap_chunks=1 (one launch).
    o = torch.empty((B, Hq, Sl, D), dtype=dtype, device=dev)
    g = Hq // Hk
    n_chunks = overlap_chunks if (overlap_chunks and B == 1 and Hk % overlap_chunks == 0 and world > 1) else 1
    hc = Hk // n_chunks
    cur = torch.cuda.current_stream(dev)
    comm = _comm_stream(dev) if n_chunks > 1 else cur
    comm.wait_stream(cur)                               # quantised shards are ready
    gathered = []
    for c in range(n_chunks):
        hs = slice(c * hc, (c + 1) * hc)
        with torch.cuda.stream(comm):
            k_all = gather_rank_major(k_int8[:, hs], group)          # [P*B,hc,Sl,D]
            v_all = gather_rank_major(v_fp8[:, hs], group)           # [P*B,hc,D,Sl]
            ks_all = gather_scales(k_scale[:, hs].contiguous(), group)   # [B,hc,P*n]
            ev = torch.cuda.Event()
            ev.record(comm)
        gathered.append((k_all, v_all, ks_all, ev))
    for c, (k_all, v_all, ks_all, ev) in enumerate(gathered):
        cur.wait_event(ev)
        for t in (k_all, v_all, ks_all):
            t.record_stream(cur)
        qs_ = slice(c * hc * g, (c + 1) * hc * g)
        ops.qk_int8_sv_f8_attn(q_int8[:, qs_], k_all, v_all, o[:, qs_], q_scale[:, qs_].contiguous(), ks_all,
                               v_scale[:, c * hc:(c + 1) * hc].contiguous(), None, 1, 1 if is_causal else 0, gran, gran,
                               sm_scale, 0, 0, rank * Sl, Sl)
    o = o[..., :head_dim_og]
    return o if lay == 1 else o.transpose(1, 2)


# ------------------------------------------------------------------ Ulysses (head-parallel) variant
def _seq_to_head_shard(x: torch.Tensor, world: int, group=None) -> torch.Tensor:
    """[B,H,S/P,D] on every rank (sequence-sharded) -> [B,H/P,S,D] (head-sharded): one all_to_all."""
    B, H, Sl, D = x.shape
    send = x.reshape(B, world, H // world, Sl, D).permute(1, 0, 2, 3, 4).contiguous()     # [P(dst rank = head group),B,H/P,Sl,D]
    recv = torch.empty_like(send)                                                        # [P(src rank = sequence slice),...]
    dist.all_to_all_single(recv, send, group=group)
    return recv.permute(1, 2, 0, 3, 4).reshape(B, H // world, world * Sl, D)


def _head_to_seq_shard(x: torch.Tensor, world: int, group=None) -> torch.Tensor:
    """inverse of _seq_to_head_shard: [B,H/P,S,D] -> [B,H,S/P,D]."""
    B, Hl, S, D = x.shape
    Sl = S // world
    send = x.reshape(B, Hl, world, Sl, D).permute(2, 0, 1, 3, 4).contiguous()             # [P(dst rank = sequence slice),B,H/P,Sl,D]
    recv = torch.empty_like(send)                                                        # [P(src rank = head group),...]
    dist.all_to_all_single(recv, send, group=group)
    return recv.permute(1, 0, 2, 3, 4).reshape(B, world * Hl, Sl, D)


def sageattn_ulysses(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, tensor_layout: str = "HND", is_causal: bool = False,
                     sm_scale: Optional[float] = None, group=None, attn_fn=None, **kwargs: Any) -> torch.Tensor:
    """Ulysses sequence parallelism around `sageattn` (what the reference's example delegates to xfuser,
    example/parallel_sageattn_cogvideo.py:32-51): every rank holds a sequence slice of ALL heads; an all_to_all turns that
    into the FULL sequence of H/P heads, the unmodified single-GPU `sageattn` runs on those heads, a second all_to_all
    restores the sequence sharding of the output.  No numerics change at all (K mean, V scales and block scales are per
    head), so each head's result is bit-identical to the single-GPU call.  Needs Hq % P == 0 and Hkv % P == 0; use
    `sageattn_sp` (KV all-gather of 8-bit tensors) otherwise — it also moves half the bytes.
    attn_fn: the local attention callable (default: sageattn_qk_int8_pv_fp8_cuda, the operator behind sageattn); the gloo tests
    inject a CPU stand-in."""
    if not dist.is_initialized():
        raise RuntimeError("sageattn_ulysses needs an initialised torch.distributed process group")
    world = dist.get_world_size(group)
    if tensor_layout not in ("HND", "NHD"):
        raise ValueError(f"Unknown tensor layout: {tensor_layout}")
    if attn_fn is None:
        from .core import sageattn_qk_int8_pv_fp8_cuda as attn_fn     # what sageattn dispatches to; honours qk_quant_gran etc.
    hnd = tensor_layout == "HND"
    qh, kh, vh = (t if hnd else t.transpose(1, 2) for t in (q, k, v))
    Hq, Hk = qh.size(1), kh.size(1)
    assert Hq % world == 0 and Hk % world == 0, f"Ulysses needs num heads ({Hq}, {Hk}) divisible by the group size {world}"
    assert qh.size(2) == kh.size(2) or not is_causal, "qo_len and kv_len must be equal for causal attention."
    if world == 1:
        return attn_fn(q, k, v, tensor_layout=tensor_layout, is_causal=is_causal, sm_scale=sm_scale, **kwargs)
    qf, kf, vf = (_seq_to_head_shard(t, world, group) for t in (qh, kh, vh))
    of = attn_fn(qf, kf, vf, tensor_layout="HND", is_causal=is_causal, sm_scale=sm_scale, **kwargs)
    o = _head_to_seq_shard(of.contiguous(), world, group)
    return o if hnd else o.transpose(1, 2)


# ------------------------------------------------------------------ ring attention over return_lse
def merge_attention_states(o_a: torch.Tensor, lse_a: torch.Tensor, o_b: torch.Tensor, lse_b: torch.Tensor, hnd: bool = True):
    """Combine two partial attention results over disjoint key sets from their natural-log LSEs (the use the reference
    gives `return_lse`, sageattention/core.py:289-293, 329): softmax weights of the union = exp(lse_x - logaddexp)."""
    lse = torch.logaddexp(lse_a, lse_b)
    wa, wb = torch.exp(lse_a - lse), torch.exp(lse_b - lse)                 # [B,H,S]
    if not hnd:
        wa, wb = wa.transpose(1, 2), wb.transpose(1, 2)
    o = o_a.float() * wa.unsqueeze(-1) + o_b.float() * wb.unsqueeze(-1)
    return o, lse


def sageattn_ring(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, tensor_layout: str = "HND", is_causal: bool = False,
                  sm_scale: Optional[float] = None, group=None, attn_fn=None, **kwargs: Any) -> torch.Tensor:
    """Ring attention: Q stays put, the K/V slices travel round the ring (P-1 send/recv steps, bf16/fp16 payload), each
    step is one `sageattn(..., return_lse=True)` on the local Q slice against the visiting K/V slice and the partial
    results are merged through their LSEs.  For sequences whose gathered K/V do not fit one GPU; otherwise prefer
    `sageattn_sp` (one 8-bit gather, one kernel) — this form quantises every visiting slice again and smooths K per
    slice (the LSE returned by the operator is already corrected to the unsmoothed keys, core.py:329), so its result
    agrees with the single-GPU call to quantisation accuracy, not bit for bit.
    Causal: slices from later ranks are skipped, the diagonal slice runs causal, earlier slices run unmasked."""
    if not dist.is_initialized():
        raise RuntimeError("sageattn_ring needs an initialised torch.distributed process group")
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    if tensor_layout not in ("HND", "NHD"):
        raise ValueError(f"Unknown tensor layout: {tensor_layout}")
    if attn_fn is None:
        from .core import sageattn_qk_int8_pv_fp8_cuda as attn_fn
    hnd = tensor_layout == "HND"
    k_cur, v_cur = k.contiguous(), v.contiguous()
    o_acc, lse_acc = None, None
    for step in range(world):
        src = (rank - step) % world                       # owner of the K/V slice held in this step
        reqs = []
        if step + 1 < world:                              # pass the slice on while computing with it
            k_nxt, v_nxt = torch.empty_like(k_cur), torch.empty_like(v_cur)
            nxt, prv = (rank + 1) % world, (rank - 1) % world
            if group is not None:      # P2POp peers are GLOBAL ranks: translate for sub-groups (SP groups inside a DPxSP job)
                nxt, prv = dist.get_global_rank(group, nxt), dist.get_global_rank(group, prv)
            ops_ = [dist.P2POp(dist.isend, k_cur, nxt, group), dist.P2POp(dist.isend, v_cur, nxt, group),
                    dist.P2POp(dist.irecv, k_nxt, prv, group), dist.P2POp(dist.irecv, v_nxt, prv, group)]
            reqs = dist.batch_isend_irecv(ops_)
        if not (is_causal and src > rank):
            o_i, lse_i = attn_fn(q, k_cur, v_cur, tensor_layout=tensor_layout, is_causal=bool(is_causal and src == rank),
                                 sm_scale=sm_scale, return_lse=True, **kwargs)
            if o_acc is None:
                o_acc, lse_acc = o_i.float(), lse_i
            else:
                o_acc, lse_acc = merge_attention_states(o_acc, lse_acc, o_i, lse_i, hnd)
        for r in reqs:
            r.wait()
        if step + 1 < world:
            k_cur, v_cur = k_nxt, v_nxt
    return o_acc.to(q.dtype)
