"""Paged KV-cache benchmark: sageattn_varlen_kvcache against the routes a caller has without it, in one run, alternated.

Setup: Hq=32, Hkv=8, D=128, bf16, page_size 16, bottom-right causal.  Workloads (the LLM prefill shapes a serving stack runs):
  chunked_prefill          four sequences with cached prefixes of 2048, 6144, 14336 and 30720 tokens, plus a 2048-token chunk each;
  prefix_caching           eight sequences sharing one 8192-token prefix through shared pages, plus 1024 new tokens each;
  speculative_verification 32 sequences, Lq = 8, Lk from 4K to 16K.  For context only: one 128-row Q tile per (sequence, head)
                           holds 8 rows, so most of the tensor-core work is idle by design.
Routes:
  kvcache  sageattn_varlen_kvcache (the quantisers read the pages);
  gather   a torch page gather into 16-bit per-sequence K / V, then sageattn_window(..., (-1, Lk - Lq)) per sequence: the same bits;
  sdpa     torch SDPA per sequence on the gathered bf16 tensors with a lower-right causal bias, for context.
Reported per workload: call ms (CUDA events, median of --reps alternated rounds of --steps calls), the attention-kernel and
quantiser ms of the new call (torch.profiler, a run of its own), 4*Hq*D*(visible pairs)/t in TFLOP/s, the peak memory each route
allocates beyond its inputs (torch.cuda.max_memory_allocated), the GPU name and power limit, and one JSON line at the end.

    python bench_kvcache.py [--steps 10] [--warmup 3] [--reps 3] [--workload NAME]
"""
import argparse
import collections
import json
import statistics
import subprocess

import torch

HQ, HKV, D, PAGE = 32, 8, 128, 16
Workload = collections.namedtuple("Workload", "name lens_q lens_k shared_prefix")
WORKLOADS = [
    Workload("chunked_prefill", [2048] * 4, [p + 2048 for p in (2048, 6144, 14336, 30720)], 0),
    Workload("prefix_caching", [1024] * 8, [8192 + 1024] * 8, 8192),
    Workload("speculative_verification", [8] * 32, [4096 + 384 * i for i in range(32)], 0),
]


def visible_pairs(lens_q, lens_k, causal=True):
    """Query-key pairs the call evaluates, summed over sequences (one head): bottom-right causal, query i of a sequence sees
    key j iff j <= i + Lk - Lq."""
    total = 0
    for lq, lk in zip(lens_q, lens_k):
        if not causal:
            total += lq * lk
            continue
        off = lk - lq
        for i in range(lq):             # rows see min(lk, max(0, i + off + 1)) keys
            total += min(lk, max(0, i + off + 1))
    return total


def _gpu():
    name = torch.cuda.get_device_name(0)
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        return {"name": name, "power_limit_w": float(r.stdout.strip())}
    except Exception as e:  # the figure is still stated next to the numbers, as unknown
        return {"name": name, "power_limit_w": None, "error": str(e)}


def _events(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def make_inputs(w, seed=0):
    """q packed [Tq,Hq,D], the paged caches, block table, cu_seqlens_q and seqused_k of a workload.  The shared prefix of
    prefix_caching is one set of pages every sequence's table names; every other page belongs to one sequence, in shuffled order."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    pages = [(n + PAGE - 1) // PAGE for n in w.lens_k]
    npre = w.shared_prefix // PAGE
    num_pages = npre + sum(p - npre for p in pages)
    perm = torch.randperm(num_pages, generator=g, device="cuda").to(torch.int32)
    table = torch.zeros(len(pages), max(pages), dtype=torch.int32, device="cuda")
    nxt = npre
    for b, p in enumerate(pages):
        table[b, :npre] = perm[:npre]
        table[b, npre:p] = perm[nxt:nxt + p - npre]
        nxt += p - npre
    kv = torch.randn(2, num_pages, PAGE, HKV, D, generator=g, device="cuda", dtype=torch.bfloat16)
    kv[0] += torch.randn(HKV, D, generator=g, device="cuda", dtype=torch.bfloat16)
    q = torch.randn(sum(w.lens_q), HQ, D, generator=g, device="cuda", dtype=torch.bfloat16)
    cu = torch.tensor([0] + torch.cumsum(torch.tensor(w.lens_q), 0).tolist(), dtype=torch.int32, device="cuda")
    used = torch.tensor(w.lens_k, dtype=torch.int32, device="cuda")
    return q, kv[0], kv[1], table, cu, used


def _gather(cache, table, n):
    t = torch.arange(n, device="cuda")
    return cache[table[t // PAGE].long(), t % PAGE]                       # [n,Hkv,D]


def routes(w, q, k_cache, v_cache, table, cu, used):
    import sageattention_b200 as sab
    from torch.nn.attention.bias import causal_lower_right
    import torch.nn.functional as F
    spans = list(zip(cu.tolist()[:-1], cu.tolist()[1:]))

    def kvcache():
        return sab.sageattn_varlen_kvcache(q, k_cache, v_cache, cu, used, table, max(w.lens_q), is_causal=True)

    def gather():
        o = torch.empty_like(q)
        for b, (s, e) in enumerate(spans):
            lk = w.lens_k[b]
            k, v = _gather(k_cache, table[b], lk), _gather(v_cache, table[b], lk)
            o[s:e] = sab.sageattn_window(q[s:e][None], k[None], v[None], (-1, lk - (e - s)), tensor_layout="NHD")[0]
        return o

    def sdpa():
        o = torch.empty_like(q)
        g = HQ // HKV
        for b, (s, e) in enumerate(spans):
            lk = w.lens_k[b]
            k, v = _gather(k_cache, table[b], lk), _gather(v_cache, table[b], lk)
            qh = q[s:e].transpose(0, 1)[None]
            kh = k.transpose(0, 1).repeat_interleave(g, 0)[None]
            vh = v.transpose(0, 1).repeat_interleave(g, 0)[None]
            o[s:e] = F.scaled_dot_product_attention(qh, kh, vh, attn_mask=causal_lower_right(e - s, lk))[0].transpose(0, 1)
        return o
    return {"kvcache": kvcache, "gather": gather, "sdpa": sdpa}


def _peak_extra_mb(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)


def _profile_split(fn, steps):
    """Mean device ms per call of the attention kernel and of everything else the call launches (the quantisers)."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
    attn = other = 0.0
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
        if getattr(e, "device_type", None) is not None and "CUDA" not in str(e.device_type):
            continue
        if "sage_attn_fwd_kernel" in e.key:
            attn += t
        elif "kernel" in e.key.lower() and ("quant" in e.key or "channel_stats" in e.key):
            other += t
    return round(attn / 1e3 / steps, 3), round(other / 1e3 / steps, 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--workload", default=None, choices=[w.name for w in WORKLOADS])
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_kvcache.py measures on a GPU; none is visible")
    gpu = _gpu()
    results = []
    for w in WORKLOADS:
        if a.workload and w.name != a.workload:
            continue
        q, kc, vc, table, cu, used = make_inputs(w)
        fns = routes(w, q, kc, vc, table, cu, used)
        same = torch.equal(fns["kvcache"](), fns["gather"]())
        times = {name: [] for name in fns}
        for _ in range(a.reps):
            for name, fn in fns.items():
                times[name].append(_events(fn, a.steps, a.warmup))
        ms = {name: round(statistics.median(t), 3) for name, t in times.items()}
        mem = {name: _peak_extra_mb(fn) for name, fn in fns.items()}
        kern_ms, quant_ms = _profile_split(fns["kvcache"], a.steps)
        flop = 4 * HQ * D * visible_pairs(w.lens_q, w.lens_k)
        r = {"workload": w.name, "nseq": len(w.lens_q), "tokens_q": sum(w.lens_q), "tokens_k": sum(w.lens_k),
             "ms": ms, "tflops": {name: round(flop / (t * 1e-3) / 1e12, 1) for name, t in ms.items()},
             "kvcache_kernel_ms": kern_ms, "kvcache_quant_ms": quant_ms,
             "kvcache_kernel_tflops": round(flop / (kern_ms * 1e-3) / 1e12, 1) if kern_ms else None,
             "speedup_vs_gather": round(ms["gather"] / ms["kvcache"], 3), "peak_extra_mb": mem, "bits_equal_gather": same}
        results.append(r)
        print(f"{w.name:26s} call ms kvcache {ms['kvcache']:8.3f}  gather {ms['gather']:8.3f}  sdpa {ms['sdpa']:8.3f} | "
              f"kernel {kern_ms:7.3f} quant {quant_ms:7.3f} | TFLOP/s {r['tflops']['kvcache']:6.1f} | "
              f"peak MB {mem['kvcache']:8.1f} / {mem['gather']:8.1f} / {mem['sdpa']:8.1f} | bits equal {same}", flush=True)
        del q, kc, vc, table, fns
        torch.cuda.empty_cache()
    print(json.dumps({"bench": "kvcache", "gpu": gpu, "heads": [HQ, HKV], "head_dim": D, "dtype": "bf16", "page_size": PAGE,
                      "steps": a.steps, "warmup": a.warmup, "reps": a.reps, "results": results}))


if __name__ == "__main__":
    main()
