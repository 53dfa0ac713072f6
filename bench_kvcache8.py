"""8-bit paged KV-cache benchmark: sageattn_kvcache8 against sageattn_varlen_kvcache on the equivalent 16-bit cache and torch SDPA,
alternated in one run.

Setup (that of bench_kvcache.py): Hq=32, Hkv=8, D=128, bf16, page_size 16, bottom-right causal.  Workloads:
  decode                    32 sequences, Lq = 1, Lk = 4096 + 384 i;
  speculative_verification  32 sequences, Lq = 8, the same Lk;
  long_context_decode       one sequence, Lq = 1, Lk = 131072.
Routes:
  kvcache8  sageattn_kvcache8 on a PagedKVCache8 holding the same tokens;
  kvcache   sageattn_varlen_kvcache on the 16-bit cache;
  sdpa      torch SDPA (enable_gqa) on a padded batch gathered from the 16-bit pages, with a lower-right causal mask, for context.
Reported per workload: call ms (CUDA events, median of --reps alternated rounds of --steps calls); the attention + combine kernel ms
of sageattn_kvcache8 (torch.profiler, a run of its own); the write kernel's ms for one decode step's 32 tokens; cache bytes read /
kernel time against the 3.35 TB/s data-sheet bandwidth of the H100 SXM (decode is bound by bytes: the FLOPs are 4 Hq D per pair);
cache bytes per token of each cache; the GPU name and power limit, and one JSON line at the end.

    python bench_kvcache8.py [--steps 20] [--warmup 5] [--reps 3] [--workload NAME]
"""
import argparse
import collections
import json
import statistics
import subprocess

import torch

HQ, HKV, D, PAGE = 32, 8, 128, 16
HBM_BYTES_PER_S = 3.35e12       # H100 SXM data sheet
Workload = collections.namedtuple("Workload", "name lens_q lens_k")
WORKLOADS = [
    Workload("decode", [1] * 32, [4096 + 384 * i for i in range(32)]),
    Workload("speculative_verification", [8] * 32, [4096 + 384 * i for i in range(32)]),
    Workload("long_context_decode", [1], [131072]),
]


def cache_bytes_per_token(hkv=HKV, d=D, bits16=False):
    """Bytes one token takes in the cache: 16-bit K and V, or 8-bit K and V plus an fp32 scale each per KV head."""
    return hkv * (4 * d if bits16 else 2 * d + 8)


def bytes_read(lens_k, hkv=HKV, d=D):
    """Cache bytes sageattn_kvcache8 reads: every key of every sequence once per KV head."""
    return sum(lens_k) * cache_bytes_per_token(hkv, d)


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
    """q packed [Tq,Hq,D], the 16-bit paged caches in shuffled pages, the 8-bit cache written from them (k_smooth: the mean key),
    block table, cu_seqlens_q and seqused_k."""
    import sageattention_b200 as sab
    g = torch.Generator(device="cuda").manual_seed(seed)
    pages = [(n + PAGE - 1) // PAGE for n in w.lens_k]
    num_pages = sum(pages)
    perm = torch.randperm(num_pages, generator=g, device="cuda").to(torch.int32)
    table = torch.zeros(len(pages), max(pages), dtype=torch.int32, device="cuda")
    nxt = 0
    for b, p in enumerate(pages):
        table[b, :p] = perm[nxt:nxt + p]
        nxt += p
    kv = torch.randn(2, num_pages, PAGE, HKV, D, generator=g, device="cuda", dtype=torch.bfloat16)
    kv[0] += torch.randn(HKV, D, generator=g, device="cuda", dtype=torch.bfloat16)
    q = torch.randn(sum(w.lens_q), HQ, D, generator=g, device="cuda", dtype=torch.bfloat16)
    cu = torch.tensor([0] + torch.cumsum(torch.tensor(w.lens_q), 0).tolist(), dtype=torch.int32, device="cuda")
    used = torch.tensor(w.lens_k, dtype=torch.int32, device="cuda")
    cache = sab.PagedKVCache8(num_pages, PAGE, HKV, D, torch.bfloat16, k_smooth=kv[0].float().mean((0, 1)))
    slots = torch.arange(num_pages * PAGE, device="cuda")
    cache.write(kv[0].reshape(-1, HKV, D), kv[1].reshape(-1, HKV, D), slots)
    return q, kv[0], kv[1], cache, table, cu, used


def _gather(cache, table, n):
    t = torch.arange(n, device="cuda")
    return cache[table[t // PAGE].long(), t % PAGE]                       # [n,Hkv,D]


def routes(w, q, k_cache, v_cache, cache8, table, cu, used):
    import sageattention_b200 as sab
    import torch.nn.functional as F
    nseq, lq, lk = len(w.lens_q), max(w.lens_q), max(w.lens_k)
    # the padded batch SDPA reads, gathered once outside the timing (SDPA has no paged form): [nseq, Hkv, lk, D], lower-right mask
    kp = torch.zeros(nseq, HKV, lk, D, dtype=q.dtype, device="cuda")
    vp = torch.zeros_like(kp)
    mask = torch.zeros(nseq, 1, lq, lk, dtype=torch.bool, device="cuda")
    for b, n in enumerate(w.lens_k):
        kp[b, :, :n] = _gather(k_cache, table[b], n).transpose(0, 1)
        vp[b, :, :n] = _gather(v_cache, table[b], n).transpose(0, 1)
        mask[b, 0] = torch.arange(lk, device="cuda")[None, :] <= torch.arange(lq, device="cuda")[:, None] + n - lq
    qp = q.view(nseq, lq, HQ, D).transpose(1, 2)

    def kvcache8():
        return sab.sageattn_kvcache8(q, cache8, cu, used, table, lq, is_causal=True)

    def kvcache():
        return sab.sageattn_varlen_kvcache(q, k_cache, v_cache, cu, used, table, lq, is_causal=True)

    def sdpa():
        return F.scaled_dot_product_attention(qp, kp, vp, attn_mask=mask, enable_gqa=True).transpose(1, 2).reshape(q.shape)
    return {"kvcache8": kvcache8, "kvcache": kvcache, "sdpa": sdpa}


def _profile_kernels(fn, steps, names):
    """Mean device ms per call of the kernels whose names contain one of `names`."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
    tot = 0.0
    for e in prof.key_averages():
        if getattr(e, "device_type", None) is not None and "CUDA" not in str(e.device_type):
            continue
        if any(n in e.key for n in names):
            tot += getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
    return round(tot / 1e3 / steps, 4)


def _errors(w, q, k_cache, v_cache, outs, table):
    """Max and mean |o - fp64 attention on the 16-bit K / V| of each route, over the first four sequences."""
    err = {name: [0.0, 0.0, 0] for name in outs}
    lq = max(w.lens_q)
    for b in range(min(4, len(w.lens_q))):
        n = w.lens_k[b]
        k, v = _gather(k_cache, table[b], n).double(), _gather(v_cache, table[b], n).double()
        qb = q[b * lq:(b + 1) * lq].double().transpose(0, 1)
        kh, vh = k.transpose(0, 1).repeat_interleave(HQ // HKV, 0), v.transpose(0, 1).repeat_interleave(HQ // HKV, 0)
        s = qb @ kh.transpose(1, 2) * D ** -0.5
        vis = torch.arange(n, device="cuda")[None, :] <= torch.arange(lq, device="cuda")[:, None] + n - lq
        ref = (torch.softmax(s.masked_fill(~vis, float("-inf")), -1) @ vh).transpose(0, 1)
        for name, o in outs.items():
            e = (o[b * lq:(b + 1) * lq].double() - ref).abs()
            err[name][0] = max(err[name][0], e.max().item())
            err[name][1] += e.sum().item()
            err[name][2] += e.numel()
    return {name: {"max": round(m, 5), "mean": round(s / c, 6)} for name, (m, s, c) in err.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--workload", default=None, choices=[w.name for w in WORKLOADS])
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_kvcache8.py measures on a GPU; none is visible")
    import sageattention_b200 as sab
    from sageattention_b200 import ops
    gpu = _gpu()
    results = []
    for w in WORKLOADS:
        if a.workload and w.name != a.workload:
            continue
        q, kc, vc, cache8, table, cu, used = make_inputs(w)
        fns = routes(w, q, kc, vc, cache8, table, cu, used)
        outs = {name: fn() for name, fn in fns.items()}
        errs = _errors(w, q, kc, vc, outs, table)
        times = {name: [] for name in fns}
        for _ in range(a.reps):
            for name, fn in fns.items():
                times[name].append(_events(fn, a.steps, a.warmup))
        ms = {name: round(statistics.median(t), 4) for name, t in times.items()}
        kern_ms = _profile_kernels(fns["kvcache8"], a.steps, ("kv8_attn_kernel", "kv8_combine_kernel"))
        # one decode step's write: 32 new tokens (K and V) into free slots of a cache of the same shape
        k_new = torch.randn(32, HKV, D, device="cuda", dtype=torch.bfloat16)
        scratch = sab.PagedKVCache8(4, PAGE, HKV, D, torch.bfloat16)
        slots = torch.arange(32, device="cuda", dtype=torch.int64)
        write_ms = _profile_kernels(lambda: scratch.write(k_new, k_new, slots), a.steps, ("kv8_write_kernel",))
        nbytes = bytes_read(w.lens_k)
        r = {"workload": w.name, "nseq": len(w.lens_q), "tokens_q": sum(w.lens_q), "tokens_k": sum(w.lens_k), "ms": ms,
             "kvcache8_kernel_ms": kern_ms, "write_ms_32_tokens": write_ms, "cache_bytes_read": nbytes,
             "kernel_tb_per_s": round(nbytes / (kern_ms * 1e-3) / 1e12, 3) if kern_ms else None,
             "share_of_hbm_peak": round(nbytes / HBM_BYTES_PER_S / (kern_ms * 1e-3), 3) if kern_ms else None,
             "speedup_vs_kvcache": round(ms["kvcache"] / ms["kvcache8"], 2), "err_vs_fp64": errs,
             "chunk_keys": ops.kvcache8_chunk_keys()}
        results.append(r)
        print(f"{w.name:26s} call ms kvcache8 {ms['kvcache8']:7.3f}  kvcache {ms['kvcache']:7.3f}  sdpa {ms['sdpa']:7.3f} | "
              f"kernel {kern_ms:7.4f} ms = {r['kernel_tb_per_s']} TB/s ({r['share_of_hbm_peak']} of 3.35) | write {write_ms:.4f} ms | "
              f"err max {errs['kvcache8']['max']:.4f} / {errs['kvcache']['max']:.4f}  mean {errs['kvcache8']['mean']:.5f} / "
              f"{errs['kvcache']['mean']:.5f}", flush=True)
        del q, kc, vc, cache8, table, fns, outs
        torch.cuda.empty_cache()
    print(json.dumps({"bench": "kvcache8", "gpu": gpu, "heads": [HQ, HKV], "head_dim": D, "dtype": "bf16", "page_size": PAGE,
                      "bytes_per_token": {"8bit": cache_bytes_per_token(), "bf16": cache_bytes_per_token(bits16=True)},
                      "steps": a.steps, "warmup": a.warmup, "reps": a.reps, "results": results}))


if __name__ == "__main__":
    main()
