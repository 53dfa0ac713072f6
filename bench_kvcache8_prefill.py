"""Chunked-prefill benchmark on the 8-bit paged KV cache: sageattn_kvcache8_prefill against sageattn_varlen_kvcache on a bf16 cache
holding the same tokens and torch SDPA, alternated in one run.

Setup (that of bench_kvcache.py): Hq=32, Hkv=8, D=128, bf16, page_size 16, bottom-right causal.  Workloads:
  chunked_prefill  four sequences with cached prefixes of 2048, 6144, 14336 and 30720 tokens, plus a 2048-token chunk each;
  prefix_caching   eight sequences sharing one 8192-token prefix through shared pages, plus 1024 new tokens each.
Routes:
  prefill8  sageattn_kvcache8_prefill on a PagedKVCache8 written with cache.write from the bf16 pages (k_smooth: the mean key);
  kvcache   sageattn_varlen_kvcache on the bf16 cache;
  sdpa      torch SDPA per sequence on K / V gathered from the bf16 pages, with a lower-right causal bias, for context.
Reported per workload: call ms (CUDA events, median of --reps alternated rounds of --steps calls); the attention kernel ms of both
cache routes (torch.profiler, a run of its own); 4*Hq*D*(visible pairs)/t in TFLOP/s and the prefill kernel's share of the dense
bound (half the FLOPs INT8 QK^T at 1979, half bf16 PV at 989 TFLOP/s, the H100 SXM data sheet); the cache bytes each cache route
reads; the max / mean error of both cache routes against fp64 attention on the bf16 K / V (four Q heads, one per pair of KV
heads); the GPU name and power limit, and one JSON line at the end.

    python bench_kvcache8_prefill.py [--steps 10] [--warmup 3] [--reps 3] [--workload NAME]
"""
import argparse
import json
import statistics

import torch

import bench_kvcache as bk

HQ, HKV, D, PAGE = bk.HQ, bk.HKV, bk.D, bk.PAGE
WORKLOADS = [w for w in bk.WORKLOADS if w.name in ("chunked_prefill", "prefix_caching")]
INT8_TFLOPS, BF16_TFLOPS = 1979e12, 989e12      # H100 SXM data sheet, dense
ERR_HEADS = (0, 9, 18, 27)


def flops(w):
    """4 Hq D per visible (query, key) pair: QK^T and PV, two FLOPs per multiply-add each."""
    return 4 * HQ * D * bk.visible_pairs(w.lens_q, w.lens_k)


def peak_seconds(w):
    """The least time the tensor cores need: half the FLOPs are INT8 QK^T, half bf16 PV."""
    f = flops(w)
    return f / 2 / INT8_TFLOPS + f / 2 / BF16_TFLOPS


def cache_bytes_read(w, bits16=False):
    """Cache bytes one call reads at least once: every key of every sequence per KV head (a shared prefix counts per sequence).
    8-bit: INT8 K and e4m3 V plus an fp32 scale each; bf16: 16-bit K and V."""
    return sum(w.lens_k) * HKV * (4 * D if bits16 else 2 * D + 8)


def make_cache8(k_cache, v_cache):
    """A PagedKVCache8 holding the bf16 pages' tokens in the same slots, k_smooth the mean key."""
    import sageattention_b200 as sab
    num_pages = k_cache.size(0)
    cache = sab.PagedKVCache8(num_pages, PAGE, HKV, D, torch.bfloat16, k_smooth=k_cache.float().mean((0, 1)))
    cache.write(k_cache.reshape(-1, HKV, D), v_cache.reshape(-1, HKV, D), torch.arange(num_pages * PAGE, device="cuda"))
    return cache


def routes(w, q, k_cache, v_cache, cache8, table, cu, used):
    import sageattention_b200 as sab
    fns = bk.routes(w, q, k_cache, v_cache, table, cu, used)
    lq = max(w.lens_q)

    def prefill8():
        return sab.sageattn_kvcache8_prefill(q, cache8, cu, used, table, lq, is_causal=True)
    return {"prefill8": prefill8, "kvcache": fns["kvcache"], "sdpa": fns["sdpa"]}


def _kernel_ms(fn, steps, name):
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
        if name in e.key:
            tot += getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
    return round(tot / 1e3 / steps, 4)


def _errors(w, q, k_cache, v_cache, outs, table):
    """Max and mean |o - fp64 attention on the bf16 K / V| of each route over every sequence, on ERR_HEADS."""
    err = {name: [0.0, 0.0, 0] for name in outs}
    s = 0
    for b, (lq, n) in enumerate(zip(w.lens_q, w.lens_k)):
        k, v = bk._gather(k_cache, table[b], n), bk._gather(v_cache, table[b], n)
        vis = torch.arange(n, device="cuda")[None, :] <= torch.arange(lq, device="cuda")[:, None] + n - lq
        for h in ERR_HEADS:
            hk = h // (HQ // HKV)
            sc = q[s:s + lq, h].double() @ k[:, hk].double().T * D ** -0.5
            ref = torch.softmax(sc.masked_fill(~vis, float("-inf")), -1) @ v[:, hk].double()
            for name, o in outs.items():
                e = (o[s:s + lq, h].double() - ref).abs()
                err[name][0] = max(err[name][0], e.max().item())
                err[name][1] += e.sum().item()
                err[name][2] += e.numel()
            del sc, ref
        s += lq
    return {name: {"max": round(m, 5), "mean": round(t / c, 6)} for name, (m, t, c) in err.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--workload", default=None, choices=[w.name for w in WORKLOADS])
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_kvcache8_prefill.py measures on a GPU; none is visible")
    gpu = bk._gpu()
    results = []
    for w in WORKLOADS:
        if a.workload and w.name != a.workload:
            continue
        q, kc, vc, table, cu, used = bk.make_inputs(w)
        cache8 = make_cache8(kc, vc)
        fns = routes(w, q, kc, vc, cache8, table, cu, used)
        outs = {name: fn() for name, fn in fns.items() if name != "sdpa"}
        errs = _errors(w, q, kc, vc, outs, table)
        del outs
        times = {name: [] for name in fns}
        for _ in range(a.reps):
            for name, fn in fns.items():
                times[name].append(_events(fn, a.steps, a.warmup))
        ms = {name: round(statistics.median(t), 4) for name, t in times.items()}
        kern = {"prefill8": _kernel_ms(fns["prefill8"], a.steps, "kv8_prefill_kernel"),
                "kvcache": _kernel_ms(fns["kvcache"], a.steps, "sage_attn_fwd_kernel")}
        f = flops(w)
        r = {"workload": w.name, "nseq": len(w.lens_q), "tokens_q": sum(w.lens_q), "tokens_k": sum(w.lens_k), "ms": ms,
             "kernel_ms": kern, "tflops_call": {name: round(f / (t * 1e-3) / 1e12, 1) for name, t in ms.items()},
             "tflops_kernel": {name: round(f / (t * 1e-3) / 1e12, 1) if t else None for name, t in kern.items()},
             "prefill8_share_of_dense_bound": round(peak_seconds(w) / (kern["prefill8"] * 1e-3), 3) if kern["prefill8"] else None,
             "cache_bytes_read": {"prefill8": cache_bytes_read(w), "kvcache": cache_bytes_read(w, bits16=True)},
             "speedup_vs_kvcache": round(ms["kvcache"] / ms["prefill8"], 3), "err_vs_fp64": errs}
        results.append(r)
        print(f"{w.name:16s} call ms prefill8 {ms['prefill8']:7.3f}  kvcache {ms['kvcache']:7.3f}  sdpa {ms['sdpa']:7.3f} | "
              f"kernel ms {kern['prefill8']:7.3f} / {kern['kvcache']:7.3f} = TFLOP/s {r['tflops_kernel']['prefill8']} / "
              f"{r['tflops_kernel']['kvcache']} ({r['prefill8_share_of_dense_bound']} of the dense bound) | "
              f"err max {errs['prefill8']['max']:.4f} / {errs['kvcache']['max']:.4f}  mean {errs['prefill8']['mean']:.5f} / "
              f"{errs['kvcache']['mean']:.5f}", flush=True)
        del q, kc, vc, cache8, table, fns
        torch.cuda.empty_cache()
    print(json.dumps({"bench": "kvcache8_prefill", "gpu": gpu, "heads": [HQ, HKV], "head_dim": D, "dtype": "bf16", "page_size": PAGE,
                      "steps": a.steps, "warmup": a.warmup, "reps": a.reps, "results": results}))


_events = bk._events

if __name__ == "__main__":
    main()
