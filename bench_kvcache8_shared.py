"""Shared-prefix decoding benchmark on the 8-bit paged KV cache: sageattn_kvcache8 with shared_prefix_len against the same call
without it and torch SDPA, alternated in one run.

Setup (that of the other cache benchmarks): Hq=32, Hkv=8, D=128, bf16, page_size 16, bottom-right causal.  Every sequence's
first pages are the prefix's pages (one set, named by every table row); the rest are its own.  Workloads:
  parallel_sampling    32 samples of one prompt: Lq = 1, an 8192-key shared prompt plus 64 i own keys (i = 0..31);
  system_prompt        64 requests behind one system prompt: Lq = 1, 4096 shared keys plus 1024..8192 own keys;
  shared_verification  16 sequences verifying 4 draft tokens each: Lq = 4, 8192 shared plus 512 own keys (4 sequences per CTA).
Routes:
  shared  sageattn_kvcache8(..., shared_prefix_len=prefix) on a PagedKVCache8 written with cache.write from the bf16 pages;
  plain   the same call with shared_prefix_len=0: its bits are checked equal to the shared route's in the run;
  sdpa    torch SDPA on a padded bf16 batch gathered from the pages outside the timing, with a causal and padding mask.
Reported per workload: call ms (CUDA events, median of --reps alternated rounds of --steps calls); the kernel ms of both cache
routes (torch.profiler, a run of its own: the attention and combine kernels); the cache bytes each route reads (bytes_read
below) over kernel time in TB/s and as a share of 3.35 TB/s; the GPU name and power limit, and one JSON line at the end.

Measured on one H100 80GB HBM3 at a 700 W power limit (one run; kernel ms shared / plain): parallel_sampling 0.136 / 0.422,
system_prompt 0.507 / 0.786, shared_verification 0.114 / 0.215, identical bits on every workload (README, "Shared-prefix decoding
on the 8-bit cache").

    python bench_kvcache8_shared.py [--steps 20] [--warmup 3] [--reps 5] [--workload NAME]
"""
import argparse
import json
import statistics

import torch

import bench_kvcache as bk
import bench_kvcache8_prefill as bp

HQ, HKV, D, PAGE = bk.HQ, bk.HKV, bk.D, bk.PAGE
CHUNK = 1024                        # ops.kvcache8_chunk_keys(), checked at run time
ROWS = 64                           # query rows per CTA and KV head
HBM_TBS = 3.35e12                   # H100 SXM data sheet
WORKLOADS = [
    bk.Workload("parallel_sampling", [1] * 32, [8192 + 64 * i for i in range(32)], 8192),
    bk.Workload("system_prompt", [1] * 64, [4096 + 1024 + 7168 * i // 63 for i in range(64)], 4096),
    bk.Workload("shared_verification", [4] * 16, [8192 + 512] * 16, 8192),
]


def taken_chunks(lq, lk, prefix):
    """Chunks of a sequence a shared CTA computes (causal): c < prefix // CHUNK with (c + 1) CHUNK <= Lk - Lq + 1, Lq >= 1."""
    if lq < 1:
        return 0
    return max(0, min(prefix // CHUNK, (lk - lq + 1) // CHUNK))


def keys_read(w, shared):
    """Keys per KV head a route reads: every key of every sequence without sharing; with it, each chunk some member of a slice
    (ROWS / (G max Lq) sequences) takes once per slice, plus every key of every sequence outside its taken chunks."""
    if not shared:
        return sum(w.lens_k)
    per = ROWS // (HQ // HKV * max(w.lens_q))
    taken = [taken_chunks(lq, lk, w.shared_prefix) for lq, lk in zip(w.lens_q, w.lens_k)]
    slices = sum(max(taken[s:s + per]) for s in range(0, len(taken), per))
    return slices * CHUNK + sum(lk - t * CHUNK for lk, t in zip(w.lens_k, taken))


def bytes_read(w, shared):
    """8-bit K and V plus an fp32 scale each, per key read and KV head."""
    return keys_read(w, shared) * HKV * (2 * D + 8)


def routes(w, q, k_cache, v_cache, cache8, table, cu, used):
    import torch.nn.functional as F
    import sageattention_b200 as sab
    lq, n, longest = max(w.lens_q), len(w.lens_q), max(w.lens_k)
    g = HQ // HKV
    kp = torch.zeros(n, HQ, longest, D, dtype=torch.bfloat16, device="cuda")
    vp = torch.zeros_like(kp)
    mask = torch.zeros(n, 1, lq, longest, dtype=torch.bool, device="cuda")
    for b, lk in enumerate(w.lens_k):
        kp[b, :, :lk] = bk._gather(k_cache, table[b], lk).transpose(0, 1).repeat_interleave(g, 0)
        vp[b, :, :lk] = bk._gather(v_cache, table[b], lk).transpose(0, 1).repeat_interleave(g, 0)
        mask[b, 0] = torch.arange(longest, device="cuda")[None, :] <= torch.arange(lq, device="cuda")[:, None] + lk - lq
    qp = q.view(n, lq, HQ, D).transpose(1, 2)

    def shared():
        return sab.sageattn_kvcache8(q, cache8, cu, used, table, lq, is_causal=True, return_lse=True,
                                     shared_prefix_len=w.shared_prefix)

    def plain():
        return sab.sageattn_kvcache8(q, cache8, cu, used, table, lq, is_causal=True, return_lse=True)

    def sdpa():
        return F.scaled_dot_product_attention(qp, kp, vp, attn_mask=mask)
    return {"shared": shared, "plain": plain, "sdpa": sdpa}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--workload", default=None, choices=[w.name for w in WORKLOADS])
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_kvcache8_shared.py measures on a GPU; none is visible")
    from sageattention_b200 import ops
    assert ops.kvcache8_chunk_keys() == CHUNK
    gpu = bk._gpu()
    results = []
    for w in WORKLOADS:
        if a.workload and w.name != a.workload:
            continue
        q, kc, vc, table, cu, used = bk.make_inputs(w)
        cache8 = bp.make_cache8(kc, vc)
        fns = routes(w, q, kc, vc, cache8, table, cu, used)
        o_s, l_s = fns["shared"]()
        o_p, l_p = fns["plain"]()
        same = torch.equal(o_s, o_p) and torch.equal(l_s, l_p)
        times = {name: [] for name in fns}
        for _ in range(a.reps):
            for name, fn in fns.items():
                times[name].append(bk._events(fn, a.steps, a.warmup))
        ms = {name: round(statistics.median(t), 4) for name, t in times.items()}
        kern = {name: bp._kernel_ms(fns[name], a.steps, "kv8_") for name in ("shared", "plain")}
        nbytes = {"shared": bytes_read(w, True), "plain": bytes_read(w, False)}
        tbs = {n: round(nbytes[n] / (kern[n] * 1e-3) / 1e12, 3) if kern[n] else None for n in kern}
        r = {"workload": w.name, "nseq": len(w.lens_q), "lq": max(w.lens_q), "shared_prefix": w.shared_prefix,
             "tokens_k": sum(w.lens_k), "ms": ms, "kernel_ms": kern, "bytes_read": nbytes, "tbs_kernel": tbs,
             "share_of_hbm": {n: round(v / (HBM_TBS / 1e12), 3) if v else None for n, v in tbs.items()},
             "call_speedup": round(ms["plain"] / ms["shared"], 3),
             "kernel_speedup": round(kern["plain"] / kern["shared"], 3) if kern["shared"] else None, "bits_equal": same}
        results.append(r)
        print(f"{w.name:20s} call ms shared {ms['shared']:7.3f}  plain {ms['plain']:7.3f}  sdpa {ms['sdpa']:7.3f} | "
              f"kernel ms {kern['shared']:7.3f} / {kern['plain']:7.3f} ({r['kernel_speedup']}x) | "
              f"MB {nbytes['shared'] / 1e6:7.1f} / {nbytes['plain'] / 1e6:7.1f} | TB/s {tbs['shared']} / {tbs['plain']} | "
              f"bits equal {same}", flush=True)
        del fns, q, kc, vc, cache8, table
        torch.cuda.empty_cache()
    print(json.dumps({"bench": "kvcache8_shared", "gpu": gpu, "heads": [HQ, HKV], "head_dim": D, "dtype": "bf16", "page_size": PAGE,
                      "steps": a.steps, "warmup": a.warmup, "reps": a.reps, "results": results}))


if __name__ == "__main__":
    main()
