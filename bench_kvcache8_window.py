"""Sliding-window benchmark on the 8-bit paged KV cache: sageattn_kvcache8 / sageattn_kvcache8_prefill with window_size=(left, 0)
against the same call without a window and torch SDPA on the window, alternated in one run.

Setup (that of the other cache benchmarks): Hq=32, Hkv=8, D=128, bf16, page_size 16, bottom-right causal; a local-attention
layer sees the last left + 1 keys, left in LEFTS.  Workloads:
  decode               32 sequences, 1 new token each, Lk 4096..16000;
  long_context_decode  1 sequence, 1 new token, Lk 131072: about left / 1024 + 1 working chunk CTAs per KV head, latency-bound;
  chunked_prefill      four 2048-token chunks after cached prefixes, Lk 4096, 8192, 16384 and 32768.
Routes:
  window  the windowed call on a PagedKVCache8 written with cache.write from the bf16 pages (k_smooth: the mean key);
  full    the same call without a window: the cost of attending over the whole cache;
  sdpa    torch SDPA per sequence on a bf16 gather of the window's keys (built outside the timing) with a bottom-right band mask.
Reported per workload and left: call ms (CUDA events, median of --reps alternated rounds of --steps calls); the kernel ms of both
cache routes (torch.profiler, a run of its own: the attention and combine kernels for decode); the cache bytes the kernel must
read (keys in the window x Hkv x (2 D + 8)) over kernel time in TB/s and as a share of 3.35 TB/s (decode), or 4 Hq D x visible
pairs over kernel time in TFLOP/s (prefill); the max / mean error of the windowed call against fp64 attention on the bf16 window
(four Q heads); the GPU name and power limit, and one JSON line at the end.

    python bench_kvcache8_window.py [--steps 20] [--warmup 3] [--reps 3] [--workload NAME]
"""
import argparse
import json
import statistics

import torch

import bench_kvcache as bk
import bench_kvcache8_prefill as bp

HQ, HKV, D, PAGE = bk.HQ, bk.HKV, bk.D, bk.PAGE
LEFTS = (1024, 4096)
HBM_TBS = 3.35e12                   # H100 SXM data sheet
ERR_HEADS = (0, 9, 18, 27)
WORKLOADS = [
    bk.Workload("decode", [1] * 32, [4096 + 384 * i for i in range(32)], 0),
    bk.Workload("long_context_decode", [1], [131072], 0),
    bk.Workload("chunked_prefill", [2048] * 4, [4096, 8192, 16384, 32768], 0),
]


def window_keys(w, left):
    """Keys the call must read, summed over sequences: j >= max(0, Lk - Lq - left), every key when left == -1."""
    return sum(lk if left < 0 else min(lk, lq + left) for lq, lk in zip(w.lens_q, w.lens_k))


def bytes_read(w, left):
    """8-bit K and V plus an fp32 scale each, per key in the window and KV head."""
    return window_keys(w, left) * HKV * (2 * D + 8)


def visible_pairs(w, left):
    """(query, key) pairs of one head: row i sees keys max(0, i + off - left) .. i + off, off = Lk - Lq."""
    total = 0
    for lq, lk in zip(w.lens_q, w.lens_k):
        for i in range(lq):
            d = i + lk - lq
            if d >= 0:
                total += (d if left < 0 else min(d, left)) + 1
    return total


def flops(w, left):
    return 4 * HQ * D * visible_pairs(w, left)


def _windows(w, left):
    """Per sequence: (first key read, the band mask [Lq, keys read]) of the windowed call."""
    out = []
    for lq, lk in zip(w.lens_q, w.lens_k):
        start = max(0, lk - lq - left)
        i = torch.arange(lq, device="cuda")[:, None] + lk - lq
        j = torch.arange(start, lk, device="cuda")[None, :]
        out.append((start, (j <= i) & (j >= i - left)))
    return out


def routes(w, left, q, k_cache, v_cache, cache8, table, cu, used):
    import torch.nn.functional as F
    import sageattention_b200 as sab
    lq = max(w.lens_q)
    call = sab.sageattn_kvcache8 if lq == 1 else sab.sageattn_kvcache8_prefill
    spans = list(zip(cu.tolist()[:-1], cu.tolist()[1:]))
    g = HQ // HKV
    gathered = []
    for b, (start, mask) in enumerate(_windows(w, left)):
        lk = w.lens_k[b]
        k, v = bk._gather(k_cache, table[b], lk)[start:], bk._gather(v_cache, table[b], lk)[start:]
        gathered.append((k.transpose(0, 1).repeat_interleave(g, 0)[None].contiguous(),
                         v.transpose(0, 1).repeat_interleave(g, 0)[None].contiguous(), mask))

    def window():
        return call(q, cache8, cu, used, table, lq, is_causal=True, window_size=(left, 0))

    def full():
        return call(q, cache8, cu, used, table, lq, is_causal=True)

    def sdpa():
        o = torch.empty_like(q)
        for (s, e), (kh, vh, mask) in zip(spans, gathered):
            o[s:e] = F.scaled_dot_product_attention(q[s:e].transpose(0, 1)[None], kh, vh, attn_mask=mask)[0].transpose(0, 1)
        return o
    return {"window": window, "full": full, "sdpa": sdpa}


def _errors(w, left, q, k_cache, v_cache, o, table):
    """Max and mean |o - fp64 attention on the bf16 window| over every sequence, on ERR_HEADS."""
    mx, tot, cnt = 0.0, 0.0, 0
    s = 0
    for b, (start, mask) in enumerate(_windows(w, left)):
        lq, lk = w.lens_q[b], w.lens_k[b]
        k, v = bk._gather(k_cache, table[b], lk)[start:], bk._gather(v_cache, table[b], lk)[start:]
        for h in ERR_HEADS:
            hk = h // (HQ // HKV)
            sc = q[s:s + lq, h].double() @ k[:, hk].double().T * D ** -0.5
            ref = torch.softmax(sc.masked_fill(~mask, float("-inf")), -1) @ v[:, hk].double()
            e = (o[s:s + lq, h].double() - ref).abs()
            mx, tot, cnt = max(mx, e.max().item()), tot + e.sum().item(), cnt + e.numel()
        s += lq
    return {"max": round(mx, 5), "mean": round(tot / cnt, 6)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--workload", default=None, choices=[w.name for w in WORKLOADS])
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_kvcache8_window.py measures on a GPU; none is visible")
    gpu = bk._gpu()
    results = []
    for w in WORKLOADS:
        if a.workload and w.name != a.workload:
            continue
        q, kc, vc, table, cu, used = bk.make_inputs(w)
        cache8 = bp.make_cache8(kc, vc)
        decode = max(w.lens_q) == 1
        kname = "kv8_" if decode else "kv8_prefill_kernel"
        for left in LEFTS:
            fns = routes(w, left, q, kc, vc, cache8, table, cu, used)
            err = _errors(w, left, q, kc, vc, fns["window"](), table)
            times = {name: [] for name in fns}
            for _ in range(a.reps):
                for name, fn in fns.items():
                    times[name].append(bk._events(fn, a.steps, a.warmup))
            ms = {name: round(statistics.median(t), 4) for name, t in times.items()}
            kern = {name: bp._kernel_ms(fns[name], a.steps, kname) for name in ("window", "full")}
            nbytes = {"window": bytes_read(w, left), "full": bytes_read(w, -1)}
            r = {"workload": w.name, "left": left, "nseq": len(w.lens_q), "tokens_q": sum(w.lens_q), "tokens_k": sum(w.lens_k),
                 "window_keys": window_keys(w, left), "ms": ms, "kernel_ms": kern, "bytes_read": nbytes,
                 "speedup_vs_full": round(ms["full"] / ms["window"], 3), "err_vs_fp64": err}
            if decode:
                r["tbs_kernel"] = {n: round(nbytes[n] / (kern[n] * 1e-3) / 1e12, 3) if kern[n] else None for n in kern}
                r["share_of_hbm"] = {n: round(v / (HBM_TBS / 1e12), 3) if v else None for n, v in r["tbs_kernel"].items()}
                rate = f"TB/s {r['tbs_kernel']['window']} / {r['tbs_kernel']['full']}"
            else:
                f = {"window": flops(w, left), "full": flops(w, -1)}
                r["visible_pairs"] = visible_pairs(w, left)
                r["tflops_kernel"] = {n: round(f[n] / (kern[n] * 1e-3) / 1e12, 1) if kern[n] else None for n in kern}
                rate = f"TFLOP/s {r['tflops_kernel']['window']} / {r['tflops_kernel']['full']}"
            results.append(r)
            print(f"{w.name:20s} left {left:5d} call ms window {ms['window']:7.3f}  full {ms['full']:7.3f}  sdpa {ms['sdpa']:7.3f} | "
                  f"kernel ms {kern['window']:7.3f} / {kern['full']:7.3f}  {rate} | err max {err['max']:.4f} mean {err['mean']:.5f}",
                  flush=True)
            del fns
        del q, kc, vc, cache8, table
        torch.cuda.empty_cache()
    print(json.dumps({"bench": "kvcache8_window", "gpu": gpu, "heads": [HQ, HKV], "head_dim": D, "dtype": "bf16", "page_size": PAGE,
                      "lefts": list(LEFTS), "steps": a.steps, "warmup": a.warmup, "reps": a.reps, "results": results}))


if __name__ == "__main__":
    main()
