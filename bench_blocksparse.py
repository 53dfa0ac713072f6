"""Block-sparse attention benchmark: sageattn_blocksparse's kernels against the dense INT8+FP8 kernels in the same run.

Workloads: B=4, H=32, S=8192 and B=1, H=30, S=32768 (D=128, bf16, non-causal).  Masks: seeded random block masks at densities
1.0, 0.5, 0.25 and 0.1, and a band ("local window": each 128-query block sees the 64-key blocks within +-1024 keys of it).
Per case: the sparse kernel ms and the dense kernel ms, timed alternately in the same run (median of --reps rounds of --steps
launches after --warmup), the whole sageattn_blocksparse call, the visible fraction and 4*D*(visible query-key pairs)/t.
--backward does the same for the gradient kernels against the dense backward's, and splits each backward call into its delta,
dQ and dK/dV kernels (torch.profiler).  Prints one JSON line with the GPU name and
power limit.  CUDA events; writes nothing.

    python bench_blocksparse.py [--steps 5] [--warmup 2] [--reps 3] [--backward] [--shapes 8k,32k]
"""
import argparse
import json
import statistics
import subprocess

import torch

SHAPES = {"8k": (4, 32, 8192, 128), "32k": (1, 30, 32768, 128)}


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


def _gpu():
    name = torch.cuda.get_device_name(0)
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        return {"name": name, "power_limit_w": float(r.stdout.strip())}
    except Exception as e:  # the figure is still stated next to the numbers, as unknown
        return {"name": name, "power_limit_w": None, "error": str(e)}


def _masks(B, H, S):
    nq, nk = (S + 127) // 128, (S + 63) // 64
    g = torch.Generator(device="cuda").manual_seed(0)
    out = {f"random_{p}": torch.rand(B, H, nq, nk, generator=g, device="cuda") < p for p in (1.0, 0.5, 0.25, 0.1)}
    qc = torch.arange(nq, device="cuda")[:, None] * 128 + 64
    kc = torch.arange(nk, device="cuda")[None, :] * 64 + 32
    out["band_1024"] = ((qc - kc).abs() <= 1024).expand(B, H, nq, nk)
    return out


def _pairs(bm, S):
    rows = torch.full((bm.size(2),), 128.0, device="cuda", dtype=torch.float64)
    rows[-1] = S - 128 * (bm.size(2) - 1)
    keys = torch.full((bm.size(3),), 64.0, device="cuda", dtype=torch.float64)
    keys[-1] = S - 64 * (bm.size(3) - 1)
    return float((rows[:, None] * bm.double() * keys[None, :]).sum())


def _split(fn, a):
    """Mean device ms per call of the delta, dQ and dK/dV kernels of a backward call (torch.profiler, --steps calls)."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(a.steps):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        for tag in ("bwd_delta", "bwd_dq", "bwd_dkdv"):
            if tag in e.key:
                t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
                out[tag] = round(out.get(tag, 0.0) + t / 1e3 / a.steps, 3)
    return out


def _alternate(fa, fb, a):
    ta, tb = [], []
    for _ in range(a.reps):
        ta.append(_events(fa, a.steps, a.warmup))
        tb.append(_events(fb, a.steps, a.warmup))
    return statistics.median(ta), statistics.median(tb)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--backward", action="store_true")
    ap.add_argument("--shapes", default="8k,32k")
    a = ap.parse_args()
    import sageattention_b200 as sab
    from sageattention_b200 import ops
    from sageattention_b200.core import _quant_qk
    from sageattention_b200.quant import per_channel_fp8

    out = {"metric": "sageattn_blocksparse " + ("backward" if a.backward else "forward") + " kernels vs dense", "gpu": _gpu(),
           "dtype": "bf16", "causal": False, "cases": []}
    for sname in a.shapes.split(","):
        B, H, S, D = SHAPES[sname]
        g = torch.Generator(device="cuda").manual_seed(0)
        q, k, v, do = (torch.randn(B, H, S, D, device="cuda", dtype=torch.bfloat16, generator=g) for _ in range(4))
        sm = D ** -0.5
        km, q8, qs, k8, ks, qg, kg, _ = _quant_qk(q, k, "fp8", "HND", "per_thread", sm, True, "cuda")
        v8, vs, vm = per_channel_fp8(v, tensor_layout="HND", scale_max=2.25, smooth_v=False)
        o = torch.empty_like(q)
        dense = lambda ret=0: ops.qk_int8_sv_f8_attn(q8, k8, v8, o, qs, ks, vs, vm, 1, 0, qg, kg, sm, 0, ret)
        for mname, bm in _masks(B, H, S).items():
            pairs = _pairs(bm, S)
            os_ = torch.empty_like(q)
            sparse = lambda ret=0: ops.qk_int8_sv_f8_attn_blocksparse(q8, k8, v8, os_, qs, ks, vs, vm, bm, 1, 0, qg, kg, sm, 0, ret)
            case = {"shape": [B, H, S, D], "mask": mname, "visible_fraction": round(pairs / (B * H * S * S), 4)}
            if not a.backward:
                ts, td = _alternate(sparse, dense, a)
                tc = _events(lambda: sab.sageattn_blocksparse(q, k, v, bm), a.steps, a.warmup)
                flops = 4.0 * D * pairs
                case.update(sparse_kernel_ms=round(ts, 3), dense_kernel_ms=round(td, 3), sparse_call_ms=round(tc, 3),
                            sparse_over_dense=round(ts / td, 3), sparse_tflops=round(flops / ts / 1e9, 1))
            else:
                lse_d, lse_s = dense(1), sparse(1)
                dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
                kmv = km
                bs = lambda: ops.qk_int8_attn_bwd_blocksparse(q8, k8, qs, ks, q, k, v, os_, do, lse_s, kmv, dq, dk, dv, bm, 1, 0,
                                                               qg, kg, sm, 0)
                bd = lambda: ops.qk_int8_attn_bwd(q8, k8, qs, ks, q, k, v, o, do, lse_d, kmv, dq, dk, dv, 1, 0, qg, kg, sm, 0)
                ts, td = _alternate(bs, bd, a)
                flops = 10.0 * D * pairs
                case.update(sparse_bwd_kernels_ms=round(ts, 3), dense_bwd_kernels_ms=round(td, 3),
                            sparse_over_dense=round(ts / td, 3), sparse_tflops=round(flops / ts / 1e9, 1),
                            per_kernel_ms={"sparse": _split(bs, a), "dense": _split(bd, a)})
            out["cases"].append(case)
            del bm
        del q, k, v, do, q8, k8, v8, o
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
