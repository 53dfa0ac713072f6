"""Block-sparse attention benchmark: sageattn_blocksparse's kernels against the dense INT8+FP8 kernels in the same run.

Workloads: B=4, H=32, S=8192 and B=1, H=30, S=32768 (D=128, bf16, non-causal).  Masks: seeded random block masks at densities
1.0, 0.5, 0.25 and 0.1, and a band ("local window": each 128-query block sees the 64-key blocks within +-1024 keys of it).
Per case: the sparse kernel ms and the dense kernel ms, timed alternately in the same run (median of --reps rounds of --steps
launches after --warmup), the whole sageattn_blocksparse call, the visible fraction and 4*D*(visible query-key pairs)/t.
--backward does the same for the gradient kernels against the dense backward's, and splits each backward call into its delta,
dQ and dK/dV kernels (torch.profiler).  Prints one JSON line with the GPU name and
power limit.  CUDA events; writes nothing.

--varlen: sageattn_varlen_blocksparse's kernels on the packed lengths of bench_varlen_fp8.py (2048, 16384, 4096, 512, 1024, 8192;
Hq=32, Hkv=8, D=128, bf16), non-causal and causal, with seeded masks of densities 1.0, 0.5, 0.25 and 0.1 and a mask from
predict_block_mask_varlen (cdf 0.9, sim 0.3) on seeded video-like data (bench_block_predict.py's generator, one T x H x W grid
per sequence; every case runs on that data).  Three kernels timed in turn in every round: the packed block-sparse kernel, the
packed kernel without a mask (sageattn_varlen_qk_int8_pv_fp8_cuda's) and the dense block-sparse kernel once per sequence on its
mask slice (summed).  Visible pairs are summed over sequences and heads; 4*D*(visible pairs)/t for every kernel, the packed
dense kernel included (it computes more pairs than the mask keeps).  The predictor is timed too (three launches), against
predict_block_mask once per sequence.  --varlen --backward does the same for the gradient kernels (10*D per pair).

    python bench_blocksparse.py [--steps 5] [--warmup 2] [--reps 3] [--backward] [--shapes 8k,32k] [--varlen]
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


VARLEN_LENS = [2048, 16384, 4096, 512, 1024, 8192]   # bench_varlen_fp8.py's packed lengths, in its order
VIDEO_GRIDS = {512: (8, 8, 8), 1024: (4, 16, 16), 2048: (8, 16, 16), 4096: (4, 32, 32), 8192: (8, 32, 32), 16384: (16, 32, 32)}
VARLEN_PREDICT = (0.9, 0.3)                            # cdf_threshold, sim_threshold of the predicted mask


def _varlen_pairs(bm, lens_q, lens_k, causal):
    """Visible query-key pairs of the packed call with block mask bm [nseq or 1, Hq or 1, ., .], summed over sequences and Q heads
    (Q heads of a broadcast mask counted as its expansion to hq = bm.size(1)); causal is top-left inside each sequence."""
    total = 0.0
    for b, (lq, lk) in enumerate(zip(lens_q, lens_k)):
        if lq == 0 or lk == 0:
            continue
        nq, nk = (lq + 127) // 128, (lk + 63) // 64
        i = torch.arange(lq, dtype=torch.float64)[:, None]
        k0 = torch.arange(nk, dtype=torch.float64)[None, :] * 64
        hi = torch.full_like(i, float(lk)).expand(lq, nk)
        if causal:
            hi = torch.minimum(hi, i + 1)
        per_row = (torch.minimum(hi, k0 + 64) - k0).clamp(min=0)                        # [lq, nk] visible keys of each tile
        per_tile = torch.nn.functional.pad(per_row, (0, 0, 0, nq * 128 - lq)).view(nq, 128, nk).sum(1)
        total += float((bm[min(b, bm.size(0) - 1), :, :nq, :nk].double().cpu() * per_tile).sum())
    return total


def _packed_video(lens, H, D, g):
    """Packed [T,H,D] q, k, v of bench_block_predict._video_like, one grid per sequence (VIDEO_GRIDS)."""
    from bench_block_predict import _video_like
    parts = [_video_like(1, H, L, D, VIDEO_GRIDS[L], g) for L in lens]
    return [torch.cat([p[i][0].transpose(0, 1) for p in parts]).contiguous() for i in range(3)]


def main_varlen(a):
    import sageattention_b200 as sab
    from sageattention_b200 import ops, quant as Q
    from sageattention_b200.core import _quant_qk, _quant_qk_varlen_f8
    from sageattention_b200._capi import SAB_GRAN_PER_THREAD as PT
    from bench_window import _alternate_all

    lens, Hq, Hkv, D = VARLEN_LENS, 32, 8, 128
    out = {"metric": "sageattn_varlen_blocksparse " + ("backward" if a.backward else "forward") +
           " kernels vs packed dense and per-sequence block-sparse", "gpu": _gpu(), "dtype": "bf16", "seqlens": lens, "Hq": Hq,
           "Hkv": Hkv, "D": D, "data": "video-like (seeded)", "cases": []}
    cu = torch.tensor([0] + torch.tensor(lens).cumsum(0).tolist(), dtype=torch.int32, device="cuda")
    L = max(lens)
    spans = [(int(cu[i]), int(cu[i + 1])) for i in range(len(lens))]
    nq, nk = (L + 127) // 128, (L + 63) // 64
    g = torch.Generator(device="cuda").manual_seed(0)
    q, _, _ = _packed_video(lens, Hq, D, g)
    _, k, v = _packed_video(lens, Hkv, D, g)
    do = torch.randn(q.shape, device="cuda", dtype=torch.bfloat16, generator=g)
    sm = D ** -0.5
    km, q8, qs, cqs, k8, ks, cks = _quant_qk_varlen_f8(q, k, cu, cu, L, L, "per_thread", True)
    v8, vs, vm, cpad = Q.per_channel_fp8_varlen_seq(v, cu, L, 2.25)
    osp, od = torch.empty_like(q), torch.empty_like(q)
    dense = []   # each sequence's dense operands (NHD, batch 1)
    for s, e in spans:
        qb, kb, vb = q[s:e][None], k[s:e][None], v[s:e][None]
        kmb, q8d, qsd, k8d, ksd, _, _, _ = _quant_qk(qb, kb, "fp8", "NHD", "per_thread", sm, True, "cuda")
        v8d, vsd, _ = Q.per_channel_fp8(vb, "NHD", 2.25, False)
        dense.append((qb, kb, vb, do[s:e][None], kmb, q8d, qsd, k8d, ksd, v8d, vsd, torch.empty_like(qb)))
    for causal in (False, True):
        c = int(causal)
        gm = torch.Generator(device="cuda").manual_seed(1)
        masks = {f"random_{p}": torch.rand(len(lens), Hq, nq, nk, generator=gm, device="cuda") < p for p in (1.0, 0.5, 0.25, 0.1)}
        pkw = dict(cdf_threshold=VARLEN_PREDICT[0], sim_threshold=VARLEN_PREDICT[1], is_causal=causal)
        masks["predicted"] = sab.predict_block_mask_varlen(q, k, cu, cu, L, L, **pkw)
        pred_ms = _events(lambda: sab.predict_block_mask_varlen(q, k, cu, cu, L, L, **pkw), a.steps, a.warmup)
        pred_seq_ms = _events(lambda: [sab.predict_block_mask(d[0], d[1], tensor_layout="NHD", **pkw) for d in dense], a.steps, a.warmup)
        out.setdefault("predictor", []).append({"causal": causal, "cdf_threshold": VARLEN_PREDICT[0],
                                                "sim_threshold": VARLEN_PREDICT[1], "packed_ms": round(pred_ms, 3),
                                                "per_sequence_ms": round(pred_seq_ms, 3)})
        dense_pairs = _varlen_pairs(torch.ones(1, Hq, nq, nk, dtype=torch.bool), lens, lens, causal)
        for mname, bm in masks.items():
            pairs = _varlen_pairs(bm, lens, lens, causal)
            sl = [bm[b:b + 1, :, :(e - s + 127) // 128, :(e - s + 63) // 64] for b, (s, e) in enumerate(spans)]
            sparse = lambda ret=0: ops.qk_int8_sv_f8_attn_varlen_blocksparse(q8, k8, v8, osp, qs, ks, vs, None, cu, cu, cpad, cqs, cks, L,
                                                                             L, bm, c, PT, PT, sm, ret)
            packed = lambda ret=0: ops.qk_int8_sv_f8_attn_varlen_seq(q8, k8, v8, od, qs, ks, vs, None, cu, cu, cpad, cqs, cks, L, c, PT,
                                                                    PT, sm, ret)
            per_seq = lambda ret=0: [ops.qk_int8_sv_f8_attn_blocksparse(d[5], d[7], d[9], d[11], d[6], d[8], d[10], None, m, 0, c, PT,
                                                                        PT, sm, 0, ret) for d, m in zip(dense, sl)]
            case = {"causal": causal, "mask": mname, "visible_pairs": pairs, "visible_fraction_of_dense": round(pairs / dense_pairs, 4)}
            per = 10.0 if a.backward else 4.0
            if not a.backward:
                t = _alternate_all({"packed_sparse": sparse, "packed_dense": packed, "per_sequence_sparse": per_seq}, a)
                tc = _events(lambda: sab.sageattn_varlen_blocksparse(q, k, v, cu, cu, L, L, bm, is_causal=causal), a.steps, a.warmup)
                case["packed_sparse_call_ms"] = round(tc, 3)
            else:
                lsp, lpk, lps = sparse(1), packed(1), per_seq(1)
                gq, gk, gv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
                bsp = lambda: ops.qk_int8_attn_bwd_varlen_blocksparse(q8, k8, qs, ks, q, k, v, osp, do, lsp, km, gq, gk, gv, cu, cu, cqs,
                                                                      cks, L, L, bm, c, PT, PT, sm)
                bpk = lambda: ops.qk_int8_attn_bwd_varlen_seq(q8, k8, qs, ks, q, k, v, od, do, lpk, km, gq, gk, gv, cu, cu, cqs, cks, L,
                                                              L, c, PT, PT, sm)
                grads = [tuple(torch.empty_like(x) for x in d[:3]) for d in dense]
                bps = lambda: [ops.qk_int8_attn_bwd_blocksparse(d[5], d[7], d[6], d[8], d[0], d[1], d[2], d[11], d[3], l, d[4], *gr, m,
                                                                0, c, PT, PT, sm, 0) for d, l, gr, m in zip(dense, lps, grads, sl)]
                t = _alternate_all({"packed_sparse": bsp, "packed_dense": bpk, "per_sequence_sparse": bps}, a)
                case["per_kernel_ms"] = {"packed_sparse": _split(bsp, a), "packed_dense": _split(bpk, a)}
            for n, tn in t.items():
                case[f"{n}_ms"] = round(tn, 3)
                case[f"{n}_tflops_visible"] = round(per * D * pairs / tn / 1e9, 1)
            case["packed_sparse_over_packed_dense"] = round(t["packed_sparse"] / t["packed_dense"], 4)
            case["packed_sparse_over_per_sequence"] = round(t["packed_sparse"] / t["per_sequence_sparse"], 4)
            out["cases"].append(case)
    print(json.dumps(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--backward", action="store_true")
    ap.add_argument("--shapes", default="8k,32k")
    ap.add_argument("--varlen", action="store_true")
    a = ap.parse_args()
    if a.varlen:
        return main_varlen(a)
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
