"""Block-mask predictor benchmark: predict_block_mask's cost and what its masks buy sageattn_blocksparse.

Workloads: B=4, H=32, S=8192 and B=1, H=30, S=32768 (D=128, bf16, non-causal).  Data, both seeded: Gaussian q, k, v, and a
synthetic "video-like" generator that puts the tokens on a T x H x W grid (8x32x32 and 8x64x64) and makes q and k smooth random
functions of the position (random Fourier features of low frequency, plus a per-head common part) plus noise.  Accuracy figures are for this synthetic data
only.  Per (cdf_threshold, sim_threshold) pair: the predictor's ms (CUDA events, the whole call: two statistics launches and one
selection launch) and its selection launch alone, the mask density, the sparse kernel with the predicted mask against the dense
kernel (alternated in one run, median of --reps rounds of --steps launches after --warmup), and the relative L2 error of the
sageattn_blocksparse output against the dense call's.  Prints one JSON line with the GPU name and power limit; writes nothing.

    python bench_block_predict.py [--steps 5] [--warmup 2] [--reps 3] [--shapes 8k,32k]
"""
import argparse
import json

import torch

from bench_blocksparse import _alternate, _events, _gpu

SHAPES = {"8k": (4, 32, 8192, 128, (8, 32, 32)), "32k": (1, 30, 32768, 128, (8, 64, 64))}
PAIRS = [(0.5, 0.3), (0.7, 0.3), (0.9, 0.3), (0.95, 0.5), (0.9, -1.0)]


def _gaussian(B, H, S, D, g):
    return [torch.randn(B, H, S, D, device="cuda", generator=g).to(torch.bfloat16) for _ in range(3)]


def _video_like(B, H, S, D, grid, g, nfeat=16, noise=0.3, offset=0.5):
    T, Hh, W = grid
    assert T * Hh * W == S
    t, y, x = torch.meshgrid(torch.arange(T, device="cuda"), torch.arange(Hh, device="cuda"), torch.arange(W, device="cuda"),
                             indexing="ij")
    pos = torch.stack([t.flatten() / T, y.flatten() / Hh, x.flatten() / W], -1).float()          # [S, 3] in [0, 1)
    out = []
    for _ in range(3):
        freq = torch.randn(3, nfeat, device="cuda", generator=g) * 6.0                              # a few cycles per axis
        phase = torch.rand(nfeat, device="cuda", generator=g) * 6.2832
        feat = torch.sin(pos @ freq + phase)                                                          # [S, nfeat]
        coef = torch.randn(B, H, nfeat, D, device="cuda", generator=g) / nfeat ** 0.5
        base = offset * torch.randn(B, H, 1, D, device="cuda", generator=g)                        # a per-head common part
        x_ = base + feat @ coef + noise * torch.randn(B, H, S, D, device="cuda", generator=g)
        out.append(x_.to(torch.bfloat16))
        del x_
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--shapes", default="8k,32k")
    a = ap.parse_args()
    import sageattention_b200 as sab
    from sageattention_b200 import ops
    from sageattention_b200.core import _quant_qk
    from sageattention_b200.quant import per_channel_fp8

    out = {"metric": "predict_block_mask cost and sageattn_blocksparse with predicted masks", "gpu": _gpu(), "dtype": "bf16",
           "causal": False, "data": "synthetic (seeded)", "cases": []}
    for sname in a.shapes.split(","):
        B, H, S, D, grid = SHAPES[sname]
        sm = D ** -0.5
        for dname in ("gaussian", "video_like"):
            g = torch.Generator(device="cuda").manual_seed(0)
            q, k, v = _gaussian(B, H, S, D, g) if dname == "gaussian" else _video_like(B, H, S, D, grid, g)
            km, q8, qs, k8, ks, qg, kg, _ = _quant_qk(q, k, "fp8", "HND", "per_thread", sm, True, "cuda")
            v8, vs, vm = per_channel_fp8(v, tensor_layout="HND", scale_max=2.25, smooth_v=False)
            o_kernel = torch.empty_like(q)
            dense = lambda: ops.qk_int8_sv_f8_attn(q8, k8, v8, o_kernel, qs, ks, vs, vm, 1, 0, qg, kg, sm, 0, 0)
            o_dense = sab.sageattn_qk_int8_pv_fp8_cuda(q, k, v).float()
            # the selection launch alone, on statistics computed once
            nq, nk = (S + 127) // 128, (S + 63) // 64
            f32 = dict(dtype=torch.float32, device="cuda")
            qm_, qs_ = torch.empty(B, H, nq, D, **f32), torch.empty(B, H, nq, **f32)
            km_, ks_ = torch.empty(B, H, nk, D, **f32), torch.empty(B, H, nk, **f32)
            ops.block_stats(q, qm_, qs_, 1, 128)
            ops.block_stats(k, km_, ks_, 1, 64)
            stats_ms = _events(lambda: (ops.block_stats(q, qm_, qs_, 1, 128), ops.block_stats(k, km_, ks_, 1, 64)), a.steps,
                               a.warmup)
            for cdf, simt in PAIRS:
                kw = dict(cdf_threshold=cdf, sim_threshold=simt)
                bm = sab.predict_block_mask(q, k, **kw)
                pred_ms = _events(lambda: sab.predict_block_mask(q, k, **kw), a.steps, a.warmup)
                bm2 = torch.empty_like(bm)
                sel_ms = _events(lambda: ops.predict_block_mask(qm_, qs_, km_, ks_, bm2, S, S, 0, sm, cdf, simt), a.steps, a.warmup)
                assert torch.equal(bm, bm2)
                os_ = torch.empty_like(q)
                sparse = lambda: ops.qk_int8_sv_f8_attn_blocksparse(q8, k8, v8, os_, qs, ks, vs, vm, bm, 1, 0, qg, kg, sm, 0, 0)
                ts, td = _alternate(sparse, dense, a)
                o_sparse = sab.sageattn_blocksparse(q, k, v, bm).float()
                rel = ((o_sparse - o_dense).norm() / o_dense.norm()).item()
                out["cases"].append({
                    "shape": [B, H, S, D], "data": dname, "cdf_threshold": cdf, "sim_threshold": simt,
                    "density": round(bm.float().mean().item(), 4),
                    "predictor_ms": round(pred_ms, 3), "stats_ms": round(stats_ms, 3), "select_ms": round(sel_ms, 3),
                    "sparse_kernel_ms": round(ts, 3), "dense_kernel_ms": round(td, 3),
                    "predictor_over_dense": round(pred_ms / td, 4), "sparse_over_dense": round(ts / td, 3),
                    "rel_l2_vs_dense": float(f"{rel:.3e}")})
                del bm, bm2, o_sparse, os_
            del q, k, v, q8, k8, v8, o_kernel, o_dense
            torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
