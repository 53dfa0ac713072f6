"""Sliding-window attention benchmark: sageattn_window's kernels against the dense INT8+FP8 kernels in the same run.

Workloads (D=128, bf16): B=1, H=32, S=32768 causal with left = 1024 and 4096 (right 0), against the causal dense kernel; B=1,
H=30, S=32768 non-causal with a symmetric +-2048 window, against the non-causal dense kernel.  Per case: the window kernel ms and
the dense kernel ms, timed alternately in the same run (median of --reps rounds of --steps launches after --warmup), the whole
sageattn_window call, the visible query-key pairs, the 128x64 tiles the window kernel visits (and how many of them an edge of
the window crosses, which take the masked path) against the dense kernel's, and 4*D*(visible pairs)/t.  --backward does the same
for the gradient kernels (10*D per pair) against the dense backward's, and splits each backward call into its delta, dQ and dK/dV
kernels (torch.profiler).  Prints one JSON line with the GPU name and power limit.  CUDA events; writes nothing.

    python bench_window.py [--steps 5] [--warmup 2] [--reps 3] [--backward]
"""
import argparse
import json
import statistics

import torch

from bench_blocksparse import _alternate, _events, _gpu, _split

CASES = [  # B, H, S, D, causal, (left, right)
    (1, 32, 32768, 128, True, (1024, 0)),
    (1, 32, 32768, 128, True, (4096, 0)),
    (1, 30, 32768, 128, False, (2048, 2048)),
]


def _visible(S, causal, left, right):
    """(visible query-key pairs, 128x64 tiles visited, of which masked, dense kernel's tiles) of one (b, h)."""
    i = torch.arange(S, dtype=torch.int64)
    lo = (i - left).clamp(min=0) if left >= 0 else torch.zeros_like(i)
    hi = torch.full_like(i, S - 1)
    if right >= 0:
        hi = torch.minimum(hi, i + right)
    if causal:
        hi = torch.minimum(hi, i)
    pairs = int((hi - lo + 1).clamp(min=0).sum())
    tiles = masked = dense = 0
    for r0 in range(0, S, 128):
        r1 = min(r0 + 128, S) - 1
        j_lo, j_hi = int(lo[r0]) // 64, int(hi[r1]) // 64 + 1
        tiles += j_hi - j_lo
        dense += (r1 // 64 + 1) if causal else (S + 63) // 64
        for j in range(j_lo, j_hi):   # a tile is masked when some row of the block does not see all of its keys
            masked += int(bool(((lo[r0:r1 + 1] > 64 * j) | (hi[r0:r1 + 1] < 64 * j + 63)).any()))
    return pairs, tiles, masked, dense


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--backward", action="store_true")
    a = ap.parse_args()
    import sageattention_b200 as sab
    from sageattention_b200 import ops
    from sageattention_b200.core import _quant_qk
    from sageattention_b200.quant import per_channel_fp8

    out = {"metric": "sageattn_window " + ("backward" if a.backward else "forward") + " kernels vs dense", "gpu": _gpu(),
           "dtype": "bf16", "cases": []}
    for B, H, S, D, causal, (left, right) in CASES:
        g = torch.Generator(device="cuda").manual_seed(0)
        q, k, v, do = (torch.randn(B, H, S, D, device="cuda", dtype=torch.bfloat16, generator=g) for _ in range(4))
        sm = D ** -0.5
        c = 1 if causal else 0
        km, q8, qs, k8, ks, qg, kg, _ = _quant_qk(q, k, "fp8", "HND", "per_thread", sm, True, "cuda")
        v8, vs, vm = per_channel_fp8(v, tensor_layout="HND", scale_max=2.25, smooth_v=False)
        o, ow = torch.empty_like(q), torch.empty_like(q)
        dense = lambda ret=0: ops.qk_int8_sv_f8_attn(q8, k8, v8, o, qs, ks, vs, vm, 1, c, qg, kg, sm, 0, ret)
        win = lambda ret=0: ops.qk_int8_sv_f8_attn_window(q8, k8, v8, ow, qs, ks, vs, vm, left, right, 1, c, qg, kg, sm, 0, ret)
        pairs, tiles, masked, dense_tiles = _visible(S, causal, left, right)
        dense_pairs = S * (S + 1) // 2 if causal else S * S
        case = {"shape": [B, H, S, D], "causal": causal, "window": [left, right], "visible_pairs_per_head": pairs,
                "visible_fraction_of_dense": round(pairs / dense_pairs, 4), "tiles_visited_per_head": tiles,
                "masked_tiles_per_head": masked, "tiles_fraction_of_dense": round(tiles / dense_tiles, 4)}
        if not a.backward:
            tw, td = _alternate(win, dense, a)
            tc = _events(lambda: sab.sageattn_window(q, k, v, (left, right), is_causal=causal), a.steps, a.warmup)
            case.update(window_kernel_ms=round(tw, 3), dense_kernel_ms=round(td, 3), window_call_ms=round(tc, 3),
                        window_over_dense=round(tw / td, 4),
                        window_tflops=round(4.0 * D * pairs * B * H / tw / 1e9, 1),
                        dense_tflops=round(4.0 * D * dense_pairs * B * H / td / 1e9, 1))
        else:
            lse_d, lse_w = dense(1), win(1)
            dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
            bw = lambda: ops.qk_int8_attn_bwd_window(q8, k8, qs, ks, q, k, v, ow, do, lse_w, km, dq, dk, dv, left, right, 1, c,
                                                     qg, kg, sm, 0)
            bd = lambda: ops.qk_int8_attn_bwd(q8, k8, qs, ks, q, k, v, o, do, lse_d, km, dq, dk, dv, 1, c, qg, kg, sm, 0)
            tw, td = _alternate(bw, bd, a)
            case.update(window_bwd_kernels_ms=round(tw, 3), dense_bwd_kernels_ms=round(td, 3), window_over_dense=round(tw / td, 4),
                        window_tflops=round(10.0 * D * pairs * B * H / tw / 1e9, 1),
                        dense_tflops=round(10.0 * D * dense_pairs * B * H / td / 1e9, 1),
                        per_kernel_ms={"window": _split(bw, a), "dense": _split(bd, a)})
        out["cases"].append(case)
        del q, k, v, do, q8, k8, v8, o, ow
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
