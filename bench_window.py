"""Sliding-window attention benchmark: sageattn_window's kernels against the dense INT8+FP8 kernels in the same run.

Workloads (D=128, bf16): B=1, H=32, S=32768 causal with left = 1024 and 4096 (right 0), against the causal dense kernel; B=1,
H=30, S=32768 non-causal with a symmetric +-2048 window, against the non-causal dense kernel.  Per case: the window kernel ms and
the dense kernel ms, timed alternately in the same run (median of --reps rounds of --steps launches after --warmup), the whole
sageattn_window call, the visible query-key pairs, the 128x64 tiles the window kernel visits (and how many of them an edge of
the window crosses, which take the masked path) against the dense kernel's, and 4*D*(visible pairs)/t.  --backward does the same
for the gradient kernels (10*D per pair) against the dense backward's, and splits each backward call into its delta, dQ and dK/dV
kernels (torch.profiler).  Prints one JSON line with the GPU name and power limit.  CUDA events; writes nothing.

--varlen: sageattn_varlen_window's kernels on the packed lengths of bench_varlen_fp8.py (2048, 16384, 4096, 512, 1024, 8192;
Hq=32, Hkv=8, D=128, bf16) with the same three windows (Hq=32 for all three), against the packed kernel without a window
(sageattn_varlen_qk_int8_pv_fp8_cuda's) and the dense window kernels run once per sequence (summed), all three timed alternately
in the same run.  Visible pairs and tiles are summed over the sequences; 4*Hq*D*(visible pairs)/t for every kernel, the packed
dense kernel included (it computes more pairs than the window keeps).  --varlen --backward does the same for the gradient kernels
(10*Hq*D per pair).

    python bench_window.py [--steps 5] [--warmup 2] [--reps 3] [--backward] [--varlen]
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


VARLEN_LENS = [2048, 16384, 4096, 512, 1024, 8192]   # bench_varlen_fp8.py's packed lengths, in its order
VARLEN_WINDOWS = [(True, (1024, 0)), (True, (4096, 0)), (False, (2048, 2048))]


def _visible_varlen(lens, causal, left, right):
    """_visible summed over packed sequences (Lq == Lk): (pairs, tiles, masked, dense tiles) of one head."""
    return tuple(sum(x) for x in zip(*(_visible(L, causal, left, right) for L in lens)))


def _alternate_all(fns, a):
    """Median ms of each function of fns, timed in turn in every round (as _alternate does for two)."""
    ts = {n: [] for n in fns}
    for _ in range(a.reps):
        for n, f in fns.items():
            ts[n].append(_events(f, a.steps, a.warmup))
    return {n: statistics.median(t) for n, t in ts.items()}


def main_varlen(a):
    import sageattention_b200 as sab
    from sageattention_b200 import ops, quant as Q
    from sageattention_b200.core import _quant_qk, _quant_qk_varlen_f8
    from sageattention_b200._capi import SAB_GRAN_PER_THREAD as PT

    lens, Hq, Hkv, D = VARLEN_LENS, 32, 8, 128
    out = {"metric": "sageattn_varlen_window " + ("backward" if a.backward else "forward") + " kernels vs packed dense and per-sequence",
           "gpu": _gpu(), "dtype": "bf16", "seqlens": lens, "Hq": Hq, "Hkv": Hkv, "D": D, "cases": []}
    cu = torch.tensor([0] + torch.tensor(lens).cumsum(0).tolist(), dtype=torch.int32, device="cuda")
    T, L = int(cu[-1]), max(lens)
    spans = [(int(cu[i]), int(cu[i + 1])) for i in range(len(lens))]
    g = torch.Generator(device="cuda").manual_seed(0)
    q, do = (torch.randn(T, Hq, D, device="cuda", dtype=torch.bfloat16, generator=g) for _ in range(2))
    k, v = (torch.randn(T, Hkv, D, device="cuda", dtype=torch.bfloat16, generator=g) for _ in range(2))
    sm = D ** -0.5
    km, q8, qs, cqs, k8, ks, cks = _quant_qk_varlen_f8(q, k, cu, cu, L, L, "per_thread", True)
    v8, vs, vm, cpad = Q.per_channel_fp8_varlen_seq(v, cu, L, 2.25)
    ow, od = torch.empty_like(q), torch.empty_like(q)
    dense = []   # each sequence's dense operands (NHD, batch 1)
    for s, e in spans:
        qb, kb, vb = q[s:e][None], k[s:e][None], v[s:e][None]
        kmb, q8d, qsd, k8d, ksd, _, _, _ = _quant_qk(qb, kb, "fp8", "NHD", "per_thread", sm, True, "cuda")
        v8d, vsd, _ = Q.per_channel_fp8(vb, "NHD", 2.25, False)
        dense.append((qb, kb, vb, do[s:e][None], kmb, q8d, qsd, k8d, ksd, v8d, vsd, torch.empty_like(qb)))
    for causal, (left, right) in VARLEN_WINDOWS:
        c = int(causal)
        win = lambda ret=0: ops.qk_int8_sv_f8_attn_varlen_window(q8, k8, v8, ow, qs, ks, vs, None, cu, cu, cpad, cqs, cks, L, left, right,
                                                                c, PT, PT, sm, ret)
        packed = lambda ret=0: ops.qk_int8_sv_f8_attn_varlen_seq(q8, k8, v8, od, qs, ks, vs, None, cu, cu, cpad, cqs, cks, L, c, PT, PT,
                                                                sm, ret)
        per_seq = lambda ret=0: [ops.qk_int8_sv_f8_attn_window(d[5], d[7], d[9], d[11], d[6], d[8], d[10], None, left, right, 0, c, PT,
                                                               PT, sm, 0, ret) for d in dense]
        pairs, tiles, masked, dense_tiles = _visible_varlen(lens, causal, left, right)
        dense_pairs = sum(Ls * (Ls + 1) // 2 if causal else Ls * Ls for Ls in lens)
        case = {"causal": causal, "window": [left, right], "visible_pairs_per_head": pairs,
                "visible_fraction_of_dense": round(pairs / dense_pairs, 4), "tiles_visited_per_head": tiles,
                "masked_tiles_per_head": masked, "tiles_fraction_of_dense": round(tiles / dense_tiles, 4)}
        per = 10.0 if a.backward else 4.0
        if not a.backward:
            t = _alternate_all({"packed_window": win, "packed_dense": packed, "per_sequence_window": per_seq}, a)
            tc = _events(lambda: sab.sageattn_varlen_window(q, k, v, cu, cu, L, L, (left, right), is_causal=causal), a.steps, a.warmup)
            case["packed_window_call_ms"] = round(tc, 3)
        else:
            lw, ld, ls = win(1), packed(1), per_seq(1)
            gq, gk, gv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
            bw = lambda: ops.qk_int8_attn_bwd_varlen_window(q8, k8, qs, ks, q, k, v, ow, do, lw, km, gq, gk, gv, cu, cu, cqs, cks, L, L,
                                                            left, right, c, PT, PT, sm)
            bd = lambda: ops.qk_int8_attn_bwd_varlen_seq(q8, k8, qs, ks, q, k, v, od, do, ld, km, gq, gk, gv, cu, cu, cqs, cks, L, L, c,
                                                         PT, PT, sm)
            grads = [tuple(torch.empty_like(x) for x in d[:3]) for d in dense]
            bs = lambda: [ops.qk_int8_attn_bwd_window(d[5], d[7], d[6], d[8], d[0], d[1], d[2], d[11], d[3], l, d[4], *gr, left, right, 0,
                                                      c, PT, PT, sm, 0) for d, l, gr in zip(dense, ls, grads)]
            t = _alternate_all({"packed_window": bw, "packed_dense": bd, "per_sequence_window": bs}, a)
            case["per_kernel_ms"] = {"packed_window": _split(bw, a), "packed_dense": _split(bd, a)}
        for n, tn in t.items():
            case[f"{n}_ms"] = round(tn, 3)
            case[f"{n}_tflops_visible"] = round(per * Hq * D * pairs / tn / 1e9, 1)
        case["packed_window_over_per_sequence"] = round(t["packed_window"] / t["per_sequence_window"], 4)
        case["packed_window_over_packed_dense"] = round(t["packed_window"] / t["packed_dense"], 4)
        out["cases"].append(case)
    print(json.dumps(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--backward", action="store_true")
    ap.add_argument("--varlen", action="store_true")
    a = ap.parse_args()
    if a.varlen:
        return main_varlen(a)
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
