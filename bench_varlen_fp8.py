"""Packed INT8+FP8 attention at BASELINE.json configs[3] (GQA Hq=32 / Hkv=8, D=128, bf16, lengths 512..16384 shuffled with seed 0):
sageattn_varlen_qk_int8_pv_fp8_cuda against sageattn_varlen's FP16-PV kernel and the dense INT8+FP8 kernel run per sequence
(summed).  The three are timed in alternation (CUDA events, median of --reps rounds of --iters launches each).  TFLOP/s count
4*Hq*D per visible query-key pair (causal: key <= query inside each sequence).  --backward times the gradient kernels instead
(varlen-seq vs sageattn_varlen's vs the dense per-sequence ones).  Prints one JSON line with the GPU name and power limit."""
import argparse, json, statistics, subprocess
import torch

import sageattention_b200 as sab
from sageattention_b200 import ops, quant as Q
from sageattention_b200.core import _quant_qk_varlen_f8, _quant_qk_varlen, _quant_qk, _attn_varlen_f8, _attn_varlen
from sageattention_b200._capi import SAB_GRAN_PER_THREAD as PT


def _power_limit():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True,
                           text=True, timeout=30)
        return float(r.stdout.strip().splitlines()[0])
    except Exception:
        return None


def _ms(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--backward", action="store_true")
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    lens = [512, 1024, 2048, 4096, 8192, 16384]
    g = torch.Generator().manual_seed(0)
    lens = [lens[i] for i in torch.randperm(len(lens), generator=g).tolist()]
    Hq, Hkv, D, dt = 32, 8, 128, torch.bfloat16
    cu = torch.tensor([0] + torch.tensor(lens).cumsum(0).tolist(), dtype=torch.int32, device=dev)
    T, L = int(cu[-1]), max(lens)
    q, do = (torch.randn(T, Hq, D, device=dev, dtype=dt) for _ in range(2))
    k, v = (torch.randn(T, Hkv, D, device=dev, dtype=dt) for _ in range(2))
    spans = [(int(cu[i]), int(cu[i + 1])) for i in range(len(lens))]
    res = {"gpu": torch.cuda.get_device_name(dev), "power_limit_w": _power_limit(), "config": "configs[3]", "seqlens": lens,
           "Hq": Hq, "Hkv": Hkv, "D": D, "dtype": "bf16", "backward": a.backward, "iters": a.iters, "reps": a.reps}
    sm = D ** -0.5
    for causal in (False, True):
        fl = sum(4.0 * Hq * D * (Ls * (Ls + 1) / 2 if causal else Ls * Ls) for Ls in lens) * (2.5 if a.backward else 1.0)
        c = int(causal)
        # operands of the three kernels, prepared once
        km, q8, qs, cqs, k8, ks, cks = _quant_qk_varlen_f8(q, k, cu, cu, L, L, "per_thread", True)
        v8, vs, _, cpad = Q.per_channel_fp8_varlen_seq(v, cu, L, 2.25)
        o = torch.empty_like(q)
        _, q8b, qsb, k8b, ksb, cqb, ckb = _quant_qk_varlen(q, k, cu, cu, L, L, sm, True)
        vt, cpad16 = Q.transpose_v_f16_varlen(v, cu, L)
        dense = []
        for s, e in spans:
            qb, kb, vb, dob = q[s:e][None], k[s:e][None], v[s:e][None], do[s:e][None]
            kmb, q8d, qsd, k8d, ksd, _, _, _ = _quant_qk(qb, kb, "fp8", "NHD", "per_thread", sm, True, "cuda")
            v8d, vsd, _ = Q.per_channel_fp8(vb, "NHD", 2.25, False)
            dense.append((qb, kb, vb, dob, kmb, q8d, qsd, k8d, ksd, v8d, vsd, torch.empty_like(qb)))
        if not a.backward:
            kern = {
                "varlen_fp8": lambda: ops.qk_int8_sv_f8_attn_varlen_seq(q8, k8, v8, o, qs, ks, vs, None, cu, cu, cpad, cqs, cks, L, c, PT,
                                                                        PT, sm, 0),
                "varlen_fp16pv": lambda: ops.qk_int8_sv_f16_attn_varlen(q8b, k8b, vt, o, qsb, ksb, cu, cu, cpad16, cqb, ckb, L, c, sm, 1, 0),
                "dense_fp8_per_seq": lambda: [ops.qk_int8_sv_f8_attn(d[5], d[7], d[9], d[11], d[6], d[8], d[10], None, 0, c, PT, PT, sm, 0, 0)
                                              for d in dense],
            }
            call = {
                "varlen_fp8": lambda: sab.sageattn_varlen_qk_int8_pv_fp8_cuda(q, k, v, cu, cu, L, L, is_causal=causal),
                "varlen_fp16pv": lambda: sab.sageattn_varlen(q, k, v, cu, cu, L, L, is_causal=causal),
                "dense_fp8_per_seq": lambda: [sab.sageattn_qk_int8_pv_fp8_cuda(d[0], d[1], d[2], tensor_layout="NHD", is_causal=causal)
                                              for d in dense],
            }
        else:
            o1, lse1, _ = _attn_varlen_f8(q, k, v, cu, cu, L, L, causal, "per_thread", sm, True, False, 2.25, True)
            o2, lse2 = _attn_varlen(q, k, v, cu, cu, L, L, causal, sm, True, True)
            lses = []
            for d in dense:
                lses.append(ops.qk_int8_sv_f8_attn(d[5], d[7], d[9], d[11], d[6], d[8], d[10], None, 0, c, PT, PT, sm, 0, 1))
            gq, gk, gv = torch.zeros_like(q), torch.zeros_like(k), torch.zeros_like(v)
            kern = {
                "varlen_fp8": lambda: ops.qk_int8_attn_bwd_varlen_seq(q8, k8, qs, ks, q, k, v, o1, do, lse1, km, gq, gk, gv, cu, cu, cqs, cks,
                                                                      L, L, c, PT, PT, sm),
                "varlen_fp16pv": lambda: ops.qk_int8_attn_bwd_varlen(q8b, k8b, qsb, ksb, q, k, v, o2, do, lse2, None, gq, gk, gv, cu, cu,
                                                                     cqb, ckb, L, L, c, sm, 1),
                "dense_fp8_per_seq": lambda: [ops.qk_int8_attn_bwd(d[5], d[7], d[6], d[8], d[0], d[1], d[2], d[11], d[3], l, d[4],
                                                                   torch.empty_like(d[0]), torch.empty_like(d[1]), torch.empty_like(d[2]), 0,
                                                                   c, PT, PT, sm, 0) for d, l in zip(dense, lses)],
            }
            call = None
        times = {n: [] for n in kern}
        ctimes = {n: [] for n in kern}
        for fn in list(kern.values()) + (list(call.values()) if call else []):
            fn()
        torch.cuda.synchronize()
        for _ in range(a.reps):
            for n in kern:
                times[n].append(_ms(kern[n], a.iters))
                if call:
                    ctimes[n].append(_ms(call[n], a.iters))
        tag = "causal" if causal else "noncausal"
        for n in kern:
            km_ = statistics.median(times[n])
            res[f"{tag}_{n}_kernel_ms"] = round(km_, 4)
            res[f"{tag}_{n}_kernel_tflops"] = round(fl / km_ / 1e9, 1)
            if call:
                cm_ = statistics.median(ctimes[n])
                res[f"{tag}_{n}_call_ms"] = round(cm_, 4)
                res[f"{tag}_{n}_call_tflops"] = round(fl / cm_ / 1e9, 1)
        del dense
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
