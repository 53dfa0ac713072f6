"""Backward benchmark: forward + backward of sageattn at the headline shape (B=4, H=32, S=8192, D=128, bf16), non-causal and
causal, on one GPU.  Prints one JSON line with, per mode:
  * bwd_kernel: the gradient kernels alone (sab_qk_int8_attn_bwd on quantised operands prepared once), ms and TFLOP/s counting
    10*B*H*S^2*D algorithmic FLOPs (halved for causal; the two-kernel design's recompute of S and dP is not counted);
  * bwd_call: the whole backward of sageattn (o.backward(dO): Q/K quantiser recompute + gradient kernels);
  * fwd_bwd: forward + backward of sageattn;
  * sdpa_flash_bwd: torch SDPA's flash-attention backward on the same inputs, for context;
and the GPU name and power limit.  CUDA events after warm-up; writes nothing.

--varlen: the same for sageattn_varlen on a packed GQA batch (lens 4096, 512, 16384, 1024, 8192, 2048; Hq=32, Hkv=8, D=128, bf16),
non-causal and causal, counting 10*Hq*D*sum(Lq*Lk) FLOPs (only the visible pairs for causal), with the sum of per-sequence torch
SDPA flash backwards for context.

--masked: the same for sageattn_qk_int8_pv_fp16_triton with attn_mask (B=1, H=32, S=8192, D=128, bf16, non-causal, 10*B*H*S^2*D
FLOPs whatever the mask hides): (a) a bool mask [1,1,S,S] and (b) a bias [1,H,S,S] that requires grad, so the kernels also write
the dense dBias.  For context, torch SDPA's memory-efficient backward on the same inputs with the same mask as a float additive
mask (False -> -inf for (a); bias*ln2, requiring grad, for (b))."""
import argparse
import json
import subprocess

import torch
import torch.nn.functional as F


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
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        pl, clk = (x.strip() for x in r.stdout.strip().split(","))
        return {"name": name, "power_limit_w": float(pl), "sm_max_mhz": float(clk)}
    except Exception as e:  # the figures are still stated next to the numbers, as unknown
        return {"name": name, "power_limit_w": None, "error": str(e)}


VARLEN_LENS = [4096, 512, 16384, 1024, 8192, 2048]


def varlen(a):
    import numpy as np
    import sageattention_b200 as sab
    from sageattention_b200 import ops
    from sageattention_b200.quant import per_block_int8_varlen, transpose_v_f16_varlen

    lens, Hq, Hkv, D = VARLEN_LENS, 32, 8, 128
    T, L = sum(lens), max(lens)
    dt = torch.bfloat16
    g = torch.Generator(device="cuda").manual_seed(0)
    q, do = (torch.randn(T, Hq, D, device="cuda", dtype=dt, generator=g) for _ in range(2))
    k, v = (torch.randn(T, Hkv, D, device="cuda", dtype=dt, generator=g) for _ in range(2))
    cu = torch.tensor([0] + list(np.cumsum(lens)), dtype=torch.int32, device="cuda")
    sm = D ** -0.5
    out = {"metric": "sageattn_varlen backward", "shape": {"lens": lens, "Hq": Hq, "Hkv": Hkv, "D": D, "dtype": "bf16"},
           "gpu": _gpu()}
    for causal in (False, True):
        pairs = sum(n * (n + 1) // 2 if causal else n * n for n in lens)
        flops = 10.0 * Hq * D * pairs
        # kernels alone, on the operands sageattn_varlen's forward uses
        km = sab.k_mean(k.unsqueeze(0), "NHD").view(Hkv, D)
        q8, qs, k8, ks, cqs, cks = per_block_int8_varlen(q, k, cu, cu, L, L, sm_scale=sm, km=km)
        v_t, cu_pad = transpose_v_f16_varlen(v, cu, L)
        o = torch.empty_like(q)
        lse = ops.qk_int8_sv_f16_attn_varlen(q8, k8, v_t, o, qs, ks, cu, cu, cu_pad, cqs, cks, L, int(causal), sm, 1, 1)
        dq, dk, dv = torch.zeros_like(q), torch.zeros_like(k), torch.zeros_like(v)
        t_kern = _events(lambda: ops.qk_int8_attn_bwd_varlen(q8, k8, qs, ks, q, k, v, o, do, lse, km, dq, dk, dv, cu, cu, cqs, cks,
                                                             L, L, int(causal), sm, 1), a.steps, a.warmup)
        # the public call
        qg, kg, vg = (t.clone().requires_grad_(True) for t in (q, k, v))

        def fwd_bwd():
            qg.grad = kg.grad = vg.grad = None
            sab.sageattn_varlen(qg, kg, vg, cu, cu, L, L, is_causal=causal).backward(do)

        t_fb = _events(fwd_bwd, a.steps, a.warmup)
        ob = sab.sageattn_varlen(qg, kg, vg, cu, cu, L, L, is_causal=causal)
        t_bwd = _events(lambda: torch.autograd.grad(ob, (qg, kg, vg), do, retain_graph=True), a.steps, a.warmup)
        # torch SDPA flash backward of each sequence alone (K / V heads repeated to Hq outside the timed region)
        seqs = []
        with torch.nn.attention.sdpa_kernel(torch.nn.attention.SDPBackend.FLASH_ATTENTION):
            for i in range(len(lens)):
                s = slice(int(cu[i]), int(cu[i + 1]))
                qi = q[s].transpose(0, 1).unsqueeze(0).detach().requires_grad_(True)
                ki, vi = (t[s].transpose(0, 1).repeat_interleave(Hq // Hkv, 0).unsqueeze(0).detach().requires_grad_(True)
                          for t in (k, v))
                oi = F.scaled_dot_product_attention(qi, ki, vi, is_causal=causal)
                seqs.append((oi, (qi, ki, vi), do[s].transpose(0, 1).unsqueeze(0)))

            def sdpa_bwd():
                for oi, ins, doi in seqs:
                    torch.autograd.grad(oi, ins, doi, retain_graph=True)

            t_sdpa = _events(sdpa_bwd, a.steps, a.warmup)
        out["causal" if causal else "non_causal"] = {
            "bwd_kernel": {"ms": round(t_kern, 3), "tflops": round(flops / t_kern / 1e9, 1)},
            "bwd_call": {"ms": round(t_bwd, 3), "tflops": round(flops / t_bwd / 1e9, 1)},
            "fwd_bwd": {"ms": round(t_fb, 3)},
            "sdpa_flash_bwd_per_sequence": {"ms": round(t_sdpa, 3), "tflops": round(flops / t_sdpa / 1e9, 1)},
        }
        del ob, seqs
    print(json.dumps(out))


def masked(a):
    import math
    import sageattention_b200 as sab
    from sageattention_b200 import ops

    B, H, S, D = 1, 32, 8192, 128
    dt = torch.bfloat16
    g = torch.Generator(device="cuda").manual_seed(0)
    q, k, v, do = (torch.randn(B, H, S, D, device="cuda", dtype=dt, generator=g) for _ in range(4))
    sm = D ** -0.5
    flops = 10.0 * B * H * S * S * D
    out = {"metric": "sageattn_qk_int8_pv_fp16_triton masked backward", "shape": {"B": B, "H": H, "S": S, "D": D, "dtype": "bf16"},
           "gpu": _gpu()}
    masks = {
        "bool_1_1_S_S": torch.rand(1, 1, S, S, device="cuda", generator=g) > 0.2,
        "bias_1_H_S_S": torch.randn(1, H, S, S, device="cuda", dtype=dt, generator=g).requires_grad_(True),
    }
    for name, mask in masks.items():
        bias = mask.dtype != torch.bool
        # kernels alone, on the operands the forward uses
        km = sab.k_mean(k)
        q8, qs, k8, ks = sab.per_block_int8(q, k, km, sm_scale=sm)
        me = mask.detach().expand(B, H, S, S)
        o = torch.empty_like(q)
        lse = ops.qk_int8_sv_f16_attn_masked(q8, k8, sab.transpose_v_f16(v), o, qs, ks, me, 1, 1, 1, sm, 1, 1)
        dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
        dbias = torch.empty(B, H, S, S, device="cuda", dtype=dt) if bias else None
        t_kern = _events(lambda: ops.qk_int8_attn_bwd_masked(q8, k8, qs, ks, q, k, v, o, do, lse, km, dq, dk, dv, me, dbias, 1, 1, 1,
                                                             sm, 1), a.steps, a.warmup)
        del dbias
        # the public call
        qg, kg, vg = (t.clone().requires_grad_(True) for t in (q, k, v))
        ins = (qg, kg, vg) + ((mask,) if bias else ())
        ob = sab.sageattn_qk_int8_pv_fp16_triton(qg, kg, vg, attn_mask=mask)
        t_bwd = _events(lambda: torch.autograd.grad(ob, ins, do, retain_graph=True), a.steps, a.warmup)
        del ob
        # torch SDPA memory-efficient backward, same inputs, the mask as a float additive mask
        fm = (mask.detach().float() * math.log(2.0)).to(dt).requires_grad_(True) if bias else \
            torch.zeros(mask.shape, device="cuda", dtype=dt).masked_fill(~mask, float("-inf"))
        with torch.nn.attention.sdpa_kernel(torch.nn.attention.SDPBackend.EFFICIENT_ATTENTION):
            os_ = F.scaled_dot_product_attention(qg, kg, vg, attn_mask=fm)
            sins = (qg, kg, vg) + ((fm,) if bias else ())
            t_sdpa = _events(lambda: torch.autograd.grad(os_, sins, do, retain_graph=True), a.steps, a.warmup)
        out[name] = {
            "bwd_kernel": {"ms": round(t_kern, 3), "tflops": round(flops / t_kern / 1e9, 1)},
            "bwd_call": {"ms": round(t_bwd, 3), "tflops": round(flops / t_bwd / 1e9, 1)},
            "sdpa_efficient_bwd": {"ms": round(t_sdpa, 3), "tflops": round(flops / t_sdpa / 1e9, 1)},
        }
        del os_, fm
    print(json.dumps(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=4)
    ap.add_argument("--H", type=int, default=32)
    ap.add_argument("--S", type=int, default=8192)
    ap.add_argument("--D", type=int, default=128)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--varlen", action="store_true", help="sageattn_varlen on a packed GQA batch instead of sageattn")
    ap.add_argument("--masked", action="store_true", help="sageattn_qk_int8_pv_fp16_triton with attn_mask instead of sageattn")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_backward.py needs a GPU"
    if a.varlen:
        return varlen(a)
    if a.masked:
        return masked(a)
    import sageattention_b200 as sab
    from sageattention_b200 import ops

    B, H, S, D = a.B, a.H, a.S, a.D
    dt = torch.bfloat16
    g = torch.Generator(device="cuda").manual_seed(0)
    q, k, v, do = (torch.randn(B, H, S, D, device="cuda", dtype=dt, generator=g) for _ in range(4))
    sm = D ** -0.5
    out = {"metric": "sageattn backward", "shape": {"B": B, "H": H, "S": S, "D": D, "dtype": "bf16"}, "gpu": _gpu()}
    for causal in (False, True):
        flops = 10.0 * B * H * S * S * D * (0.5 if causal else 1.0)
        # kernels alone, on the operands sageattn's forward uses
        km = sab.k_mean(k)
        q8, qs, k8, ks = sab.per_thread_int8(q, k, km)
        v8, vs, _ = sab.per_channel_fp8(v, scale_max=2.25, smooth_v=False)
        o = torch.empty_like(q)
        lse = ops.qk_int8_sv_f8_attn(q8, k8, v8, o, qs, ks, vs, None, 1, int(causal), 3, 3, sm, 0, 1)
        dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
        t_kern = _events(lambda: ops.qk_int8_attn_bwd(q8, k8, qs, ks, q, k, v, o, do, lse, km, dq, dk, dv, 1, int(causal), 3, 3, sm, 0),
                         a.steps, a.warmup)
        # the public call
        qg, kg, vg = (t.clone().requires_grad_(True) for t in (q, k, v))

        def fwd_bwd():
            qg.grad = kg.grad = vg.grad = None
            sab.sageattn(qg, kg, vg, is_causal=causal).backward(do)

        t_fb = _events(fwd_bwd, a.steps, a.warmup)
        ob = sab.sageattn(qg, kg, vg, is_causal=causal)
        t_bwd = _events(lambda: torch.autograd.grad(ob, (qg, kg, vg), do, retain_graph=True), a.steps, a.warmup)
        # torch SDPA flash backward, same inputs
        with torch.nn.attention.sdpa_kernel(torch.nn.attention.SDPBackend.FLASH_ATTENTION):
            os_ = F.scaled_dot_product_attention(qg, kg, vg, is_causal=causal)
            t_sdpa = _events(lambda: torch.autograd.grad(os_, (qg, kg, vg), do, retain_graph=True), a.steps, a.warmup)
        out["causal" if causal else "non_causal"] = {
            "bwd_kernel": {"ms": round(t_kern, 3), "tflops": round(flops / t_kern / 1e9, 1)},
            "bwd_call": {"ms": round(t_bwd, 3), "tflops": round(flops / t_bwd / 1e9, 1)},
            "fwd_bwd": {"ms": round(t_fb, 3)},
            "sdpa_flash_bwd": {"ms": round(t_sdpa, 3), "tflops": round(flops / t_sdpa / 1e9, 1)},
        }
        del ob, os_
    print(json.dumps(out))


if __name__ == "__main__":
    main()
