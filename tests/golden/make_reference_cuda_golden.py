"""Store what the reference's own CUDA kernels compute for the comparisons in tests/test_gpu_parity.py (a seeded sample of rows of
each output, see `_row_idx`; 16-bit attention outputs as their bit patterns), so that those tests need neither the reference sources nor its compiled extensions.

Run on an H100 once oracle/build_ref.py has built oracle/_ref/*.so (the reference's csrc/fused quantisers, its sm89 FP8-PV attention
kernels and its sm80 FP16-PV kernel, compiled unmodified for sm_90a):
    python tests/golden/make_reference_cuda_golden.py
Output: tests/golden/reference_cuda_kernels.npz.
"""
import importlib.util, os, sys
import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
import sageattention_b200 as sab  # noqa: E402
import test_gpu_parity as T  # noqa: E402


def _ref(name):
    p = os.path.join(ROOT, "oracle", "_ref", name + ".so")
    spec = importlib.util.spec_from_file_location(name, p)
    m = importlib.util.module_from_spec(spec); spec.loader.exec_module(m); return m


def ref_v_fp8(rf, v, smax):
    """The reference's V path (transpose_pad_permute + scale_fuse_quant), its 16-token permutation undone (quant.py:233)."""
    B, H, S, D = v.shape
    pl = (S + 63) // 64 * 64
    vt = torch.empty((B, H, D, pl), dtype=v.dtype, device="cuda")
    rf.transpose_pad_permute_cuda(v, vt, 1)
    r8 = torch.empty(vt.shape, dtype=torch.float8_e4m3fn, device="cuda")
    rs = torch.empty((B, H, D), dtype=torch.float32, device="cuda")
    rf.scale_fuse_quant_cuda(vt, r8, rs, S, smax, 1)
    perm = torch.tensor([0, 1, 8, 9, 2, 3, 10, 11, 4, 5, 12, 13, 6, 7, 14, 15], device="cuda")
    ar = torch.arange(pl, device="cuda")
    src = (ar // 16) * 16 + perm[ar % 16]
    unperm = torch.empty(pl, dtype=torch.long, device="cuda"); unperm[src] = ar
    return r8, rs, r8.view(torch.uint8)[..., unperm][..., :S]


def main():
    rf, ra, r80 = _ref("ref_fused"), _ref("ref_qattn"), _ref("ref_qattn80")
    out = {}
    for ci, (B, H, S, D, dt) in enumerate(T.QREF_CASES):
        q, k, v = T._mk_host(B, H, S, D, dt, seed=ci)
        km = k.mean(dim=2, keepdim=True)
        q8, qs, k8, ks = sab.per_warp_int8(q, k, km)
        rq8, rk8, rqs, rks = torch.empty_like(q8), torch.empty_like(k8), torch.empty_like(qs), torch.empty_like(ks)
        rf.quant_per_warp_int8_cuda(q, rq8, rqs, 128, 32, 1)
        rf.quant_per_block_int8_fuse_sub_mean_cuda(k, km.squeeze(2), rk8, rks, 64, 1)
        ridx = T._row_idx(B * H * S, 10 + ci)
        out[f"quant{ci}_q8"], out[f"quant{ci}_qs"] = T._rows(rq8, ridx).numpy(), rqs.cpu().numpy()
        out[f"quant{ci}_k8"], out[f"quant{ci}_ks"] = T._rows(rk8, ridx).numpy(), rks.cpu().numpy()
        vidx = T._row_idx(B * H * D, 20 + ci)
        for smax in (448.0, 2.25):
            _, rs, r8u = ref_v_fp8(rf, v, smax)
            out[f"quant{ci}_v8_{smax:g}"], out[f"quant{ci}_vs_{smax:g}"] = T._rows(r8u, vidx).numpy(), rs.cpu().numpy()
    for ci, (B, H, S, D, dt, causal, gran) in enumerate(T.ATT_REF_CASES):
        q, k, v = T._mk_host(B, H, S, D, dt, seed=100 + ci)
        km = k.mean(dim=2, keepdim=True)
        q8, qs, k8, ks = (sab.per_warp_int8 if gran == "per_warp" else sab.per_thread_int8)(q, k, km)
        g = 2 if gran == "per_warp" else 3
        ridx = T._row_idx(B * H * S, 100 + ci)
        for smax, fn in [(2.25, ra.qk_int8_sv_f8_accum_f16_fuse_v_scale_attn_inst_buf), (448.0, ra.qk_int8_sv_f8_accum_f32_fuse_v_scale_attn_inst_buf)]:
            r8, rs, _ = ref_v_fp8(rf, v, smax)
            o_ref = torch.empty_like(q)
            lse_ref = fn(q8, k8, r8, o_ref, qs, ks, rs, 1, int(causal), g, D ** -0.5, 1)
            out[f"attn{ci}_o_{smax:g}"] = T._rows(o_ref, ridx).view(torch.int16).numpy()
            out[f"attn{ci}_lse_{smax:g}"] = T._rows(lse_ref.reshape(-1, 1), ridx).reshape(-1).numpy()
    for ci, case in enumerate(T._A16_CASES):
        B, H, S, D, dt, causal, gran, vshift = case
        q, k, v = T._a16_inputs(ci, case)
        km = k.mean(dim=2, keepdim=True)
        q8, qs, k8, ks = (sab.per_warp_int8 if gran == "per_warp" else sab.per_thread_int8)(q, k, km)
        gi = 2 if gran == "per_warp" else 3
        r8, rs, _ = ref_v_fp8(rf, v, 2.25)
        o_ref = torch.empty_like(q)
        ra.qk_int8_sv_f8_accum_f16_fuse_v_scale_attn_inst_buf(q8, k8, r8, o_ref, qs, ks, rs, 1, int(causal), gi, D ** -0.5, 0)
        out[f"a16_{ci}_o"] = T._rows(o_ref, T._row_idx(B * H * S, 200 + ci)).view(torch.int16).numpy()
    for ci, (B, H, Hk, S, D, dt, causal, gran) in enumerate(T.F16PV_CASES):
        q, k, v = T._mk_host(B, H, S, D, dt, Hk=Hk, seed=300 + ci)
        km = k.mean(dim=2, keepdim=True)
        q8, qs, k8, ks = (sab.per_warp_int8 if gran == "per_warp" else sab.per_thread_int8)(q, k, km)
        g = 2 if gran == "per_warp" else 3
        o_ref = torch.empty_like(q)
        lse_ref = r80.qk_int8_sv_f16_accum_f32_attn(q8, k8, v.to(torch.float16), o_ref, qs, ks, 1, int(causal), g, D ** -0.5, 1)
        ridx = T._row_idx(B * H * S, 300 + ci)
        out[f"f16pv{ci}_o"] = T._rows(o_ref, ridx).view(torch.int16).numpy()
        out[f"f16pv{ci}_lse"] = T._rows(lse_ref.reshape(-1, 1), ridx).reshape(-1).numpy()
    torch.cuda.synchronize()
    dst = os.path.join(HERE, "reference_cuda_kernels.npz")
    np.savez_compressed(dst, **out)
    print(f"wrote {dst}: {len(out)} arrays, {os.path.getsize(dst)} bytes")


if __name__ == "__main__":
    main()
