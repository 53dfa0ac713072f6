"""Generate golden fixtures from the REAL reference Triton kernels (executed on CPU).

Run once in the build container (needs /root/reference; not available on the GPU box):
    TRITON_INTERPRET=1 python tests/golden/make_golden.py
The reference package cannot be imported (`sageattention/quant.py:20` needs the compiled
`_fused`), so its Triton modules are loaded by file path; the ~30 lines of host glue around them
(`sageattention/core.py:260-331`, `:399-448`) are restated here.  Outputs: tests/golden/*.npz
(inputs stored as raw fp16/bf16 bit patterns so the fixtures do not depend on RNG versions).
"""
import os, sys, importlib.util
os.environ["TRITON_INTERPRET"] = "1"
import numpy as np
import torch

REF = "/root/reference/sageattention/triton"
HERE = os.path.dirname(os.path.abspath(__file__))


def load(name):
    spec = importlib.util.spec_from_file_location("ref_" + name, f"{REF}/{name}.py")
    m = importlib.util.module_from_spec(spec); spec.loader.exec_module(m); return m


def bits(t):
    return t.contiguous().view(torch.int16).numpy()


def mk(shape, dtype, seed, outlier=False):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(shape, generator=g).to(dtype)
    k = torch.randn(shape, generator=g)
    if outlier:
        k = k + 4.0 * torch.randn((shape[0], shape[1], 1, shape[3]), generator=g)
    k = k.to(dtype)
    v = torch.randn(shape, generator=g)
    if outlier:
        v = v + 2.0
    return q, k, v.to(dtype)


def xattn_fixture(qpb, att):
    """2c. qo_len != kv_len (non-causal cross-attention) with head_dim 96 in bf16: the host glue of
    sageattn_qk_int8_pv_fp16_triton zero-pads the head dim to 128 (core.py:262-271), keeps sm_scale = 96**-0.5 (:288-289), casts V to
    fp16 (:297-298), and slices the output back (:327)."""
    g = torch.Generator().manual_seed(777)
    dtype, D, Dp = torch.bfloat16, 96, 128
    q = torch.randn((1, 2, 192, D), generator=g).to(dtype)
    k = (torch.randn((1, 2, 320, D), generator=g) + 3.0 * torch.randn((1, 2, 1, D), generator=g)).to(dtype)
    v = (torch.randn((1, 2, 320, D), generator=g) + 1.0).to(dtype)
    qp, kp, vp = (torch.nn.functional.pad(t, (0, Dp - D)) for t in (q, k, v))
    km = kp.mean(dim=2, keepdim=True)
    lse_corr = torch.matmul(qp, km.transpose(2, 3)).squeeze(-1).to(torch.float32)
    sm_scale = 1.0 / (D ** 0.5)
    q8, qs, k8, ks = qpb.per_block_int8(qp, kp, km=km, sm_scale=sm_scale)
    o, lse = att.forward(q8, k8, vp.to(torch.float16), qs, ks, tensor_layout="HND", output_dtype=dtype, return_lse=True)
    o = o[..., :D]
    lse = lse / 1.44269504 + lse_corr * sm_scale
    np.savez_compressed(f"{HERE}/attn_xattn_d96_bf16.npz", q=bits(q), k=bits(k), v=bits(v), o=bits(o), lse=lse.numpy(),
                        causal=False, dtype=str(dtype))
    print("wrote attn_xattn_d96_bf16")


def main():
    qpb, qpt, qpbv = load("quant_per_block"), load("quant_per_thread"), load("quant_per_block_varlen")
    att, attc = load("attn_qk_int8_per_block"), load("attn_qk_int8_per_block_causal")
    attv, attvc = load("attn_qk_int8_block_varlen"), load("attn_qk_int8_per_block_causal_varlen")

    only_mask = "--only-mask" in sys.argv      # regenerate just the attn_mask fixtures (section 2b)
    only_xattn = "--only-xattn" in sys.argv    # regenerate just the cross-attention / padded head-dim fixture (section 2c)
    if only_xattn:
        xattn_fixture(qpb, att)
        return

    # ---- 1. quantisation fixtures (bit-exact targets) ----------------------------------------
    for name, shape, dtype, outlier in [] if only_mask else [
        ("quant_d64_fp16", (1, 2, 200, 64), torch.float16, True),
        ("quant_d128_bf16", (2, 1, 333, 128), torch.bfloat16, False),
    ]:
        q, k, _ = mk(shape, dtype, 1234, outlier)
        km = k.mean(dim=2, keepdim=True)
        D = shape[-1]
        out = {"q": bits(q), "k": bits(k), "km": bits(km), "dtype": str(dtype)}
        q8, qs, k8, ks = qpb.per_block_int8(q, k, km=km, sm_scale=D ** -0.5)
        out.update(pb_q8=q8.numpy(), pb_qs=qs.numpy(), pb_k8=k8.numpy(), pb_ks=ks.numpy())
        q8, qs, k8, ks = qpt.per_thread_int8(q, k, km)
        out.update(pt_q8=q8.numpy(), pt_qs=qs.numpy(), pt_k8=k8.numpy(), pt_ks=ks.numpy())
        # NHD layout variant
        qn, kn = q.transpose(1, 2).contiguous(), k.transpose(1, 2).contiguous()
        q8, qs, k8, ks = qpt.per_thread_int8(qn, kn, km.transpose(1, 2), tensor_layout="NHD")
        out.update(ptn_q8=q8.numpy(), ptn_qs=qs.numpy(), ptn_k8=k8.numpy(), ptn_ks=ks.numpy())
        np.savez_compressed(f"{HERE}/{name}.npz", **out)
        print("wrote", name)

    # ---- 2. Triton attention path (sageattn_qk_int8_pv_fp16_triton internals, core.py:260-331) ----
    for name, shape, dtype, causal in [] if only_mask else [
        ("attn_d64_fp16_nc", (1, 2, 320, 64), torch.float16, False),
        ("attn_d64_fp16_c", (1, 2, 320, 64), torch.float16, True),
        ("attn_d128_fp16_nc_ragged", (1, 2, 200, 128), torch.float16, False),
    ]:
        q, k, v = mk(shape, dtype, 99, True)
        D = shape[-1]
        km = k.mean(dim=2, keepdim=True)
        lse_corr = torch.matmul(q, km.transpose(2, 3)).squeeze(-1).to(torch.float32)
        sm_scale = 1.0 / (D ** 0.5)
        q8, qs, k8, ks = qpb.per_block_int8(q, k, km=km, sm_scale=sm_scale)
        fwd = attc.forward if causal else att.forward
        o, lse = fwd(q8, k8, v, qs, ks, tensor_layout="HND", output_dtype=dtype, return_lse=True)
        lse = lse / 1.44269504 + lse_corr * sm_scale
        np.savez_compressed(f"{HERE}/{name}.npz", q=bits(q), k=bits(k), v=bits(v), o=bits(o),
                            lse=lse.numpy(), causal=causal, dtype=str(dtype))
        print("wrote", name)

    if not only_mask:
        xattn_fixture(qpb, att)

    # ---- 2b. attn_mask of the Triton path (core.py:248-250, 310-325; attn_qk_int8_per_block.py:33-52) ----
    for name, shape, kind in [("attn_mask_bool_d64", (1, 2, 256, 64), "bool"), ("attn_mask_bias_d128", (1, 2, 200, 128), "bias")]:
        dtype = torch.float16
        q, k, v = mk(shape, dtype, 4242, True)
        B, H, S, D = shape
        g = torch.Generator().manual_seed(17)
        if kind == "bool":
            mask = torch.rand((1, 1, S, S), generator=g) < 0.6           # broadcast over heads (stride 0 after expand)
            mask[:, :, :128, 64:128] = False                             # one all-false 128 x 64 block: the reference skips it
            mask[:, :, :, 0] = True                                      # every row keeps at least one key
        else:
            mask = torch.randn((1, H, S, S), generator=g)
            mask[torch.rand((1, H, S, S), generator=g) < 0.3] = -30000.0  # "minus infinity" of fp16 pipelines
            mask[:, :, :, 0] = 0.0
            mask = mask.to(dtype)
        km = k.mean(dim=2, keepdim=True)
        lse_corr = torch.matmul(q, km.transpose(2, 3)).squeeze(-1).to(torch.float32)
        sm_scale = 1.0 / (D ** 0.5)
        q8, qs, k8, ks = qpb.per_block_int8(q, k, km=km, sm_scale=sm_scale)
        o, lse = att.forward(q8, k8, v, qs, ks, tensor_layout="HND", output_dtype=dtype, attn_mask=mask.expand(B, H, S, S), return_lse=True)
        lse = lse / 1.44269504 + lse_corr * sm_scale
        mk_arr = mask.numpy() if kind == "bool" else bits(mask)
        np.savez_compressed(f"{HERE}/{name}.npz", q=bits(q), k=bits(k), v=bits(v), o=bits(o), lse=lse.numpy(), mask=mk_arr,
                            mask_shape=np.array(mask.shape), kind=kind, dtype=str(dtype))
        print("wrote", name)
    if only_mask:
        return

    # ---- 3. varlen (core.py:399-448) ---------------------------------------------------------
    for name, causal in [("varlen_gqa_d128_nc", False), ("varlen_gqa_d128_c", True)]:
        g = torch.Generator().manual_seed(7)
        lens = [200, 130, 77]
        T, Hq, Hk, D = sum(lens), 2, 1, 128
        q = torch.randn((T, Hq, D), generator=g).half()
        k = (torch.randn((T, Hk, D), generator=g) + 2.0 * torch.randn((1, Hk, D), generator=g)).half()
        v = torch.randn((T, Hk, D), generator=g).half()
        cu = torch.tensor([0] + list(np.cumsum(lens)), dtype=torch.int32)
        km = k.mean(dim=0, keepdim=True)
        ks_ = k - km
        sm_scale = 1.0 / (D ** 0.5)
        q8, qs, k8, ks, cuqs, cuks = qpbv.per_block_int8(q, ks_, cu, cu, max(lens), max(lens), sm_scale=sm_scale)
        fwd = attvc.forward if causal else attv.forward
        o = fwd(q8, k8, v, cu, cu, max(lens), qs, ks, cuqs, cuks, output_dtype=torch.float16)
        np.savez_compressed(f"{HERE}/{name}.npz", q=bits(q), k=bits(k), v=bits(v), o=bits(o),
                            cu=cu.numpy(), q8=q8.numpy(), qs=qs.numpy(), k8=k8.numpy(), ks=ks.numpy(),
                            cuqs=cuqs.numpy(), cuks=cuks.numpy(), causal=causal)
        print("wrote", name)


if __name__ == "__main__":
    main()
