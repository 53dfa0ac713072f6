"""GPU tests (-m gpu) of the gradient kernels (csrc/attn_bwd.cu) at their edges:
  1. stride independence: q8, k8, q, k, v, o, dO and the outputs as row- and head-padded views of wider buffers, each with its
     own strides, give the bits of the contiguous call and leave the outputs' padding alone; HND gives the bits of NHD;
  2. every differentiable dense entry point and option through autograd, elementwise against the fp64 reference on that entry's
     own operands (attn_bwd_oracle), and against fp64 exact attention; the autograd plumbing (packed qkv, strided dO, partial
     requires_grad, return_lse);
  3. full-size gradients (the backward benchmark's shape and a 32K causal one): every element written, bit-reproducible, and
     every head inside the elementwise bound of the row-chunked fp64 reference evaluated on the GPU;
  4. the backward ops refuse o / dout / q_int8 / k_int8 of the wrong shape or dtype before launching anything.
The elementwise bound and its derivation are in tests/attn_bwd_oracle.py; the tests print the worst ratio of error to bound and
the normwise relative error (pytest -s).  Measured on an H100 80GB HBM3 (400 W power limit):
  * entry points (ENTRY_CASES): worst ratio 0.81; normwise at most 2.4e-3 for bf16 and 3.0e-4 for fp16; against exact attention
    0.6-2.3 % (TOL_EXACT 3e-2);
  * full size: worst ratio 0.254 (S=8192, non-causal), 0.839 (S=8192, causal), 0.941 (S=32768, causal); normwise at most 2.4e-3
    for bf16 and 3.1e-4 for fp16."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from attn_bwd_oracle import attn_bwd, check_elementwise

pytestmark = pytest.mark.gpu
BF, FP = torch.bfloat16, torch.float16
GRAN = {"per_block": 1, "per_warp": 2, "per_thread": 3}      # SAB_GRAN_*
ORACLE_GRAN = {"per_thread": ("per_thread", "per_thread"), "per_warp": ("per_warp", "per_block"), "per_block": ("per_block", "per_block")}
TOL_EXACT = 3e-2      # normwise against fp64 exact attention (tests/test_gpu_backward.py)
SENTINEL = 7.0


def _shape(B, H, S, D, layout):
    return (B, H, S, D) if layout == "HND" else (B, S, H, D)


def _hnd(x, layout):
    return x if layout == "HND" else x.transpose(1, 2)


def _randn(shape, seed, dt):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed)).to(dt).cuda()


def _padded(x, extra_cols, extra_heads, head_dim, fill):
    """x as a view of a wider buffer: extra_cols more elements per row and extra_heads more heads (dimension head_dim), the rest
    filled with `fill`.  Returns (view, buffer)."""
    shape = list(x.shape)
    shape[-1] += extra_cols
    shape[head_dim] += extra_heads
    buf = torch.full(shape, fill, dtype=x.dtype, device=x.device)
    view = buf.narrow(head_dim, 0, x.size(head_dim))[..., :x.size(-1)]
    view.copy_(x)
    return view, buf


# ------------------------------------------------------------------------------------------- 1. stride independence
def _dense_operands(D, dt, gran, layout, causal, B=2, Hq=4, Hkv=2, Sq=200, Skv=200, seed=0):
    import sageattention_b200 as sab
    from sageattention_b200 import ops
    lay = 1 if layout == "HND" else 0
    q = _randn(_shape(B, Hq, Sq, D, layout), seed, dt)
    k = _randn(_shape(B, Hkv, Skv, D, layout), seed + 1, dt) + 2.0
    v = _randn(_shape(B, Hkv, Skv, D, layout), seed + 2, dt)
    do = _randn(_shape(B, Hq, Sq, D, layout), seed + 3, dt)
    sm = D ** -0.5
    km = sab.k_mean(k, layout)
    o = torch.empty_like(q)
    if gran == "per_block":
        q8, qs, k8, ks = sab.per_block_int8(q, k, km, sm_scale=sm, tensor_layout=layout)
        lse = ops.qk_int8_sv_f16_attn(q8, k8, sab.transpose_v_f16(v, layout), o, qs, ks, lay, int(causal), 1, 1, sm, 1, 1)
        fold = 1
    else:
        q8, qs, k8, ks = (sab.per_thread_int8 if gran == "per_thread" else sab.per_warp_int8)(q, k, km, tensor_layout=layout)
        v8, vs, _ = sab.per_channel_fp8(v, tensor_layout=layout, scale_max=448.0, smooth_v=False)
        lse = ops.qk_int8_sv_f8_attn(q8, k8, v8, o, qs, ks, vs, None, lay, int(causal), GRAN[gran], GRAN[gran], sm, 0, 1)
        fold = 0
    return dict(q8=q8, k8=k8, qs=qs, ks=ks, q=q, k=k, v=v, o=o, do=do, lse=lse, km=km, lay=lay, causal=int(causal),
                gran=GRAN[gran], sm=sm, fold=fold)


def _dense_bwd(c, outs=None, **views):
    from sageattention_b200 import ops
    t = dict(c, **views)
    dq, dk, dv = outs or (torch.full_like(t[n], float("nan")) for n in ("q", "k", "v"))
    ops.qk_int8_attn_bwd(t["q8"], t["k8"], t["qs"], t["ks"], t["q"], t["k"], t["v"], t["o"], t["do"], t["lse"], t["km"], dq, dk, dv,
                         t["lay"], t["causal"], t["gran"], t["gran"], t["sm"], t["fold"])
    return dq, dk, dv


def _strided_views(c, head_dim):
    """Every 16-bit input and both int8 operands as a view with its own strides: tensor i gets 8 (i + 1) extra elements per row
    (16 (i + 1) for int8, whose strides must be multiples of 16) and, every other tensor, one extra head."""
    views = {}
    for i, n in enumerate(("q8", "k8", "q", "k", "v", "o", "do")):
        cols = (16 if c[n].dtype == torch.int8 else 8) * (i + 1)
        views[n] = _padded(c[n], cols, i % 2, head_dim, 0)[0]
    return views


def _strided_outputs(c, head_dim):
    """dq / dk / dv as views of SENTINEL-filled buffers with the strides of the q / k / v views (same padding recipe)."""
    outs, bufs = [], []
    for i, n in zip((2, 3, 4), ("q", "k", "v")):
        view, buf = _padded(torch.full_like(c[n], float("nan")), 8 * (i + 1), i % 2, head_dim, SENTINEL)
        outs.append(view)
        bufs.append(buf)
    return outs, bufs


def _outside(view, buf):
    """The elements of buf that are not in view (view = buf.narrow(...)[..., :D])."""
    inside = torch.zeros(buf.shape, dtype=torch.bool, device=buf.device)
    idx = tuple(slice(0, s) for s in view.shape)
    inside[idx] = True
    return buf[~inside]


DENSE_INSTANTIATIONS = [   # (D, dtype, gran, layout, causal): every (D, per-thread K scales or not, dtype) of attn_bwd.cu
    (128, BF, "per_thread", "HND", False), (128, FP, "per_thread", "NHD", True), (128, BF, "per_warp", "NHD", True),
    (128, FP, "per_block", "HND", False), (64, BF, "per_thread", "NHD", False), (64, FP, "per_thread", "HND", True),
    (64, BF, "per_block", "HND", True), (64, FP, "per_warp", "NHD", False),
]


@pytest.mark.parametrize("case", DENSE_INSTANTIATIONS, ids=lambda c: f"D{c[0]}-{str(c[1])[6:]}-{c[2]}-{c[3]}-causal{int(c[4])}")
def test_dense_gradients_do_not_depend_on_strides(case):
    D, dt, gran, layout, causal = case
    c = _dense_operands(D, dt, gran, layout, causal)
    hd = 1 if layout == "HND" else 2
    ref = _dense_bwd(c)
    views = _strided_views(c, hd)
    outs, bufs = _strided_outputs(views, hd)
    got = _dense_bwd(c, outs, **views)
    for name, a, b, buf in zip(("dq", "dk", "dv"), got, ref, bufs):
        assert a.stride() != b.stride()
        assert torch.equal(a, b), name
        assert torch.all(_outside(a, buf) == SENTINEL), f"{name}: the padding of the output buffer was written"


@pytest.mark.parametrize("case", DENSE_INSTANTIATIONS, ids=lambda c: f"D{c[0]}-{str(c[1])[6:]}-{c[2]}-causal{int(c[4])}")
def test_hnd_gradients_are_the_nhd_gradients(case):
    D, dt, gran, _, causal = case
    c = _dense_operands(D, dt, gran, "HND", causal)
    hnd = _dense_bwd(c)
    nhd_in = {n: c[n].transpose(1, 2).contiguous() for n in ("q8", "k8", "q", "k", "v", "o", "do")}
    nhd = _dense_bwd(c, lay=0, km=c["km"].transpose(1, 2).contiguous(), **nhd_in)
    for name, a, b in zip(("dq", "dk", "dv"), hnd, nhd):
        assert torch.equal(a, b.transpose(1, 2)), name


def test_varlen_gradients_do_not_depend_on_strides():
    import sageattention_b200 as sab
    from sageattention_b200 import ops
    from sageattention_b200.quant import per_block_int8_varlen, transpose_v_f16_varlen
    lq, lk, Hq, Hk, D, dt = [100, 0, 129], [64, 30, 200], 4, 2, 64, BF
    cq, ck = (torch.tensor([0] + list(np.cumsum(x)), dtype=torch.int32, device="cuda") for x in (lq, lk))
    q, do = _randn((sum(lq), Hq, D), 1, dt), _randn((sum(lq), Hq, D), 2, dt)
    k, v = _randn((sum(lk), Hk, D), 3, dt) + 2.0, _randn((sum(lk), Hk, D), 4, dt)
    sm = D ** -0.5
    km = sab.k_mean(k.unsqueeze(0), "NHD").view(Hk, D)
    q8, qs, k8, ks, cqs, cks = per_block_int8_varlen(q, k, cq, ck, max(lq), max(lk), sm_scale=sm, km=km)
    v_t, cu_pad = transpose_v_f16_varlen(v, ck, max(lk))
    o = torch.empty_like(q)
    lse = ops.qk_int8_sv_f16_attn_varlen(q8, k8, v_t, o, qs, ks, cq, ck, cu_pad, cqs, cks, max(lq), 1, sm, 1, 1)
    c = dict(q8=q8, k8=k8, q=q, k=k, v=v, o=o, do=do)

    def run(t, outs):
        ops.qk_int8_attn_bwd_varlen(t["q8"], t["k8"], qs, ks, t["q"], t["k"], t["v"], t["o"], t["do"], lse, km, *outs, cq, ck, cqs,
                                    cks, max(lq), max(lk), 1, sm, 1)
        return outs

    ref = run(c, [torch.full_like(c[n], float("nan")) for n in ("q", "k", "v")])
    views = _strided_views(c, 1)
    outs, bufs = _strided_outputs(views, 1)
    for name, a, b, buf in zip(("dq", "dk", "dv"), run(views, outs), ref, bufs):
        assert torch.equal(a, b), name
        assert torch.all(_outside(a, buf) == SENTINEL), name


@pytest.mark.parametrize("family", ["masked", "blocksparse"])
def test_masked_and_blocksparse_gradients_do_not_depend_on_strides(family):
    import sageattention_b200 as sab
    from sageattention_b200 import ops
    layout, D, dt = "NHD", 128, FP
    B, Hq, Hkv, Sq, Skv = 2, 4, 2, 200, 260
    q, do = _randn(_shape(B, Hq, Sq, D, layout), 1, dt), _randn(_shape(B, Hq, Sq, D, layout), 2, dt)
    k, v = _randn(_shape(B, Hkv, Skv, D, layout), 3, dt) + 2.0, _randn(_shape(B, Hkv, Skv, D, layout), 4, dt)
    sm = D ** -0.5
    km = sab.k_mean(k, layout)
    o = torch.empty_like(q)
    if family == "masked":
        mask = (_randn((B, Hq, Sq, Skv), 5, torch.float32) * 2).to(dt)
        q8, qs, k8, ks = sab.per_block_int8(q, k, km, sm_scale=sm, tensor_layout=layout)
        lse = ops.qk_int8_sv_f16_attn_masked(q8, k8, sab.transpose_v_f16(v, layout), o, qs, ks, mask, 0, 1, 1, sm, 1, 1)

        def run(t, outs):
            ops.qk_int8_attn_bwd_masked(t["q8"], t["k8"], qs, ks, t["q"], t["k"], t["v"], t["o"], t["do"], lse, km, *outs, mask, None,
                                        0, 1, 1, sm, 1)
            return outs
    else:
        bm = torch.rand((B, Hq, (Sq + 127) // 128, (Skv + 63) // 64), generator=torch.Generator(device="cuda").manual_seed(6),
                        device="cuda") < 0.6
        q8, qs, k8, ks = sab.per_thread_int8(q, k, km, tensor_layout=layout)
        v8, vs, _ = sab.per_channel_fp8(v, tensor_layout=layout, scale_max=448.0, smooth_v=False)
        lse = ops.qk_int8_sv_f8_attn_blocksparse(q8, k8, v8, o, qs, ks, vs, None, bm, 0, 0, 3, 3, sm, 0, 1)

        def run(t, outs):
            ops.qk_int8_attn_bwd_blocksparse(t["q8"], t["k8"], qs, ks, t["q"], t["k"], t["v"], t["o"], t["do"], lse, km, *outs, bm, 0,
                                             0, 3, 3, sm, 0)
            return outs
    c = dict(q8=q8, k8=k8, q=q, k=k, v=v, o=o, do=do)
    ref = run(c, [torch.full_like(c[n], float("nan")) for n in ("q", "k", "v")])
    views = _strided_views(c, 2)
    outs, bufs = _strided_outputs(views, 2)
    for name, a, b, buf in zip(("dq", "dk", "dv"), run(views, outs), ref, bufs):
        assert torch.equal(a, b), name
        assert torch.all(_outside(a, buf) == SENTINEL), name


# ------------------------------------------------------------------------------------------- 2. entry points through autograd
def _entries():
    """name -> (entry point, kind, qk_quant_gran, V range, quantization backend) as core.py calls _attn_dense."""
    import sageattention_b200 as sab
    return {
        "sageattn": (sab.sageattn, "fp8", "per_thread", 2.25, "cuda"),
        "fp8_cuda_per_warp": (lambda *a, **kw: sab.sageattn_qk_int8_pv_fp8_cuda(*a, qk_quant_gran="per_warp", **kw), "fp8", "per_warp",
                              2.25, "cuda"),
        "fp8_cuda_per_thread": (sab.sageattn_qk_int8_pv_fp8_cuda, "fp8", "per_thread", 2.25, "cuda"),
        "fp8_cuda_sm90": (sab.sageattn_qk_int8_pv_fp8_cuda_sm90, "fp8", "per_thread", 448.0, "cuda"),
        "fp16_cuda": (sab.sageattn_qk_int8_pv_fp16_cuda, "fp16_cuda", "per_thread", 0.0, "cuda"),
        "fp16_cuda_per_warp": (lambda *a, **kw: sab.sageattn_qk_int8_pv_fp16_cuda(*a, qk_quant_gran="per_warp", **kw), "fp16_cuda",
                               "per_warp", 0.0, "cuda"),
        "fp16_triton": (sab.sageattn_qk_int8_pv_fp16_triton, "fp16_triton", "per_block", 0.0, "triton"),
        "fp16_triton_cuda_quant": (lambda *a, **kw: sab.sageattn_qk_int8_pv_fp16_triton(*a, quantization_backend="cuda", **kw),
                                   "fp16_triton", "per_block", 0.0, "cuda"),
    }


# (entry, D, dtype, layout, causal, options)
ENTRY_CASES = [
    ("sageattn", 128, BF, "HND", True, {}),
    ("fp8_cuda_per_warp", 64, FP, "NHD", False, {}),
    ("fp8_cuda_per_thread", 128, FP, "HND", False, {}),
    ("fp8_cuda_sm90", 128, BF, "NHD", True, {}),
    ("fp16_cuda", 64, BF, "HND", True, {}),
    ("fp16_cuda_per_warp", 128, FP, "NHD", False, {}),
    ("fp16_triton", 128, FP, "HND", False, {}),
    ("fp16_triton", 64, BF, "NHD", True, {}),
    ("fp16_triton_cuda_quant", 128, BF, "HND", True, {}),
    ("fp8_cuda_per_thread", 64, BF, "HND", True, {"smooth_k": False}),
    ("fp16_triton", 128, FP, "NHD", False, {"smooth_k": False}),
    ("fp16_cuda", 128, FP, "HND", False, {"sm_scale": 0.05}),
    ("fp16_triton", 64, FP, "HND", True, {"sm_scale": 0.2}),
    ("fp8_cuda_per_thread", 128, BF, "NHD", False, {"pv_accum_dtype": "fp32", "smooth_v": True}),
    ("sageattn", 32, BF, "HND", False, {}),
    ("fp16_triton", 40, FP, "NHD", True, {}),
    ("fp8_cuda_per_warp", 72, BF, "HND", True, {}),
    ("fp16_cuda", 80, FP, "NHD", False, {}),
    ("fp8_cuda_sm90", 112, FP, "HND", False, {}),
]


def _exact_grads(q, k, v, do, causal, layout, sm):
    q, k, v = (_hnd(t, layout).detach().double().requires_grad_(True) for t in (q, k, v))
    o = F.scaled_dot_product_attention(q, k, v, is_causal=causal, enable_gqa=True, scale=sm)
    (o * _hnd(do, layout).double()).sum().backward()
    return q.grad, k.grad, v.grad


@pytest.mark.parametrize("case", ENTRY_CASES, ids=lambda c: f"{c[0]}-D{c[1]}-{str(c[2])[6:]}-{c[3]}-causal{int(c[4])}-" +
                         ("-".join(f"{k}={v}" for k, v in c[5].items()) or "default"))
def test_entry_point_gradients_match_oracle_elementwise(case):
    from sageattention_b200 import core
    name, D, dt, layout, causal, opts = case
    fn, kind, gran, v_range, backend = _entries()[name]
    B, Hq, Hkv, S = 2, 4, 2, 300
    q, k, v = (_randn(_shape(B, H, S, D, layout), s, dt).requires_grad_(True) for s, H in ((1, Hq), (2, Hkv), (3, Hkv)))
    do = _randn(_shape(B, Hq, S, D, layout), 4, dt)
    o = fn(q, k, v, tensor_layout=layout, is_causal=causal, **opts)
    o.backward(do)
    # the entry's own operands: head-dim-padded q, k, v, the forward's quantisers, o and raw LSE
    qp, kp, vp, d0 = core._pad_head_dim(q.detach(), k.detach(), v.detach())
    sm = opts.get("sm_scale", 1.0 / (d0 ** 0.5) if kind == "fp16_triton" else d0 ** -0.5)   # as each entry computes it
    smooth_k = opts.get("smooth_k", True)
    smooth_v = opts.get("smooth_v", False)
    if "pv_accum_dtype" in opts:
        v_range = 448.0
    km, q8, qs, k8, ks, _, _, fold = core._quant_qk(qp, kp, kind, layout, gran, sm, smooth_k, backend)
    op, lse, _ = core._attn_dense(qp, kp, vp, kind, layout, causal, gran, sm, smooth_k, smooth_v, v_range, backend, True)
    assert torch.equal(op[..., :D], o.detach())
    qg, kg = ORACLE_GRAN[gran]
    *ref, bounds = attn_bwd(_hnd(q8, layout), _hnd(k8, layout), qs, ks, _hnd(qp, layout), _hnd(kp, layout), _hnd(vp, layout),
                            _hnd(op, layout), _hnd(F.pad(do, (0, qp.size(-1) - D)), layout), lse, q_gran=qg, k_gran=kg,
                            is_causal=causal, sm_scale=sm, fold_sm_scale=bool(fold), k_mean=None if km is None else _hnd(km, layout),
                            bound=True)
    res = {n: check_elementwise(n, _hnd(t.grad, layout), r[..., :D], b[..., :D])
           for n, t, r, b in zip(("dq", "dk", "dv"), (q, k, v), ref, bounds)}
    exact = _exact_grads(q, k, v, do, causal, layout, sm)
    errs = {n: float((_hnd(t.grad, layout).double() - e).norm() / e.norm()) for n, t, e in zip(("dq", "dk", "dv"), (q, k, v), exact)}
    print(f"[entry] {case}: " + ", ".join(f"{n} ratio {w:.3f} normwise {e:.2e}" for n, (w, e) in res.items()) +
          "; exact " + ", ".join(f"{n} {e:.2e}" for n, e in errs.items()))
    assert max(errs.values()) <= TOL_EXACT, errs


def _grads(fn, q, k, v, do, **kw):
    q, k, v = (t.detach().clone().requires_grad_(True) for t in (q, k, v))
    fn(q, k, v, **kw).backward(do)
    return q.grad, k.grad, v.grad


def test_packed_qkv_and_strided_dout_give_the_contiguous_gradients():
    import sageattention_b200 as sab
    B, S, H, D = 2, 300, 4, 128
    qkv = _randn((B, S, 3, H, D), 1, BF).requires_grad_(True)
    q, k, v = qkv.unbind(2)                                          # NHD views with a 3*H*D sequence stride
    do_wide = _randn((B, S, H, 2 * D), 2, BF)
    do = do_wide[..., ::2]                                           # a non-contiguous dO (element stride 2)
    o = sab.sageattn(q, k, v, tensor_layout="NHD", is_causal=True)
    o.backward(do)
    ref = _grads(sab.sageattn, q.contiguous(), k.contiguous(), v.contiguous(), do.contiguous(), tensor_layout="NHD", is_causal=True)
    for i, (name, r) in enumerate(zip(("dq", "dk", "dv"), ref)):
        assert torch.equal(qkv.grad[:, :, i], r), name


def test_partial_requires_grad_and_return_lse_keep_the_bits():
    import sageattention_b200 as sab
    q, k, v = (_randn((1, 4, 257, 128), s, FP) for s in (1, 2, 3))
    do = _randn((1, 4, 257, 128), 4, FP)
    full = _grads(sab.sageattn, q, k, v, do, is_causal=True)
    vg = v.clone().requires_grad_(True)
    sab.sageattn(q, k, vg, is_causal=True).backward(do)
    assert torch.equal(vg.grad, full[2])
    qg, kg, vg = (t.clone().requires_grad_(True) for t in (q, k, v))
    o, lse = sab.sageattn(qg, kg, vg, is_causal=True, return_lse=True)
    assert not lse.requires_grad
    o.backward(do)
    for name, a, b in zip(("dq", "dk", "dv"), (qg.grad, kg.grad, vg.grad), full):
        assert torch.equal(a, b), name


# ------------------------------------------------------------------------------------------- 3. full size
FULL_CASES = [   # (B, H, S, D, dtype, causal): bench_backward.py's shape, causal or not, and a 32K causal sequence
    (4, 32, 8192, 128, BF, False),
    (4, 32, 8192, 128, BF, True),
    (1, 32, 32768, 64, FP, True),
]
CHUNK_ELEMENTS = 2 ** 26        # rows x keys of one fp64 [rows, Skv] temporary: 512 MiB


@pytest.mark.parametrize("case", FULL_CASES, ids=lambda c: f"B{c[0]}-H{c[1]}-S{c[2]}-D{c[3]}-{str(c[4])[6:]}-causal{int(c[5])}")
def test_full_size_gradients_every_head_inside_the_bound(case):
    from sageattention_b200 import core, ops
    B, H, S, D, dt, causal = case
    g = torch.Generator(device="cuda").manual_seed(S + D)
    q, k, v, do = (torch.randn((B, H, S, D), generator=g, device="cuda").to(dt) for _ in range(4))
    k += 2.0
    sm = D ** -0.5
    km, q8, qs, k8, ks, qgran, kgran, fold = core._quant_qk(q, k, "fp8", "HND", "per_thread", sm, True, "cuda")
    o, lse, _ = core._attn_dense(q, k, v, "fp8", "HND", causal, "per_thread", sm, True, False, 2.25, "cuda", True)
    runs = []
    for _ in range(2):
        grads = tuple(torch.full_like(t, float("nan")) for t in (q, k, v))
        ops.qk_int8_attn_bwd(q8, k8, qs, ks, q, k, v, o, do, lse, km, *grads, 1, int(causal), qgran, kgran, sm, fold)
        runs.append(grads)
    for name, a, b in zip(("dq", "dk", "dv"), *runs):
        assert torch.equal(a, b), f"{name}: two calls differ"
    dq, dk, dv = runs[0]
    rows = max(128, CHUNK_ELEMENTS // S // 128 * 128)
    worst = {"dq": (0.0, 0.0), "dk": (0.0, 0.0), "dv": (0.0, 0.0)}
    for b in range(B):
        for h in range(H):
            sl = (slice(b, b + 1), slice(h, h + 1))
            acc = None
            for r0 in range(0, S, rows):
                r1 = min(S, r0 + rows)
                part = attn_bwd(q8[sl][:, :, r0:r1], k8[sl], qs[sl], ks[sl], q[sl][:, :, r0:r1], k[sl], v[sl], o[sl][:, :, r0:r1],
                                do[sl][:, :, r0:r1], lse[sl][:, :, r0:r1], q_gran="per_thread", k_gran="per_thread", is_causal=causal,
                                sm_scale=sm, k_mean=km[sl], q_offset=r0, q_len=S, bound=True)
                w = check_elementwise(f"dq b={b} h={h}", dq[sl][:, :, r0:r1], part[0], part[3][0])
                worst["dq"] = max(worst["dq"], w)
                kv = (part[1], part[2], part[3][1], part[3][2])
                acc = kv if acc is None else tuple(x + y for x, y in zip(acc, kv))
                del part
            for name, got, r, bd in (("dk", dk, acc[0], acc[2]), ("dv", dv, acc[1], acc[3])):
                worst[name] = max(worst[name], check_elementwise(f"{name} b={b} h={h}", got[sl], r, bd))
    print(f"[full] {case}: " + ", ".join(f"{n} ratio {w:.3f} normwise {e:.2e}" for n, (w, e) in worst.items()))


# ------------------------------------------------------------------------------------------- 4. validation
def _bwd_call(family, **bad):
    """One small, valid call of a backward op with `bad` substituted; returns (call, outputs)."""
    import sageattention_b200 as sab
    from sageattention_b200 import ops
    if family == "varlen":
        T, H, D = 128, 2, 64
        q, k, v = (_randn((T, H, D), s, FP) for s in (1, 2, 3))
        cu = torch.tensor([0, T], dtype=torch.int32, device="cuda")
        cus = torch.tensor([0, 1], dtype=torch.int32, device="cuda")
        q8, k8 = torch.zeros_like(q, dtype=torch.int8), torch.zeros_like(k, dtype=torch.int8)
        qs, ks = torch.ones(1, H, device="cuda"), torch.ones(2, H, device="cuda")
        lse = torch.zeros(H, T, device="cuda")
        a = dict(q8=q8, k8=k8, o=q.clone(), dout=q.clone())
        a.update(bad)
        outs = [torch.full_like(t, float("nan")) for t in (q, k, v)]
        return (lambda: ops.qk_int8_attn_bwd_varlen(a["q8"], a["k8"], qs, ks, q, k, v, a["o"], a["dout"], lse, None, *outs, cu, cu,
                                                    cus, torch.tensor([0, 2], dtype=torch.int32, device="cuda"), T, T, 0, 0.125, 1)), outs
    B, H, S, D = 1, 2, 128, 64
    q, k, v = (_randn((B, H, S, D), s, FP) for s in (1, 2, 3))
    q8, qs, k8, ks = sab.per_warp_int8(q, k, None)
    lse = torch.zeros(B, H, S, device="cuda")
    a = dict(q8=q8, k8=k8, o=q.clone(), dout=q.clone())
    a.update(bad)
    outs = [torch.full_like(t, float("nan")) for t in (q, k, v)]
    args = (a["q8"], a["k8"], qs, ks, q, k, v, a["o"], a["dout"], lse, None, *outs)
    if family == "dense":
        return (lambda: ops.qk_int8_attn_bwd(*args, 1, 0, 2, 2, 0.125, 0)), outs
    if family == "masked":
        mask = torch.ones(B, H, S, S, dtype=torch.bool, device="cuda")
        return (lambda: ops.qk_int8_attn_bwd_masked(*args, mask, None, 1, 2, 2, 0.125, 0)), outs
    bm = torch.ones(B, H, 1, 2, dtype=torch.bool, device="cuda")
    return (lambda: ops.qk_int8_attn_bwd_blocksparse(*args, bm, 1, 0, 2, 2, 0.125, 0)), outs


def _bad_arguments(family):
    ref = _randn((128, 2, 64), 9, FP) if family == "varlen" else _randn((1, 2, 128, 64), 9, FP)
    fewer_rows = ref[:-1] if family == "varlen" else ref[:, :, :-1]
    return {
        "o_fewer_rows": dict(o=fewer_rows),
        "o_bf16": dict(o=ref.to(BF)),
        "dout_fewer_rows": dict(dout=fewer_rows),
        "dout_fp32": dict(dout=ref.float()),
        "q8_fewer_rows": dict(q8=fewer_rows.to(torch.int8)),
        "k8_wider": dict(k8=torch.zeros(ref.shape[:-1] + (128,), dtype=torch.int8, device="cuda")),
        "q8_not_int8": dict(q8=ref.to(torch.uint8)),
    }


@pytest.mark.parametrize("family", ["dense", "varlen", "masked", "blocksparse"])
@pytest.mark.parametrize("bad", ["o_fewer_rows", "o_bf16", "dout_fewer_rows", "dout_fp32", "q8_fewer_rows", "k8_wider", "q8_not_int8"])
def test_backward_ops_refuse_mismatched_operands_before_launching(family, bad):
    call, outs = _bwd_call(family)
    call()                                                              # the valid call runs
    torch.cuda.synchronize()
    call, outs = _bwd_call(family, **_bad_arguments(family)[bad])
    with pytest.raises(AssertionError, match="must"):
        call()
    torch.cuda.synchronize()
    assert all(torch.isnan(t).all() for t in outs), "an output was written: the op launched before refusing"
