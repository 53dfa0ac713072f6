"""CPU tests (no GPU) of the FP16-PV restatement and its bound (tests/attn_fp16pv_oracle.py):
  1. with bound=False it is the reference's FP16-PV arithmetic: oracle.sage_oracle.attn_int8_fp16_cuda on unmasked inputs, and
     attn_int8_fp16_triton on masked inputs where the kernel and the reference agree (every row sees a key in its first visited
     tile), within the bound (the references sum in fp32, and the Triton one rounds each tile's PV to fp16: 2^-11 of its terms);
     row chunks give the whole call's rows bit for bit;
  2. a CPU emulation of the kernel's arithmetic stays inside the bound: ex2 perturbed within its error, every ambiguous fp16 P
     flipped at random, the in-place accumulation cut to the U_TC16 model, fp32 d and epilogue;
  3. each planted mistake of the kernel breaks the bound.  The table printed by test_planted_mistakes_break_the_bound gives each
     one's worst error / bound ratio and whether the max-abs gate of test_gpu_kernel_edges.test_every_instantiation_vs_oracle
     (2e-3 fp16-cuda, 4e-3 Triton fp16, 2e-2 Triton bf16) would have caught it on the same input."""
import math

import pytest
import torch

from attn_bwd_oracle import elementwise_ratio
from attn_fp16pv_oracle import F16, attn_fp16pv, attn_fp16pv_varlen
from attn_window_oracle import check_forward
from oracle import sage_oracle as O

BF = torch.bfloat16
GATE = {("cuda", F16): 2e-3, ("cuda", BF): 2e-3 + 2.0 ** -7, ("triton", F16): 4e-3, ("triton", BF): 2e-2}


def _qkv(B, Hq, Hk, Sq, Sk, D, dt, seed, kind="randn"):
    """randn inputs; "ramp": the scores grow along the keys, so the running max moves on most tiles; "peak": rows whose logits
    span some 40 binades, so P reaches fp16 subnormals."""
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(B, Hq, Sq, D, generator=g)
    k = torch.randn(B, Hk, Sk, D, generator=g) + torch.randn(B, Hk, 1, D, generator=g)
    v = torch.randn(B, Hk, Sk, D, generator=g)
    if kind != "randn":
        u = torch.randn(D, generator=g)
        u = u / u.norm()
        c, R = (2.0, 48.0) if kind == "ramp" else (8.0, 30.0)
        q = q + c * u
        k = k + torch.linspace(0.0, R, Sk)[:, None] * u
    return q.to(dt), k.to(dt), v.to(dt)


def _operands(q, k, path, gran="per_block", sm=None):
    """The reference quantisers' operands (K smoothed by its mean): (q8, qs, k8, ks, gran, fold)."""
    D = q.size(-1)
    km = k.mean(dim=2, keepdim=True)
    if path == "triton":
        q8, qs, k8, ks = O.per_block_int8_triton(q, k, km, sm_scale=sm if sm is not None else D ** -0.5)
        return q8, qs, k8, ks, "per_block", True
    f = O.per_warp_int8_cuda if gran == "per_warp" else O.quant_per_thread_int8_triton
    q8, qs, k8, ks = f(q, k, km)
    return q8, qs, k8, ks, gran, False


def _restate(ops, v, dt, **kw):
    q8, qs, k8, ks, gran, fold = ops
    D = q8.size(-1)
    return attn_fp16pv(q8, k8, v, qs, ks, q_gran=gran, fold_sm_scale=fold, sm_scale=D ** -0.5, out_dtype=dt, return_lse=True,
                       **kw)


def _within(ref32, bd, slack):
    """Worst |ref32 - restatement| / (bound + slack + 2^-22 |o|) over the rows that see a key."""
    tol = bd.o_bound + slack + 2.0 ** -22 * bd.o.abs()
    err = (ref32.double() - bd.o).abs()
    return float(torch.where(err == 0, 0.0, err / tol).max())


# ------------------------------------------------------------------------------------------------ 1. the reference's arithmetic
@pytest.mark.parametrize("gran", ["per_warp", "per_thread"])
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("dt", [F16, BF])
def test_unmasked_equals_the_reference_cuda_restatement(gran, causal, dt):
    Sq, Sk = (200, 200) if causal else (150, 333)
    q, k, v = _qkv(2, 4, 2, Sq, Sk, 64, dt, seed=Sq + int(causal))
    ops = _operands(q, k, "cuda", gran)
    _, lse, bd = _restate(ops, v, dt, is_causal=causal, bound=True)
    oe, le = O.attn_int8_fp16_cuda(ops[0], ops[2], v, ops[1], ops[3], qk_quant_gran=gran, is_causal=causal, sm_scale=64 ** -0.5,
                                   out_dtype=torch.float32, return_lse=True)
    assert _within(oe, bd, 0.0) <= 1.0
    assert ((le.double() - lse).abs() <= bd.lse_bound + 1e-6).all()


@pytest.mark.parametrize("kind", ["none", "bool", "bias"])
@pytest.mark.parametrize("dt", [F16, BF])
def test_triton_path_equals_the_reference_triton_restatement(kind, dt):
    """Masks where the two agree: key 0 visible to every row (bool), bias 0 there (bias, else randn * 4 and a quarter -inf)."""
    q, k, v = _qkv(1, 4, 2, 200, 333, 64, dt, seed=7)
    ops = _operands(q, k, "triton")
    g = torch.Generator().manual_seed(3)
    mask = None
    if kind == "bool":
        mask = torch.rand(1, 4, 200, 333, generator=g) < 0.4
        mask[..., 0] = True
    elif kind == "bias":
        mask = 4.0 * torch.randn(1, 4, 200, 333, generator=g)
        mask[torch.rand(mask.shape, generator=g) < 0.25] = -math.inf
        mask[..., 0] = 0.0
        mask = mask.to(dt)
    _, lse, bd = _restate(ops, v, dt, mask=mask, bound=True)
    oe, le = O.attn_int8_fp16_triton(ops[0], ops[2], v, ops[1], ops[3], out_dtype=torch.float32, return_lse=True, attn_mask=mask)
    assert _within(oe, bd, 2.0 ** -11 * bd.mag) <= 1.0
    assert ((le.double() - lse).abs() <= bd.lse_bound + 1e-6).all()


def test_row_chunks_equal_the_whole_call():
    q, k, v = _qkv(1, 2, 1, 333, 333, 64, F16, seed=5)
    ops = _operands(q, k, "cuda", "per_thread")
    o, l = _restate(ops, v, F16, is_causal=True)
    for r0, r1 in ((0, 128), (128, 256), (256, 333), (64, 65)):
        oc, lc = _restate((ops[0][:, :, r0:r1],) + ops[1:], v, F16, is_causal=True, q_offset=r0, q_len=333)
        assert torch.equal(oc, o[:, :, r0:r1]) and torch.equal(lc, l[:, :, r0:r1]), (r0, r1)
    rows = torch.tensor([0, 7, 127, 128, 300, 332])
    oc, lc = _restate((ops[0][:, :, rows],) + ops[1:], v, F16, is_causal=True, q_rows=rows, q_len=333)
    assert torch.equal(oc, o[:, :, rows]) and torch.equal(lc, l[:, :, rows])


# ------------------------------------------------------------------------------------------------ 2. the emulation stays inside
EMU_CASES = [("cuda", "per_thread", F16, "ramp", None, False), ("cuda", "per_warp", BF, "peak", None, True),
             ("triton", "per_block", F16, "randn", "bool", False), ("triton", "per_block", BF, "ramp", "bias", False),
             ("triton", "per_block", F16, "peak", "bias40", False)]


def _emu_mask(kind, dt, Sq, Sk, seed):
    g = torch.Generator().manual_seed(seed)
    if kind is None:
        return None
    if kind == "bool":
        m = torch.rand(1, 2, Sq, Sk, generator=g) < 0.3
        m[:, :, :40, :130] = False          # rows whose first tiles are fully masked
        m[:, :, 50] = False                 # a fully masked row
        return m
    m = (torch.randn(1, 2, Sq, Sk, generator=g) * (40.0 if kind == "bias40" else 4.0))
    m[torch.rand(m.shape, generator=g) < 0.2] = -math.inf
    m[:, :, 60] = -math.inf
    m[:, :, 61] = torch.finfo(BF).min
    m[:, :, 62] = torch.finfo(F16).min
    return m.to(dt)


@pytest.mark.parametrize("case", EMU_CASES, ids=lambda c: "-".join(str(x) for x in c))
def test_emulated_kernel_stays_inside_the_bound(case):
    path, gran, dt, kind, mkind, causal = case
    Sq, Sk = (200, 200) if causal else (130, 333)
    q, k, v = _qkv(1, 2, 1, Sq, Sk, 64, dt, seed=11, kind=kind)
    ops = _operands(q, k, path, gran)
    mask = _emu_mask(mkind, dt, Sq, Sk, seed=2)
    _, lse, bd = _restate(ops, v, dt, mask=mask, is_causal=causal, bound=True)
    assert bd.ambiguous > 0, "no ambiguous fp16 P: the emulation flips nothing"
    worst = 0.0
    for s in range(3):
        o_e, l_e = _restate(ops, v, dt, mask=mask, is_causal=causal, emulate=torch.Generator().manual_seed(s))
        worst = max(worst, check_forward(f"emulated {case} seed {s}", o_e, l_e, lse, bd)[0])
    print(f"[emulation] {case}: worst ratio {worst:.3f}, ambiguous {bd.ambiguous} of {bd.visible}, moved {bd.moved} of {bd.rows}")
    if mkind is not None and mkind.startswith("bias"):
        # finfo(bf16).min and -inf rows are fully masked (exact zeros), finfo(fp16).min rows attend over their keys
        assert (bd.lse_bound[:, :, 60:62] == 0).all() and (bd.lse_bound[:, :, 62] > 0).all()


# ------------------------------------------------------------------------------------------------ 3. planted mistakes
def _shift(t, dim, n=1):
    """t read n elements late along dim (the last element repeated)."""
    idx = torch.clamp(torch.arange(t.size(dim)) + n, max=t.size(dim) - 1)
    return t.index_select(dim, idx)


def _mistake(name):
    """(reference output, mutated output, bound, gate) of one planted mistake on an input where it matters."""
    S = 333
    if name in ("mask_key_off", "mask_row_off", "mask_strides_swapped", "bias_natural_log", "bias_after_max"):
        dt = BF
        q, k, v = _qkv(1, 2, 1, S, S, 64, dt, seed=21)
        ops = _operands(q, k, "triton")
        g = torch.Generator().manual_seed(4)
        if name.startswith("bias"):
            mask = (torch.randn(1, 2, S, S, generator=g) * 8.0).to(dt)
        else:
            mask = torch.rand(1, 2, S, S, generator=g) < 0.5
        mut = {"mask_key_off": lambda m: _shift(m, 3), "mask_row_off": lambda m: _shift(m, 2),
               "mask_strides_swapped": lambda m: m.transpose(2, 3), "bias_natural_log": lambda m: (m.double() * O.LOG2E_CU).to(dt),
               "bias_after_max": lambda m: m}[name](mask)
        ref, _, bd = _restate(ops, v, dt, mask=mask, bound=True)
        out, _ = _restate(ops, v, dt, mask=mut, mutation="bias_after_max" if name == "bias_after_max" else None)
        return ref, out, bd, GATE[("triton", dt)]
    if name == "varlen_k_offset":
        lens = [200, 1, 333, 64]
        cu = torch.tensor([0, 200, 201, 534, 598], dtype=torch.int32)
        g = torch.Generator().manual_seed(9)
        q, k, v = (torch.randn(598, 2, 64, generator=g).half() for _ in range(3))
        k = k + torch.randn(1, 2, 64, generator=g).half()
        q8, qs, cqs = O.quant_per_block_int8_varlen_triton(q, cu, 128, 64 ** -0.5 * O.LOG2E_PY)
        k8, ks, cks = O.quant_per_block_int8_varlen_triton(k - k.mean(0, keepdim=True), cu, 64, 1.0)
        k8p = torch.cat([k8, k8[-1:]])
        ref = attn_fp16pv_varlen(q8, k8p, v, qs, ks, cu, cu, cqs, cks, bound=True)
        mut = attn_fp16pv_varlen(q8, k8p, v, qs, ks, cu, cu, cqs, cks, k_shift=1)
        assert len(lens) == len(ref)
        cat = lambda rs, i: torch.cat([r[i].flatten() for r in rs])
        bd = ref[0][4]._replace(o=torch.cat([r[4].o.flatten() for r in ref]), o_bound=torch.cat([r[4].o_bound.flatten() for r in ref]))
        return cat(ref, 2), cat(mut, 2), bd, GATE[("triton", F16)]
    dt = F16
    kind = "ramp" if name == "skip_alpha" else "randn"
    q, k, v = _qkv(1, 2, 1, S, S, 64, dt, seed=31, kind=kind)
    path = "cuda" if name == "causal_off_by_one" else "triton"
    ops = _operands(q, k, path, "per_warp")
    causal = name == "causal_off_by_one"
    ref, _, bd = _restate(ops, v, dt, is_causal=causal, bound=True)
    if name == "causal_off_by_one":
        out, _ = _restate(ops, v, dt, mask=torch.ones(S, S, dtype=torch.bool).tril(1))
    elif name == "k_scale_neighbour":
        ks = ops[3].clone()
        ks[..., 1] = ks[..., 2]
        out, _ = _restate(ops[:3] + (ks,) + ops[4:], v, dt)
    elif name == "partial_tile_dropped":
        n = S // 64 * 64
        out, _ = _restate(ops[:2] + (ops[2][:, :, :n],) + ops[3:], v[:, :, :n], dt)
    else:
        out, _ = _restate(ops, v, dt, mutation=name)
    return ref, out, bd, GATE[(path, dt)]


MISTAKES = ["mask_key_off", "mask_row_off", "mask_strides_swapped", "bias_natural_log", "bias_after_max", "skip_alpha", "p_bf16",
            "k_scale_neighbour", "partial_tile_dropped", "causal_off_by_one", "varlen_k_offset"]


@pytest.mark.parametrize("name", MISTAKES)
def test_planted_mistakes_break_the_bound(name):
    ref, out, bd, gate = _mistake(name)
    ratio = float(elementwise_ratio(out, bd.o, bd.o_bound).max())
    maxabs = float((out.double() - ref.double()).abs().max())
    caught = not (maxabs <= gate)        # the gate's test also asserts a finite output
    print(f"[mistake] {name:22s} worst error / bound {ratio:10.3g}   max abs {maxabs:.3e}   gate {gate:.2e} "
          f"{'caught' if caught else 'NOT caught'} by the max-abs gate")
    assert ratio > 1.0, f"{name}: the bound does not catch it (worst ratio {ratio:.3g})"


# ------------------------------------------------------------------------------------------------ 4. the GPU file's coverage guard
def test_the_gpu_file_guards_every_fp16pv_instantiation():
    """tests/test_gpu_fp16pv_forward_edges.py asserts at import that its case lists launch every kPV16 instantiation of attn.cu:
    a new instantiation, or a case list that loses one, breaks that equality."""
    import os
    import test_gpu_fp16pv_forward_edges as G
    src = open(os.path.join(G.ROOT, "sageattention_b200", "csrc", "attn.cu")).read()
    assert G.source_pv16_instantiations(src) == G.case_pv16_instantiations() and len(G._SRC) == 12
    extra = src + "\n  return launch_attn<96, false, __half, true, true>(tq, tk, tv, p, grid, s);\n"
    assert G.source_pv16_instantiations(extra) != G.case_pv16_instantiations()
    saved = list(G.MASK_CASES)
    try:
        del G.MASK_CASES[0]
        assert G.source_pv16_instantiations(src) != G.case_pv16_instantiations()
    finally:
        G.MASK_CASES[:] = saved


# ------------------------------------------------------------------------------------------------ 5. planted mistakes at long S
_LONG = {}


def _long_reference(S):
    """Triton path, fp16, D = 64, one head, non-causal, S keys: the first and last 128-row blocks, restated with the bound."""
    if S not in _LONG:
        q, k, v = _qkv(1, 1, 1, S, S, 64, F16, seed=S)
        ops = _operands(q, k, "triton")
        rows = torch.cat([torch.arange(128), torch.arange(S - 128, S)])
        ops = (ops[0][:, :, rows],) + ops[1:]
        _LONG[S] = (ops, v, rows) + tuple(_restate(ops, v, F16, q_rows=rows, q_len=S, bound=True))
    return _LONG[S]


LONG_MISTAKES = [(32768, n) for n in ("k_scale_neighbour", "p_bf16", "tile_dropped", "v_key_late")] + [(16384, "p_bf16"),
                                                                                                       (16384, "k_scale_neighbour")]


@pytest.mark.parametrize("case", LONG_MISTAKES, ids=lambda c: f"S{c[0]}-{c[1]}")
def test_planted_mistakes_at_long_sequences_break_the_bound(case):
    """One wrong 64-key tile in the middle of a 16K / 32K-key row (or P rounded to bf16 everywhere) must break the bound of the
    in-place accumulation, which grows with the number of tiles."""
    S, name = case
    ops, v, rows, ref, _, bd = _long_reference(S)
    j = S // 128                                  # a tile in the middle
    kw = dict(q_rows=rows, q_len=S)
    if name == "k_scale_neighbour":
        ks = ops[3].clone()
        ks[..., j] = ks[..., j + 1]
        out, _ = _restate(ops[:3] + (ks,) + ops[4:], v, F16, **kw)
    elif name == "tile_dropped":
        keep = torch.cat([torch.arange(64 * j), torch.arange(64 * j + 64, S)])
        ks = torch.cat([ops[3][..., :j], ops[3][..., j + 1:]], dim=-1)
        out, _ = _restate(ops[:2] + (ops[2][:, :, keep], ks) + ops[4:], v[:, :, keep], F16, **kw)
    elif name == "v_key_late":
        vm = v.clone()
        vm[:, :, 64 * j:64 * j + 64] = v[:, :, 64 * j + 1:64 * j + 65]
        out, _ = _restate(ops, vm, F16, **kw)
    else:
        out, _ = _restate(ops, v, F16, mutation=name, **kw)
    ratio = float(elementwise_ratio(out, bd.o, bd.o_bound).max())
    maxabs = float((out.double() - ref.double()).abs().max())
    print(f"[mistake] S={S} {name:18s} worst error / bound {ratio:10.3g}   max abs {maxabs:.3e}   gate {GATE[('triton', F16)]:.2e} "
          f"{'caught' if not maxabs <= GATE[('triton', F16)] else 'NOT caught'} by the max-abs gate")
    assert ratio > 1.0, f"S={S} {name}: the bound does not catch it (worst ratio {ratio:.3g})"
