"""GPU tests (-m gpu) of the FP16-PV forward kernel (sage_attn_fwd_kernel with kPV16, csrc/attn.cu), element by element: the
kernel's raw output and log2 lse against the restatement of tests/attn_fp16pv_oracle.py on the kernel's own quantised operands,
within its bound (attn_window_oracle.check_forward), the restatement evaluated in fp64 on the GPU.  Every case also checks that
the public entry point gives the same bits as the op it calls.
  1. dense: every unmasked kPV16 instantiation through sageattn_qk_int8_pv_fp16_cuda (per_warp, per_thread) and
     sageattn_qk_int8_pv_fp16_triton (per_block, both quantisation backends): Skv 1 .. 4097 against Sq 1 .. 200, causal S 1 .. 257,
     cross lengths, B > 1, GQA 4 and 8, HND and NHD, head dims 40 / 72 / 96 / 112, an explicit sm_scale, smooth_k off;
  2. data that stresses this path: ramp and sink inputs that move the running max, peaked rows whose P reaches fp16 subnormals, V
     with large per-channel offsets, bf16 V beyond fp16's range;
  3. long sequences, where O accumulates in place in the tensor core: whole 128-row blocks at S = 16K and 32K;
  4. attn_mask, bool and bias, every masked instantiation: mask shapes and views, masked regions, bias values, the public lse;
  5. packed sageattn_varlen, fp16 and bf16, and the BASELINE configs[3] shape, every head on whole 128-row blocks.
Scope of 4: the restatement reads the same [B,Hq,Sq,Skv] view of attn_mask (core._expand_mask) that the kernel is given, so this
file checks the kernel's reading of that view (strides, stride-0 broadcasts, bool and bias), not the host's broadcasting of the mask
or the units of the bias (log2, as the reference's Triton kernel adds it); test_gpu_parity.test_triton_path_attn_mask_vs_oracle
compares those end to end with the reference's restatement.
Each test prints its group's worst error / bound ratio, worst lse ratio and share of ambiguous elements ([fp16pv] lines).
Measured on an H100 80GB HBM3 at a 700 W power limit with U_TC16 = 2^-23 (one run; the file took 44 s):
  group       worst o ratio   beyond rounding   worst lse ratio   ambiguous
  dense           0.991           0.923             0.047          9.2e-3
  data            0.986           0.569             0.043          1.8e-2
  long            0.612           0.006             0.028          1.1e-2
  masked          0.992           0.881             0.047          1.4e-2
  packed          0.990           0.965             0.049          8.1e-3
  configs[3]      0.975           0.420             0.048          1.0e-2
The output ratio near 1 is the 16-bit rounding of the output (see _Stats); on the long sequences, where the accumulation term
dominates the bound, the error beyond that rounding used at most 0.006 of it."""
import math
import os
import re

import numpy as np
import pytest
import torch

from attn_fp16pv_oracle import attn_fp16pv, attn_fp16pv_varlen
from attn_window_oracle import check_forward

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BF, FP = torch.bfloat16, torch.float16
LOG2E = 1.44269504


# ------------------------------------------------------------------------------------------------ coverage guard
def source_pv16_instantiations(src):
    """{(D, kKT, OutT, masked)} of the kPV16 kernels attn.cu launches: each SAB_LAUNCH(D, KT, T) launches one unmasked FP16-PV
    kernel, and the masked ones are spelled out as launch_attn<D, KT, T, true, true>."""
    found = {(int(d), kt == "true", t, False) for d, kt, t in re.findall(r"SAB_LAUNCH\((\d+), (true|false), ([\w:]+)\)", src)}
    for d, kt, t, pv16, msk in re.findall(r"launch_attn<(\d+), (true|false), ([\w:]+), (true|false), (true|false)>\(", src):
        if pv16 == "true":
            found.add((int(d), kt == "true", t, msk == "true"))
    return found


def _t(dt):
    return "__nv_bfloat16" if dt == BF else "__half"


# (path, head dim, dtype, gran, layout, B, Hq, Hkv, sm_scale or None, smooth_k, quantization_backend)
DENSE_CASES = [
    ("cuda", 64, FP, "per_thread", "HND", 2, 4, 1, None, True, "cuda"),
    ("cuda", 128, BF, "per_thread", "NHD", 1, 8, 1, 0.1, True, "cuda"),
    ("cuda", 96, FP, "per_thread", "HND", 1, 2, 2, None, False, "cuda"),
    ("cuda", 40, BF, "per_thread", "NHD", 2, 4, 2, None, True, "cuda"),
    ("cuda", 128, FP, "per_warp", "NHD", 1, 2, 1, None, True, "cuda"),
    ("cuda", 64, BF, "per_warp", "HND", 2, 4, 4, None, False, "cuda"),
    ("triton", 64, FP, "per_block", "HND", 2, 8, 2, None, True, "cuda"),
    ("triton", 112, BF, "per_block", "NHD", 1, 8, 1, 0.07, True, "triton"),
    ("triton", 128, FP, "per_block", "HND", 1, 4, 4, None, False, "triton"),
    ("triton", 72, BF, "per_block", "HND", 1, 2, 1, None, True, "triton"),
]
# (head dim, dtype, layout, B, Hq, Hkv): the triton entry with attn_mask
MASK_CASES = [(64, FP, "HND", 2, 4, 2), (128, BF, "NHD", 2, 4, 1), (40, BF, "HND", 1, 2, 2), (112, FP, "NHD", 2, 2, 1)]


def _pad(D):
    return 64 if D <= 64 else 128


def case_pv16_instantiations():
    got = {(_pad(c[1]), c[3] == "per_thread", _t(c[2]), False) for c in DENSE_CASES}
    return got | {(_pad(c[0]), False, _t(c[1]), True) for c in MASK_CASES}


# Checked when the module is imported, so also on machines without a GPU: a new kPV16 instantiation needs a case here.
_SRC = source_pv16_instantiations(open(os.path.join(ROOT, "sageattention_b200", "csrc", "attn.cu")).read())
assert len(_SRC) == 12 and case_pv16_instantiations() == _SRC, (
    f"DENSE_CASES / MASK_CASES must launch every kPV16 instantiation of csrc/attn.cu; missing: "
    f"{sorted(_SRC - case_pv16_instantiations(), key=str)}")


# ------------------------------------------------------------------------------------------------ helpers
class _Stats:
    """Worst ratios of one group.  The output's ratio includes its 16-bit rounding, which alone reaches ~0.95 (fp16) / ~0.99
    (bf16) of the tolerance where the bound is small; "beyond rounding" is max(0, |o - ref| - (u + 2^-22) |ref|) / bound, the part
    of the error the rounding cannot explain, over the bound of the module docstring of attn_fp16pv_oracle."""

    def __init__(self, name):
        self.name, self.o, self.lse, self.ex, self.amb, self.vis, self.n = name, 0.0, 0.0, 0.0, 0, 0, 0

    def add(self, ratios, bd, excess=0.0):
        self.o, self.lse, self.ex = max(self.o, ratios[0]), max(self.lse, ratios[1]), max(self.ex, excess)
        self.amb, self.vis, self.n = self.amb + bd.ambiguous, self.vis + bd.visible, self.n + 1

    def report(self):
        print(f"[fp16pv] {self.name}: {self.n} comparisons, worst ratio o {self.o:.3f} (beyond rounding {self.ex:.3f}) lse "
              f"{self.lse:.3f}, ambiguous {self.amb} of {self.vis} ({self.amb / max(self.vis, 1):.2e})")


def _hnd(x, layout):
    return x if layout == "HND" else x.transpose(1, 2)


def _inputs(B, Hq, Hkv, Sq, Sk, D, dt, layout, seed, kind="randn"):
    """HND randn inputs (K with a per-head offset, which smooth_k takes out), in the layout; kind as _data_inputs."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    q = torch.randn(B, Hq, Sq, D, generator=g, device="cuda")
    k = torch.randn(B, Hkv, Sk, D, generator=g, device="cuda") + torch.randn(B, Hkv, 1, D, generator=g, device="cuda")
    v = torch.randn(B, Hkv, Sk, D, generator=g, device="cuda")
    if layout == "NHD":
        q, k, v = (t.transpose(1, 2).contiguous() for t in (q, k, v))
    return q.to(dt), k.to(dt), v.to(dt)


def _run_dense(q, k, v, path, gran, layout, causal=False, sm_scale=None, smooth_k=True, backend="triton", mask=None, lse_api=False):
    """The op the public entry calls, on the entry's own quantised operands, with its raw log2 lse; asserts the public entry gives
    the same output bits.  Returns (o HND [..., :D], lse, restatement kwargs)."""
    import sageattention_b200 as sab
    from sageattention_b200 import ops
    from sageattention_b200.core import _expand_mask, _pad_head_dim, _quant_qk
    from sageattention_b200.quant import transpose_v_f16
    D = q.size(-1)
    sm = sm_scale if sm_scale is not None else D ** -0.5
    qp, kp, vp, _ = _pad_head_dim(q, k, v)
    kind = "fp16_triton" if path == "triton" else "fp16_cuda"
    km, q8, qs, k8, ks, qg, kg, fold = _quant_qk(qp, kp, kind, layout, gran, sm, smooth_k, backend)
    lay = 0 if layout == "NHD" else 1
    o = torch.empty_like(qp)
    vt = transpose_v_f16(vp, tensor_layout=layout)
    if mask is None:
        lse = ops.qk_int8_sv_f16_attn(q8, k8, vt, o, qs, ks, lay, int(causal), qg, kg, sm, fold, 1)
    else:
        lse = ops.qk_int8_sv_f16_attn_masked(q8, k8, vt, o, qs, ks, _expand_mask(mask, qp, kp, layout), lay, qg, kg, sm, fold, 1)
    if path == "triton":
        api = sab.sageattn_qk_int8_pv_fp16_triton(q, k, v, tensor_layout=layout, quantization_backend=backend, is_causal=causal,
                                                  sm_scale=sm_scale, smooth_k=smooth_k, attn_mask=mask, return_lse=lse_api)
    else:
        api = sab.sageattn_qk_int8_pv_fp16_cuda(q, k, v, tensor_layout=layout, is_causal=causal, qk_quant_gran=gran,
                                                sm_scale=sm_scale, smooth_k=smooth_k, return_lse=lse_api)
    o_api = api[0] if lse_api else api
    assert torch.equal(o_api, o[..., :D]), "the public entry and the op it calls differ"
    kw = dict(q8=_hnd(q8, layout), k8=_hnd(k8, layout), v=_hnd(vp, layout), q_scale=qs, k_scale=ks,
              q_gran="per_block" if path == "triton" else gran, fold_sm_scale=bool(fold), sm_scale=sm, is_causal=causal,
              out_dtype=q.dtype, mask=None if mask is None else _hnd_mask(mask, qp, kp, layout))
    if lse_api:
        kw["_api"] = (api[1], _hnd(q, layout), _hnd(k, layout), sm)
    return _hnd(o, layout)[..., :D], lse, kw


def _hnd_mask(mask, qp, kp, layout):
    from sageattention_b200.core import _expand_mask
    return _expand_mask(mask, qp, kp, layout)          # [B,Hq,Sq,Skv] in either layout


def _check(name, o, lse, lr, bd, stats, cols):
    """check_forward on the CPU, on the output columns cols of the restatement's Bound."""
    from attn_bwd_oracle import U
    bd = bd._replace(o=bd.o[..., cols].cpu(), o_bound=bd.o_bound[..., cols].cpu(), lse_bound=bd.lse_bound.cpu(), mag=None)
    ratios = check_forward(name, o, lse, lr.cpu(), bd)
    err = (o.cpu().double() - bd.o).abs() - (U[o.dtype] + 2.0 ** -22) * bd.o.abs()
    ex = torch.where((bd.o_bound > 0) & (err > 0), err / bd.o_bound, 0.0)
    stats.add(ratios, bd, float(ex.max()) if ex.numel() else 0.0)
    return bd


def _compare(name, o, lse, kw, stats, D, rows=None):
    """o / lse against the restatement (all rows, or the LongTensor rows), within the bound."""
    kw = {k: v for k, v in kw.items() if not k.startswith("_")}
    if rows is not None:
        kw["q8"], kw["q_rows"], kw["q_len"] = kw["q8"][:, :, rows.cuda()], rows, o.size(2)
        if kw["mask"] is not None:
            kw["mask"] = kw["mask"][:, :, rows.cuda()]
        o, lse = o[:, :, rows.cuda()], lse[:, :, rows.cuda()]
    _, lr, bd = attn_fp16pv(**kw, return_lse=True, bound=True)
    return lr, _check(name, o, lse, lr, bd, stats, slice(0, D))


# ------------------------------------------------------------------------------------------------ 1. dense tile edges
SKV = [1, 63, 64, 65, 127, 128, 129, 333, 4097]
SQ = [1, 127, 128, 129, 200]
CAUSAL_S = [1, 63, 64, 65, 128, 129, 255, 257]
XLEN = [(4096, 77), (64, 4096)]


def _cid(c):
    return f"{c[0]}-D{c[1]}-{str(c[2])[6:]}-{c[3]}-{c[4]}-B{c[5]}H{c[6]}x{c[7]}-sm{c[8]}-smk{int(c[9])}-{c[10]}"


@pytest.mark.parametrize("i", range(len(DENSE_CASES)), ids=lambda i: _cid(DENSE_CASES[i]))
def test_dense_tile_edges_against_the_bound(i):
    """Each case runs every Skv with a rotating Sq (so the cases together cover every (Sq, Skv) pair), every causal S, and the two
    cross lengths."""
    path, D, dt, gran, layout, B, Hq, Hkv, sm, smk, be = DENSE_CASES[i]
    stats = _Stats(f"dense {_cid(DENSE_CASES[i])}")
    shapes = [(SQ[(i + s) % len(SQ)], sk, False) for s, sk in enumerate(SKV)] + [(s, s, True) for s in CAUSAL_S]
    shapes += [(sq, sk, False) for sq, sk in XLEN]
    for n, (Sq, Sk, causal) in enumerate(shapes):
        q, k, v = _inputs(B, Hq, Hkv, Sq, Sk, D, dt, layout, seed=100 * i + n)
        o, lse, kw = _run_dense(q, k, v, path, gran, layout, causal, sm, smk, be)
        _compare(f"{_cid(DENSE_CASES[i])} {Sq}x{Sk} causal={causal}", o, lse, kw, stats, D)
    stats.report()


# ------------------------------------------------------------------------------------------------ 2. data that stresses the path
def _data_inputs(kind, D, dt, S=1024, H=2, seed=0):
    """ramp48 / ramp160 / sink (test_gpu_kernel_edges._max_inputs): the running max moves on most rows; "peak": q = 8u + randn,
    k = randn + ramp(0..30) u, rows whose logits span ~40 binades (P reaches fp16 subnormals); "voffset": V with per-channel
    offsets of +-300 (|V| ~ 300, spread 1)."""
    from test_gpu_kernel_edges import _max_inputs
    if kind in ("ramp48", "ramp160", "sink"):
        return _max_inputs(D, dt, kind, S=S, H=H, seed=seed)
    g = torch.Generator().manual_seed(seed)
    u = torch.randn(D, generator=g)
    u = u / u.norm()
    q = torch.randn(1, H, S, D, generator=g)
    k = torch.randn(1, H, S, D, generator=g)
    v = torch.randn(1, H, S, D, generator=g)
    if kind == "peak":
        q, k = q + 8.0 * u, k + torch.linspace(0.0, 30.0, S)[:, None] * u
    else:
        v = v + 300.0 * torch.sign(torch.randn(D, generator=g))
    return q.to(dt).cuda(), k.to(dt).cuda(), v.to(dt).cuda()


DATA_CASES = [("cuda", 128, FP, "per_thread", "ramp48", False), ("cuda", 64, BF, "per_warp", "ramp160", True),
              ("triton", 128, BF, "per_block", "sink", False), ("triton", 64, FP, "per_block", "peak", False),
              ("cuda", 64, FP, "per_thread", "peak", True), ("triton", 128, FP, "per_block", "voffset", False),
              ("cuda", 128, BF, "per_warp", "voffset", True)]


@pytest.mark.parametrize("case", DATA_CASES, ids=lambda c: "-".join(str(x).replace("torch.", "") for x in c))
def test_stressing_data_against_the_bound(case):
    path, D, dt, gran, kind, causal = case
    q, k, v = _data_inputs(kind, D, dt)
    o, lse, kw = _run_dense(q, k, v, path, gran, "HND", causal)
    stats = _Stats(f"dense data {case}")
    _, bd = _compare(str(case), o, lse, kw, stats, D)
    stats.report()
    if kind.startswith("ramp") or kind == "sink":
        assert bd.moved >= 0.25 * bd.rows, f"the running max moves on only {bd.moved} of {bd.rows} rows"
    if kind == "peak":
        assert bd.ambiguous > 0


def test_bf16_v_beyond_fp16_range():
    """transpose_v_f16 converts a bf16 V as v.to(torch.float16) does, which the reference's FP16-PV entries run: values beyond
    65504 become inf and values below 2^-24 become fp16 subnormals or 0 (round to nearest).  The kernel's output is then inf or
    NaN in every row of a channel that holds an inf (a row's P16 V sum takes the inf), and within the bound in every other
    channel."""
    from sageattention_b200.quant import transpose_v_f16
    import sageattention_b200 as sab  # noqa: F401
    q, k, v = _inputs(1, 2, 2, 200, 333, 64, BF, "HND", seed=77)
    v = v.clone()
    v[:, :, 5, 3] = 1.0e5                       # beyond fp16: inf
    v[:, :, 9, 7] = -7.0e4                      # -inf
    v[:, :, :, 11] = v[:, :, :, 11] * 1.0e-7    # fp16 subnormals and zeros
    vt = transpose_v_f16(v)
    ref = v.to(FP).transpose(2, 3)
    assert torch.equal(vt[..., :333].view(torch.int16), ref.contiguous().view(torch.int16))
    assert torch.isinf(ref[:, :, 3, 5]).all() and torch.isinf(ref[:, :, 7, 9]).all()
    sub = ref[:, :, 11].abs()
    assert ((sub > 0) & (sub < 2.0 ** -14)).any() and (sub == 0).any()
    o, lse, kw = _run_dense(q, k, v, "triton", "per_block", "HND")
    bad = [3, 7]
    assert not torch.isfinite(o[..., bad]).any(), "a channel holding an inf V must be non-finite in every row"
    keep = [c for c in range(64) if c not in bad]
    kw["v"] = kw["v"].clone()
    kw["v"][..., bad] = 0
    _, lr, bd = attn_fp16pv(**{a: b for a, b in kw.items() if not a.startswith("_")}, return_lse=True, bound=True)
    stats = _Stats("dense bf16 V beyond fp16")
    _check("bf16 V", o[..., keep], lse, lr, bd, stats, keep)
    stats.report()


# ------------------------------------------------------------------------------------------------ 3. long sequences
# (S, D, causal, path, gran, dtype); 16461 has a ragged last block of 77 rows
LONG_CASES = [(16384, 64, False, "cuda", "per_thread", FP), (16384, 128, True, "triton", "per_block", BF),
              (32768, 64, True, "cuda", "per_warp", BF), (32768, 128, False, "triton", "per_block", FP),
              (16461, 128, True, "cuda", "per_thread", FP), (16461, 64, False, "triton", "per_block", BF)]


def _blocks(S, every=None):
    """Rows of whole 128-row blocks: first, middle, last full, ragged last (every: also every block b with b % every == 0)."""
    n = (S + 127) // 128
    sel = {b for b in {0, n // 2, S // 128 - 1, n - 1} if b >= 0} | (set(range(0, n, every)) if every else set())
    return torch.cat([torch.arange(128 * b, min(128 * b + 128, S)) for b in sorted(sel)])


@pytest.mark.parametrize("case", LONG_CASES, ids=lambda c: f"S{c[0]}-D{c[1]}-{'c' if c[2] else 'n'}-{c[3]}-{str(c[5])[6:]}")
def test_long_sequence_blocks_against_the_bound(case):
    S, D, causal, path, gran, dt = case
    q, k, v = _inputs(1, 2, 2, S, S, D, dt, "HND", seed=S + D)
    o, lse, kw = _run_dense(q, k, v, path, gran, "HND", causal)
    stats = _Stats(f"long {case}")
    _compare(str(case), o, lse, kw, stats, D, rows=_blocks(S))
    stats.report()


# ------------------------------------------------------------------------------------------------ 4. attn_mask
def _masks(kind, dt, B, Hq, Sq, Sk, seed):
    """[(name, mask)] of one kind, each broadcastable to [B,Hq,Sq,Skv]: bool (True = visible) or a bias of dtype dt."""
    g = torch.Generator().manual_seed(seed)
    rnd = lambda *s: torch.rand(*s, generator=g)
    lens = torch.randint(1, Sk + 1, (B,), generator=g)
    keys = torch.arange(Sk)
    right = (keys[None, :] < lens[:, None]).view(B, 1, 1, Sk)                 # key padding, right padded
    left = (keys[None, :] >= (Sk - lens)[:, None]).view(B, 1, 1, Sk)          # left padded
    regions = rnd(B, 1, Sq, Sk) < 0.5
    regions[:, :, :70, :200] = False            # rows whose first tiles are fully masked
    regions[:, :, 70:90, :] = False
    regions[:, :, 70:90, Sk - 3:] = True        # rows visible only in the last partial tile
    regions[:, :, 90:95, :] = False             # fully masked rows
    regions[:, :, 128:256, 64:128] = False      # a whole 128 x 64 block
    # (name, mask, sliced): a sliced mask is every other key of a [B,Hq,Sq,2 Skv] tensor on the device, a view with key stride 2
    out = [("2d", rnd(Sq, Sk) < 0.3, False), ("pad-right", right, False), ("pad-left", left, False),
           ("b1qk-regions", regions, False), ("1hqk", rnd(1, Hq, Sq, Sk) < 0.7, False), ("sliced", rnd(B, Hq, Sq, 2 * Sk) < 0.5, True)]

    def dev(m, sliced):
        m = m.cuda()
        return m[..., ::2] if sliced else m
    if kind == "bool":
        return [(n, dev(m, sl)) for n, m, sl in out]
    big = -65504.0 if dt == FP else torch.finfo(BF).min

    def bias(m, scale=4.0):
        b = torch.randn(m.shape, generator=g) * scale
        return torch.where(m, b, -math.inf).to(dt)
    res = [(n + "-inf", dev(bias(m), sl)) for n, m, sl in out]
    b40 = torch.randn(B, Hq, Sq, Sk, generator=g) * 40.0                     # moves the max by tens of binades
    b40[:, :, :, :64] = -40.0
    b40[:, :, 10] = big                                                       # finfo(dt).min on every key of a row
    b40[:, :, 11, :100] = torch.finfo(BF).min if dt == BF else -65504.0
    b40[:, :, 12] = -math.inf
    res.append(("pm40-min", b40.to(dt).cuda()))
    return res


@pytest.mark.parametrize("kind", ["bool", "bias"])
@pytest.mark.parametrize("case", MASK_CASES, ids=lambda c: f"D{c[0]}-{str(c[1])[6:]}-{c[2]}-B{c[3]}H{c[4]}x{c[5]}")
def test_attn_mask_against_the_bound(case, kind):
    """Every mask of _masks at Sq = 300 x Skv = 333 (a partial Q tile, a partial last key tile); fully masked rows (also a
    finfo(bf16).min bias, below the kernel's -5e6 mask value) must be exactly 0 with lse -inf, a finfo(fp16).min bias row
    attends over its keys, and so does a row whose first 100 keys have a finfo(bf16).min bias."""
    D, dt, layout, B, Hq, Hkv = case
    Sq, Sk = 300, 333
    stats = _Stats(f"masked {kind} {case}")
    for n, (name, m) in enumerate(_masks(kind, dt, B, Hq, Sq, Sk, seed=D)):
        q, k, v = _inputs(B, Hq, Hkv, Sq, Sk, D, dt, layout, seed=D + 7 * n)
        if name == "sliced":
            assert m.stride(-1) == 2
        o, lse, kw = _run_dense(q, k, v, "triton", "per_block", layout, mask=m, lse_api=(n == 0))
        lr, bd = _compare(f"{case} {name}", o, lse, kw, stats, D)
        if name == "pm40-min":
            full = [12] + ([10] if dt == BF else [])
            seen = [11] + ([10] if dt == FP else [])
            assert (bd.lse_bound[:, :, full] == 0).all() and (o[:, :, full] == 0).all()
            assert (bd.lse_bound[:, :, seen] > 0).all()
        if n == 0:
            _check_public_lse(kw, lr)
    stats.report()


def _check_public_lse(kw, lr):
    """The public return_lse: the kernel's log2 lse / log2(e) plus the K-mean correction q . mean(k) * sm_scale, taken in the input
    dtype as the reference's core.py takes it, within the 1e-2 that test_every_instantiation_vs_oracle already allows the public
    lse; -inf on rows that see no key."""
    lse_api, q, k, sm = kw["_api"]
    g = q.size(1) // k.size(1)
    km = k.mean(dim=2, keepdim=True).repeat_interleave(g, dim=1)
    want = lr / LOG2E + (q @ km.transpose(-1, -2)).squeeze(-1).double() * sm
    seen = torch.isfinite(lr)
    assert torch.equal(torch.isneginf(lse_api), ~seen)
    err = (lse_api.double() - want)[seen].abs().max().item()
    assert err <= 1e-2, f"public lse off by {err:.3e}"


# ------------------------------------------------------------------------------------------------ 5. packed sageattn_varlen
def _cu(lens):
    return torch.tensor([0] + list(np.cumsum(lens)), dtype=torch.int32, device="cuda")


def _run_varlen(lens_q, lens_k, Hq, Hkv, D, dt, causal, seed, extra_q=0, over=0):
    """sageattn_varlen and the op it calls (output prefilled with a sentinel), on extra_q rows past cu_seqlens_q[-1] and with
    max_seqlen over-stated by `over`.  Returns (o, lse, restatement operands)."""
    import sageattention_b200 as sab
    from sageattention_b200 import ops
    from sageattention_b200.core import _pad_head_dim, _quant_qk_varlen
    from sageattention_b200.quant import transpose_v_f16_varlen
    g = torch.Generator(device="cuda").manual_seed(seed)
    Tq, Tk = sum(lens_q) + extra_q, sum(lens_k)
    q = torch.randn(Tq, Hq, D, generator=g, device="cuda").to(dt)
    k = (torch.randn(Tk, Hkv, D, generator=g, device="cuda") + torch.randn(1, Hkv, D, generator=g, device="cuda")).to(dt)
    v = torch.randn(Tk, Hkv, D, generator=g, device="cuda").to(dt)
    cq, ck = _cu(lens_q), _cu(lens_k)
    mq, mk = max(lens_q) + over, max(lens_k) + over
    sm = D ** -0.5
    qp, kp, vp, _ = _pad_head_dim(q, k, v)
    _, q8, qs, k8, ks, cqs, cks = _quant_qk_varlen(qp, kp, cq, ck, mq, mk, sm, True)
    vt, cpad = transpose_v_f16_varlen(vp, ck, mk)
    o = torch.full(qp.shape, -77.0, dtype=dt, device="cuda")
    lse = ops.qk_int8_sv_f16_attn_varlen(q8, k8, vt, o, qs, ks, cq, ck, cpad, cqs, cks, mq, int(causal), sm, 1, 1)
    api = sab.sageattn_varlen(q, k, v, cq, ck, mq, mk, is_causal=causal)
    T = sum(lens_q)
    assert torch.equal(api[:T], o[:T, :, :D]), "sageattn_varlen and the op it calls differ"
    assert (o[T:] == -77.0).all(), "rows past cu_seqlens_q[-1] must not be written"
    return o[..., :D], lse, (q8, k8, vp, qs, ks, cq, ck, cqs, cks)


def _compare_varlen(name, o, lse, opnds, D, dt, causal, stats, rows=None):
    q8, k8, vp, qs, ks, cq, ck, cqs, cks = opnds
    res = attn_fp16pv_varlen(q8, k8, vp, qs, ks, cq.cpu(), ck.cpu(), cqs.cpu(), cks.cpu(), rows=rows, is_causal=causal,
                             out_dtype=dt, bound=True)
    cqc = cq.cpu()
    for b, r, _, lr, bd in res:
        idx = (int(cqc[b]) + r).cuda()
        ob = o[idx].transpose(0, 1)[None]
        lb = lse[:, idx][None]
        _check(f"{name} sequence {b}", ob, lb, lr, bd, stats, slice(0, D))


# (lens_q, lens_k, Hq, Hkv, D): empty and 1-token sequences, Lq != Lk
VARLEN_CASES = [([200, 0, 1, 130, 77], [333, 0, 1, 64, 300], 4, 2, 128), ([1, 300, 0, 64, 129], [257, 100, 0, 1, 129], 2, 2, 64),
                ([65, 128, 5], [3, 200, 128], 8, 1, 96),
                ([100, 50, 30], [0, 130, 0], 4, 2, 64)]        # rows with no key at all (Lk = 0): zeros and lse -inf


@pytest.mark.parametrize("dt", [FP, BF])
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("case", VARLEN_CASES, ids=lambda c: f"D{c[4]}-H{c[2]}x{c[3]}-{len(c[0])}seq")
def test_packed_varlen_edges_against_the_bound(case, causal, dt):
    lq, lk, Hq, Hkv, D = case
    o, lse, opnds = _run_varlen(lq, lk, Hq, Hkv, D, dt, causal, seed=D + int(causal), extra_q=37, over=70)
    stats = _Stats(f"packed {case} causal={causal} {str(dt)[6:]}")
    _compare_varlen(str(case), o, lse, opnds, D, dt, causal, stats)
    stats.report()


CONFIG3_LENS = [4096, 512, 16384, 1024, 8192, 2048]


@pytest.mark.parametrize("causal", [False, True])
def test_config3_varlen_every_head_against_the_bound(causal):
    """BASELINE configs[3]: lens 4096, 512, 16384, 1024, 8192, 2048; Hq = 32, Hkv = 8; D = 128; bf16: every head on whole 128-row
    blocks of each sequence (first, middle, last)."""
    o, lse, opnds = _run_varlen(CONFIG3_LENS, CONFIG3_LENS, 32, 8, 128, BF, causal, seed=3)
    stats = _Stats(f"configs[3] causal={causal}")
    _compare_varlen("configs[3]", o, lse, opnds, 128, BF, causal, stats, rows=_blocks)
    stats.report()
