"""GPU tests (-m gpu) of the paths of the sm_90a attention kernel (csrc/attn.cu) that the parity suite cannot see:
  B. the O rescale of the lazy running max, on inputs that make the max move (default kernel and SAB_ATTN_KERNEL=exact);
  C. segmented K/V (kv_seg_len, causal_q_offset) and the flag-polling entry point, on one GPU;
  D. every template instantiation of the kernel, reached through the public entry points;
  E. the smooth_v (V mean) quantiser and epilogue;
  F. whole 128-row blocks of 16K / 32K-token sequences;
  G. cross-length dense inputs, varlen batches with empty and 1-token sequences, strided (packed qkv) inputs.
The kernel is compared with the CPU oracle (oracle/sage_oracle.py) run on the kernel's own quantised operands with the kernel's
arithmetic, or with itself where the arithmetic is the same (bit identity).

Tolerances of the kernel-vs-oracle comparisons (stated once):
  TOL_ELEM  every element within 2e-2 + one output ulp: exact exp2 on the CPU vs ex2.approx on the GPU can flip the e4m3 rounding
            of an isolated P, and one flipped top-binade P (7 %) on a peaked row moves its output by up to ~1e-2 (as in
            test_gpu_parity.py); the 16-bit rounding of the result adds one ulp (2^-5 for a bf16 output in [4, 8));
  ULP_FRAC  at least 98 % of elements within one output ulp + 2e-4 (P, m and d are the oracle's; only the fp32 accumulation order
            and those rare flips differ);
  TOL_LSE   LSE within 5e-4 in log2 units (d is summed from un-rounded fp32 P on both sides).
A wrong register index or offset in any of the paths above moves most rows of a case, not a few elements."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from test_gpu_parity import LAZY_TAU, ROOT, _kernel_tau, _mk, _out_ulp, env  # noqa: F401  (env: fixture)

pytestmark = pytest.mark.gpu

TOL_ELEM = 2e-2
ULP_FRAC = 0.98
TOL_LSE = 5e-4
GRAN = {"per_warp": 2, "per_thread": 3}      # SAB_GRAN_PER_WARP / SAB_GRAN_PER_THREAD
BM = 128


def _assert_matches_oracle(o, oe, lse=None, le=None, what=""):
    """o: kernel output (16-bit, any device), oe: oracle output of the same shape; lse / le in log2 units."""
    dt = o.dtype
    o, oe = o.float().cpu(), oe.float().cpu()
    assert torch.isfinite(o).all(), what
    err = (o - oe).abs()
    ulp = _out_ulp(oe, dt)
    assert (err <= TOL_ELEM + 1.01 * ulp).all(), f"{what}: max abs {err.max().item():.3e}"
    good = (err <= 1.01 * ulp + 2e-4).float().mean().item()
    assert good >= ULP_FRAC, f"{what}: only {good:.4f} of elements within 1 ulp + 2e-4 (max abs {err.max().item():.3e})"
    if lse is not None:
        d = (lse.float().cpu() - le).abs().max().item()
        assert d <= TOL_LSE, f"{what}: lse differs by {d:.3e}"


def _quant(q, k, v, gran, layout="HND", scale_max=448.0, smooth_v=False):
    """The kernel's own quantised operands (the product quantisers, K smoothed by its mean as sageattn does)."""
    import sageattention_b200 as sab
    km = sab.k_mean(k, layout)
    q8, qs, k8, ks = (sab.per_warp_int8 if gran == "per_warp" else sab.per_thread_int8)(q, k, km, tensor_layout=layout)
    v8, vs, vm = sab.per_channel_fp8(v, tensor_layout=layout, scale_max=scale_max, smooth_v=smooth_v)
    return q8, qs, k8, ks, v8, vs, vm


def _hnd_cpu(x, layout):
    return (x if layout == "HND" else x.transpose(1, 2)).cpu()


def _v_logical(v8, Skv):
    """[B,Hk,D,S_pad] e4m3 as the oracle's logical [B,Hk,Skv,D]."""
    return v8[..., :Skv].transpose(2, 3).contiguous().cpu()


def _oracle(q8, qs, k8, ks, v8, vs, gran, causal, sm, dt, tau, layout="HND", v_mean=None, causal_q_offset=0, Skv=None):
    from oracle import sage_oracle as O
    Skv = Skv if Skv is not None else (k8.shape[2] if layout == "HND" else k8.shape[1])
    return O.attn_int8_fp8_cuda(_hnd_cpu(q8, layout), _hnd_cpu(k8, layout), _v_logical(v8, Skv), qs.cpu(), ks.cpu(), vs.cpu(),
                                qk_quant_gran=gran, is_causal=causal, sm_scale=sm, pv_accum_dtype="fp32+fp32", out_dtype=dt,
                                return_lse=True, lazy_tau=tau, causal_q_offset=causal_q_offset,
                                v_mean=None if v_mean is None else v_mean.cpu())


# ------------------------------------------------------------------------------------------- B. running-max movement
MAX_CASES = [(D, dt, causal, gran, "ramp48" if i % 2 == 0 else "ramp160")
             for i, (D, dt, causal, gran) in enumerate((D, dt, c, g) for D in (64, 128) for dt in (torch.float16, torch.bfloat16)
                                                       for c in (False, True) for g in ("per_warp", "per_thread"))]
MAX_CASES += [(128, torch.float16, False, "per_thread", "sink"), (64, torch.bfloat16, False, "per_warp", "sink")]


def _max_inputs(D, dt, kind, S=1024, H=2, seed=0):
    """Q = randn + 2u, K = randn + ramp(s) u with u a unit vector and the ramp running from 0 to R along the sequence: the scores
    grow along the keys, so the running max keeps moving (on the CPU oracle at S=1024, D=128: R=48 moves the lazy max of 92 % of
    rows, 2.1 times on average; R=160 of 96 %, 6.5 times).  "sink": plain randn K plus ONE key in the last tile whose score
    jumps ~12 binades above every other, so every row moves its max on the last tile."""
    g = torch.Generator().manual_seed(seed)
    u = torch.randn(D, generator=g)
    u = u / u.norm()
    q = torch.randn(1, H, S, D, generator=g) + 2.0 * u
    k = torch.randn(1, H, S, D, generator=g)
    if kind == "sink":
        S = S - 24                                        # partial last K tile, the sink inside it
        q, k = q[:, :, :S], k[:, :, :S]
        k[:, :, S - 5] += 48.0 * u
    else:
        R = 48.0 if kind == "ramp48" else 160.0
        k = k + torch.linspace(0.0, R, S)[:, None] * u
    v = torch.randn(1, H, S, D, generator=g)
    return q.to(dt).cuda(), k.to(dt).cuda(), v.to(dt).cuda()


def _lazy_max_moves(q8, qs, k8, ks, gran, causal, sm):
    """Fraction of rows whose lazy running max (tau = LAZY_TAU) moves after the first tile, restated from the oracle's rule."""
    from oracle import sage_oracle as O
    q8, qs, k8, ks = q8.cpu(), qs.cpu(), k8.cpu(), ks.cpu()
    Sq, Sk = q8.shape[2], k8.shape[2]
    sm2 = torch.tensor(sm, dtype=torch.float32) * torch.tensor(O.LOG2E_CU, dtype=torch.float32)
    coef = (sm2 * O._expand_q_scale(qs, gran, Sq)[:, :, :Sq])[..., None] * O._expand_k_scale(ks, gran, Sk)[:, :, None, :Sk]
    s = (q8.float() @ k8.float().transpose(-1, -2)) * coef
    if causal:
        s = s.masked_fill(torch.arange(Sk)[None, :] > torch.arange(Sq)[:, None], O.MASK_VALUE)
    m = torch.full(s.shape[:3], O.MASK_VALUE)
    moved = torch.zeros(s.shape[:3], dtype=torch.bool)
    for j, s0 in enumerate(range(0, Sk, 64)):
        m_true = torch.maximum(m, s[..., s0:s0 + 64].amax(-1) - (O.S_FP8_OFFSET - LAZY_TAU))
        mv = m_true - m > LAZY_TAU
        if j > 0:
            moved |= mv
        m = torch.where(mv, m_true, m)
    return moved.float().mean().item()


def _check_max_case(case):
    import sageattention_b200 as sab
    from sageattention_b200 import ops
    D, dt, causal, gran, kind = case
    q, k, v = _max_inputs(D, dt, kind)
    sm = D ** -0.5
    q8, qs, k8, ks, v8, vs, _ = _quant(q, k, v, gran)
    o = torch.empty_like(q)
    lse = ops.qk_int8_sv_f8_attn(q8, k8, v8, o, qs, ks, vs, None, 1, int(causal), GRAN[gran], GRAN[gran], sm, 0, 1)
    torch.cuda.synchronize()
    frac = _lazy_max_moves(q8, qs, k8, ks, gran, causal, sm)
    # the suite's ordinary inputs move it on < 1 % of rows; causal rows early in the sequence see little of the ramp
    assert frac >= 0.25, f"{case}: the lazy max moves on only {frac:.2f} of rows; the input does not exercise the rescale"
    oe, le = _oracle(q8, qs, k8, ks, v8, vs, gran, causal, sm, dt, _kernel_tau(D))
    _assert_matches_oracle(o, oe, lse, le, str(case))
    return frac


@pytest.mark.parametrize("case", MAX_CASES, ids=lambda c: f"D{c[0]}-{str(c[1])[6:]}-{'c' if c[2] else 'n'}-{c[3]}-{c[4]}")
def test_running_max_moves_vs_oracle(env, case):
    _check_max_case(case)


def test_running_max_moves_vs_oracle_exact_max_kernel():
    """The same cases with SAB_ATTN_KERNEL=exact (the reference's running max, which moves on almost every tile).  The kernel
    choice is read once per process, so the check runs in a subprocess."""
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    env_ = dict(os.environ, SAB_ATTN_KERNEL="exact")
    code = ("import sys; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
            "import test_gpu_kernel_edges as T\n"
            "assert T._kernel_tau(128) is None\n"
            "for c in T.MAX_CASES:\n    T._check_max_case(c)\n"
            "print('EXACT_OK')\n" % (ROOT, os.path.join(ROOT, "tests")))
    p = subprocess.run([sys.executable, "-c", code], env=env_, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0 and "EXACT_OK" in p.stdout, p.stdout[-2000:] + p.stderr[-3000:]


# ------------------------------------------------------------------------------------------- C. segmented K/V on one GPU
# (P, causal, gran, D, Hq, Hk, Sl, dtype); Sl % 128 == 0, so the Q tiles and K tiles of a segment are those of the dense call
SEG_CASES = [(2, False, "per_warp", 128, 2, 2, 256, torch.float16),
             (2, True, "per_thread", 64, 2, 2, 256, torch.bfloat16),
             (4, True, "per_warp", 128, 8, 2, 128, torch.bfloat16),
             (4, False, "per_thread", 64, 8, 2, 256, torch.float16),
             (8, True, "per_thread", 128, 2, 2, 128, torch.float16),
             (8, False, "per_warp", 64, 2, 1, 256, torch.bfloat16),
             (2, True, "per_thread", 128, 30, 30, 128, torch.bfloat16),      # the head count of BASELINE configs[4]
             (4, False, "per_warp", 128, 30, 30, 128, torch.float16)]


def _seg_operands(case):
    """The dense call's quantised operands, and K / V^T rearranged into the rank-major layout the sequence-parallel all-gather
    produces ([P*B,Hk,Sl,D] / [P*B,Hk,D,Sl]); K scales keep the dense layout (global 64-key blocks)."""
    P, causal, gran, D, Hq, Hk, Sl, dt = case
    B = 1
    q, k, v = _mk(B, Hq, P * Sl, D, dt, Hk=Hk, seed=P)
    q8, qs, k8, ks, v8, vs, _ = _quant(q, k, v, gran)
    k_all = k8.view(B, Hk, P, Sl, D).permute(2, 0, 1, 3, 4).reshape(P * B, Hk, Sl, D).contiguous()
    v_all = v8.view(B, Hk, D, P, Sl).permute(3, 0, 1, 2, 4).reshape(P * B, Hk, D, Sl).contiguous()   # B=1: reshape is a view
    return q8, qs, k8, ks, v8, vs, k_all, v_all


def _q_segment(q8, qs, r, P, Sl):
    """Rank r's Q block and its Q scales."""
    B, Hq = q8.shape[:2]
    return q8[:, :, r * Sl:(r + 1) * Sl], qs.view(B, Hq, P, -1)[:, :, r].contiguous()


@pytest.mark.parametrize("case", SEG_CASES, ids=lambda c: f"P{c[0]}-{'c' if c[1] else 'n'}-{c[2]}-D{c[3]}-H{c[4]}x{c[5]}")
def test_segmented_kv_is_bit_identical_to_dense(env, case):
    """qk_int8_sv_f8_attn(..., causal_q_offset=r*Sl, kv_seg_len=Sl) on rank r's Q block == rows r*Sl.. of the dense call, output
    and LSE bit for bit: the segment-major TMA coordinates, the causal offset in the tile count, the mask and the causal limit
    change where the data comes from, not the arithmetic."""
    sab, ops, O = env
    P, causal, gran, D, Hq, Hk, Sl, dt = case
    q8, qs, k8, ks, v8, vs, k_all, v_all = _seg_operands(case)
    g, sm = GRAN[gran], D ** -0.5
    o = torch.empty(q8.shape, dtype=dt, device="cuda")
    lse = ops.qk_int8_sv_f8_attn(q8, k8, v8, o, qs, ks, vs, None, 1, int(causal), g, g, sm, 0, 1)
    for r in range(P):
        qr, qsr = _q_segment(q8, qs, r, P, Sl)
        orr = torch.empty(qr.shape, dtype=dt, device="cuda")
        lr = ops.qk_int8_sv_f8_attn(qr, k_all, v_all, orr, qsr, ks, vs, None, 1, int(causal), g, g, sm, 0, 1, r * Sl, Sl)
        rows = slice(r * Sl, (r + 1) * Sl)
        assert torch.equal(orr, o[:, :, rows]), (case, r, (orr.float() - o[:, :, rows].float()).abs().max().item())
        assert torch.equal(lr, lse[:, :, rows]), (case, r)


@pytest.mark.parametrize("case", [c for c in SEG_CASES if not c[1]], ids=lambda c: f"P{c[0]}-{c[2]}-D{c[3]}-H{c[4]}x{c[5]}")
def test_flag_polling_entry_is_bit_identical_to_dense(env, case):
    """qk_int8_sv_f8_attn_sp (the fused-gather entry whose producer polls one flag per (KV-head group, segment)) with EVERY flag
    raised to the call's epoch in stream order before the launch, so the producer never waits: bit-identical to the dense call
    for 1, Hk/2 and Hk heads per flag (the flag index (hk / heads_per_flag) * P + seg)."""
    sab, ops, O = env
    P, causal, gran, D, Hq, Hk, Sl, dt = case
    q8, qs, k8, ks, v8, vs, k_all, v_all = _seg_operands(case)
    g, sm = GRAN[gran], D ** -0.5
    o = torch.empty(q8.shape, dtype=dt, device="cuda")
    ops.qk_int8_sv_f8_attn(q8, k8, v8, o, qs, ks, vs, None, 1, 0, g, g, sm, 0, 0)
    epoch = 7
    for hpf in sorted({h for h in (1, Hk // 2, Hk) if h > 0 and Hk % h == 0}):
        flags = torch.full(((Hk // hpf) * P,), epoch, dtype=torch.int32, device="cuda")
        for r in range(P):
            qr, qsr = _q_segment(q8, qs, r, P, Sl)
            orr = torch.empty(qr.shape, dtype=dt, device="cuda")
            ops.qk_int8_sv_f8_attn_sp(qr, k_all, v_all, orr, qsr, ks, vs, g, g, sm, Sl, flags, epoch, hpf)
            assert torch.equal(orr, o[:, :, r * Sl:(r + 1) * Sl]), (case, hpf, r)
        epoch += 1


# ------------------------------------------------------------------------------------------- D. every instantiation
# (entry point, head dim, dtype, variant): variant = Q/K granularity, or the attn_mask kind of the masked entry
INST_CASES = [(e, D, dt, gran) for e in ("fp8", "fp16") for D in (64, 128) for dt in (torch.float16, torch.bfloat16)
              for gran in ("per_warp", "per_thread")]
INST_CASES += [("triton", D, dt, None) for D in (64, 128) for dt in (torch.float16, torch.bfloat16)]
INST_CASES += [("triton_mask", 64, torch.float16, "bool"), ("triton_mask", 64, torch.bfloat16, "bias"),
               ("triton_mask", 128, torch.float16, "bias"), ("triton_mask", 128, torch.bfloat16, "bool")]


def _instantiation(case):
    """The kernel template sage_attn_fwd_kernel<D, kKT, OutT, kPV16, kMask> a case launches (csrc/attn.cu attn_entry)."""
    entry, D, dt, variant = case
    out = "__nv_bfloat16" if dt == torch.bfloat16 else "__half"
    kt = entry in ("fp8", "fp16") and variant == "per_thread"
    return (D, kt, out, entry != "fp8", entry == "triton_mask")


def _source_instantiations():
    """Every instantiation attn_entry can launch, read from csrc/attn.cu: each SAB_LAUNCH(D, KT, T) launches the FP8-PV and
    the FP16-PV kernel; the masked launches are spelled out."""
    src = open(os.path.join(ROOT, "sageattention_b200", "csrc", "attn.cu")).read()
    found = set()
    for d, kt, t in re.findall(r"SAB_LAUNCH\((\d+), (true|false), ([\w:]+)\)", src):
        for pv16 in (False, True):
            found.add((int(d), kt == "true", t, pv16, False))
    for d, kt, t, pv16, msk in re.findall(r"launch_attn<(\d+), (true|false), ([\w:]+), (true|false), (true|false)>\(", src):
        found.add((int(d), kt == "true", t, pv16 == "true", msk == "true"))
    return found


# Checked when the module is imported, so also on machines without a GPU: a new kernel instantiation needs a case here.
_SRC_INST = _source_instantiations()
assert len(_SRC_INST) == 20 and {_instantiation(c) for c in INST_CASES} == _SRC_INST, (
    "INST_CASES must launch every kernel instantiation of csrc/attn.cu; missing: "
    f"{sorted(_SRC_INST - {_instantiation(c) for c in INST_CASES}, key=str)}")


@pytest.mark.parametrize("case", INST_CASES, ids=lambda c: f"{c[0]}-D{c[1]}-{str(c[2])[6:]}-{c[3]}")
def test_every_instantiation_vs_oracle(env, case):
    """S=333 (a partial last K tile and a partial Q tile), GQA 2:1, return_lse.  The CUDA-semantics entries (fp8, fp16) equal the
    kernel on the product quantisers' operands, which is compared with the oracle on those same operands (the oracle's own
    per-warp quantiser uses IEEE division, so end to end the operands themselves could differ): fp8 at the criteria above, fp16 at
    test_gpu_parity.py's 2e-3 (+ one bf16 ulp) and LSE 1e-3.  The Triton entries quantise bit-exactly and are compared end to end,
    at test_gpu_parity.py's 4e-3 (fp16) / 2e-2 (bf16) and LSE 1e-2."""
    sab, ops, O = env
    entry, D, dt, variant = case
    causal = entry in ("fp8", "fp16") and D == 64
    sm = D ** -0.5
    q, k, v = _mk(1, 4, 333, D, dt, Hk=2, seed=D)
    o = torch.empty_like(q)
    if entry == "fp8":
        o_api, lse_api = sab.sageattn_qk_int8_pv_fp8_cuda(q, k, v, is_causal=causal, qk_quant_gran=variant, pv_accum_dtype="fp32+fp32",
                                                          return_lse=True)
        q8, qs, k8, ks, v8, vs, _ = _quant(q, k, v, variant)
        lse = ops.qk_int8_sv_f8_attn(q8, k8, v8, o, qs, ks, vs, None, 1, int(causal), GRAN[variant], GRAN[variant], sm, 0, 1)
        assert torch.equal(o_api, o), case
        oe, le = _oracle(q8, qs, k8, ks, v8, vs, variant, causal, sm, dt, _kernel_tau(D))
        _assert_matches_oracle(o, oe, lse, le, str(case))
    elif entry == "fp16":
        o_api, lse_api = sab.sageattn_qk_int8_pv_fp16_cuda(q, k, v, is_causal=causal, qk_quant_gran=variant, return_lse=True)
        q8, qs, k8, ks, _, _, _ = _quant(q, k, v, variant)
        lse = ops.qk_int8_sv_f16_attn(q8, k8, sab.transpose_v_f16(v), o, qs, ks, 1, int(causal), GRAN[variant], GRAN[variant], sm, 0, 1)
        assert torch.equal(o_api, o), case
        oe, le = O.attn_int8_fp16_cuda(q8.cpu(), k8.cpu(), v.cpu(), qs.cpu(), ks.cpu(), qk_quant_gran=variant, is_causal=causal,
                                       sm_scale=sm, out_dtype=dt, return_lse=True)
        tol = 2e-3 + (2.0 ** -7 if dt == torch.bfloat16 else 0.0)
        assert (o.cpu().float() - oe.float()).abs().max().item() <= tol, case
        assert (lse.cpu() - le).abs().max().item() <= 1e-3, case
    else:
        mask = None
        if entry == "triton_mask":
            g = torch.Generator().manual_seed(D)
            if variant == "bool":
                mask = torch.rand(333, 333, generator=g) < 0.5
                mask[..., 0] = True
            else:
                mask = torch.randn(1, 4, 333, 333, generator=g)
                mask[torch.rand(mask.shape, generator=g) < 0.25] = float("-inf")
                mask[..., 0] = 0.0
                mask = mask.to(dt)
        o_api, lse_api = sab.sageattn_qk_int8_pv_fp16_triton(q, k, v, return_lse=True, attn_mask=None if mask is None else mask.cuda())
        oe, le = O.sageattn_qk_int8_pv_fp16_triton(q.cpu(), k.cpu(), v.cpu(), return_lse=True, attn_mask=mask)
        tol = 4e-3 if dt == torch.float16 else 2e-2
        assert (o_api.cpu().float() - oe.float()).abs().max().item() <= tol, case
        assert (lse_api.cpu() - le).abs().max().item() <= 1e-2, case
    assert o_api.shape == q.shape and lse_api.shape == q.shape[:3] and torch.isfinite(o_api).all() and torch.isfinite(lse_api).all()


# ------------------------------------------------------------------------------------------- E. smooth_v
SMOOTH_CASES = [(1, 2, 1000, 128, torch.float16), (2, 2, 333, 64, torch.bfloat16)]


def _smooth_inputs(B, H, S, D, dt):
    q, k, v = _mk(B, H, S, D, dt, seed=S)
    g = torch.Generator(device="cuda").manual_seed(S + 1)
    v = (v.float() + 3.0 * torch.randn(D, device="cuda", generator=g)).to(dt)     # a per-channel offset
    return q, k, v


@pytest.mark.parametrize("case", SMOOTH_CASES, ids=lambda c: f"B{c[0]}S{c[2]}D{c[3]}-{str(c[4])[6:]}")
def test_smooth_v_quantiser_vs_oracle(env, case):
    """per_channel_fp8(smooth_v=True), dense and fused, against per_channel_fp8_cuda(smooth_v=True): the V mean over the
    16-padded length and the smoothed scales within rtol 1e-5 (fp32 sums in another order; atol 1e-6 for channels whose mean is
    near zero), bytes differ on < 1e-3 of elements (a rounding-boundary value can fall either side after that last-bit
    difference)."""
    sab, ops, O = env
    B, H, S, D, dt = case
    _, _, v = _smooth_inputs(*case)
    e8, es, em = O.per_channel_fp8_cuda(v.cpu(), "HND", 448.0, smooth_v=True)
    for fused in (False, True):
        v8, vs, vm = sab.per_channel_fp8(v, scale_max=448.0, smooth_v=True, fused=fused)
        assert torch.allclose(vm.cpu(), em, rtol=1e-5, atol=1e-6), (case, fused, (vm.cpu() - em).abs().max().item())
        assert torch.allclose(vs.cpu(), es, rtol=1e-5, atol=0), (case, fused)
        got = v8[..., :S].transpose(2, 3).cpu()
        assert (got.view(torch.uint8) != e8.view(torch.uint8)).float().mean().item() < 1e-3, (case, fused)
        assert float(v8[..., S:].float().abs().sum()) == 0.0


@pytest.mark.parametrize("case", SMOOTH_CASES, ids=lambda c: f"B{c[0]}S{c[2]}D{c[3]}-{str(c[4])[6:]}")
def test_smooth_v_attention_vs_oracle(env, case):
    """pv_accum_dtype="fp32", smooth_v=True: the public call equals the kernel on its own quantised operands, and that matches the
    oracle with v_mean (added after * v_scale) at the criteria of B.  End to end against exact fp32 attention, smoothing V is
    more accurate than not smoothing it on this input: on an H100 80GB HBM3 (700 W) the mean error ratio smoothed / plain was
    0.34 (fp16, D=128) and 0.54 (bf16, D=64); the bound 0.75 leaves room for other seeds, not for smoothing that does nothing."""
    sab, ops, O = env
    B, H, S, D, dt = case
    q, k, v = _smooth_inputs(*case)
    sm = D ** -0.5
    q8, qs, k8, ks, v8, vs, vm = _quant(q, k, v, "per_thread", smooth_v=True)
    o = torch.empty_like(q)
    lse = ops.qk_int8_sv_f8_attn(q8, k8, v8, o, qs, ks, vs, vm, 1, 0, 3, 3, sm, 0, 1)
    o_api = sab.sageattn_qk_int8_pv_fp8_cuda(q, k, v, pv_accum_dtype="fp32", smooth_v=True)
    assert torch.equal(o_api, o)
    oe, le = _oracle(q8, qs, k8, ks, v8, vs, "per_thread", False, sm, dt, _kernel_tau(D), v_mean=vm)
    _assert_matches_oracle(o, oe, lse, le, f"smooth_v {case}")
    o_plain = sab.sageattn_qk_int8_pv_fp8_cuda(q, k, v, pv_accum_dtype="fp32", smooth_v=False)
    ex = O.sdpa_fp32(q.cpu(), k.cpu(), v.cpu())
    e_s = (o.cpu().float() - ex).abs().mean().item()
    e_u = (o_plain.cpu().float() - ex).abs().mean().item()
    print(f"smooth_v {case}: mean abs error {e_s:.3e} smoothed vs {e_u:.3e} plain (ratio {e_s / e_u:.3f})")
    assert e_s <= 0.75 * e_u, (case, e_s, e_u)


# ------------------------------------------------------------------------------------------- F. long sequences
# (S, D, causal, gran, dtype); 16461 has a ragged last block of 77 rows
LONG_CASES = [(16384, 64, False, "per_thread", torch.bfloat16), (16384, 64, True, "per_warp", torch.float16),
              (16384, 128, False, "per_warp", torch.float16), (16384, 128, True, "per_thread", torch.bfloat16),
              (32768, 64, False, "per_warp", torch.bfloat16), (32768, 64, True, "per_thread", torch.float16),
              (32768, 128, False, "per_thread", torch.float16), (32768, 128, True, "per_warp", torch.bfloat16),
              (16461, 128, True, "per_thread", torch.float16)]


@pytest.mark.parametrize("case", LONG_CASES, ids=lambda c: f"S{c[0]}-D{c[1]}-{'c' if c[2] else 'n'}-{c[3]}")
def test_long_sequence_blocks_vs_oracle(env, case):
    """B=1, H=2: five whole 128-row blocks (first, quarter, middle, last full, last) against the oracle's block evaluation
    (causal_q_offset) on the kernel's quantised operands, at the criteria of B — drift of the two-level FP8 accumulation or a
    wrong ring phase late in the loop shows in every late row."""
    sab, ops, O = env
    S, D, causal, gran, dt = case
    q, k, v = _mk(1, 2, S, D, dt, seed=S + D)
    sm = D ** -0.5
    q8, qs, k8, ks, v8, vs, _ = _quant(q, k, v, gran)
    o = torch.empty_like(q)
    lse = ops.qk_int8_sv_f8_attn(q8, k8, v8, o, qs, ks, vs, None, 1, int(causal), GRAN[gran], GRAN[gran], sm, 0, 1)
    torch.cuda.synchronize()
    per = 4 if gran == "per_warp" else 32
    n_blk = (S + BM - 1) // BM
    k8c, v8c, ksc, vsc = k8.cpu(), _v_logical(v8, S), ks.cpu(), vs.cpu()
    for bi in sorted({0, n_blk // 4, n_blk // 2, S // BM - 1, n_blk - 1}):
        r0 = bi * BM
        qb = q8[:, :, r0:r0 + BM].cpu()
        qsb = qs[:, :, bi * per:(bi + 1) * per].cpu()
        oe, le = O.attn_int8_fp8_cuda(qb, k8c, v8c, qsb, ksc, vsc, qk_quant_gran=gran, is_causal=causal, sm_scale=sm,
                                      pv_accum_dtype="fp32+fp32", out_dtype=dt, return_lse=True, lazy_tau=_kernel_tau(D),
                                      causal_q_offset=r0)
        _assert_matches_oracle(o[:, :, r0:r0 + BM], oe, lse[:, :, r0:r0 + BM], le, f"{case} block {bi}")


# ------------------------------------------------------------------------------------------- G. cross-length, varlen, strides
# (Sq, Skv, Hq, Hk, D, dtype, gran, layout)
XLEN_CASES = [(4096, 77, 2, 2, 128, torch.float16, "per_thread", "HND"),       # text-encoder cross attention
              (1000, 226, 2, 2, 64, torch.bfloat16, "per_warp", "NHD"),
              (64, 4096, 2, 2, 128, torch.bfloat16, "per_thread", "NHD"),
              (1, 333, 2, 2, 64, torch.float16, "per_warp", "HND"),
              (1000, 226, 8, 1, 128, torch.float16, "per_thread", "HND"),
              (4096, 77, 8, 1, 64, torch.bfloat16, "per_warp", "NHD")]


@pytest.mark.parametrize("case", XLEN_CASES, ids=lambda c: f"{c[0]}x{c[1]}-H{c[2]}x{c[3]}-D{c[4]}-{c[6]}-{c[7]}")
def test_cross_length_vs_oracle(env, case):
    sab, ops, O = env
    Sq, Skv, Hq, Hk, D, dt, gran, layout = case
    q, k, v = _mk(1, Hq, Sq, D, dt, Hk=Hk, Sk=Skv, seed=Sq + Skv)
    if layout == "NHD":
        q, k, v = (t.transpose(1, 2).contiguous() for t in (q, k, v))
    sm = D ** -0.5
    q8, qs, k8, ks, v8, vs, _ = _quant(q, k, v, gran, layout)
    o = torch.empty_like(q)
    lse = ops.qk_int8_sv_f8_attn(q8, k8, v8, o, qs, ks, vs, None, 0 if layout == "NHD" else 1, 0, GRAN[gran], GRAN[gran], sm, 0, 1)
    oe, le = _oracle(q8, qs, k8, ks, v8, vs, gran, False, sm, dt, _kernel_tau(D), layout=layout)
    _assert_matches_oracle(o if layout == "HND" else o.transpose(1, 2), oe, lse, le, str(case))


# (lens_q, lens_k, Hq, Hk, D): an empty sequence in the middle, 1-token sequences, q and k lengths that differ
VARLEN_CASES = [([200, 0, 1, 130, 77], [333, 0, 1, 64, 300], 4, 2, 128),
                ([1, 300, 0, 64, 129], [257, 100, 0, 1, 129], 2, 2, 64)]


@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("case", VARLEN_CASES, ids=lambda c: f"D{c[4]}-H{c[2]}x{c[3]}")
def test_varlen_edges_vs_oracle(env, case, causal):
    """sageattn_varlen against the oracle's restatement of the reference Triton varlen kernels, 4e-3 (fp16, as the varlen
    fixtures); empty sequences write nothing and are skipped by both."""
    sab, ops, O = env
    lq, lk, Hq, Hk, D = case
    g = torch.Generator().manual_seed(D + int(causal))
    q = torch.randn(sum(lq), Hq, D, generator=g).half()
    k = (torch.randn(sum(lk), Hk, D, generator=g) + 2.0 * torch.randn(1, Hk, D, generator=g)).half()
    v = torch.randn(sum(lk), Hk, D, generator=g).half()
    cq = torch.tensor([0] + list(np.cumsum(lq)), dtype=torch.int32)
    ck = torch.tensor([0] + list(np.cumsum(lk)), dtype=torch.int32)
    o = sab.sageattn_varlen(q.cuda(), k.cuda(), v.cuda(), cq.cuda(), ck.cuda(), max(lq), max(lk), is_causal=causal)
    oe = O.sageattn_varlen(q, k, v, cq, ck, max(lq), max(lk), is_causal=causal)
    assert o.shape == q.shape and torch.isfinite(o).all()
    err = (o.cpu().float() - oe.float()).abs()
    assert err.max().item() <= 4e-3, (case, causal, err.max().item())


def _same_bits(f, views):
    """f on strided views == f on .contiguous() copies, bit for bit."""
    a = f(*views)
    b = f(*(t.contiguous() for t in views))
    assert torch.equal(a, b)


def test_strided_inputs_are_bit_identical_to_contiguous(env):
    """Views of a packed qkv tensor (how most models call attention) and row-padded views go through the quantisers' stride
    arguments; the result is the same bits as on contiguous copies."""
    sab, ops, O = env
    g = torch.Generator(device="cuda").manual_seed(21)
    B, S, H, D = 2, 333, 4, 128
    qkv = torch.randn(B, S, 3, H, D, device="cuda", generator=g).half()
    nhd = qkv.unbind(2)                                   # [B,S,H,D], stride_s = 3HD
    hnd = tuple(t.transpose(1, 2) for t in nhd)           # [B,H,S,D]
    for lay, views in (("NHD", nhd), ("HND", hnd)):
        _same_bits(lambda a, b, c: sab.sageattn(a, b, c, tensor_layout=lay), views)
        _same_bits(lambda a, b, c: sab.sageattn(a, b, c, tensor_layout=lay, is_causal=True), views)
        _same_bits(lambda a, b, c: sab.sageattn_qk_int8_pv_fp16_triton(a, b, c, tensor_layout=lay), views)
    padded = tuple(torch.randn(B, H, S, D + 16, device="cuda", generator=g).bfloat16()[..., 8:8 + D] for _ in range(3))
    _same_bits(lambda a, b, c: sab.sageattn(a, b, c), padded)                       # 16-byte aligned row-padded views
    _same_bits(lambda a, b, c: sab.sageattn_qk_int8_pv_fp16_triton(a, b, c), padded)
    lens = [100, 0, 1, 232]
    cu = torch.tensor([0] + list(np.cumsum(lens)), dtype=torch.int32, device="cuda")
    packed = torch.randn(sum(lens), 3, H, 64, device="cuda", generator=g).half().unbind(1)   # [T,H,D], stride_t = 3HD
    _same_bits(lambda a, b, c: sab.sageattn_varlen(a, b, c, cu, cu, max(lens), max(lens)), packed)
    _same_bits(lambda a, b, c: sab.sageattn_varlen(a, b, c, cu, cu, max(lens), max(lens), is_causal=True), packed)


def test_misaligned_and_strided_operands_are_rejected(env):
    """A view 8 bytes off a 16-byte boundary cannot be read with 16-byte vector loads, and a strided V^T operand not with the
    kernel's tensor map: the host checks raise ValueError before any launch."""
    sab, ops, O = env
    B, H, S, D = 1, 2, 200, 64
    mis = tuple(torch.randn(B, H, S, D + 16, device="cuda").half()[..., 4:4 + D] for _ in range(3))
    with pytest.raises(ValueError):
        sab.sageattn(*mis)
    with pytest.raises(ValueError):
        sab.sageattn_qk_int8_pv_fp16_triton(*mis)
    misp = tuple(torch.randn(S, H, D + 16, device="cuda").half()[..., 4:4 + D] for _ in range(3))
    cu = torch.tensor([0, 120, S], dtype=torch.int32, device="cuda")
    with pytest.raises(ValueError):
        sab.sageattn_varlen(*misp, cu, cu, 120, 120)
    # the kernel reads V^T through a tensor map built for the quantisers' packed layout: a strided V operand is refused
    q, k, v = _mk(1, 2, 256, 64, torch.float16)
    q8, qs, k8, ks, v8, vs, _ = _quant(q, k, v, "per_thread")
    v_strided = torch.zeros((*v8.shape[:-1], 512), dtype=torch.uint8, device="cuda").view(torch.float8_e4m3fn)[..., :256]
    with pytest.raises(ValueError):
        ops.qk_int8_sv_f8_attn(q8, k8, v_strided, torch.empty_like(q), qs, ks, vs, None, 1, 0, 3, 3, 0.125, 0, 0)
