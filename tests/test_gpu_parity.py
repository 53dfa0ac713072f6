"""GPU parity tests (-m gpu): the sm_90a kernels, called through the public API / C ABI, against
  (1) the CPU oracle (oracle/sage_oracle.py, pinned to reference-Triton golden fixtures),
  (2) the golden fixtures themselves (tests/golden/*.npz, produced by the real reference Triton kernels),
  (3) the REAL reference CUDA kernels: their outputs on seeded inputs, stored as a fixed sample of rows in
      tests/golden/reference_cuda_kernels.npz (tests/golden/make_reference_cuda_golden.py, run on an H100 with oracle/_ref built).
Tolerances (stated once): quantised tensors and scales bit-exact; attention output max-abs <= 1e-2 against the
reference kernel (north-star tolerance), <= 5e-3 against the oracle run with the kernel's arithmetic."""
import os
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = os.path.join(ROOT, "tests", "golden")
TOL_REF = 1e-2      # north-star tolerance vs the reference kernel
LAZY_TAU = 4        # csrc/attn.cu kLazyTau: the kernel's lazy-max threshold (binades)
REF_GOLDEN = os.path.join(G, "reference_cuda_kernels.npz")
REF_ROWS = 144      # rows of each reference output kept in the golden file (16-bit outputs stored as their bits)


def _kernel_tau(D):
    """Which running-max rule the INT8+FP8 kernel uses: by default a LAZY max (csrc/attn.cu) — it moves only when a P would overflow
    e4m3; SAB_ATTN_KERNEL=exact keeps the reference's exact max.  The oracle restates both (lazy_tau=...), so the CUDA path is always compared with the oracle run with ITS arithmetic;
    against the reference kernel (exact max) a lazy-max result is a different e4m3 rounding realisation of the same P — compared
    statistically."""
    if os.environ.get("SAB_ATTN_KERNEL", "")[:1] == "e":
        return None
    return LAZY_TAU


def assert_close_ulp(a, b, what=""):
    """P, m and d are bit-identical to the reference by construction, so outputs may differ only through fp32
    accumulation order: allow ONE unit in the last place of the 16-bit output format plus 2e-4 absolute."""
    a32, b32 = a.float(), b.float()
    eps = 2.0 ** -10 if a.dtype == torch.float16 else 2.0 ** -7
    mag = torch.maximum(a32.abs(), b32.abs()).clamp_min(2.0 ** -14)
    ulp = torch.exp2(torch.floor(torch.log2(mag))) * eps
    bad = (a32 - b32).abs() > 1.01 * ulp + 2e-4
    assert not bad.any(), f"{what}: {int(bad.sum())} elements differ by more than 1 ulp; max abs {(a32 - b32).abs().max().item():.3e}"


@pytest.fixture(scope="module")
def env():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import sageattention_b200 as sab
    from sageattention_b200 import ops, _capi
    from oracle import sage_oracle as O
    assert _capi.lib().sab_check_device() == 0, "not an sm_90 device"
    return sab, ops, O


def _ref_golden():
    assert os.path.exists(REF_GOLDEN), "tests/golden/reference_cuda_kernels.npz missing"
    return np.load(REF_GOLDEN)


def _row_idx(nrows, seed, n=REF_ROWS):
    """Fixed, seeded sample of row indices (rows of the tensor viewed as [-1, last dim])."""
    return np.sort(np.random.RandomState(seed).choice(nrows, min(n, nrows), replace=False))


def _rows(t, idx):
    """Rows `idx` of t viewed as [-1, t.shape[-1]], as a CPU tensor."""
    return t.reshape(-1, t.shape[-1])[torch.from_numpy(idx).to(t.device)].cpu()


def _golden16(z, key, dt):
    """A stored 16-bit reference output (its bit pattern as int16) as float32."""
    return torch.from_numpy(z[key].copy()).view(dt).float()


def _mk_host(B, H, S, D, dt, Hk=None, seed=0):
    """Inputs of the comparisons with the reference CUDA kernels: drawn on the CPU, so they are the same on every machine."""
    g = torch.Generator().manual_seed(seed)
    Hk = Hk or H
    q = torch.randn(B, H, S, D, generator=g).to(dt)
    k = torch.randn(B, Hk, S, D, generator=g) + 4.0 * torch.randn(B, Hk, 1, D, generator=g)
    v = torch.randn(B, Hk, S, D, generator=g)
    return q.cuda(), k.to(dt).cuda(), v.to(dt).cuda()


def _t(a, dtype):
    return torch.from_numpy(a.copy()).view(dtype)


def _mk(B, H, S, D, dt, Hk=None, outlier=True, seed=0, Sk=None):
    g = torch.Generator(device="cuda").manual_seed(seed)
    Hk, Sk = Hk or H, Sk or S
    q = torch.randn(B, H, S, D, device="cuda", generator=g).to(dt)
    k = torch.randn(B, Hk, Sk, D, device="cuda", generator=g)
    if outlier:
        k = k + 4.0 * torch.randn(B, Hk, 1, D, device="cuda", generator=g)
    v = torch.randn(B, Hk, Sk, D, device="cuda", generator=g)
    return q, k.to(dt), v.to(dt)


def _check_k_mean(got, k, km_torch):
    """K smoothing mean (sageattention/core.py:773 `k.mean(dim=seq)`): torch reduces in fp32 in ITS launch-dependent order and
    rounds to the input dtype; the sm_90a kernel reduces in fp32 in a fixed order (csrc/quant.cu channel_stats).  Both are
    roundings of the same fp32-accurate sum, so they can only differ where the exact mean sits on a rounding boundary of
    the 16-bit format.  Pin: the kernel's value is a CORRECT rounding of the fp64 mean up to the fp32 summation noise
    (half an ulp + 2^-20 relative), and it is bit-identical to torch.mean on all but a handful of channels.  (Given the
    same km, the quantised K and its scales are bit-exact — that is what the quantiser tests pin.)"""
    exact = k.double().mean(dim=2, keepdim=True)
    eps = 2.0 ** -10 if k.dtype == torch.float16 else 2.0 ** -7
    ulp = torch.exp2(torch.floor(torch.log2(exact.abs().clamp_min(2.0 ** -14)))) * eps
    assert ((got.double() - exact).abs() <= 0.5 * ulp * (1 + 1e-3) + exact.abs() * 2.0 ** -20 + 1e-7).all()
    same = (got == km_torch).float().mean().item()
    assert same >= 0.98, f"k_mean equals torch.mean on only {same:.4f} of the channels"
    assert ((got.float() - km_torch.float()).abs() <= 1.001 * ulp.float()).all()      # never more than one 16-bit ulp apart


# ------------------------------------------------------------------------------------------- quantisation
@pytest.mark.parametrize("name", ["quant_d64_fp16", "quant_d128_bf16"])
def test_quant_bit_exact_vs_reference_triton_fixtures(env, name):
    sab, ops, O = env
    z = np.load(f"{G}/{name}.npz")
    dt = torch.bfloat16 if "bfloat16" in str(z["dtype"]) else torch.float16
    q, k, km = (_t(z[n], dt).cuda() for n in ("q", "k", "km"))
    D = q.shape[-1]
    q8, qs, k8, ks = sab.per_block_int8(q, k, km, sm_scale=D ** -0.5)
    for got, key in ((q8, "pb_q8"), (qs, "pb_qs"), (k8, "pb_k8"), (ks, "pb_ks")):
        assert np.array_equal(got.cpu().numpy(), z[key]), key
    q8, qs, k8, ks = sab.per_thread_int8(q, k, km)
    for got, key in ((q8, "pt_q8"), (qs, "pt_qs"), (k8, "pt_k8"), (ks, "pt_ks")):
        assert np.array_equal(got.cpu().numpy(), z[key]), key
    qn, kn = q.transpose(1, 2).contiguous(), k.transpose(1, 2).contiguous()
    q8, qs, k8, ks = sab.per_thread_int8(qn, kn, km.transpose(1, 2), tensor_layout="NHD")
    for got, key in ((q8, "ptn_q8"), (qs, "ptn_qs"), (k8, "ptn_k8"), (ks, "ptn_ks")):
        assert np.array_equal(got.cpu().numpy(), z[key]), key


@pytest.mark.parametrize("shape", [(1, 2, 200, 64, torch.float16), (2, 3, 333, 128, torch.bfloat16), (1, 2, 1, 64, torch.float16),
                                   (1, 1, 129, 128, torch.float16)])
def test_quant_vs_oracle(env, shape):
    sab, ops, O = env
    B, H, S, D, dt = shape
    q, k, v = _mk(B, H, S, D, dt)
    km = k.mean(dim=2, keepdim=True)
    _check_k_mean(sab.k_mean(k), k, km)
    qc, kc, kmc = q.cpu(), k.cpu(), km.cpu()
    for got, exp in ((sab.per_block_int8(q, k, km, sm_scale=D ** -0.5), O.per_block_int8_triton(qc, kc, kmc, sm_scale=D ** -0.5)),
                     (sab.per_thread_int8(q, k, km), O.quant_per_thread_int8_triton(qc, kc, kmc))):
        for g_, e_ in zip(got, exp):
            assert torch.equal(g_.cpu(), e_)                         # Triton semantics: bit exact
    got, exp = sab.per_warp_int8(q, k, km), O.per_warp_int8_cuda(qc, kc, kmc)
    for g_, e_ in zip(got, exp):                                       # CUDA semantics: oracle uses IEEE division
        if g_.dtype == torch.int8:
            d = (g_.cpu().int() - e_.int()).abs()
            assert d.max() <= 1 and (d > 0).float().mean() < 1e-3
        else:
            assert torch.allclose(g_.cpu(), e_, rtol=3e-7, atol=0)
    for smax in (448.0, 2.25):
        v8, vs, _ = sab.per_channel_fp8(v, scale_max=smax, smooth_v=False)
        e8, es, _ = O.per_channel_fp8_cuda(v.cpu(), "HND", smax)
        got8 = v8[..., :S].transpose(2, 3).float().cpu()
        assert v8.shape[-1] % 128 == 0 and float(v8[..., S:].float().abs().sum()) == 0.0     # zero padding
        assert ((got8 - e8.float()).abs() > 0).float().mean() < 1e-3
        assert torch.allclose(vs.cpu(), es, rtol=3e-7, atol=0)


def test_quant_per_thread_bit_exact_at_full_size(env):
    """BASELINE-size tensor (4x32x8192x128): the fast-path/exact-division split of the Triton-semantics quantiser must be
    bit-identical to the plain IEEE formula (quant_per_thread.py:41-44), restated here with torch ops on the GPU."""
    sab, ops, O = env
    g = torch.Generator(device="cuda").manual_seed(9)
    B, H, S, D = 4, 32, 8192, 128
    q = torch.randn(B, H, S, D, device="cuda", generator=g).bfloat16()
    k = (torch.randn(B, H, S, D, device="cuda", generator=g) + 2.0).bfloat16()
    km = k.mean(dim=2, keepdim=True)
    q8, qs, k8, ks = sab.per_thread_int8(q, k, km)
    xf = q.float().view(B, H, S // 32, 4, 8, D)
    c127 = torch.tensor(127.0, device="cuda")   # tensor divisor: torch turns division by a python scalar into a multiply
    sc = xf.abs().amax(dim=(3, 5)) / c127 + 0.0000001
    y = xf / sc[:, :, :, None, :, None]
    e8 = torch.trunc(y + 0.5 * torch.where(y >= 0, 1.0, -1.0)).to(torch.int8).view(B, H, S, D)
    assert torch.equal(qs, sc.reshape(B, H, -1)) and torch.equal(q8, e8)
    kf = (k - km).float().view(B, H, S // 64, 8, 4, 2, D)
    sc = kf.abs().amax(dim=(3, 5, 6)) / c127 + 0.0000001
    y = kf / sc[:, :, :, None, :, None, None]
    e8 = torch.trunc(y + 0.5 * torch.where(y >= 0, 1.0, -1.0)).to(torch.int8).view(B, H, S, D)
    assert torch.equal(ks, sc.reshape(B, H, -1)) and torch.equal(k8, e8)


QREF_CASES = [(2, 3, 333, 128, torch.bfloat16), (1, 2, 1000, 64, torch.float16)]


def test_quant_bit_exact_vs_real_reference_kernels(env):
    """Per-warp Q / per-block K INT8 and per-channel FP8 V against the reference's csrc/fused quantisers (stored rows of their
    output, the reference's 16-token V permutation undone): bit-exact, scales complete."""
    sab, ops, O = env
    z = _ref_golden()
    for ci, (B, H, S, D, dt) in enumerate(QREF_CASES):
        q, k, v = _mk_host(B, H, S, D, dt, seed=ci)
        km = k.mean(dim=2, keepdim=True)
        q8, qs, k8, ks = sab.per_warp_int8(q, k, km)
        ridx = _row_idx(B * H * S, 10 + ci)
        assert np.array_equal(_rows(q8, ridx).numpy(), z[f"quant{ci}_q8"]) and np.array_equal(qs.cpu().numpy(), z[f"quant{ci}_qs"])
        assert np.array_equal(_rows(k8, ridx).numpy(), z[f"quant{ci}_k8"]) and np.array_equal(ks.cpu().numpy(), z[f"quant{ci}_ks"])
        vidx = _row_idx(B * H * D, 20 + ci)
        for smax in (448.0, 2.25):
            v8, vs, _ = sab.per_channel_fp8(v, scale_max=smax, smooth_v=False)
            assert np.array_equal(_rows(v8.view(torch.uint8)[..., :S], vidx).numpy(), z[f"quant{ci}_v8_{smax:g}"])
            assert np.array_equal(vs.cpu().numpy(), z[f"quant{ci}_vs_{smax:g}"])


def test_fused_front_end_matches_the_two_step_calls(env):
    """The single-launch front-end (opt-in): `smooth_quant_k` (K mean + INT8 K in one cluster
    launch) and `per_channel_fp8(fused=True)`.  INT8 / FP8 bytes and scales are bit-identical to the two-step entry points given the
    same mean; the fused mean itself is another fp32 summation order (within one 16-bit ulp of k_mean on rare channels)."""
    sab, ops, O = env
    from sageattention_b200.quant import quant_k_int8, smooth_quant_k
    for (B, Hk, S, D, dt, layout) in [(2, 3, 333, 128, torch.bfloat16, "HND"), (1, 2, 1000, 64, torch.float16, "NHD"), (1, 1, 1, 64, torch.float16, "HND"),
                                      (1, 4, 8192, 128, torch.bfloat16, "HND"), (2, 2, 130, 128, torch.float16, "NHD")]:
        _, k, v = _mk(B, Hk, S, D, dt, Hk=Hk)
        if layout == "NHD":
            k, v = k.transpose(1, 2).contiguous(), v.transpose(1, 2).contiguous()
        km = sab.k_mean(k, layout)
        for gran in ("per_thread", "per_warp"):
            km2, k8b, ksb = smooth_quant_k(k, gran, layout)
            k8, ks = quant_k_int8(k, km2, gran, layout)
            assert torch.equal(k8b, k8) and torch.equal(ksb, ks), (B, Hk, S, D, dt, layout, gran)
            kh = k if layout == "HND" else k.transpose(1, 2)
            _check_k_mean(km2.reshape(B, Hk, 1, D), kh, km.reshape(B, Hk, 1, D))
        for smax in (448.0, 2.25):
            for smooth_v in (False, True):
                v8, vs, vm = sab.per_channel_fp8(v, tensor_layout=layout, scale_max=smax, smooth_v=smooth_v, fused=True)
                r8, rs, rm = sab.per_channel_fp8(v, tensor_layout=layout, scale_max=smax, smooth_v=smooth_v)
                if not smooth_v:     # max / min reductions are order-independent: identical scales and bytes
                    assert torch.equal(v8.view(torch.uint8), r8.view(torch.uint8)) and torch.equal(vs, rs), (B, Hk, S, D, dt, layout, smax)
                else:                # the V mean is an fp32 sum whose order differs between the two kernels: last-bit differences only
                    assert torch.allclose(vm, rm, rtol=1e-5, atol=1e-6) and torch.allclose(vs, rs, rtol=1e-5, atol=0)
                    assert (v8.view(torch.uint8) != r8.view(torch.uint8)).float().mean().item() < 1e-3


# ------------------------------------------------------------------------------------------- attention
CFGS = [
    dict(B=1, H=2, S=320, D=64, dt=torch.float16, causal=False, gran="per_warp", acc="fp32+fp32"),
    dict(B=1, H=2, S=320, D=64, dt=torch.float16, causal=True, gran="per_thread", acc="fp32+fp16"),
    dict(B=2, H=4, S=200, D=128, dt=torch.bfloat16, causal=False, gran="per_thread", acc="fp32+fp16", Hk=2),
    dict(B=1, H=2, S=1000, D=128, dt=torch.float16, causal=True, gran="per_warp", acc="fp32+fp16"),
    dict(B=1, H=2, S=1024, D=128, dt=torch.bfloat16, causal=False, gran="per_thread", acc="fp32+fp32"),
    dict(B=1, H=2, S=77, D=72, dt=torch.float16, causal=False, gran="per_thread", acc="fp32+fp16"),
    dict(B=1, H=3, S=1, D=64, dt=torch.float16, causal=False, gran="per_warp", acc="fp32+fp16"),
    dict(B=1, H=2, S=130, D=40, dt=torch.bfloat16, causal=True, gran="per_thread", acc="fp32"),
    dict(B=1, H=8, S=1024, D=64, dt=torch.float16, causal=False, gran="per_thread", acc="fp32+fp16"),   # BASELINE configs[0]
]


@pytest.mark.parametrize("c", CFGS, ids=lambda c: f"B{c['B']}H{c['H']}S{c['S']}D{c['D']}{'c' if c['causal'] else 'n'}-{c['gran']}-{c['acc']}")
def test_attention_vs_oracle(env, c):
    sab, ops, O = env
    q, k, v = _mk(c["B"], c["H"], c["S"], c["D"], c["dt"], Hk=c.get("Hk"))
    o, lse = sab.sageattn_qk_int8_pv_fp8_cuda(q, k, v, is_causal=c["causal"], qk_quant_gran=c["gran"], pv_accum_dtype=c["acc"], return_lse=True)
    torch.cuda.synchronize()
    tau = _kernel_tau(c["D"])
    kw = dict(is_causal=c["causal"], qk_quant_gran=c["gran"], pv_accum_dtype=c["acc"], return_lse=True, emulate_f16_accum=False)
    oe, le = O.sageattn_qk_int8_pv_fp8_cuda(q.cpu(), k.cpu(), v.cpu(), lazy_tau=tau, **kw)     # the kernel's own arithmetic
    assert o.shape == q.shape and o.dtype == q.dtype and lse.shape == q.shape[:3] and lse.dtype == torch.float32
    assert not torch.isnan(o).any()
    # exact exp2 on the CPU vs ex2.approx on the GPU can flip the e4m3 rounding of an isolated P (prob. ~1e-5/element):
    # demand 1-ulp agreement for all but a handful of elements, and the north-star bound for every element
    err = (o.cpu().float() - oe.float()).abs()
    assert err.max().item() <= 2 * TOL_REF   # one flipped top-binade P (7 %) on a peaked row; the GPU-vs-GPU test below is tight
    eps = 2.0 ** -10 if q.dtype == torch.float16 else 2.0 ** -7
    ulp = torch.exp2(torch.floor(torch.log2(oe.float().abs().clamp_min(2.0 ** -14)))) * eps
    assert (err > 1.01 * ulp + 2e-4).float().mean().item() < 2e-2   # a flipped P touches every column of its row
    # lse = kernel lse (agrees to 1e-4 with the reference kernel, test below) + q.km correction computed by torch.matmul in
    # the INPUT dtype (core.py:782-786): cuBLAS vs CPU rounding of that fp16/bf16 product dominates
    assert (lse.cpu() - le).abs().max().item() <= (1e-2 if q.dtype == torch.float16 else 6e-2)
    if tau is not None:
        # lazy max vs the reference's exact max: another rounding realisation of the same P, not a less accurate one — the error
        # against exact fp32 attention must stay at the exact-max arithmetic's level (mean within 10 %, max within 50 % + 5e-3)
        ox, _ = O.sageattn_qk_int8_pv_fp8_cuda(q.cpu(), k.cpu(), v.cpu(), **kw)
        sd = O.sdpa_fp32(q.cpu(), k.cpu(), v.cpu(), is_causal=c["causal"])
        e_k, e_x = (o.cpu().float() - sd).abs(), (ox.float() - sd).abs()
        assert e_k.mean().item() <= 1.10 * e_x.mean().item() + 1e-4
        assert e_k.max().item() <= 1.5 * e_x.max().item() + 5e-3      # a single-element statistic: loose
    # NHD layout: same numbers through the other stride set
    qn, kn, vn = (t.transpose(1, 2).contiguous() for t in (q, k, v))
    on = sab.sageattn_qk_int8_pv_fp8_cuda(qn, kn, vn, tensor_layout="NHD", is_causal=c["causal"], qk_quant_gran=c["gran"], pv_accum_dtype=c["acc"])
    assert torch.equal(on.transpose(1, 2), o)


ATT_REF_CASES = [(1, 4, 1024, 128, torch.float16, False, "per_warp"), (1, 4, 1024, 64, torch.bfloat16, True, "per_warp"),
                 (2, 4, 2000, 128, torch.bfloat16, False, "per_thread"), (1, 2, 4096, 128, torch.bfloat16, True, "per_thread"),
                 (1, 8, 1024, 64, torch.float16, False, "per_thread"), (1, 2, 333, 128, torch.float16, True, "per_thread")]


def _check_vs_real_reference_kernel(sab, ops, O):
    """The CUDA path against the REAL reference sm89 kernels (qk_int8_sv_f8_accum_f{16,32}_fuse_v_scale_attn_inst_buf) on the same
    quantised operands (stored rows of their output and LSE).
    Exact max (SAB_ATTN_KERNEL=exact): same P / m / d bits as the reference -> <= 4e-3 vs its fp32+fp32 kernel (the residual is the
    reduced-precision accumulator of the reference's legacy fp8 mma.sync), <= 2e-2 vs its fp32+fp16 kernel (that kernel's own per-tile
    f16 rounding, attn_utils.cuh:896-974).  Lazy max (default): a different e4m3 rounding realisation of the same P, so the comparison
    is statistical — mean |diff| <= 2.5e-3, and the error against exact fp32 attention is at the reference kernel's level (mean within
    10 %, max within 50 % + 5e-3).  LSE agrees to 5e-4 (log2 units) in every case."""
    z = _ref_golden()
    worst, worst_mean = 0.0, 0.0
    for ci, (B, H, S, D, dt, causal, gran) in enumerate(ATT_REF_CASES):
        q, k, v = _mk_host(B, H, S, D, dt, seed=100 + ci)
        km = k.mean(dim=2, keepdim=True)
        sm = D ** -0.5
        q8, qs, k8, ks = (sab.per_warp_int8 if gran == "per_warp" else sab.per_thread_int8)(q, k, km)
        g = 2 if gran == "per_warp" else 3
        tau = _kernel_tau(D)
        ridx = _row_idx(B * H * S, 100 + ci)
        sd = _rows(O.sdpa_fp32(q.cpu(), k.cpu(), v.cpu(), is_causal=causal), ridx) if tau is not None else None
        for smax in (2.25, 448.0):
            o_ref = _golden16(z, f"attn{ci}_o_{smax:g}", dt)
            lse_ref = torch.from_numpy(z[f"attn{ci}_lse_{smax:g}"])
            v8, vs, _ = sab.per_channel_fp8(v, scale_max=smax, smooth_v=False)
            o = torch.empty_like(q)
            lse = ops.qk_int8_sv_f8_attn(q8, k8, v8, o, qs, ks, vs, None, 1, int(causal), g, g, sm, 0, 1)
            torch.cuda.synchronize()
            o = _rows(o, ridx).float()
            lse = _rows(lse.reshape(-1, 1), ridx).reshape(-1)
            diff = (o - o_ref).abs()
            err = diff.max().item()
            worst, worst_mean = max(worst, err), max(worst_mean, diff.mean().item())
            if tau is None:
                assert err <= (4e-3 if smax == 448.0 else 2e-2), (B, H, S, D, dt, causal, gran, smax, err)
            else:
                assert diff.mean().item() <= 2.5e-3, (B, H, S, D, dt, causal, gran, smax, diff.mean().item())
                e_k, e_r = (o - sd).abs(), (o_ref - sd).abs()
                assert e_k.mean().item() <= 1.10 * e_r.mean().item() + 1e-4, (B, H, S, D, dt, causal, gran, smax)
                assert e_k.max().item() <= 1.5 * e_r.max().item() + 5e-3, (B, H, S, D, dt, causal, gran, smax)
            assert (lse - lse_ref).abs().max().item() <= 5e-4
    return worst, worst_mean


def _out_ulp(x, dt):
    eps = 2.0 ** -10 if dt == torch.float16 else 2.0 ** -7
    return torch.exp2(torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -14)))) * eps


_A16_CASES = [(1, 4, 1024, 128, torch.float16, False, "per_warp", 0.0), (1, 2, 2048, 128, torch.bfloat16, True, "per_thread", 0.0),
              (1, 2, 333, 128, torch.float16, True, "per_thread", 0.0), (1, 2, 2048, 128, torch.float16, False, "per_thread", 2.0),
              (1, 2, 1024, 128, torch.float16, True, "per_thread", 2.0), (1, 4, 1024, 64, torch.float16, True, "per_warp", 2.0)]


def _a16_inputs(ci, case):
    B, H, S, D, dt, causal, gran, vshift = case
    g = torch.Generator().manual_seed(ci)
    q = torch.randn(B, H, S, D, generator=g).to(dt)
    k = (torch.randn(B, H, S, D, generator=g) + 4.0 * torch.randn(B, H, 1, D, generator=g)).to(dt)
    v = (torch.randn(B, H, S, D, generator=g) + vshift).to(dt)
    return q.cuda(), k.cuda(), v.cuda()


def _a16_case(sab, ops, O, z, ci, case):
    """One case of the a16 study (two-level f16/f32 PV accumulation, attn_utils.cuh:896-974; v += 2 stresses the f16
    accumulator): the real reference "fp32+fp16" kernel (stored rows), our kernel, and the oracle's f16-emulating / fp32 branches — all
    on the SAME quantised operands.  Returns the same rows of each."""
    B, H, S, D, dt, causal, gran, vshift = case
    q, k, v = _a16_inputs(ci, case)
    km = k.mean(dim=2, keepdim=True)
    sm = D ** -0.5
    q8, qs, k8, ks = (sab.per_warp_int8 if gran == "per_warp" else sab.per_thread_int8)(q, k, km)
    gi = 2 if gran == "per_warp" else 3
    v8, vs, _ = sab.per_channel_fp8(v, scale_max=2.25, smooth_v=False)
    o = torch.empty_like(q)
    ops.qk_int8_sv_f8_attn(q8, k8, v8, o, qs, ks, vs, None, 1, int(causal), gi, gi, sm, 0, 0)
    torch.cuda.synchronize()
    v8l = v8[..., :S].transpose(2, 3).contiguous().cpu()
    args = (q8.cpu(), k8.cpu(), v8l, qs.cpu(), ks.cpu(), vs.cpu())
    kw = dict(qk_quant_gran=gran, is_causal=causal, sm_scale=sm, out_dtype=torch.float32)
    o_f16 = O.attn_int8_fp8_cuda(*args, pv_accum_dtype="fp32+fp16", **kw)
    o_f32 = O.attn_int8_fp8_cuda(*args, pv_accum_dtype="fp32+fp32", **kw)
    ridx = _row_idx(B * H * S, 200 + ci)
    return _rows(o, ridx).float(), _golden16(z, f"a16_{ci}_o", dt), _rows(o_f16, ridx), _rows(o_f32, ridx), dt


def test_a16_oracle_f16_accumulate_branch_vs_real_f16_kernel(env):
    """Pins the oracle's emulate_f16_accum branch (oracle/sage_oracle.py attn_int8_fp8_cuda, pv_accum_dtype="fp32+fp16") to the REAL
    reference kernel `qk_int8_sv_f8_accum_f16_fuse_v_scale_attn_inst_buf`: within 2e-3 plus two units in the last place of the output
    (the real mma accumulates its 32-key steps with an internal precision the step-wise f16 rounding of the restatement only
    approximates; the v += 2 causal stress case reaches 2 fp16 ulps)."""
    sab, ops, O = env
    z = _ref_golden()
    for ci, case in enumerate(_A16_CASES):
        _, o_ref, o_f16, _, dt = _a16_case(sab, ops, O, z, ci, case)
        err = (o_f16 - o_ref).abs()
        assert (err <= 2e-3 + 2.02 * _out_ulp(o_ref, dt)).all(), (case, err.max().item())


def _check_a16_attribution(sab, ops, O):
    """With the EXACT-max kernel (same P bits as the reference): where our output differs from the reference's default "fp32+fp16"
    kernel, the difference IS that kernel's per-tile f16 rounding — our result sits on the exact evaluation of the quantised operands
    (oracle, fp32 accumulation) to 2e-3 + 1 ulp everywhere, and on the rows that differ by more than 5e-3 the reference is the farther one."""
    z = _ref_golden()
    worst = 0.0
    for ci, case in enumerate(_A16_CASES):
        o, o_ref, o_f16, o_f32, dt = _a16_case(sab, ops, O, z, ci, case)
        e_o, e_r = (o - o_f32).abs(), (o_ref - o_f32).abs()
        assert (e_o <= 2e-3 + 1.01 * _out_ulp(o_f32, dt)).all(), (case, e_o.max().item())
        rows = (o - o_ref).abs().amax(dim=-1) > 5e-3
        worst = max(worst, (o - o_ref).abs().max().item())
        if rows.any():
            assert e_o[rows].max().item() <= e_r[rows].max().item() + 1e-4, (case, e_o[rows].max().item(), e_r[rows].max().item())
    return worst


def test_attention_vs_real_reference_kernel(env):
    sab, ops, O = env
    r = _check_vs_real_reference_kernel(sab, ops, O)
    print(f"worst max-abs / mean-abs vs real reference kernels: {r[0]:.3e} / {r[1]:.3e}")


def test_exact_max_kernel_matches_reference_kernel_bits():
    """SAB_ATTN_KERNEL=exact keeps the reference's exact running max at head_dim 128 as well (csrc/attn.cu): P, m and d are then the
    reference kernel's, and the output agrees with its fp32+fp32 kernel to 4e-3 (the bound VERDICT r01 asks to keep selectable).
    The kernel choice is read once per process, so the check runs in a subprocess."""
    import subprocess, sys
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    env_ = dict(os.environ, SAB_ATTN_KERNEL="exact")
    code = ("import sys; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
            "import torch, sageattention_b200 as sab\nfrom sageattention_b200 import ops\nfrom oracle import sage_oracle as O\n"
            "import test_gpu_parity as T\nr = T._check_vs_real_reference_kernel(sab, ops, O)\nprint('EXACT', r)\n"
            "a = T._check_a16_attribution(sab, ops, O)\nprint('A16', a)\n" % (ROOT, os.path.join(ROOT, "tests")))
    p = subprocess.run([sys.executable, "-c", code], env=env_, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-2000:]
    assert "EXACT" in p.stdout and "A16" in p.stdout
    print(p.stdout[-300:])


F16PV_CASES = [(1, 4, 4, 1024, 128, torch.float16, False, "per_thread"), (1, 4, 2, 1000, 64, torch.float16, True, "per_warp"),
               (2, 2, 2, 333, 128, torch.bfloat16, True, "per_thread"), (1, 2, 2, 2048, 64, torch.bfloat16, False, "per_thread")]


def test_fp16_pv_cuda_entry_vs_real_reference_kernel_and_oracle(env):
    """sageattn_qk_int8_pv_fp16_cuda (core.py:451-633): per-warp / per-thread INT8 Q,K + FP16 P and V.  Against the REAL
    reference sm80 kernel (`qk_int8_sv_f16_accum_f32_attn`, csrc/qattn/qk_int_sv_f16_cuda_sm80.cu; stored rows of its output) on the
    same quantised operands, and end to end against the oracle restatement.  Tolerance 2e-3 (fp16 P, fp32 accumulation on both
    sides; summation order differs) + one output ulp for bf16."""
    sab, ops, O = env
    z = _ref_golden()
    worst = 0.0
    for ci, (B, H, Hk, S, D, dt, causal, gran) in enumerate(F16PV_CASES):
        q, k, v = _mk_host(B, H, S, D, dt, Hk=Hk, seed=300 + ci)
        km = k.mean(dim=2, keepdim=True)
        sm = D ** -0.5
        q8, qs, k8, ks = (sab.per_warp_int8 if gran == "per_warp" else sab.per_thread_int8)(q, k, km)
        g = 2 if gran == "per_warp" else 3
        vt = sab.transpose_v_f16(v)
        o = torch.empty_like(q)
        lse = ops.qk_int8_sv_f16_attn(q8, k8, vt, o, qs, ks, 1, int(causal), g, g, sm, 0, 1)
        tol = 2e-3 + (2.0 ** -7 if dt == torch.bfloat16 else 0.0)
        ridx = _row_idx(B * H * S, 300 + ci)
        err = (_rows(o, ridx).float() - _golden16(z, f"f16pv{ci}_o", dt)).abs().max().item()
        worst = max(worst, err)
        assert err <= tol, (B, H, S, D, dt, causal, gran, err)
        assert (_rows(lse.reshape(-1, 1), ridx).reshape(-1) - torch.from_numpy(z[f"f16pv{ci}_lse"])).abs().max().item() <= 5e-4
        oe, le = O.attn_int8_fp16_cuda(q8.cpu(), k8.cpu(), v.cpu(), qs.cpu(), ks.cpu(), qk_quant_gran=gran, is_causal=causal,
                                       sm_scale=sm, out_dtype=dt, return_lse=True)
        assert (o.cpu().float() - oe.float()).abs().max().item() <= tol
        assert (lse.cpu() - le).abs().max().item() <= 1e-3
        # the public entry point (all pv_accum_dtype spellings of the reference are served with fp32 accumulation)
        for acc in ("fp32", "fp16+fp32"):
            o2, lse2 = sab.sageattn_qk_int8_pv_fp16_cuda(q, k, v, is_causal=causal, qk_quant_gran=gran, pv_accum_dtype=acc, return_lse=True)
            assert torch.equal(o2, o)
        oe2 = O.sageattn_qk_int8_pv_fp16_cuda(q.cpu(), k.cpu(), v.cpu(), is_causal=causal, qk_quant_gran=gran)
        assert (o2.cpu().float() - oe2.float()).abs().max().item() <= 2 * tol      # km: torch CPU vs kernel rounding of the mean
    print(f"worst max-abs vs real reference sm80 f16 kernel: {worst:.3e}")


@pytest.mark.parametrize("name", ["attn_d64_fp16_nc", "attn_d64_fp16_c", "attn_d128_fp16_nc_ragged"])
def test_triton_path_shell_vs_reference_triton_fixtures(env, name):
    """sageattn_qk_int8_pv_fp16_triton on sm_90a = bit-exact per-block quantisation + the FP16-PV kernel variant
    (kind::f16, Triton-path softmax): output within 4e-3 of the reference Triton kernel (whose tl.dot accumulates each
    64-key partial product in fp16; our kernel accumulates in fp32), LSE within 2e-3."""
    sab, ops, O = env
    z = np.load(f"{G}/{name}.npz")
    q, k, v, o_ref = (_t(z[n], torch.float16).cuda() for n in ("q", "k", "v", "o"))
    o, lse = sab.sageattn_qk_int8_pv_fp16_triton(q, k, v, is_causal=bool(z["causal"]), return_lse=True)
    assert np.allclose(lse.cpu().numpy(), z["lse"], atol=2e-3)
    assert (o.float() - o_ref.float()).abs().max().item() <= 4e-3


def test_triton_path_shell_cross_attention_padded_head_dim(env):
    """qo_len != kv_len, head_dim 96 (padded to 128, sm_scale from 96), bf16 (V cast to fp16): against the reference Triton
    kernel's output (tests/golden/attn_xattn_d96_bf16.npz); one bf16 output ulp + the fp16-accumulate slack."""
    sab, ops, O = env
    z = np.load(f"{G}/attn_xattn_d96_bf16.npz")
    q, k, v, o_ref = (_t(z[n], torch.bfloat16).cuda() for n in ("q", "k", "v", "o"))
    o, lse = sab.sageattn_qk_int8_pv_fp16_triton(q, k, v, is_causal=False, return_lse=True)
    assert o.shape == o_ref.shape
    assert np.allclose(lse.cpu().numpy(), z["lse"], atol=2e-3)
    assert (o.float() - o_ref.float()).abs().max().item() <= 2.0 ** -7 + 4e-3


@pytest.mark.parametrize("name", ["attn_mask_bool_d64", "attn_mask_bias_d128"])
def test_triton_path_attn_mask_vs_reference_triton_fixtures(env, name):
    """attn_mask of sageattn_qk_int8_pv_fp16_triton (core.py:248-250, 310-325; attn_qk_int8_per_block.py:33-52): bool mask
    (broadcast over heads, one all-false block) and additive fp16 bias, against the reference Triton kernel's output."""
    sab, ops, O = env
    z = np.load(f"{G}/{name}.npz")
    q, k, v, o_ref = (_t(z[n], torch.float16).cuda() for n in ("q", "k", "v", "o"))
    shape = tuple(int(x) for x in z["mask_shape"])
    mask = torch.from_numpy(z["mask"].copy()).view(shape) if str(z["kind"]) == "bool" else _t(z["mask"], torch.float16).view(shape)
    o, lse = sab.sageattn_qk_int8_pv_fp16_triton(q, k, v, attn_mask=mask.cuda(), return_lse=True)
    assert np.allclose(lse.cpu().numpy(), z["lse"], atol=2e-3)
    assert (o.float() - o_ref.float()).abs().max().item() <= 4e-3


def test_triton_path_attn_mask_vs_oracle(env):
    """More mask shapes against the CPU oracle: NHD layout, bf16 bias, GQA, 2-D / per-batch broadcast masks, ragged lengths,
    qo_len != kv_len; plus the host-side contract (dtype / causal asserts, broadcast failure)."""
    sab, ops, O = env
    g = torch.Generator().manual_seed(5)
    cases = [dict(B=2, H=4, Hk=2, Sq=200, Sk=333, D=128, dt=torch.bfloat16, layout="HND", mshape=(200, 333), kind="bool"),
             dict(B=2, H=2, Hk=2, Sq=130, Sk=130, D=64, dt=torch.float16, layout="NHD", mshape=(2, 1, 130, 130), kind="bias"),
             dict(B=1, H=4, Hk=1, Sq=257, Sk=64, D=96, dt=torch.bfloat16, layout="HND", mshape=(1, 4, 257, 64), kind="bias")]
    for c in cases:
        q, k, v = _mk(c["B"], c["H"], c["Sq"], c["D"], c["dt"], Hk=c["Hk"], Sk=c["Sk"])
        if c["kind"] == "bool":
            mask = torch.rand(c["mshape"], generator=g) < 0.5
            mask[..., 0] = True
        else:
            mask = torch.randn(c["mshape"], generator=g)
            mask[torch.rand(c["mshape"], generator=g) < 0.25] = float("-inf")
            mask[..., 0] = 0.0
            mask = mask.to(c["dt"])
        ref, ref_lse = O.sageattn_qk_int8_pv_fp16_triton(q.cpu(), k.cpu(), v.cpu(), return_lse=True, attn_mask=mask)
        qd, kd, vd = q, k, v
        if c["layout"] == "NHD":
            qd, kd, vd = (t.transpose(1, 2).contiguous() for t in (q, k, v))
        o, lse = sab.sageattn_qk_int8_pv_fp16_triton(qd, kd, vd, tensor_layout=c["layout"], attn_mask=mask.cuda(), return_lse=True)
        if c["layout"] == "NHD":
            o = o.transpose(1, 2)
        tol = 4e-3 if c["dt"] == torch.float16 else 2e-2
        assert (o.cpu().float() - ref.float()).abs().max().item() <= tol, c
        assert (lse.cpu() - ref_lse).abs().max().item() <= 1e-2, c
    q, k, v = _mk(1, 2, 128, 64, torch.float16)
    m = torch.ones(128, 128, dtype=torch.bool, device="cuda")
    with pytest.raises(AssertionError):
        sab.sageattn_qk_int8_pv_fp16_triton(q, k, v, attn_mask=m, is_causal=True)          # core.py:310
    with pytest.raises(AssertionError):
        sab.sageattn_qk_int8_pv_fp16_triton(q, k, v, attn_mask=m.float())                  # core.py:249
    with pytest.raises(AssertionError):
        sab.sageattn_qk_int8_pv_fp16_triton(q, k, v, attn_mask=m[:, :100])                 # cannot broadcast, core.py:322
    # a row with no visible key: zeros, not NaN (documented divergence: the reference returns an unmasked softmax)
    m2 = m.clone(); m2[5] = False
    o = sab.sageattn_qk_int8_pv_fp16_triton(q, k, v, attn_mask=m2)
    assert torch.isfinite(o).all() and o[:, :, 5].abs().max().item() == 0.0


# ------------------------------------------------------------------------------------------- API behaviour
def test_api_behaviour(env):
    sab, ops, O = env
    q, k, v = _mk(1, 4, 256, 64, torch.float16)
    base = sab.sageattn(q, k, v)
    # 1. unknown kwargs are accepted and ignored (SDPA monkey-patch contract, core.py:79-88)
    assert torch.equal(sab.sageattn(q, k, v, attn_mask=None, dropout_p=0.0, scale=0.3), base)
    # 2/3. sm_scale default uses the UN-padded head dim; padded output is sliced back
    q2, k2, v2 = _mk(1, 2, 128, 72, torch.float16)
    o2 = sab.sageattn(q2, k2, v2)
    assert o2.shape == q2.shape
    ex = O.sdpa_fp32(q2.cpu(), k2.cpu(), v2.cpu(), sm_scale=72 ** -0.5)
    assert (o2.cpu().float() - ex).abs().max().item() < 6e-2
    # 5. return_lse: natural-log LSE w.r.t. the UNSMOOTHED keys
    o3, lse = sab.sageattn(q, k, v, return_lse=True)
    s = (q.float() @ k.float().transpose(-1, -2)) * 64 ** -0.5
    assert (lse - torch.logsumexp(s, -1)).abs().max().item() < 5e-2
    # 6. qo_len != kv_len allowed for non-causal
    qs_, ks_, vs_ = _mk(1, 2, 100, 64, torch.float16, Sk=333)
    o4 = sab.sageattn(qs_, ks_, vs_)
    assert (o4.cpu().float() - O.sdpa_fp32(qs_.cpu(), ks_.cpu(), vs_.cpu())).abs().max().item() < 6e-2
    # 7. GQA divisibility, 10. unknown pv_accum_dtype raises, head_dim > 128 raises, fp32 rejected
    with pytest.raises(ValueError):
        sab.sageattn_qk_int8_pv_fp8_cuda(q, k, v, pv_accum_dtype="fp64")
    with pytest.raises(ValueError):
        sab.sageattn(torch.zeros(1, 1, 8, 160, device="cuda", dtype=torch.float16), torch.zeros(1, 1, 8, 160, device="cuda", dtype=torch.float16),
                     torch.zeros(1, 1, 8, 160, device="cuda", dtype=torch.float16))
    with pytest.raises(AssertionError):
        sab.sageattn(q.float(), k.float(), v.float())
    with pytest.raises(ValueError):
        sab.sageattn(_mk(1, 3, 64, 64, torch.float16)[0], *_mk(1, 2, 64, 64, torch.float16)[1:])
    # 9. smooth_v honoured for "fp32" (fuse_v_mean), warned + ignored otherwise
    vb = v + 3.0
    o5 = sab.sageattn_qk_int8_pv_fp8_cuda(q, k, vb, pv_accum_dtype="fp32", smooth_v=True)
    exb = O.sdpa_fp32(q.cpu(), k.cpu(), vb.cpu())
    o6 = sab.sageattn_qk_int8_pv_fp8_cuda(q, k, vb, pv_accum_dtype="fp32", smooth_v=False)
    assert (o5.cpu().float() - exb).abs().max().item() < (o6.cpu().float() - exb).abs().max().item() + 1e-3
    with pytest.warns(UserWarning):
        sab.sageattn_qk_int8_pv_fp8_cuda(q, k, vb, pv_accum_dtype="fp32+fp16", smooth_v=True)
    # 13. torch.compile traces through the custom ops (non-cudagraph), sm89_compile.py:48-101
    f = torch.compile(lambda a, b, c: sab.sageattn(a, b, c), fullgraph=False, backend="eager")   # dynamo + fake impls, no inductor
    assert torch.equal(f(q, k, v), base)


# ------------------------------------------------------------------------------------------- varlen (configs[3] family)
@pytest.mark.parametrize("name", ["varlen_gqa_d128_nc", "varlen_gqa_d128_c"])
def test_varlen_vs_reference_triton_fixtures(env, name):
    """Quantised tensors + packed scales bit-exact vs the reference Triton kernels; output (FP16-PV kernel variant) within
    4e-3 of the reference Triton varlen kernel."""
    sab, ops, O = env
    from sageattention_b200.quant import per_block_int8_varlen
    z = np.load(f"{G}/{name}.npz")
    q, k, v, o_ref = (_t(z[n], torch.float16).cuda() for n in ("q", "k", "v", "o"))
    cu = torch.from_numpy(z["cu"]).cuda()
    lens = (cu[1:] - cu[:-1]).tolist()
    km = k.mean(dim=0, keepdim=True)
    q8, qs, k8, ks, cuqs, cuks = per_block_int8_varlen(q, k, cu, cu, max(lens), max(lens), sm_scale=1.0 / 128 ** 0.5, km=km)
    assert np.array_equal(q8.cpu().numpy(), z["q8"]) and np.array_equal(k8.cpu().numpy(), z["k8"])
    n1, n2 = z["qs"].shape[0], z["ks"].shape[0]
    assert np.array_equal(qs[:n1].cpu().numpy(), z["qs"]) and np.array_equal(ks[:n2].cpu().numpy(), z["ks"])
    assert np.array_equal(cuqs.cpu().numpy(), z["cuqs"]) and np.array_equal(cuks.cpu().numpy(), z["cuks"])
    o = sab.sageattn_varlen(q, k, v, cu, cu, max(lens), max(lens), is_causal=bool(z["causal"]))
    assert not torch.isnan(o).any()
    assert (o.float() - o_ref.float()).abs().max().item() <= 4e-3


def test_varlen_equals_dense_per_sequence(env):
    """Size-independent property: a packed batch equals running each sequence alone through the dense per-block path
    with the same (batch-wide) K mean — checks cu_seqlens indexing, padding and scale offsets exactly."""
    sab, ops, O = env
    torch.manual_seed(3)
    lens = [512, 130, 77, 1000, 64]
    Hq, Hk, D = 8, 2, 128
    T = sum(lens)
    q = torch.randn(T, Hq, D, device="cuda").half(); k = torch.randn(T, Hk, D, device="cuda").half(); v = torch.randn(T, Hk, D, device="cuda").half()
    cu = torch.tensor([0] + list(np.cumsum(lens)), dtype=torch.int32, device="cuda")
    o = sab.sageattn_varlen(q, k, v, cu, cu, max(lens), max(lens), smooth_k=False)
    for i, L in enumerate(lens):
        a, b = int(cu[i]), int(cu[i + 1])
        oi = sab.sageattn_varlen(q[a:b].contiguous(), k[a:b].contiguous(), v[a:b].contiguous(), cu[:2] * 0 + torch.tensor([0, L], device="cuda", dtype=torch.int32),
                                 cu[:2] * 0 + torch.tensor([0, L], device="cuda", dtype=torch.int32), L, L, smooth_k=False)
        assert torch.equal(o[a:b], oi)   # same blocks, same scales, same kernel arithmetic -> same bits


# ------------------------------------------------------------------------------------------- full-size properties
def _full_size_checks(sab, O, B, H, S, D, causal, dt=torch.bfloat16):
    q, k, v = _mk(B, H, S, D, dt, seed=5)
    o, lse = sab.sageattn(q, k, v, is_causal=causal, return_lse=True)
    assert not torch.isnan(o).any() and not torch.isinf(lse).any()
    # (a) linearity in V by powers of two is EXACT (per-channel scales absorb it, fp8 payload identical)
    o2 = sab.sageattn(q, k, v * 2, is_causal=causal)
    assert torch.equal(o2, o * 2)
    # (b) heads / batches are independent: recomputing one (b,h) alone gives the same bits
    o1 = sab.sageattn(q[1:2, 3:4], k[1:2, 3:4], v[1:2, 3:4], is_causal=causal) if B > 1 else sab.sageattn(q[:, 3:4], k[:, 3:4], v[:, 3:4], is_causal=causal)
    assert torch.equal(o1, o[1:2, 3:4] if B > 1 else o[:, 3:4])
    # (c) sampled rows against exact fp32 attention and exact log-sum-exp
    rows = torch.randint(0, S, (48,), device="cuda")
    b, h = (1 if B > 1 else 0), 3
    s = (q[b, h, rows].float() @ k[b, h].float().T) * D ** -0.5
    if causal:
        s = s.masked_fill(torch.arange(S, device="cuda")[None, :] > rows[:, None], float("-inf"))
    ex = torch.softmax(s, -1) @ v[b, h].float()
    assert (o[b, h, rows].float() - ex).abs().max().item() < (1.5e-1 if causal else 3e-2)
    assert (lse[b, h, rows] - torch.logsumexp(s, -1)).abs().max().item() < 5e-2


def test_full_size_config1_hd128_seq8192(env):
    sab, ops, O = env
    _full_size_checks(sab, O, 4, 32, 8192, 128, False)


def test_full_size_config2_hd64_seq32768_causal(env):
    sab, ops, O = env
    _full_size_checks(sab, O, 1, 32, 32768, 64, True)


def test_full_size_config3_varlen_gqa(env):
    """configs[3]: GQA 32/8, hd=128, lens 512..16384 (T=32256): packed result vs exact fp32 attention on sampled rows."""
    sab, ops, O = env
    lens = [4096, 512, 16384, 1024, 8192, 2048]
    Hq, Hk, D = 32, 8, 128
    T = sum(lens)
    g = torch.Generator(device="cuda").manual_seed(11)
    q = torch.randn(T, Hq, D, device="cuda", generator=g).bfloat16()
    k = torch.randn(T, Hk, D, device="cuda", generator=g).bfloat16()
    v = torch.randn(T, Hk, D, device="cuda", generator=g).bfloat16()
    cu = torch.tensor([0] + list(np.cumsum(lens)), dtype=torch.int32, device="cuda")
    o = sab.sageattn_varlen(q, k, v, cu, cu, max(lens), max(lens))
    assert not torch.isnan(o).any()
    for i in (1, 2, 5):
        a, b = int(cu[i]), int(cu[i + 1])
        rows = torch.randint(a, b, (16,), device="cuda")
        h = 5
        s = (q[rows, h].float() @ k[a:b, h // 4].float().T) * D ** -0.5
        ex = torch.softmax(s, -1) @ v[a:b, h // 4].float()
        assert (o[rows, h].float() - ex).abs().max().item() < 3e-2


# ------------------------------------------------------------------------------------------- callers either side of the path
@pytest.mark.gpu
def test_prequantized_kv_is_bit_identical_to_one_shot_call(env):
    """quantize_kv once + sageattn_prequantized per call == sageattn_qk_int8_pv_fp8_cuda, bit for bit (same kernels)."""
    sab, ops, O = env
    cases = [dict(B=2, H=4, Hk=2, S=320, D=128, dt=torch.bfloat16, layout="HND", causal=False, gran="per_thread", acc="fp32+fp16"),
             dict(B=1, H=4, Hk=4, S=257, D=64, dt=torch.float16, layout="NHD", causal=True, gran="per_warp", acc="fp32+fp32"),
             dict(B=1, H=2, Hk=1, S=200, D=96, dt=torch.float16, layout="HND", causal=False, gran="per_thread", acc="fp32+fp16")]
    for c in cases:
        q, k, v = _mk(c["B"], c["H"], c["S"], c["D"], c["dt"], Hk=c["Hk"])
        if c["layout"] == "NHD":
            q, k, v = (t.transpose(1, 2).contiguous() for t in (q, k, v))
        ref, ref_lse = sab.sageattn_qk_int8_pv_fp8_cuda(q, k, v, tensor_layout=c["layout"], is_causal=c["causal"], qk_quant_gran=c["gran"],
                                                        pv_accum_dtype=c["acc"], return_lse=True)
        kv = sab.quantize_kv(k, v, tensor_layout=c["layout"], qk_quant_gran=c["gran"], pv_accum_dtype=c["acc"])
        assert kv.kv_len == c["S"] and kv.nbytes() < (k.numel() + v.numel()) * k.element_size()
        for _ in range(2):   # the cache is reusable
            o, lse = sab.sageattn_prequantized(q, kv, is_causal=c["causal"], return_lse=True)
            assert torch.equal(o, ref) and torch.equal(lse, ref_lse)
        # a different query block against the same K/V (non-causal): equals the one-shot call on that block
        if not c["causal"]:
            q2 = torch.randn_like(q)[:, :, :130] if c["layout"] == "HND" else torch.randn_like(q)[:, :130]
            q2 = q2.contiguous()
            assert torch.equal(sab.sageattn_prequantized(q2, kv),
                               sab.sageattn_qk_int8_pv_fp8_cuda(q2, k, v, tensor_layout=c["layout"], qk_quant_gran=c["gran"], pv_accum_dtype=c["acc"]))
    with pytest.raises(AssertionError):
        sab.sageattn_prequantized(q.to(torch.bfloat16), kv)


@pytest.mark.gpu
def test_host_pipeline_equals_device_call(env):
    """sageattn_host (chunked H2D / compute / D2H pipeline over pinned host tensors) == sageattn on device copies."""
    sab, ops, O = env
    for (B, H, Hk, S, D, dt, layout, causal, hpc) in [(2, 8, 4, 384, 128, torch.bfloat16, "HND", False, 2),
                                                      (2, 6, 6, 300, 64, torch.float16, "HND", True, 4),      # ragged last chunk
                                                      (3, 4, 2, 256, 128, torch.float16, "NHD", False, None),
                                                      (1, 4, 4, 200, 80, torch.bfloat16, "HND", False, 1)]:    # padded head dim
        q, k, v = _mk(B, H, S, D, dt, Hk=Hk)
        if layout == "NHD":
            q, k, v = (t.transpose(1, 2).contiguous() for t in (q, k, v))
        ref = sab.sageattn(q, k, v, tensor_layout=layout, is_causal=causal).cpu()
        qh, kh, vh = (t.cpu().pin_memory() for t in (q, k, v))
        out = sab.sageattn_host(qh, kh, vh, tensor_layout=layout, is_causal=causal, heads_per_chunk=hpc)
        assert out.device.type == "cpu" and out.is_pinned() and torch.equal(out, ref)
        # caller-provided (pageable) output, pageable inputs, sync=False + explicit stream sync
        out2 = torch.empty_like(ref)
        r = sab.sageattn_host(q.cpu(), k.cpu(), v.cpu(), out=out2, tensor_layout=layout, is_causal=causal, heads_per_chunk=hpc, sync=False)
        torch.cuda.current_stream().synchronize()
        assert r is out2 and torch.equal(out2, ref)
    with pytest.raises(AssertionError):
        sab.sageattn_host(q, k, v)   # device tensors belong to sageattn()


# ------------------------------------------------------------------------------------------- sequence parallel (configs[4])
def test_sequence_parallel_two_gpus(env):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import subprocess, sys
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
                        "--master-port", "29611", os.path.join(ROOT, "tests", "sp_check.py")], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "SP_CHECK_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
