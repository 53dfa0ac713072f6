"""The quantisation kernels (csrc/quant.cu) where they can go wrong (-m gpu): rounding ties, the fast path's two fallbacks,
degenerate blocks, every instantiation the C ABI reaches, strides and guard bands, the packed varlen forms, the reduction
seams and the FP16 V transpose.  Every check compares a kernel, called through sageattention_b200.ops with caller-owned
output buffers, with oracle/sage_oracle.py or an fp32/fp64 restatement written here.

Criteria (stated once):
* Triton rounding semantics (IEEE division in the kernel): INT8 bytes and scales bit for bit.
* CUDA rounding semantics (the reference is built with --use_fast_math, so amax/127 and 127/amax are approximate divisions):
  scales within 2 ulp of the IEEE quotient; for every scale group ONE multiplier within 2 ulp of RN(127/amax) reproduces every
  byte of the group as rne(RN(x * mult)) — the multiply rounded on its own, ties to even; and against the IEEE oracle a byte may
  differ by exactly 1, and only where the exact quotient lies within 127 * 2^-21 of a tie.
* FP8 V: the same form — one reciprocal per channel within 2 ulp of RN(scale_max/amax) reproduces every byte; against the IEEE
  reciprocal a byte may move to the adjacent e4m3 code, and only within |y| * 2^-21 of an e4m3 rounding boundary.
The worst value each criterion met is collected in WORST and printed by the last test."""
import math
import pytest
import torch

import quant_cases as QC
from test_gpu_parity import _check_k_mean

pytestmark = pytest.mark.gpu
DTYPES = [torch.float16, torch.bfloat16]
SEM = {"cuda": 0, "triton": 1}
S_LIST = [1, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 1023, 1024, 1025, 2049, 8192]
WORST = {}


def _worst(key, value):
    WORST[key] = max(WORST.get(key, 0.0), float(value))


@pytest.fixture(scope="module")
def env():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    import sageattention_b200 as sab
    from sageattention_b200 import ops, _capi
    from oracle import sage_oracle as O
    assert _capi.lib().sab_check_device() == 0, "not an sm_90 device"
    return sab, ops, O


# ------------------------------------------------------------------------------------------------ helpers
def _guarded(shape, dtype, sentinel=0xA5, margin=4096):
    """A contiguous tensor inside a byte buffer pre-filled with `sentinel`, `margin` bytes of it on both sides."""
    n = math.prod(shape) * torch.empty((), dtype=dtype).element_size()
    buf = torch.full((2 * margin + n,), sentinel, dtype=torch.uint8, device="cuda")
    return buf, buf[margin:margin + n].view(dtype).view(shape)


def _only_these_written(buf, views, sentinel=0xA5):
    """Every byte of `buf` outside `views` still holds the sentinel (the views are consumed: they are overwritten)."""
    for v in views:
        v.view(torch.uint8).fill_(sentinel)
    return bool((buf == sentinel).all())


def _ulps(a, b):
    return (a.contiguous().view(torch.int32) - b.contiguous().view(torch.int32)).abs()


def _blocks(t, blk):
    """[B,H,S,D] -> [B,H,nblk,blk*D], rows zero-padded to a multiple of blk."""
    B, H, S, D = t.shape
    t = torch.nn.functional.pad(t, (0, 0, 0, (-S) % blk))
    return t.reshape(B, H, -1, blk * D)


def _expect_block(O, x, blk, sem, mean, sm):
    """The oracle for ops.quant_per_block_int8 on CPU tensors: x [B,H,S,D], mean [B,H,D] or None, sm a float or None."""
    if sem == "triton":
        xx = x if mean is None else x - mean[:, :, None, :]            # `k - km` in the input dtype (quant_per_block.py:53-54)
        e8, es = O.quant_per_block_int8_triton(xx, blk, 1.0 if sm is None else sm)
        zero = es.repeat_interleave(blk, dim=2)[:, :, :x.shape[2], None] == 0
        return torch.where(zero, torch.zeros_like(e8), e8), es          # all-zero block: 0/0 = NaN stores 0
    return O.quant_int8_cuda(x, blk, mean, sm)


def _check_cuda_sem(x, mean, sm, blk, got8, gots, e8, es, tag):
    """The CUDA-semantics criterion of the module docstring, on CPU tensors in HND order."""
    xf = x.float()
    if mean is not None:
        xf = xf - mean.float()[:, :, None, :]
    if sm is not None:
        xf = xf * torch.tensor(sm, dtype=torch.float32)
    xb, gb = _blocks(xf, blk), _blocks(got8, blk)
    amax = xb.abs().amax(dim=-1).clamp_min(0.0000001)
    assert torch.isfinite(gots).all() and int(_ulps(gots, es).max()) <= 2, f"{tag}: scale off by {int(_ulps(gots, es).max())} ulp"
    _worst("int8 scale ulps", _ulps(gots, es).max())
    diff = got8.int() - e8.int()
    assert int(diff.abs().max()) <= 1, f"{tag}: a byte differs from the oracle by {int(diff.abs().max())}"
    if bool((diff != 0).any()):
        rows_scale = (amax.double() / 127.0).repeat_interleave(blk, dim=2)[:, :, :x.shape[2], None]
        dist = QC.exact_distance_to_tie(xf, rows_scale)[diff != 0]
        _worst("int8 tie distance of a differing byte / (127 * 2^-21)", dist.max() / QC.TIE_BAND_INT8)
        assert float(dist.max()) < QC.TIE_BAND_INT8, f"{tag}: byte differs {float(dist.max()):.3e} away from a tie"
    m0 = torch.tensor(127.0) / amax
    ok = torch.zeros_like(amax, dtype=torch.bool)
    for j in range(-2, 3):
        m = (m0.view(torch.int32) + j).view(torch.float32)
        ok |= (torch.round(xb * m[..., None]).clamp(-128, 127) == gb.float()).all(dim=-1)
    assert bool(ok.all()), f"{tag}: {int((~ok).sum())} groups are not rne(RN(x * mult)) for any mult within 2 ulp of 127/amax"


def _run_block(ops, x, mean, blk, sem, sm, layout="HND"):
    """ops.quant_per_block_int8 into sentinel-guarded buffers; x / outputs in `layout`; returns HND CPU tensors."""
    xh = x if layout == "HND" else x.transpose(1, 2)
    B, H, S, D = xh.shape
    buf8, o8 = _guarded(x.shape, torch.int8)
    bufs, osc = _guarded((B, H, (S + blk - 1) // blk), torch.float32)
    ops.quant_per_block_int8(x, mean, o8, osc, blk, 1 if layout == "HND" else 0, SEM[sem], sm is not None, 1.0 if sm is None else sm)
    torch.cuda.synchronize()
    r8 = (o8 if layout == "HND" else o8.transpose(1, 2)).contiguous().cpu()
    rs = osc.cpu()
    assert _only_these_written(buf8, [o8]) and _only_these_written(bufs, [osc])
    return r8, rs


def _check_block(env, x, mean, blk, sem, sm, tag, layout="HND"):
    sab, ops, O = env
    got8, gots = _run_block(ops, x, mean, blk, sem, sm, layout)
    xc = (x if layout == "HND" else x.transpose(1, 2)).cpu()
    mc = None if mean is None else mean.cpu()
    e8, es = _expect_block(O, xc, blk, sem, mc, sm)
    if sem == "triton":
        assert torch.equal(gots, es), f"{tag}: scales"
        assert torch.equal(got8, e8), f"{tag}: {int((got8 != e8).sum())} bytes differ from the oracle"
    else:
        _check_cuda_sem(xc, mc, sm, blk, got8, gots, e8, es, tag)
    return got8, gots


def _run_thread(ops, x, mean, is_key, layout="HND"):
    xh = x if layout == "HND" else x.transpose(1, 2)
    B, H, S, D = xh.shape
    ncol = (S + 63) // 64 * 4 if is_key else (S + 127) // 128 * 32
    buf8, o8 = _guarded(x.shape, torch.int8)
    bufs, osc = _guarded((B, H, ncol), torch.float32)
    ops.quant_per_thread_int8(x, mean, o8, osc, 1 if layout == "HND" else 0, is_key)
    torch.cuda.synchronize()
    r8, rs = (o8 if layout == "HND" else o8.transpose(1, 2)).contiguous().cpu(), osc.cpu()
    assert _only_these_written(buf8, [o8]) and _only_these_written(bufs, [osc])
    return r8, rs


def _check_thread(env, x, mean, is_key, tag, layout="HND"):
    """ops.quant_per_thread_int8 against quant_per_thread_int8_triton (Triton semantics: bit for bit, scales complete)."""
    sab, ops, O = env
    got8, gots = _run_thread(ops, x, mean, is_key, layout)
    xc = (x if layout == "HND" else x.transpose(1, 2)).cpu()
    xx = xc if mean is None else xc - mean.cpu()[:, :, None, :]
    q8, qs, k8, ks = O.quant_per_thread_int8_triton(xx, xx)
    e8, es = (k8, ks) if is_key else (q8, qs)
    assert torch.equal(gots, es), f"{tag}: scales"
    assert torch.equal(got8, e8), f"{tag}: {int((got8 != e8).sum())} bytes differ from the oracle"


def _tie_tensor(dtype, D, blk, S, k0=-2, amax_every_row=False):
    """[1,1,S,D]: consecutive tie blocks (each its own power-of-two scale), so the first, the middle and the last, partial
    block of the tensor all hold exact ties."""
    n = (S + blk - 1) // blk
    x = torch.cat([QC.tie_block(dtype, blk, D, k0 + (i % 5), seed=i) for i in range(n)])[:S]
    if amax_every_row:      # per-thread groups interleave rows: give every row of a 128-row tile the tile's amax
        for t in range(0, S, 128):
            x[t:t + 128, 0] = x[t:t + 128].float().abs().max().to(dtype)
    return x.view(1, 1, S, D)


def _v_expect_check(v, got8, gots, gotm, smax, tag):
    """The FP8 criterion of the module docstring.  v [B,H,S,D] CPU, got8 [B,H,D,S_pad] uint8, gots [B,H,D], gotm [B,H,D] or None.
    With smooth_v the per-channel amax is max(|max - mean|, |min - mean|) in fp32 with the kernel's own mean."""
    B, H, S, D = v.shape
    vf = v.float()
    assert int(got8[..., S:].max() if got8.shape[-1] > S else 0) == 0, f"{tag}: padding columns are not zero"
    assert torch.isfinite(gots).all()
    if gotm is None:
        amax, c = vf.abs().amax(dim=2), vf
    else:
        amax = torch.maximum((vf.amax(dim=2) - gotm).abs(), (vf.amin(dim=2) - gotm).abs())
        c = vf - gotm[:, :, None, :]
    es = amax / torch.tensor(smax)
    assert int(_ulps(gots, es).max()) <= 2, f"{tag}: v_scale off by {int(_ulps(gots, es).max())} ulp"
    _worst("fp8 scale ulps", _ulps(gots, es).max())
    r0 = torch.where(amax > 0, torch.tensor(smax) / amax, torch.zeros_like(amax))       # zero channel: recp 0, bytes 0
    g = got8[..., :S].transpose(2, 3)                                                   # [B,H,S,D]
    ok = torch.zeros_like(amax, dtype=torch.bool)
    for j in range(-2, 3):
        r = torch.where(amax > 0, (r0.view(torch.int32) + j).view(torch.float32), r0)
        ok |= (QC.e4m3_satfinite(c * r[:, :, None, :]) == g).all(dim=2)
    assert bool(ok.all()), f"{tag}: {int((~ok).sum())} channels are not e4m3(RN((v - mean) * recp)) for any recp within 2 ulp"
    y = c * r0[:, :, None, :]
    e = QC.e4m3_satfinite(y)
    bad = e != g
    if bool(bad.any()):
        assert int((e[bad].int() - g[bad].int()).abs().max()) == 1, f"{tag}: not the adjacent e4m3 code"
        rel = QC.exact_distance_to_e4m3_boundary(c.double() * (smax / amax.double())[:, :, None, :])[bad] / y[bad].abs().double()
        _worst("fp8 boundary distance of a differing byte / (|y| * 2^-21)", rel.max() * 2.0 ** 21)
        assert float(rel.max()) < 2.0 ** -21, f"{tag}: byte differs {float(rel.max()):.3e} (relative) away from a boundary"


def _run_v(ops, v, smax, smooth_v, fused=False, layout="HND", sentinel=0xA5):
    vh = v if layout == "HND" else v.transpose(1, 2)
    B, H, S, D = vh.shape
    b8, o8 = _guarded((B, H, D, (S + 127) // 128 * 128), torch.uint8, sentinel)
    bs, osc = _guarded((B, H, D), torch.float32, sentinel)
    bm, om = _guarded((B, H, D), torch.float32, sentinel)
    fn = ops.per_channel_fp8_fused if fused else ops.per_channel_fp8
    fn(v, o8.view(torch.float8_e4m3fn), osc, om if smooth_v else None, 1 if layout == "HND" else 0, smax)
    torch.cuda.synchronize()
    r = o8.cpu(), osc.cpu(), om.cpu() if smooth_v else None
    assert _only_these_written(b8, [o8], sentinel) and _only_these_written(bs, [osc], sentinel)
    assert _only_these_written(bm, [om] if smooth_v else [], sentinel)
    return r


def _data(kind, B, H, S, D, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    torch.manual_seed(seed)         # the chi-square draw below uses the global generator
    x = torch.randn(B, H, S, D, generator=g)
    if kind == "outlier":          # K-like: a per-channel offset several sigma wide
        x = x + 4.0 * torch.randn(B, H, 1, D, generator=g)
    elif kind == "heavy":          # Student-t(2) plus a few 100x outliers
        x = x / torch.sqrt(torch.distributions.Chi2(2.0).sample((B, H, S, D)) / 2.0).clamp_min(1e-2)
        x = torch.where(torch.rand(B, H, S, D, generator=g) < 1e-3, 100.0 * x, x).clamp(-3e4, 3e4)
    return x.to(dtype).cuda()


# ------------------------------------------------------------------------------------------------ A. ties and fallbacks
@pytest.mark.parametrize("dtype", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("blk", [64, 128])
@pytest.mark.parametrize("sem", ["triton", "cuda"])
@pytest.mark.parametrize("with_mean", [False, True])
@pytest.mark.parametrize("with_sm", [False, True])
def test_ties_per_block(env, dtype, D, blk, sem, with_mean, with_sm):
    S = 2 * 128 + 77                      # the last tile and the last block are partial
    x = _tie_tensor(dtype, D, blk, S)
    mean = None
    if with_mean:                         # fp16 can hold tie + 256 * 2^k exactly, so the centred values are the ties again
        c = 256.0 * 2.0 ** -2 if dtype == torch.float16 else 0.0
        x = (x.float() + c).to(dtype)
        mean = torch.full((1, 1, D), c, dtype=dtype)
    sm = D ** -0.5 * QC.LOG2E if with_sm else None
    _check_block(env, x.cuda(), None if mean is None else mean.cuda(), blk, sem, sm, "ties")


@pytest.mark.parametrize("dtype", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("is_key", [False, True])
def test_ties_per_thread(env, dtype, D, is_key):
    """scale = amax/127 + 1e-7: with amax = 127 * 2^8 the epsilon is absorbed and the quotients are exact ties again."""
    x = _tie_tensor(dtype, D, 128, 333, k0=6, amax_every_row=True).cuda()
    _check_thread(env, x, None, is_key, "ties per-thread")
    _check_thread(env, x, torch.zeros(1, 1, D, dtype=dtype, device="cuda"), is_key, "ties per-thread, zero mean")


@pytest.mark.parametrize("dtype", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("with_sm", [False, True])
def test_near_ties_per_block(env, dtype, D, with_sm):
    """Quotients 2^-20 .. 1e-4 from a tie (the row has to fall back) next to quotients 1.5e-4 .. 5e-3 away (it does not)."""
    sm = D ** -0.5 * QC.LOG2E if with_sm else None
    x, _ = QC.near_tie_rows(dtype, D, sm_scale=sm, n_tiles=6)
    x = x[:6 * 128 - 50].view(1, 1, -1, D).cuda()
    for blk in (64, 128):
        for sem in ("triton", "cuda"):
            _check_block(env, x, None, blk, sem, sm, f"near ties blk{blk} {sem}")
    if not with_sm:
        _check_block(env, x, torch.zeros(1, 1, D, dtype=dtype, device="cuda"), 64, "triton", None, "near ties, zero mean")


@pytest.mark.parametrize("dtype", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("D", [64, 128])
def test_near_ties_per_thread(env, dtype, D):
    x, _ = QC.near_tie_rows(dtype, D, eps_after=True, n_tiles=6)
    x = x[:6 * 128 - 50].view(1, 1, -1, D).cuda()
    for is_key in (False, True):
        _check_thread(env, x, None, is_key, "near ties per-thread")


@pytest.mark.parametrize("dtype", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("gran", ["per_thread", "per_warp"])
def test_ties_smooth_quant_k(env, dtype, D, gran):
    """The single-launch K path computes its own mean; with THAT mean its bytes and scales are the oracle's."""
    sab, ops, O = env
    from sageattention_b200 import _capi
    ties = _tie_tensor(dtype, D, 64, 1152 + 40, k0=-2)                         # 10 tiles: more tiles than cluster ranks
    near, _ = QC.near_tie_rows(dtype, D, eps_after=gran == "per_thread", n_tiles=2)
    k = torch.cat([ties, near.view(1, 1, -1, D)], dim=2).cuda()
    S = k.shape[2]
    ncol = (S + 63) // 64 * (4 if gran == "per_thread" else 1)
    b8, o8 = _guarded(k.shape, torch.int8)
    bs, osc = _guarded((1, 1, ncol), torch.float32)
    bm, om = _guarded((1, 1, D), dtype)
    ops.k_smooth_quant_int8(k, om, o8, osc, 1, _capi.SAB_GRAN_PER_THREAD if gran == "per_thread" else _capi.SAB_GRAN_PER_WARP)
    torch.cuda.synchronize()
    got8, gots, km = o8.cpu(), osc.cpu(), om.clone()
    assert _only_these_written(b8, [o8]) and _only_these_written(bs, [osc]) and _only_these_written(bm, [om])
    _check_k_mean(km.view(1, 1, 1, D), k, k.mean(dim=2, keepdim=True))
    kc, kmc = k.cpu(), km.cpu()
    if gran == "per_thread":
        xx = kc - kmc[:, :, None, :]
        _, _, e8, es = O.quant_per_thread_int8_triton(xx, xx)
        assert torch.equal(gots, es) and torch.equal(got8, e8)
    else:
        e8, es = O.quant_int8_cuda(kc, 64, kmc)
        _check_cuda_sem(kc, kmc, None, 64, got8, gots, e8, es, "smooth_quant_k per_warp")


# ------------------------------------------------------------------------------------------------ B. inexact scales
@pytest.mark.parametrize("S", S_LIST)
@pytest.mark.parametrize("kind", ["gauss", "outlier", "heavy"])
def test_cuda_semantics_criteria(env, S, kind):
    sab, ops, O = env
    i = S_LIST.index(S)
    dtype, D, H = DTYPES[i % 2], (64, 128)[(i // 2) % 2], 1 if S > 2049 else 2
    x = _data(kind, 1, H, S, D, dtype, seed=S)
    _check_block(env, x, None, 32, "cuda", None, f"per-warp Q {kind} S{S}")
    _check_block(env, x, sab.k_mean(x).view(1, H, D), 64, "cuda", None, f"per-warp K {kind} S{S}")
    for smax in (448.0, 2.25):
        for smooth_v in (False, True):
            got8, gots, gotm = _run_v(ops, x, smax, smooth_v)
            _v_expect_check(x.cpu(), got8, gots, gotm, smax, f"fp8 {kind} S{S} smax{smax} smooth{smooth_v}")


# ------------------------------------------------------------------------------------------------ C. degenerate blocks
@pytest.mark.parametrize("dtype", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("D", [64, 128])
def test_degenerate_blocks(env, dtype, D):
    sab, ops, O = env
    for name, (x, m) in QC.degenerate_qk_cases(dtype, D).items():
        x = x.view(1, 1, *x.shape).cuda()
        mean = None if m is None else m.view(1, 1, D).cuda()
        sms = (None,) if mean is not None else (None, D ** -0.5 * QC.LOG2E)
        for sm in sms:
            for blk in (64, 128):
                _check_block(env, x, mean, blk, "triton", sm, f"{name} triton blk{blk} sm{sm}")
                if name == "format_max" and dtype == torch.bfloat16:
                    continue              # CUDA semantics at amax > 2^126: test_cuda_semantics_at_bf16_max
                _check_block(env, x, mean, blk, "cuda", sm, f"{name} cuda blk{blk} sm{sm}")
        for is_key in (False, True):
            _check_thread(env, x, mean, is_key, f"{name} per-thread")


def test_tiny_amax_bf16_block_takes_the_exact_path(env):
    """A bf16 block with amax below 127 * 2^-128 (finite, normal inputs reach 1.2e-38) has a denormal Triton-semantics scale
    whose fp32 reciprocal is inf.  The reference formula trunc(x / scale + 0.5 sign) still gives +-127 for +-amax and 0 for 0."""
    sab, ops, O = env
    for name in ("1e-38", "bf16_min_subnormal"):
        x = QC.tiny_amax_block(QC.TINY_AMAX[name], 192, 64).view(1, 1, 192, 64).cuda()
        got8, gots = _check_block(env, x, None, 64, "triton", None, f"tiny {name}")
        assert int(got8.max()) == 127 and int(got8.min()) == -127 and torch.equal(got8 == 0, x.cpu() == 0)
        assert float(gots.min()) > 0 and not torch.isfinite(1.0 / gots).all()
        q8, qs, k8, ks = sab.per_block_int8(x, x)                               # the Python front end, K side without sm_scale
        assert torch.equal(k8.cpu(), got8) and torch.equal(ks.cpu(), gots)


def test_cuda_semantics_at_bf16_max(env):
    """CUDA semantics with amax in (2^126, 2^128).  The reference is built with --use_fast_math, whose division returns 0 for a
    divisor in that range (CUDA C++ Programming Guide, __fdividef): its multiplier 127/amax is 0 and every byte it stores is 0,
    while the scale amax/127 is an ordinary quotient.  No stored row of tests/golden/reference_cuda_kernels.npz covers this
    input; the reference's own quantiser (built by oracle/build_ref.py) was run on it on an H100 and stores exactly that, bytes
    and scale bits equal to this kernel's.  So the reference's answer is pinned here, not the IEEE oracle's +-127."""
    sab, ops, O = env
    x, _ = QC.degenerate_qk_cases(torch.bfloat16, 64)["format_max"]
    x = x.view(1, 1, *x.shape).cuda()
    assert float(x.float().abs().max()) > 2.0 ** 126
    for blk in (32, 64):
        got8, gots = _run_block(ops, x, None, blk, "cuda", None)
        es = _blocks(x.cpu().float(), blk).abs().amax(dim=-1) / 127.0
        assert int(_ulps(gots, es).max()) <= 2 and int(got8.abs().max()) == 0


@pytest.mark.parametrize("dtype", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("fused", [False, True])
def test_degenerate_v(env, dtype, fused):
    sab, ops, O = env
    D, S = 64, 208
    v = QC.degenerate_v(dtype, S, D).view(1, 1, S, D).cuda()
    for smax in (448.0, 2.25):
        for smooth_v in (False, True):
            got8, gots, gotm = _run_v(ops, v, smax, smooth_v, fused)
            _v_expect_check(v.cpu(), got8, gots, gotm, smax, f"degenerate V smax{smax} smooth{smooth_v} fused{fused}")
            zero = [0, 1] if smooth_v else [0]                      # the constant channel is zero after centring
            assert int(got8[0, 0, zero].max()) == 0 and float(gots[0, 0, zero].abs().max()) == 0.0
            if smooth_v:
                assert float(gotm[0, 0, 1]) == 2.5 and float(gotm[0, 0, 0]) == 0.0


def test_nan_stays_in_its_head(env):
    """Non-finite inputs are outside the contract; the one promise is that they do not leak into another (b, h)."""
    sab, ops, O = env
    x = _data("gauss", 1, 3, 200, 64, torch.float16, seed=3)
    bad = x.clone()
    bad[0, 1, 17, 5] = float("nan")
    for sem in ("triton", "cuda"):
        a8, a_s = _run_block(ops, x, None, 64, sem, None)
        b8, b_s = _run_block(ops, bad, None, 64, sem, None)
        assert torch.equal(a8[:, [0, 2]], b8[:, [0, 2]]) and torch.equal(a_s[:, [0, 2]], b_s[:, [0, 2]])
    a, b = _run_v(ops, x, 448.0, True), _run_v(ops, bad, 448.0, True)
    for t, u in zip(a, b):
        assert torch.equal(t[:, [0, 2]], u[:, [0, 2]])


def _degenerate_attention_inputs(dtype, H=2, S=256, D=64):
    """q with an all-zero first 128-row tile; k whose keys 64..127 equal the sequence mean exactly (the other keys are +-pairs on
    a 1/16 grid around it, so the fp32 sum is exact); v with channel 0 all zero."""
    g = torch.Generator().manual_seed(21)
    q = (0.25 * torch.randn(1, H, S, D, generator=g)).to(dtype)
    q[:, :, :128] = 0
    c = torch.randint(-16, 17, (1, H, 1, D), generator=g).float() / 16
    n = torch.randint(-24, 25, (1, H, (S - 64) // 2, D), generator=g).float() / 16
    k = torch.cat([c + n[:, :, :32], c.expand(1, H, 64, D), c + n[:, :, 32:], c - n], dim=2).to(dtype)
    assert torch.equal(k.float().mean(dim=2, keepdim=True), c)
    v = torch.randn(1, H, S, D, generator=g).to(dtype)
    v[..., 0] = 0
    return q, k, v


@pytest.mark.parametrize("dtype", DTYPES, ids=["fp16", "bf16"])
def test_degenerate_inputs_end_to_end(env, dtype):
    sab, ops, O = env
    q, k, v = _degenerate_attention_inputs(dtype)
    ref = O.sdpa_fp32(q, k, v)
    qc, kc, vc = q.cuda(), k.cuda(), v.cuda()
    outs = {"sageattn": sab.sageattn(qc, kc, vc), "fp16_triton": sab.sageattn_qk_int8_pv_fp16_triton(qc, kc, vc)}
    cu = torch.tensor([0, 256], dtype=torch.int32, device="cuda")
    pk = lambda t: t[0].transpose(0, 1).contiguous()
    ov = sab.sageattn_varlen(pk(qc), pk(kc), pk(vc), cu, cu, 256, 256)
    outs["varlen"] = ov.transpose(0, 1).unsqueeze(0)
    for name, o in outs.items():
        o = o.float().cpu()
        assert torch.isfinite(o).all(), name
        assert float(o[..., 0].abs().max()) == 0.0, f"{name}: the all-zero V channel"
        err = float((o - ref).abs().max())
        _worst(f"end to end max-abs vs fp32 attention ({name})", err)
        # the FP8 entry rounds P and V to e4m3 (2^-4 relative each): 2e-2 against exact attention, 1e-2 against the oracle below
        assert err <= (2e-2 if name == "sageattn" else 1e-2), f"{name}: {err:.3e}"
    oe = O.sageattn_qk_int8_pv_fp8_cuda(q, k, v, lazy_tau=4, emulate_f16_accum=False)      # the FP8 kernel's own arithmetic
    # (channels 1..: the oracle's reciprocal of the zero channel's amax is inf, where the kernel and the reference guard)
    err = float((outs["sageattn"].float().cpu() - oe.float())[..., 1:].abs().max())
    _worst("end to end max-abs vs the oracle (sageattn)", err)
    assert err <= 1e-2, f"sageattn against the oracle: {err:.3e}"


# ------------------------------------------------------------------------------------------------ D. every instantiation
@pytest.mark.parametrize("dtype", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("blk", [16, 32, 64, 128])
@pytest.mark.parametrize("sem", ["triton", "cuda"])
@pytest.mark.parametrize("with_mean", [False, True])
@pytest.mark.parametrize("with_sm", [False, True])
def test_every_per_block_instantiation(env, dtype, D, blk, sem, with_mean, with_sm):
    x = _data("outlier", 2, 3, 333, D, dtype, seed=blk + D)
    mean = x.float().mean(dim=2).to(dtype) if with_mean else None
    sm = D ** -0.5 * QC.LOG2E if with_sm else None
    _check_block(env, x, mean, blk, sem, sm, "HND")
    xn = x.transpose(1, 2).contiguous()
    _check_block(env, xn, mean, blk, sem, sm, "NHD", layout="NHD")


@pytest.mark.parametrize("dtype", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("is_key", [False, True])
@pytest.mark.parametrize("with_mean", [False, True])
def test_every_per_thread_instantiation(env, dtype, D, is_key, with_mean):
    x = _data("outlier", 2, 3, 333, D, dtype, seed=7 + D)
    mean = x.float().mean(dim=2).to(dtype) if with_mean else None
    _check_thread(env, x, mean, is_key, "HND")
    _check_thread(env, x.transpose(1, 2).contiguous(), mean, is_key, "NHD", layout="NHD")


def test_rejected_arguments_return_their_codes(env):
    sab, ops, O = env
    from sageattention_b200 import _capi
    L = _capi.lib()
    INVALID, UNSUPPORTED = -1, -2
    B, H, S = 1, 2, 100

    def call(D=64, blk=64, ss=None, cols=None, out_off=0, dt=_capi.SAB_DTYPE_FP16, sem=1):
        x = torch.zeros(B, H, S, D, dtype=torch.float16, device="cuda")
        buf, o8 = _guarded((B * H * S * D + 64,), torch.int8)
        bs, sc = _guarded((B, H, 8), torch.float32)
        ss = D if ss is None else ss
        r = L.sab_quant_per_block_int8(x.data_ptr(), dt, None, o8.data_ptr() + out_off, sc.data_ptr(), B, H, S, D, H * S * D, S * D, ss,
                                       H * S * D, S * D, D, 8 if cols is None else cols, blk, sem, 0, 1.0, None)
        torch.cuda.synchronize()
        assert bool((buf == 0xA5).all()) and bool((bs == 0xA5).all()) or r == 0, "a rejected call wrote to its outputs"
        return r

    assert call() == 0
    assert call(blk=48) == UNSUPPORTED and call(D=96) == UNSUPPORTED and call(dt=7) == UNSUPPORTED
    assert call(ss=68) == INVALID and call(cols=1) == INVALID and call(out_off=4) == INVALID and call(sem=2) == INVALID
    x = torch.zeros(B, H, S, 64, dtype=torch.float16, device="cuda")
    o8, sc = torch.zeros(B, H, S, 64, dtype=torch.int8, device="cuda"), torch.zeros(B, H, 4, device="cuda")
    assert L.sab_quant_per_thread_int8(x.data_ptr(), 0, None, o8.data_ptr(), sc.data_ptr(), B, H, S, 64, H * S * 64, S * 64, 64,
                                       H * S * 64, S * 64, 64, 4, 1, None) == INVALID          # needs ceil(100/64)*4 = 8 columns


# ------------------------------------------------------------------------------------------------ E. strides and guard bands
def _input_views(dtype, D):
    """name -> (x, layout): slices and views of larger buffers; every one is [2,3,200,D] in HND order."""
    g = torch.Generator().manual_seed(2)
    big = (torch.randn(2, 5, 232, D, generator=g) + 2.0).to(dtype).cuda()
    nhd = (torch.randn(2, 200, 3, D, generator=g) + 2.0).to(dtype).cuda()
    return {"head slice": (big[:, 1:4, :200], "HND"), "token slice": (big[:, :3, 24:224], "HND"),
            "NHD view of an HND buffer": (big[:, :3, 8:208].transpose(1, 2), "NHD"), "NHD": (nhd, "NHD"),
            "batch stride 0": (big[:1, 2:5, 3:203].expand(2, 3, 200, D), "HND")}


@pytest.mark.parametrize("dtype", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("D", [64, 128])
def test_strided_inputs_and_outputs(env, dtype, D):
    """Each entry point on strided inputs, writing into a strided view of a sentinel-filled buffer: same bytes as the contiguous
    call, nothing written outside the view (gaps included), nothing that depends on the sentinel."""
    sab, ops, O = env
    from sageattention_b200 import _capi
    for name, (x, layout) in _input_views(dtype, D).items():
        lay = 1 if layout == "HND" else 0
        xh = x if layout == "HND" else x.transpose(1, 2)
        B, H, S, _ = xh.shape
        xc = xh.contiguous()
        mean = xc.float().mean(dim=2).to(dtype)
        results = []
        for sentinel in (0xA5, 0x5A):
            # the int8 output is a view with gaps in every dimension: [B, H+1, S+5, 2D] -> [:, :H, 3:3+S, D:]
            buf, big8 = _guarded((B, H + 1, S + 5, 2 * D), torch.int8, sentinel)
            o8h = big8[:, :H, 3:3 + S, D:]
            o8 = o8h if layout == "HND" else o8h.transpose(1, 2)
            got = []
            calls = [("block triton", lambda o, s: ops.quant_per_block_int8(x, mean, o, s, 64, lay, 1, False, 1.0), (S + 63) // 64),
                     ("block cuda", lambda o, s: ops.quant_per_block_int8(x, None, o, s, 32, lay, 0, True, 0.25), (S + 31) // 32),
                     ("thread q", lambda o, s: ops.quant_per_thread_int8(x, None, o, s, lay, False), (S + 127) // 128 * 32),
                     ("thread k", lambda o, s: ops.quant_per_thread_int8(x, mean, o, s, lay, True), (S + 63) // 64 * 4)]
            for cname, fn, ncol in calls:
                bs, sc = _guarded((B, H, ncol), torch.float32, sentinel)
                fn(o8, sc)
                torch.cuda.synchronize()
                got += [o8h.contiguous(), sc.clone()]
                assert _only_these_written(bs, [sc], sentinel), f"{name} / {cname}: scale guard band"
                assert _only_these_written(buf, [o8h], sentinel), f"{name} / {cname}: int8 guard band or gap"
            bm, om = _guarded((B, H, D), dtype, sentinel)
            ops.k_mean(x, om, lay)
            got.append(om.clone())
            bs, sc = _guarded((B, H, (S + 63) // 64), torch.float32, sentinel)
            bm2, om2 = _guarded((B, H, D), dtype, sentinel)
            ops.k_smooth_quant_int8(x, om2, o8, sc, lay, _capi.SAB_GRAN_PER_WARP)
            torch.cuda.synchronize()
            got += [o8h.contiguous(), sc.clone(), om2.clone()]
            assert _only_these_written(bm, [om], sentinel) and _only_these_written(bm2, [om2], sentinel)
            assert _only_these_written(bs, [sc], sentinel) and _only_these_written(buf, [o8h], sentinel), f"{name}: fused K"
            for smooth_v in (False, True):
                for fused in (False, True):
                    got += [t for t in _run_v(ops, x, 448.0, smooth_v, fused, layout, sentinel) if t is not None]
            bt, vt = _guarded((B, H, D, (S + 127) // 128 * 128), torch.float16, sentinel)
            ops.v_transpose_f16(x, vt, lay)
            torch.cuda.synchronize()
            got.append(vt.clone())
            assert _only_these_written(bt, [vt], sentinel)
            results.append(got)
        assert all(torch.equal(a, b) for a, b in zip(*results)), f"{name}: an output depends on what the buffer held before"
        # the same entry points on the contiguous copy, contiguous outputs
        ref = []
        for blk, sem, m, sm in ((64, "triton", mean, None), (32, "cuda", None, 0.25)):
            ref += [t.cuda() for t in _run_block(ops, xc, m, blk, sem, sm)]
        for is_key, m in ((False, None), (True, mean)):
            ref += [t.cuda() for t in _run_thread(ops, xc, m, is_key)]
        km, k8, ks = sab.quant.smooth_quant_k(xc, "per_warp")
        ref += [sab.k_mean(xc).view(B, H, D), k8, ks, km.view(B, H, D)]
        for smooth_v in (False, True):
            for fused in (False, True):
                ref += [t.cuda() for t in _run_v(ops, xc, 448.0, smooth_v, fused) if t is not None]
        ref.append(sab.quant.transpose_v_f16(xc))
        assert len(ref) == len(results[0])
        for i, (a, b) in enumerate(zip(results[0], ref)):
            assert torch.equal(a.cuda(), b), f"{name}: output {i} differs from the contiguous call"


# ------------------------------------------------------------------------------------------------ F. varlen
VARLEN_CASES = [dict(lq=l, lk=l) for l in QC.VARLEN_LENS] + [
    dict(lq=[100, 7, 260], lk=[300, 64, 1], Hq=4, Hk=2),                       # Lq != Lk, GQA
    dict(lq=[129, 1, 64], lk=[129, 1, 64], trailing=37, overstate=300, cu_dtype=torch.int64)]


@pytest.mark.parametrize("case", VARLEN_CASES, ids=lambda c: "q" + "_".join(map(str, c["lq"])) + "-k" + "_".join(map(str, c["lk"])))
@pytest.mark.parametrize("dtype,D", [(torch.float16, 64), (torch.bfloat16, 128)], ids=["fp16-d64", "bf16-d128"])
def test_varlen_quantisers(env, case, dtype, D):
    """Packed [T,H,D] forms.  INT8: every sequence equals the dense Triton-semantics quantiser on that sequence alone (with the
    packed mean), scale rows follow cu_seqlens_scale, everything else keeps the sentinel.  V: the per-channel scale is taken over
    ALL T packed tokens — tokens past cu_seqlens[-1] included, as the kernel reduces the whole tensor — and given that amax
    the columns [cu_pad[i], cu_pad[i] + L_i) are the dense quantiser's, the rest of each 128-padded segment is zero."""
    sab, ops, O = env
    from sageattention_b200 import quant
    Hq, Hk, trailing = case.get("Hq", 2), case.get("Hk", 2), case.get("trailing", 0)
    cu_dt = case.get("cu_dtype", torch.int32)
    g = torch.Generator().manual_seed(sum(case["lq"]))
    sm = D ** -0.5 * QC.LOG2E
    for lens, H, blk, is_k in ((case["lq"], Hq, 128, False), (case["lk"], Hk, 64, True)):
        cu, cu_scale, cu_pad = QC.varlen_layout(lens, blk)
        T = cu[-1] + trailing
        max_len = max(lens) + case.get("overstate", 0)
        x = (torch.randn(T, H, D, generator=g) + (2.0 if is_k else 0.0)).to(dtype).cuda()
        if trailing:
            x[cu[-1]:] = 50.0                                                   # the trailing tokens would dominate any statistic
        mean = x.float().mean(dim=0).to(dtype) if is_k else None
        cu_t = torch.tensor(cu, dtype=torch.int32, device="cuda")
        cus_t = torch.tensor(cu_scale, dtype=torch.int32, device="cuda")
        b8, o8 = _guarded((T, H, D), torch.int8)
        nrow = T // blk + len(lens)                                             # the front end's upper bound
        bs, sc = _guarded((nrow, H), torch.float32)
        ops.quant_per_block_int8_varlen(x, mean, o8, sc, cu_t, cus_t, max_len, blk, not is_k, sm if not is_k else 1.0)
        torch.cuda.synchronize()
        xx = (x if mean is None else x - mean[None]).cpu()
        e8, es, ecs = O.quant_per_block_int8_varlen_triton(xx[:cu[-1]], cu, blk, 1.0 if is_k else sm)
        assert ecs.tolist() == cu_scale
        assert torch.equal(o8[:cu[-1]].cpu(), e8) and torch.equal(sc[:cu_scale[-1]].cpu(), es)
        for i, L in enumerate(lens):                                            # and the dense kernel on the sequence alone
            if L:
                seg = x[cu[i]:cu[i + 1]].transpose(0, 1).unsqueeze(0)
                d8, ds = _run_block(ops, seg, None if mean is None else mean.view(1, H, D), blk, "triton", None if is_k else sm)
                assert torch.equal(d8[0].transpose(0, 1), o8[cu[i]:cu[i + 1]].cpu())
                assert torch.equal(ds[0].transpose(0, 1), sc[cu_scale[i]:cu_scale[i + 1]].cpu())
        assert _only_these_written(b8, [o8[:cu[-1]]]) and _only_these_written(bs, [sc[:cu_scale[-1]]]), "unused rows were written"
        if not is_k:
            continue
        # the front end: int64 or int32 cu_seqlens, its own cu arrays
        cu_user = torch.tensor(cu, dtype=cu_dt, device="cuda")
        cuq = torch.tensor(QC.varlen_layout(case["lq"], 128)[0], dtype=cu_dt, device="cuda")
        xq = torch.randn(int(cuq[-1]), Hq, D, generator=g).to(dtype).cuda()
        r = quant.per_block_int8_varlen(xq, x, cuq, cu_user, max(case["lq"]), max_len, km=mean.view(1, H, D))
        assert r[5].tolist() == cu_scale and r[4].tolist() == QC.varlen_layout(case["lq"], 128)[1]
        assert torch.equal(r[2][:cu[-1]].cpu(), e8)
        assert torch.equal(r[3][:cu_scale[-1]].cpu(), es)
        # V, FP8 and FP16, over the same packed tensor
        t_pad = (T + 127 * len(lens) + 127) // 128 * 128
        cup_t = torch.tensor(cu_pad, dtype=torch.int32, device="cuda")
        amax = x.float().abs().amax(dim=0)                                      # [H, D], over all T tokens
        for smax in (448.0, 2.25):
            bv, v8 = _guarded((H, D, t_pad), torch.uint8)
            bvs, vs = _guarded((H, D), torch.float32)
            ops.per_channel_fp8_varlen(x, v8.view(torch.float8_e4m3fn), vs, cu_t, cup_t, max_len, smax)
            torch.cuda.synchronize()
            written = []
            for i, L in enumerate(lens):
                if not L:
                    continue
                seg = x[cu[i]:cu[i + 1]].transpose(0, 1).unsqueeze(0).contiguous()
                Lp = (L + 127) // 128 * 128
                d8 = torch.empty(1, H, D, Lp, dtype=torch.float8_e4m3fn, device="cuda")
                dsc = torch.empty(1, H, D, device="cuda")
                ops.v_quant_with_amax(seg, d8, amax.view(1, H, D).contiguous(), dsc, 1, smax)
                assert cu_pad[i + 1] - cu_pad[i] == Lp
                assert torch.equal(v8[:, :, cu_pad[i]:cu_pad[i + 1]], d8[0].view(torch.uint8)), f"sequence {i}"
                assert int(d8.view(torch.uint8)[..., L:].max() if Lp > L else 0) == 0
                assert torch.equal(vs, dsc[0])
                written.append(v8[:, :, cu_pad[i]:cu_pad[i + 1]])
            assert _only_these_written(bv, written) and _only_these_written(bvs, [vs]), "columns past cu_pad[-1] were written"
        r8, rs, rpad = quant.per_channel_fp8_varlen(x, cu_user, max_len)
        assert rpad.tolist() == cu_pad and r8.shape[-1] == t_pad
        bt, vt = _guarded((H, D, t_pad), torch.float16)
        ops.v_transpose_f16_varlen(x, vt, cu_t, cup_t, max_len)
        torch.cuda.synchronize()
        written = []
        for i, L in enumerate(lens):
            if L:
                exp = torch.zeros(H, D, cu_pad[i + 1] - cu_pad[i], dtype=torch.float16, device="cuda")
                exp[:, :, :L] = x[cu[i]:cu[i + 1]].to(torch.float16).permute(1, 2, 0)
                assert torch.equal(vt[:, :, cu_pad[i]:cu_pad[i + 1]].view(torch.int16), exp.view(torch.int16)), f"fp16 V, sequence {i}"
                written.append(vt[:, :, cu_pad[i]:cu_pad[i + 1]])
        assert _only_these_written(bt, written)
        rt, rpad = quant.transpose_v_f16_varlen(x, cu_user, max_len)
        assert rpad.tolist() == cu_pad and rt.shape == (H, D, t_pad)


# ------------------------------------------------------------------------------------------------ G. reductions
@pytest.mark.parametrize("S", [1, 15, 16, 17, 127, 128, 1023, 1024, 1025, 1152, 2048, 2176, 32768])
@pytest.mark.parametrize("dtype,D", [(torch.float16, 128), (torch.bfloat16, 64)], ids=["fp16-d128", "bf16-d64"])
def test_reduction_seams(env, S, dtype, D):
    """Per-channel offset 100 with unit noise: the case where an fp32 summation order shows.  Against fp64; every kernel twice."""
    sab, ops, O = env
    from sageattention_b200.quant import quant_k_int8, smooth_quant_k
    B, H = 1, 2
    g = torch.Generator().manual_seed(S)
    x = (100.0 + torch.randn(B, H, S, D, generator=g)).to(dtype).cuda()
    xd = x.double()
    eps16 = 2.0 ** -10 if dtype == torch.float16 else 2.0 ** -7
    sum_tol = min(S, 1024) * 2.0 ** -24     # no kernel chains more than 1024 fp32 additions per channel, whatever S is

    def mean_ok(got, exact, what):      # a correct rounding of the fp64 mean, up to the fp32 summation error
        ulp = torch.exp2(torch.floor(torch.log2(exact.abs()))) * eps16
        err = ((got.double() - exact).abs() - exact.abs() * sum_tol).clamp_min(0) / ulp
        _worst(f"{what} error beyond the summation bound, in 16-bit ulps (limit 0.5)", err.max())
        assert float(err.max()) <= 0.5 * (1 + 1e-6), f"{what}: {float(err.max()):.3f} ulp"

    km = sab.k_mean(x)
    assert torch.equal(km, sab.k_mean(x))
    mean_ok(km.view(B, H, D), xd.mean(dim=2), "k_mean")
    st = [torch.empty(B, H, D, device="cuda") for _ in range(6)]
    ops.channel_stats(x, st[0], st[1], st[2], 1)
    ops.channel_stats(x, st[3], st[4], st[5], 1)
    assert all(torch.equal(st[i], st[i + 3]) for i in range(3))
    rel = ((st[0].double() - xd.sum(dim=2)).abs() / xd.abs().sum(dim=2)).max()
    _worst("channel_stats sum relative error / (min(S, 1024) * 2^-24)", rel / sum_tol)
    assert float(rel) <= sum_tol
    assert torch.equal(st[1], x.float().amax(dim=2)) and torch.equal(st[2], x.float().amin(dim=2))
    for gran in ("per_thread", "per_warp"):
        km2, k8, ks = smooth_quant_k(x, gran)
        again = smooth_quant_k(x, gran)
        assert torch.equal(km2, again[0]) and torch.equal(k8, again[1]) and torch.equal(ks, again[2])
        mean_ok(km2.view(B, H, D), xd.mean(dim=2), "smooth_quant_k mean")
        ulp = torch.exp2(torch.floor(torch.log2(km.float().abs()))) * eps16
        assert bool(((km2.float() - km.float()).abs() <= ulp).all())            # the two summation orders: one 16-bit ulp at most
        r8, rs = quant_k_int8(x, km2, gran)
        assert torch.equal(k8, r8) and torch.equal(ks, rs)
    pad16 = (S + 15) // 16 * 16
    outs = {}
    for fused in (False, True):
        a, b = _run_v(ops, x, 448.0, True, fused), _run_v(ops, x, 448.0, True, fused)
        assert all(torch.equal(t, u) for t, u in zip(a, b))
        exact = xd.sum(dim=2).cpu() / pad16                                     # the reference divides by the 16-padded length
        rel = ((a[2].double() - exact).abs() / exact.abs()).max()
        _worst("smooth-V mean relative error / ((min(S, 1024) + 1) * 2^-24)", rel / (sum_tol + 2.0 ** -24))
        assert float(rel) <= sum_tol + 2.0 ** -24, f"smooth-V mean (fused={fused}): {float(rel):.3e}"
        _v_expect_check(x.cpu(), a[0], a[1], a[2], 448.0, f"smooth V S{S} fused{fused}")
        outs[fused] = a
    assert torch.allclose(outs[True][2], outs[False][2], rtol=2 * sum_tol + 2.0 ** -23, atol=0)
    if torch.equal(outs[True][2], outs[False][2]):                               # given the same mean: identical scales and bytes
        assert torch.equal(outs[True][0], outs[False][0]) and torch.equal(outs[True][1], outs[False][1])
    a, b = _run_v(ops, x, 448.0, False, False), _run_v(ops, x, 448.0, False, True)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])                   # max / min do not depend on the order


# ------------------------------------------------------------------------------------------------ H. FP16 V
@pytest.mark.parametrize("dtype", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("layout", ["HND", "NHD"])
def test_transpose_v_f16_bit_for_bit(env, dtype, D, layout):
    sab, ops, O = env
    for S in S_LIST:
        H = 1 if S > 2049 else 2
        v = _data("gauss", 1, H, S, D, dtype, seed=S).cpu()
        if dtype == torch.bfloat16:      # values that overflow (inf), round to the fp16 maximum, or underflow in fp16
            edge = torch.tensor([1e5, -7e4, 65520.0, 65504.0, 3e-8, -2.9e-8, 6e-8, 1e-6, 3.38e38, 1e-30], dtype=dtype)
            v[0, 0, 0, :10] = edge
            v[0, -1, -1, -10:] = edge
        v = v.cuda()
        vin = v if layout == "HND" else v.transpose(1, 2).contiguous()
        bt, vt = _guarded((1, H, D, (S + 127) // 128 * 128), torch.float16)
        ops.v_transpose_f16(vin, vt, 1 if layout == "HND" else 0)
        torch.cuda.synchronize()
        exp = torch.zeros_like(vt)
        exp[..., :S] = v.to(torch.float16).transpose(2, 3)
        assert torch.equal(vt.view(torch.int16), exp.view(torch.int16)), f"S={S}"
        assert _only_these_written(bt, [vt])


def test_zz_report_margins(env):
    """Not a check: prints the worst value every criterion above met (run with -rP to see it)."""
    for k in sorted(WORST):
        print(f"[quant-edges] {k}: {WORST[k]:.4g}")
