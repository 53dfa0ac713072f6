"""The constructors of tests/quant_cases.py do what they claim (CPU only), so that a failure of tests/test_gpu_quant_edges.py
is a finding about a kernel and not about its input."""
import pytest
import torch

import quant_cases as QC
from oracle import sage_oracle as O

DTYPES = [torch.float16, torch.bfloat16]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("blk,D,k", [(16, 64, -3), (64, 128, 0), (128, 64, 4)])
def test_tie_block_reaches_every_int8_and_separates_the_two_roundings(dtype, blk, D, k):
    x = QC.tie_block(dtype, blk, D, k).view(1, 1, blk, D)
    t8, ts = O.quant_per_block_int8_triton(x, blk)
    c8, cs = O.quant_int8_cuda(x, blk)
    assert float(ts) == 2.0 ** k and float(cs) == 2.0 ** k
    assert sorted(set(t8.flatten().tolist())) == list(range(-127, 128)) == sorted(set(c8.flatten().tolist()))
    y = x.double() / 2.0 ** k
    tie = (y.abs() - y.abs().floor()) == 0.5
    assert int(tie.sum()) == 254
    differ = t8 != c8
    even_tie = tie & (y.abs().floor() % 2 == 0)            # half-away and half-even disagree exactly on n + 0.5 with n even
    assert torch.equal(differ, even_tie)
    assert torch.equal(t8[tie].double(), (y[tie].abs() + 0.5) * y[tie].sign())


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("D,sm,eps", [(64, None, False), (128, None, True), (64, 64 ** -0.5 * QC.LOG2E, False),
                                       (128, 128 ** -0.5 * QC.LOG2E, False)])
def test_near_tie_rows_straddle_the_fast_path_threshold(dtype, D, sm, eps):
    x, info = QC.near_tie_rows(dtype, D, sm_scale=sm, eps_after=eps, n_tiles=4)
    assert x.shape == (512, D) and torch.isfinite(x.float()).all()
    xb = x.view(1, 1, 512, D)
    if eps:   # the per-thread form: every group of a tile has the tile's amax
        _, qs, _, _ = O.quant_per_thread_int8_triton(xb, xb)
        scale = qs.view(4, 32)
    else:
        _, s = O.quant_per_block_int8_triton(xb, 128, 1.0 if sm is None else sm)
        scale = s.view(4, 1)
    assert (scale == info["scale"].view(4, 1)).all()
    sc = info["scale"].view(4, 1, 1).expand(4, 128, D).reshape(512, D)
    assert (torch.log2(sc) % 1 != 0).all()                                      # not a power of two: 1/scale is inexact
    res = QC.fast_path_residual(x, sc, sm).view(4, 128, D // 8, 8).amax(dim=-1)  # per 8-element group, as the kernel decides
    near, off = res[:, 0::2], res[:, 1::2]
    assert (near.amax(dim=-1) > QC.FAST_PATH_THRESHOLD).all()                    # every near-tie row has a group that falls back
    assert (off < QC.FAST_PATH_THRESHOLD).all() and (off.amax(dim=-1) > 0.49).all()
    d = info["dist"]
    for band in (1e-5, 1e-4):
        assert int((d < band).sum()) > 0
    assert int((x.float() < 0).sum()) > 0 and int((x.float() > 0).sum()) > 0


@pytest.mark.parametrize("name,amax", list(QC.TINY_AMAX.items()))
def test_tiny_amax_blocks_have_the_stated_scale(name, amax):
    x = QC.tiny_amax_block(amax, 64, 64)
    assert torch.isfinite(x.float()).all() and int((x != 0).sum()) > 0
    a = x.float().abs().max()
    assert a == torch.tensor(amax, dtype=torch.float64).float().bfloat16().float()
    q8, scale = O.quant_per_block_int8_triton(x.view(1, 1, 64, 64), 64)
    assert float(scale) == float(a / 127.0) and float(scale) > 0
    overflow = not torch.isfinite(torch.ones((), dtype=torch.float32) / scale).all()
    assert overflow == (amax < 127 * 2.0 ** -128)                            # 1e-38 and the subnormal overflow, 4e-37 does not
    assert int(q8.max()) == 127 and torch.equal(q8 == 0, x.view_as(q8) == 0)      # the reference formula: +-127 reached, 0 only for 0


@pytest.mark.parametrize("dtype", DTYPES)
def test_degenerate_cases_are_finite_and_degenerate(dtype):
    cases = QC.degenerate_qk_cases(dtype, 64)
    assert {"all_zero", "single_nonzero", "equal_to_mean", "minus_amax_only", "format_max"} <= set(cases)
    assert ("tiny_1e-38" in cases) == (dtype == torch.bfloat16)
    x, m = cases["equal_to_mean"]
    assert float((x - m).abs().max()) == 0.0
    x, _ = cases["minus_amax_only"]
    assert set(O.quant_int8_cuda(x.view(1, 1, *x.shape), 64)[0].flatten().tolist()) == {-127}
    x, _ = cases["all_zero"]
    q8, s = O.quant_int8_cuda(x.view(1, 1, *x.shape), 64)
    assert float(s.max()) == pytest.approx(1e-7 / 127, rel=1e-6) and int(q8.abs().max()) == 0
    v = QC.degenerate_v(dtype, 208, 64)
    assert float(v[:, 0].abs().max()) == 0 and float((v[:, 1] - 2.5).abs().max()) == 0
    y = v[:, 2].double() / 2.0 ** -3
    assert float(QC.exact_distance_to_e4m3_boundary(y[1:]).max()) == 0.0 and float(y.abs().max()) == 448.0
    assert float(QC.exact_distance_to_e4m3_boundary(v[1:, 3].double() / 2.0 ** -3).min()) > 0


def test_e4m3_helpers():
    y = torch.tensor([0.0, 1.0, 17.0, 18.0, 19.0, 447.9, 448.0, 470.0, 1e6, -1e6])
    got = QC.e4m3_satfinite(y).view(torch.float8_e4m3fn).float()
    assert got.tolist() == [0.0, 1.0, 16.0, 18.0, 20.0, 448.0, 448.0, 448.0, 448.0, -448.0]   # 17 and 19 are ties: to even
    d = QC.exact_distance_to_e4m3_boundary(torch.tensor([17.0, 17.5, 1.0625, 2.0 ** -10]))
    assert d.tolist() == [0.0, 0.5, 0.0, 0.0]
    assert QC.exact_distance_to_tie(torch.tensor([2.5, -7.0, 0.26]), torch.tensor(1.0)).tolist() == pytest.approx([0.0, 0.5, 0.24])


def test_varlen_layouts():
    """cu_seqlens_scale and cu_pad as sageattention_b200.quant.per_block_int8_varlen / per_channel_fp8_varlen compute them
    (cumsum of ceil(L/BLK), cumsum of ceil(L/128)*128), restated with Python integers and with torch on CPU tensors."""
    assert QC.varlen_layout([5, 0, 300], 64) == ([0, 5, 5, 305], [0, 1, 1, 6], [0, 128, 128, 512])
    assert QC.varlen_layout([129, 1, 64], 128) == ([0, 129, 130, 194], [0, 2, 3, 4], [0, 256, 384, 512])
    for lens in QC.VARLEN_LENS:
        for blk in (64, 128):
            cu, cu_scale, cu_pad = QC.varlen_layout(lens, blk)
            cu32 = torch.tensor(cu, dtype=torch.int32)
            L = cu32[1:] - cu32[:-1]
            pad = torch.nn.functional.pad
            assert pad(torch.cumsum((L + blk - 1) // blk, dim=0), (1, 0), value=0).tolist() == cu_scale
            assert pad(torch.cumsum((L + 127) // 128 * 128, dim=0), (1, 0), value=0).tolist() == cu_pad
            T, n = cu[-1], len(lens)
            assert cu_scale[-1] <= T // blk + n and cu_pad[-1] <= (T + 127 * n + 127) // 128 * 128   # the front end's upper bounds
