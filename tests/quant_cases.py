"""Seeded input constructors and exact (fp64) predicates for the quantiser tests.  Plain torch on the CPU.

The INT8 quantisers of csrc/quant.cu round y = x/scale with a byte trick and fall back to the reference's own sequence only
for rows whose |y - round(y)| maximum exceeds 0.4999 (Triton rounding) or whose |y| exceeds 127.49 (CUDA rounding).  Random
data reaches those branches by chance; the constructors here reach them on purpose: exact ties, quotients a chosen distance
from a tie, and blocks whose scale is zero, denormal, or at the top of the input format.  The expected bytes always come from
oracle/sage_oracle.py (or from the fp32 restatements below); nothing here computes an expectation from the construction.
Consumers: tests/test_quant_cases_cpu.py (the constructors do what they claim) and tests/test_gpu_quant_edges.py."""
import math
import torch

FAST_PATH_THRESHOLD = 0.4999     # csrc/quant.cu quant_int8_tile: rows with max |y - n| above it redo the exact sequence
TIE_BAND_INT8 = 127 * 2.0 ** -21  # what two approximate divisions (2 ulp each) can move a quotient of magnitude <= 127
LOG2E = 1.44269504


def _neighbours(x: torch.Tensor):
    """The next representable value above and below each element, in x's own 16-bit format (finite non-zero x)."""
    bits = x.view(torch.int16)
    return (bits + 1).view(x.dtype), (bits - 1).view(x.dtype)     # +1 / -1 on the bit pattern: away from / towards zero


def tie_block(dtype, blk_rows: int, D: int, k: int, seed: int = 0) -> torch.Tensor:
    """[blk_rows, D] block whose amax is exactly 127 * 2^k, so scale = 2^k and 1/scale are exact.  It holds, times 2^k: +-127,
    (n + 0.5) for n in 0..126 with both signs (the ties, where half-away and half-even disagree for even n), every integer
    -126..126, and the neighbours of each tie one unit in the last place of `dtype` away; the rest is zero.  All are exact in
    fp16 and bf16 (8 significant bits reach 127.5).  Positions are shuffled by `seed`."""
    assert blk_rows * D >= 1017
    n = torch.arange(127, dtype=torch.float32)
    ties = torch.cat([n + 0.5, -(n + 0.5)])
    ints = torch.arange(-127, 128, dtype=torch.float32)
    t16 = ties.to(dtype)
    assert torch.equal(t16.float(), ties)
    up, down = _neighbours(t16)
    vals = torch.cat([ties, ints, up.float(), down.float()])
    blk = torch.zeros(blk_rows * D, dtype=torch.float32)
    blk[:vals.numel()] = vals
    perm = torch.randperm(blk.numel(), generator=torch.Generator().manual_seed(seed))
    out = (blk[perm] * 2.0 ** k).to(dtype)
    assert torch.equal(out.float(), blk[perm] * 2.0 ** k)
    return out.view(blk_rows, D)


def exact_distance_to_tie(x: torch.Tensor, scale: torch.Tensor) -> torch.Tensor:
    """|frac(|x| / scale) - 0.5| in fp64: how far the exact quotient is from a rounding tie of the INT8 grid."""
    q = (x.double() / scale.double()).abs()
    return (q - q.floor() - 0.5).abs()


def _e4m3_boundaries() -> torch.Tensor:
    """Midpoints between adjacent non-negative e4m3 values (the points where cvt.rn.e4m3 changes its answer), fp64."""
    vals = torch.arange(0, 127, dtype=torch.uint8).view(torch.float8_e4m3fn).double()      # 0 .. 448
    return (vals[1:] + vals[:-1]) / 2


def exact_distance_to_e4m3_boundary(y: torch.Tensor) -> torch.Tensor:
    """Distance (fp64) of |y| to the nearest e4m3 rounding boundary."""
    b = _e4m3_boundaries()
    a = y.double().abs().clamp(max=480.0)
    i = torch.searchsorted(b, a.contiguous()).clamp(1, b.numel() - 1)
    return torch.minimum((a - b[i - 1]).abs(), (a - b[i]).abs())


def e4m3_satfinite(y: torch.Tensor) -> torch.Tensor:
    """cvt.rn.satfinite.e4m3x2.f32 as bytes: torch's cast rounds to nearest even but turns |y| > 464 into NaN, so clamp first."""
    return y.float().clamp(-448.0, 448.0).to(torch.float8_e4m3fn).view(torch.uint8)


def _positive_values(dtype, lo: float, hi: float) -> torch.Tensor:
    """Every finite value of the 16-bit format in [lo, hi], ascending."""
    allv = torch.arange(0, 0x7C00 if dtype == torch.float16 else 0x7F80, dtype=torch.int32).to(torch.int16).view(dtype)
    f = allv.float()
    return allv[(f >= lo) & (f <= hi)]


def near_tie_rows(dtype, D: int, sm_scale=None, eps_after: bool = False, n_tiles: int = 12, seed: int = 0):
    """Brute force over the 16-bit values: 128-row tiles, each with ONE amax `a` (in column 0 of every row, so every per-block,
    per-warp and per-thread group of the tile has the scale RN(a [* sm_scale] / 127) [+ 1e-7], not a power of two), whose other
    elements are values x with the exact quotient x [* sm_scale] / scale close to a half-integer.  Even rows of a tile hold
    quotients within 1e-4 of a tie (bands 2^-20, 1e-5, 1e-4: the fast path's |y - n| exceeds 0.4999 and the row must take the
    exact sequence); odd rows hold quotients between 1.5e-4 and 5e-3 from a tie (|y - n| stays below 0.4999: the fast path
    decides, and has to be right on its own).  Both signs.  Returns (x [n_tiles*128, D], info) with info['dist'] the fp64 tie
    distance of every element and info['scale'] the per-tile scale."""
    g = torch.Generator().manual_seed(seed)
    sm = None if sm_scale is None else torch.tensor(sm_scale, dtype=torch.float32)
    amaxes = _positive_values(dtype, 1.0, 1.999)
    amaxes = amaxes[torch.randperm(amaxes.numel(), generator=g)[:256]]
    found = []
    for a in amaxes:      # bf16 has ~1e5 (amax, x) pairs in all, a few dozen of them within 1e-4 of a tie: keep the richest amaxes
        af = a.float() * sm if sm is not None else a.float()
        scale = af / 127.0 + (0.0000001 if eps_after else 0.0)
        cand = _positive_values(dtype, float(a) / 300.0, float(a))
        cf = cand.float() * sm if sm is not None else cand.float()
        d = exact_distance_to_tie(cf, scale)
        near, off = cand[d < 1e-4], cand[(d > 1.5e-4) & (d < 5e-3)]
        if near.numel() >= 1 and off.numel() >= 4:
            found.append((float(d[d < 1e-4].min()), a, scale, near, off))
    assert len(found) >= n_tiles, "not enough near-tie candidates"
    found.sort(key=lambda f: f[0])
    tiles, scales, dists = [], [], []
    for _, a, scale, near, off in found[:n_tiles]:
        tile = torch.zeros(128, D, dtype=dtype)
        for r in range(128):
            src = near if r % 2 == 0 else off
            pick = src[torch.randint(src.numel(), (D,), generator=g)]
            sign = torch.where(torch.rand(D, generator=g) < 0.5, -1.0, 1.0).to(dtype)
            keep = torch.rand(D, generator=g) < (0.25 if r % 2 == 0 else 0.5)    # near-tie rows stay sparse: most 8-groups clean
            tile[r] = torch.where(keep, pick * sign, torch.zeros((), dtype=dtype))
        tile[:, 0] = a
        tiles.append(tile)
        scales.append(scale)
        tf = tile.float() * sm if sm is not None else tile.float()
        dists.append(exact_distance_to_tie(tf, scale))
    return torch.cat(tiles), {"dist": torch.cat(dists), "scale": torch.stack(scales)}


def fast_path_residual(x: torch.Tensor, scale: torch.Tensor, sm_scale=None) -> torch.Tensor:
    """|y - rne(y)| with y = RN(x [* sm_scale]) * RN(1/scale) in fp32: the quantity csrc/quant.cu compares with 0.4999."""
    xf = x.float() * torch.tensor(sm_scale, dtype=torch.float32) if sm_scale is not None else x.float()
    y = xf * (torch.ones((), dtype=torch.float32) / scale.float())
    return (y - torch.round(y)).abs()


TINY_AMAX = {"bf16_min_subnormal": 2.0 ** -133, "1e-38": 1e-38, "3e-37": 3e-37, "4e-37": 4e-37, "1e-30": 1e-30}


def tiny_amax_block(amax: float, rows: int, D: int, seed: int = 0) -> torch.Tensor:
    """bf16 [rows, D]: finite values j/127 * amax, j in -127..127 (rounded to bf16), zeros, and +amax itself.  For amax below
    127 * 2^-128 the Triton-semantics scale amax/127 is an fp32 denormal whose reciprocal overflows."""
    g = torch.Generator().manual_seed(seed)
    j = torch.randint(-127, 128, (rows, D), generator=g).double()
    x = (j / 127.0 * amax).to(torch.float32).to(torch.bfloat16)
    x[torch.rand(rows, D, generator=g) < 0.2] = 0
    a = torch.tensor(amax, dtype=torch.float64).to(torch.float32).to(torch.bfloat16)
    x = torch.where(x.float().abs() > a.float(), a, x)
    x[::3, 1] = a
    return x


def degenerate_qk_cases(dtype, D: int, S: int = 192):
    """name -> (x [S, D], mean [D] or None).  S = 192: one full 128-row tile and a partial one."""
    g = torch.Generator().manual_seed(11)
    rnd = torch.randn(S, D, generator=g)
    cases = {"all_zero": (torch.zeros(S, D, dtype=dtype), None)}
    one = torch.zeros(S, D, dtype=dtype)
    one[70, 5] = 3.0
    cases["single_nonzero"] = (one, None)
    row = torch.randn(D, generator=g).to(dtype)
    cases["equal_to_mean"] = (row.expand(S, D).contiguous(), row.clone())
    cases["minus_amax_only"] = (torch.full((S, D), -1.5, dtype=dtype), None)
    mixed = rnd.to(dtype).clone()
    mixed[0:64] = 0                      # one all-zero 64-row block next to ordinary ones
    mixed[128:144] = 0
    cases["zero_block_among_others"] = (mixed, None)
    top = 65504.0 if dtype == torch.float16 else 3.38e38
    huge = (rnd.clamp(-1, 1) * top).to(dtype)
    huge[::5, 3] = top
    cases["format_max"] = (huge, None)
    if dtype == torch.bfloat16:
        for name, a in TINY_AMAX.items():
            cases["tiny_" + name] = (tiny_amax_block(a, S, D, seed=len(name)), None)
    for x, m in cases.values():
        assert torch.isfinite(x.float()).all() and (m is None or torch.isfinite(m.float()).all())
    return cases


def degenerate_v(dtype, S: int, D: int, k: int = -3, seed: int = 5) -> torch.Tensor:
    """V [S, D] (S a multiple of 16, so the smooth-V mean of a constant channel is that constant):
    channel 0 all zero; channel 1 constant 2.5 (zero after centring); channel 2 amax 448 * 2^k with the other tokens ON the e4m3
    rounding boundaries times 2^k, both signs; channel 3 the same boundaries moved one unit in the last place; rest Gaussian."""
    assert S % 16 == 0
    g = torch.Generator().manual_seed(seed)
    v = torch.randn(S, D, generator=g).to(dtype)
    v[:, 0] = 0
    v[:, 1] = 2.5
    b = _e4m3_boundaries().float()
    b = b[b >= 2.0 ** -5]               # boundaries with at most 8 significant bits after scaling stay exact in bf16
    idx = torch.randint(b.numel(), (S,), generator=g)
    sign = torch.where(torch.rand(S, generator=g) < 0.5, -1.0, 1.0)
    col = (b[idx] * sign * 2.0 ** k).to(dtype)
    assert torch.equal(col.float(), b[idx] * sign * 2.0 ** k)
    up, down = _neighbours(col)
    v[:, 2] = col
    v[:, 3] = torch.where(torch.rand(S, generator=g) < 0.5, up, down)
    v[0, 2] = v[0, 3] = 448.0 * 2.0 ** k
    return v


def varlen_layout(lens, blk: int):
    """Python-int restatement of the packed layouts: cu_seqlens, cu_seqlens_scale (one scale row per `blk` tokens of each sequence,
    quant_per_block_varlen.py:77-85) and cu_pad (every sequence's V columns padded to a multiple of 128)."""
    cu, cu_scale, cu_pad = [0], [0], [0]
    for L in lens:
        cu.append(cu[-1] + L)
        cu_scale.append(cu_scale[-1] + math.ceil(L / blk))
        cu_pad.append(cu_pad[-1] + math.ceil(L / 128) * 128)
    return cu, cu_scale, cu_pad


VARLEN_LENS = [[1], [128], [129, 1, 64], [5, 0, 300], [127, 128, 129, 1000]]
