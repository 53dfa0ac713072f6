"""GPU tests (-m gpu) of the block-mask predictor (predict_block_mask; sab_block_stats and sab_predict_block_mask):
  1. the kernels' block statistics against the fp64 restatement (block_predict_oracle), elementwise, within a bound derived from
     the fp32 accumulation;
  2. the selection kernel fed its own statistics against the restatement: equal masks except at decisions within 1e-5 of a
     threshold (counted and reported);
  3. coverage: Sq != Skv, partial blocks, Skv in {1, 64, 65}, GQA with B > 1, D in {64, 96, 128}, both layouts and strided q / k
     (bitwise the same mask), causal or not, one head at Skv = 1048576;
  4. identities: thresholds that keep everything, the dense call's bits through sageattn_blocksparse, reproducibility, no empty
     row, the captured attention mass on piecewise-constant data, the gradient with a predicted mask; 5. validation, compile."""
import math

import pytest
import torch

import sageattention_b200 as sab
from sageattention_b200 import ops
from block_predict_oracle import block_stats, select

pytestmark = pytest.mark.gpu
BF, FP = torch.bfloat16, torch.float16
U = 2.0 ** -24
EPS = 1e-5


def _smooth(B, H, S, D, dt, seed, layout="HND"):
    """Seeded tokens that vary smoothly along the sequence, plus noise whose level changes every 64 tokens: blocks range from
    nearly constant (self-similarity near 1) to noise-dominated (near 0)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    pos = torch.arange(S, device="cuda", dtype=torch.float32)[:, None]
    freq = torch.rand(1, 4, generator=g, device="cuda") * 0.02
    phase = torch.rand(1, 4, generator=g, device="cuda") * 6.3
    basis = torch.sin(pos * freq + phase)                                              # [S, 4]
    coef = torch.randn(B, H, 4, D, generator=g, device="cuda")
    base = torch.randn(B, H, 1, D, generator=g, device="cuda")
    level = torch.rand(B, H, (S + 63) // 64, 1, generator=g, device="cuda").pow(3) * 4.0
    noise = torch.randn(B, H, S, D, generator=g, device="cuda") * level.repeat_interleave(64, 2)[:, :, :S]
    x = (base + basis @ coef + noise).to(dt)
    return x if layout == "HND" else x.transpose(1, 2).contiguous()


def _hnd(x, layout):
    return x if layout == "HND" else x.transpose(1, 2)


def _kernel_stats(x, layout, blk):
    lay = 1 if layout == "HND" else 0
    B, H, S, D = ops._bhsd(x, lay)
    nb = (S + blk - 1) // blk
    mean = torch.empty(B, H, nb, D, device="cuda")
    sim = torch.empty(B, H, nb, device="cuda")
    ops.block_stats(x, mean, sim, lay, blk)
    return mean, sim


def _check_stats(x, layout, blk):
    """The kernel's mean and self-similarity against fp64, elementwise.  Bounds from the fp32 accumulation over a block of n rows:
    mean: (n + 4) u mean|x|;  sim: with S_d = sum_r u_rd and A_d = sum_r |u_rd|, each S_d is within e A_d, e = (n + D + 4) u (n
    additions, plus the unit vector's D-term norm), so sim is within (2 sum_d |S_d| e A_d + sum_d (e A_d)^2) / n^2 + (D + 4) u sim.
    Returns the worst ratio of error to bound for each."""
    mean, sim = _kernel_stats(x, layout, blk)
    xh = _hnd(x, layout).double().cpu()
    B, H, S, D = xh.shape
    m_ref, s_ref = block_stats(xh, blk)
    nb = m_ref.size(2)
    pad = nb * blk - S
    n = torch.full((nb,), float(blk), dtype=torch.float64)
    n[-1] = S - blk * (nb - 1)
    xs = torch.nn.functional.pad(xh, (0, 0, 0, pad)).view(B, H, nb, blk, D)
    norm = xs.norm(dim=-1, keepdim=True)
    us = torch.where(norm > 0, xs / norm.clamp_min(1e-300), torch.zeros_like(xs))
    bound_m = (n[:, None] + 4) * U * xs.abs().sum(3) / n[:, None] + 1e-30
    e = (n[:, None] + D + 4) * U * us.abs().sum(3)
    Sd = us.sum(3)
    bound_s = (2 * (Sd.abs() * e).sum(-1) + (e ** 2).sum(-1)) / n ** 2 + (D + 4) * U * s_ref + 1e-30
    rm = ((mean.cpu().double() - m_ref).abs() / bound_m).max().item()
    rs = ((sim.cpu().double() - s_ref).abs() / bound_s).max().item()
    return rm, rs, mean, sim


# B, Hq, Hkv, Sq, Skv, D, dtype, layout, causal
CASES = [
    (1, 2, 2, 1000, 777, 64, FP, "HND", False),
    (2, 8, 2, 1024, 2048, 128, BF, "NHD", False),
    (1, 4, 4, 512, 1, 96, BF, "HND", False),
    (1, 2, 1, 256, 64, 128, FP, "NHD", False),
    (1, 2, 2, 300, 65, 64, BF, "HND", False),
    (2, 4, 2, 2048, 2048, 128, BF, "HND", True),
    (1, 2, 2, 1000, 1000, 96, FP, "NHD", True),
]
THRESHOLDS = [(0.9, 0.5), (0.5, 0.8), (0.99, 0.2)]


def _ids(c):
    return "-".join(str(x).replace("torch.", "") for x in c)


@pytest.mark.parametrize("case", CASES, ids=_ids)
def test_kernels_against_the_restatement(case):
    B, Hq, Hkv, Sq, Sk, D, dt, layout, causal = case
    q = _smooth(B, Hq, Sq, D, dt, seed=Sq + D, layout=layout)
    k = _smooth(B, Hkv, Sk, D, dt, seed=Sk + 7 * D, layout=layout)
    rq, sq_, qm, qs = _check_stats(q, layout, 128)
    rk, sk_, km, ks = _check_stats(k, layout, 64)
    print(f"[stats] {_ids(case)}: worst ratio to bound: q mean {rq:.3f} sim {sq_:.3f}, k mean {rk:.3f} sim {sk_:.3f}")
    assert max(rq, sq_, rk, sk_) <= 1.0
    other = "NHD" if layout == "HND" else "HND"
    q2, k2 = (_hnd(t, layout) if other == "HND" else _hnd(t, layout).transpose(1, 2) for t in (q, k))
    q2, k2 = q2.contiguous(), k2.contiguous()
    for cdf, sim in THRESHOLDS:
        kw = dict(cdf_threshold=cdf, sim_threshold=sim, is_causal=causal)
        m = sab.predict_block_mask(q, k, tensor_layout=layout, **kw)
        assert m.dtype == torch.bool and m.is_contiguous() and tuple(m.shape) == (B, Hq, (Sq + 127) // 128, (Sk + 63) // 64)
        ref, near = select(qm.cpu(), qs.cpu(), km.cpu(), ks.cpu(), Sq, Sk, sm_scale=D ** -0.5, eps=EPS, **kw)
        far = ~near
        print(f"[select] {_ids(case)} cdf {cdf} sim {sim}: density {m.float().mean().item():.3f}, "
              f"forced q blocks {(qs < sim).float().mean().item():.2f}, near-threshold rows {int(near.sum())}")
        assert torch.equal(m.cpu()[far], ref[far])
        assert near.float().mean().item() <= 0.01
        assert torch.all(m.any(-1))
        assert torch.equal(sab.predict_block_mask(q, k, tensor_layout=layout, **kw), m)          # reproducible
        assert torch.equal(sab.predict_block_mask(q2, k2, tensor_layout=other, **kw), m)         # the other layout


def test_strided_q_k_from_a_packed_qkv_give_the_same_bits():
    B, S, H, D = 2, 1536, 4, 64
    x = _smooth(B, 3 * H, S, D, BF, seed=11, layout="NHD")               # [B, S, 3H, D]
    qkv = x.view(B, S, 3, H, D)
    q, k = qkv[:, :, 0], qkv[:, :, 1]
    assert not q.is_contiguous() and not k.is_contiguous()
    for causal in (False, True):
        kw = dict(cdf_threshold=0.9, sim_threshold=0.5, tensor_layout="NHD", is_causal=causal)
        assert torch.equal(sab.predict_block_mask(q, k, **kw), sab.predict_block_mask(q.contiguous(), k.contiguous(), **kw))


def test_one_head_at_the_key_limit():
    """nk = 16384 (Skv = 1048576): one Q block per CTA, the sort over up to 16384 keys.  The restatement on the kernel's
    statistics.  sim_threshold -1 makes every key block a candidate; the other threshold sits in the middle of the widest gap
    between the key blocks' self-similarities near their median, so no column decision is within 1e-5 of it.  With thousands of
    candidates a prefix mass lands within 1e-5 of cdf_threshold more often: those rows are counted, not compared."""
    Sq, Sk, D = 4096, 1 << 20, 128
    q = _smooth(1, 1, Sq, D, BF, seed=21)
    k = _smooth(1, 1, Sk, D, BF, seed=22)
    qm, qs = _kernel_stats(q, "HND", 128)
    km, ks = _kernel_stats(k, "HND", 64)
    srt = ks.flatten().double().sort().values
    mid = srt[4096:12288]
    gap = (mid[1:] - mid[:-1]).argmax()
    sim_gap = float((mid[gap] + mid[gap + 1]) / 2)
    for cdf, sim in ((0.9, -1.0), (0.5, sim_gap), (0.9, sim_gap)):
        m = sab.predict_block_mask(q, k, cdf_threshold=cdf, sim_threshold=sim)
        assert tuple(m.shape) == (1, 1, 32, 16384)
        ref, near = select(qm.cpu(), qs.cpu(), km.cpu(), ks.cpu(), Sq, Sk, cdf_threshold=cdf, sim_threshold=sim,
                           sm_scale=D ** -0.5, eps=EPS)
        print(f"[limit] cdf {cdf} sim {sim:.6f}: density {m.float().mean().item():.4f}, near-threshold rows {int(near.sum())} of 32")
        assert int((~near).sum()) >= 8
        assert torch.equal(m.cpu()[~near], ref[~near])
        assert torch.equal(sab.predict_block_mask(q, k, cdf_threshold=cdf, sim_threshold=sim), m)
        assert torch.all(m.any(-1))
    assert torch.all(sab.predict_block_mask(q, k, cdf_threshold=1.0, sim_threshold=0.5))


@pytest.mark.parametrize("causal", [False, True])
def test_thresholds_that_keep_everything(causal):
    B, H, S, D = 1, 4, 1000, 128
    q = _smooth(B, H, S, D, FP, seed=31)
    k = _smooth(B, H, S, D, FP, seed=32)
    nq, nk = (S + 127) // 128, (S + 63) // 64
    i = torch.arange(nq, device="cuda")[:, None]
    j = torch.arange(nk, device="cuda")[None, :]
    full = (64 * j <= 128 * i + 127) if causal else torch.ones(nq, nk, dtype=torch.bool, device="cuda")
    for cdf, sim in ((1.0, 0.5), (1.5, -1.0), (0.5, 1.01), (0.01, math.inf)):
        m = sab.predict_block_mask(q, k, cdf_threshold=cdf, sim_threshold=sim, is_causal=causal)
        assert torch.equal(m, full.expand(B, H, nq, nk)), (cdf, sim)


@pytest.mark.parametrize("causal", [False, True])
def test_all_true_prediction_gives_the_dense_call_bitwise(causal):
    B, Hq, Hkv, S, D = 1, 4, 2, 768, 128
    q, k, v = (_smooth(B, h, S, D, BF, seed=40 + h) for h in (Hq, Hkv, Hkv))
    m = sab.predict_block_mask(q, k, cdf_threshold=1.0, sim_threshold=0.5, is_causal=causal)
    o = sab.sageattn_blocksparse(q, k, v, m, is_causal=causal)
    assert torch.equal(o, sab.sageattn_qk_int8_pv_fp8_cuda(q, k, v, is_causal=causal))


def _piecewise(B, Hq, Hkv, nq, nk, D, dt, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    q = (torch.randn(B, Hq, nq, 1, D, generator=g, device="cuda") * 2).to(dt).expand(-1, -1, -1, 128, -1)
    k = (torch.randn(B, Hkv, nk, 1, D, generator=g, device="cuda") * 2).to(dt).expand(-1, -1, -1, 64, -1)
    return q.reshape(B, Hq, nq * 128, D), k.reshape(B, Hkv, nk * 64, D)


@pytest.mark.parametrize("cdf", [0.5, 0.9, 0.99])
def test_piecewise_constant_data_captures_cdf_mass(cdf):
    """Every block is one token repeated, so pooled scores are the true block scores: the exact fp64 attention mass inside the
    mask reaches cdf_threshold in every row (less the fp32 rounding of the kernel's p)."""
    B, Hq, Hkv, nq, nk, D = 2, 4, 2, 8, 16, 64
    q, k = _piecewise(B, Hq, Hkv, nq, nk, D, BF, seed=int(cdf * 100))
    m = sab.predict_block_mask(q, k, cdf_threshold=cdf, sim_threshold=0.99)
    p = torch.softmax(D ** -0.5 * q.double() @ k.double().repeat_interleave(Hq // Hkv, 1).transpose(-1, -2), -1)
    mass = (p * m.repeat_interleave(128, 2).repeat_interleave(64, 3)).sum(-1)
    print(f"[piecewise] cdf {cdf}: density {m.float().mean().item():.3f}, least captured mass {mass.min().item():.6f}")
    assert mass.min().item() >= cdf - 1e-4
    assert m.float().mean().item() < 1.0


def test_gradients_with_a_predicted_mask_are_those_of_the_same_mask_passed_in():
    B, Hq, Hkv, S, D = 1, 4, 2, 640, 64
    q, k, v = (_smooth(B, h, S, D, BF, seed=50 + h).requires_grad_() for h in (Hq, Hkv, Hkv))
    do = torch.randn_like(q)
    m = sab.predict_block_mask(q, k, cdf_threshold=0.8, sim_threshold=0.5, is_causal=True)
    assert not m.requires_grad and 0.0 < m.float().mean().item() < 1.0
    given = m.cpu().clone().cuda()
    res = []
    for mask in (m, given):
        o = sab.sageattn_blocksparse(q, k, v, mask, is_causal=True)
        res.append((o,) + torch.autograd.grad(o, (q, k, v), do))
    for x, y in zip(*res):
        assert torch.equal(x, y)


def test_validation_raises_before_any_launch():
    q = _smooth(1, 4, 256, 64, FP, seed=60)
    k = _smooth(1, 2, 256, 64, FP, seed=61)
    kw = dict(cdf_threshold=0.9, sim_threshold=0.5)
    bad = [
        (ValueError, dict(q=q, k=k, cdf_threshold=0.0, sim_threshold=0.5)),
        (ValueError, dict(q=q, k=k, cdf_threshold=math.nan, sim_threshold=0.5)),
        (ValueError, dict(q=q, k=k, cdf_threshold=0.9, sim_threshold=math.nan)),
        (ValueError, dict(q=q, k=k, tensor_layout="XYZ", **kw)),
        (ValueError, dict(q=q, k=_smooth(1, 3, 256, 64, FP, seed=62), **kw)),
        (ValueError, dict(q=torch.zeros(1, 4, 128, 136, dtype=FP, device="cuda"),
                          k=torch.zeros(1, 2, 128, 136, dtype=FP, device="cuda"), **kw)),
        (ValueError, dict(q=q, k=k, sm_scale=math.inf, **kw)),
        (AssertionError, dict(q=q, k=_smooth(1, 2, 320, 64, FP, seed=63), is_causal=True, **kw)),
        (AssertionError, dict(q=q, k=k.float(), **kw)),
        (AssertionError, dict(q=q.cpu(), k=k.cpu(), **kw)),
    ]
    torch.cuda.synchronize()
    for exc, args in bad:
        with pytest.raises(exc):
            sab.predict_block_mask(**args)
    with pytest.raises(TypeError):
        sab.predict_block_mask(q, k, cdf_threshold=0.9)          # sim_threshold is required


def test_compile_gives_the_eager_mask():
    q = _smooth(2, 4, 1000, 96, BF, seed=70)
    k = _smooth(2, 2, 700, 96, BF, seed=71)
    fn = lambda q, k: sab.predict_block_mask(q, k, cdf_threshold=0.9, sim_threshold=0.5)
    assert torch.equal(torch.compile(fn, fullgraph=True)(q, k), fn(q, k))
