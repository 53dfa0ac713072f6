"""CPU tests of the 8-bit paged KV cache at the inputs serving engines pass it (tests/test_gpu_kvcache8_edges.py runs the kernels
on the same inputs):
  1. quant_rows pinned to values worked out by hand, so a restatement sharing a kernel's rounding bug cannot pass: int8 and e4m3
     ties round half to even, products that round above qmax saturate, and a denormal-range amax takes the exact quotient;
  2. the quantiser edges the GPU tests feed the kernels exist in bf16 and fp16: amax values whose amax * RN(qmax / amax) rounds
     above qmax, and the amax thresholds below which RN(qmax / amax) overflows;
  3. the host passes strided q, a column slice of a wider block table and int64 cu_seqlens_q to the ops as they are (no copy of q
     or of the table, offsets as int32), and accepts a max_seqlen_q below a sequence's length;
  4. the restatements at GQA ratios 7 and 64, at sm_scale 1.0 / 0.02 / 0.3, and with a large common K offset against fp64
     attention on the 16-bit tokens; the 131072-key decode restatement the GPU tests use runs in seconds."""
import math
import time

import pytest
import torch

from attn_kvcache8_oracle import attend, quant_rows, write
from attn_kvcache8_prefill_oracle import attend_folded
from attn_kvcache8_window_oracle import attend as attend_w, visible_keys

FLT_MAX = torch.finfo(torch.float32).max


def _fp64(q, k, v, is_causal, sm_scale, window=(-1, -1)):
    """fp64 attention of one sequence on its 16-bit tokens, bottom-right, with an optional window."""
    Lq, Hq, D = q.shape
    Lk = k.size(0)
    g = Hq // k.size(1)
    kh = k.double().repeat_interleave(g, 1).transpose(0, 1)
    vh = v.double().repeat_interleave(g, 1).transpose(0, 1)
    s = (q.double().transpose(0, 1) @ kh.transpose(1, 2)) * sm_scale
    first, last = visible_keys(Lq, Lk, is_causal, window)
    j = torch.arange(Lk)[None, :]
    s = s.masked_fill(~((j <= last) & (j >= first)), -math.inf)
    lse = torch.logsumexp(s, -1)
    p = torch.exp(s - lse[..., None]).nan_to_num(0.0)
    return (p @ vh).transpose(0, 1), lse


# ------------------------------------------------------------------------------------------------ 1. hand-computed anchors
def test_int8_ties_round_half_to_even():
    # amax 127: scale = 127 / 127 = 1 and RN(127 / 127) = 1, so every element reaches the rounding as it is
    x = torch.tensor([[0.5, -0.5, 1.5, -1.5, 2.5, -2.5, 126.5, -126.5, 3.5, 127.0]])
    q, s = quant_rows(x, 127.0, fp8=False)
    assert s.tolist() == [1.0]
    assert q[0].tolist() == [0.0, 0.0, 2.0, -2.0, 2.0, -2.0, 126.0, -126.0, 4.0, 127.0]


def test_e4m3_ties_round_half_to_even():
    # amax 448: scale 1, RN(448 / 448) = 1.  e4m3 steps are 2 on [16, 32), 2^-9 below 2^-6 (subnormals); each x is a midpoint
    u = 2.0 ** -9
    x = torch.tensor([[17.0, 19.0, -17.0, 1.5 * u, 2.5 * u, 0.5 * u, -1.5 * u, 3.5 * u, 232.0, 448.0]])
    q, s = quant_rows(x, 448.0, fp8=True)
    assert s.tolist() == [1.0]
    # 17 -> 16 (mantissa 000), 19 -> 20 (010), 1.5u -> 2u, 2.5u -> 2u, 0.5u -> 0, 3.5u -> 4u; 232 (steps of 16) -> 224
    assert q[0].tolist() == [16.0, 20.0, -16.0, 2 * u, 2 * u, 0.0, -2 * u, 4 * u, 224.0, 448.0]


def test_products_that_round_above_qmax_saturate():
    # bf16 4.408103815583578e-37 (0x03160000): RN(127 / a) * a = 127.0000076 in fp32, which must give 127, not overflow
    a = torch.tensor([0x0316], dtype=torch.int16).view(torch.bfloat16).float()
    assert a.item() == pytest.approx(4.408103815583578e-37, rel=1e-12)
    assert (a * (torch.tensor(127.0) / a)).item() == 127.00000762939453
    q, _ = quant_rows(torch.cat([a, -a, a / 2]).view(1, 3), 127.0, fp8=False)
    assert q[0].tolist() == [127.0, -127.0, 64.0]
    # fp16 7.748603820800781e-07 (13 x 2^-24): RN(448 / a) * a = 448.0000305; e4m3 saturates to 448
    b = torch.tensor([13 * 2.0 ** -24])
    assert (b * (torch.tensor(448.0) / b)).item() == 448.0000305175781
    v, _ = quant_rows(torch.cat([b, -b]).view(1, 2), 448.0, fp8=True)
    assert v[0].tolist() == [448.0, -448.0]


def test_the_exact_branch_below_the_overflow_threshold():
    # amax = 2^-126: RN(127 / amax) = inf, so x / scale with scale = RN(2^-126 / 127) = 66052 x 2^-149 (a denormal; 2^23 / 127 =
    # 66052.03).  x = amax gives 2^23 / 66052 = 127.00006 -> 127; x = amax / 2 gives 63.50003 -> 64 (no tie); amax / 127 gives 1.0
    a = 2.0 ** -126
    x = torch.tensor([[a, -a, a / 2, 0.75 * a, -a / 4, a / 127, 0.0]])
    q, s = quant_rows(x, 127.0, fp8=False)
    assert s.item() == 66052 * 2.0 ** -149
    assert q[0].tolist() == [127.0, -127.0, 64.0, 95.0, -32.0, 1.0, 0.0]
    # V: scale = RN(2^-126 / 448) = 18725 x 2^-149 (2^23 / 448 = 18724.57); amax / scale = 447.99 -> 448, -0.3 amax -> -134.4 -> -128
    v, vs = quant_rows(torch.tensor([[a, a / 2, -0.3 * a]]), 448.0, fp8=True)
    assert vs.item() == 18725 * 2.0 ** -149
    assert v[0].tolist() == [448.0, 224.0, -128.0]


def test_k_zero_with_a_denormal_k_smooth():
    # k = 0 and k_smooth in the fp32 denormal range: x = -k_smooth, amax = 3 x 2^-140 = 1536 x 2^-149, so RN(127 / amax) = inf and
    # the exact branch runs with scale = RN(1536 x 2^-149 / 127) = 12 x 2^-149 (1536 / 127 = 12.09).  x / scale is then
    ksm = torch.zeros(1, 64)
    ksm[0, :4] = torch.tensor([3.0, -1.5, 0.75, 2.0]) * 2.0 ** -140
    k8, ks, _, _ = write(torch.zeros(1, 1, 64, dtype=torch.bfloat16), torch.ones(1, 1, 64, dtype=torch.bfloat16), ksm)
    assert ks.item() == 12 * 2.0 ** -149
    # -1536 / 12 = -128 (int8's own minimum), 768 / 12 = 64, -384 / 12 = -32, -1024 / 12 = -85.33 -> -85, and 0
    assert k8[0, 0, :5].tolist() == [-128.0, 64.0, -32.0, -85.0, 0.0]


# ------------------------------------------------------------------------------------------------ 2. searched edges
def _positive_finite(dt):
    top = 0x7C00 if dt == torch.float16 else 0x7F80
    return torch.arange(1, top, dtype=torch.int32).to(torch.int16).view(dt).float()


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("qmax", [127.0, 448.0])
def test_amax_values_whose_product_rounds_above_qmax_exist_and_saturate(dt, qmax):
    a = _positive_finite(dt)
    mult = torch.tensor(qmax) / a
    over = torch.isfinite(mult) & (a * mult > qmax)
    assert over.sum() > 1000
    x = torch.stack([a[over], -a[over]], -1)
    q, _ = quant_rows(x, qmax, fp8=qmax == 448.0)
    assert (q[:, 0] == qmax).all() and (q[:, 1] == -qmax).all()


@pytest.mark.parametrize("qmax", [127.0, 448.0])
def test_the_overflow_threshold_of_bf16_amax(qmax):
    """bf16 reaches below qmax / FLT_MAX: the amax values on either side of the point where RN(qmax / amax) overflows."""
    a = _positive_finite(torch.bfloat16)
    inf = torch.isinf(torch.tensor(qmax) / a)
    below, above = a[inf].max(), a[~inf].min()
    assert below < qmax / FLT_MAX <= above and (a[inf] < above).all()
    assert torch.isfinite(torch.tensor(qmax) / above)
    for amax in (below, above):
        q, s = quant_rows(torch.stack([amax, -amax / 3]).view(1, 2), qmax, fp8=qmax == 448.0)
        assert s.item() == (amax / qmax).item() and abs(q[0, 0].item()) == qmax
    # fp16 never gets there: its smallest denormal, 2^-24, is far above 448 / FLT_MAX
    assert torch.isfinite(torch.tensor(127.0) / _positive_finite(torch.float16)).all()


# ------------------------------------------------------------------------------------------------ 3. host handling
def _cpu_cache(Hkv, D, page_size=16, num_pages=8):
    from sageattention_b200 import kvcache8
    cache = kvcache8.PagedKVCache8.__new__(kvcache8.PagedKVCache8)
    cache.dtype, cache.device = torch.bfloat16, torch.device("cpu")
    cache.k_pages = torch.zeros(num_pages, page_size, Hkv, D, dtype=torch.int8)
    cache.v_pages = torch.zeros(num_pages, page_size, Hkv, D, dtype=torch.float8_e4m3fn)
    cache.k_scale = cache.v_scale = torch.zeros(num_pages, page_size, Hkv)
    cache.k_smooth = torch.zeros(Hkv, D)
    return cache


@pytest.mark.parametrize("prefill", [False, True])
@pytest.mark.parametrize("window", [(-1, -1), (7, 5)])
def test_views_and_int64_offsets_reach_the_op_unchanged(monkeypatch, prefill, window):
    import sageattention_b200 as sab
    from sageattention_b200 import kvcache8
    Hq, Hkv, D = 28, 4, 64
    cache = _cpu_cache(Hkv, D)
    calls = []
    name = ("kvcache8_prefill" if prefill else "kvcache8_attn") + ("" if window == (-1, -1) else "_window")
    monkeypatch.setattr(kvcache8.ops, name, lambda *a: calls.append(a) or torch.empty(0))
    qkv = torch.zeros(5, Hq + 2 * Hkv, D, dtype=torch.bfloat16)
    q = qkv[:, :Hq]
    wide = torch.arange(2 * 11, dtype=torch.int32).view(2, 11) % 8
    table = wide[:, :3]
    cu = torch.tensor([0, 2, 5], dtype=torch.int64)
    used = torch.tensor([20, 40], dtype=torch.int32)
    fn = sab.sageattn_kvcache8_prefill if prefill else sab.sageattn_kvcache8
    fn(q, cache, cu, used, table, 2, window_size=window)        # max_seqlen_q 2 < Lq_1 = 3: accepted, no host sync
    (a,) = calls
    assert a[0].data_ptr() == q.data_ptr() and a[0].stride() == q.stride()
    assert a[7].dtype == torch.int32 and a[7].tolist() == [0, 2, 5]
    assert a[9].data_ptr() == wide.data_ptr() and a[9].stride() == (11, 1) and tuple(a[9].shape) == (2, 3)
    assert a[10] == 2
    if window != (-1, -1):
        assert a[-2:] == window


# ------------------------------------------------------------------------------------------------ 4. the restatements
@pytest.mark.parametrize("Hq,Hkv", [(28, 4), (64, 1)])
@pytest.mark.parametrize("window", [(-1, -1), (7, 5)])
def test_restatements_at_odd_gqa_ratios_against_fp64(Hq, Hkv, window):
    causal = window == (-1, -1)
    g = torch.Generator().manual_seed(Hq + Hkv)
    Lq, Lk, D = 1, 300, 64
    q = torch.randn(Lq, Hq, D, generator=g).bfloat16()
    k = (torch.randn(Lk, Hkv, D, generator=g) + torch.randn(1, Hkv, D, generator=g)).bfloat16()
    v = torch.randn(Lk, Hkv, D, generator=g).bfloat16()
    ksm = k.float().mean(0)
    k8, ks, v8, vs = write(k, v, ksm)
    oe, le = _fp64(q, k, v, causal, D ** -0.5, window)
    for o, lse in (attend_w(q, k8, ks, v8, vs, ksm, causal, D ** -0.5, 128, window=window),
                   attend_folded(q, k8, ks, v8, vs, ksm, causal, D ** -0.5) if causal else
                   attend_w(q, k8, ks, v8, vs, ksm, causal, D ** -0.5, 1 << 20, window=window)):
        assert (o - oe).abs().max() < 0.1 and (o - oe).abs().mean() < 0.02
        assert (lse - le).abs().max() < 0.05
    # a row's heads follow head h // G of the KV heads: moving one KV head's keys moves exactly its G query heads
    k2 = k.clone()
    k2[:, Hkv - 1] = torch.randn(Lk, D, generator=g).bfloat16()
    o2, _ = attend(q, *write(k2, v, ksm), ksm, causal, D ** -0.5, 128)
    o1, _ = attend(q, k8, ks, v8, vs, ksm, causal, D ** -0.5, 128)
    G = Hq // Hkv
    changed = (o1 != o2).any(-1).any(0)
    assert changed[(Hkv - 1) * G:].all() and not changed[:(Hkv - 1) * G].any()


@pytest.mark.parametrize("sm_scale", [1.0, 0.02, 0.3])
def test_restatement_at_other_sm_scales_against_fp64(sm_scale):
    g = torch.Generator().manual_seed(int(sm_scale * 100))
    q = torch.randn(3, 8, 128, generator=g).bfloat16()
    k = (torch.randn(500, 2, 128, generator=g) + torch.randn(1, 2, 128, generator=g)).bfloat16()
    v = torch.randn(500, 2, 128, generator=g).bfloat16()
    ksm = k.float().mean(0)
    o, lse = attend(q, *write(k, v, ksm), ksm, True, sm_scale, 256)
    oe, le = _fp64(q, k, v, True, sm_scale)
    # sm_scale 1.0 makes the softmax nearly one-hot, so the 8-bit logit error shows more there
    assert (o - oe).abs().max() < (0.5 if sm_scale == 1.0 else 0.1)
    assert ((lse - le).abs() / le.abs().clamp_min(1.0)).max() < 0.05


def test_k_smooth_absorbs_a_large_common_offset():
    """Keys with a common bf16 offset of 50 and residual std 0.3: with k_smooth the mean, the 8-bit logits keep the residual's
    resolution; without it the offset takes the whole int8 range."""
    g = torch.Generator().manual_seed(50)
    q = torch.randn(2, 8, 128, generator=g).bfloat16()
    k = (50.0 + 0.3 * torch.randn(800, 2, 128, generator=g)).bfloat16()
    v = torch.randn(800, 2, 128, generator=g).bfloat16()
    oe, le = _fp64(q, k, v, True, 128 ** -0.5)
    errs = []
    for ksm in (torch.zeros(2, 128), k.float().mean(0)):
        o, lse = attend(q, *write(k, v, ksm), ksm, True, 128 ** -0.5, 1024)
        errs.append(((o - oe).abs().max().item(), (lse - le).abs().max().item()))
    print(f"offset 50: max error without / with k_smooth: o {errs[0][0]:.4f} / {errs[1][0]:.4f}, lse {errs[0][1]:.4f} / {errs[1][1]:.4f}")
    assert errs[1][0] < 0.05 and errs[1][1] < 0.05
    assert errs[1][0] < errs[0][0] / 4 and errs[1][1] < errs[0][1] / 4


def test_the_long_decode_restatement_runs_in_seconds():
    """The GPU tests restate 1 x 131072 keys at Hq 8, Hkv 2, D 128, Lq 4 with a bound: it has to stay a few seconds."""
    g = torch.Generator().manual_seed(0)
    Lk = 131072
    k8 = torch.randint(-127, 128, (Lk, 2, 128), generator=g).float()
    v8 = torch.randn(Lk, 2, 128, generator=g).to(torch.float8_e4m3fn).float()
    ks, vs = torch.rand(Lk, 2, generator=g) * 0.02, torch.rand(Lk, 2, generator=g) * 0.01
    q = torch.randn(4, 8, 128, generator=g).bfloat16()
    t = time.perf_counter()
    o, lse, ob, lb = attend(q, k8, ks, v8, vs, torch.zeros(2, 128), True, 128 ** -0.5, 1024, bound=True)
    took = time.perf_counter() - t
    print(f"131072-key decode restatement: {took:.2f} s")
    assert torch.isfinite(o).all() and torch.isfinite(lse).all() and took < 60
