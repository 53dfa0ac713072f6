"""GPU tests (-m gpu) of the masked forms of the INT8+FP8 forward kernel (sage_attn_fwd_kernel with kWindow or the block mask,
csrc/attn.cu) at their edges, element by element against the bound of attn_window_oracle (check_forward) on the kernel's own
quantised operands:
  1. every dense window instantiation: windows (0,0), (1,0), (63,64), (127,0), (130,0), (200,37), (-1,100) at lengths 1 to 129,
     300 x 700 and 700 x 300; B = 2, GQA, HND and NHD, D 64 / 96 / 128, V range 448 and 2.25, smooth_v with its v_mean, causal or
     not; rows with no visible key must be exactly 0 with lse -inf;
  2. every dense block-sparse instantiation, causal: masks that hide exactly one tile of a diagonal 64-key pair (either one),
     whole rows, and list the partial last tile; and one packed causal call with Lq != Lk, per sequence on the dense quantisers'
     operands of that sequence (the packed quantisers give the same bits, tests/test_gpu_varlen_fp8.py);
  3. the ramp and sink inputs of test_gpu_kernel_edges, under windows and sparse masks, where the lazy running max moves after a
     row's first visible tile on at least 25 % of rows;
  4. all of the above with SAB_ATTN_KERNEL=exact (lazy_tau = 0), in a subprocess.
Each test prints the worst error / bound ratio of its family and the share of ambiguous elements."""
import os
import subprocess
import sys

import pytest
import torch

from attn_bwd_oracle import check_elementwise
from attn_window_oracle import attn_int8_fp8_blocksparse_causal, attn_int8_fp8_window, check_forward
from test_gpu_kernel_edges import _max_inputs
from test_gpu_parity import ROOT, _kernel_tau

pytestmark = pytest.mark.gpu
BF, FP = torch.bfloat16, torch.float16

WINDOWS = [(0, 0), (1, 0), (63, 64), (127, 0), (130, 0), (200, 37), (-1, 100)]
LENGTHS = [(1, 1), (63, 63), (64, 64), (65, 65), (127, 127), (129, 129), (300, 700), (700, 300)]
# (D, dtype, gran, layout, B, Hq, Hkv, pv_accum_dtype, smooth_v, causal): every (padded D, per-thread K scales, dtype)
WINDOW_CASES = [
    (128, FP, "per_thread", "HND", 2, 4, 2, "fp32+fp32", False, False),
    (96, BF, "per_thread", "NHD", 1, 4, 1, "fp32", True, True),
    (96, FP, "per_warp", "NHD", 1, 2, 2, "fp32+fp16", False, True),
    (128, BF, "per_warp", "HND", 2, 2, 1, "fp32", True, False),
    (64, FP, "per_thread", "NHD", 2, 2, 2, "fp32+fp16", False, False),
    (64, BF, "per_thread", "HND", 1, 4, 2, "fp32", True, True),
    (64, FP, "per_warp", "HND", 1, 4, 1, "fp32", False, False),
    (64, BF, "per_warp", "NHD", 2, 2, 2, "fp32+fp16", False, True),
]
# (D, dtype, gran, layout, B, Hq, Hkv, pv_accum_dtype, smooth_v), causal, at every length of SPARSE_LENGTHS
SPARSE_CASES = [
    (128, BF, "per_thread", "NHD", 2, 4, 2, "fp32", True),
    (128, FP, "per_thread", "HND", 1, 2, 2, "fp32+fp16", False),
    (96, BF, "per_warp", "HND", 1, 4, 1, "fp32+fp32", False),
    (128, FP, "per_warp", "NHD", 2, 2, 1, "fp32", True),
    (64, BF, "per_thread", "HND", 2, 2, 2, "fp32+fp16", False),
    (64, FP, "per_thread", "NHD", 1, 4, 2, "fp32", True),
    (64, BF, "per_warp", "NHD", 1, 2, 2, "fp32+fp32", False),
    (64, FP, "per_warp", "HND", 2, 4, 2, "fp32", False),
]
SPARSE_LENGTHS = [65, 129, 300, 700]


def _tau():
    return _kernel_tau(128) or 0


def _inputs(B, Hq, Hkv, Sq, Sk, D, dt, layout, seed, v_offset=False):
    g = torch.Generator(device="cuda").manual_seed(seed)
    q = torch.randn(B, Hq, Sq, D, generator=g, device="cuda")
    k = torch.randn(B, Hkv, Sk, D, generator=g, device="cuda") + torch.randn(B, Hkv, 1, D, generator=g, device="cuda")
    v = torch.randn(B, Hkv, Sk, D, generator=g, device="cuda")
    if v_offset:     # a per-channel offset, which smooth_v takes out
        v = v + 3.0 * torch.randn(D, generator=g, device="cuda")
    if layout == "NHD":
        q, k, v = (t.transpose(1, 2).contiguous() for t in (q, k, v))
    return q.to(dt), k.to(dt), v.to(dt)


def _hnd(x, layout):
    return (x if layout == "HND" else x.transpose(1, 2)).cpu()


def _operands(q, k, v, layout, gran, acc, smooth_v):
    """The public entry's quantised operands (head dim padded, K smoothed, V range of acc) on padded q, k, v, for the
    restatement: (q8, k8, v8, qs, ks, vs, vm), HND, on the CPU."""
    from sageattention_b200.core import _quant_qk
    from sageattention_b200.quant import per_channel_fp8
    _, q8, qs, k8, ks, _, _, _ = _quant_qk(q, k, "fp8", layout, gran, q.size(-1) ** -0.5, True, "cuda")
    v8, vs, vm = per_channel_fp8(v, tensor_layout=layout, scale_max=2.25 if acc == "fp32+fp16" else 448.0, smooth_v=smooth_v)
    Sk = k.size(2 if layout == "HND" else 1)
    return (_hnd(q8, layout), _hnd(k8, layout), v8[..., :Sk].transpose(-1, -2).cpu(), qs.cpu(), ks.cpu(), vs.cpu(),
            None if vm is None else vm.cpu())


def _run(q, k, v, layout, causal, gran, acc, smooth_v, window=None, block_mask=None):
    """The kernel as the public entry runs it, with its raw log2 lse, and its operands: (o, lse, *_operands(...)), o HND on the
    CPU without the padded columns."""
    from sageattention_b200.core import _attn_dense, _pad_head_dim
    D = q.size(-1)
    qp, kp, vp, _ = _pad_head_dim(q, k, v)
    o, lse, _ = _attn_dense(qp, kp, vp, "fp8", layout, causal, gran, D ** -0.5, True, smooth_v,
                            2.25 if acc == "fp32+fp16" else 448.0, "cuda", True, block_mask=block_mask, window=window)
    return (_hnd(o, layout)[..., :D], lse.cpu()) + _operands(qp, kp, vp, layout, gran, acc, smooth_v)


class _Stats:
    """Worst error / bound ratios and ambiguous elements of one family."""

    def __init__(self, name):
        self.name, self.o, self.lse, self.amb, self.vis, self.n = name, 0.0, 0.0, 0, 0, 0

    def add(self, ratios, bd):
        self.o, self.lse = max(self.o, ratios[0]), max(self.lse, ratios[1])
        self.amb, self.vis, self.n = self.amb + bd.ambiguous, self.vis + bd.visible, self.n + 1

    def report(self):
        print(f"[bound] {self.name} (tau {_tau()}): {self.n} calls, worst ratio o {self.o:.3f} lse {self.lse:.3f}, "
              f"ambiguous {self.amb} of {self.vis} visible elements ({self.amb / max(self.vis, 1):.2e})")


def _compare(name, res, D, dt, gran, oracle, stats, **kw):
    o, lse, q8, k8, v8, qs, ks, vs, vm = res
    oc, lc, bd = oracle(q8, k8, v8, qs, ks, vs, qk_quant_gran=gran, sm_scale=D ** -0.5, lazy_tau=_tau(), out_dtype=dt,
                        return_lse=True, v_mean=vm, bound=True, **kw)
    bd = bd._replace(o=bd.o[..., :D], o_bound=bd.o_bound[..., :D])
    stats.add(check_forward(name, o, lse, lc, bd), bd)
    return bd


# ------------------------------------------------------------------------------------------------ 1. windows
def _window_case(case):
    D, dt, gran, layout, B, Hq, Hkv, acc, smooth_v, causal = case
    stats = _Stats(f"window {case}")
    for i, (Sq, Sk) in enumerate(LENGTHS):
        if causal and Sq != Sk:
            continue
        q, k, v = _inputs(B, Hq, Hkv, Sq, Sk, D, dt, layout, seed=10 * i + D, v_offset=smooth_v)
        for window in WINDOWS:
            res = _run(q, k, v, layout, causal, gran, acc, smooth_v, window=window)
            _compare(f"{case} {Sq}x{Sk} window {window}", res, D, dt, gran, attn_int8_fp8_window, stats, window=window,
                     is_causal=causal)
    return stats


@pytest.mark.parametrize("case", WINDOW_CASES, ids=lambda c: "-".join(str(x).replace("torch.", "") for x in c))
def test_window_edges_against_the_bound(case):
    _window_case(case).report()


# ------------------------------------------------------------------------------------------------ 2. block-sparse, causal
def _edge_mask(B, Hq, S, seed):
    """A causal block mask [B,Hq,nq,nk]: Q-block rows cycle through hiding the diagonal pair's first tile only, its second tile
    only, the whole row (Q block 1) and a random row; every row that is not hidden lists the partial last tile."""
    nq, nk = (S + 127) // 128, (S + 63) // 64
    g = torch.Generator().manual_seed(seed)
    bm = torch.rand(B, Hq, nq, nk, generator=g) < 0.6
    for b in range(B):
        for h in range(Hq):
            for i in range(nq):
                kind = (b * Hq + h + i) % 4
                d0, d1 = 2 * i, min(2 * i + 1, nk - 1)
                if kind == 0:
                    bm[b, h, i, d0], bm[b, h, i, d1] = False, True
                elif kind == 1:
                    bm[b, h, i, d0], bm[b, h, i, d1] = True, d1 == d0
                if kind == 2 and i == 1:
                    bm[b, h, i] = False
                else:
                    bm[b, h, i, nk - 1] = True
    return bm


def _sparse_case(case):
    D, dt, gran, layout, B, Hq, Hkv, acc, smooth_v = case
    stats = _Stats(f"block-sparse {case}")
    for S in SPARSE_LENGTHS:
        q, k, v = _inputs(B, Hq, Hkv, S, S, D, dt, layout, seed=S + D, v_offset=smooth_v)
        bm = _edge_mask(B, Hq, S, seed=S)
        res = _run(q, k, v, layout, True, gran, acc, smooth_v, block_mask=bm.cuda())
        _compare(f"{case} S={S}", res, D, dt, gran, attn_int8_fp8_blocksparse_causal, stats, block_mask=bm)
    return stats


@pytest.mark.parametrize("case", SPARSE_CASES, ids=lambda c: "-".join(str(x).replace("torch.", "") for x in c))
def test_causal_block_sparse_edges_against_the_bound(case):
    _sparse_case(case).report()


def _packed_causal_case():
    """sageattn_varlen_blocksparse, causal (top-left) with Lq != Lk: each sequence's rows against the restatement on the dense
    quantisers' operands of that sequence (whose bits the packed quantisers give), output within the bound and 0 on rows that see
    no key."""
    import sageattention_b200 as sab
    from test_gpu_varlen_fp8 import _cu, _packed, _spans
    lens_q, lens_k = [100, 64, 1, 300, 129, 200], [300, 64, 129, 50, 1, 200]
    Hq, Hkv, D, dt, gran = 4, 2, 128, FP, "per_warp"
    q, k, v, _ = _packed(lens_q, lens_k, Hq, Hkv, D, dt, seed=31)
    mq, mk = max(lens_q), max(lens_k)
    bm = _edge_mask(len(lens_q), Hq, max(mq, mk), seed=5)[:, :, :(mq + 127) // 128, :(mk + 63) // 64].contiguous()
    bm[:, :, 0, 0] = False                         # the first rows of every sequence see nothing
    o = sab.sageattn_varlen_blocksparse(q, k, v, _cu(lens_q), _cu(lens_k), mq, mk, bm.cuda(), is_causal=True,
                                        qk_quant_gran=gran, pv_accum_dtype="fp32+fp32")
    stats = _Stats("packed block-sparse causal Lq != Lk")
    for b, ((s, e), (sk, ek)) in enumerate(zip(_spans(lens_q), _spans(lens_k))):
        q8, k8, v8, qs, ks, vs, _ = _operands(q[s:e][None], k[sk:ek][None], v[sk:ek][None], "NHD", gran, "fp32+fp32", False)
        mb = bm[b:b + 1, :, :(e - s + 127) // 128, :(ek - sk + 63) // 64]
        _, _, bd = attn_int8_fp8_blocksparse_causal(q8, k8, v8, qs, ks, vs, mb, qk_quant_gran=gran, sm_scale=D ** -0.5,
                                                    lazy_tau=_tau(), out_dtype=dt, return_lse=True, bound=True)
        worst, _ = check_elementwise(f"sequence {b}", o[s:e].transpose(0, 1)[None].cpu(), bd.o, bd.o_bound)
        stats.add((worst, 0.0), bd)
    return stats


def test_packed_causal_block_sparse_with_unequal_lengths_against_the_bound():
    _packed_causal_case().report()


# ------------------------------------------------------------------------------------------------ 3. running-max movement
MAX_CASES = [(128, FP, "per_thread", "ramp48"), (64, BF, "per_warp", "ramp160"), (128, BF, "per_warp", "sink"),
             (64, FP, "per_thread", "sink")]


def _max_case(case):
    """Ramps under a causal window, a non-causal window and a causal sparse mask; the sink (one key in the last tile) under two
    non-causal windows whose every row sees it.  At least 25 % of the rows that see a key must move their running max after their
    first visible tile (restated), or the inputs do not exercise the rescale."""
    D, dt, gran, kind = case
    q, k, v = _max_inputs(D, dt, kind)
    S = q.size(2)
    stats = _Stats(f"running max {case}")
    if kind == "sink":
        runs = [(False, dict(window=(900, -1))), (False, dict(window=(100, 1000)))]
    else:
        bm = _edge_mask(1, 2, S, seed=D)
        runs = [(True, dict(window=(300, 0))), (False, dict(window=(200, 150))), (True, dict(block_mask=bm))]
    for causal, kw in runs:
        what = kw.get("window", "sparse")
        if "window" in kw:
            res = _run(q, k, v, "HND", causal, gran, "fp32+fp32", False, window=kw["window"])
            bd = _compare(f"{case} {what}", res, D, dt, gran, attn_int8_fp8_window, stats, is_causal=causal, **kw)
        else:
            res = _run(q, k, v, "HND", causal, gran, "fp32+fp32", False, block_mask=bm.cuda())
            bd = _compare(f"{case} {what}", res, D, dt, gran, attn_int8_fp8_blocksparse_causal, stats, **kw)
        frac = bd.moved / bd.rows
        print(f"[max] {case} {what}: the running max moves after the first visible tile on {frac:.2f} of rows")
        assert frac >= 0.25, f"{case} {what}: the running max moves on only {frac:.2f} of rows"
    return stats


@pytest.mark.parametrize("case", MAX_CASES, ids=lambda c: f"D{c[0]}-{str(c[1])[6:]}-{c[2]}-{c[3]}")
def test_running_max_moves_under_masks_against_the_bound(case):
    _max_case(case).report()


# ------------------------------------------------------------------------------------------------ 4. exact running max
def test_everything_again_with_the_exact_running_max():
    """SAB_ATTN_KERNEL=exact is read once per process: a subprocess runs every case above with lazy_tau = 0."""
    code = ("import sys; sys.path[:0] = [%r, %r]\n" % (os.path.join(ROOT, "tests"), ROOT) +
            "import test_gpu_masked_forward_edges as T\n"
            "assert T._tau() == 0\n"
            "for c in T.WINDOW_CASES: T._window_case(c).report()\n"
            "for c in T.SPARSE_CASES: T._sparse_case(c).report()\n"
            "T._packed_causal_case().report()\n"
            "for c in T.MAX_CASES: T._max_case(c).report()\n"
            "print('EXACT_OK')\n")
    env = dict(os.environ, SAB_ATTN_KERNEL="exact")
    p = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=1800)
    print(p.stdout[-6000:])
    assert p.returncode == 0 and "EXACT_OK" in p.stdout, p.stdout[-3000:] + p.stderr[-3000:]
