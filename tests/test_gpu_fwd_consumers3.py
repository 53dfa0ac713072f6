"""GPU tests (-m gpu): the three-consumer form of the dense INT8+FP8 forward kernel at head dim 128 (csrc/attn.cu, kNC = 3, 192-row
Q tiles) against the two-consumer form (SAB_ATTN_CONSUMERS=2, 128-row Q tiles), bit for bit in the output and the lse.

Both forms run each row through the same per-element arithmetic: the same 64-key tiles in the same order, the FP8 tile product
accumulated from zero in the tensor core (a column's value does not depend on whether it is computed in an N = 128 or an N = 64
product) and folded into O in fp32 after the same rescale.  A row of the bigger tile can see more fully masked causal tiles,
which add exactly zero.  So any difference is a defect: a row base, a scale index, a masked-tile decision or a fold.

The selectors are read once per process, so each form runs in a subprocess of its own on the same seeded inputs.  Lengths cover
one Q tile and less (64, 128, 191), the tile boundary (192, 193), the benchmark length (8192: 43 tiles, the last one with 128 valid
rows), Sq != Skv without causal, and grouped-query heads; each with bf16 and fp16 outputs, per-warp and per-thread scales,
causal and not.  The default run also shows, by kernel name in a profiler trace, that it ran the three-consumer kernel."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (B, Hq, Hkv, Sq, Skv, causal)
SHAPES = [(1, 2, 2, s, s, c) for s in (64, 128, 191, 192, 193, 8192) for c in (False, True)] + [
    (2, 2, 2, 193, 1000, False),
    (1, 2, 2, 500, 129, False),
    (1, 2, 2, 64, 4096, False),
    (2, 8, 2, 777, 777, False),
    (2, 8, 2, 777, 777, True),
]
CASES = [(shape, dt, gran) for shape in SHAPES for dt in ("bfloat16", "float16") for gran in ("per_warp", "per_thread")]


def _dump(path):
    """Runs every case on this process's kernel forms and saves the outputs, lse and the forward kernels' names to path."""
    sys.path.insert(0, ROOT)
    import sageattention_b200 as sab
    dev = torch.device("cuda:0")
    res = {}
    for i, ((B, Hq, Hkv, Sq, Skv, causal), dt, gran) in enumerate(CASES):
        g = torch.Generator(device=dev).manual_seed(1000 + i)
        dtype = getattr(torch, dt)
        q = torch.randn(B, Hq, Sq, 128, device=dev, dtype=dtype, generator=g)
        k = torch.randn(B, Hkv, Skv, 128, device=dev, dtype=dtype, generator=g)
        v = torch.randn(B, Hkv, Skv, 128, device=dev, dtype=dtype, generator=g)
        k = k + 2.0 * torch.randn(B, Hkv, 1, 128, device=dev, dtype=dtype, generator=g)   # a common K offset, as in real models
        o, lse = sab.sageattn_qk_int8_pv_fp8_cuda(q, k, v, tensor_layout="HND", is_causal=causal, qk_quant_gran=gran,
                                                  return_lse=True)
        res[i] = (o.cpu(), lse.cpu())
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    q = torch.randn(1, 2, 1024, 128, device=dev, dtype=torch.bfloat16)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        sab.sageattn_qk_int8_pv_fp8_cuda(q, q, q, tensor_layout="HND")
        torch.cuda.synchronize()
    res["kernels"] = sorted({e.key for e in prof.key_averages() if "sage_attn_fwd_kernel" in e.key})
    torch.save(res, path)


def _run(tmp_path, consumers, max_mode):
    path = str(tmp_path / f"c{consumers}_{max_mode}.pt")
    env = dict(os.environ)
    env.pop("SAB_ATTN_CONSUMERS", None)
    env.pop("SAB_ATTN_KERNEL", None)
    if consumers == 2:
        env["SAB_ATTN_CONSUMERS"] = "2"
    if max_mode == "exact":
        env["SAB_ATTN_KERNEL"] = "exact"
    code = "import sys; sys.path[:0] = [%r, %r]\nimport test_gpu_fwd_consumers3 as T\nT._dump(%r)\n" % (
        os.path.join(ROOT, "tests"), ROOT, path)
    p = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=1800)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
    return torch.load(path)


@pytest.mark.parametrize("max_mode", ["lazy", "exact"])
def test_three_consumers_match_two_bit_for_bit(tmp_path, max_mode):
    three, two = _run(tmp_path, 3, max_mode), _run(tmp_path, 2, max_mode)
    assert any(", 3>" in k for k in three["kernels"]), f"the default run did not use the three-consumer kernel: {three['kernels']}"
    assert not any(", 3>" in k for k in two["kernels"]), f"SAB_ATTN_CONSUMERS=2 still ran three consumers: {two['kernels']}"
    bad = []
    for i, case in enumerate(CASES):
        (o3, l3), (o2, l2) = three[i], two[i]
        assert o3.shape == o2.shape and l3.shape == l2.shape
        if not torch.equal(o3.view(torch.int16), o2.view(torch.int16)) or not torch.equal(l3.view(torch.int32), l2.view(torch.int32)):
            n = (o3.view(torch.int16) != o2.view(torch.int16)).sum().item()
            bad.append(f"{case}: {n} output elements differ, lse max diff {(l3 - l2).abs().max().item():.3e}")
    assert not bad, "\n".join(bad[:20])
