"""CPU tests of the block-mask predictor: properties of the fp64 restatement (block_predict_oracle), the C entries' argument
checks (no GPU needed: they run before anything touches the device) and the public function's guards."""
import math

import pytest
import torch

from block_predict_oracle import block_stats, predict_block_mask, scores, select


def _qk(B, Hq, Hkv, Sq, Sk, D, seed=0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(B, Hq, Sq, D, generator=g, dtype=torch.float64),
            torch.randn(B, Hkv, Sk, D, generator=g, dtype=torch.float64))


def test_self_similarity_is_the_mean_of_the_cosine_matrix():
    g = torch.Generator().manual_seed(1)
    x = torch.randn(1, 2, 300, 48, generator=g, dtype=torch.float64)
    x[0, 0, 5] = 0.0                                  # a zero row: unit vector 0, cosine 0 against every row
    mean, sim = block_stats(x, 128)
    for h in range(2):
        for c in range(3):
            blk = x[0, h, 128 * c:128 * c + 128]
            n = blk.norm(dim=-1, keepdim=True)
            u = torch.where(n > 0, blk / n.clamp_min(1e-300), torch.zeros_like(blk))
            assert torch.allclose(sim[0, h, c], (u @ u.T).mean(), rtol=1e-12, atol=0)
            assert torch.allclose(mean[0, h, c], blk.mean(0), rtol=1e-12, atol=1e-15)
            assert 0 <= sim[0, h, c] <= 1
    assert block_stats(x[..., :40], 64)[1].shape == (1, 2, 5)


def test_softmax_ignores_a_k_mean():
    q, k = _qk(1, 2, 1, 256, 320, 64, seed=2)
    qm, _ = block_stats(q, 128)
    km, _ = block_stats(k, 64)
    km2, _ = block_stats(k - k.mean(dim=2, keepdim=True), 64)
    p1 = torch.softmax(scores(qm, km, 0.125), -1)
    p2 = torch.softmax(scores(qm, km2, 0.125), -1)
    assert torch.allclose(p1, p2, rtol=1e-12, atol=1e-15)


@pytest.mark.parametrize("causal", [False, True])
def test_raising_cdf_never_removes_a_block(causal):
    q, k = _qk(2, 4, 2, 640, 640, 64, seed=3)
    prev = None
    for cdf in (0.05, 0.2, 0.5, 0.8, 0.95, 0.999, 1.0):
        m, _ = predict_block_mask(q, k, cdf_threshold=cdf, sim_threshold=0.0, is_causal=causal)
        if prev is not None:
            assert torch.all(m | ~prev), cdf
        prev = m
    assert torch.all(prev == predict_block_mask(q, k, cdf_threshold=1.0, sim_threshold=2.0, is_causal=causal)[0])


def test_ties_are_taken_in_ascending_j():
    D = 16
    qm = torch.zeros(1, 1, 1, D, dtype=torch.float64)
    km = torch.zeros(1, 1, 6, D, dtype=torch.float64)
    km[0, 0, 4, 0] = 1.0
    qm[0, 0, 0, 0] = 1.0                              # block 4 scores sm_scale, the others 0 (tied)
    one = torch.ones(1, 1, 1, dtype=torch.float64)
    ks = torch.ones(1, 1, 6, dtype=torch.float64)
    p = torch.softmax(torch.tensor([0, 0, 0, 0, 1.0, 0]), 0)
    # order: 4, then 0, 1, 2, 3, 5; block 4 plus two tied blocks carry p4 + 2 p0
    cdf = p[4].item() + 1.5 * p[0].item()
    m, near = select(qm, one, km, ks, 128, 384, cdf_threshold=cdf, sim_threshold=0.5, sm_scale=1.0, eps=1e-9)
    assert m[0, 0, 0].tolist() == [True, True, False, False, True, False] and not near.any()


def test_causal_horizon_diagonal_and_no_empty_row():
    q, k = _qk(1, 4, 2, 1000, 1000, 64, seed=4)
    for cdf, sim in ((0.01, 0.0), (0.5, 0.3), (0.9, -1.0), (1.0, 2.0)):
        m, _ = predict_block_mask(q, k, cdf_threshold=cdf, sim_threshold=sim, is_causal=True)
        nq, nk = m.shape[2:]
        i = torch.arange(nq)[:, None]
        j = torch.arange(nk)[None, :]
        assert not torch.any(m & (64 * j > 128 * i + 127))
        diag = (128 * i <= 64 * j + 63) & (64 * j <= 128 * i + 127)
        assert torch.all(m[..., diag])
        assert torch.all(m.any(-1))


def _piecewise(B, Hq, Hkv, nq, nk, D, seed):
    """Every 128-query block and every 64-key block is one token repeated: pooled scores are the true block scores."""
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(B, Hq, nq, 1, D, generator=g, dtype=torch.float64).mul(2.0).expand(-1, -1, -1, 128, -1)
    k = torch.randn(B, Hkv, nk, 1, D, generator=g, dtype=torch.float64).mul(2.0).expand(-1, -1, -1, 64, -1)
    return q.reshape(B, Hq, nq * 128, D), k.reshape(B, Hkv, nk * 64, D)


def _captured_mass(q, k, mask, sm_scale):
    """Per query row, the exact fp64 attention mass inside the element-expanded block mask: [B,Hq,Sq]."""
    g = q.size(1) // k.size(1)
    p = torch.softmax(sm_scale * q @ k.repeat_interleave(g, 1).transpose(-1, -2), -1)
    em = mask.repeat_interleave(128, 2)[:, :, :q.size(2)].repeat_interleave(64, 3)[..., :k.size(2)]
    return (p * em).sum(-1)


@pytest.mark.parametrize("cdf", [0.3, 0.7, 0.9, 0.99])
@pytest.mark.parametrize("sim", [-1.0, 0.5, 0.99])
def test_piecewise_constant_data_captures_cdf_mass(cdf, sim):
    q, k = _piecewise(1, 4, 2, 4, 12, 32, seed=int(cdf * 100 + sim * 10))
    m, _ = predict_block_mask(q, k, cdf_threshold=cdf, sim_threshold=sim)
    mass = _captured_mass(q, k, m, 32 ** -0.5)
    assert mass.min().item() >= cdf - 1e-12, (mass.min().item(), cdf)
    assert m.float().mean() < 1.0 or cdf > 0.9      # the selection really drops blocks


# ------------------------------------------------------------------------------------------------ C entries, no GPU
def _stats(lib, x=16, dtype=0, D=64, strides=(0, 0, 64), blk=128):
    return lib.sab_block_stats(x, dtype, 16, 16, 1, 1, 128, D, *strides, blk, None)


def _pred(lib, ptr=16, Hq=2, Hkv=2, Sq=128, Skv=128, D=64, causal=0, cdf=0.5, sim=0.5, scale=0.125):
    return lib.sab_predict_block_mask(ptr, 16, 16, 16, 16, 1, Hq, Hkv, Sq, Skv, D, causal, scale, cdf, sim, None)


def test_c_entries_validate_without_a_gpu():
    from sageattention_b200 import _capi
    lib = _capi.lib()
    err = lambda: lib.sab_last_error()
    assert _stats(lib, x=None) == -1 and b"null" in err()
    assert _stats(lib, dtype=2) == -2 and b"half and bfloat16" in err()
    assert _stats(lib, D=136) == -2 and b"head dim" in err()
    assert _stats(lib, D=60) == -2 and b"head dim" in err()
    assert _stats(lib, strides=(0, -64, 64)) == -1 and b">= 0" in err()
    assert _stats(lib, strides=(0, 0, 60)) == -1 and b"multiple of 8" in err()
    assert _stats(lib, blk=32) == -1 and b"64 or 128" in err()
    assert _pred(lib, ptr=None) == -1 and b"null" in err()
    assert _pred(lib, D=0) == -2 and b"head dim" in err()
    assert _pred(lib, Hq=3) == -1 and b"divisible" in err()
    assert _pred(lib, Skv=(1 << 20) + 1) == -2 and b"kv_len <= 1048576" in err()
    assert _pred(lib, causal=1, Skv=256) == -1 and b"must be equal for causal" in err()
    assert _pred(lib, cdf=0.0) == -1 and b"cdf_threshold" in err()
    assert _pred(lib, cdf=-0.5) == -1 and b"cdf_threshold" in err()
    assert _pred(lib, cdf=math.nan) == -1 and b"cdf_threshold" in err()
    assert _pred(lib, sim=math.nan) == -1 and b"sim_threshold" in err()
    assert _pred(lib, scale=math.inf) == -1 and b"sm_scale" in err()


def test_public_function_exists_and_rejects_cpu_tensors():
    import inspect
    import sageattention_b200 as sab
    assert "predict_block_mask" in sab.__all__ and callable(sab.predict_block_mask)
    sig = inspect.signature(sab.predict_block_mask)
    assert list(sig.parameters)[:2] == ["q", "k"]
    for name in ("cdf_threshold", "sim_threshold"):     # required: no tuned default exists
        assert sig.parameters[name].kind == inspect.Parameter.KEYWORD_ONLY
        assert sig.parameters[name].default is inspect.Parameter.empty
    q = torch.randn(1, 2, 128, 64, dtype=torch.float16)
    with pytest.raises(AssertionError):
        sab.predict_block_mask(q, q, cdf_threshold=0.9, sim_threshold=0.5)
