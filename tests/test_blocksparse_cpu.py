"""CPU tests of the block-sparse attention: the CPU restatement (attn_blocksparse_oracle) against the dense restatement and
exact attention, the C entries' argument checks (no GPU needed: they run before anything touches the device) and the public
function's guards."""
import math

import pytest
import torch

from attn_blocksparse_oracle import attn_int8_fp8_blocksparse, expand_block_mask
from attn_bwd_oracle import elementwise_ratio
from attn_window_oracle import attn_int8_fp8_blocksparse_causal, attn_int8_fp8_tiles
from oracle import sage_oracle as O


def _operands(B, Hq, Hkv, Sq, Sk, D, gran, seed=0):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(B, Hq, Sq, D, generator=g).half()
    k = (torch.randn(B, Hkv, Sk, D, generator=g) + 2.0 * torch.randn(B, Hkv, 1, D, generator=g)).half()
    v = torch.randn(B, Hkv, Sk, D, generator=g).half()
    km = k.mean(dim=2, keepdim=True)
    if gran == "per_warp":
        q8, qs, k8, ks = O.per_warp_int8_cuda(q, k, km)
    else:
        q8, qs, k8, ks = O.quant_per_thread_int8_triton(q, k, km)
    v8, vs, _ = O.per_channel_fp8_cuda(v, "HND", 448.0)
    return q, k, v, q8, qs, k8, ks, v8, vs


def _mask(B, H, Sq, Sk, p, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(B, H, (Sq + 127) // 128, (Sk + 63) // 64, generator=g) < p


@pytest.mark.parametrize("gran", ["per_thread", "per_warp"])
def test_all_true_mask_is_the_dense_restatement_bitwise(gran):
    B, Hq, Hkv, Sq, Sk, D = 1, 2, 1, 200, 300, 64
    _, _, _, q8, qs, k8, ks, v8, vs = _operands(B, Hq, Hkv, Sq, Sk, D, gran)
    kw = dict(qk_quant_gran=gran, sm_scale=D ** -0.5, lazy_tau=4, return_lse=True)
    o_ref, l_ref = O.attn_int8_fp8_cuda(q8, k8, v8, qs, ks, vs, **kw)
    o, l = attn_int8_fp8_blocksparse(q8, k8, v8, qs, ks, vs, torch.ones(1, 1, 2, 5, dtype=torch.bool), **kw)
    assert torch.equal(o, o_ref) and torch.equal(l, l_ref)


def test_sparse_mask_matches_exact_masked_attention():
    B, Hq, Hkv, Sq, Sk, D = 1, 2, 1, 256, 320, 64
    q, k, v, q8, qs, k8, ks, v8, vs = _operands(B, Hq, Hkv, Sq, Sk, D, "per_thread", seed=1)
    bm = _mask(B, Hq, Sq, Sk, 0.5, 2)
    bm[0, 0, 0] = False          # a fully hidden Q-block row
    bm[0, 1, 1] = True           # a fully visible one
    o, lse = attn_int8_fp8_blocksparse(q8, k8, v8, qs, ks, vs, bm, sm_scale=D ** -0.5, lazy_tau=4, return_lse=True)
    em = expand_block_mask(bm, Sq, Sk)
    s = (q.double() @ k.double().repeat_interleave(Hq // Hkv, 1).transpose(-1, -2)) * D ** -0.5
    s = s.masked_fill(~em, -math.inf)
    p = torch.softmax(s, dim=-1).nan_to_num(0.0)
    ref = p @ v.double().repeat_interleave(Hq // Hkv, 1)
    rows = em.any(-1)
    err = (o.double() - ref)[rows].abs().max().item()
    assert err < 6e-2, err       # the parity suite's max-abs tolerance against exact attention
    assert torch.all(o[~rows] == 0) and torch.all(torch.isneginf(lse[~rows])) and not torch.isnan(o).any()


def test_broadcast_mask_equals_expanded():
    B, Hq, Hkv, Sq, Sk, D = 2, 2, 2, 130, 100, 64
    _, _, _, q8, qs, k8, ks, v8, vs = _operands(B, Hq, Hkv, Sq, Sk, D, "per_warp", seed=3)
    bm = _mask(1, 1, Sq, Sk, 0.6, 4)
    kw = dict(qk_quant_gran="per_warp", sm_scale=0.125, lazy_tau=4)
    assert torch.equal(attn_int8_fp8_blocksparse(q8, k8, v8, qs, ks, vs, bm, **kw),
                       attn_int8_fp8_blocksparse(q8, k8, v8, qs, ks, vs, bm.expand(B, Hq, -1, -1).clone(), **kw))


@pytest.mark.parametrize("tau", [4, 0])
@pytest.mark.parametrize("gran", ["per_thread", "per_warp"])
def test_tile_list_restatement_on_all_visible_tiles_is_the_dense_restatement_bitwise(gran, tau):
    """The tile-list restatement (attn_window_oracle.attn_int8_fp8_tiles) through its causal block-sparse caller with an all-True
    mask is the dense causal restatement, and with every tile listed and nothing masked the dense non-causal one."""
    B, Hq, Hkv, S, D = 2, 4, 2, 333, 64
    _, _, _, q8, qs, k8, ks, v8, vs = _operands(B, Hq, Hkv, S, S, D, gran, seed=5)
    kw = dict(qk_quant_gran=gran, sm_scale=D ** -0.5, lazy_tau=tau, return_lse=True)
    for causal in (False, True):
        ref = O.attn_int8_fp8_cuda(q8, k8, v8, qs, ks, vs, is_causal=causal, **kw)
        if causal:
            got = attn_int8_fp8_blocksparse_causal(q8, k8, v8, qs, ks, vs, torch.ones(1, 1, 3, 6, dtype=torch.bool), **kw)
        else:
            got = attn_int8_fp8_tiles(q8, k8, v8, qs, ks, vs, lambda b, h, i: range(6), torch.ones(1, 1, 1, 1, dtype=torch.bool), **kw)
        assert torch.equal(got[0], ref[0]) and torch.equal(got[1], ref[1]), causal


@pytest.mark.parametrize("gran", ["per_thread", "per_warp"])
def test_tile_list_restatement_is_the_gathered_restatement_bitwise(gran):
    """Non-causal, the tile-list loop over the visible tiles of each mask row with the expanded element mask gives the bits of the
    gathered restatement (attn_int8_fp8_blocksparse), per (batch, head) masks, hidden rows and a partial last tile included."""
    B, Hq, Hkv, Sq, Sk, D = 2, 4, 2, 300, 333, 64
    _, _, _, q8, qs, k8, ks, v8, vs = _operands(B, Hq, Hkv, Sq, Sk, D, gran, seed=6)
    bm = _mask(B, Hq, Sq, Sk, 0.5, 7)
    bm[0, 0, 1] = False
    bm[1, 3, :, -1] = True
    kw = dict(qk_quant_gran=gran, sm_scale=D ** -0.5, lazy_tau=4, return_lse=True, v_mean=torch.randn(B, Hkv, D))
    ref = attn_int8_fp8_blocksparse(q8, k8, v8, qs, ks, vs, bm, **kw)
    got = attn_int8_fp8_tiles(q8, k8, v8, qs, ks, vs, lambda b, h, i: [j for j in range(bm.size(3)) if bm[b, h, i, j]],
                              expand_block_mask(bm, Sq, Sk), **kw)
    assert torch.equal(got[0], ref[0]) and torch.equal(got[1], ref[1])


def test_bound_rejects_a_flipped_diagonal_tile():
    """Causal: the restatement on a mask with one tile of a diagonal 64-key pair flipped, either way, is outside the bound of the
    true mask's restatement."""
    B, Hq, Hkv, S, D = 1, 2, 1, 384, 64
    _, _, _, q8, qs, k8, ks, v8, vs = _operands(B, Hq, Hkv, S, S, D, "per_thread", seed=8)
    bm = _mask(B, Hq, S, S, 0.6, 9)
    bm[..., 0] = True
    kw = dict(qk_quant_gran="per_thread", sm_scale=D ** -0.5, lazy_tau=4)
    o, bd = attn_int8_fp8_blocksparse_causal(q8, k8, v8, qs, ks, vs, bm, bound=True, **kw)
    assert float(elementwise_ratio(o, bd.o, bd.o_bound).max()) <= 1.0
    for i, j in ((1, 2), (1, 3), (2, 5)):
        flip = bm.clone()
        flip[0, 1, i, j] = ~flip[0, 1, i, j]
        bad = attn_int8_fp8_blocksparse_causal(q8, k8, v8, qs, ks, vs, flip, **kw)
        assert float(elementwise_ratio(bad, bd.o, bd.o_bound).max()) > 1.0, (i, j)


def _call_fwd(lib, mask, strides=(0, 0, 1, 1), is_causal=0, q_gran=3, Sq=128, Skv=128):
    return lib.sab_qk_int8_sv_f8_attn_blocksparse(1, 1, 1, 1, None, 1, 1, None, None, 0, 1, 2, 2, Sq, Skv, 128, *([0] * 10),
                                                  is_causal, q_gran, 3, 1.0, 0, mask, *strides, None)


def _call_bwd(lib, mask, strides=(0, 0, 1, 1), is_causal=0, q_gran=3, Sq=128, Skv=128):
    return lib.sab_qk_int8_attn_bwd_blocksparse(*([16] * 15), 0, 1, 2, 2, Sq, Skv, 128, *([0] * 21), is_causal, q_gran, 3, 1.0, 0,
                                                mask, *strides, None)


@pytest.mark.parametrize("call", [_call_fwd, _call_bwd])
def test_c_entries_reject_bad_masks_without_a_gpu(call):
    from sageattention_b200 import _capi
    lib = _capi.lib()
    assert call(lib, None) == -1 and b"block_mask: null" in lib.sab_last_error()
    assert call(lib, 16, strides=(0, -1, 1, 1)) == -1 and b">= 0" in lib.sab_last_error()
    assert call(lib, 16, q_gran=1) == -2 and b"per-warp or per-thread" in lib.sab_last_error()
    assert call(lib, 16, is_causal=1, Skv=256) == -1 and b"must be equal for causal" in lib.sab_last_error()
    assert call(lib, 16, Skv=(1 << 20) + 64) == -2 and b"kv_len <= 1048576" in lib.sab_last_error()


def test_public_function_exists_and_rejects_cpu_tensors():
    import sageattention_b200 as sab
    assert "sageattn_blocksparse" in sab.__all__ and callable(sab.sageattn_blocksparse)
    q = torch.randn(1, 2, 128, 64, dtype=torch.float16)
    with pytest.raises(AssertionError):
        sab.sageattn_blocksparse(q, q, q, torch.ones(1, 1, 1, 2, dtype=torch.bool))
