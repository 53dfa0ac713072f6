"""CPU restatement of the block-sparse forward (sab_qk_int8_sv_f8_attn_blocksparse, csrc/attn.cu).  TEST INFRASTRUCTURE ONLY:
imported by tests/test_blocksparse_cpu.py and tests/test_gpu_blocksparse.py, never by the product package.

Non-causal, the kernel's CTA for 128-row Q block i runs the dense loop over the visible 64-key tiles of mask row i, in ascending
order.  That is the dense restatement (oracle.sage_oracle.attn_int8_fp8_cuda) on Q block i with those tiles of k8, k_scale and
v8 gathered in order: the per-tile arithmetic only depends on the tile's keys and scales, and a partial last tile stays last.
A row with no visible key gives 0 and lse -inf."""
import torch

from oracle import sage_oracle as O


def expand_block_mask(block_mask, Sq, Sk):
    """[.,.,ceil(Sq/128),ceil(Sk/64)] bool -> the element mask [.,.,Sq,Sk]."""
    return block_mask.repeat_interleave(128, dim=2)[:, :, :Sq].repeat_interleave(64, dim=3)[:, :, :, :Sk]


def _q_scale_block(q_scale, gran, i):
    mult = {"per_warp": 4, "per_thread": 32}[gran]
    return q_scale[:, :, i * mult:(i + 1) * mult]


def _k_scale_blocks(k_scale, gran, idx):
    mult = 4 if gran == "per_thread" else 1
    cols = torch.cat([torch.arange(j * mult, (j + 1) * mult) for j in idx])
    return k_scale[:, :, cols]


def attn_int8_fp8_blocksparse(q8, k8, v8, q_scale, k_scale, v_scale, block_mask, *, qk_quant_gran="per_thread",
                              out_dtype=torch.float16, return_lse=False, v_mean=None, **kw):
    """attn_int8_fp8_cuda (non-causal) restricted to the visible tiles of block_mask ([B or 1, Hq or 1, ceil(Sq/128),
    ceil(Sk/64)] bool, indexed by the Q head).  v8 is the LOGICAL [B,Hkv,Sk,D] fp8 tensor; kw go to attn_int8_fp8_cuda."""
    assert not kw.get("is_causal", False), "the gathered restatement is non-causal"
    B, Hq, Sq, D = q8.shape
    _, Hk, Sk, _ = k8.shape
    g = Hq // Hk
    bm = block_mask.expand(B, Hq, (Sq + 127) // 128, (Sk + 63) // 64)
    out = torch.zeros((B, Hq, Sq, D), dtype=out_dtype)
    lse = torch.full((B, Hq, Sq), -float("inf"), dtype=torch.float32)
    for b in range(B):
        for h in range(Hq):
            hk = h // g
            for i in range(bm.size(2)):
                r0, r1 = 128 * i, min(128 * i + 128, Sq)
                idx = [j for j in range(bm.size(3)) if bool(bm[b, h, i, j])]
                if not idx:
                    continue
                keys = torch.cat([torch.arange(64 * j, min(64 * j + 64, Sk)) for j in idx])
                res = O.attn_int8_fp8_cuda(
                    q8[b:b + 1, h:h + 1, r0:r1], k8[b:b + 1, hk:hk + 1, keys], v8[b:b + 1, hk:hk + 1, keys],
                    _q_scale_block(q_scale[b:b + 1, h:h + 1], qk_quant_gran, i),
                    _k_scale_blocks(k_scale[b:b + 1, hk:hk + 1], qk_quant_gran, idx), v_scale[b:b + 1, hk:hk + 1],
                    qk_quant_gran=qk_quant_gran, out_dtype=out_dtype, return_lse=True,
                    v_mean=None if v_mean is None else v_mean[b:b + 1, hk:hk + 1], **kw)
                out[b, h, r0:r1] = res[0][0, 0]
                lse[b, h, r0:r1] = res[1][0, 0]
    return (out, lse) if return_lse else out
