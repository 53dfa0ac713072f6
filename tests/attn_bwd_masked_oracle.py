"""fp64 CPU reference of the masked backward (sab_qk_int8_attn_bwd_masked, csrc/attn_bwd.cu).  TEST INFRASTRUCTURE ONLY: imported by
tests/test_backward_masked_cpu.py and tests/test_gpu_backward_masked.py, never by the product package.

The masked P has one definition here, and the gradient formulas stay those of attn_bwd_oracle.attn_bwd: a mask is an additive
log2-unit term M on the logits, S + M, and attn_bwd is evaluated on operands extended by Sk columns that add exactly that term.
  * q8 gains the columns M[i, j] / (q_scale_i * sm_scale*log2e) and k8 the diagonal 1 / k_scale_j, so that attn_bwd's
    S = float(q8 k8^T) * q_scale * k_scale * sm_scale*log2e becomes S + M;
  * k gains the identity (k_mean, when given, zeros), so that dQ = dS K * sm_scale carries dS itself in its extra columns;
  * q, v, o, dout gain zero columns, which change neither dP, delta, dK nor dV.
The extra columns are sliced off the results."""
import math

import torch

from attn_bwd_oracle import attn_bwd
from oracle import sage_oracle as O

# log2-unit stand-in for a masked element: exp2(S - lse + MASKED) is exactly 0 in fp64 for any logits these tests produce
MASKED = -1.0e4


def attn_bwd_masked(q8, k8, q_scale, k_scale, q, k, v, o, do, lse, attn_mask, *, q_gran="per_block", k_gran="per_block",
                    sm_scale=1.0, fold_sm_scale=False, log2e=O.LOG2E_CU, k_mean=None, bound=False):
    """attn_bwd (non-causal) with the forward's masked logits.  attn_mask, broadcastable to [B,Hq,Sq,Sk]: bool (False = masked out:
    P = 0) or an additive bias in log2 units, added to the scaled logits as the forward adds it (-inf: P = 0).  A row with
    lse = -inf has no visible key (the forward returned zeros): its P is 0.  Other arguments as attn_bwd.  Returns
    (dq, dk, dv, dbias) in fp64, dbias = ln2 * dS as [B,Hq,Sq,Sk]; with bound=True also attn_bwd's elementwise bounds of the four,
    dBias's being ln2 / sm_scale times that of dS's extra dQ columns (e_dS plus the accumulation term, which only widens it)."""
    B, Hq, Sq, D = q8.shape
    _, Hk, Sk, _ = k8.shape
    if attn_mask.dtype == torch.bool:
        M = torch.where(attn_mask, 0.0, MASKED).double()
    else:
        M = attn_mask.double().masked_fill(attn_mask == float("-inf"), MASKED)
    M = M.expand(B, Hq, Sq, Sk)
    qs = O._expand_q_scale(q_scale, q_gran, Sq)[:, :, :Sq].double()
    ks = O._expand_k_scale(k_scale, k_gran or q_gran, Sk)[:, :, :Sk].double()
    sm2 = 1.0 if fold_sm_scale else float(sm_scale) * log2e
    q8x = torch.cat([q8.double(), M / (qs[..., None] * sm2)], dim=-1)
    k8x = torch.cat([k8.double(), torch.diag_embed(1.0 / ks)], dim=-1)
    eye = torch.eye(Sk, dtype=k.dtype).expand(B, Hk, Sk, Sk)
    kx = torch.cat([k, eye], dim=-1)
    kmx = None if k_mean is None else torch.cat([k_mean.reshape(B, Hk, 1, D), torch.zeros(B, Hk, 1, Sk, dtype=k_mean.dtype)], dim=-1)

    def zpad(t):
        return torch.cat([t, torch.zeros(t.shape[:-1] + (Sk,), dtype=t.dtype)], dim=-1)

    # no visible key: lse = +inf makes P = exp2(S - lse) exactly 0 (the kernel's -lse = -inf)
    lsex = lse.double().masked_fill(lse == float("-inf"), float("inf"))
    res = attn_bwd(q8x, k8x, q_scale, k_scale, zpad(q), kx, zpad(v), zpad(o), zpad(do), lsex, q_gran=q_gran, k_gran=k_gran,
                   sm_scale=sm_scale, fold_sm_scale=fold_sm_scale, log2e=log2e, k_mean=kmx, head_dim=D, bound=bound)
    dq, dk, dv = res[:3]
    out = (dq[..., :D], dk[..., :D], dv[..., :D], math.log(2.0) / sm_scale * dq[..., D:])
    if not bound:
        return out
    bq, bk, bv = res[3]
    return out + ((bq[..., :D], bk[..., :D], bv[..., :D], math.log(2.0) / sm_scale * bq[..., D:]),)
