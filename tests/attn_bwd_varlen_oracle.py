"""fp64 CPU reference of the packed varlen backward (sab_qk_int8_attn_bwd_varlen, csrc/attn_bwd.cu).  TEST INFRASTRUCTURE ONLY:
imported by tests/test_backward_varlen_cpu.py and tests/test_gpu_backward_varlen.py, never by the product package.  Each sequence
is an independent dense call of attn_bwd_oracle.attn_bwd on the per-block, folded-scale path (the scales sageattn_varlen uses)."""
import torch

from attn_bwd_oracle import attn_bwd


def attn_bwd_varlen(q8, k8, q_scale, k_scale, q, k, v, o, do, lse, cu_seqlens_q, cu_seqlens_k, cu_q_scale, cu_k_scale, *,
                    is_causal=False, sm_scale=1.0, k_mean=None, bound=False):
    """q8 / q / o / do packed [Tq,Hq,D], k8 / k / v packed [Tk,Hkv,D]; q_scale [nblocks,Hq] and k_scale [nblocks,Hkv] with sequence b's
    128-row / 64-key blocks starting at cu_q_scale[b] / cu_k_scale[b]; lse [Hq,Tq] in log2 units (the forward kernel's);
    k_mean [Hkv,D] (any shape with Hkv*D elements, k's dtype) or None.  sm_scale*log2e is folded into q_scale, as sageattn_varlen
    quantises.  Returns (dq, dk, dv) in fp64, packed like q, k, v; tokens of no sequence, and sequences without queries or keys,
    get zeros.  bound=True: also the elementwise bounds of attn_bwd, packed the same way (zero where the gradient is zero)."""
    Hk, D = k.shape[1], k.shape[2]
    km = None if k_mean is None else k_mean.reshape(1, Hk, D)
    dq, dk, dv = (torch.zeros(t.shape, dtype=torch.float64) for t in (q, k, v))
    bq, bk, bv = (torch.zeros(t.shape, dtype=torch.float64) for t in (q, k, v))

    def hnd(t, s):
        return t[s].transpose(0, 1).unsqueeze(0)              # [1,H,L,D]

    for b in range(len(cu_seqlens_q) - 1):
        sq = slice(int(cu_seqlens_q[b]), int(cu_seqlens_q[b + 1]))
        sk = slice(int(cu_seqlens_k[b]), int(cu_seqlens_k[b + 1]))
        Lq, Lk = sq.stop - sq.start, sk.stop - sk.start
        if Lq == 0 or Lk == 0:
            continue
        qb, kb = int(cu_q_scale[b]), int(cu_k_scale[b])
        qs = q_scale[qb:qb + (Lq + 127) // 128].transpose(0, 1).unsqueeze(0)   # [1,Hq,nblocks]
        ks = k_scale[kb:kb + (Lk + 63) // 64].transpose(0, 1).unsqueeze(0)
        g = attn_bwd(hnd(q8, sq), hnd(k8, sk), qs, ks, hnd(q, sq), hnd(k, sk), hnd(v, sk), hnd(o, sq), hnd(do, sq),
                     lse[:, sq].unsqueeze(0), q_gran="per_block", k_gran="per_block", is_causal=is_causal, sm_scale=sm_scale,
                     fold_sm_scale=True, k_mean=km, bound=bound)
        dq[sq], dk[sk], dv[sk] = (x[0].transpose(0, 1) for x in g[:3])
        if bound:
            bq[sq], bk[sk], bv[sk] = (x[0].transpose(0, 1) for x in g[3])
    return (dq, dk, dv, (bq, bk, bv)) if bound else (dq, dk, dv)
