"""fp64 CPU reference of the backward kernels (sageattention_b200/csrc/attn_bwd.cu).  TEST INFRASTRUCTURE ONLY: imported by
tests/test_backward_cpu.py and tests/test_gpu_backward.py, never by the product package.  It expands the packed Q / K scales with
the oracle's own helpers (oracle/sage_oracle.py), so it reads the scales exactly as the forward's oracle does."""
import torch

from oracle import sage_oracle as O


def attn_bwd(q8, k8, q_scale, k_scale, q, k, v, o, do, lse, *, q_gran="per_thread", k_gran=None, is_causal=False,
             sm_scale=1.0, fold_sm_scale=False, log2e=O.LOG2E_CU, k_mean=None):
    """Gradients of the sm_90a backward kernels (csrc/attn_bwd.cu) in fp64: the gradient of attention evaluated at the forward's
    quantised logits (a straight-through estimator through the INT8 / FP8 roundings; no reference counterpart):
      S  = float(q8 k8^T) * q_scale * k_scale * sm_scale*log2e    (log2 units; fold_sm_scale: sm_scale*log2e is already in q_scale)
      P  = exp2(S - lse)  (0 where causal masks),   dV = P^T dO,   dP = dO V^T,   delta = rowsum(dO o O),   dS = P o (dP - delta)
      dQ = dS K * sm_scale,   dK = dS^T Q * sm_scale,   summed over the Q heads of each KV head (GQA).
    q8 / k8 int8 and q / k / v / o / do [B,H,S,D] (HND), the scales packed as the kernel reads them, lse [B,Hq,Sq] in log2 units
    (the forward kernel's own).  k_mean ([B,Hkv,1,D] or [B,Hkv,D], k's dtype): dQ is taken with the smoothed K, (k - k_mean) rounded
    to k's dtype, as the kernel does when it receives the mean.  Returns (dq, dk, dv) in fp64."""
    B, Hq, Sq, D = q8.shape
    _, Hk, Sk, _ = k8.shape
    g = Hq // Hk
    qs = O._expand_q_scale(q_scale, q_gran, Sq)[:, :, :Sq].double()
    ks = O._expand_k_scale(k_scale, k_gran or q_gran, Sk)[:, :, :Sk].double().repeat_interleave(g, dim=1)
    sm2 = 1.0 if fold_sm_scale else float(sm_scale) * log2e
    S = (q8.double() @ k8.double().repeat_interleave(g, dim=1).transpose(-1, -2)) * (qs[..., None] * ks[:, :, None, :]) * sm2
    P = torch.exp2(S - lse.double()[..., None])
    if is_causal:
        P = P.masked_fill(torch.arange(Sk)[None, :] > torch.arange(Sq)[:, None], 0.0)
    qf, dof, of = q.double(), do.double(), o.double()
    kf, vf = k.double().repeat_interleave(g, dim=1), v.double().repeat_interleave(g, dim=1)
    dP = dof @ vf.transpose(-1, -2)
    dS = P * (dP - (dof * of).sum(dim=-1, keepdim=True))
    if k_mean is not None:
        kf = (k - k_mean.reshape(B, Hk, 1, D)).double().repeat_interleave(g, dim=1)
    dq = dS @ kf * sm_scale
    dk = (dS.transpose(-1, -2) @ qf * sm_scale).view(B, Hk, g, Sk, D).sum(dim=2)
    dv = (P.transpose(-1, -2) @ dof).view(B, Hk, g, Sk, D).sum(dim=2)
    return dq, dk, dv
