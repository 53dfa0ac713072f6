"""fp64 reference of the backward kernels (sageattention_b200/csrc/attn_bwd.cu), with an elementwise error bound.  TEST
INFRASTRUCTURE ONLY: imported by the backward tests, never by the product package.  It expands the packed Q / K scales with the
oracle's own helpers (oracle/sage_oracle.py), so it reads the scales exactly as the forward's oracle does.  It runs on the device of
its inputs (the CPU for small cases, the GPU in fp64 for full-size ones).

The bound (attn_bwd(..., bound=True), then check_elementwise) is derived from the kernels' rounding model, with the same
constants for every case and family:
  * P is ex2.approx of an fp32 logit x = fmaf(float(s), coef, -lse), coef = k_scale * (q_scale * sm_scale*log2e) in fp32: a few
    fp32 roundings of |S| (the log2 logit) and of |x| <= |S| + |lse| and the relative error of ex2.approx.  Relative error of P:
      eps_P = EPS_EXP * (1 + |S| + |lse|),   EPS_EXP = 2^-21 (ex2.approx and the four fp32 roundings, with room to spare);
  * dP = dO V^T and delta = rowsum(dO o O) are fp32 sums of D products: absolute error of dP - delta at most
      a = D * U32 * (|dO| |V|^T + rowsum(|dO| o |O|)),   U32 = 2^-23 (one fp32 addition, truncated as tensor cores may);
  * the kernels round P and dS to the input dtype T (unit roundoff u = 2^-8 for bf16, 2^-11 for fp16; fp16 also has an absolute
    TINY = 2^-25 for values in its subnormal range) before the products that take them.  Per element:
      e_P  = |P| (u + eps_P) + TINY [P > 0],   e_dS = |dS| (u + eps_P) + P a + TINY [P > 0];
  * each gradient is an fp32 accumulation over the loop of its kernel (n = Skv keys for dQ, G * Sq rows of the GQA group for dK
    and dV), at most n * U32 times the sum of absolute terms.  So, before the store:
      dV: (e_P + n U32 |P|)^T |dO|,   dQ: (e_dS + n U32 |dS|) |K - mean| sm_scale,   dK: (e_dS + n U32 |dS|)^T |Q| sm_scale,
    whose main terms are u P^T|dO|, u |dS| |K - mean| sm_scale and u |dS|^T |Q| sm_scale;
  * the store multiplies by sm_scale in fp32 and rounds to T once: check_elementwise adds (u + 2^-22)(|ref| + bound) and, for
    fp16, TINY where the bound is not zero.
These bounds are linear in the Q rows, so a row-chunked evaluation (q_offset) sums the dK / dV bounds of its chunks, and the
store's rounding is applied once, by check_elementwise.  The masked oracle (attn_bwd_masked_oracle) carries dS in extra dQ
columns; their bound, times ln2 / sm_scale, is dBias's: e_dS + n U32 |dS| before dBias = ln2 dS is rounded to T."""
import math

import torch

from oracle import sage_oracle as O

U = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}
TINY = {torch.bfloat16: 0.0, torch.float16: 2.0 ** -25}
U32 = 2.0 ** -23
EPS_EXP = 2.0 ** -21


def attn_bwd(q8, k8, q_scale, k_scale, q, k, v, o, do, lse, *, q_gran="per_thread", k_gran=None, is_causal=False,
             sm_scale=1.0, fold_sm_scale=False, log2e=O.LOG2E_CU, k_mean=None, q_offset=0, q_len=None, head_dim=None,
             bound=False):
    """Gradients of the sm_90a backward kernels (csrc/attn_bwd.cu) in fp64: the gradient of attention evaluated at the forward's
    quantised logits (a straight-through estimator through the INT8 / FP8 roundings; no reference counterpart):
      S  = float(q8 k8^T) * q_scale * k_scale * sm_scale*log2e    (log2 units; fold_sm_scale: sm_scale*log2e is already in q_scale)
      P  = exp2(S - lse)  (0 where causal masks),   dV = P^T dO,   dP = dO V^T,   delta = rowsum(dO o O),   dS = P o (dP - delta)
      dQ = dS K * sm_scale,   dK = dS^T Q * sm_scale,   summed over the Q heads of each KV head (GQA).
    q8 / k8 int8 and q / k / v / o / do [B,H,S,D] (HND), the scales packed as the kernel reads them, lse [B,Hq,Sq] in log2 units
    (the forward kernel's own).  k_mean ([B,Hkv,1,D] or [B,Hkv,D], k's dtype): dQ is taken with the smoothed K, (k - k_mean) rounded
    to k's dtype, as the kernel does when it receives the mean.
    Row chunks: q8, q, o, do and lse may hold rows [q_offset, q_offset + n) of a call with q_len Q rows (default q_offset + n);
    q_scale stays the whole call's.  dQ is then that of the chunk's rows, dK / dV the chunk's share (sum them over the chunks).
    head_dim: the D of the dP and delta sums when the operands carry extra columns (default D).
    Returns (dq, dk, dv) in fp64, and with bound=True also the tuple of their elementwise bounds before the store (see the module
    docstring; q's dtype selects the unit roundoff)."""
    dev = q8.device
    B, Hq, Sq, D = q8.shape
    _, Hk, Sk, _ = k8.shape
    g = Hq // Hk
    n_q = q_len if q_len is not None else q_offset + Sq
    qs = O._expand_q_scale(q_scale.cpu(), q_gran, n_q)[:, :, q_offset:q_offset + Sq].to(dev).double()
    ks = O._expand_k_scale(k_scale.cpu(), k_gran or q_gran, Sk)[:, :, :Sk].to(dev).double().repeat_interleave(g, dim=1)
    sm2 = 1.0 if fold_sm_scale else float(sm_scale) * log2e
    S = (q8.double() @ k8.double().repeat_interleave(g, dim=1).transpose(-1, -2)) * (qs[..., None] * ks[:, :, None, :]) * sm2
    lse = lse.double()[..., None]
    P = torch.exp2(S - lse)
    if is_causal:
        rows = torch.arange(q_offset, q_offset + Sq, device=dev)
        P = P.masked_fill(torch.arange(Sk, device=dev)[None, :] > rows[:, None], 0.0)
    qf, dof, of = q.double(), do.double(), o.double()
    vf = v.double().repeat_interleave(g, dim=1)
    kc = k if k_mean is None else k - k_mean.reshape(B, Hk, 1, D)
    kf = kc.double().repeat_interleave(g, dim=1)
    dP = dof @ vf.transpose(-1, -2)
    dS = P * (dP - (dof * of).sum(dim=-1, keepdim=True))
    dq = dS @ kf * sm_scale
    dk = (dS.transpose(-1, -2) @ qf * sm_scale).reshape(B, Hk, g, Sk, D).sum(dim=2)
    dv = (P.transpose(-1, -2) @ dof).reshape(B, Hk, g, Sk, D).sum(dim=2)
    if not bound:
        return dq, dk, dv
    del dP
    u, tiny = U[q.dtype], TINY[q.dtype]
    visible = P > 0
    eps_p = torch.where(visible, EPS_EXP * (1.0 + S.abs() + lse.abs()), 0.0)
    del S
    ado = dof.abs()
    a = (head_dim or D) * U32 * (ado @ vf.abs().transpose(-1, -2) + (ado * of.abs()).sum(dim=-1, keepdim=True))
    tiny_p = tiny * visible if tiny else 0.0
    adS = dS.abs()
    e_ds = adS * (u + eps_p) + P * a + tiny_p
    del a
    bq = (e_ds + Sk * U32 * adS) @ kf.abs() * sm_scale
    n_kv = g * n_q
    bk = ((e_ds + n_kv * U32 * adS).transpose(-1, -2) @ qf.abs() * sm_scale).reshape(B, Hk, g, Sk, D).sum(dim=2)
    del e_ds, adS
    e_p = P * (u + eps_p + n_kv * U32) + tiny_p
    bv = (e_p.transpose(-1, -2) @ ado).reshape(B, Hk, g, Sk, D).sum(dim=2)
    return dq, dk, dv, (bq, bk, bv)


def elementwise_ratio(got, ref, bound):
    """Per element |got - ref| / tol with tol = bound + (u + 2^-22)(|ref| + bound) + TINY [bound > 0] for got's 16-bit dtype
    (the store's fp32 scaling and rounding, see the module docstring); 0 where got == ref, inf where got is not finite or the
    tolerance is 0 and got differs."""
    t = got.dtype
    got = got.to(ref.device).double()
    tol = bound + (U[t] + 2.0 ** -22) * (ref.abs() + bound) + TINY[t] * (bound > 0)
    err = (got - ref).abs()
    ratio = torch.where(err == 0, torch.zeros_like(err), err / tol)
    return torch.where(torch.isfinite(got), ratio, torch.full_like(err, math.inf))


def check_elementwise(name, got, ref, bound, dims=("b", "h", "row", "col")):
    """Assert |got - ref| <= tol elementwise (elementwise_ratio <= 1); on failure report the worst ratio and its index.  Returns
    (worst ratio, normwise relative error ||got - ref|| / ||ref||) for the caller to print."""
    ratio = elementwise_ratio(got, ref, bound)
    flat = int(ratio.argmax())
    worst = float(ratio.reshape(-1)[flat])
    idx = []
    for s in reversed(ratio.shape):
        idx.append(flat % s)
        flat //= s
    where = ", ".join(f"{n}={i}" for n, i in zip(dims, reversed(idx)))
    g = got.to(ref.device).double()
    bad = ~torch.isfinite(g)
    norm = float((g.nan_to_num() - ref).norm() / ref.norm()) if ref.norm() > 0 else float((g.nan_to_num() - ref).norm())
    assert worst <= 1.0, (f"{name}: |got - ref| / bound = {worst:.3g} at ({where}); {int(bad.sum())} non-finite elements; "
                          f"normwise {norm:.3e}")
    return worst, norm
