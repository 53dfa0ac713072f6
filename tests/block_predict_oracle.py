"""fp64 CPU restatement of predict_block_mask (include/sageattn_b200.h, sab_block_stats / sab_predict_block_mask).

block_stats(x, blk)             -> per-block mean [B,H,nb,D] and self-similarity [B,H,nb]
select(q_mean, q_sim, ...)      -> the bool [B,Hq,nq,nk] mask from given statistics (e.g. the kernel's own), and the rows with a
                                   decision within `eps` of a threshold
predict_block_mask(q, k, ...)   -> both steps from the inputs
"""
import torch


def block_stats(x, blk):
    """x: [B,H,S,D] (any float dtype).  Returns (mean, sim) in fp64."""
    B, H, S, D = x.shape
    nb = (S + blk - 1) // blk
    x = x.double()
    norm = x.norm(dim=-1, keepdim=True)
    u = torch.where(norm > 0, x / torch.where(norm > 0, norm, torch.ones_like(norm)), torch.zeros_like(x))
    pad = nb * blk - S
    xs = torch.nn.functional.pad(x, (0, 0, 0, pad)).view(B, H, nb, blk, D)
    us = torch.nn.functional.pad(u, (0, 0, 0, pad)).view(B, H, nb, blk, D)
    n = torch.full((nb,), float(blk), dtype=torch.float64)
    n[-1] = S - blk * (nb - 1)
    mean = xs.sum(3) / n[:, None]
    sim = us.sum(3).pow(2).sum(-1) / n ** 2
    return mean, sim


def scores(q_mean, k_mean, sm_scale):
    """sm_scale * (m_q . m_k) for every (row, key block): [B,Hq,nq,nk] fp64, the K head broadcast over its Q heads."""
    g = q_mean.size(1) // k_mean.size(1)
    return sm_scale * q_mean.double() @ k_mean.double().repeat_interleave(g, 1).transpose(-1, -2)


def select(q_mean, q_sim, k_mean, k_sim, Sq, Skv, *, cdf_threshold, sim_threshold, is_causal=False, sm_scale, eps=0.0, rows=None):
    """The mask from block statistics.  Returns (mask, near): near[b,h,i] is True where a decision of row i lies within eps of a
    threshold (a prefix mass within eps of cdf_threshold, a self-similarity within eps of sim_threshold, or two distinct p within
    a relative eps at the cut), where fp32 statistics may legitimately decide the other way.  rows: optional 1-D tensor of the Q-block
    indices to evaluate (the result then has len(rows) rows)."""
    B, Hq, nq, _ = q_mean.shape
    nk = k_mean.size(2)
    g = Hq // k_mean.size(1)
    rows = torch.arange(nq) if rows is None else torch.as_tensor(rows)
    q_mean, q_sim = q_mean[:, :, rows], q_sim[:, :, rows]
    s = scores(q_mean, k_mean, sm_scale)
    qs, ks = q_sim.double(), k_sim.double().repeat_interleave(g, 1)[:, :, None, :]
    i = rows[:, None]
    j = torch.arange(nk)[None, :]
    horizon = (64 * j <= 128 * i + 127) if is_causal else torch.ones(len(rows), nk, dtype=torch.bool)
    diag = ((128 * i <= 64 * j + 63) & horizon) if is_causal else torch.zeros(len(rows), nk, dtype=torch.bool)
    cand = (ks >= sim_threshold) & horizon
    p = torch.softmax(s.masked_fill(~cand, float("-inf")), -1).nan_to_num(0.0)
    # descending p; a stable sort keeps equal p in ascending j
    ps, order = torch.sort(p, dim=-1, descending=True, stable=True)
    cs = torch.gather(cand, -1, order)
    before = torch.cumsum(ps, -1) - ps
    keep_sorted = cs & ((before < cdf_threshold) | (cdf_threshold >= 1))
    kept = torch.zeros_like(cand).scatter(-1, order, keep_sorted)
    near = ((ks - sim_threshold).abs() < eps).expand_as(cand).logical_and(horizon).any(-1)
    near |= (qs - sim_threshold).abs() < eps
    if cdf_threshold < 1:
        near |= (cs & ((before - cdf_threshold).abs() < eps)).any(-1)
        cut = keep_sorted[..., :-1] & ~keep_sorted[..., 1:] & cs[..., 1:]
        gap = (ps[..., :-1] - ps[..., 1:]).abs()
        near |= (cut & (gap > 0) & (gap < eps * ps[..., :-1])).any(-1)
    mask = kept | (ks < sim_threshold) | diag | (qs < sim_threshold)[..., None]
    return mask & horizon, near


def predict_block_mask(q, k, *, cdf_threshold, sim_threshold, tensor_layout="HND", is_causal=False, sm_scale=None, eps=0.0):
    """From the inputs (q [B,Hq,Sq,D], k [B,Hkv,Skv,D] for "HND").  Returns (mask, near) as select()."""
    if tensor_layout == "NHD":
        q, k = q.transpose(1, 2), k.transpose(1, 2)
    Sq, Skv = q.size(2), k.size(2)
    if sm_scale is None:
        sm_scale = q.size(-1) ** -0.5
    qm, qs = block_stats(q, 128)
    km, ks = block_stats(k, 64)
    return select(qm, qs, km, ks, Sq, Skv, cdf_threshold=cdf_threshold, sim_threshold=sim_threshold, is_causal=is_causal,
                  sm_scale=sm_scale, eps=eps)
