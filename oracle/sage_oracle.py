"""CPU oracle for the SageAttention INT8-QK / FP8-PV hot path.  TEST INFRASTRUCTURE ONLY.

Nothing in the product package (``sageattention_b200``) may import this module: only ``tests/``,
``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` / ``--impl reference`` legs do.

It is a plain torch-on-CPU restatement (fp32/int arithmetic, no GPU) of the reference algorithm.
Every function cites the reference file:line (relative to /root/reference) that it follows.

Pinning status
--------------
* The reference ships NO tests / golden vectors, so parity is pinned against outputs
  of the reference code itself:
  - Triton-semantics functions (``quant_per_block_int8_triton``, ``quant_per_thread_int8_triton``,
    ``quant_per_block_int8_varlen_triton``, ``attn_int8_fp16_triton``) are checked bit-exact /
    to 2e-3 against the reference Triton kernels executed in this container under
    TRITON_INTERPRET=1; fixtures and generator: tests/golden/make_golden.py, tests/golden/*.npz.
  - CUDA-semantics functions (``quant_int8_cuda``, ``per_channel_fp8_cuda``, ``attn_int8_fp8_cuda``)
    are checked on the GPU box against the real reference kernels built for sm_90a into
    oracle/_ref/ (oracle/build_ref.py) by tests/test_gpu_parity.py.
"""
from __future__ import annotations

import math
from typing import Optional, Tuple

import torch

LOG2E_PY = 1.44269504                      # sageattention/core.py:304, quant_per_block.py:87
LOG2E_CU = 1.44269504088896340736          # csrc/math.cuh:32
S_FP8_OFFSET = 8.807                       # csrc/qattn/attn_utils.cuh:30  (log2(448))
MASK_VALUE = -5000000.0                    # csrc/qattn/attn_utils.cuh:310,344


# --------------------------------------------------------------------------------------------
# helpers
# --------------------------------------------------------------------------------------------
def _to_hnd(x: torch.Tensor, tensor_layout: str) -> torch.Tensor:
    """Return a [B,H,S,D] view (reference kernels take strides; layout only changes strides)."""
    if tensor_layout == "HND":
        return x
    if tensor_layout == "NHD":
        return x.transpose(1, 2)
    raise ValueError(f"Unknown tensor layout: {tensor_layout}")


def _pad_seq(x: torch.Tensor, blk: int) -> torch.Tensor:
    s = x.shape[2]
    pad = (-s) % blk
    if pad:
        x = torch.nn.functional.pad(x, (0, 0, 0, pad))
    return x


def _round_half_away_to_int8(y: torch.Tensor) -> torch.Tensor:
    """x_int8 += 0.5*where(x>=0,1,-1); .to(int8) truncates toward zero
    (sageattention/triton/quant_per_block.py:43-45)."""
    y = y + 0.5 * torch.where(y >= 0, 1.0, -1.0).to(y.dtype)
    return torch.trunc(y).to(torch.int8)


# --------------------------------------------------------------------------------------------
# INT8 quantisation of Q / K
# --------------------------------------------------------------------------------------------
def quant_per_block_int8_triton(x: torch.Tensor, BLK: int, sm_scale: float = 1.0,
                                tensor_layout: str = "HND") -> Tuple[torch.Tensor, torch.Tensor]:
    """sageattention/triton/quant_per_block.py:21-47.  scale = amax/127 (no epsilon),
    round-half-away, out-of-range rows read as 0.  Returns (int8 same layout as x, scale [B,H,nblk])."""
    xh = _to_hnd(x, tensor_layout)
    B, H, S, D = xh.shape
    xf = _pad_seq(xh.float(), BLK) * torch.tensor(sm_scale, dtype=torch.float32)
    nblk = xf.shape[2] // BLK
    xb = xf.reshape(B, H, nblk, BLK * D)
    scale = xb.abs().amax(dim=-1) / 127.0
    q = _round_half_away_to_int8(xb / scale[..., None]).view(B, H, nblk * BLK, D)[:, :, :S]
    if tensor_layout == "NHD":
        q = q.transpose(1, 2)
    return q.contiguous(), scale.contiguous()


def per_block_int8_triton(q, k, km=None, BLKQ=128, BLKK=64, sm_scale=None, tensor_layout="HND"):
    """sageattention/triton/quant_per_block.py:49-101 (host glue)."""
    if km is not None:
        k = k - km                                             # in input dtype, :53-54
    D = q.shape[-1]
    if sm_scale is None:
        sm_scale = D ** -0.5
    q8, qs = quant_per_block_int8_triton(q, BLKQ, sm_scale * LOG2E_PY, tensor_layout)
    k8, ks = quant_per_block_int8_triton(k, BLKK, 1.0, tensor_layout)
    return q8, qs, k8, ks


def quant_per_thread_int8_triton(q, k, km=None, BLKQ=128, WARPQ=32, BLKK=64, WARPK=64,
                                 tensor_layout="HND"):
    """sageattention/triton/quant_per_thread.py:21-98,154-203.
    Q: inside each WARPQ(32)-row block, group g = rows {g, g+8, g+16, g+24} (:32);
    K: inside each WARPK(64)-key block, group t = keys {8j+2t, 8j+2t+1} (:75-76);
    scale = amax/127 + 1e-7, round-half-away, `k - km` done first in input dtype (:158-159)."""
    if km is not None:
        k = k - km
    qh, kh = _to_hnd(q, tensor_layout), _to_hnd(k, tensor_layout)
    B, Hq, Sq, D = qh.shape
    _, Hk, Sk, _ = kh.shape
    # ---- Q
    qf = _pad_seq(qh.float(), BLKQ)
    nwq = qf.shape[2] // WARPQ
    qg = qf.reshape(B, Hq, nwq, WARPQ // 8, 8, D)                  # row = w*32 + i*8 + g
    q_scale = qg.abs().amax(dim=(3, 5)) / 127.0 + 0.0000001     # [B,H,nwq,8]
    q8 = _round_half_away_to_int8(qg / q_scale[:, :, :, None, :, None]).view(B, Hq, -1, D)[:, :, :Sq]
    q_scale = q_scale.reshape(B, Hq, nwq * 8)
    # ---- K
    kf = _pad_seq(kh.float(), BLKK)
    nwk = kf.shape[2] // WARPK
    kg = kf.reshape(B, Hk, nwk, WARPK // 8, 4, 2, D)               # key = w*64 + j*8 + t*2 + e
    k_scale = kg.abs().amax(dim=(3, 5, 6)) / 127.0 + 0.0000001  # [B,H,nwk,4]
    k8 = _round_half_away_to_int8(kg / k_scale[:, :, :, None, :, None, None]).view(B, Hk, -1, D)[:, :, :Sk]
    k_scale = k_scale.reshape(B, Hk, nwk * 4)
    if tensor_layout == "NHD":
        q8, k8 = q8.transpose(1, 2), k8.transpose(1, 2)
    return q8.contiguous(), q_scale.contiguous(), k8.contiguous(), k_scale.contiguous()


def quant_int8_cuda(x: torch.Tensor, BLK: int, mean: Optional[torch.Tensor] = None,
                    sm_scale: Optional[float] = None, tensor_layout: str = "HND"):
    """csrc/fused/fused.cu:64-198 (QuantInt8Kernel).  x_f = float(x) [- float(mean)] [* sm_scale];
    amax floored at 1e-7; scale = amax/127; q = cvt.rni.sat.s8(x_f * (127/amax))
    (round-half-even, csrc/numeric_conversion.cuh:144-148).  `mean` is [B,H,D] in x.dtype.
    NOTE: the reference is compiled with --use_fast_math (setup.py:56) so its two divisions are
    approximate; this restatement uses IEEE division, the GPU test against oracle/_ref is the pin."""
    xh = _to_hnd(x, tensor_layout)
    B, H, S, D = xh.shape
    xf = xh.float()
    if mean is not None:
        xf = xf - mean.float().view(B, H, 1, D)
    if sm_scale is not None:
        xf = xf * torch.tensor(sm_scale, dtype=torch.float32)
    xf = _pad_seq(xf, BLK)
    nblk = xf.shape[2] // BLK
    xb = xf.reshape(B, H, nblk, BLK * D)
    amax = xb.abs().amax(dim=-1).clamp_min(0.0000001)
    scale = amax / 127.0
    tmp = 127.0 / amax
    q = torch.round(xb * tmp[..., None]).clamp(-128, 127).to(torch.int8)   # torch.round = half-even
    q = q.view(B, H, nblk * BLK, D)[:, :, :S]
    if tensor_layout == "NHD":
        q = q.transpose(1, 2)
    return q.contiguous(), scale.contiguous()


def per_warp_int8_cuda(q, k, km=None, BLKQ=128, WARPQ=32, BLKK=64, tensor_layout="HND"):
    """sageattention/quant.py:105-180: Q per WARPQ-row block, K per BLKK block with fused (k - km);
    q_scale is laid out [B,H,ceil(Sq/BLKQ)*(BLKQ/WARPQ)] (rows beyond Sq contribute zeros)."""
    qh = _to_hnd(q, tensor_layout)
    B, Hq, Sq, D = qh.shape
    q8, qs = quant_int8_cuda(q, WARPQ, None, None, tensor_layout)
    n_expected = (Sq + BLKQ - 1) // BLKQ * (BLKQ // WARPQ)
    if qs.shape[-1] < n_expected:   # fully out-of-range warp blocks: amax floor 1e-7 -> scale 1e-7/127
        fill = torch.full((B, Hq, n_expected - qs.shape[-1]), 0.0000001 / 127.0, dtype=torch.float32)
        qs = torch.cat([qs, fill], dim=-1)
    kmean = None
    if km is not None:
        kmean = km.squeeze(1) if tensor_layout == "NHD" else km.squeeze(2)
    k8, ks = quant_int8_cuda(k, BLKK, kmean, None, tensor_layout)
    return q8, qs, k8, ks


# --------------------------------------------------------------------------------------------
# FP8 quantisation of V
# --------------------------------------------------------------------------------------------
def per_channel_fp8_cuda(v: torch.Tensor, tensor_layout: str = "HND", scale_max: float = 448.0,
                         smooth_v: bool = False):
    """sageattention/quant.py:224-293 + csrc/fused/fused.cu:316-427 (MeanScaleKernel).
    Per (b,h,d) channel: scale = amax/scale_max, v8 = cvt.rn.satfinite.e4m3(v * (scale_max/amax)).
    Returns the quantised values in LOGICAL order [B,H,S,D] (fp8 e4m3fn) — the reference's
    transposed/padded/16-token-permuted storage (fused.cu:262-313) is an mma.sync layout artefact
    and not part of the numerical contract — plus v_scale [B,H,D] and (optional) mean."""
    vh = _to_hnd(v, tensor_layout).float()
    B, H, S, D = vh.shape
    vm = None
    if smooth_v:
        pad16 = (S + 15) // 16 * 16                               # fused.cu:349,381
        vm = vh.sum(dim=2) / pad16
        vh = vh - vm[:, :, None, :]
    amax = vh.abs().amax(dim=2)
    scale = amax / scale_max
    recp = scale_max / amax
    v8 = (vh * recp[:, :, None, :]).to(torch.float8_e4m3fn)
    return v8, scale.contiguous(), vm


# --------------------------------------------------------------------------------------------
# attention: CUDA fp8 path
# --------------------------------------------------------------------------------------------
def _expand_q_scale(q_scale, gran, Sq, BLKQ=128, WARPQ=32):
    """Per-row dequant scale [B,H,Sq_pad] from the packed layouts
    (csrc/qattn/qk_int_sv_f8_cuda_sm89.cuh:98-114)."""
    B, H, n = q_scale.shape
    Sp = (Sq + BLKQ - 1) // BLKQ * BLKQ
    rows = torch.arange(Sp)
    if gran == "per_block":
        idx = rows // BLKQ
    elif gran == "per_warp":
        idx = rows // WARPQ
    elif gran == "per_thread":
        idx = (rows // WARPQ) * 8 + rows % 8
    else:
        raise ValueError(gran)
    return q_scale[:, :, idx]


def _expand_k_scale(k_scale, gran, Sk, BLKK=64):
    """Per-key dequant scale [B,H,Sk_pad] (…sm89.cuh:116-132)."""
    Sp = (Sk + BLKK - 1) // BLKK * BLKK
    keys = torch.arange(Sp)
    if gran in ("per_block", "per_warp"):
        idx = keys // BLKK
    elif gran == "per_thread":
        idx = (keys // BLKK) * 4 + (keys % 8) // 2
    else:
        raise ValueError(gran)
    return k_scale[:, :, idx]


def attn_int8_fp8_cuda(q8, k8, v8, q_scale, k_scale, v_scale, *, qk_quant_gran="per_thread",
                       k_quant_gran=None, is_causal=False, sm_scale=1.0, pv_accum_dtype="fp32+fp32",
                       out_dtype=torch.float16, kv_tile=64, return_lse=False, log2e=LOG2E_CU, exp2_fn=None, lazy_tau=None,
                       v_mean=None, causal_q_offset=0):
    """csrc/qattn/qk_int_sv_f8_cuda_sm89.cuh:44-704 restated on [B,H,S,D] tensors.

    q8/k8 int8 [B,Hq|Hkv,S,D]; v8 fp8-e4m3 LOGICAL [B,Hkv,Skv,D]; scales packed as the reference.
    Per kv tile of `kv_tile` keys (reference CTA_K = 64):
      S_f   = float(S_i32) * (sm_scale*log2e*q_scale*k_scale)                 (:255-257, 287-301)
      masks = -5e6 for causal kv>q and kv>=kv_len                             (attn_utils.cuh:296-351)
      m_new = max(m_old, rowmax(S_f) - 8.807);  alpha = exp2(m_old-m_new)    (attn_utils.cuh:354-400)
      P     = exp2(S_f - m_new) in (0,448];  d = d*alpha + sum(P) (fp32)     (:440-458, 529-556)
      P8    = e4m3_rn_satfinite(P)                                           (:478-493)
      O     = O*alpha + P8 @ V8   (fp32, or f16 per-tile accumulate)         (:896-974)
    epilogue: O/d * v_scale -> out_dtype;  lse = log2(d) + m                  (…sm89.cuh:572-703)
    Causal uses top-left alignment (kv_idx > q_idx masked).
    `exp2_fn` (default torch.exp2) replaces the exponential of P only — used by tests/test_poly_exp_numerics.py to
    quantify the opt-in FMA-pipe polynomial of the sm_90a kernel (csrc/ptx.cuh ex2_poly2) against this restatement.
    `lazy_tau` (default None = the reference rule) restates the lazy running max of the sm_90a kernel: the
    running max only moves when it grew by more than tau (log2 units) and the exponent offset is 8.807 - tau.
    `v_mean` ([B,Hkv,D] fp32, the smooth_v channel mean) is added after `* v_scale`, as the reference's fuse-v-mean epilogue
    (…sm89.cuh:572-703) and the sm_90a kernel do.
    `causal_q_offset` is the global index of q8's first row (the kernel parameter of the same name): the causal mask and the
    causal early exit use global rows, q_scale stays indexed by local row.  So one 128-row-aligned block of Q
    (q8[:, :, r0:r0+128] with q_scale sliced to that block) evaluates to exactly those rows of the full evaluation."""
    B, Hq, Sq, D = q8.shape
    _, Hk, Sk, _ = k8.shape
    g = Hq // Hk
    kgran = k_quant_gran or qk_quant_gran
    qs_row = _expand_q_scale(q_scale, qk_quant_gran, Sq)[:, :, :Sq]               # [B,Hq,Sq]
    ks_key = _expand_k_scale(k_scale, kgran, Sk)[:, :, :Sk]                       # [B,Hk,Sk]
    ks_key = ks_key.repeat_interleave(g, dim=1)
    kf = k8.float().repeat_interleave(g, dim=1)
    vf = v8.float().repeat_interleave(g, dim=1)
    vsc = v_scale.repeat_interleave(g, dim=1)                                     # [B,Hq,D]
    qf = q8.float()
    sm2 = torch.tensor(sm_scale, dtype=torch.float32) * torch.tensor(log2e, dtype=torch.float32)

    m = torch.full((B, Hq, Sq), MASK_VALUE, dtype=torch.float32)
    d = torch.ones((B, Hq, Sq), dtype=torch.float32)
    O = torch.zeros((B, Hq, Sq, D), dtype=torch.float32)
    qi = torch.arange(Sq)[:, None] + causal_q_offset
    for s0 in range(0, Sk, kv_tile):
        s1 = min(s0 + kv_tile, Sk)
        if is_causal and s0 > causal_q_offset + Sq - 1:
            break
        S_i = qf @ kf[:, :, s0:s1].transpose(-1, -2)                               # exact in fp32
        coef = (sm2 * qs_row)[..., None] * ks_key[:, :, None, s0:s1]               # sm_scale*dequant
        S = S_i * coef
        if is_causal:
            kj = torch.arange(s0, s1)[None, :]
            S = torch.where(kj > qi, torch.tensor(MASK_VALUE), S)
        if lazy_tau is None:
            m_new = torch.maximum(m, S.amax(dim=-1) - S_FP8_OFFSET)
        else:
            m_true = torch.maximum(m, S.amax(dim=-1) - (S_FP8_OFFSET - float(lazy_tau)))
            m_new = torch.where(m_true - m > float(lazy_tau), m_true, m)
        alpha = torch.exp2(m - m_new)
        P = (exp2_fn or torch.exp2)(S - m_new[..., None])
        d = d * alpha + P.sum(dim=-1)
        P8 = P.to(torch.float8_e4m3fn).float()
        Vt = vf[:, :, s0:s1]
        if pv_accum_dtype == "fp32+fp16":
            # f16 accumulators zeroed per 64-key tile, two k32 mma steps (attn_utils.cuh:896-974)
            T = torch.zeros((B, Hq, Sq, D), dtype=torch.float16)
            for c0 in range(0, s1 - s0, 32):
                T = (T.float() + P8[..., c0:c0 + 32] @ Vt[:, :, c0:c0 + 32]).half()
            O = O * alpha[..., None] + T.float()
        else:
            O = O * alpha[..., None] + P8 @ Vt
        m = m_new
    out = (O / d[..., None]) * vsc[:, :, None, :]
    if v_mean is not None:
        out = out + v_mean.float().repeat_interleave(g, dim=1)[:, :, None, :]
    out = out.to(out_dtype)
    if return_lse:
        return out, torch.log2(d) + m
    return out


# --------------------------------------------------------------------------------------------
# attention: Triton fp16-PV path (per-block scales)
# --------------------------------------------------------------------------------------------
def attn_int8_fp16_triton(q8, k8, v, q_scale, k_scale, *, is_causal=False, out_dtype=torch.float16,
                          BLOCK_M=128, BLOCK_N=64, return_lse=False, attn_mask=None):
    """sageattention/triton/attn_qk_int8_per_block.py:22-128 and _causal.py:22-122.
    qk = dot(q,k).f32 * (q_scale*k_scale) [q already carries sm_scale*log2e]; OOB keys -1e6
    (non-causal, :53) / -inf (causal, :46); p = exp2(qk - m); l += sum(p) (fp32, l init 1.0 with
    m init -inf -> alpha 0); acc = acc*alpha + dot(p.f16, v.f16, out_dtype=f16).
    attn_mask (non-causal, :33-52): [B,Hq,Sq,Sk] bool -> qk += where(mask, 0, -1e6) and a 128 x 64 block with no True
    element is skipped; otherwise an additive bias (promoted to fp32)."""
    B, Hq, Sq, D = q8.shape
    _, Hk, Sk, _ = k8.shape
    g = Hq // Hk
    qs_row = q_scale[:, :, torch.arange((Sq + BLOCK_M - 1) // BLOCK_M * BLOCK_M) // BLOCK_M][:, :, :Sq]
    kf = k8.float().repeat_interleave(g, dim=1)
    vf = v.to(torch.float16).float().repeat_interleave(g, dim=1)
    ksr = k_scale.repeat_interleave(g, dim=1)
    qf = q8.float()
    m = torch.full((B, Hq, Sq), float("-inf"))
    l = torch.ones((B, Hq, Sq))
    acc = torch.zeros((B, Hq, Sq, D))
    qi = torch.arange(Sq)[:, None]
    for s0 in range(0, Sk, BLOCK_N):
        s1 = min(s0 + BLOCK_N, Sk)
        S = (qf @ kf[:, :, s0:s1].transpose(-1, -2)) * (qs_row * ksr[:, :, s0 // BLOCK_N, None])[..., None]
        if is_causal:
            kj = torch.arange(s0, s1)[None, :]
            S = torch.where(kj > qi, torch.tensor(float("-inf")), S)
            # rows whose whole tile is masked keep m=-inf in the reference only for tiles the
            # reference never visits (it stops at the diagonal block); emulate by skipping them.
            live = (qi[:, 0] >= s0)
        else:
            live = torch.ones(Sq, dtype=torch.bool)
        lv = live[None, None, :]
        if attn_mask is not None:
            mb = attn_mask[:, :, :, s0:s1]
            if attn_mask.dtype == torch.bool:
                S = S + torch.where(mb, 0.0, -1.0e6)
                # block skip (:35-36): per (b, h, 128-row block) when the whole block is False
                nblk = (Sq + BLOCK_M - 1) // BLOCK_M
                anyt = torch.stack([mb[:, :, i * BLOCK_M:(i + 1) * BLOCK_M].flatten(2).any(-1) for i in range(nblk)], dim=-1)
                lv = anyt.repeat_interleave(BLOCK_M, dim=-1)[:, :, :Sq]
            else:
                S = S + mb.float()
        m_new = torch.maximum(m, S.amax(dim=-1))
        m_safe = torch.where(torch.isinf(m_new), torch.zeros_like(m_new), m_new)
        P = torch.exp2(S - m_safe[..., None])
        alpha = torch.where(torch.isinf(m_new), torch.ones_like(m), torch.exp2(m - m_safe))
        l = torch.where(lv, l * alpha + P.sum(-1), l)
        pv = (P.half().float() @ vf[:, :, s0:s1]).half().float()
        acc = torch.where(lv[..., None], acc * alpha[..., None] + pv, acc)
        m = torch.where(lv, m_new, m)
    out = (acc / l[..., None]).to(out_dtype)
    if return_lse:
        return out, torch.log2(l) + m
    return out


# --------------------------------------------------------------------------------------------
# whole-call restatements (host glue of sageattention/core.py)
# --------------------------------------------------------------------------------------------
def _pad_head_dim(q, k, v):
    """sageattention/core.py:752-761."""
    hd = q.size(-1)
    if hd < 64:
        tgt = 64
    elif 64 < hd < 128:
        tgt = 128
    elif hd > 128:
        raise ValueError(f"Unsupported head_dim: {hd}")
    else:
        tgt = hd
    if tgt != hd:
        q, k, v = (torch.nn.functional.pad(t, (0, tgt - hd)) for t in (q, k, v))
    return q, k, v, hd


def sageattn_qk_int8_pv_fp8_cuda(q, k, v, tensor_layout="HND", is_causal=False,
                                 qk_quant_gran="per_thread", sm_scale=None,
                                 pv_accum_dtype="fp32+fp16", smooth_k=True, smooth_v=False,
                                 return_lse=False, kv_tile=64, emulate_f16_accum=True, exp2_fn=None, lazy_tau=None):
    """sageattention/core.py:636-826 end to end (CPU).  emulate_f16_accum=False keeps the reference's V range
    for "fp32+fp16" (2.25) but accumulates PV in fp32 — the sm_90a kernel's arithmetic (fp32 accumulation)."""
    dtype = q.dtype
    q, k, v, hd_og = _pad_head_dim(q, k, v)
    if sm_scale is None:
        sm_scale = hd_og ** -0.5
    seq_dim = 1 if tensor_layout == "NHD" else 2
    km = k.mean(dim=seq_dim, keepdim=True) if smooth_k else None                    # core.py:773
    lse_corr = None
    if smooth_k and return_lse:                                                     # core.py:775-786
        qh, kmh = _to_hnd(q, tensor_layout), _to_hnd(km, tensor_layout)
        g = qh.shape[1] // kmh.shape[1]
        lse_corr = torch.matmul(qh, kmh.repeat_interleave(g, dim=1).transpose(2, 3)).squeeze(-1).to(torch.float32)  # input dtype, as the reference
    if qk_quant_gran == "per_warp":
        q8, qs, k8, ks = per_warp_int8_cuda(q, k, km, tensor_layout=tensor_layout)
    elif qk_quant_gran == "per_thread":
        q8, qs, k8, ks = quant_per_thread_int8_triton(q, k, km, tensor_layout=tensor_layout)
    else:
        raise AssertionError("qk_quant_gran must be either 'per_warp' or 'per_thread'.")
    scale_max = 2.25 if pv_accum_dtype == "fp32+fp16" else 448.0                    # core.py:805-807
    v8, vs, _ = per_channel_fp8_cuda(v, tensor_layout, scale_max, smooth_v=False)
    o = attn_int8_fp8_cuda(_to_hnd(q8, tensor_layout), _to_hnd(k8, tensor_layout), v8, qs, ks, vs,
                           qk_quant_gran=qk_quant_gran, is_causal=is_causal, sm_scale=sm_scale,
                           pv_accum_dtype=pv_accum_dtype if emulate_f16_accum else "fp32+fp32", out_dtype=dtype,
                           kv_tile=kv_tile, return_lse=return_lse, exp2_fn=exp2_fn, lazy_tau=lazy_tau)
    lse = None
    if return_lse:
        o, lse = o
        lse = lse / LOG2E_PY + (lse_corr * sm_scale if smooth_k else 0.0)           # core.py:823-826
    if tensor_layout == "NHD":
        o = o.transpose(1, 2)
    o = o[..., :hd_og]
    return (o, lse) if return_lse else o


def attn_int8_fp16_cuda(q8, k8, v, q_scale, k_scale, *, qk_quant_gran="per_thread", is_causal=False, sm_scale=1.0,
                        out_dtype=torch.float16, kv_tile=64, return_lse=False):
    """csrc/qattn/qk_int_sv_f16_cuda_sm80.cu:46-640 (`qk_int_sv_f16_attn_kernel`, the accum_f32 instantiation) restated:
    the fp8 kernel's loop without the exponent offset and with fp16 P and V —
      S_f = float(S_i32) * (sm_scale*log2e*q_scale*k_scale)   (:92, 255-300)   masks -5e6 (attn_utils.cuh:296-351)
      m_new = max(m_old, rowmax(S_f)); P = exp2(S_f - m_new)  (update_mdo<..., exp_offset=false>, :303-307)
      d += sum(P) in fp32 (accumulate_d kCudaCore, :312); P16 = half(P) (RS_32_to_16, :316)
      O = O*alpha + P16 @ V16 with f32 accumulators          (compute_fp16_sv_permuted, :339)
    epilogue O/d -> out dtype, lse = log2(d) + m              (normalize_d :540, :560-640)."""
    B, Hq, Sq, D = q8.shape
    _, Hk, Sk, _ = k8.shape
    g = Hq // Hk
    qs_row = _expand_q_scale(q_scale, qk_quant_gran, Sq)[:, :, :Sq]
    ks_key = _expand_k_scale(k_scale, qk_quant_gran, Sk)[:, :, :Sk].repeat_interleave(g, dim=1)
    kf = k8.float().repeat_interleave(g, dim=1)
    vf = v.to(torch.float16).float().repeat_interleave(g, dim=1)
    qf = q8.float()
    sm2 = torch.tensor(sm_scale, dtype=torch.float32) * torch.tensor(LOG2E_CU, dtype=torch.float32)
    m = torch.full((B, Hq, Sq), MASK_VALUE, dtype=torch.float32)
    d = torch.ones((B, Hq, Sq), dtype=torch.float32)
    O = torch.zeros((B, Hq, Sq, D), dtype=torch.float32)
    qi = torch.arange(Sq)[:, None]
    for s0 in range(0, Sk, kv_tile):
        s1 = min(s0 + kv_tile, Sk)
        if is_causal and s0 > Sq - 1:
            break
        S = (qf @ kf[:, :, s0:s1].transpose(-1, -2)) * ((sm2 * qs_row)[..., None] * ks_key[:, :, None, s0:s1])
        if is_causal:
            S = torch.where(torch.arange(s0, s1)[None, :] > qi, torch.tensor(MASK_VALUE), S)
        m_new = torch.maximum(m, S.amax(dim=-1))
        alpha = torch.exp2(m - m_new)
        P = torch.exp2(S - m_new[..., None])
        d = d * alpha + P.sum(dim=-1)
        O = O * alpha[..., None] + P.half().float() @ vf[:, :, s0:s1]
        m = m_new
    out = (O / d[..., None]).to(out_dtype)
    if return_lse:
        return out, torch.log2(d) + m
    return out


def sageattn_qk_int8_pv_fp16_cuda(q, k, v, tensor_layout="HND", is_causal=False, qk_quant_gran="per_thread", sm_scale=None,
                                  smooth_k=True, return_lse=False):
    """sageattention/core.py:451-633 end to end (CPU), pv_accum_dtype="fp32" (f32 accumulators, :601-603)."""
    dtype = q.dtype
    q, k, v, hd_og = _pad_head_dim(q, k, v)
    if sm_scale is None:
        sm_scale = hd_og ** -0.5
    seq_dim = 1 if tensor_layout == "NHD" else 2
    km = k.mean(dim=seq_dim, keepdim=True) if smooth_k else None                    # core.py:573
    lse_corr = None
    if smooth_k and return_lse:
        qh, kmh = _to_hnd(q, tensor_layout), _to_hnd(km, tensor_layout)
        g = qh.shape[1] // kmh.shape[1]
        lse_corr = torch.matmul(qh, kmh.repeat_interleave(g, dim=1).transpose(2, 3)).squeeze(-1).to(torch.float32)
    if qk_quant_gran == "per_warp":
        q8, qs, k8, ks = per_warp_int8_cuda(q, k, km, tensor_layout=tensor_layout)
    else:
        q8, qs, k8, ks = quant_per_thread_int8_triton(q, k, km, tensor_layout=tensor_layout)
    o = attn_int8_fp16_cuda(_to_hnd(q8, tensor_layout), _to_hnd(k8, tensor_layout), _to_hnd(v, tensor_layout), qs, ks,
                            qk_quant_gran=qk_quant_gran, is_causal=is_causal, sm_scale=sm_scale, out_dtype=dtype,
                            return_lse=return_lse)
    lse = None
    if return_lse:
        o, lse = o
        lse = lse / LOG2E_PY + (lse_corr * sm_scale if smooth_k else 0.0)
    if tensor_layout == "NHD":
        o = o.transpose(1, 2)
    o = o[..., :hd_og]
    return (o, lse) if return_lse else o


def sageattn_qk_int8_pv_fp16_triton(q, k, v, tensor_layout="HND", is_causal=False, sm_scale=None,
                                    smooth_k=True, return_lse=False, attn_mask=None):
    """sageattention/core.py:160-331 end to end (CPU); attn_mask: bool or q.dtype, broadcastable to [B,Hq,Sq,Sk]."""
    dtype = q.dtype
    q, k, v, hd_og = _pad_head_dim(q, k, v)
    seq_dim = 1 if tensor_layout == "NHD" else 2
    km = k.mean(dim=seq_dim, keepdim=True) if smooth_k else None
    lse_corr = None
    if smooth_k and return_lse:
        qh, kmh = _to_hnd(q, tensor_layout), _to_hnd(km, tensor_layout)
        g = qh.shape[1] // kmh.shape[1]
        lse_corr = torch.matmul(qh, kmh.repeat_interleave(g, dim=1).transpose(2, 3)).squeeze(-1).to(torch.float32)  # input dtype, as the reference
    if sm_scale is None:
        sm_scale = 1.0 / (hd_og ** 0.5)
    q8, qs, k8, ks = per_block_int8_triton(q, k, km=km, sm_scale=sm_scale, tensor_layout=tensor_layout)
    o = attn_int8_fp16_triton(_to_hnd(q8, tensor_layout), _to_hnd(k8, tensor_layout),
                              _to_hnd(v, tensor_layout), qs, ks, is_causal=is_causal, out_dtype=dtype,
                              return_lse=return_lse,
                              attn_mask=None if attn_mask is None else attn_mask.expand(
                                  _to_hnd(q, tensor_layout).shape[0], _to_hnd(q, tensor_layout).shape[1],
                                  _to_hnd(q, tensor_layout).shape[2], _to_hnd(k, tensor_layout).shape[2]))
    lse = None
    if return_lse:
        o, lse = o
        lse = lse / LOG2E_PY + (lse_corr * sm_scale if smooth_k else 0.0)
    if tensor_layout == "NHD":
        o = o.transpose(1, 2)
    o = o[..., :hd_og]
    return (o, lse) if return_lse else o


def quant_per_block_int8_varlen_triton(x, cu_seqlens, BLK, sm_scale=1.0):
    """sageattention/triton/quant_per_block_varlen.py:21-58: x [T,H,D]; per sequence, per BLK block;
    scale stored [sum_i ceil(L_i/BLK), H] (block-major, head-minor)."""
    T, H, D = x.shape
    cu = [int(c) for c in cu_seqlens]
    q_out = torch.empty((T, H, D), dtype=torch.int8)
    scales = []
    for i in range(len(cu) - 1):
        seg = x[cu[i]:cu[i + 1]].transpose(0, 1).unsqueeze(0)              # [1,H,L,D]
        if seg.shape[2] == 0:
            continue
        q8, sc = quant_per_block_int8_triton(seg, BLK, sm_scale, "HND")
        q_out[cu[i]:cu[i + 1]] = q8[0].transpose(0, 1)
        scales.append(sc[0].transpose(0, 1))                               # [nblk,H]
    scale = torch.cat(scales, dim=0) if scales else torch.empty((0, H))
    lens = torch.tensor([cu[i + 1] - cu[i] for i in range(len(cu) - 1)])
    cu_scale = torch.nn.functional.pad(torch.cumsum((lens + BLK - 1) // BLK, 0), (1, 0))
    return q_out, scale.contiguous(), cu_scale


def sageattn_varlen(q, k, v, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k,
                    is_causal=False, sm_scale=None, smooth_k=True):
    """sageattention/core.py:334-448 + triton/attn_qk_int8_block_varlen.py / _causal_varlen.py:
    packed [T,H,D]; K mean over ALL tokens of ALL sequences (core.py:433); per-block int8 per
    sequence; fp16 PV."""
    dtype = q.dtype
    q, k, v, hd_og = _pad_head_dim(q, k, v)
    if smooth_k:
        km = k.mean(dim=0, keepdim=True)
        k = k - km
    if sm_scale is None:
        sm_scale = 1.0 / (hd_og ** 0.5)
    q8, qs, cuqs = quant_per_block_int8_varlen_triton(q, cu_seqlens_q, 128, sm_scale * LOG2E_PY)
    k8, ks, cuks = quant_per_block_int8_varlen_triton(k, cu_seqlens_k, 64, 1.0)
    o = torch.zeros(q.shape, dtype=dtype)
    cq = [int(c) for c in cu_seqlens_q]
    ck = [int(c) for c in cu_seqlens_k]
    for i in range(len(cq) - 1):
        if cq[i + 1] == cq[i]:
            continue
        qi = q8[cq[i]:cq[i + 1]].transpose(0, 1).unsqueeze(0)
        ki = k8[ck[i]:ck[i + 1]].transpose(0, 1).unsqueeze(0)
        vi = v[ck[i]:ck[i + 1]].transpose(0, 1).unsqueeze(0)
        qsi = qs[int(cuqs[i]):int(cuqs[i + 1])].transpose(0, 1).unsqueeze(0)
        ksi = ks[int(cuks[i]):int(cuks[i + 1])].transpose(0, 1).unsqueeze(0)
        oi = attn_int8_fp16_triton(qi, ki, vi, qsi, ksi, is_causal=is_causal, out_dtype=dtype)
        o[cq[i]:cq[i + 1]] = oi[0].transpose(0, 1)
    return o[..., :hd_og]


def sdpa_fp32(q, k, v, is_causal=False, sm_scale=None, tensor_layout="HND"):
    """Exact fp32 attention, the accuracy yard-stick (not a reference function)."""
    qh, kh, vh = (_to_hnd(t, tensor_layout).float() for t in (q, k, v))
    g = qh.shape[1] // kh.shape[1]
    kh, vh = kh.repeat_interleave(g, 1), vh.repeat_interleave(g, 1)
    if sm_scale is None:
        sm_scale = qh.shape[-1] ** -0.5
    S = qh @ kh.transpose(-1, -2) * sm_scale
    if is_causal:
        Sq, Sk = S.shape[-2:]
        S = S.masked_fill(torch.arange(Sk)[None, :] > torch.arange(Sq)[:, None], float("-inf"))
    o = torch.softmax(S, dim=-1) @ vh
    return o.transpose(1, 2) if tensor_layout == "NHD" else o
