/*
 * sageattn_b200 — C ABI of the H100-native (sm_90a) SageAttention hot path.
 *
 * Plain C: raw device pointers, sizes, element strides and a cudaStream_t (passed as void*).
 * No torch types.  Every entry point returns 0 on success or a negative sab_status; the message of
 * the last failure on the calling thread is available from sab_last_error().  Nothing is allocated
 * or retained by the library: the caller owns every buffer (the reference convention).
 *
 * Each function names the reference interface it replaces (paths relative to thu-ml/SageAttention):
 *   csrc/fused/fused.h:19-76            the eight `_fused` quantisation entry points
 *   csrc/qattn/attn_cuda_sm89.h:19-104  the seven `_qattn_sm89` attention entry points
 *   sageattention/triton/quant_per_thread.py:154-203, quant_per_block.py:49-101,
 *   quant_per_block_varlen.py:60-104    the Triton quantisation launchers
 *   sageattention/triton/attn_qk_int8_block_varlen.py:123-150 (+ causal)   the varlen attention launcher
 *
 * Tensor convention: a "bhsd" tensor is addressed as ptr[b*stride_b + h*stride_h + s*stride_s + d]
 * (strides in ELEMENTS, innermost dimension contiguous) which covers both reference layouts
 * ("HND" [B,H,S,D] and "NHD" [B,S,H,D], tensor_layout 1 / 0 in the csrc/qattn launchers).
 */
#ifndef SAGEATTN_B200_H_
#define SAGEATTN_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
  SAB_OK = 0,
  SAB_ERR_INVALID = -1,     /* bad argument (reference: TORCH_CHECK / std::invalid_argument) */
  SAB_ERR_UNSUPPORTED = -2, /* unsupported head_dim / dtype / granularity                     */
  SAB_ERR_CUDA = -3,        /* CUDA runtime / driver failure (launch, tensor-map encode)       */
  SAB_ERR_ARCH = -4         /* device is not sm_90 (no fallback path exists)                   */
} sab_status;

/* element types of the 16-bit inputs / outputs */
#define SAB_DTYPE_FP16 0
#define SAB_DTYPE_BF16 1

/* QuantGranularity, csrc/qattn/attn_utils.cuh:52-58 (ints 2/3 cross the reference op boundary) */
#define SAB_GRAN_PER_BLOCK 1
#define SAB_GRAN_PER_WARP 2
#define SAB_GRAN_PER_THREAD 3

/* rounding / epsilon semantics of the INT8 quantisers */
#define SAB_SEM_CUDA 0   /* csrc/fused/fused.cu:147-184: amax floored 1e-7, x*(127/amax), cvt.rni       */
#define SAB_SEM_TRITON 1 /* triton/quant_per_block.py:41-45: scale=amax/127, x/scale, round-half-away    */

const char* sab_last_error(void);
/* 0 if the current device can run this library (compute capability 9.0), else SAB_ERR_ARCH. */
int sab_check_device(void);
int sab_version(void);

/* ------------------------------------------------------------------------------------------------
 * K smoothing mean.  Replaces `km = k.mean(dim=seq, keepdim=True)` (sageattention/core.py:773,
 * :433 for varlen): fp32 accumulation, result rounded to the input dtype.  mean is [B,H,D]
 * contiguous in `dtype`.  For the varlen form pass B=1, S=total tokens (mean over all sequences).
 * workspace: >= sab_k_mean_workspace_bytes(B,H,S,D) bytes of device scratch.
 * ---------------------------------------------------------------------------------------------- */
int64_t sab_k_mean_workspace_bytes(int B, int H, int S, int D);
int sab_k_mean(const void* k, int dtype, void* mean, int B, int H, int S, int D, int64_t stride_b,
               int64_t stride_h, int64_t stride_s, void* workspace, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Per-block INT8 quantisation of one tensor.  Replaces
 *   quant_per_block_int8_cuda (both overloads), quant_per_block_int8_fuse_sub_mean_cuda,
 *   quant_per_warp_int8_cuda            (csrc/fused/fused.h:19-49; semantics SAB_SEM_CUDA)
 *   triton quant_per_block_int8_kernel  (triton/quant_per_block.py:21-47; SAB_SEM_TRITON)
 * Every `blk` consecutive rows of a (b,h) share one scale; scale is [B,H,scale_cols] fp32 with
 * scale_cols >= ceil(S/blk) (the reference pads per_warp scales to ceil(S/BLKQ)*(BLKQ/WARPQ); the
 * padding entries are written with the all-zero-rows value).
 *   mean     : optional [B,H,D] (`dtype`), subtracted before quantisation.  SAB_SEM_CUDA subtracts
 *              in fp32 (fused.cu:119-126); SAB_SEM_TRITON first rounds (x-mean) to `dtype`
 *              (`k = k - km` in torch, quant_per_block.py:53-54).
 *   sm_scale : multiplied in fp32 before quantisation when has_sm_scale != 0.
 * blk in {16,32,64,128}; D in {64,128}.
 * ---------------------------------------------------------------------------------------------- */
int sab_quant_per_block_int8(const void* x, int dtype, const void* mean, int8_t* out, float* scale,
                             int B, int H, int S, int D, int64_t x_stride_b, int64_t x_stride_h,
                             int64_t x_stride_s, int64_t o_stride_b, int64_t o_stride_h,
                             int64_t o_stride_s, int scale_cols, int blk, int semantics,
                             int has_sm_scale, float sm_scale, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Per-thread INT8 quantisation.  Replaces triton quant_query_per_thread_int8_kernel /
 * quant_key_per_thread_int8_kernel (triton/quant_per_thread.py:21-98).
 *   is_key == 0: inside each 32-row block, group g = rows {g, g+8, g+16, g+24}; 8 scales / block;
 *                scale [B,H,ceil(S/128)*4*8].
 *   is_key != 0: inside each 64-key block, group t = keys {8j+2t, 8j+2t+1}; 4 scales / block;
 *                scale [B,H,ceil(S/64)*4].
 * scale = amax/127 + 1e-7, round-half-away; `mean` (optional) handled as SAB_SEM_TRITON above.
 * ---------------------------------------------------------------------------------------------- */
int sab_quant_per_thread_int8(const void* x, int dtype, const void* mean, int8_t* out, float* scale,
                              int B, int H, int S, int D, int64_t x_stride_b, int64_t x_stride_h,
                              int64_t x_stride_s, int64_t o_stride_b, int64_t o_stride_h,
                              int64_t o_stride_s, int scale_cols, int is_key, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Varlen per-block INT8 quantisation.  Replaces triton/quant_per_block_varlen.py:21-58.
 * x, out: packed [T,H,D] (token stride = stride_t, head stride = stride_h); cu_seqlens [nseq+1]
 * int32 device; cu_scale [nseq+1] int32 device = exclusive cumsum of ceil(L_i/blk); scale is
 * [cu_scale[nseq], H] (block-major, head-minor).  Semantics SAB_SEM_TRITON.
 * ---------------------------------------------------------------------------------------------- */
int sab_quant_per_block_int8_varlen(const void* x, int dtype, const void* mean, int8_t* out, float* scale,
                                    const int32_t* cu_seqlens, const int32_t* cu_scale, int nseq,
                                    int max_seqlen, int H, int D, int64_t x_stride_t, int64_t x_stride_h,
                                    int64_t o_stride_t, int64_t o_stride_h, int blk, int has_sm_scale,
                                    float sm_scale, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Per-channel FP8 (e4m3) quantisation of V.  Replaces transpose_pad_permute_cuda +
 * scale_fuse_quant_cuda / mean_scale_fuse_quant_cuda (csrc/fused/fused.h:58-76,
 * sageattention/quant.py:224-293).
 *   v      : bhsd, `dtype`.
 *   v_fp8  : [B,H,D,S_pad] bytes, token-contiguous ("V transposed"), S_pad = ceil(S/128)*128, tokens
 *            >= S are written as 0.  Unlike the reference there is NO 16-token permutation: that is
 *            an mma.sync fragment artefact (fused.cu:287-291); wgmma reads V^T tiles directly.
 *   v_scale: [B,H,D] fp32 = amax/scale_max;  v_fp8 = cvt.rn.satfinite.e4m3(v*(scale_max/amax)).
 *   v_mean : optional [B,H,D] fp32 (smooth_v): mean over tokens (denominator: S rounded up to 16,
 *            fused.cu:349,381), subtracted before quantisation.
 * Varlen form (cu_seqlens != NULL): v packed [T,H,D] (B ignored, stride_b ignored, stride_s = token
 * stride), per-channel statistics over ALL tokens, output [H,D,T_pad] where sequence i starts at
 * token column cu_pad[i] (cu_pad = exclusive cumsum of ceil(L_i/128)*128, int32 device, nseq+1).
 * workspace: >= sab_per_channel_fp8_workspace_bytes(...) bytes.
 * ---------------------------------------------------------------------------------------------- */
int64_t sab_per_channel_fp8_workspace_bytes(int B, int H, int S, int D);
int sab_per_channel_fp8(const void* v, int dtype, uint8_t* v_fp8, float* v_scale, float* v_mean, int B,
                        int H, int S, int D, int64_t stride_b, int64_t stride_h, int64_t stride_s,
                        int64_t s_pad, float scale_max, const int32_t* cu_seqlens,
                        const int32_t* cu_pad, int nseq, int max_seqlen, void* workspace, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Single-pass front-end (quantisation fused into the statistics pass).  One launch each; a thread-block
 * cluster per (b,h) reduces the statistic through distributed shared memory and then quantises, so K / V
 * are read from HBM once (the second read hits L2) instead of twice:
 *  sab_k_smooth_quant_int8   = sab_k_mean + sab_quant_per_thread_int8(is_key) [SAB_GRAN_PER_THREAD] or
 *                              sab_k_mean + sab_quant_per_block_int8(blk 64, SAB_SEM_CUDA) [SAB_GRAN_PER_WARP / PER_BLOCK],
 *                              i.e. `km = k.mean(...)` + the K half of per_thread_int8 / per_warp_int8
 *                              (sageattention/core.py:773, 788-795); mean_out [B,H,D] in `dtype` is also returned
 *                              (needed for the LSE correction, core.py:782-786).  Dense layouts only.
 *  sab_per_channel_fp8_fused = sab_per_channel_fp8 (dense form) without workspace.
 * The INT8 / FP8 outputs and scales are bit-identical to the two-step entry points given the same mean.
 * ---------------------------------------------------------------------------------------------- */
int sab_k_smooth_quant_int8(const void* k, int dtype, void* mean_out, int8_t* out, float* scale, int B, int H, int S,
                            int D, int64_t x_stride_b, int64_t x_stride_h, int64_t x_stride_s, int64_t o_stride_b,
                            int64_t o_stride_h, int64_t o_stride_s, int scale_cols, int granularity, void* stream);
int sab_per_channel_fp8_fused(const void* v, int dtype, uint8_t* v_fp8, float* v_scale, float* v_mean, int B, int H,
                              int S, int D, int64_t stride_b, int64_t stride_h, int64_t stride_s, int64_t s_pad,
                              float scale_max, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Building blocks of the sequence-parallel path (no reference counterpart: the reference ships no SP
 * code; semantics chosen so that the sharded result equals the single-GPU one):
 *  sab_channel_stats   : per-(b,h,d) fp32 sum / max / min over the LOCAL tokens (all-reduced by the host:
 *                        SUM for the global K mean, MAX/MIN for the global per-channel V range).
 *  sab_v_quant_with_amax: sab_per_channel_fp8 with the per-channel |max| supplied by the caller.
 * ---------------------------------------------------------------------------------------------- */
int sab_channel_stats(const void* x, int dtype, float* sum_out, float* max_out, float* min_out, int B, int H,
                      int S, int D, int64_t stride_b, int64_t stride_h, int64_t stride_s, void* workspace,
                      void* stream);
int sab_v_quant_with_amax(const void* v, int dtype, uint8_t* v_fp8, const float* amax, float* v_scale, int B,
                          int H, int S, int D, int64_t stride_b, int64_t stride_h, int64_t stride_s,
                          int64_t s_pad, float scale_max, void* workspace, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Fused attention: INT8 QK^T (wgmma s8) -> fp32 online softmax -> FP8 P -> FP8 PV
 * (wgmma e4m3, fp32 accumulation) -> fp16/bf16 O.
 * Replaces qk_int8_sv_f8_accum_{f32,f16}[_fuse_v_scale][_fuse_v_mean]_attn[_inst_buf]
 * (csrc/qattn/attn_cuda_sm89.h:19-104) and, with cu_seqlens, the Triton varlen launchers.
 *   q_int8 : bhsd int8 [B,Hq,Sq,D];  k_int8: bhsd int8 [B,Hkv,Skv,D];
 *   v_fp8  : [B,Hkv,D,s_pad] e4m3 as produced by sab_per_channel_fp8;
 *   out    : bhsd `out_dtype` [B,Hq,Sq,D];  lse: optional [B,Hq,Sq] fp32 (log2 units, as the
 *            reference kernel writes it, qk_int_sv_f8_cuda_sm89.cuh:691-703).
 *   q_scale/k_scale : fp32, packed exactly as the reference packs them for the given granularity
 *            (q: [B,Hq,ceil(Sq/128)*{1,4,32}], k: [B,Hkv,ceil(Skv/64)*{1,1,4}]);
 *   v_scale: optional [B,Hkv,D] (fuse_v_scale); v_mean: optional [B,Hkv,D] (fuse_v_mean).
 *   sm_scale: softmax scale; the kernel multiplies by log2(e) itself.  Pass fold_sm_scale != 0 when
 *            sm_scale*log2e is already folded into q (per_block Triton path, core.py:304).
 *   is_causal: top-left aligned (kv_idx > q_idx masked, attn_utils.cuh:310).
 * Sequence-parallel form (kv_seg_len > 0, dense only): k_int8 is [P*B,Hkv,kv_seg_len,D] and v_fp8 is
 * [P*B,Hkv,D,kv_seg_len] exactly as an all-gather of the P ranks' local shards lays them out (rank-major);
 * key t of batch b lives in segment t / kv_seg_len.  Skv = P*kv_seg_len, kv_seg_len % 128 == 0.
 * causal_q_offset: global index of this call's first query row (top-left causal alignment on global
 * indices); 0 on a single GPU.
 * Varlen form (cu_seqlens_q != NULL): q/out packed [Tq,Hq,D], k packed [Tk,Hkv,D] (B = number of
 * sequences, *_stride_b ignored), v_fp8 [Hkv,D,T_pad] with cu_pad_v offsets, scales
 * [nblocks_total,H] with cu_*_scale offsets (quant_per_block_varlen.py:72-79), per_block only.
 * ---------------------------------------------------------------------------------------------- */
int sab_qk_int8_sv_f8_attn(const int8_t* q_int8, const int8_t* k_int8, const uint8_t* v_fp8, void* out,
                           float* lse, const float* q_scale, const float* k_scale, const float* v_scale,
                           const float* v_mean, int out_dtype, int B, int Hq, int Hkv, int Sq, int Skv,
                           int D, int64_t q_stride_b, int64_t q_stride_h, int64_t q_stride_s,
                           int64_t k_stride_b, int64_t k_stride_h, int64_t k_stride_s, int64_t v_s_pad,
                           int64_t o_stride_b, int64_t o_stride_h, int64_t o_stride_s, int is_causal,
                           int q_gran, int k_gran, float sm_scale, int fold_sm_scale,
                           const int32_t* cu_seqlens_q, const int32_t* cu_seqlens_k,
                           const int32_t* cu_pad_v, const int32_t* cu_q_scale, const int32_t* cu_k_scale,
                           int max_seqlen_q, int causal_q_offset, int kv_seg_len, int32_t* debug_dump,
                           void* stream);

/* Block-sparse form of sab_qk_int8_sv_f8_attn (dense tensors only: no varlen, sequence-parallel or debug arguments).
 *   block_mask : bool (uint8, 0 = hidden) [Bm,Hm,ceil(Sq/128),ceil(Skv/64)] read through the element strides
 *                mask_stride_b / _h / _qb / _kb (0 broadcasts a dimension; Bm in {1,B}, Hm in {1,Hq}, indexed by the Q head).
 *   Key j is visible to query i of head h iff block_mask[b, h, i/128, j/64] (and j <= i when is_causal, which needs Sq == Skv).
 *   The kernel visits only the visible 128x64 tiles; with an all-visible mask it computes the bytes of sab_qk_int8_sv_f8_attn.
 *   A row with no visible key returns 0 and lse -inf.
 *   q_gran per-warp or per-thread (the INT8+FP8 path's), Skv <= 1048576: each CTA keeps its list of visible key blocks in shared
 *   memory (2 bytes per 64-key block).  The mask is checked before anything touches the device. */
int sab_qk_int8_sv_f8_attn_blocksparse(const int8_t* q_int8, const int8_t* k_int8, const uint8_t* v_fp8, void* out,
                                       float* lse, const float* q_scale, const float* k_scale, const float* v_scale,
                                       const float* v_mean, int out_dtype, int B, int Hq, int Hkv, int Sq, int Skv,
                                       int D, int64_t q_stride_b, int64_t q_stride_h, int64_t q_stride_s,
                                       int64_t k_stride_b, int64_t k_stride_h, int64_t k_stride_s, int64_t v_s_pad,
                                       int64_t o_stride_b, int64_t o_stride_h, int64_t o_stride_s, int is_causal,
                                       int q_gran, int k_gran, float sm_scale, int fold_sm_scale,
                                       const uint8_t* block_mask, int64_t mask_stride_b, int64_t mask_stride_h,
                                       int64_t mask_stride_qb, int64_t mask_stride_kb, void* stream);

/* Sliding-window form of sab_qk_int8_sv_f8_attn (dense tensors only, as the block-sparse form).
 *   Key j is visible to query i iff i - window_left <= j <= i + window_right (and j <= i when is_causal, which needs Sq == Skv);
 *   -1 leaves that side unbounded.  Top-left alignment (query i and key i are the same position); Sq != Skv is allowed when not
 *   causal.  Each 128-row Q tile visits only the 64-key tiles that meet its rows' windows and masks the elements on the tiles
 *   an edge crosses.  (-1, -1) computes the bytes of sab_qk_int8_sv_f8_attn, (-1, 0) those of its causal call.
 *   A row with no visible key returns 0 and lse -inf.  window_left / window_right < -1 and causal with Sq != Skv are refused
 *   before anything touches the device. */
int sab_qk_int8_sv_f8_attn_window(const int8_t* q_int8, const int8_t* k_int8, const uint8_t* v_fp8, void* out, float* lse,
                                  const float* q_scale, const float* k_scale, const float* v_scale, const float* v_mean,
                                  int out_dtype, int B, int Hq, int Hkv, int Sq, int Skv, int D, int64_t q_stride_b,
                                  int64_t q_stride_h, int64_t q_stride_s, int64_t k_stride_b, int64_t k_stride_h,
                                  int64_t k_stride_s, int64_t v_s_pad, int64_t o_stride_b, int64_t o_stride_h,
                                  int64_t o_stride_s, int is_causal, int q_gran, int k_gran, float sm_scale,
                                  int fold_sm_scale, int window_left, int window_right, void* stream);

/* ------------------------------------------------------------------------------------------------
 * FP16-PV variant: INT8 QK^T -> fp32 online softmax WITHOUT exponent offset -> FP16 P -> FP16 PV
 * (wgmma f16, fp32 accumulation).  Replaces the Triton attention launchers
 * `forward` of sageattention/triton/attn_qk_int8_per_block.py:130-183, attn_qk_int8_per_block_causal.py,
 * attn_qk_int8_block_varlen.py:123-150, attn_qk_int8_per_block_causal_varlen.py (the kernels behind
 * sageattn_qk_int8_pv_fp16_triton and sageattn_varlen).  Arguments as sab_qk_int8_sv_f8_attn except:
 *   v_f16t : [B,Hkv,D,s_pad] fp16 (token-contiguous, zero padded) from sab_v_transpose_f16;
 *   no v_scale / v_mean (V is not quantised); no sequence-parallel form.
 * sab_v_transpose_f16 replaces `v.to(torch.float16)` (sageattention/core.py:297-298) plus the K-major
 * re-layout the wgmma B operand needs; varlen form as sab_per_channel_fp8.
 * ---------------------------------------------------------------------------------------------- */
int sab_v_transpose_f16(const void* v, int dtype, void* v_f16t, int B, int H, int S, int D, int64_t stride_b,
                        int64_t stride_h, int64_t stride_s, int64_t s_pad, const int32_t* cu_seqlens,
                        const int32_t* cu_pad, int nseq, int max_seqlen, void* stream);
int sab_qk_int8_sv_f16_attn(const int8_t* q_int8, const int8_t* k_int8, const void* v_f16t, void* out, float* lse,
                            const float* q_scale, const float* k_scale, int out_dtype, int B, int Hq, int Hkv,
                            int Sq, int Skv, int D, int64_t q_stride_b, int64_t q_stride_h, int64_t q_stride_s,
                            int64_t k_stride_b, int64_t k_stride_h, int64_t k_stride_s, int64_t v_s_pad,
                            int64_t o_stride_b, int64_t o_stride_h, int64_t o_stride_s, int is_causal, int q_gran,
                            int k_gran, float sm_scale, int fold_sm_scale, const int32_t* cu_seqlens_q,
                            const int32_t* cu_seqlens_k, const int32_t* cu_pad_v, const int32_t* cu_q_scale,
                            const int32_t* cu_k_scale, int max_seqlen_q, void* stream);

/* Masked form of sab_qk_int8_sv_f16_attn: the `attn_mask` argument of sageattn_qk_int8_pv_fp16_triton
 * (sageattention/core.py:160-331: bool or q.dtype, broadcast to [B,Hq,Sq,Skv], non-causal only) as consumed by
 * sageattention/triton/attn_qk_int8_per_block.py:33-52:
 *   SAB_MASK_BOOL : uint8 elements, 0 = masked out (the reference adds -1e6 and skips all-false blocks);
 *   SAB_MASK_BIAS : additive bias in the output dtype (fp16 / bf16), added to S*scale in fp32 before the softmax.
 * mask_stride_* are ELEMENT strides of the broadcast view (0 for broadcast dimensions).  Dense, non-causal, K scales
 * per block / per warp; a row whose keys are all masked returns zeros (the reference: an unmasked softmax). */
#define SAB_MASK_BOOL 1
#define SAB_MASK_BIAS 2
int sab_qk_int8_sv_f16_attn_masked(const int8_t* q_int8, const int8_t* k_int8, const void* v_f16t, void* out, float* lse,
                                   const float* q_scale, const float* k_scale, int out_dtype, int B, int Hq, int Hkv,
                                   int Sq, int Skv, int D, int64_t q_stride_b, int64_t q_stride_h, int64_t q_stride_s,
                                   int64_t k_stride_b, int64_t k_stride_h, int64_t k_stride_s, int64_t v_s_pad,
                                   int64_t o_stride_b, int64_t o_stride_h, int64_t o_stride_s, int q_gran, int k_gran,
                                   float sm_scale, int fold_sm_scale, const void* attn_mask, int mask_kind,
                                   int64_t mask_stride_b, int64_t mask_stride_h, int64_t mask_stride_m,
                                   int64_t mask_stride_n, void* stream);

/* Sequence-parallel attention with the K/V gather fused into the launch (no reference counterpart: the reference ships no
 * sequence-parallel operator, example/parallel_sageattn_cogvideo.py:44-51 only wires sageattn into xfuser).  Same tensors as the
 * kv_seg_len > 0 form of sab_qk_int8_sv_f8_attn (k_int8 [P*B,Hkv,kv_seg_len,D], v_fp8 [P*B,Hkv,D,kv_seg_len], rank-major), but
 * the segments may still be arriving: the kernel's TMA producer waits until
 *     seg_flags[(kv_head / heads_per_flag) * (Skv / kv_seg_len) + segment] == seg_epoch      (32-bit, system-scope acquire)
 * before it loads the first tile of a segment.  The caller writes each flag in stream order behind the copies that fill that
 * (KV-head group, segment) — e.g. cudaMemcpyAsync from peer memory followed by cuStreamWriteValue32 on a second stream — and
 * passes a fresh epoch per call, so flags never need resetting.  The copies and flag writes must not need SMs that the
 * waiting CTAs occupy (copy engines + stream memory operations do not).  Dense, non-causal. */
int sab_qk_int8_sv_f8_attn_sp(const int8_t* q_int8, const int8_t* k_int8, const uint8_t* v_fp8, void* out, float* lse,
                              const float* q_scale, const float* k_scale, const float* v_scale, int out_dtype, int B, int Hq,
                              int Hkv, int Sq, int Skv, int D, int64_t q_stride_b, int64_t q_stride_h, int64_t q_stride_s,
                              int64_t k_stride_b, int64_t k_stride_h, int64_t k_stride_s, int64_t v_s_pad, int64_t o_stride_b,
                              int64_t o_stride_h, int64_t o_stride_s, int q_gran, int k_gran, float sm_scale, int kv_seg_len,
                              const uint32_t* seg_flags, uint32_t seg_epoch, int heads_per_flag, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Backward of the INT8-QK attention (no reference counterpart: the reference is forward-only).  The gradient of attention
 * evaluated at the forward's quantised logits, a straight-through estimator through the INT8 Q/K, FP8 V and FP8 P roundings:
 *   S = dequant(q_int8 k_int8^T) * sm_scale (the logits the forward kernel computed: same scales, granularities, fold),
 *   P = exp2(S*log2e - lse), dV = P^T dO, dP = dO V^T, delta = rowsum(dO o O), dS = P o (dP - delta),
 *   dQ = dS K * sm_scale, dK = dS^T Q * sm_scale.
 *   q_int8, k_int8, q_scale, k_scale, q_gran, k_gran, sm_scale, fold_sm_scale : exactly what the forward call received;
 *   q, k, v : the original 16-bit bhsd tensors (`dtype`); k must be UNsmoothed (the K mean has no gradient term: the rows of dS
 *             sum to zero), while k_int8 is the smoothed K the forward used, because lse is relative to it;
 *   o, dout : the forward's output and its gradient (bhsd, `dtype`); lse : [B,Hq,Sq] fp32, the forward's log2 LSE;
 *   k_mean : optional [B,Hkv,D] (`dtype`), the K smoothing mean the forward subtracted.  dQ is then taken as dS (K - k_mean): the
 *            same value in exact arithmetic, but the small residue in the row sums of dS (delta comes from the quantised
 *            forward's O) is not multiplied by a large K mean;
 *   dq, dk, dv : outputs in `dtype` with the strides of q, k, v.  GQA: dk / dv are summed over the Q heads of each KV head.
 *   workspace : >= sab_attn_bwd_workspace_bytes(B, Hq, Sq) bytes of device scratch.
 * Dense (packed sequences: sab_qk_int8_attn_bwd_varlen below; with the masked forward's attn_mask: sab_qk_int8_attn_bwd_masked);
 * is_causal needs Sq == Skv (top-left).  Deterministic: no atomics, a fixed summation order.
 * ---------------------------------------------------------------------------------------------- */
int64_t sab_attn_bwd_workspace_bytes(int B, int Hq, int Sq);
int sab_qk_int8_attn_bwd(const int8_t* q_int8, const int8_t* k_int8, const float* q_scale, const float* k_scale, const void* q,
                         const void* k, const void* v, const void* o, const void* dout, const float* lse, const void* k_mean,
                         void* dq, void* dk, void* dv, void* workspace, int dtype, int B, int Hq, int Hkv, int Sq, int Skv, int D,
                         int64_t q8_stride_b, int64_t q8_stride_h, int64_t q8_stride_s, int64_t k8_stride_b,
                         int64_t k8_stride_h, int64_t k8_stride_s, int64_t q_stride_b, int64_t q_stride_h, int64_t q_stride_s,
                         int64_t k_stride_b, int64_t k_stride_h, int64_t k_stride_s, int64_t v_stride_b, int64_t v_stride_h,
                         int64_t v_stride_s, int64_t o_stride_b, int64_t o_stride_h, int64_t o_stride_s, int64_t do_stride_b,
                         int64_t do_stride_h, int64_t do_stride_s, int is_causal, int q_gran, int k_gran, float sm_scale,
                         int fold_sm_scale, void* stream);

/* Varlen form of sab_qk_int8_attn_bwd: the gradient of the packed FP16-PV forward (sab_qk_int8_sv_f16_attn with cu_seqlens, the
 * kernel behind sageattn_varlen), each sequence on its own.  Same definition as above; the causal mask is top-left inside each
 * sequence (key j visible to row i iff j <= i), and Lq != Lk is allowed, as in the forward.
 *   q_int8, k_int8, q, k, v, o, dout, dq, dk, dv : packed [T,H,D] (Tq rows for q / o / dout / dq, Tk for k / v / dk / dv); the
 *            strides are (stride_t, stride_h) pairs in elements; dq / dk / dv have the strides of q / k / v;
 *   q_scale, k_scale : per-block [nblocks,Hq] / [nblocks,Hkv], sequence b's blocks starting at cu_q_scale[b] / cu_k_scale[b],
 *            as sab_quant_per_block_int8_varlen writes them (per_block Q and K, the only varlen granularity);
 *   lse    : [Hq,Tq] fp32 log2 units, the forward's (row h*Tq + cu_seqlens_q[b] + i);
 *   k_mean : optional [Hkv,D] (`dtype`), the K mean over all packed tokens the forward subtracted;
 *   cu_seqlens_q / cu_seqlens_k : [nseq+1] int32 token offsets; max_seqlen_q / max_seqlen_k : the longest sequence of each.
 *   workspace : >= sab_attn_bwd_workspace_bytes(1, Hq, Tq) bytes of device scratch.
 * Rows of dq and keys of dk / dv past cu_seqlens_*[nseq] belong to no sequence and are not written; a sequence with keys but no
 * queries gets zero dk / dv.  Deterministic like the dense form. */
int sab_qk_int8_attn_bwd_varlen(const int8_t* q_int8, const int8_t* k_int8, const float* q_scale, const float* k_scale, const void* q,
                                const void* k, const void* v, const void* o, const void* dout, const float* lse, const void* k_mean,
                                void* dq, void* dk, void* dv, void* workspace, int dtype, int nseq, int Hq, int Hkv, int Tq, int Tk,
                                int D, int64_t q8_stride_t, int64_t q8_stride_h, int64_t k8_stride_t, int64_t k8_stride_h,
                                int64_t q_stride_t, int64_t q_stride_h, int64_t k_stride_t, int64_t k_stride_h, int64_t v_stride_t,
                                int64_t v_stride_h, int64_t o_stride_t, int64_t o_stride_h, int64_t do_stride_t, int64_t do_stride_h,
                                const int32_t* cu_seqlens_q, const int32_t* cu_seqlens_k, const int32_t* cu_q_scale,
                                const int32_t* cu_k_scale, int max_seqlen_q, int max_seqlen_k, int is_causal, float sm_scale,
                                int fold_sm_scale, void* stream);

/* Masked form of sab_qk_int8_attn_bwd: the gradient of sab_qk_int8_sv_f16_attn_masked (the kernel behind
 * sageattn_qk_int8_pv_fp16_triton with attn_mask).  Same definition and arguments as sab_qk_int8_attn_bwd without is_causal (the
 * masked forward is non-causal), with the forward's masked logits:
 *   SAB_MASK_BOOL : P = 0 where the mask element is 0;
 *   SAB_MASK_BIAS : P = exp2(x - lse) with x = S*log2e + bias in fp32 (the forward's expression; bias -inf gives P = 0);
 *   a row with lse = -inf has no visible key (the forward returned zeros): its P and gradients are 0.
 *   attn_mask, mask_kind, mask_stride_* : exactly what the forward received (element strides of the [B,Hq,Sq,Skv] broadcast view,
 *            0 allowed); K scales per block / per warp, as the forward requires;
 *   dbias  : nullable, SAB_MASK_BIAS only: dense row-major [B,Hq,Sq,Skv] in `dtype`, 16-byte aligned, written with
 *            dBias = ln2 * dS (the bias is added to log2-unit logits, so it acts as bias*ln2 in natural-log units); masked and -inf
 *            positions get 0.  Summing it over the broadcast dimensions is the caller's (autograd's expand backward).
 * Deterministic like the dense form: every dBias element is written once, by the CTA that owns its Q row. */
int sab_qk_int8_attn_bwd_masked(const int8_t* q_int8, const int8_t* k_int8, const float* q_scale, const float* k_scale, const void* q,
                                const void* k, const void* v, const void* o, const void* dout, const float* lse, const void* k_mean,
                                void* dq, void* dk, void* dv, void* workspace, int dtype, int B, int Hq, int Hkv, int Sq, int Skv, int D,
                                int64_t q8_stride_b, int64_t q8_stride_h, int64_t q8_stride_s, int64_t k8_stride_b,
                                int64_t k8_stride_h, int64_t k8_stride_s, int64_t q_stride_b, int64_t q_stride_h, int64_t q_stride_s,
                                int64_t k_stride_b, int64_t k_stride_h, int64_t k_stride_s, int64_t v_stride_b, int64_t v_stride_h,
                                int64_t v_stride_s, int64_t o_stride_b, int64_t o_stride_h, int64_t o_stride_s, int64_t do_stride_b,
                                int64_t do_stride_h, int64_t do_stride_s, int q_gran, int k_gran, float sm_scale, int fold_sm_scale,
                                const void* attn_mask, int mask_kind, int64_t mask_stride_b, int64_t mask_stride_h,
                                int64_t mask_stride_m, int64_t mask_stride_n, void* dbias, void* stream);

/* Block-sparse form of sab_qk_int8_attn_bwd: the gradient of sab_qk_int8_sv_f8_attn_blocksparse.  Same definition and arguments as
 * sab_qk_int8_attn_bwd plus exactly the block mask the forward received (same checks, codes and messages); P = 0 on hidden tiles,
 * and a row with lse = -inf gets zero gradients.  The dQ kernel visits only the visible key blocks of each 128-row Q block; the
 * dK/dV kernel skips a (Q head, 64-row Q tile) step whose two 64-key blocks are both hidden.  Keys hidden from every row get zero
 * dk and dv.  Deterministic like the dense form. */
int sab_qk_int8_attn_bwd_blocksparse(const int8_t* q_int8, const int8_t* k_int8, const float* q_scale, const float* k_scale,
                                     const void* q, const void* k, const void* v, const void* o, const void* dout, const float* lse,
                                     const void* k_mean, void* dq, void* dk, void* dv, void* workspace, int dtype, int B, int Hq,
                                     int Hkv, int Sq, int Skv, int D, int64_t q8_stride_b, int64_t q8_stride_h,
                                     int64_t q8_stride_s, int64_t k8_stride_b, int64_t k8_stride_h, int64_t k8_stride_s,
                                     int64_t q_stride_b, int64_t q_stride_h, int64_t q_stride_s, int64_t k_stride_b,
                                     int64_t k_stride_h, int64_t k_stride_s, int64_t v_stride_b, int64_t v_stride_h,
                                     int64_t v_stride_s, int64_t o_stride_b, int64_t o_stride_h, int64_t o_stride_s,
                                     int64_t do_stride_b, int64_t do_stride_h, int64_t do_stride_s, int is_causal, int q_gran,
                                     int k_gran, float sm_scale, int fold_sm_scale, const uint8_t* block_mask,
                                     int64_t mask_stride_b, int64_t mask_stride_h, int64_t mask_stride_qb, int64_t mask_stride_kb,
                                     void* stream);

/* Sliding-window form of sab_qk_int8_attn_bwd: the gradient of sab_qk_int8_sv_f8_attn_window.  Same definition and arguments as
 * sab_qk_int8_attn_bwd plus exactly the window the forward received (same checks, codes and messages); P = 0 outside the window,
 * and a row with lse = -inf gets zero gradients.  The dQ kernel walks the forward's tile range of each 128-row Q tile; the dK/dV
 * kernel of the 128 keys at k0 visits only the 64-row Q tiles that meet rows [k0 - right, k0 + 127 + left].  Keys no row sees
 * get zero dk and dv.  Deterministic like the dense form. */
int sab_qk_int8_attn_bwd_window(const int8_t* q_int8, const int8_t* k_int8, const float* q_scale, const float* k_scale, const void* q,
                                const void* k, const void* v, const void* o, const void* dout, const float* lse, const void* k_mean,
                                void* dq, void* dk, void* dv, void* workspace, int dtype, int B, int Hq, int Hkv, int Sq, int Skv, int D,
                                int64_t q8_stride_b, int64_t q8_stride_h, int64_t q8_stride_s, int64_t k8_stride_b,
                                int64_t k8_stride_h, int64_t k8_stride_s, int64_t q_stride_b, int64_t q_stride_h, int64_t q_stride_s,
                                int64_t k_stride_b, int64_t k_stride_h, int64_t k_stride_s, int64_t v_stride_b, int64_t v_stride_h,
                                int64_t v_stride_s, int64_t o_stride_b, int64_t o_stride_h, int64_t o_stride_s, int64_t do_stride_b,
                                int64_t do_stride_h, int64_t do_stride_s, int is_causal, int q_gran, int k_gran, float sm_scale,
                                int fold_sm_scale, int window_left, int window_right, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Block-mask prediction from pooled Q/K statistics (no reference counterpart; SpargeAttn's training-free first stage): the
 * block_mask of sab_qk_int8_sv_f8_attn_blocksparse chosen from per-block means and self-similarities.
 *
 * sab_block_stats: x bhsd (`dtype`), D <= 128 and a multiple of 8 (zero padding changes no statistic), 16-byte aligned, strides
 * multiples of 8 elements; blk 128 (Q) or 64 (K).  For block c of each (b,h), with n = min(blk, S - c*blk) rows, in fp32:
 *   mean[b,h,c,:] = (1/n) sum_r x_r                                   ([B,H,ceil(S/blk),D] contiguous)
 *   sim[b,h,c]    = |sum_r x_r/|x_r||^2 / n^2  (a zero row counts 0)   ([B,H,ceil(S/blk)] contiguous)
 * sim is the mean of the block's n x n cosine-similarity matrix, diagonal included, so 0 <= sim <= 1.
 *
 * sab_predict_block_mask: q_mean / q_sim from sab_block_stats(q, blk 128), k_mean / k_sim from sab_block_stats(k, blk 64), the same D;
 * block_mask: bool bytes [B,Hq,nq,nk] contiguous, nq = ceil(Sq/128), nk = ceil(Skv/64).  Row (b,h,i), hk = h / (Hq/Hkv):
 *   candidates C_i = { j : k_sim[j] >= sim_threshold }, and 64 j <= 128 i + 127 when is_causal;
 *   p = softmax over C_i of sm_scale * (q_mean_i . k_mean_j);
 *   order C_i by p descending, ties by ascending j; j is kept iff the sum of p over the blocks before it in that order is
 *   < cdf_threshold (the top block is always kept; cdf_threshold >= 1 keeps every candidate);
 *   forced visible: the whole row if q_sim[i] < sim_threshold, the whole column j if k_sim[j] < sim_threshold, and when is_causal the
 *   diagonal blocks 128 i <= 64 j + 63 (so no row is empty);
 *   when is_causal every block with 64 j > 128 i + 127 is hidden, forced ones included.
 * Checks before touching the device: null pointers, D, Hq % Hkv, Skv <= 1048576, is_causal with Sq != Skv, cdf_threshold <= 0 or
 * NaN, a NaN sim_threshold, a non-finite sm_scale.  Deterministic (fixed summation orders, no atomics).
 * ---------------------------------------------------------------------------------------------- */
int sab_block_stats(const void* x, int dtype, float* mean, float* sim, int B, int H, int S, int D, int64_t stride_b,
                    int64_t stride_h, int64_t stride_s, int blk, void* stream);
int sab_predict_block_mask(const float* q_mean, const float* q_sim, const float* k_mean, const float* k_sim, uint8_t* block_mask,
                           int B, int Hq, int Hkv, int Sq, int Skv, int D, int is_causal, float sm_scale, float cdf_threshold,
                           float sim_threshold, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Packed variable-length INT8+FP8 attention with per-sequence statistics (no reference counterpart): the building blocks of
 * sageattn_varlen_qk_int8_pv_fp8_cuda.  Inputs are packed [T,H,D] (token stride stride_t, head stride stride_h); cu_seqlens
 * [nseq+1] int32 device, sequence b = tokens [cu_seqlens[b], cu_seqlens[b+1]) (empty sequences allowed); max_seqlen >= every
 * length (it sizes the grids; a larger value only adds idle CTAs).  Every statistic is taken per sequence, so sequence b gets
 * the bits of the dense entry points on that sequence alone; tokens past cu_seqlens[nseq] belong to no sequence and are not
 * read or written.  Unlike the varlen forms above (one K mean and one V scale over all packed tokens).
 *
 * sab_k_mean_varlen: mean [nseq,H,D] (`dtype`), bit for bit sab_k_mean of each sequence (same 1024-token chunks, aligned to the
 *   sequence's first token, same fold); an empty sequence gets 0.  workspace >= sab_k_mean_varlen_workspace_bytes(...).
 * sab_quant_int8_varlen: the Q (is_key == 0) or K (is_key != 0) half of per_thread_int8 (granularity SAB_GRAN_PER_THREAD,
 *   sab_quant_per_thread_int8's semantics) or per_warp_int8 (SAB_GRAN_PER_WARP, sab_quant_per_block_int8 with blk 32 / 64 and
 *   SAB_SEM_CUDA) on each sequence.  Blocks restart at every sequence: cu_scale [nseq+1] int32 device is the exclusive cumsum of
 *   ceil(L_b/128) (Q) or ceil(L_b/64) (K), and sequence b's scales are rows [cu_scale[b]*mult, (cu_scale[b]+nblk_b)*mult) of
 *   scale [rows,H] fp32, mult = 4 (per-warp Q), 32 (per-thread Q), 1 (per-warp K), 4 (per-thread K), in the column order of
 *   the dense call.  mean: optional [nseq,H,D] (`dtype`) K smoothing mean of each sequence (K only).
 * sab_per_channel_fp8_varlen: v_scale (and v_mean when not NULL, smooth_v) [nseq,H,D] fp32 of each sequence as
 *   sab_per_channel_fp8 computes them (v_mean's denominator is L_b rounded up to 16); an empty sequence gets 0.  v_fp8
 *   [H,D,t_pad] e4m3, sequence b at token columns [cu_pad[b], cu_pad[b] + ceil(L_b/128)*128), zero padded (cu_pad: exclusive
 *   cumsum of ceil(L_b/128)*128, int32 device).  workspace >= sab_per_channel_fp8_varlen_workspace_bytes(...).
 * sab_qk_int8_sv_f8_attn_varlen: the forward of sab_qk_int8_sv_f8_attn's varlen form with per-warp / per-thread scales from
 *   sab_quant_int8_varlen (q_gran, k_gran) and the per-sequence v_scale / v_mean [nseq,Hkv,D] of sab_per_channel_fp8_varlen
 *   (sm_scale never folded).  out [Tq,Hq,D]; lse (optional) [Hq,Tq] fp32 log2 units.  Causal is top-left inside each sequence
 *   (Lq != Lk allowed).  A sequence with no keys gets zero rows and lse -inf; rows past cu_seqlens_q[nseq] are not written.
 *   Needs Tk > 0.
 * sab_qk_int8_attn_bwd_varlen_seq: the gradient of sab_qk_int8_sv_f8_attn_varlen; sab_qk_int8_attn_bwd_varlen's arguments plus
 *   q_gran / k_gran, with k_mean the per-sequence [nseq,Hkv,D] mean of sab_k_mean_varlen (NULL without smoothing) and lse the
 *   forward's [Hq,Tq] log2 LSE.  For every sequence, dq / dk / dv are the bits of sab_qk_int8_attn_bwd on that sequence alone;
 *   rows and keys past cu_seqlens_*[nseq] are not written, and keys of a sequence with no queries get zeros.
 * ---------------------------------------------------------------------------------------------- */
int64_t sab_k_mean_varlen_workspace_bytes(int nseq, int H, int max_seqlen, int D);
int sab_k_mean_varlen(const void* k, int dtype, void* mean, const int32_t* cu_seqlens, int nseq, int max_seqlen, int H, int D,
                      int64_t stride_t, int64_t stride_h, void* workspace, void* stream);
int sab_quant_int8_varlen(const void* x, int dtype, const void* mean, int8_t* out, float* scale, const int32_t* cu_seqlens,
                          const int32_t* cu_scale, int nseq, int max_seqlen, int H, int D, int64_t x_stride_t, int64_t x_stride_h,
                          int64_t o_stride_t, int64_t o_stride_h, int granularity, int is_key, void* stream);
int64_t sab_per_channel_fp8_varlen_workspace_bytes(int nseq, int H, int max_seqlen, int D);
int sab_per_channel_fp8_varlen(const void* v, int dtype, uint8_t* v_fp8, float* v_scale, float* v_mean, const int32_t* cu_seqlens,
                               const int32_t* cu_pad, int nseq, int max_seqlen, int H, int D, int64_t stride_t, int64_t stride_h,
                               int64_t t_pad, float scale_max, void* workspace, void* stream);
int sab_qk_int8_sv_f8_attn_varlen(const int8_t* q_int8, const int8_t* k_int8, const uint8_t* v_fp8, void* out, float* lse,
                                  const float* q_scale, const float* k_scale, const float* v_scale, const float* v_mean, int out_dtype,
                                  int nseq, int Hq, int Hkv, int Tq, int Tk, int D, int64_t q_stride_t, int64_t q_stride_h,
                                  int64_t k_stride_t, int64_t k_stride_h, int64_t v_t_pad, int64_t o_stride_t, int64_t o_stride_h,
                                  int is_causal, int q_gran, int k_gran, float sm_scale, const int32_t* cu_seqlens_q,
                                  const int32_t* cu_seqlens_k, const int32_t* cu_pad_v, const int32_t* cu_q_scale,
                                  const int32_t* cu_k_scale, int max_seqlen_q, void* stream);
int sab_qk_int8_attn_bwd_varlen_seq(const int8_t* q_int8, const int8_t* k_int8, const float* q_scale, const float* k_scale, const void* q,
                                    const void* k, const void* v, const void* o, const void* dout, const float* lse, const void* k_mean,
                                    void* dq, void* dk, void* dv, void* workspace, int dtype, int nseq, int Hq, int Hkv, int Tq, int Tk,
                                    int D, int64_t q8_stride_t, int64_t q8_stride_h, int64_t k8_stride_t, int64_t k8_stride_h,
                                    int64_t q_stride_t, int64_t q_stride_h, int64_t k_stride_t, int64_t k_stride_h, int64_t v_stride_t,
                                    int64_t v_stride_h, int64_t o_stride_t, int64_t o_stride_h, int64_t do_stride_t, int64_t do_stride_h,
                                    const int32_t* cu_seqlens_q, const int32_t* cu_seqlens_k, const int32_t* cu_q_scale,
                                    const int32_t* cu_k_scale, int max_seqlen_q, int max_seqlen_k, int is_causal, int q_gran,
                                    int k_gran, float sm_scale, void* stream);

/* Sliding-window forms of the packed per-sequence INT8+FP8 attention (no reference counterpart): sab_qk_int8_sv_f8_attn_varlen and
 * sab_qk_int8_attn_bwd_varlen_seq with the window of sab_qk_int8_sv_f8_attn_window, applied inside each sequence.  Key j of
 * sequence b is visible to its query i iff i - window_left <= j <= i + window_right (-1: that side unbounded; top-left inside the
 * sequence), j < Lk_b, and j <= i when is_causal (Lq != Lk allowed); no window reaches into a neighbouring sequence.  Each
 * sequence's window is clamped at its own lengths (a side >= Lq_b or >= Lk_b becomes -1, as sab_qk_int8_sv_f8_attn_window clamps
 * it for the dense call), so sequence b gets the bits of the dense window entry on that sequence alone, forward and gradient.
 * Causal with (left, right) is non-causal with (left, 0).  (-1, -1) computes the bits of the entries without a window, (-1, 0)
 * non-causal those of their causal call.  A row with no visible key returns 0 and lse -inf and gets zero gradients; keys no row
 * sees get zero dk and dv.  window_left / window_right < -1 and missing sequence tables are refused before anything touches the
 * device; a side is first clamped at max_seqlen_q (left) and at Tk (forward) or max_seqlen_k (gradient, right). */
int sab_qk_int8_sv_f8_attn_varlen_window(const int8_t* q_int8, const int8_t* k_int8, const uint8_t* v_fp8, void* out, float* lse,
                                         const float* q_scale, const float* k_scale, const float* v_scale, const float* v_mean,
                                         int out_dtype, int nseq, int Hq, int Hkv, int Tq, int Tk, int D, int64_t q_stride_t,
                                         int64_t q_stride_h, int64_t k_stride_t, int64_t k_stride_h, int64_t v_t_pad,
                                         int64_t o_stride_t, int64_t o_stride_h, int is_causal, int q_gran, int k_gran, float sm_scale,
                                         const int32_t* cu_seqlens_q, const int32_t* cu_seqlens_k, const int32_t* cu_pad_v,
                                         const int32_t* cu_q_scale, const int32_t* cu_k_scale, int max_seqlen_q, int window_left,
                                         int window_right, void* stream);
int sab_qk_int8_attn_bwd_varlen_window(const int8_t* q_int8, const int8_t* k_int8, const float* q_scale, const float* k_scale,
                                       const void* q, const void* k, const void* v, const void* o, const void* dout, const float* lse,
                                       const void* k_mean, void* dq, void* dk, void* dv, void* workspace, int dtype, int nseq, int Hq,
                                       int Hkv, int Tq, int Tk, int D, int64_t q8_stride_t, int64_t q8_stride_h, int64_t k8_stride_t,
                                       int64_t k8_stride_h, int64_t q_stride_t, int64_t q_stride_h, int64_t k_stride_t,
                                       int64_t k_stride_h, int64_t v_stride_t, int64_t v_stride_h, int64_t o_stride_t,
                                       int64_t o_stride_h, int64_t do_stride_t, int64_t do_stride_h, const int32_t* cu_seqlens_q,
                                       const int32_t* cu_seqlens_k, const int32_t* cu_q_scale, const int32_t* cu_k_scale,
                                       int max_seqlen_q, int max_seqlen_k, int is_causal, int q_gran, int k_gran, float sm_scale,
                                       int window_left, int window_right, void* stream);

/* Attention against a paged KV cache (no reference counterpart): the building blocks of sageattn_varlen_kvcache.
 *   The paged quantisers read K or V from a cache [num_pages, page_size, H, D] (`dtype`; page stride page_stride, slot stride
 *   stride_t, head stride stride_h, in elements, each a multiple of 8, 16-byte aligned base) through block_table [nseq, *] int32
 *   device (row stride table_stride): token t of sequence b is slot t % page_size of page block_table[b * table_stride + t /
 *   page_size].  cu_seqlens [nseq+1] int32 device is the exclusive cumsum of the sequence lengths Lk_b (the tokens read) and places
 *   sequence b of the outputs, which are exactly those of the packed entries above on the gathered tensor, bit for bit:
 *   sab_k_mean_paged = sab_k_mean_varlen, sab_quant_int8_paged = sab_quant_int8_varlen with is_key = 1 (out [Tk,H,D] at row
 *   cu_seqlens[b] + t), sab_per_channel_fp8_paged = sab_per_channel_fp8_varlen (v_fp8 [H,D,t_pad] at column cu_pad[b] + t).
 *   Slots past Lk_b and pages the first ceil(Lk_b/page_size) table entries do not name are never read.  The table entries are
 *   trusted: each must lie in [0, num_pages).  Workspaces: sab_k_mean_varlen_workspace_bytes / sab_per_channel_fp8_varlen_workspace_bytes.
 * sab_qk_int8_sv_f8_attn_varlen_bottom_right: sab_qk_int8_sv_f8_attn_varlen with causal aligned bottom-right inside each sequence:
 *   query i of sequence b sees key j iff j <= i + Lk_b - Lq_b (Lk_b < Lq_b allowed: its first Lq_b - Lk_b rows see no key and
 *   return 0 and lse -inf).  For Lk_b >= Lq_b sequence b gets the bits of sab_qk_int8_sv_f8_attn_window on that sequence alone with
 *   the window (-1, Lk_b - Lq_b), non-causal.  Non-causal (is_causal == 0) is sab_qk_int8_sv_f8_attn_varlen itself. */
int sab_k_mean_paged(const void* k_cache, int dtype, void* mean, const int32_t* cu_seqlens, const int32_t* block_table,
                     int64_t table_stride, int page_size, int nseq, int max_seqlen, int H, int D, int64_t page_stride, int64_t stride_t,
                     int64_t stride_h, void* workspace, void* stream);
int sab_quant_int8_paged(const void* k_cache, int dtype, const void* mean, int8_t* out, float* scale, const int32_t* cu_seqlens,
                         const int32_t* cu_scale, const int32_t* block_table, int64_t table_stride, int page_size, int nseq,
                         int max_seqlen, int H, int D, int64_t page_stride, int64_t stride_t, int64_t stride_h, int64_t o_stride_t,
                         int64_t o_stride_h, int granularity, void* stream);
int sab_per_channel_fp8_paged(const void* v_cache, int dtype, uint8_t* v_fp8, float* v_scale, float* v_mean, const int32_t* cu_seqlens,
                              const int32_t* cu_pad, const int32_t* block_table, int64_t table_stride, int page_size, int nseq,
                              int max_seqlen, int H, int D, int64_t page_stride, int64_t stride_t, int64_t stride_h, int64_t t_pad,
                              float scale_max, void* workspace, void* stream);
int sab_qk_int8_sv_f8_attn_varlen_bottom_right(const int8_t* q_int8, const int8_t* k_int8, const uint8_t* v_fp8, void* out, float* lse,
                                               const float* q_scale, const float* k_scale, const float* v_scale, const float* v_mean,
                                               int out_dtype, int nseq, int Hq, int Hkv, int Tq, int Tk, int D, int64_t q_stride_t,
                                               int64_t q_stride_h, int64_t k_stride_t, int64_t k_stride_h, int64_t v_t_pad,
                                               int64_t o_stride_t, int64_t o_stride_h, int is_causal, int q_gran, int k_gran,
                                               float sm_scale, const int32_t* cu_seqlens_q, const int32_t* cu_seqlens_k,
                                               const int32_t* cu_pad_v, const int32_t* cu_q_scale, const int32_t* cu_k_scale,
                                               int max_seqlen_q, void* stream);

/* Block-sparse forms of the packed per-sequence INT8+FP8 attention (no reference counterpart): sab_qk_int8_sv_f8_attn_varlen and
 * sab_qk_int8_attn_bwd_varlen_seq with the block mask of sab_qk_int8_sv_f8_attn_blocksparse, applied inside each sequence.
 *   block_mask : bool (uint8, 0 = hidden) [nseq or 1, Hq or 1, ceil(max_seqlen_q/128), ceil(max_seqlen_k/64)] read through the
 *                element strides mask_stride_b / _h / _qb / _kb (0 broadcasts a dimension; indexed by the Q head).  Sequence b's
 *                blocks start at its own first token, as its INT8 blocks do; entries past its own ceil(Lq_b/128) x ceil(Lk_b/64)
 *                blocks are never read.
 *   Key j of sequence b is visible to its query i iff block_mask[b, h, i/128, j/64], j < Lk_b, and j <= i when is_causal (top-left
 *   inside the sequence, Lq != Lk allowed).  Sequence b gets the bits of the dense block-sparse entry on that sequence alone with
 *   mask slice [b, :, :ceil(Lq_b/128), :ceil(Lk_b/64)], forward and gradient; with an all-visible mask, the bits of the entries
 *   without a mask.  A row with no visible key returns 0 and lse -inf and gets zero gradients; keys no row sees get zero dk and dv.
 *   max_seqlen_k <= 1048576 (each CTA keeps its list of visible key blocks in shared memory, 2 bytes per 64-key block of the longest
 *   sequence).  Refused before anything touches the device: a null mask, negative strides, per-block Q scales, max_seqlen_k >
 *   1048576, missing sequence tables. */
int sab_qk_int8_sv_f8_attn_varlen_blocksparse(const int8_t* q_int8, const int8_t* k_int8, const uint8_t* v_fp8, void* out, float* lse,
                                              const float* q_scale, const float* k_scale, const float* v_scale, const float* v_mean,
                                              int out_dtype, int nseq, int Hq, int Hkv, int Tq, int Tk, int D, int64_t q_stride_t,
                                              int64_t q_stride_h, int64_t k_stride_t, int64_t k_stride_h, int64_t v_t_pad,
                                              int64_t o_stride_t, int64_t o_stride_h, int is_causal, int q_gran, int k_gran,
                                              float sm_scale, const int32_t* cu_seqlens_q, const int32_t* cu_seqlens_k,
                                              const int32_t* cu_pad_v, const int32_t* cu_q_scale, const int32_t* cu_k_scale,
                                              int max_seqlen_q, int max_seqlen_k, const uint8_t* block_mask, int64_t mask_stride_b,
                                              int64_t mask_stride_h, int64_t mask_stride_qb, int64_t mask_stride_kb, void* stream);
int sab_qk_int8_attn_bwd_varlen_blocksparse(const int8_t* q_int8, const int8_t* k_int8, const float* q_scale, const float* k_scale,
                                            const void* q, const void* k, const void* v, const void* o, const void* dout,
                                            const float* lse, const void* k_mean, void* dq, void* dk, void* dv, void* workspace,
                                            int dtype, int nseq, int Hq, int Hkv, int Tq, int Tk, int D, int64_t q8_stride_t,
                                            int64_t q8_stride_h, int64_t k8_stride_t, int64_t k8_stride_h, int64_t q_stride_t,
                                            int64_t q_stride_h, int64_t k_stride_t, int64_t k_stride_h, int64_t v_stride_t,
                                            int64_t v_stride_h, int64_t o_stride_t, int64_t o_stride_h, int64_t do_stride_t,
                                            int64_t do_stride_h, const int32_t* cu_seqlens_q, const int32_t* cu_seqlens_k,
                                            const int32_t* cu_q_scale, const int32_t* cu_k_scale, int max_seqlen_q, int max_seqlen_k,
                                            int is_causal, int q_gran, int k_gran, float sm_scale, const uint8_t* block_mask,
                                            int64_t mask_stride_b, int64_t mask_stride_h, int64_t mask_stride_qb,
                                            int64_t mask_stride_kb, void* stream);

/* Packed forms of the block-mask prediction (no reference counterpart): sab_block_stats and sab_predict_block_mask of every packed
 * sequence on its own.  Inputs and sequence tables as the packed entries above (cu_seqlens int32 device, max_seqlen >= every length).
 * sab_block_stats_varlen: x packed [T,H,D]; blocks of blk rows restart at each sequence's first token.  mean [nseq,H,nblk,D] and
 *   sim [nseq,H,nblk] contiguous fp32 with nblk = ceil(max_seqlen/blk); block c of sequence b gets the bits of sab_block_stats on
 *   that sequence alone, and blocks past the end of a sequence get 0.  Checks of sab_block_stats.
 * sab_predict_block_mask_varlen: statistics from sab_block_stats_varlen (q: blk 128, k: blk 64); block_mask bool bytes
 *   [nseq,Hq,ceil(max_seqlen_q/128),ceil(max_seqlen_k/64)] contiguous.  Slice [b, :, :ceil(Lq_b/128), :ceil(Lk_b/64)] is the bits
 *   of sab_predict_block_mask on sequence b alone (each sequence sorts on its own power-of-two length, so its prefix masses are
 *   summed in the dense call's order); every other byte is 0, and so is every byte of a sequence without queries or keys.  Causal
 *   is top-left inside each sequence with the same rules, Lq != Lk allowed.  The lengths are read on the device.  Checks of
 *   sab_predict_block_mask (with max_seqlen_k for kv_len), except that causal needs no Lq == Lk; missing sequence tables are
 *   refused too. */
int sab_block_stats_varlen(const void* x, int dtype, float* mean, float* sim, const int32_t* cu_seqlens, int nseq, int max_seqlen,
                           int H, int D, int64_t stride_t, int64_t stride_h, int blk, void* stream);
int sab_predict_block_mask_varlen(const float* q_mean, const float* q_sim, const float* k_mean, const float* k_sim,
                                  uint8_t* block_mask, const int32_t* cu_seqlens_q, const int32_t* cu_seqlens_k, int nseq, int Hq,
                                  int Hkv, int max_seqlen_q, int max_seqlen_k, int D, int is_causal, float sm_scale,
                                  float cdf_threshold, float sim_threshold, void* stream);

/* 8-bit paged KV cache for decoding (no reference counterpart): the building blocks of PagedKVCache8 and sageattn_kvcache8.
 *   The cache is token-major and contiguous: k_pages int8 and v_pages e4m3 [num_pages, page_size, Hkv, D], k_scale and v_scale fp32
 *   [num_pages, page_size, Hkv], k_smooth fp32 [Hkv, D].  D is 64 or 128, page_size a multiple of 16, `dtype` the 16-bit type of
 *   the tokens written and of q / out.  Slot s is token s % page_size of page s / page_size.
 * sab_kvcache8_write: quantises T tokens k, v [T, Hkv, D] (element strides k_stride_t / k_stride_h, v_stride_t / v_stride_h, last
 *   dim contiguous) into the slots slot_mapping[t] (int64 device, page * page_size + slot; a negative entry skips the token, and so
 *   does an entry >= num_pages * page_size), one launch.  Per (token, head), in fp32: K x = k - k_smooth[h], amax = max|x|, k_scale
 *   = amax / 127 (IEEE), k8 = cvt.rni.sat.s8(x * RN(127 / amax)); V amax = max|v|, v_scale = amax / 448, v8 =
 *   cvt.rn.satfinite.e4m3(v * RN(448 / amax)).  amax == 0 stores scale 0 and zeros; when RN(qmax / amax) overflows (a denormal
 *   amax) the quotient x / scale is used instead.  The result depends on the token alone; unmapped slots are never written.
 * sab_kvcache8_attn: attention of packed q [Tq, Hq, D] (cu_seqlens_q [nseq+1] int32 device) against the cache: sequence b has
 *   Lk_b = seqused_k[b] keys (int32 device, read only on the device; clamped to max_pages * page_size), key j at slot j % page_size
 *   of page block_table[b * table_stride + j / page_size] (trusted, in [0, num_pages)).  Causal is bottom-right: query i sees key j
 *   iff j <= i + Lk_b - Lq_b, with Lq_b = cu_seqlens_q[b + 1] - cu_seqlens_q[b] even when it exceeds max_seqlen_q (only the
 *   first max_seqlen_q rows are then written, each seeing what it sees in the whole sequence).  Q is quantised per (token, head) as K is, without smoothing; logits in log2 units are
 *   float(dot(q8, k8)) * (q_scale * sm_scale * log2e) * k_scale.  Keys are cut into chunks of sab_kvcache8_chunk_keys() keys, one
 *   CTA per (sequence, KV head, chunk) holding all max_seqlen_q * Hq / Hkv <= 64 query rows of that KV head (rows past
 *   max_seqlen_q are not written); within a chunk an exact running max over 64-key tiles, P = bf16(p * v_scale) times bf16(v8)
 *   with fp32 accumulation.  A second kernel merges the chunks of a row in ascending order (no atomics: bit-reproducible).  out
 *   [Tq, Hq, D] (strides o_stride_t / o_stride_h) in `dtype`; lse (optional) [Hq, Tq] fp32 in natural-log units including
 *   (q . k_smooth) * sm_scale.  A row that sees no key returns 0 and lse -inf.  workspace: sab_kvcache8_workspace_bytes(Tq, Hq, D,
 *   max_pages * page_size) bytes.  No host synchronisation: the grid follows nseq, Hkv and max_pages * page_size.  Launch-grid
 *   limits, refused with SAB_ERR_INVALID: Hq <= 65535, nseq * ceil(max_pages * page_size / chunk) < 2^31, nseq * max_seqlen_q
 *   < 2^31 and max_pages * page_size < 2^31. */
int sab_kvcache8_chunk_keys(void);
int64_t sab_kvcache8_workspace_bytes(int Tq, int Hq, int D, int64_t max_keys);
int sab_kvcache8_write(const void* k, const void* v, int dtype, const float* k_smooth, const int64_t* slot_mapping, int T, int Hkv,
                       int D, int64_t k_stride_t, int64_t k_stride_h, int64_t v_stride_t, int64_t v_stride_h, int8_t* k_pages,
                       float* k_scale, uint8_t* v_pages, float* v_scale, int64_t num_pages, int page_size, void* stream);
int sab_kvcache8_attn(const void* q, int dtype, const int8_t* k_pages, const float* k_scale, const uint8_t* v_pages,
                      const float* v_scale, const float* k_smooth, void* out, float* lse, const int32_t* cu_seqlens_q,
                      const int32_t* seqused_k, const int32_t* block_table, int64_t table_stride, int max_pages, int nseq, int Tq,
                      int Hq, int Hkv, int D, int page_size, int64_t q_stride_t, int64_t q_stride_h, int64_t o_stride_t,
                      int64_t o_stride_h, int max_seqlen_q, int is_causal, float sm_scale, void* workspace, void* stream);
/* sab_kvcache8_prefill: attention of packed query chunks of any length against the same cache (chunked prefill, prefix caching):
 *   the arguments, checks and causal rule of sab_kvcache8_attn without its row limit and without a workspace.  One CTA per
 *   (sequence, 128-row Q tile, Q head), grid nseq * ceil(max_seqlen_q / 128) x Hq, so no host synchronisation.  Numerics: those of
 *   sab_kvcache8_attn with one chunk: Q quantised per (token, head) to INT8, logits in log2 units float(dot(q8, k8)) * (q_scale *
 *   sm_scale * log2e) * k_scale, one exact running max per row over 64-key tiles from key 0, P = bf16(p * v_scale) times bf16(v8)
 *   with fp32 accumulation (wgmma), O / l.  A row's bits depend only on its own q, keys and values.  out [Tq, Hq, D] (strides
 *   o_stride_t / o_stride_h, even, 4-byte aligned) in `dtype`; lse (optional) [Hq, Tq] fp32 as in sab_kvcache8_attn.  A row that
 *   sees no key returns 0 and lse -inf; rows past max_seqlen_q are not written, and the rows written take Lq_b from
 *   cu_seqlens_q as in sab_kvcache8_attn.  Launch-grid limits, refused with SAB_ERR_INVALID:
 *   Hq <= 65535, nseq * ceil(max_seqlen_q / 128) < 2^31 and max_pages * page_size < 2^31. */
int sab_kvcache8_prefill(const void* q, int dtype, const int8_t* k_pages, const float* k_scale, const uint8_t* v_pages,
                         const float* v_scale, const float* k_smooth, void* out, float* lse, const int32_t* cu_seqlens_q,
                         const int32_t* seqused_k, const int32_t* block_table, int64_t table_stride, int max_pages, int nseq, int Tq,
                         int Hq, int Hkv, int D, int page_size, int64_t q_stride_t, int64_t q_stride_h, int64_t o_stride_t,
                         int64_t o_stride_h, int max_seqlen_q, int is_causal, float sm_scale, void* stream);
/* sab_kvcache8_attn_window / sab_kvcache8_prefill_window: sab_kvcache8_attn / sab_kvcache8_prefill with a sliding window, the same
 *   arguments plus window_left / window_right (>= -1, else SAB_ERR_INVALID before any launch; -1 leaves a side unbounded) and the
 *   same workspace size.  With off_b = Lk_b - Lq_b, query i sees key j iff i + off_b - window_left <= j <= i + off_b +
 *   window_right, and j <= i + off_b as well when is_causal.  Table entries read: only keys j >= max(0, Lk_b - Lq_b -
 *   window_left) are ever loaded; the table entries, K / V bytes and scales of keys below that bound are never read, so those
 *   entries may name any page in [0, num_pages) (a shared null page, or pages reused for newer tokens).  Numerics and the bits
 *   of a row are those of the call without a window on the visible keys: tiles left of the window are skipped, and a tile in
 *   which a row sees nothing leaves it unchanged.  A row that sees no key returns 0 and lse -inf. */
int sab_kvcache8_attn_window(const void* q, int dtype, const int8_t* k_pages, const float* k_scale, const uint8_t* v_pages,
                             const float* v_scale, const float* k_smooth, void* out, float* lse, const int32_t* cu_seqlens_q,
                             const int32_t* seqused_k, const int32_t* block_table, int64_t table_stride, int max_pages, int nseq,
                             int Tq, int Hq, int Hkv, int D, int page_size, int64_t q_stride_t, int64_t q_stride_h,
                             int64_t o_stride_t, int64_t o_stride_h, int max_seqlen_q, int is_causal, float sm_scale,
                             void* workspace, int window_left, int window_right, void* stream);
int sab_kvcache8_prefill_window(const void* q, int dtype, const int8_t* k_pages, const float* k_scale, const uint8_t* v_pages,
                                const float* v_scale, const float* k_smooth, void* out, float* lse, const int32_t* cu_seqlens_q,
                                const int32_t* seqused_k, const int32_t* block_table, int64_t table_stride, int max_pages, int nseq,
                                int Tq, int Hq, int Hkv, int D, int page_size, int64_t q_stride_t, int64_t q_stride_h,
                                int64_t o_stride_t, int64_t o_stride_h, int max_seqlen_q, int is_causal, float sm_scale,
                                int window_left, int window_right, void* stream);
/* sab_kvcache8_attn_shared: sab_kvcache8_attn with a prefix every sequence shares, read once for many sequences (parallel
 *   sampling, beam search, requests behind one system prompt).  The same arguments plus shared_prefix_len (>= 0, else
 *   SAB_ERR_INVALID before any launch) and the same workspace size.  Only whole chunks are shared: with C =
 *   sab_kvcache8_chunk_keys() and P = min(shared_prefix_len, max_pages * page_size), P' = (P / C) * C; P' = 0 runs
 *   sab_kvcache8_attn's kernels.  Promise (trusted, as table entries are): keys j < P' of every sequence are the same tokens,
 *   stored in the pages block_table[0 .. P' / page_size - 1] name; row 0 is the only table row read for a shared chunk.
 *   Chunk c < P' / C of sequence b goes to a shared CTA iff Lq_b >= 1 and (c + 1) * C <= Lk_b (non-causal) or
 *   (c + 1) * C <= Lk_b - Lq_b + 1 (causal), decided on the device (no host synchronisation); such a CTA holds the rows of
 *   S = 64 / (max_seqlen_q * Hq / Hkv) sequences and writes each row's partial for the chunk with the arithmetic of that row's
 *   own CTA.  Every other chunk runs as in sab_kvcache8_attn.  Where the promise holds, out and lse are bit for bit those of
 *   sab_kvcache8_attn.  Launch-grid limits: those of sab_kvcache8_attn, and nseq * ceil(max_pages * page_size / C) +
 *   ceil(nseq / S) * P' / C < 2^31. */
int sab_kvcache8_attn_shared(const void* q, int dtype, const int8_t* k_pages, const float* k_scale, const uint8_t* v_pages,
                             const float* v_scale, const float* k_smooth, void* out, float* lse, const int32_t* cu_seqlens_q,
                             const int32_t* seqused_k, const int32_t* block_table, int64_t table_stride, int max_pages, int nseq,
                             int Tq, int Hq, int Hkv, int D, int page_size, int64_t q_stride_t, int64_t q_stride_h,
                             int64_t o_stride_t, int64_t o_stride_h, int max_seqlen_q, int is_causal, float sm_scale,
                             void* workspace, int shared_prefix_len, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SAGEATTN_B200_H_ */
