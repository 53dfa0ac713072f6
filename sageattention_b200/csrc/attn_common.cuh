// Shared declarations of the attention kernel (attn.cu).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <type_traits>
#include "common.cuh"
#include "ptx.cuh"

namespace sab {

constexpr int BM = 128;  // Q rows per CTA
constexpr int BN = 64;   // keys per softmax / MMA tile (reference CTA_K)
constexpr int LK = 128;  // keys per TMA stage (two tiles)
constexpr float kFp8Offset = 8.807f;      // attn_utils.cuh:30
constexpr float kMaskValue = -5000000.0f; // attn_utils.cuh:310
constexpr int kIntSentinel = -(1 << 30);
struct AttnParams {
  const float* q_scale;
  const float* k_scale;
  const float* v_scale;  // nullable
  const float* v_mean;   // nullable
  void* out;
  float* lse;  // nullable
  int64_t o_stride_b, o_stride_h, o_stride_s;
  int B, Hq, Hkv, Sq, Sk;
  int n_q_tiles;
  int causal;
  float sm_scale_log2;
  int q_mult;            // scales per 128-row Q block: 1 / 4 / 32
  int q_gran;            // 1 / 2 / 3
  int k_mult;            // scales per 64-key block: 1 / 4
  int64_t qs_stride_bh;  // dense: scales per (b,h); varlen: unused
  int64_t ks_stride_bh;
  int qs_stride_idx;     // dense 1, varlen Hq
  int ks_stride_idx;     // dense 1, varlen Hkv
  const int32_t* cu_q;   // varlen (nullable)
  const int32_t* cu_k;
  const int32_t* cu_v;
  const int32_t* cu_qs;
  const int32_t* cu_ks;
  int causal_q_offset;   // global index of query row 0 (sequence-parallel causal)
  int kv_seg_len;        // > 0: K/V are rank-major all-gathered segments of this many keys
  float lazy_tau;        // INT8+FP8 path: the running max moves only by more than this many binades (0: exact max)
  // attention mask of the Triton-path shell (attn_qk_int8_per_block.py:33-52): [B,Hq,Sq,Skv] with arbitrary (also 0) strides
  const void* mask;      // nullable
  int mask_kind;         // 1: bool (uint8, false = masked out), 2: additive bias in the output dtype (fp16 / bf16)
  int64_t mask_sb, mask_sh, mask_sm, mask_sn;   // element strides
  // sequence-parallel gather fused into the launch (seg_flags != nullptr): K/V segment `seg` of KV-head group g is complete in
  // this GPU's memory once seg_flags[g * n_segments + seg] == seg_epoch (written in stream order behind the peer copies)
  const uint32_t* seg_flags;   // nullable
  uint32_t seg_epoch;
  int seg_heads;               // KV heads per flag group
};

// ---- logits of the INT8 path.  The forward (attn.cu) and the backward (attn_bwd.cu) both evaluate them with these helpers: the
// backward's P must be the forward's P, so the dequantised logit has one definition.
// Dequant scale of Q row `row` (0..127) of 128-row scale block `blk`, times sm_scale*log2e (1 when folded into q)
// (…sm89.cuh:98-114).
__device__ __forceinline__ float q_dequant_log2(const AttnParams& p, const float* qs_base, int blk, int row) {
  int q_idx = blk * p.q_mult;
  if (p.q_gran == SAB_GRAN_PER_WARP) q_idx += row >> 5;
  if (p.q_gran == SAB_GRAN_PER_THREAD) q_idx += (row >> 5) * 8 + (row & 7);
  return qs_base[int64_t(q_idx) * p.qs_stride_idx] * p.sm_scale_log2;
}
// Dequant scale of 64-key block `blk`; per-thread K scales (kKT): of scale group `grp` = keys 8i+2grp, 8i+2grp+1 (…sm89.cuh:116-132).
template <bool kKT>
__device__ __forceinline__ float k_dequant(const AttnParams& p, const float* ks_base, int blk, int grp) {
  return ks_base[int64_t(blk * (kKT ? 4 : 1) + (kKT ? grp : 0)) * p.ks_stride_idx];
}
// S * coef - m in log2 units for an int32 logit S, coef = k_dequant * q_dequant_log2.  I2FP is exact (|S| < 2^24) and the FMA is
// the reference's fmaf(S, sm_scale', -m) (attn_utils.cuh:450).
__device__ __forceinline__ float logit_log2(uint32_t s, float coef, float neg_m) {
  return fmaf(__int2float_rn(int(s)), coef, neg_m);
}

__device__ __forceinline__ void mbar_wait_wd(uint64_t* bar, uint32_t parity) {
#ifdef SAB_WATCHDOG
  // Debug build: bounded spin.  A wait that never completes reports itself (block 0 only) and is ABANDONED, so the kernel
  // runs to the end with wrong results instead of hanging the GPU, and the printf buffer is flushed.
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 22)) {
      if (blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0 && (threadIdx.x & 31) == 0)
        printf("sab: mbarrier timeout warp %d bar@%u parity %u\n", threadIdx.x >> 5, smem_u32(bar) & 0xfffu, parity);
      break;
    }
  }
#else
  mbar_wait(bar, parity);
#endif
}

// ---- attention mask of the masked entries (sab_qk_int8_sv_f16_attn_masked / sab_qk_int8_attn_bwd_masked): AttnParams::mask,
// mask_kind and the mask_s* strides
struct MaskArgs {
  const void* ptr; int kind; int64_t sb, sh, sm, sn;
};

// ---- block-sparse attention (sab_qk_int8_sv_f8_attn_blocksparse / sab_qk_int8_attn_bwd_blocksparse).  A kernel argument, not an
// AttnParams field, so the parameter offsets of the other kernels do not move.
struct BlockMask {
  const uint8_t* ptr;              // bool [Bm,Hm,ceil(Sq/128),ceil(Skv/64)]: key block j visible to 128-row Q block i of head h
  int64_t sb, sh, sqb, skb;        // element strides, 0 for a broadcast dimension
};
// Each visible key block costs one 2-byte entry of shared memory in the kernels that compact a mask row (build_kv_list).
constexpr int kMaxKvBlocks = 16384;                        // Skv <= 16384 * 64 = 1048576 keys
constexpr size_t kv_list_bytes(int n_blocks) { return 64 + (size_t(n_blocks) * 2 + 15) / 16 * 16; }   // + per-warp counts

// Ascending indices j < n of the visible 64-key blocks of mask row (b, h, qb) into list, by all NT threads of the CTA (uniform
// control flow: it synchronises the CTA); returns their count to every thread.  scratch: 64 bytes of shared memory.
template <int NT>
__device__ __forceinline__ int build_kv_list(const BlockMask& m, int b, int h, int qb, int n, uint16_t* list, int* scratch) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint8_t* row = m.ptr + int64_t(b) * m.sb + int64_t(h) * m.sh + int64_t(qb) * m.sqb;
  int total = 0;
  for (int base = 0; base < n; base += NT) {
    const int j = base + int(threadIdx.x);
    const bool vis = j < n && __ldg(row + int64_t(j) * m.skb) != 0;
    const uint32_t bal = __ballot_sync(0xffffffffu, vis);
    if (lane == 0) scratch[warp] = __popc(bal);
    __syncthreads();
    int pos = total + __popc(bal & ((1u << lane) - 1u));
    for (int w = 0; w < NT / 32; ++w) {
      if (w < warp) pos += scratch[w];
      total += scratch[w];
    }
    if (vis) list[pos] = uint16_t(j);
    __syncthreads();   // the list is complete and scratch may be rewritten
  }
  return total;
}

// Host: the block-sparse entries' checks of the mask arguments, before anything touches the device (forward and backward)
inline int check_block_mask(const void* block_mask, int64_t sb, int64_t sh, int64_t sqb, int64_t skb, int q_gran, int is_causal,
                            int Sq, int Skv) {
  SAB_REQUIRE(block_mask != nullptr, SAB_ERR_INVALID, "block_mask: null pointer");
  SAB_REQUIRE(sb >= 0 && sh >= 0 && sqb >= 0 && skb >= 0, SAB_ERR_INVALID, "block_mask strides must be >= 0 (0 broadcasts)");
  SAB_REQUIRE(q_gran == SAB_GRAN_PER_WARP || q_gran == SAB_GRAN_PER_THREAD, SAB_ERR_UNSUPPORTED,
              "the block-sparse path needs per-warp or per-thread Q scales (q_gran %d)", q_gran);
  SAB_REQUIRE(!is_causal || Sq == Skv, SAB_ERR_INVALID, "qo_len and kv_len must be equal for causal attention.");
  SAB_REQUIRE(Skv <= kMaxKvBlocks * BN, SAB_ERR_UNSUPPORTED, "the block-sparse path supports kv_len <= %d (got %d)",
              kMaxKvBlocks * BN, Skv);
  return SAB_OK;
}

// Host: the packed block-sparse entries' checks (sab_qk_int8_sv_f8_attn_varlen_blocksparse / sab_qk_int8_attn_bwd_varlen_blocksparse):
// those of check_block_mask, except that causal is top-left inside each sequence and needs no Lq == Lk, and that the key limit
// applies to max_seqlen_k (it sizes each CTA's list of visible key blocks), not to the packed total.
inline int check_block_mask_varlen(const void* block_mask, int64_t sb, int64_t sh, int64_t sqb, int64_t skb, int q_gran, int max_q,
                                   int max_k) {
  SAB_REQUIRE(block_mask != nullptr, SAB_ERR_INVALID, "block_mask: null pointer");
  SAB_REQUIRE(sb >= 0 && sh >= 0 && sqb >= 0 && skb >= 0, SAB_ERR_INVALID, "block_mask strides must be >= 0 (0 broadcasts)");
  SAB_REQUIRE(q_gran == SAB_GRAN_PER_WARP || q_gran == SAB_GRAN_PER_THREAD, SAB_ERR_UNSUPPORTED,
              "the block-sparse path needs per-warp or per-thread Q scales (q_gran %d)", q_gran);
  SAB_REQUIRE(max_q > 0 && max_k > 0, SAB_ERR_INVALID, "the packed block mask needs max_seqlen_q and max_seqlen_k > 0 (got %d, %d)",
              max_q, max_k);
  SAB_REQUIRE(max_k <= kMaxKvBlocks * BN, SAB_ERR_UNSUPPORTED, "the block-sparse path supports max_seqlen_k <= %d (got %d)",
              kMaxKvBlocks * BN, max_k);
  return SAB_OK;
}

// ---- sliding-window attention (sab_qk_int8_sv_f8_attn_window / sab_qk_int8_attn_bwd_window).  A kernel argument, not an
// AttnParams field, so the parameter offsets of the other kernels do not move.
struct Window {
  int left, right;                 // key j visible to query i iff i - left <= j <= i + right (top-left); -1: that side unbounded
};

// Window::right of the packed bottom-right causal form (sab_qk_int8_sv_f8_attn_varlen_kvcache), as handed to the launch: sequence
// b's right side is Lk_b - Lq_b.  That side may be negative and is never unbounded, so the kernel derives it per sequence under
// its own flag (kBR) and reads it with kRightBounded below; this value only selects that kernel.
constexpr int kWindowBottomRight = -(1 << 30);

// The 64-key tiles [j_lo, j_hi) that hold a key visible to some row of [r_lo, r_hi] (r_hi inclusive): the window, the causal
// horizon and kv_len.  Empty (j_lo == j_hi) when no row of the range sees any key.  kRightBounded: w.right bounds the right side
// whatever its sign (a negative right side hides keys up to |right| before the row's own position).
template <bool kRightBounded = false>
__device__ __forceinline__ void window_tiles(const Window& w, bool causal, int r_lo, int r_hi, int kv_len, int& j_lo, int& j_hi) {
  const int k_lo = w.left < 0 ? 0 : max(0, r_lo - w.left);
  int k_hi = kv_len - 1;
  if (kRightBounded || w.right >= 0) k_hi = min(k_hi, r_hi + w.right);
  if (causal) k_hi = min(k_hi, r_hi);
  j_lo = k_lo / BN;
  j_hi = k_hi >= k_lo ? k_hi / BN + 1 : j_lo;
}

// Host: the window entries' checks, before anything touches the device (forward and backward).  A side that reaches past every
// row (left >= Sq) or every key (right >= Skv) is set to -1: the same visibility, and the kernels' index arithmetic then stays
// below Sq + Skv.
inline int check_window(int& left, int& right, int is_causal, int Sq, int Skv) {
  SAB_REQUIRE(left >= -1 && right >= -1, SAB_ERR_INVALID, "window_size sides must be >= -1 (-1: unbounded), got (%d, %d)", left,
              right);
  SAB_REQUIRE(!is_causal || Sq == Skv, SAB_ERR_INVALID, "qo_len and kv_len must be equal for causal attention.");
  if (left >= Sq) left = -1;
  if (right >= Skv) right = -1;
  return SAB_OK;
}

// Host: the packed window entries' checks (sab_qk_int8_sv_f8_attn_varlen_window / sab_qk_int8_attn_bwd_varlen_window).  Causal is
// top-left inside each sequence and needs no Lq == Lk.  A side is clamped at the longest sequence (max_q rows, max_k keys) so
// that the kernels' index arithmetic stays in int32; each kernel then clamps it again at its own sequence's lengths
// (seq_window), which is what the dense entry does for that sequence alone.
inline int check_window_varlen(int& left, int& right, int max_q, int max_k) {
  SAB_REQUIRE(left >= -1 && right >= -1, SAB_ERR_INVALID, "window_size sides must be >= -1 (-1: unbounded), got (%d, %d)", left,
              right);
  SAB_REQUIRE(max_q > 0 && max_k > 0, SAB_ERR_INVALID, "the packed window needs a query bound and a key bound > 0 (got %d, %d)",
              max_q, max_k);
  if (left >= max_q) left = -1;
  if (right >= max_k) right = -1;
  return SAB_OK;
}

// Device: the window a packed sequence of q_len rows and kv_len keys sees, clamped as check_window clamps it for the dense call
// on that sequence.  The clamp keeps the visibility and decides which tiles take the masked path (tile_setup in attn.cu).
__device__ __forceinline__ Window seq_window(const Window& w, int q_len, int kv_len) {
  return Window{w.left >= q_len ? -1 : w.left, w.right >= kv_len ? -1 : w.right};
}

// Host: opt a kernel into its dynamic shared-memory size once PER DEVICE (cudaFuncSetAttribute applies to the current
// device only; a process that drives several GPUs — sageattn_host(device=...), tests — must set it on each).
template <typename Kern>
inline int ensure_dynamic_smem(Kern kern, size_t smem, bool (&done)[64]) {
  int dev = 0;
  SAB_CUDA_OK(cudaGetDevice(&dev));
  const bool tracked = dev >= 0 && dev < 64;
  if (!tracked || !done[dev]) {
    SAB_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
    if (tracked) done[dev] = true;
  }
  return SAB_OK;
}

template <typename T>
__device__ __forceinline__ uint32_t pack2(float a, float b);
template <>
__device__ __forceinline__ uint32_t pack2<__half>(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}
template <>
__device__ __forceinline__ uint32_t pack2<__nv_bfloat16>(float a, float b) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}


}  // namespace sab
