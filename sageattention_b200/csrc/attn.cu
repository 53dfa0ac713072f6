// Fused INT8-QK attention for sm_90a (H100): INT8 QK^T -> fp32 online softmax -> FP8 (or FP16) P -> PV, all products on the
// warpgroup tensor core (wgmma) with register accumulators.
//
// Serves (a) the INT8+FP8 path (sageattn_qk_int8_pv_fp8_cuda and everything built on it) and (b) the FP16-PV numerics of the
// reference's Triton kernels (kPV16: sageattn_varlen, sageattn_qk_int8_pv_fp16_triton incl. attn_mask,
// sageattn_qk_int8_pv_fp16_cuda).  One CTA = one 128-row Q tile of one (batch, head), 384 threads (the dense INT8+FP8 kernel at
// D = 128: one 192-row tile, 512 threads, a third consumer warpgroup; see kNC below):
//   warps 0-3 / 4-7 : two consumer warpgroups, 64 Q rows each.  Per 64-key tile: S = Q K^T (wgmma s8, int32 accumulators in
//                     registers), online softmax in registers, P (e4m3 or f16) handed to the PV wgmma as its register A operand,
//                     O (fp32, 64 x D) accumulated in registers.  The loop is rotated so that each warpgroup issues PV(j-1)
//                     and QK(j) as one tensor-core phase per tile, and the two warpgroups ping-pong: named barriers hand the
//                     turn to issue from one to the other, so one's softmax runs while the other's MMAs are on the tensor cores.
//                     The loop is bound by each warpgroup's serial path (phase, then softmax), not by the tensor cores, so at
//                     D = 128 softmax(j) starts when QK(j) is done and runs under PV(j-1): a step at hd=128, S=8192 went from
//                     1693 to 1555 cycles (H100 SXM, 700 W; -DSAB_PHASE_CLOCKS, tools/phase_clocks.py).
//   warp 8          : TMA producer (Q once; K and V^T 64-key tiles through a kStages-deep mbarrier ring, swizzled smem);
//                     warps 9-11 only hand their registers over (setmaxnreg: 24 for the producer warpgroup, 240 for consumers).
// The softmax / MMA tile is 64 keys — the reference's CTA_K — so the running-max sequence, P and d follow
// csrc/qattn/qk_int_sv_f8_cuda_sm89.cuh: base-2 online softmax, -8.807 exponent offset so P fills (0,448], d from un-rounded fp32
// P, top-left causal alignment, rcp/lg2/ex2 .approx.  FP8 PV is accumulated in two levels: each tile's product starts from zero in
// the tensor core and is added to O in fp32 on the CUDA cores (Hopper's FP8 wgmma keeps fewer accumulator bits than fp32, so a
// long accumulation inside the tensor core drifts; the reference's sm90 kernel does the same).  FP16 PV accumulates in place.
// Running max of the INT8+FP8 path: LAZY by default (lazy_tau = 4 binades): the max moves only when an element of the tile would
// overflow e4m3 (P > 448); when it moves, the new row maximum is placed tau binades below 448 (exponent offset 8.807 - tau), so O
// is rarely rescaled.  P keeps e4m3's relative precision; it is a different rounding realisation than the reference kernel's (same
// accuracy against exact attention, tests/test_gpu_parity.py).  SAB_ATTN_KERNEL=exact selects the reference's exact running max
// (lazy_tau = 0): P, m and d are then the reference kernel's.
#include <cstdlib>
#include "attn_common.cuh"

namespace sab {

// kNC consumer warpgroups of 64 Q rows each: 2 (a 128-row Q tile), or 3 (192 rows) in the dense INT8+FP8 kernel at D = 128
template <int kNC>
constexpr int kNumThreads = (kNC + 1) * 128;   // + the producer warpgroup (one TMA warp; setmaxnreg is per warpgroup)
constexpr int kStages = 6;                     // K / V^T ring depth (64-key tiles)

template <int D, bool kPV16, int kNC = 2>
constexpr size_t attn_smem_bytes() {
  return size_t(kNC * 64) * D + size_t(kStages) * (BN * D + BN * D * (kPV16 ? 2 : 1)) + (1 + 2 * kStages) * 8 + 1024;
}

// Shared memory of the block-sparse form behind the INT8+FP8 kernel's barriers: build_kv_list's 64 bytes of counts, then the list
// of visible 64-key tiles (kv_list_bytes)
template <int D>
constexpr uint32_t kKvScratchOff = uint32_t(BM) * D + kStages * (2 * BN * D) + (1 + 2 * kStages) * 8;
template <int D>
__device__ __forceinline__ int* kv_scratch(uint8_t* smem) { return reinterpret_cast<int*>(smem + kKvScratchOff<D>); }
template <int D>
__device__ __forceinline__ uint16_t* kv_list(uint8_t* smem) { return reinterpret_cast<uint16_t*>(smem + kKvScratchOff<D> + 64); }

// Per-phase cycle counts of the consumer loop, for measurement builds only (-DSAB_PHASE_CLOCKS; tools/phase_clocks.py reads
// them).  Each consumer warpgroup sums clock64() spans over its main-loop steps j >= 1 (PV(j-1) + QK(j)): from taking its turn
// to the end of the wait for S(j) (the tensor-core phase, including any wait behind the other warpgroup's phase; at D = 128 it
// ends when QK(j) is done), and from there to the end of the fold + softmax; the whole loop is timed as well.  The sums over all warpgroups of a launch are added to
// g_phase_clk: {phase cycles, fold + softmax cycles, loop cycles, steps, warpgroups}.  The product build compiles none of it.
#ifdef SAB_PHASE_CLOCKS
__device__ unsigned long long g_phase_clk[5];
struct PhaseClocks {
  long long mma = 0, soft = 0, loop0 = 0, t = 0;
  int n = 0;
  __device__ __forceinline__ void loop_start() { loop0 = clock64(); }
  __device__ __forceinline__ void turn() { t = clock64(); }
  __device__ __forceinline__ void mma_done() { const long long c = clock64(); mma += c - t; t = c; ++n; }
  __device__ __forceinline__ void soft_done() { soft += clock64() - t; }
  __device__ __forceinline__ void flush() {
    const long long loop = clock64() - loop0;
    if ((threadIdx.x & 127) == 0 && n > 0) {
      atomicAdd(&g_phase_clk[0], (unsigned long long)mma);
      atomicAdd(&g_phase_clk[1], (unsigned long long)soft);
      atomicAdd(&g_phase_clk[2], (unsigned long long)loop);
      atomicAdd(&g_phase_clk[3], (unsigned long long)n);
      atomicAdd(&g_phase_clk[4], 1ull);
    }
  }
};
#else
struct PhaseClocks {
  __device__ __forceinline__ void loop_start() {}
  __device__ __forceinline__ void turn() {}
  __device__ __forceinline__ void mma_done() {}
  __device__ __forceinline__ void soft_done() {}
  __device__ __forceinline__ void flush() {}
};
#endif

// D: head dim (64 / 128).  kKT: per-thread K scales (4 per 64-key block) instead of 1.  OutT: __half / bf16.
// kPV16: P and V in fp16 with the Triton path's softmax (no exponent offset) — the numerics of the reference's
// sageattn_qk_int8_pv_fp16_triton / sageattn_varlen kernels (triton/attn_qk_int8_per_block.py:22-128).
// kMask with kPV16: attn_mask of sageattn_qk_int8_pv_fp16_triton — a bool mask marks elements like the out-of-range keys
// (integer sentinel), an additive bias takes the float path below.
// Sequence-parallel fused gather (p.seg_flags != nullptr): K/V segments arrive WHILE the kernel runs (peer copies on another
// stream); the TMA producer polls one flag per (KV-head group, segment) before the first tile of a segment.
// the two meanings of kMask (namespace-scope, not kernel locals: a local constexpr perturbs the code ptxas emits for the kernel)
template <bool kPV16, bool kMask>
constexpr bool kElemMask = kMask && kPV16;    // attn_mask of the FP16-PV path
template <bool kPV16, bool kMask>
constexpr bool kSparse = kMask && !kPV16;     // block mask of the INT8+FP8 path

// kMask without kPV16 (INT8+FP8 only): the block-sparse form.  p.mask is then the bool block mask [.,.,ceil(Sq/128),ceil(Skv/64)]
// with element strides mask_sb / mask_sh / mask_sm (128-row Q blocks) / mask_sn (64-key blocks), and the dynamic shared memory
// adds kv_list_bytes(ceil(Skv/64)).  The CTA first compacts its row (b, h, qt) of the mask into a shared-memory list of the visible
// 64-key tiles, ascending and cut at the causal horizon; the loop below then runs over that list, with tile kv_list[j] wherever the
// dense kernel uses tile j (TMA coordinates, K-scale block, limit, masked_tile).  A row whose list is empty takes the n_kv == 0
// path; a row that sees none of the listed keys (causal) gets zeros and lse -inf.
// kWindow (INT8+FP8 only, dense): the sliding-window form; win holds the window (unused by the other forms).  The CTA's rows see
// the 64-key tiles [j0, j0 + n_kv) (window_tiles), and step j runs tile j0 + j wherever the dense kernel uses tile j.  Each row
// part has a lower bound lo next to limit (visible keys of the tile: lo <= key < limit), and every tile that crosses either edge
// of the window for some row of the CTA takes the masked path.  A row part that sees nothing of a tile keeps m and d (its
// maximum is the mask value, so the lazy max does not move) and adds P = 0, also before its first visible tile; a row that sees
// no key at all gets zeros and lse -inf.
// kSeqV (INT8+FP8 only, varlen): per-sequence V statistics, v_scale / v_mean [nseq,Hkv,D] indexed by the sequence, where the other
// varlen forms read one [Hkv,D] table for the whole packed batch.
// kWindow with kSeqV: the packed window form.  Each sequence sees the window clamped at its own lengths (seq_window), so its rows
// take the dense window kernel's path on that sequence alone, tile for tile.
// kMask (block-sparse) with kSeqV: the packed block-sparse form.  b is the sequence and qt its own Q tile, so the CTA compacts mask
// row (b, h, qt) of a [nseq,Hq,ceil(max_seqlen_q/128),ceil(max_seqlen_k/64)] mask, cut at its sequence's n_kv and causal horizon:
// the dense block-sparse kernel's path on that sequence alone.
// kBR with kWindow and kSeqV: the packed bottom-right causal form.  Sequence b's rows see the window (-1, Lk_b - Lq_b), derived
// here instead of read from win_arg: the window kernel's path on that window, tile for tile.  The right side may be negative
// (Lk_b < Lq_b: the first Lq_b - Lk_b rows see no key) and always bounds, so it is read as bounded whatever its sign.
// kNC = 3 (dense INT8+FP8 at D = 128 only): three consumer warpgroups on a 192-row Q tile, so each SM sub-partition has more
// independent warps to hide the softmax's latency, and each K/V tile serves 192 rows.  160 registers per consumer thread hold
// O (64) but not a 64-register tile product next to S: the FP8 PV runs as two m64n64 halves into 32 registers, each folded
// into O before the next (a column's product does not depend on N, so O is the same to the bit), and softmax(j) runs under
// the second half.  The turn passes round the three warpgroups (see the main loop).  At 160 registers ptxas keeps three values
// (a turn barrier id and the two rows' Q scales) in 12 bytes of local memory, reloaded once per 64-key step.
template <int D, bool kKT, typename OutT, bool kPV16, bool kMask = false, bool kWindow = false, bool kSeqV = false, bool kBR = false,
          int kNC = 2>
__global__ void __launch_bounds__(kNumThreads<kNC>, 1)
sage_attn_fwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                     const __grid_constant__ CUtensorMap tmV, const __grid_constant__ AttnParams p,
                     const __grid_constant__ Window win_arg) {
  constexpr uint32_t K_TILE = BN * D;
  constexpr uint32_t V_TILE = D * BN * (kPV16 ? 2 : 1);
  constexpr int SWQK = D;                        // swizzle span of the Q/K tiles (= row bytes)
  constexpr int SWV = kPV16 ? 128 : 64;          // V^T rows: 64 keys = 64 B (fp8) / 128 B (fp16)
  static_assert(kNC == 2 || (kNC == 3 && D == 128 && !kPV16 && !kMask && !kWindow && !kSeqV), "three consumers: dense INT8+FP8, D = 128");
  constexpr int QM = kNC * 64;                   // Q rows per CTA
  constexpr uint32_t Q_BYTES = QM * D;
  constexpr int NO = D / 2;                      // fp32 O accumulators per thread (64 x D over 128 threads)
  constexpr bool kHalfPV = kNC == 3;             // the FP8 PV as two m64n64 halves (see above)

  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + Q_BYTES;
  uint8_t* sV = sK + kStages * K_TILE;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + kStages * V_TILE);
  uint64_t* q_full = bars;
  uint64_t* kv_full = bars + 1;                  // [kStages] TMA bytes landed (K + V^T tile)
  uint64_t* kv_empty = kv_full + kStages;        // [kStages] both consumer warpgroups finished with the slot

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  // ---------------- work decode (uniform across the CTA)
  int qt = blockIdx.x;
  if (p.causal || kBR) qt = p.n_q_tiles - 1 - qt;  // heaviest tiles first
  const int h = blockIdx.y;
  const int b = blockIdx.z;
  const int hk = h / (p.Hq / p.Hkv);
  const bool varlen = p.cu_q != nullptr;
  int q_len = p.Sq, kv_len = p.Sk, q_off = 0, k_off = 0, v_off = 0, tb = b;
  int q_blk0 = 0, k_blk0 = 0;  // first 128-row / 64-key scale block of this sequence
  if (varlen) {
    q_off = p.cu_q[b];
    q_len = p.cu_q[b + 1] - q_off;
    k_off = p.cu_k[b];
    kv_len = p.cu_k[b + 1] - k_off;
    v_off = p.cu_v[b];
    q_blk0 = p.cu_qs[b];
    k_blk0 = p.cu_ks[b];
    tb = 0;
    if (qt * QM >= q_len) return;  // attn_qk_int8_block_varlen.py:84-85
  }
  // the packed window form reads its sequence's clamped copy; every other form reads the kernel argument itself
  [[maybe_unused]] Window seq_win;
  if constexpr (kWindow && kSeqV) seq_win = kBR ? Window{-1, kv_len - q_len} : seq_window(win_arg, q_len, kv_len);
  const Window& win = (kWindow && kSeqV) ? seq_win : win_arg;
  int n_kv = (kv_len + BN - 1) / BN;                 // 64-key tiles
  if (p.causal) n_kv = min(n_kv, (p.causal_q_offset + (qt + 1) * QM + BN - 1) / BN);
  if constexpr (kSparse<kPV16, kMask>) {
    const BlockMask bm{static_cast<const uint8_t*>(p.mask), p.mask_sb, p.mask_sh, p.mask_sm, p.mask_sn};
    n_kv = build_kv_list<kNumThreads<kNC>>(bm, b, h, qt, n_kv, kv_list<D>(smem), kv_scratch<D>(smem));
  }
  [[maybe_unused]] int j0 = 0;   // window form: the first 64-key tile of the CTA's range
  if constexpr (kWindow) {
    int j1;
    window_tiles<kBR>(win, p.causal != 0, qt * QM, min(qt * QM + QM, q_len) - 1, kv_len, j0, j1);
    n_kv = j1 - j0;
  }

  if (threadIdx.x == 0) {
    if ((smem_u32(smem) & 1023u) != 0) __trap();     // swizzled tiles need a 1 KB-aligned base
    mbar_init(q_full, 1);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(kv_full + i, 1);
      mbar_init(kv_empty + i, kNC);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >= kNC * 4) {
    // =============================== TMA producer ===============================
    setmaxnreg_dec<24>();
    if (warp == kNC * 4 && lane == 0 && n_kv > 0) {
      tma_prefetch_desc(&tmQ);
      tma_prefetch_desc(&tmK);
      tma_prefetch_desc(&tmV);
      mbar_expect_tx(q_full, Q_BYTES);
      tma_load_4d(sQ, &tmQ, q_full, 0, q_off + qt * QM, h, tb);   // the host's Q box is QM rows
      int ready_seg = -1;
      for (int j = 0; j < n_kv; ++j) {
        const int s = j % kStages;
        const uint32_t ph = (j / kStages) & 1;
        int kj = j;   // the 64-key tile loaded in step j
        if constexpr (kSparse<kPV16, kMask>) kj = kv_list<D>(smem)[j];
        if constexpr (kWindow) kj = j0 + j;
        int kc = k_off + kj * BN, vc = v_off + kj * BN, kb = tb;
        if (p.kv_seg_len > 0) {  // all-gathered layout: segment-major
          const int seg = (j * BN) / p.kv_seg_len;
          kc = vc = j * BN - seg * p.kv_seg_len;
          kb = seg * p.B + b;
          if (p.seg_flags != nullptr && seg != ready_seg) {
            // first tile of a segment: has the peer copy of this (head group, segment) landed?
            const uint32_t* flag = p.seg_flags + (hk / p.seg_heads) * (p.Sk / p.kv_seg_len) + seg;
            const long long t0 = clock64();
            while (ld_acquire_sys_u32(flag) != p.seg_epoch) {
              __nanosleep(200);
              if (clock64() - t0 > (8ll << 30)) __trap();   // ~4 s: the copies never came; fail the launch instead of hanging
            }
            fence_proxy_async_all();
            ready_seg = seg;
          }
        }
        mbar_wait_wd(kv_empty + s, ph ^ 1);
        mbar_expect_tx(kv_full + s, K_TILE + V_TILE);
        tma_load_4d(sK + s * K_TILE, &tmK, kv_full + s, 0, kc, hk, kb);
        tma_load_4d(sV + s * V_TILE, &tmV, kv_full + s, vc * (kPV16 ? 2 : 1), 0, hk, kb);   // byte coordinate
      }
    }
    return;
  }

  // =============================== consumer warpgroups ===============================
  setmaxnreg_inc<kNC == 2 ? 240 : 160>();   // 3 x 128 x 160 + 128 x 24 = 64512 of the SM's 65536
  // wgmma accumulator layout (m64nN): warp w of the warpgroup owns rows 16w..16w+15; lane = 4 g + t holds rows 16w+g (registers
  // 4i, 4i+1) and 16w+g+8 (4i+2, 4i+3) at columns 8i+2t, 8i+2t+1.  A row is spread over the 4 lanes of a quad.
  const int wg = warp >> 2;
  const int t = lane & 3;
  const int row0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // rows row0 and row0 + 8 of the Q tile
  int q_row[2];
  float qss[2];
  const float* qs_base = p.q_scale + (varlen ? int64_t(h) : (int64_t(b) * p.Hq + h) * p.qs_stride_bh);
  const float* ks_base = p.k_scale + (varlen ? int64_t(hk) : (int64_t(b) * p.Hkv + hk) * p.ks_stride_bh);
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int row = row0 + 8 * i;
    q_row[i] = qt * QM + row;  // row index inside the sequence
    if constexpr (kNC == 2) {
      qss[i] = q_dequant_log2(p, qs_base, q_blk0 + qt, row);
    } else {
      // a 192-row tile covers parts of two 128-row scale blocks; a row past the end (never stored) reads the last row's scale,
      // which exists
      const int r = min(q_row[i], q_len - 1);
      qss[i] = q_dequant_log2(p, qs_base, q_blk0 + r / BM, r % BM);
    }
  }
  const float tau = p.lazy_tau;
  float m[2] = {kMaskValue, kMaskValue};   // running max (log2 units, includes the -8.807 offset on the fp8 path)
  float d[2] = {0.f, 0.f};                 // this thread's part of the running sum of fp32 P
  float o[NO];
#pragma unroll
  for (int i = 0; i < NO; ++i) o[i] = 0.f;

  const uint64_t dQ = make_wgmma_desc<SWQK>(smem_u32(sQ + wg * 64 * D));
  const uint64_t dK0 = make_wgmma_desc<SWQK>(smem_u32(sK));
  const uint64_t dV0 = make_wgmma_desc<SWV>(smem_u32(sV));
  // P handed from the accumulator layout to the 8-bit A-operand layout (lane t of a quad holds keys 4t..4t+3 and 16+4t..16+4t+3
  // of each 32-key chunk): two 16-bit pairs from lanes 2(t&1) and 2(t&1)+1 of the quad, from block 0 or 1 of the chunk
  const int src0 = (lane & ~3) | ((t & 1) << 1);
  const uint32_t psel = (t >> 1) ? 0x7632u : 0x5410u;

  // ---- per-tile operands of the softmax, set before the tile's GEMM phase so the K-scale load overlaps it
  float coef[2];           // dequant coefficient of each row part
  int limit[2];            // number of visible keys of this tile per row (OOB + causal, attn_utils.cuh:296-351)
  [[maybe_unused]] int lo[2];   // window form: first visible key of this tile per row (keys lo <= key < limit are visible)
  bool masked_tile = false;
  auto tile_setup = [&](int j) {
    int kj = j;   // the 64-key tile of step j
    if constexpr (kSparse<kPV16, kMask>) kj = kv_list<D>(smem)[j];
    if constexpr (kWindow) kj = j0 + j;
    // dequant coefficient (…sm89.cuh:116-132, 255-257); tile kj == 64-key block kj.  Per-thread K scales: the keys of lane t
    // (8i+2t, 8i+2t+1) are all in scale group t.
    const float ksv = k_dequant<kKT>(p, ks_base, k_blk0 + kj, t);
    coef[0] = ksv * qss[0];
    coef[1] = ksv * qss[1];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      limit[i] = kv_len - kj * BN;
      if (p.causal) limit[i] = min(limit[i], p.causal_q_offset + q_row[i] - kj * BN + 1);
      if (kElemMask<kPV16, kMask> && q_row[i] >= q_len) limit[i] = 0;   // rows past the end: nothing visible, no mask bytes read
      if constexpr (kWindow) {
        if (kBR || win.right >= 0) limit[i] = min(limit[i], q_row[i] + win.right + 1 - kj * BN);
        lo[i] = win.left >= 0 ? q_row[i] - win.left - kj * BN : 0;
      }
    }
    masked_tile = kElemMask<kPV16, kMask> || (kv_len - kj * BN < BN) || (p.causal && (kj + 1) * BN > p.causal_q_offset + qt * QM + 1);
    if constexpr (kWindow) {
      // the top row's window ends inside the tile, or the bottom row's starts after its first key
      masked_tile = masked_tile || ((kBR || win.right >= 0) && (kj + 1) * BN - 1 > qt * QM + win.right) ||
                    (win.left >= 0 && kj * BN < qt * QM + QM - 1 - win.left);
    }
  };

  uint32_t s[32];                   // S of the tile in flight (int32)
  float alpha[2];                   // O rescale factor of the last softmax'd tile
  uint32_t a[kPV16 ? 4 : 2][4];     // P of the tile whose PV comes next, as the PV A operand
  constexpr int NOT = kHalfPV ? NO / 2 : NO;
  [[maybe_unused]] float ot[NOT];   // FP8 path: its P V (kHalfPV: one half of it), from zero

  // ---- S (registers, int32) -> P: running max m, sum d, rescale factor alpha, P as A fragments
  float e[32];                      // P of the last softmax in fp32, same register order as S
  auto softmax = [&](int j) {
    [[maybe_unused]] const char* mrow[2] = {nullptr, nullptr};   // this row's 64 mask elements of tile j
    if constexpr (kElemMask<kPV16, kMask>) {
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int64_t off = int64_t(b) * p.mask_sb + int64_t(h) * p.mask_sh + int64_t(q_row[i]) * p.mask_sm + int64_t(j) * BN * p.mask_sn;
        mrow[i] = reinterpret_cast<const char*>(p.mask) + off * (p.mask_kind == 1 ? 1 : 2);
        if (p.mask_kind == 1) {
#pragma unroll
          for (int c = 0; c < 16; ++c) {
            const int key = 8 * (c >> 1) + 2 * t + (c & 1);
            if (key < limit[i] && __ldg(reinterpret_cast<const uint8_t*>(mrow[i]) + int64_t(key) * p.mask_sn) == 0)
              s[4 * (c >> 1) + 2 * i + (c & 1)] = uint32_t(kIntSentinel);
          }
        }
      }
    }

    auto tile = [&](auto masked_tag) {
      constexpr bool MASKED = decltype(masked_tag)::value;
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        // ---- row max.  Scales are positive, so max_c(S_c*coef) = coef * max_c S_c: integer max, one conversion per row part
        int v = kIntSentinel;
#pragma unroll
        for (int c = 0; c < 16; ++c) {
          const int idx = 4 * (c >> 1) + 2 * i + (c & 1);
          if constexpr (MASKED && kWindow) {
            const int key = 8 * (c >> 1) + 2 * t + (c & 1);
            if (key >= limit[i] || key < lo[i]) s[idx] = uint32_t(kIntSentinel);
          } else if constexpr (MASKED) {
            if (8 * (c >> 1) + 2 * t + (c & 1) >= limit[i]) s[idx] = uint32_t(kIntSentinel);
          }
          v = max(v, int(s[idx]));
        }
        float mx = float(v) * coef[i];
        if constexpr (MASKED) mx = (v == kIntSentinel) ? kMaskValue : mx;
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
        float m_new;
        if constexpr (kPV16) {
          m_new = fmaxf(m[i], mx);                             // plain running max (Triton path)
        } else {
          // update_mdo with the -log2(448) offset (attn_utils.cuh:377-396); lazy: move only by more than tau binades
          const float m_true = fmaxf(m[i], mx - (kFp8Offset - tau));
          m_new = (m_true - m[i] > tau) ? m_true : m[i];
        }
        alpha[i] = (m_new != m[i]) ? ex2_approx(m[i] - m_new) : 1.0f;
        d[i] *= alpha[i];
        m[i] = m_new;
        // ---- P = exp2(S*coef - m_new), bit-identical to the reference kernel's at the same m (logit_log2)
        const float nm = -m_new;
        float sum = 0.f;
#pragma unroll
        for (int c = 0; c < 16; c += 2) {
          const int idx = 4 * (c >> 1) + 2 * i;
          const float y0 = logit_log2(s[idx], coef[i], nm), y1 = logit_log2(s[idx + 1], coef[i], nm);
          float x[2];
#ifdef SAB_POLY_EXP_PAIRS
          if (t < SAB_POLY_EXP_PAIRS) {   // column pair t of every 8 columns
            ex2_poly2(y0, y1, x[0], x[1]);
          } else {
            x[0] = ex2_approx(y0);
            x[1] = ex2_approx(y1);
          }
#else
          x[0] = ex2_approx(y0);
          x[1] = ex2_approx(y1);
#endif
#pragma unroll
          for (int u = 0; u < 2; ++u) {
            if constexpr (MASKED && kElemMask<kPV16, kMask>) x[u] = (int(s[idx + u]) != kIntSentinel) ? x[u] : 0.f;   // masked-out elements: not a prefix
            else if constexpr (MASKED && kWindow) x[u] = (8 * (c >> 1) + 2 * t + u < limit[i] && 8 * (c >> 1) + 2 * t + u >= lo[i]) ? x[u] : 0.f;
            else if constexpr (MASKED) x[u] = (8 * (c >> 1) + 2 * t + u < limit[i]) ? x[u] : 0.f;
            e[idx + u] = x[u];
            sum += x[u];
          }
        }
        d[i] += sum;
      }
    };
    // additive bias (attn_qk_int8_per_block.py:41,50-51): qk = S*scale + bias in fp32, then the plain online softmax
    auto tile_bias = [&]() {
      if constexpr (kElemMask<kPV16, kMask>) {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          float mx = -INFINITY;
#pragma unroll
          for (int c = 0; c < 16; ++c) {
            const int idx = 4 * (c >> 1) + 2 * i + (c & 1);
            const int key = 8 * (c >> 1) + 2 * t + (c & 1);
            float y = -INFINITY;
            if (key < limit[i]) {
              const float bias = float(__ldg(reinterpret_cast<const OutT*>(mrow[i]) + int64_t(key) * p.mask_sn));
              y = fmaf(__int2float_rn(int(s[idx])), coef[i], bias);
            }
            e[idx] = y;
            mx = fmaxf(mx, y);
          }
          mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
          mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
          const float m_new = fmaxf(m[i], mx);     // m starts at the finite mask value: never -inf
          alpha[i] = ex2_approx(m[i] - m_new);
          d[i] *= alpha[i];
          m[i] = m_new;
          float sum = 0.f;
#pragma unroll
          for (int c = 0; c < 16; ++c) {
            const int idx = 4 * (c >> 1) + 2 * i + (c & 1);
            e[idx] = ex2_approx(e[idx] - m_new);
            sum += e[idx];
          }
          d[i] += sum;
        }
      }
    };
    if (kElemMask<kPV16, kMask> && p.mask_kind == 2) tile_bias();
    else if (masked_tile) tile(std::true_type{});
    else tile(std::false_type{});

  };

  // ---- P -> A fragments of the PV operand.  Only once the PV that read a has completed.
  auto pack_p = [&]() {
    if constexpr (kPV16) {
      // k16 step kk: keys 16kk..16kk+15 = accumulator blocks 2kk, 2kk+1 (same layout: no exchange)
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        const int i0 = 8 * kk, i1 = 8 * kk + 4;
        a[kk][0] = pack_f16x2(e[i0], e[i0 + 1]);   // p.to(tl.float16), attn_qk_int8_per_block.py:62
        a[kk][1] = pack_f16x2(e[i0 + 2], e[i0 + 3]);
        a[kk][2] = pack_f16x2(e[i1], e[i1 + 1]);
        a[kk][3] = pack_f16x2(e[i1 + 2], e[i1 + 3]);
      }
    } else {
      // k32 chunk c: keys 32c..32c+31 = accumulator blocks 4c..4c+3
#pragma unroll
      for (int c = 0; c < 2; ++c) {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int b0 = 16 * c + 2 * i;   // register of block 4c, this row
          const uint32_t x = pack_e4m3x4(e[b0], e[b0 + 1], e[b0 + 4], e[b0 + 5]);         // blocks 4c, 4c+1
          const uint32_t y = pack_e4m3x4(e[b0 + 8], e[b0 + 9], e[b0 + 12], e[b0 + 13]);   // blocks 4c+2, 4c+3
          a[c][i] = __byte_perm(__shfl_sync(0xffffffffu, x, src0), __shfl_sync(0xffffffffu, x, src0 + 1), psel);
          a[c][2 + i] = __byte_perm(__shfl_sync(0xffffffffu, y, src0), __shfl_sync(0xffffffffu, y, src0 + 1), psel);
        }
      }
    }
  };

  // ---- rescale O (registers) by alpha of the tile whose PV comes next.  A separate rounding step, never contracted into an
  // FMA with the add of that tile's P V: O's per-element sequence is o *= alpha(j); o += PV(j); o *= alpha(j+1); ...
  auto rescale_o = [&]() {
    if (alpha[0] != 1.0f || alpha[1] != 1.0f) {
#pragma unroll
      for (int i = 0; i < NO; i += 4) {
        o[i] = __fmul_rn(o[i], alpha[0]);
        o[i + 1] = __fmul_rn(o[i + 1], alpha[0]);
        o[i + 2] = __fmul_rn(o[i + 2], alpha[1]);
        o[i + 3] = __fmul_rn(o[i + 3], alpha[1]);
      }
    }
  };
  auto issue_qk = [&](int j) {   // S = Q K(j)^T
    const uint64_t dK = dK0 + uint64_t(j % kStages) * (K_TILE >> 4);
#pragma unroll
    for (int k = 0; k < D / 32; ++k) wgmma_qk_i8(s, dQ + 2 * k, dK + 2 * k, k > 0);
  };
  auto issue_pv = [&](int j) {   // FP16: O += P V(j) in place (O already rescaled); FP8: ot = P V(j)
    const uint64_t dV = dV0 + uint64_t(j % kStages) * (V_TILE >> 4);
    if constexpr (kPV16) {
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) wgmma_pv_f16(o, a[kk], dV + 2 * kk, 1);
    } else {
#pragma unroll
      for (int c = 0; c < 2; ++c) wgmma_pv_f8(ot, a[c], dV + 2 * c, c > 0);
    }
  };
  auto finish_pv = [&](int j) {  // after the wait: fold the FP8 tile product into O, release slot j
    if constexpr (kPV16) {
      fence_regs(o);
    } else {
      fence_regs(ot);
#pragma unroll
      for (int i = 0; i < NOT; ++i) o[i] += ot[i];
    }
    if ((threadIdx.x & 127) == 0) mbar_arrive(kv_empty + j % kStages);   // K(j) and V(j) consumed by this warpgroup
  };
  // kHalfPV: ot = P V(j) for output columns 64 hh .. 64 hh + 63 (V^T rows from 64 hh: 64 rows of 64 B, a whole number of 64-B
  // swizzle atoms), and its fold into those columns of O
  auto issue_pv_half = [&](int j, int hh) {
    const uint64_t dV = dV0 + uint64_t(j % kStages) * (V_TILE >> 4) + uint64_t(hh) * ((64 * SWV) >> 4);
#pragma unroll
    for (int c = 0; c < 2; ++c) wgmma_pv_f8(ot, a[c], dV + 2 * c, c > 0);
  };
  auto fold_half = [&](int hh) {
    fence_regs(ot);
#pragma unroll
    for (int i = 0; i < NOT; ++i) o[NOT * hh + i] += ot[i];
  };

  // ---- main loop, rotated so each warpgroup has ONE tensor-core phase per tile: QK(j) and PV(j-1) issued back to back, then
  // softmax(j) and the fold of PV(j-1) into O on the CUDA cores.  At D = 128 the two products are separate commit groups, QK(j)
  // first, and softmax(j) starts as soon as QK(j) has completed, under PV(j-1) (an m64n128k32 pair, half the phase); O is folded
  // after it.  At D = 64 PV(j-1) is an m64n64k32 pair with little to hide, and one commit group measured faster (hd=64 rows of
  // bench.py 1.3 % slower with the split, H100 SXM, 700 W).  Either way O's per-element sequence is o *= alpha(j-1), then
  // o += PV(j-1) (softmax(j) does not touch O) and P(j) overwrites the PV operand a only after PV(j-1) has completed (pack_p),
  // so the output is the same to the bit.  The two warpgroups take turns at issuing their phases (named barrier 1 + wg is this
  // warpgroup's turn, arrived at by the other one right after its commit), so one's softmax runs while the other's MMAs are on
  // the tensor cores.  Each warpgroup has n_kv + 1 phases; warpgroup 1 hands the first turn to warpgroup 0 and skips the
  // hand-over after its last phase, so no arrival is left over at exit.  n_kv is uniform per CTA; with n_kv == 0 no barrier is
  // touched.  Slot j-1 is released one phase later than it was consumed; the ring absorbs it.
  constexpr bool kSoftmaxUnderPV = D == 128;
  constexpr uint32_t kTurnThreads = 2 * 128;
  const uint32_t my_turn = 1 + wg;
  [[maybe_unused]] const uint32_t their_turn = 2 - wg;   // two warpgroups
  PhaseClocks clk;
  clk.loop_start();
  if constexpr (kHalfPV) {
    // Three warpgroups: the turn goes round them (warpgroup w waits on barrier 1 + w and hands the turn to barrier
    // 1 + (w + 1) % 3, each barrier counting its owner and its predecessor).  Warpgroup 2 hands the first turn to warpgroup 0
    // and skips the hand-over after its last phase, so each barrier sees n_kv + 1 arrivals and n_kv + 1 waits and none is left
    // over.  Warpgroups whose rows all lie past Sq run the same phases (n_kv is uniform per CTA), so the rotation never skips
    // one.  A phase is PV(j-1) half 0 and QK(j), two commit groups; half 0 is folded into O as soon as it lands (under QK(j)) and
    // half 1 is issued before the turn passes, so the phase reaches the tensor cores in one piece; softmax(j) then runs under
    // half 1.  O's per-element sequence stays o *= alpha(j-1), o += PV(j-1).
    const uint32_t next_turn = 1 + (wg + 1) % kNC;
    if (n_kv > 0) {
      mbar_wait_wd(q_full, 0);
      if (wg == kNC - 1) named_bar_arrive(next_turn, kTurnThreads);
      tile_setup(0);
      mbar_wait_wd(kv_full, 0);                // never hold the turn while waiting on TMA
      named_bar_sync(my_turn, kTurnThreads);
      wgmma_fence();
      issue_qk(0);
      wgmma_commit();
      named_bar_arrive(next_turn, kTurnThreads);
      wgmma_wait<0>();
      fence_regs(s);
      softmax(0);
      pack_p();
    }
    for (int j = 1; j < n_kv; ++j) {
      tile_setup(j);
      mbar_wait_wd(kv_full + j % kStages, (j / kStages) & 1);
      named_bar_sync(my_turn, kTurnThreads);
      clk.turn();
      wgmma_fence();
      issue_pv_half(j - 1, 0);
      wgmma_commit();
      issue_qk(j);
      wgmma_commit();
      rescale_o();
      wgmma_wait<1>();                         // PV(j-1) half 0 is ready; QK(j) may still run
      fold_half(0);
      wgmma_fence();
      issue_pv_half(j - 1, 1);
      wgmma_commit();
      named_bar_arrive(next_turn, kTurnThreads);
      wgmma_wait<1>();                         // S(j) is ready; half 1 may still run
      fence_regs(s);
      clk.mma_done();
      softmax(j);
      wgmma_wait<0>();
      fold_half(1);
      if ((threadIdx.x & 127) == 0) mbar_arrive(kv_empty + (j - 1) % kStages);
      pack_p();
      clk.soft_done();
    }
    if (n_kv > 0) {
      named_bar_sync(my_turn, kTurnThreads);
      wgmma_fence();
      issue_pv_half(n_kv - 1, 0);
      wgmma_commit();
      rescale_o();
      wgmma_wait<0>();
      fold_half(0);
      wgmma_fence();
      issue_pv_half(n_kv - 1, 1);
      wgmma_commit();
      if (wg != kNC - 1) named_bar_arrive(next_turn, kTurnThreads);
      wgmma_wait<0>();
      fold_half(1);
      if ((threadIdx.x & 127) == 0) mbar_arrive(kv_empty + (n_kv - 1) % kStages);
    }
  } else {
    if (n_kv > 0) {
      mbar_wait_wd(q_full, 0);
      if (wg == 1) named_bar_arrive(their_turn, kTurnThreads);
      tile_setup(0);
      mbar_wait_wd(kv_full, 0);                  // never hold the turn while waiting on TMA
      named_bar_sync(my_turn, kTurnThreads);
      wgmma_fence();
      issue_qk(0);
      wgmma_commit();
      named_bar_arrive(their_turn, kTurnThreads);
      wgmma_wait<0>();
      fence_regs(s);
      softmax(0);
      pack_p();
    }
    for (int j = 1; j < n_kv; ++j) {
      tile_setup(j);
      mbar_wait_wd(kv_full + j % kStages, (j / kStages) & 1);
      named_bar_sync(my_turn, kTurnThreads);
      clk.turn();
      if constexpr (kPV16) rescale_o();          // before the in-place PV
      wgmma_fence();
      if constexpr (kSoftmaxUnderPV) {
        issue_qk(j);
        wgmma_commit();
        issue_pv(j - 1);
        wgmma_commit();
      } else {
        issue_pv(j - 1);
        issue_qk(j);
        wgmma_commit();
      }
      named_bar_arrive(their_turn, kTurnThreads);
      if constexpr (!kPV16) rescale_o();         // overlaps the MMAs
      if constexpr (kSoftmaxUnderPV) {
        wgmma_wait<1>();                         // S(j) is ready; PV(j-1) may still run
        fence_regs(s);
        clk.mma_done();
        softmax(j);
        wgmma_wait<0>();
        finish_pv(j - 1);
      } else {
        wgmma_wait<0>();
        fence_regs(s);
        clk.mma_done();
        finish_pv(j - 1);
        softmax(j);
      }
      pack_p();
      clk.soft_done();
    }
    if (n_kv > 0) {
      named_bar_sync(my_turn, kTurnThreads);
      if constexpr (kPV16) rescale_o();
      wgmma_fence();
      issue_pv(n_kv - 1);
      wgmma_commit();
      if (wg == 0) named_bar_arrive(their_turn, kTurnThreads);
      if constexpr (!kPV16) rescale_o();
      wgmma_wait<0>();
      finish_pv(n_kv - 1);
    }
  }
  clk.flush();

  // ---- epilogue: O / d * v_scale (+ v_mean) -> fp16/bf16 (…sm89.cuh:572-703)
  const float* vs = p.v_scale ? p.v_scale + (int64_t(varlen && !kSeqV ? 0 : b) * p.Hkv + hk) * D : nullptr;
  const float* vm = p.v_mean ? p.v_mean + (int64_t(varlen && !kSeqV ? 0 : b) * p.Hkv + hk) * D : nullptr;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    float dt = d[i];
    dt += __shfl_xor_sync(0xffffffffu, dt, 1);
    dt += __shfl_xor_sync(0xffffffffu, dt, 2);
    const bool row_ok = q_row[i] < q_len;
    OutT* orow = reinterpret_cast<OutT*>(p.out) + (varlen ? 0 : int64_t(b) * p.o_stride_b) + int64_t(h) * p.o_stride_h +
                 int64_t(q_off + q_row[i]) * p.o_stride_s;
    // a fully masked row yields zeros, not NaN; block-sparse causal or a window: a row may see none of the CTA's keys
    const float inv = (n_kv == 0 || ((kMask || kWindow) && !(dt > 0.f))) ? 0.f : rcp_approx(dt);
    if (row_ok) {
#pragma unroll
      for (int nb = 0; nb < D / 8; ++nb) {
        const int col = 8 * nb + 2 * t;
        float x0 = o[4 * nb + 2 * i] * inv, x1 = o[4 * nb + 2 * i + 1] * inv;
        if (vs) {
          x0 *= vs[col];
          x1 *= vs[col + 1];
        }
        if (vm) {
          x0 += vm[col];
          x1 += vm[col + 1];
        }
        if (n_kv == 0 || ((kSparse<kPV16, kMask> || kWindow) && !(dt > 0.f))) x0 = x1 = 0.f;
        *reinterpret_cast<uint32_t*>(orow + col) = pack2<OutT>(x0, x1);
      }
      if (p.lse != nullptr && t == 0) {
        // log2 units like the reference kernel (…sm89.cuh:691-703); the offset cancels: log2(sum 2^x)
        const int64_t li = varlen ? (int64_t(h) * p.Sq + q_off + q_row[i]) : ((int64_t(b) * p.Hq + h) * p.Sq + q_row[i]);
        p.lse[li] = n_kv > 0 ? lg2_approx(dt) + m[i] : -INFINITY;   // block-sparse / window, no visible key: lg2(0) = -inf
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ host
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn == nullptr) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(ptr);
  }
  return fn;
}

// 4-D byte tensor map: dims (innermost first) d0..d3, strides in bytes for d1..d3, box (b0,b1,1,1).
static int make_map_u8(CUtensorMap* map, const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t d3,
                       uint64_t s1, uint64_t s2, uint64_t s3, uint32_t b0, uint32_t b1, int swizzle_bytes) {
  EncodeTiledFn fn = get_encode_fn();
  SAB_REQUIRE(fn != nullptr, SAB_ERR_CUDA, "cuTensorMapEncodeTiled entry point not found");
  cuuint64_t dims[4] = {d0, d1, d2 ? d2 : 1, d3 ? d3 : 1};
  cuuint64_t strides[3] = {s1, s2 ? s2 : s1 * dims[1], s3 ? s3 : (s2 ? s2 : s1 * dims[1]) * dims[2]};
  cuuint32_t box[4] = {b0, b1, 1, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  for (int i = 0; i < 3; ++i)
    SAB_REQUIRE(strides[i] % 16 == 0, SAB_ERR_INVALID, "tensor stride %d (%llu bytes) must be a multiple of 16",
                i + 1, (unsigned long long)strides[i]);
  SAB_REQUIRE((reinterpret_cast<uintptr_t>(base) & 15) == 0, SAB_ERR_INVALID, "tensor base must be 16-byte aligned");
  CUtensorMapSwizzle sw = swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 4, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  SAB_REQUIRE(r == CUDA_SUCCESS, SAB_ERR_CUDA, "cuTensorMapEncodeTiled failed with CUresult %d", int(r));
  return SAB_OK;
}

// SAB_ATTN_KERNEL=exact selects the reference's exact running max on the INT8+FP8 path: P / m / d are then bit-identical to the
// reference kernel's.  Default: the lazy max (4 binades).
static bool exact_max_mode() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("SAB_ATTN_KERNEL");
    v = (e != nullptr && e[0] == 'e') ? 1 : 0;
  }
  return v == 1;
}
constexpr float kLazyTau = 4.0f;
// The dense INT8+FP8 kernel at D = 128 runs three consumer warpgroups on 192-row Q tiles.  SAB_ATTN_CONSUMERS=2 keeps it on two
// (128-row tiles, as every other form), so the two forms can be compared; they compute the same bits.
static int dense_consumers() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("SAB_ATTN_CONSUMERS");
    v = (e != nullptr && e[0] == '2') ? 2 : 3;
  }
  return v;
}

// nc: consumer warpgroups, 3 only for the dense INT8+FP8 instantiations at D = 128 (the tensor map of Q has nc * 64-row boxes
// and the grid nc * 64-row tiles)
template <int D, bool kKT, typename OutT, bool kPV16, bool kMask = false>
static int launch_attn(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, AttnParams p,
                       dim3 grid, cudaStream_t stream, int nc = 2) {
  p.lazy_tau = (kPV16 || exact_max_mode()) ? 0.0f : kLazyTau;
  if constexpr (D == 128 && !kPV16 && !kMask) {
    if (nc == 3) {
      constexpr size_t smem = attn_smem_bytes<D, false, 3>();
      auto kern = sage_attn_fwd_kernel<D, kKT, OutT, false, false, false, false, false, 3>;
      static bool configured[64] = {};
      if (int st = ensure_dynamic_smem(kern, smem, configured)) return st;
      kern<<<grid, kNumThreads<3>, smem, stream>>>(tq, tk, tv, p, Window{-1, -1});
      SAB_CUDA_OK(cudaGetLastError());
      return SAB_OK;
    }
  }
  SAB_REQUIRE(nc == 2, SAB_ERR_INVALID, "three consumer warpgroups need the dense INT8+FP8 kernel at head dim 128");
  constexpr size_t smem = attn_smem_bytes<D, kPV16>();
  auto kern = sage_attn_fwd_kernel<D, kKT, OutT, kPV16, kMask>;
  static bool configured[64] = {};
  if (int st = ensure_dynamic_smem(kern, smem, configured)) return st;
  kern<<<grid, kNumThreads<2>, smem, stream>>>(tq, tk, tv, p, Window{-1, -1});
  SAB_CUDA_OK(cudaGetLastError());
  return SAB_OK;
}

// the sliding-window form (sage_attn_fwd_kernel<D, kKT, OutT, false, false, true, kSeqV, kBR>); kSeqV: the packed form with
// per-sequence V statistics; kBR (with kSeqV): the packed bottom-right causal form, whose kernel ignores w
template <int D, bool kKT, typename OutT, bool kSeqV = false, bool kBR = false>
static int launch_attn_window(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, AttnParams p, Window w,
                              dim3 grid, cudaStream_t stream) {
  p.lazy_tau = exact_max_mode() ? 0.0f : kLazyTau;
  constexpr size_t smem = attn_smem_bytes<D, false>();
  auto kern = sage_attn_fwd_kernel<D, kKT, OutT, false, false, true, kSeqV, kBR>;
  static bool configured[64] = {};
  if (int st = ensure_dynamic_smem(kern, smem, configured)) return st;
  kern<<<grid, kNumThreads<2>, smem, stream>>>(tq, tk, tv, p, w);
  SAB_CUDA_OK(cudaGetLastError());
  return SAB_OK;
}

// the varlen form with per-sequence V statistics (sage_attn_fwd_kernel<D, kKT, OutT, false, false, false, true>)
template <int D, bool kKT, typename OutT>
static int launch_attn_seqv(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, AttnParams p, dim3 grid,
                            cudaStream_t stream) {
  p.lazy_tau = exact_max_mode() ? 0.0f : kLazyTau;
  constexpr size_t smem = attn_smem_bytes<D, false>();
  auto kern = sage_attn_fwd_kernel<D, kKT, OutT, false, false, false, true>;
  static bool configured[64] = {};
  if (int st = ensure_dynamic_smem(kern, smem, configured)) return st;
  kern<<<grid, kNumThreads<2>, smem, stream>>>(tq, tk, tv, p, Window{-1, -1});
  SAB_CUDA_OK(cudaGetLastError());
  return SAB_OK;
}

// the block-sparse form (sage_attn_fwd_kernel<D, kKT, OutT, false, true, false, kSeqV>): p.mask holds the block mask; kSeqV: the
// packed form with per-sequence V statistics.  max_k: the longest key range a CTA compacts (Skv dense, max_seqlen_k packed).
template <int D, bool kKT, typename OutT, bool kSeqV = false>
static int launch_attn_blocksparse(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, AttnParams p, int max_k,
                                   dim3 grid, cudaStream_t stream) {
  p.lazy_tau = exact_max_mode() ? 0.0f : kLazyTau;
  constexpr size_t smem_max = attn_smem_bytes<D, false>() + kv_list_bytes(kMaxKvBlocks);
  const size_t smem = attn_smem_bytes<D, false>() + kv_list_bytes((max_k + BN - 1) / BN);
  auto kern = sage_attn_fwd_kernel<D, kKT, OutT, false, true, false, kSeqV>;
  static bool configured[64] = {};
  if (int st = ensure_dynamic_smem(kern, smem_max, configured)) return st;
  kern<<<grid, kNumThreads<2>, smem, stream>>>(tq, tk, tv, p, Window{-1, -1});
  SAB_CUDA_OK(cudaGetLastError());
  return SAB_OK;
}

}  // namespace sab

// segment flags of the fused sequence-parallel entry point (sab_qk_int8_sv_f8_attn_sp)
struct SegArgs {
  const uint32_t* flags;
  uint32_t epoch;
  int heads_per_flag;
};

// Every forward entry.  The variant, each null / false when absent: a window (sab_qk_int8_sv_f8_attn_window and, through
// attn_varlen_seq, the packed window and bottom-right forms); a block mask bm, already checked (the block-sparse entries), with
// bm_max_k the packed max_seqlen_k; an attention mask m (sab_qk_int8_sv_f16_attn_masked); segment flags seg
// (sab_qk_int8_sv_f8_attn_sp); seq_v: v_scale / v_mean are per sequence (attn_varlen_seq).
static int attn_entry(int pv16, const int8_t* q_int8, const int8_t* k_int8, const uint8_t* v_fp8, void* out,
                                      float* lse, const float* q_scale, const float* k_scale, const float* v_scale,
                                      const float* v_mean, int out_dtype, int B, int Hq, int Hkv, int Sq, int Skv,
                                      int D, int64_t q_stride_b, int64_t q_stride_h, int64_t q_stride_s,
                                      int64_t k_stride_b, int64_t k_stride_h, int64_t k_stride_s, int64_t v_s_pad,
                                      int64_t o_stride_b, int64_t o_stride_h, int64_t o_stride_s, int is_causal,
                                      int q_gran, int k_gran, float sm_scale, int fold_sm_scale,
                                      const int32_t* cu_seqlens_q, const int32_t* cu_seqlens_k,
                                      const int32_t* cu_pad_v, const int32_t* cu_q_scale, const int32_t* cu_k_scale,
                                      int max_seqlen_q, int causal_q_offset, int kv_seg_len, int32_t* debug_dump,
                                      void* stream, const sab::Window* window, const sab::BlockMask* bm, int bm_max_k,
                                      const sab::MaskArgs* m, const SegArgs* seg, bool seq_v) {
  using namespace sab;
  SAB_REQUIRE(q_int8 && k_int8 && v_fp8 && out && q_scale && k_scale, SAB_ERR_INVALID, "null tensor pointer");
  SAB_REQUIRE(D == 64 || D == 128, SAB_ERR_UNSUPPORTED, "Unsupported head dim: %d (64 or 128 after padding)", D);
  SAB_REQUIRE(out_dtype == SAB_DTYPE_FP16 || out_dtype == SAB_DTYPE_BF16, SAB_ERR_UNSUPPORTED, "output dtype must be fp16 or bf16");
  SAB_REQUIRE(B > 0 && Hq > 0 && Hkv > 0 && Sq > 0 && Skv >= 0, SAB_ERR_INVALID, "bad sizes B=%d Hq=%d Hkv=%d Sq=%d Skv=%d", B, Hq, Hkv, Sq, Skv);
  SAB_REQUIRE(Hq % Hkv == 0, SAB_ERR_INVALID, "num_qo_heads (%d) must be divisible by num_kv_heads (%d)", Hq, Hkv);
  const uint64_t vb = pv16 ? 2 : 1;   // bytes per V element
  SAB_REQUIRE(q_gran >= 1 && q_gran <= 3 && k_gran >= 1 && k_gran <= 3, SAB_ERR_INVALID, "unknown quant granularity q=%d k=%d", q_gran, k_gran);
  SAB_REQUIRE(v_s_pad % 128 == 0 && (v_s_pad >= Skv || kv_seg_len > 0), SAB_ERR_INVALID, "v_fp8 token dimension (%lld) must be a multiple of 128 and >= kv_len", (long long)v_s_pad);
  SAB_REQUIRE(aligned16(out) && o_stride_s % 8 == 0 && o_stride_h % 8 == 0 && o_stride_b % 8 == 0, SAB_ERR_INVALID, "output must be 16-byte aligned with strides multiple of 8 elements");
  const bool varlen = cu_seqlens_q != nullptr;
  SAB_REQUIRE(causal_q_offset >= 0 && kv_seg_len >= 0, SAB_ERR_INVALID, "negative causal_q_offset / kv_seg_len");
  if (kv_seg_len > 0)
    SAB_REQUIRE(!varlen && kv_seg_len % 128 == 0 && Skv % kv_seg_len == 0 && v_s_pad == kv_seg_len, SAB_ERR_INVALID,
                "sequence-parallel form needs dense tensors, kv_seg_len %% 128 == 0, Skv %% kv_seg_len == 0, v_s_pad == kv_seg_len");
  if (varlen)
    SAB_REQUIRE(cu_seqlens_k && cu_pad_v && cu_q_scale && cu_k_scale && max_seqlen_q > 0, SAB_ERR_INVALID, "varlen needs cu_seqlens_k, cu_pad_v, cu_q_scale, cu_k_scale and max_seqlen_q");
  SAB_REQUIRE(debug_dump == nullptr, SAB_ERR_UNSUPPORTED, "debug_dump is not supported by the sm_90a kernel (pass NULL)");
  int st = sab_check_device();
  if (st != SAB_OK) return st;

  // the dense INT8+FP8 kernel at D = 128 (also sequence-parallel): three consumer warpgroups unless SAB_ATTN_CONSUMERS=2
  const int nc = (D == 128 && !pv16 && !varlen && !m && !bm && !window && !seq_v) ? dense_consumers() : 2;
  const uint32_t qbox = uint32_t(nc) * 64;   // Q rows per CTA
  CUtensorMap tq, tk, tv;
  const int swqk = D == 128 ? 128 : 64;
  const uint32_t kbox = BN;                 // 64-key tiles
  const uint32_t vbox = pv16 ? 128 : BN;    // bytes of one V^T row in the box
  const int swv = pv16 ? 128 : 64;
  if (kv_seg_len > 0) {
    const int P = Skv / kv_seg_len;
    if ((st = make_map_u8(&tq, q_int8, D, Sq, Hq, B, q_stride_s, q_stride_h, q_stride_b, D, qbox, swqk))) return st;
    if ((st = make_map_u8(&tk, k_int8, D, kv_seg_len, Hkv, uint64_t(B) * P, k_stride_s, k_stride_h, k_stride_b, D, kbox, swqk))) return st;
    if ((st = make_map_u8(&tv, v_fp8, v_s_pad * vb, D, Hkv, uint64_t(B) * P, v_s_pad * vb, uint64_t(v_s_pad) * D * vb, uint64_t(v_s_pad) * D * Hkv * vb, vbox, D, swv))) return st;
  } else if (!varlen) {
    if ((st = make_map_u8(&tq, q_int8, D, Sq, Hq, B, q_stride_s, q_stride_h, q_stride_b, D, qbox, swqk))) return st;
    if ((st = make_map_u8(&tk, k_int8, D, Skv > 0 ? Skv : 1, Hkv, B, k_stride_s, k_stride_h, k_stride_b, D, kbox, swqk))) return st;
    if ((st = make_map_u8(&tv, v_fp8, v_s_pad * vb, D, Hkv, B, v_s_pad * vb, uint64_t(v_s_pad) * D * vb, uint64_t(v_s_pad) * D * Hkv * vb, vbox, D, swv))) return st;
  } else {
    // packed [T,H,D]: Sq / Skv are the TOTAL token counts
    if ((st = make_map_u8(&tq, q_int8, D, Sq, Hq, 1, q_stride_s, q_stride_h, 0, D, BM, swqk))) return st;
    if ((st = make_map_u8(&tk, k_int8, D, Skv, Hkv, 1, k_stride_s, k_stride_h, 0, D, kbox, swqk))) return st;
    if ((st = make_map_u8(&tv, v_fp8, v_s_pad * vb, D, Hkv, 1, v_s_pad * vb, uint64_t(v_s_pad) * D * vb, 0, vbox, D, swv))) return st;
  }

  AttnParams p{};
  p.q_scale = q_scale; p.k_scale = k_scale; p.v_scale = v_scale; p.v_mean = v_mean;
  p.out = out; p.lse = lse;
  p.o_stride_b = o_stride_b; p.o_stride_h = o_stride_h; p.o_stride_s = o_stride_s;
  p.B = B; p.Hq = Hq; p.Hkv = Hkv; p.Sq = Sq; p.Sk = Skv;
  const int max_q = varlen ? max_seqlen_q : Sq;
  p.n_q_tiles = (max_q + int(qbox) - 1) / int(qbox);
  p.causal = is_causal ? 1 : 0;
  p.sm_scale_log2 = fold_sm_scale ? 1.0f : sm_scale * 1.44269504088896340736f;
  p.q_gran = q_gran;
  p.q_mult = q_gran == SAB_GRAN_PER_BLOCK ? 1 : (q_gran == SAB_GRAN_PER_WARP ? 4 : 32);
  p.k_mult = k_gran == SAB_GRAN_PER_THREAD ? 4 : 1;
  p.qs_stride_bh = int64_t((Sq + BM - 1) / BM) * p.q_mult;
  p.ks_stride_bh = int64_t((Skv + 63) / 64) * p.k_mult;
  p.qs_stride_idx = varlen ? Hq : 1;
  p.ks_stride_idx = varlen ? Hkv : 1;
  p.cu_q = cu_seqlens_q; p.cu_k = cu_seqlens_k; p.cu_v = cu_pad_v; p.cu_qs = cu_q_scale; p.cu_ks = cu_k_scale;
  p.causal_q_offset = causal_q_offset; p.kv_seg_len = kv_seg_len;

  dim3 grid(p.n_q_tiles, Hq, B);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const bool kt = k_gran == SAB_GRAN_PER_THREAD;
  const bool bf = out_dtype == SAB_DTYPE_BF16;
  if (m != nullptr) {
    // attn_qk_int8_per_block.py:33-52 (non-causal kernel only; sageattention/core.py:310-325 asserts mask is None when causal)
    SAB_REQUIRE(!kt, SAB_ERR_UNSUPPORTED,
                "attn_mask is supported by the dense non-causal fp16-PV path with per-block / per-warp K scales only");
    SAB_REQUIRE(m->ptr != nullptr && (m->kind == SAB_MASK_BOOL || m->kind == SAB_MASK_BIAS), SAB_ERR_INVALID,
                "attn_mask: null pointer or unknown kind %d", m->kind);
    p.mask = m->ptr; p.mask_kind = m->kind;
    p.mask_sb = m->sb; p.mask_sh = m->sh; p.mask_sm = m->sm; p.mask_sn = m->sn;
    if (D == 128) {
      if (bf) return launch_attn<128, false, __nv_bfloat16, true, true>(tq, tk, tv, p, grid, s);
      return launch_attn<128, false, __half, true, true>(tq, tk, tv, p, grid, s);
    }
    if (bf) return launch_attn<64, false, __nv_bfloat16, true, true>(tq, tk, tv, p, grid, s);
    return launch_attn<64, false, __half, true, true>(tq, tk, tv, p, grid, s);
  }
  if (seg != nullptr) {
    SAB_REQUIRE(kv_seg_len > 0, SAB_ERR_UNSUPPORTED,
                "segment flags need the sequence-parallel INT8/FP8 form (kv_seg_len > 0), non-causal");
    SAB_REQUIRE(seg->flags != nullptr && seg->heads_per_flag > 0 && Hkv % seg->heads_per_flag == 0, SAB_ERR_INVALID,
                "segment flags: null pointer or heads_per_flag (%d) does not divide num_kv_heads (%d)", seg->heads_per_flag, Hkv);
    p.seg_flags = seg->flags; p.seg_epoch = seg->epoch; p.seg_heads = seg->heads_per_flag;   // polled by the producer
  }
  if (bm != nullptr) {
    p.mask = bm->ptr;
    p.mask_sb = bm->sb; p.mask_sh = bm->sh; p.mask_sm = bm->sqb; p.mask_sn = bm->skb;
    if (seq_v) {
      const int mk = bm_max_k;
      if (D == 128) {
        if (kt) return bf ? launch_attn_blocksparse<128, true, __nv_bfloat16, true>(tq, tk, tv, p, mk, grid, s)
                          : launch_attn_blocksparse<128, true, __half, true>(tq, tk, tv, p, mk, grid, s);
        return bf ? launch_attn_blocksparse<128, false, __nv_bfloat16, true>(tq, tk, tv, p, mk, grid, s)
                  : launch_attn_blocksparse<128, false, __half, true>(tq, tk, tv, p, mk, grid, s);
      }
      if (kt) return bf ? launch_attn_blocksparse<64, true, __nv_bfloat16, true>(tq, tk, tv, p, mk, grid, s)
                        : launch_attn_blocksparse<64, true, __half, true>(tq, tk, tv, p, mk, grid, s);
      return bf ? launch_attn_blocksparse<64, false, __nv_bfloat16, true>(tq, tk, tv, p, mk, grid, s)
                : launch_attn_blocksparse<64, false, __half, true>(tq, tk, tv, p, mk, grid, s);
    }
    if (D == 128) {
      if (kt) return bf ? launch_attn_blocksparse<128, true, __nv_bfloat16>(tq, tk, tv, p, Skv, grid, s)
                        : launch_attn_blocksparse<128, true, __half>(tq, tk, tv, p, Skv, grid, s);
      return bf ? launch_attn_blocksparse<128, false, __nv_bfloat16>(tq, tk, tv, p, Skv, grid, s)
                : launch_attn_blocksparse<128, false, __half>(tq, tk, tv, p, Skv, grid, s);
    }
    if (kt) return bf ? launch_attn_blocksparse<64, true, __nv_bfloat16>(tq, tk, tv, p, Skv, grid, s)
                      : launch_attn_blocksparse<64, true, __half>(tq, tk, tv, p, Skv, grid, s);
    return bf ? launch_attn_blocksparse<64, false, __nv_bfloat16>(tq, tk, tv, p, Skv, grid, s)
              : launch_attn_blocksparse<64, false, __half>(tq, tk, tv, p, Skv, grid, s);
  }
  if (window != nullptr) {
    const Window w = *window;
    if (seq_v && w.right == kWindowBottomRight) {
      if (D == 128) {
        if (kt) return bf ? launch_attn_window<128, true, __nv_bfloat16, true, true>(tq, tk, tv, p, w, grid, s)
                          : launch_attn_window<128, true, __half, true, true>(tq, tk, tv, p, w, grid, s);
        return bf ? launch_attn_window<128, false, __nv_bfloat16, true, true>(tq, tk, tv, p, w, grid, s)
                  : launch_attn_window<128, false, __half, true, true>(tq, tk, tv, p, w, grid, s);
      }
      if (kt) return bf ? launch_attn_window<64, true, __nv_bfloat16, true, true>(tq, tk, tv, p, w, grid, s)
                        : launch_attn_window<64, true, __half, true, true>(tq, tk, tv, p, w, grid, s);
      return bf ? launch_attn_window<64, false, __nv_bfloat16, true, true>(tq, tk, tv, p, w, grid, s)
                : launch_attn_window<64, false, __half, true, true>(tq, tk, tv, p, w, grid, s);
    }
    if (seq_v) {
      if (D == 128) {
        if (kt) return bf ? launch_attn_window<128, true, __nv_bfloat16, true>(tq, tk, tv, p, w, grid, s)
                          : launch_attn_window<128, true, __half, true>(tq, tk, tv, p, w, grid, s);
        return bf ? launch_attn_window<128, false, __nv_bfloat16, true>(tq, tk, tv, p, w, grid, s)
                  : launch_attn_window<128, false, __half, true>(tq, tk, tv, p, w, grid, s);
      }
      if (kt) return bf ? launch_attn_window<64, true, __nv_bfloat16, true>(tq, tk, tv, p, w, grid, s)
                        : launch_attn_window<64, true, __half, true>(tq, tk, tv, p, w, grid, s);
      return bf ? launch_attn_window<64, false, __nv_bfloat16, true>(tq, tk, tv, p, w, grid, s)
                : launch_attn_window<64, false, __half, true>(tq, tk, tv, p, w, grid, s);
    }
    if (D == 128) {
      if (kt) return bf ? launch_attn_window<128, true, __nv_bfloat16>(tq, tk, tv, p, w, grid, s)
                        : launch_attn_window<128, true, __half>(tq, tk, tv, p, w, grid, s);
      return bf ? launch_attn_window<128, false, __nv_bfloat16>(tq, tk, tv, p, w, grid, s)
                : launch_attn_window<128, false, __half>(tq, tk, tv, p, w, grid, s);
    }
    if (kt) return bf ? launch_attn_window<64, true, __nv_bfloat16>(tq, tk, tv, p, w, grid, s)
                      : launch_attn_window<64, true, __half>(tq, tk, tv, p, w, grid, s);
    return bf ? launch_attn_window<64, false, __nv_bfloat16>(tq, tk, tv, p, w, grid, s)
              : launch_attn_window<64, false, __half>(tq, tk, tv, p, w, grid, s);
  }
  if (seq_v) {
    if (D == 128) {
      if (kt) return bf ? launch_attn_seqv<128, true, __nv_bfloat16>(tq, tk, tv, p, grid, s)
                        : launch_attn_seqv<128, true, __half>(tq, tk, tv, p, grid, s);
      return bf ? launch_attn_seqv<128, false, __nv_bfloat16>(tq, tk, tv, p, grid, s)
                : launch_attn_seqv<128, false, __half>(tq, tk, tv, p, grid, s);
    }
    if (kt) return bf ? launch_attn_seqv<64, true, __nv_bfloat16>(tq, tk, tv, p, grid, s)
                      : launch_attn_seqv<64, true, __half>(tq, tk, tv, p, grid, s);
    return bf ? launch_attn_seqv<64, false, __nv_bfloat16>(tq, tk, tv, p, grid, s)
              : launch_attn_seqv<64, false, __half>(tq, tk, tv, p, grid, s);
  }
#define SAB_LAUNCH(DD, KT, T)                                                      \
  do {                                                                             \
    if (pv16) return launch_attn<DD, KT, T, true>(tq, tk, tv, p, grid, s);         \
    return launch_attn<DD, KT, T, false>(tq, tk, tv, p, grid, s, nc);              \
  } while (0)
  if (D == 128) {
    if (kt) { if (bf) SAB_LAUNCH(128, true, __nv_bfloat16); else SAB_LAUNCH(128, true, __half); }
    else    { if (bf) SAB_LAUNCH(128, false, __nv_bfloat16); else SAB_LAUNCH(128, false, __half); }
  } else {
    if (kt) { if (bf) SAB_LAUNCH(64, true, __nv_bfloat16); else SAB_LAUNCH(64, true, __half); }
    else    { if (bf) SAB_LAUNCH(64, false, __nv_bfloat16); else SAB_LAUNCH(64, false, __half); }
  }
#undef SAB_LAUNCH
}

extern "C" int sab_qk_int8_sv_f8_attn(const int8_t* q_int8, const int8_t* k_int8, const uint8_t* v_fp8, void* out,
                                      float* lse, const float* q_scale, const float* k_scale, const float* v_scale,
                                      const float* v_mean, int out_dtype, int B, int Hq, int Hkv, int Sq, int Skv,
                                      int D, int64_t q_stride_b, int64_t q_stride_h, int64_t q_stride_s,
                                      int64_t k_stride_b, int64_t k_stride_h, int64_t k_stride_s, int64_t v_s_pad,
                                      int64_t o_stride_b, int64_t o_stride_h, int64_t o_stride_s, int is_causal,
                                      int q_gran, int k_gran, float sm_scale, int fold_sm_scale,
                                      const int32_t* cu_seqlens_q, const int32_t* cu_seqlens_k,
                                      const int32_t* cu_pad_v, const int32_t* cu_q_scale, const int32_t* cu_k_scale,
                                      int max_seqlen_q, int causal_q_offset, int kv_seg_len, int32_t* debug_dump,
                                      void* stream) {
  return attn_entry(0, q_int8, k_int8, v_fp8, out, lse, q_scale, k_scale, v_scale, v_mean, out_dtype, B, Hq, Hkv, Sq, Skv, D,
                    q_stride_b, q_stride_h, q_stride_s, k_stride_b, k_stride_h, k_stride_s, v_s_pad, o_stride_b, o_stride_h,
                    o_stride_s, is_causal, q_gran, k_gran, sm_scale, fold_sm_scale, cu_seqlens_q, cu_seqlens_k, cu_pad_v,
                    cu_q_scale, cu_k_scale, max_seqlen_q, causal_q_offset, kv_seg_len, debug_dump, stream, nullptr, nullptr, 0,
                    nullptr, nullptr, false);
}

extern "C" int sab_qk_int8_sv_f8_attn_sp(const int8_t* q_int8, const int8_t* k_int8, const uint8_t* v_fp8, void* out,
                                         float* lse, const float* q_scale, const float* k_scale, const float* v_scale,
                                         int out_dtype, int B, int Hq, int Hkv, int Sq, int Skv, int D, int64_t q_stride_b,
                                         int64_t q_stride_h, int64_t q_stride_s, int64_t k_stride_b, int64_t k_stride_h,
                                         int64_t k_stride_s, int64_t v_s_pad, int64_t o_stride_b, int64_t o_stride_h,
                                         int64_t o_stride_s, int q_gran, int k_gran, float sm_scale, int kv_seg_len,
                                         const uint32_t* seg_flags, uint32_t seg_epoch, int heads_per_flag, void* stream) {
  const SegArgs a{seg_flags, seg_epoch, heads_per_flag};
  return attn_entry(0, q_int8, k_int8, v_fp8, out, lse, q_scale, k_scale, v_scale, nullptr, out_dtype, B, Hq, Hkv, Sq, Skv, D,
                    q_stride_b, q_stride_h, q_stride_s, k_stride_b, k_stride_h, k_stride_s, v_s_pad, o_stride_b, o_stride_h,
                    o_stride_s, 0, q_gran, k_gran, sm_scale, 0, nullptr, nullptr, nullptr, nullptr, nullptr, 0, 0, kv_seg_len,
                    nullptr, stream, nullptr, nullptr, 0, nullptr, &a, false);
}

extern "C" int sab_qk_int8_sv_f16_attn(const int8_t* q_int8, const int8_t* k_int8, const void* v_f16t, void* out, float* lse,
                                       const float* q_scale, const float* k_scale, int out_dtype, int B, int Hq, int Hkv,
                                       int Sq, int Skv, int D, int64_t q_stride_b, int64_t q_stride_h, int64_t q_stride_s,
                                       int64_t k_stride_b, int64_t k_stride_h, int64_t k_stride_s, int64_t v_s_pad,
                                       int64_t o_stride_b, int64_t o_stride_h, int64_t o_stride_s, int is_causal, int q_gran,
                                       int k_gran, float sm_scale, int fold_sm_scale, const int32_t* cu_seqlens_q,
                                       const int32_t* cu_seqlens_k, const int32_t* cu_pad_v, const int32_t* cu_q_scale,
                                       const int32_t* cu_k_scale, int max_seqlen_q, void* stream) {
  return attn_entry(1, q_int8, k_int8, reinterpret_cast<const uint8_t*>(v_f16t), out, lse, q_scale, k_scale, nullptr, nullptr,
                    out_dtype, B, Hq, Hkv, Sq, Skv, D, q_stride_b, q_stride_h, q_stride_s, k_stride_b, k_stride_h, k_stride_s,
                    v_s_pad, o_stride_b, o_stride_h, o_stride_s, is_causal, q_gran, k_gran, sm_scale, fold_sm_scale,
                    cu_seqlens_q, cu_seqlens_k, cu_pad_v, cu_q_scale, cu_k_scale, max_seqlen_q, 0, 0, nullptr, stream, nullptr,
                    nullptr, 0, nullptr, nullptr, false);
}

extern "C" int sab_qk_int8_sv_f16_attn_masked(const int8_t* q_int8, const int8_t* k_int8, const void* v_f16t, void* out, float* lse,
                                              const float* q_scale, const float* k_scale, int out_dtype, int B, int Hq, int Hkv,
                                              int Sq, int Skv, int D, int64_t q_stride_b, int64_t q_stride_h, int64_t q_stride_s,
                                              int64_t k_stride_b, int64_t k_stride_h, int64_t k_stride_s, int64_t v_s_pad,
                                              int64_t o_stride_b, int64_t o_stride_h, int64_t o_stride_s, int q_gran, int k_gran,
                                              float sm_scale, int fold_sm_scale, const void* attn_mask, int mask_kind,
                                              int64_t mask_stride_b, int64_t mask_stride_h, int64_t mask_stride_m,
                                              int64_t mask_stride_n, void* stream) {
  const sab::MaskArgs m{attn_mask, mask_kind, mask_stride_b, mask_stride_h, mask_stride_m, mask_stride_n};
  return attn_entry(1, q_int8, k_int8, reinterpret_cast<const uint8_t*>(v_f16t), out, lse, q_scale, k_scale, nullptr, nullptr,
                    out_dtype, B, Hq, Hkv, Sq, Skv, D, q_stride_b, q_stride_h, q_stride_s, k_stride_b, k_stride_h, k_stride_s,
                    v_s_pad, o_stride_b, o_stride_h, o_stride_s, 0, q_gran, k_gran, sm_scale, fold_sm_scale, nullptr, nullptr,
                    nullptr, nullptr, nullptr, 0, 0, 0, nullptr, stream, nullptr, nullptr, 0, &m, nullptr, false);
}

extern "C" int sab_qk_int8_sv_f8_attn_blocksparse(const int8_t* q_int8, const int8_t* k_int8, const uint8_t* v_fp8, void* out,
                                                  float* lse, const float* q_scale, const float* k_scale, const float* v_scale,
                                                  const float* v_mean, int out_dtype, int B, int Hq, int Hkv, int Sq, int Skv,
                                                  int D, int64_t q_stride_b, int64_t q_stride_h, int64_t q_stride_s,
                                                  int64_t k_stride_b, int64_t k_stride_h, int64_t k_stride_s, int64_t v_s_pad,
                                                  int64_t o_stride_b, int64_t o_stride_h, int64_t o_stride_s, int is_causal,
                                                  int q_gran, int k_gran, float sm_scale, int fold_sm_scale,
                                                  const uint8_t* block_mask, int64_t mask_stride_b, int64_t mask_stride_h,
                                                  int64_t mask_stride_qb, int64_t mask_stride_kb, void* stream) {
  if (int st = sab::check_block_mask(block_mask, mask_stride_b, mask_stride_h, mask_stride_qb, mask_stride_kb, q_gran, is_causal, Sq, Skv))
    return st;
  const sab::BlockMask bm{block_mask, mask_stride_b, mask_stride_h, mask_stride_qb, mask_stride_kb};
  return attn_entry(0, q_int8, k_int8, v_fp8, out, lse, q_scale, k_scale, v_scale, v_mean, out_dtype, B, Hq, Hkv, Sq, Skv, D,
                    q_stride_b, q_stride_h, q_stride_s, k_stride_b, k_stride_h, k_stride_s, v_s_pad, o_stride_b, o_stride_h,
                    o_stride_s, is_causal, q_gran, k_gran, sm_scale, fold_sm_scale, nullptr, nullptr, nullptr, nullptr, nullptr, 0,
                    0, 0, nullptr, stream, nullptr, &bm, 0, nullptr, nullptr, false);
}

extern "C" int sab_qk_int8_sv_f8_attn_window(const int8_t* q_int8, const int8_t* k_int8, const uint8_t* v_fp8, void* out, float* lse,
                                             const float* q_scale, const float* k_scale, const float* v_scale, const float* v_mean,
                                             int out_dtype, int B, int Hq, int Hkv, int Sq, int Skv, int D, int64_t q_stride_b,
                                             int64_t q_stride_h, int64_t q_stride_s, int64_t k_stride_b, int64_t k_stride_h,
                                             int64_t k_stride_s, int64_t v_s_pad, int64_t o_stride_b, int64_t o_stride_h,
                                             int64_t o_stride_s, int is_causal, int q_gran, int k_gran, float sm_scale,
                                             int fold_sm_scale, int window_left, int window_right, void* stream) {
  if (int st = sab::check_window(window_left, window_right, is_causal, Sq, Skv)) return st;
  const sab::Window w{window_left, window_right};
  return attn_entry(0, q_int8, k_int8, v_fp8, out, lse, q_scale, k_scale, v_scale, v_mean, out_dtype, B, Hq, Hkv, Sq, Skv, D,
                    q_stride_b, q_stride_h, q_stride_s, k_stride_b, k_stride_h, k_stride_s, v_s_pad, o_stride_b, o_stride_h,
                    o_stride_s, is_causal, q_gran, k_gran, sm_scale, fold_sm_scale, nullptr, nullptr, nullptr, nullptr, nullptr, 0,
                    0, 0, nullptr, stream, &w, nullptr, 0, nullptr, nullptr, false);
}

// sab_qk_int8_sv_f8_attn_varlen and, with a window w or a block mask bm (already checked; bm_max_k: max_seqlen_k),
// sab_qk_int8_sv_f8_attn_varlen_window / _varlen_bottom_right / _varlen_blocksparse
static int attn_varlen_seq(const int8_t* q_int8, const int8_t* k_int8, const uint8_t* v_fp8, void* out, float* lse,
                           const float* q_scale, const float* k_scale, const float* v_scale, const float* v_mean, int out_dtype,
                           int nseq, int Hq, int Hkv, int Tq, int Tk, int D, int64_t q_stride_t, int64_t q_stride_h,
                           int64_t k_stride_t, int64_t k_stride_h, int64_t v_t_pad, int64_t o_stride_t, int64_t o_stride_h,
                           int is_causal, int q_gran, int k_gran, float sm_scale, const int32_t* cu_seqlens_q,
                           const int32_t* cu_seqlens_k, const int32_t* cu_pad_v, const int32_t* cu_q_scale,
                           const int32_t* cu_k_scale, int max_seqlen_q, const sab::Window* w, const sab::BlockMask* bm, int bm_max_k,
                           void* stream) {
  SAB_REQUIRE(q_gran == SAB_GRAN_PER_WARP || q_gran == SAB_GRAN_PER_THREAD, SAB_ERR_INVALID,
              "q_gran must be SAB_GRAN_PER_WARP or SAB_GRAN_PER_THREAD (got %d)", q_gran);
  SAB_REQUIRE(k_gran == SAB_GRAN_PER_WARP || k_gran == SAB_GRAN_PER_THREAD, SAB_ERR_INVALID,
              "k_gran must be SAB_GRAN_PER_WARP or SAB_GRAN_PER_THREAD (got %d)", k_gran);
  SAB_REQUIRE(v_scale != nullptr && cu_seqlens_q != nullptr && nseq > 0 && Tk > 0, SAB_ERR_INVALID,
              "the packed INT8/FP8 form needs v_scale, cu_seqlens_q, nseq > 0 and Tk > 0");
  return attn_entry(0, q_int8, k_int8, v_fp8, out, lse, q_scale, k_scale, v_scale, v_mean, out_dtype, nseq, Hq, Hkv, Tq, Tk, D, 0,
                    q_stride_h, q_stride_t, 0, k_stride_h, k_stride_t, v_t_pad, 0, o_stride_h, o_stride_t, is_causal, q_gran, k_gran,
                    sm_scale, 0, cu_seqlens_q, cu_seqlens_k, cu_pad_v, cu_q_scale, cu_k_scale, max_seqlen_q, 0, 0, nullptr, stream,
                    w, bm, bm_max_k, nullptr, nullptr, true);
}

extern "C" int sab_qk_int8_sv_f8_attn_varlen(const int8_t* q_int8, const int8_t* k_int8, const uint8_t* v_fp8, void* out, float* lse,
                                             const float* q_scale, const float* k_scale, const float* v_scale, const float* v_mean,
                                             int out_dtype, int nseq, int Hq, int Hkv, int Tq, int Tk, int D, int64_t q_stride_t,
                                             int64_t q_stride_h, int64_t k_stride_t, int64_t k_stride_h, int64_t v_t_pad,
                                             int64_t o_stride_t, int64_t o_stride_h, int is_causal, int q_gran, int k_gran,
                                             float sm_scale, const int32_t* cu_seqlens_q, const int32_t* cu_seqlens_k,
                                             const int32_t* cu_pad_v, const int32_t* cu_q_scale, const int32_t* cu_k_scale,
                                             int max_seqlen_q, void* stream) {
  return attn_varlen_seq(q_int8, k_int8, v_fp8, out, lse, q_scale, k_scale, v_scale, v_mean, out_dtype, nseq, Hq, Hkv, Tq, Tk, D,
                         q_stride_t, q_stride_h, k_stride_t, k_stride_h, v_t_pad, o_stride_t, o_stride_h, is_causal, q_gran, k_gran,
                         sm_scale, cu_seqlens_q, cu_seqlens_k, cu_pad_v, cu_q_scale, cu_k_scale, max_seqlen_q, nullptr, nullptr, 0,
                         stream);
}

extern "C" int sab_qk_int8_sv_f8_attn_varlen_window(const int8_t* q_int8, const int8_t* k_int8, const uint8_t* v_fp8, void* out,
                                                    float* lse, const float* q_scale, const float* k_scale, const float* v_scale,
                                                    const float* v_mean, int out_dtype, int nseq, int Hq, int Hkv, int Tq, int Tk, int D,
                                                    int64_t q_stride_t, int64_t q_stride_h, int64_t k_stride_t, int64_t k_stride_h,
                                                    int64_t v_t_pad, int64_t o_stride_t, int64_t o_stride_h, int is_causal, int q_gran,
                                                    int k_gran, float sm_scale, const int32_t* cu_seqlens_q,
                                                    const int32_t* cu_seqlens_k, const int32_t* cu_pad_v, const int32_t* cu_q_scale,
                                                    const int32_t* cu_k_scale, int max_seqlen_q, int window_left, int window_right,
                                                    void* stream) {
  // no sequence is longer than the packed batch: the right side is clamped at Tk
  if (int st = sab::check_window_varlen(window_left, window_right, max_seqlen_q, Tk)) return st;
  SAB_REQUIRE(cu_seqlens_q && cu_seqlens_k && cu_pad_v && cu_q_scale && cu_k_scale && nseq > 0, SAB_ERR_INVALID,
              "the packed window needs cu_seqlens_q, cu_seqlens_k, cu_pad_v, cu_q_scale, cu_k_scale and nseq > 0");
  const sab::Window w{window_left, window_right};
  return attn_varlen_seq(q_int8, k_int8, v_fp8, out, lse, q_scale, k_scale, v_scale, v_mean, out_dtype, nseq, Hq, Hkv, Tq, Tk, D,
                         q_stride_t, q_stride_h, k_stride_t, k_stride_h, v_t_pad, o_stride_t, o_stride_h, is_causal, q_gran, k_gran,
                         sm_scale, cu_seqlens_q, cu_seqlens_k, cu_pad_v, cu_q_scale, cu_k_scale, max_seqlen_q, &w, nullptr, 0, stream);
}

extern "C" int sab_qk_int8_sv_f8_attn_varlen_bottom_right(const int8_t* q_int8, const int8_t* k_int8, const uint8_t* v_fp8, void* out,
                                                          float* lse, const float* q_scale, const float* k_scale,
                                                          const float* v_scale, const float* v_mean, int out_dtype, int nseq, int Hq,
                                                          int Hkv, int Tq, int Tk, int D, int64_t q_stride_t, int64_t q_stride_h,
                                                          int64_t k_stride_t, int64_t k_stride_h, int64_t v_t_pad, int64_t o_stride_t,
                                                          int64_t o_stride_h, int is_causal, int q_gran, int k_gran, float sm_scale,
                                                          const int32_t* cu_seqlens_q, const int32_t* cu_seqlens_k,
                                                          const int32_t* cu_pad_v, const int32_t* cu_q_scale,
                                                          const int32_t* cu_k_scale, int max_seqlen_q, void* stream) {
  SAB_REQUIRE(cu_seqlens_q && cu_seqlens_k && cu_pad_v && cu_q_scale && cu_k_scale && nseq > 0, SAB_ERR_INVALID,
              "the packed bottom-right form needs cu_seqlens_q, cu_seqlens_k, cu_pad_v, cu_q_scale, cu_k_scale and nseq > 0");
  // non-causal has no alignment: the packed form itself.  Causal: the bottom-right window, whose kernel takes is_causal = 0.
  const sab::Window w{-1, sab::kWindowBottomRight};
  return attn_varlen_seq(q_int8, k_int8, v_fp8, out, lse, q_scale, k_scale, v_scale, v_mean, out_dtype, nseq, Hq, Hkv, Tq, Tk, D,
                         q_stride_t, q_stride_h, k_stride_t, k_stride_h, v_t_pad, o_stride_t, o_stride_h, 0, q_gran, k_gran, sm_scale,
                         cu_seqlens_q, cu_seqlens_k, cu_pad_v, cu_q_scale, cu_k_scale, max_seqlen_q, is_causal ? &w : nullptr, nullptr,
                         0, stream);
}

extern "C" int sab_qk_int8_sv_f8_attn_varlen_blocksparse(const int8_t* q_int8, const int8_t* k_int8, const uint8_t* v_fp8, void* out,
                                                         float* lse, const float* q_scale, const float* k_scale,
                                                         const float* v_scale, const float* v_mean, int out_dtype, int nseq, int Hq,
                                                         int Hkv, int Tq, int Tk, int D, int64_t q_stride_t, int64_t q_stride_h,
                                                         int64_t k_stride_t, int64_t k_stride_h, int64_t v_t_pad, int64_t o_stride_t,
                                                         int64_t o_stride_h, int is_causal, int q_gran, int k_gran, float sm_scale,
                                                         const int32_t* cu_seqlens_q, const int32_t* cu_seqlens_k,
                                                         const int32_t* cu_pad_v, const int32_t* cu_q_scale, const int32_t* cu_k_scale,
                                                         int max_seqlen_q, int max_seqlen_k, const uint8_t* block_mask,
                                                         int64_t mask_stride_b, int64_t mask_stride_h, int64_t mask_stride_qb,
                                                         int64_t mask_stride_kb, void* stream) {
  if (int st = sab::check_block_mask_varlen(block_mask, mask_stride_b, mask_stride_h, mask_stride_qb, mask_stride_kb, q_gran,
                                            max_seqlen_q, max_seqlen_k))
    return st;
  SAB_REQUIRE(cu_seqlens_q && cu_seqlens_k && cu_pad_v && cu_q_scale && cu_k_scale && nseq > 0, SAB_ERR_INVALID,
              "the packed block mask needs cu_seqlens_q, cu_seqlens_k, cu_pad_v, cu_q_scale, cu_k_scale and nseq > 0");
  const sab::BlockMask bm{block_mask, mask_stride_b, mask_stride_h, mask_stride_qb, mask_stride_kb};
  return attn_varlen_seq(q_int8, k_int8, v_fp8, out, lse, q_scale, k_scale, v_scale, v_mean, out_dtype, nseq, Hq, Hkv, Tq, Tk, D,
                         q_stride_t, q_stride_h, k_stride_t, k_stride_h, v_t_pad, o_stride_t, o_stride_h, is_causal, q_gran, k_gran,
                         sm_scale, cu_seqlens_q, cu_seqlens_k, cu_pad_v, cu_q_scale, cu_k_scale, max_seqlen_q, nullptr, &bm,
                         max_seqlen_k, stream);
}

#ifdef SAB_PHASE_CLOCKS
// measurement builds: copy out the phase-cycle sums of sab::g_phase_clk (see PhaseClocks) and reset them
extern "C" int sab_phase_clocks_read(unsigned long long* out5) {
  SAB_CUDA_OK(cudaDeviceSynchronize());
  SAB_CUDA_OK(cudaMemcpyFromSymbol(out5, sab::g_phase_clk, sizeof(unsigned long long) * 5));
  const unsigned long long zero[5] = {};
  SAB_CUDA_OK(cudaMemcpyToSymbol(sab::g_phase_clk, zero, sizeof(zero)));
  return SAB_OK;
}
#endif
