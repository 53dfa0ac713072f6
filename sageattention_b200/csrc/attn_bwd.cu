// Backward of the INT8-QK attention for sm_90a (H100): the gradient of softmax(S) V evaluated at the forward's quantised logits, a
// straight-through estimator through the INT8 Q/K, FP8 V and FP8 P roundings:
//   S  = dequant(q8 k8^T) * sm_scale        (logit_log2, attn_common.cuh: the forward kernel's logits to the bit)
//   P  = exp2(S*log2e - lse)                 (lse: the forward kernel's own log2 LSE, before the smoothing correction)
//   dV = P^T dO    dP = dO V^T    delta = rowsum(dO o O)    dS = P o (dP - delta)
//   dQ = dS K * sm_scale    dK = dS^T Q * sm_scale            (Q, K, V: the original 16-bit tensors)
// K smoothing needs no term: the rows of dS sum to zero, so the K mean drops out of dQ and dK.  S is still recomputed from the
// smoothed k8, because the LSE is relative to it, and dQ is taken with the smoothed K (K - mean, rounded to the input dtype): with
// delta from the quantised forward's O the rows of dS sum to a small residue, which K itself would multiply by its mean.
//
// Three launches on the caller's stream, no atomics, so the gradients are bit-reproducible:
//   bwd_delta_kernel : delta of every Q row (fp32) into the caller's workspace;
//   bwd_dq_kernel    : one CTA per 128-row Q tile of one (batch, Q head), shaped like the forward: two warpgroups of 64 rows, a loop
//                      over 64-key tiles; S = Q K^T (INT8), dP = dO V^T, dQ += dS K with dS as the register A operand;
//   bwd_dkdv_kernel  : one CTA per 128-key tile of one (batch, KV head), two warpgroups of 64 keys, a loop over every Q head of the
//                      GQA group and every 64-row Q tile, so dK and dV are written once.  S^T = K Q^T (INT8) and dP^T = V dO^T put
//                      P^T and dS^T in the accumulator layout; rounded to the input dtype they are the register A operand of
//                      dV += P^T dO and dK += dS^T Q.
// Varlen (p.a.cu_q != nullptr, packed [T,H,D] tensors, per-block scales [nblocks,H]): blockIdx.z is the sequence; the top of each
// CTA decodes its sequence's token offsets, lengths and first scale blocks once, as the forward does (attn.cu), and the loops below
// read those.  The causal mask is top-left inside each sequence.  delta runs on the packed rows as B = 1, so it has the LSE's
// [Hq,Tq] layout.
// Masked (p.a.mask != nullptr, the attn_mask of the dense non-causal FP16-PV forward, per-block / per-warp K scales): separate
// kernels bwd_dq_masked_kernel / bwd_dkdv_masked_kernel branch once on the mask kind into the same bodies compiled with the mask.
// P is the forward's masked P: a bool mask (0 = masked out) zeroes elements, a bias enters as exp2(fmaf(S, coef, bias) - lse)
// (the forward's tile_bias), and a row with lse = -inf (no visible key: the forward returned zeros) has P = 0.  The dQ kernel
// reads the mask along its rows, as the forward does, and writes dBias = ln2 * dS (the bias is added to log2-unit logits) for
// the elements of its own rows, so dBias needs no atomics either.  The dK/dV kernel stages each [64 Q rows x 128 keys] mask tile
// of Q head h in shared memory with the other operands.
// Products are wgmma with fp32 accumulation: INT8 for S as in the forward, bf16 / f16 for the rest.  Every B operand is K-major in
// shared memory, in the swizzled layout the forward's TMA loads write; the operands the math needs transposed (dO^T, Q^T, K^T) are
// transposed by the loaders.  Loads are plain: all threads copy a tile, the CTA synchronises, then computes (no load/compute
// overlap yet).
#include <type_traits>
#include "attn_common.cuh"

namespace sab {

constexpr int kBwdThreads = 256;   // two warpgroups

struct BwdParams {
  AttnParams a;                    // the forward's scale / size / causal / varlen parameters (a.lse, a.out unused)
  int n_k_tiles;                   // 128-key tiles per (batch or sequence, KV head): the dK/dV grid's x
  const int8_t* q8;
  const int8_t* k8;
  int64_t q8_sb, q8_sh, q8_ss, k8_sb, k8_sh, k8_ss;
  const uint16_t* q;               // 16-bit tensors (bf16 / f16 bits); dq / dk / dv have the strides of q / k / v
  const uint16_t* k;
  const uint16_t* v;
  const uint16_t* o;
  const uint16_t* dout;
  const uint16_t* kmean;           // nullable [B,Hkv,D] (varlen [Hkv,D]): the K smoothing mean, subtracted from the K of dQ += dS K
  int64_t q_sb, q_sh, q_ss, k_sb, k_sh, k_ss, v_sb, v_sh, v_ss, o_sb, o_sh, o_ss, do_sb, do_sh, do_ss;
  const float* lse;                // [B,Hq,Sq] log2 units (varlen [Hq,Tq])
  float* delta;                    // [B,Hq,Sq] workspace (varlen [Hq,Tq])
  void* dq;
  void* dk;
  void* dv;
  float sm_scale;
};

// Byte offset of 16-byte chunk c of row r in a K-major tile of `rows` rows of RB bytes, laid out as a TMA load with swizzle
// min(RB, 128) writes it: 128-byte column slabs (a longer row continues in the next slab), Swizzle<., 4, 3> inside a slab
// (address bits [4, 7) ^= bits [7, 10)).  Tile bases are 1024-byte aligned.
template <int RB>
__device__ __forceinline__ uint32_t tile_off(int r, int c, int rows) {
  constexpr int SW = RB < 128 ? RB : 128;
  constexpr int CPS = SW / 16;
  const uint32_t o = uint32_t(r) * SW + uint32_t(c % CPS) * 16;
  return uint32_t(c / CPS) * uint32_t(rows) * SW + (o ^ (((o >> 7) & (CPS - 1)) << 4));
}
// wgmma descriptor of rows [r0, r0 + 64) of such a tile, at byte kb along K (one instruction's 32-byte K extent, inside a slab)
template <int RB>
__device__ __forceinline__ uint64_t tile_desc(const uint8_t* tile, int rows, int r0, int kb) {
  constexpr int SW = RB < 128 ? RB : 128;
  return make_wgmma_desc<SW>(smem_u32(tile + (kb / SW) * rows * SW + r0 * SW)) + uint64_t((kb % SW) >> 4);
}

// rows [row0, row0 + R) of one (b, h) of a bhsd tensor (E-byte elements, row stride ss elements) into a K-major tile; rows >= limit
// read as zeros
template <int R, int D, int E>
__device__ __forceinline__ void load_tile(uint8_t* tile, const void* base, int64_t ss, int row0, int limit) {
  constexpr int RB = D * E, CPR = RB / 16;
  const uint8_t* src = reinterpret_cast<const uint8_t*>(base);
  for (int idx = threadIdx.x; idx < R * CPR; idx += kBwdThreads) {
    const int r = idx / CPR, c = idx % CPR;
    uint4 x = make_uint4(0u, 0u, 0u, 0u);
    if (row0 + r < limit) x = __ldg(reinterpret_cast<const uint4*>(src + int64_t(row0 + r) * ss * E) + c);
    *reinterpret_cast<uint4*>(tile + tile_off<RB>(r, c, R)) = x;
  }
}
template <typename T>
__device__ __forceinline__ uint32_t sub_rn(uint32_t x, float m) {   // 16-bit x - m, rounded to T
  if constexpr (std::is_same_v<T, __half>) return __half_as_ushort(__float2half_rn(__half2float(__ushort_as_half(uint16_t(x))) - m));
  else return __bfloat16_as_ushort(__float2bfloat16_rn(__bfloat162float(__ushort_as_bfloat16(uint16_t(x))) - m));
}
// the same 64 rows of 16-bit elements transposed: tile row d (128 bytes) holds column d of the 64 rows.  sub (nullable, [D]): a
// per-column value subtracted in fp32 and rounded to T
template <int D, typename T>
__device__ __forceinline__ void load_tile_t(uint8_t* tile, const uint16_t* base, int64_t ss, int row0, int limit,
                                            const uint16_t* sub = nullptr) {
  for (int idx = threadIdx.x; idx < D * 8; idx += kBwdThreads) {
    const int d = idx % D, c = idx / D;   // consecutive threads read consecutive columns of one row
    float m = 0.f;
    if (sub != nullptr) {
      if constexpr (std::is_same_v<T, __half>) m = __half2float(__ushort_as_half(sub[d]));
      else m = __bfloat162float(__ushort_as_bfloat16(sub[d]));
    }
    uint32_t w[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int r = row0 + 8 * c + 2 * j;
      uint32_t lo = r < limit ? __ldg(base + int64_t(r) * ss + d) : 0u;
      uint32_t hi = r + 1 < limit ? __ldg(base + int64_t(r + 1) * ss + d) : 0u;
      if (sub != nullptr) {
        lo = r < limit ? sub_rn<T>(lo, m) : 0u;
        hi = r + 1 < limit ? sub_rn<T>(hi, m) : 0u;
      }
      w[j] = lo | (hi << 16);
    }
    *reinterpret_cast<uint4*>(tile + tile_off<128>(d, c, D)) = make_uint4(w[0], w[1], w[2], w[3]);
  }
}

template <typename T>
__device__ __forceinline__ void wgmma_ss(float (&d)[32], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
  if constexpr (std::is_same_v<T, __half>) wgmma_ss_f16(d, a_desc, b_desc, accumulate);
  else wgmma_ss_bf16(d, a_desc, b_desc, accumulate);
}
template <typename T, int N>
__device__ __forceinline__ void wgmma_rs(float (&d)[N], const uint32_t (&a)[4], uint64_t b_desc, uint32_t accumulate) {
  if constexpr (std::is_same_v<T, __half>) wgmma_pv_f16(d, a, b_desc, accumulate);
  else wgmma_rs_bf16(d, a, b_desc, accumulate);
}
// 64 x 64 fp32 accumulator tile -> A fragments of four k16 steps: step kk = accumulator blocks 2kk, 2kk+1 (same layout, no exchange)
template <typename T>
__device__ __forceinline__ void acc_to_a(const float (&e)[32], uint32_t (&a)[4][4]) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    const int i0 = 8 * kk, i1 = 8 * kk + 4;
    a[kk][0] = pack2<T>(e[i0], e[i0 + 1]);
    a[kk][1] = pack2<T>(e[i0 + 2], e[i0 + 3]);
    a[kk][2] = pack2<T>(e[i1], e[i1 + 1]);
    a[kk][3] = pack2<T>(e[i1 + 2], e[i1 + 3]);
  }
}
// rows r, r + 8 of a 64 x D fp32 accumulator tile (times `scale`) -> 16-bit row-major memory
template <typename T, int D>
__device__ __forceinline__ void store_rows(const float (&acc)[D / 2], T* row0, T* row1, bool ok0, bool ok1, int t, float scale) {
#pragma unroll
  for (int nb = 0; nb < D / 8; ++nb) {
    const int col = 8 * nb + 2 * t;
    if (ok0) *reinterpret_cast<uint32_t*>(row0 + col) = pack2<T>(acc[4 * nb] * scale, acc[4 * nb + 1] * scale);
    if (ok1) *reinterpret_cast<uint32_t*>(row1 + col) = pack2<T>(acc[4 * nb + 2] * scale, acc[4 * nb + 3] * scale);
  }
}

// ------------------------------------------------------------------------------------------------ attention mask
// kMask: 0 (unmasked kernels), SAB_MASK_BOOL (uint8 elements, 0 = masked out) or SAB_MASK_BIAS (16-bit elements of T)
template <int kMask>
using MaskElem = std::conditional_t<kMask == SAB_MASK_BOOL, uint8_t, uint16_t>;
constexpr float kLn2 = 0.69314718055994530942f;

// -lse of a row of the masked kernels.  A row whose keys are all masked has lse = -inf (the forward returned zeros): -inf here
// makes its P exactly 0, where -lse = +inf would give exp2(+inf) on a bool row and -inf + inf = NaN on a bias row.
__device__ __forceinline__ float masked_nlse(float lse) { return lse == -INFINITY ? -INFINITY : -lse; }

// P of one visible element of a masked kernel: s its int32 logit, coef its dequant coefficient, m its mask element
template <int kMask, typename T>
__device__ __forceinline__ float masked_p(uint32_t s, float coef, float nlse, uint32_t m) {
  if constexpr (kMask == SAB_MASK_BOOL) {
    return m != 0 ? ex2_approx(logit_log2(s, coef, nlse)) : 0.f;
  } else {
    float bias;
    if constexpr (std::is_same_v<T, __half>) bias = __half2float(__ushort_as_half(uint16_t(m)));
    else bias = __bfloat162float(__ushort_as_bfloat16(uint16_t(m)));
    return ex2_approx(fmaf(__int2float_rn(int(s)), coef, bias) + nlse);   // the forward's tile_bias logit, then - lse
  }
}

// Row stride (elements) of the dK/dV kernel's staged mask tile: the 4 lanes of a quad read 4 different Q rows of one key, and
// these strides put them in different banks (272 / 144 bytes, multiples of 16 for the vector stores)
template <int kMask>
constexpr int kMaskTileRow = kMask == SAB_MASK_BOOL ? 144 : 136;
constexpr size_t kMaskTileBytes = size_t(64) * 136 * 2;   // the larger of the two kinds

// Mask elements of rows [q0, q0 + 64) x keys [k0, k0 + 128) of (b, h) into a row-major tile (Q row r at r * kMaskTileRow);
// elements of rows >= q_len or keys >= kv_len are stored masked (bool 0, bias -inf).  16-byte loads along the keys when the
// keys are contiguous and the rows 16-byte aligned, element loads with general strides otherwise.
template <int kMask, typename T>
__device__ __forceinline__ void load_mask_tile(uint8_t* tile, const AttnParams& a, int b, int h, int q0, int k0, int q_len,
                                               int kv_len) {
  using E = MaskElem<kMask>;
  constexpr int EB = sizeof(E), ROW = kMaskTileRow<kMask>, V = 16 / EB, KB = 128, QB = 64;
  constexpr E fill = kMask == SAB_MASK_BOOL ? E(0) : E(std::is_same_v<T, __half> ? 0xFC00u : 0xFF80u);   // -inf
  const E* base = reinterpret_cast<const E*>(a.mask) + int64_t(b) * a.mask_sb + int64_t(h) * a.mask_sh;
  const bool vec = a.mask_sn == 1 &&
                   ((reinterpret_cast<uintptr_t>(a.mask) | uint64_t(a.mask_sb * EB) | uint64_t(a.mask_sh * EB) | uint64_t(a.mask_sm * EB)) & 15) == 0;
  const int step = vec ? V : 1;
  for (int idx = threadIdx.x * step; idx < QB * KB; idx += kBwdThreads * step) {
    const int r = idx / KB, c = idx % KB, q = q0 + r, key = k0 + c;
    const E* src = base + int64_t(q) * a.mask_sm + int64_t(key) * a.mask_sn;
    E* dst = reinterpret_cast<E*>(tile) + r * ROW + c;
    if (vec && q < q_len && key + V <= kv_len) {
      *reinterpret_cast<uint4*>(dst) = __ldg(reinterpret_cast<const uint4*>(src));
    } else {
      for (int u = 0; u < step; ++u) dst[u] = (q < q_len && key + u < kv_len) ? __ldg(src + u) : fill;   // sn == 1 when step > 1
    }
  }
}

// ------------------------------------------------------------------------------------------------ work decode
// The tokens of this CTA's batch entry (attn.cu's work decode).  Dense: batch b, all Sq / Sk rows.  Varlen: sequence b of the
// packed tensors (stride_b 0), whose scales start at 128-row Q block q_blk0 and 64-key block k_blk0; the scale bases are then h and
// hk (qs_stride_bh = ks_stride_bh = 1, stride qs_stride_idx = Hq / ks_stride_idx = Hkv), the LSE / delta row h*Tq + q_off + row and
// the K mean [Hkv,D] (tb = 0).  Each kernel branches on p.a.cu_q once, at the top, into a body compiled for one form: the dense
// body sees the span as constants (offsets and first blocks 0), so its code is that of a kernel without varlen support.
struct SeqSpan {
  int tb;                          // batch index of the scales, LSE, delta and K mean
  int q_off, q_len, k_off, kv_len;
  int q_blk0, k_blk0;
};
template <bool kVarlen>
__device__ __forceinline__ SeqSpan seq_span(const AttnParams& a, int b) {
  if constexpr (!kVarlen) {
    return SeqSpan{b, 0, a.Sq, 0, a.Sk, 0, 0};
  } else {
    const int q_off = a.cu_q[b], k_off = a.cu_k[b];
    return SeqSpan{0, q_off, a.cu_q[b + 1] - q_off, k_off, a.cu_k[b + 1] - k_off, a.cu_qs[b], a.cu_ks[b]};
  }
}

// ------------------------------------------------------------------------------------------------ delta = rowsum(dO o O)
// one warp per Q row, fixed summation order
template <typename T>
__global__ void __launch_bounds__(256) bwd_delta_kernel(const __grid_constant__ BwdParams p, int D) {
  const int64_t row = int64_t(blockIdx.x) * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= int64_t(p.a.B) * p.a.Hq * p.a.Sq) return;
  const int s = int(row % p.a.Sq), h = int((row / p.a.Sq) % p.a.Hq), b = int(row / (int64_t(p.a.Sq) * p.a.Hq));
  const T* o = reinterpret_cast<const T*>(p.o) + b * p.o_sb + h * p.o_sh + s * p.o_ss;
  const T* g = reinterpret_cast<const T*>(p.dout) + b * p.do_sb + h * p.do_sh + s * p.do_ss;
  float acc = 0.f;
  for (int d = 2 * lane; d < D; d += 64) {
    acc = fmaf(float(o[d]), float(g[d]), acc);
    acc = fmaf(float(o[d + 1]), float(g[d + 1]), acc);
  }
#pragma unroll
  for (int x = 16; x > 0; x >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, x);
  if (lane == 0) p.delta[row] = acc;
}

// ------------------------------------------------------------------------------------------------ dQ
template <int D>
constexpr size_t bwd_dq_smem_bytes() {
  return size_t(128) * D + size_t(128) * D * 2 + size_t(64) * D + size_t(64) * D * 2 + size_t(D) * 64 * 2 + 1024;
}

// dbias (masked, nullable): dense [B,Hq,Sq,Skv] in T, written with ln2 * dS.  kSparse: the block-sparse form, which loops over
// the visible 64-key tiles of its row of *bm (build_kv_list, as the forward does) instead of every tile.  kWindow: the
// sliding-window form, which walks the forward's tile range of the window *win with the forward's per-row bounds lo <= key < limit.
// kSeqMean (varlen): the K mean is [nseq,Hkv,D], one per sequence, instead of one [Hkv,D] mean for the packed batch.
template <int D, bool kKT, typename T, bool kVarlen, int kMask = 0, bool kSparse = false, bool kWindow = false, bool kSeqMean = false>
__device__ __forceinline__ void bwd_dq_tile(const BwdParams& p, void* dbias = nullptr, const BlockMask* bm = nullptr,
                                            const Window* win = nullptr) {
  constexpr int QB = 128, KB = 64;
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* sQ8 = smem;                       // [128 x D] int8        A of S = Q K^T
  uint8_t* sdO = sQ8 + QB * D;               // [128 x D] 16-bit      A of dP = dO V^T
  uint8_t* sK8 = sdO + QB * D * 2;           // [64 x D] int8         B of S
  uint8_t* sV = sK8 + KB * D;                // [64 x D] 16-bit       B of dP
  uint8_t* sKt = sV + KB * D * 2;            // [D x 64] 16-bit       B of dQ += dS K
  [[maybe_unused]] int* s_scratch = reinterpret_cast<int*>(sKt + D * KB * 2);     // block-sparse: build_kv_list's counts
  [[maybe_unused]] uint16_t* s_idx = reinterpret_cast<uint16_t*>(s_scratch + 16); // block-sparse: visible 64-key tiles
  const AttnParams& a = p.a;

  int qt = blockIdx.x;
  if (a.causal) qt = a.n_q_tiles - 1 - qt;   // heaviest tiles first
  const int h = blockIdx.y, b = blockIdx.z;
  const int hk = h / (a.Hq / a.Hkv);
  const SeqSpan sq = seq_span<kVarlen>(a, b);
  if (qt * QB >= sq.q_len) return;           // varlen: a sequence shorter than the longest
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2, t = lane & 3;
  const int row0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // rows row0, row0 + 8 of the Q tile (forward's accumulator layout)

  if ((smem_u32(smem) & 1023u) != 0) __trap();
  load_tile<QB, D, 1>(sQ8, p.q8 + b * p.q8_sb + h * p.q8_sh + sq.q_off * p.q8_ss, p.q8_ss, qt * QB, sq.q_len);
  load_tile<QB, D, 2>(sdO, p.dout + b * p.do_sb + h * p.do_sh + sq.q_off * p.do_ss, p.do_ss, qt * QB, sq.q_len);

  const float* qs_base = a.q_scale + (int64_t(sq.tb) * a.Hq + h) * a.qs_stride_bh;
  const float* ks_base = a.k_scale + (int64_t(sq.tb) * a.Hkv + hk) * a.ks_stride_bh;
  int q_row[2];
  float qss[2], nlse[2], dlt[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    q_row[i] = qt * QB + row0 + 8 * i;
    qss[i] = q_dequant_log2(a, qs_base, sq.q_blk0 + qt, row0 + 8 * i);   // scales are padded to whole 128-row blocks
    const bool ok = q_row[i] < sq.q_len;
    const int64_t li = (int64_t(sq.tb) * a.Hq + h) * a.Sq + sq.q_off + q_row[i];
    if constexpr (kMask != 0 || kSparse || kWindow) nlse[i] = ok ? masked_nlse(p.lse[li]) : -INFINITY;
    else nlse[i] = ok ? -p.lse[li] : 0.f;
    dlt[i] = ok ? p.delta[li] : 0.f;
  }
  // masked: this thread's two rows of the mask (dense, non-varlen); rows >= Sq are never read
  [[maybe_unused]] const MaskElem<kMask>* mrow[2];
  if constexpr (kMask != 0) {
#pragma unroll
    for (int i = 0; i < 2; ++i)
      mrow[i] = reinterpret_cast<const MaskElem<kMask>*>(a.mask) + int64_t(b) * a.mask_sb + int64_t(h) * a.mask_sh +
                int64_t(q_row[i]) * a.mask_sm;
  }
  int n_kv = (sq.kv_len + KB - 1) / KB;
  if (a.causal) n_kv = min(n_kv, ((qt + 1) * QB + KB - 1) / KB);
  if constexpr (kSparse) n_kv = build_kv_list<kBwdThreads>(*bm, b, h, qt, n_kv, s_idx, s_scratch);
  [[maybe_unused]] int j0 = 0;   // window form: the first 64-key tile of the CTA's range
  if constexpr (kWindow) {
    int j1;
    window_tiles(*win, a.causal != 0, qt * QB, min(qt * QB + QB, sq.q_len) - 1, sq.kv_len, j0, j1);
    n_kv = j1 - j0;
  }

  float dq[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) dq[i] = 0.f;

  for (int jt = 0; jt < n_kv; ++jt) {
    int j = kSparse ? int(s_idx[jt]) : jt;   // the 64-key tile of step jt
    if constexpr (kWindow) j = j0 + jt;
    // masked: the mask elements of this thread's S elements of tile j, issued first so that their latency overlaps the tile loads
    // and the MMAs; rows >= Sq and keys >= Skv are not read
    [[maybe_unused]] uint32_t mv[32];
    if constexpr (kMask != 0) {
#pragma unroll
      for (int c = 0; c < 16; ++c) {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int key = j * KB + 8 * (c >> 1) + 2 * t + (c & 1);
          mv[4 * (c >> 1) + 2 * i + (c & 1)] =
              q_row[i] < sq.q_len && key < sq.kv_len ? __ldg(mrow[i] + int64_t(key) * a.mask_sn) : 0u;
        }
      }
    }
    __syncthreads();   // the previous tile's operands are consumed
    load_tile<KB, D, 1>(sK8, p.k8 + b * p.k8_sb + hk * p.k8_sh + sq.k_off * p.k8_ss, p.k8_ss, j * KB, sq.kv_len);
    load_tile<KB, D, 2>(sV, p.v + b * p.v_sb + hk * p.v_sh + sq.k_off * p.v_ss, p.v_ss, j * KB, sq.kv_len);
    // K - mean: the same product in exact arithmetic (the rows of dS sum to zero), but the residue that delta = rowsum(dO o O) of
    // the quantised forward leaves in those row sums is not multiplied by a large K mean
    load_tile_t<D, T>(sKt, p.k + b * p.k_sb + hk * p.k_sh + sq.k_off * p.k_ss, p.k_ss, j * KB, sq.kv_len,
                      p.kmean ? p.kmean + (int64_t(kSeqMean ? b : sq.tb) * a.Hkv + hk) * D : nullptr);
    fence_proxy_async_smem();   // generic-proxy stores -> visible to wgmma
    __syncthreads();

    uint32_t s[32];
    float dp[32];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < D / 32; ++k) wgmma_qk_i8(s, tile_desc<D>(sQ8, QB, wg * 64, 32 * k), tile_desc<D>(sK8, KB, 0, 32 * k), k > 0);
#pragma unroll
    for (int k = 0; k < D / 16; ++k) wgmma_ss<T>(dp, tile_desc<2 * D>(sdO, QB, wg * 64, 32 * k), tile_desc<2 * D>(sV, KB, 0, 32 * k), k > 0);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(s);
    fence_regs(dp);

    float coef[2];
    int limit[2];
    [[maybe_unused]] int lo[2];   // window form: first visible key of the tile per row
    const float ksv = k_dequant<kKT>(a, ks_base, sq.k_blk0 + j, t);
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      coef[i] = ksv * qss[i];
      limit[i] = q_row[i] < sq.q_len ? sq.kv_len - j * KB : 0;
      if (a.causal) limit[i] = min(limit[i], q_row[i] - j * KB + 1);
      if constexpr (kWindow) {
        if (win->right >= 0) limit[i] = min(limit[i], q_row[i] + win->right + 1 - j * KB);
        lo[i] = win->left >= 0 ? q_row[i] - win->left - j * KB : 0;
      }
    }
    float ds[32];
#pragma unroll
    for (int c = 0; c < 16; ++c) {
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int idx = 4 * (c >> 1) + 2 * i + (c & 1);
        const int key = 8 * (c >> 1) + 2 * t + (c & 1);
        float pe;
        if constexpr (kMask != 0)
          pe = key < limit[i] ? masked_p<kMask, T>(s[idx], coef[i], nlse[i], mv[idx]) : 0.f;
        else if constexpr (kWindow)
          pe = key < limit[i] && key >= lo[i] ? ex2_approx(logit_log2(s[idx], coef[i], nlse[i])) : 0.f;
        else
          pe = key < limit[i] ? ex2_approx(logit_log2(s[idx], coef[i], nlse[i])) : 0.f;
        ds[idx] = pe * (dp[idx] - dlt[i]);
      }
    }
    if constexpr (kMask == SAB_MASK_BIAS) {
      // dBias = ln2 * dS of this thread's elements (keys 8n + 2t, 8n + 2t + 1 of both rows), rows < Sq and keys < Skv only
      if (dbias != nullptr) {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          if (q_row[i] >= sq.q_len) continue;
          T* drow = reinterpret_cast<T*>(dbias) + ((int64_t(b) * a.Hq + h) * a.Sq + q_row[i]) * a.Sk;
#pragma unroll
          for (int n = 0; n < 8; ++n) {
            const int key = j * KB + 8 * n + 2 * t, idx = 4 * n + 2 * i;
            const float g0 = kLn2 * ds[idx], g1 = kLn2 * ds[idx + 1];
            if (key + 1 < a.Sk && (a.Sk & 1) == 0) {   // an even row length keeps the pair 4-byte aligned
              *reinterpret_cast<uint32_t*>(drow + key) = pack2<T>(g0, g1);
            } else {
              if (key < a.Sk) drow[key] = T(g0);
              if (key + 1 < a.Sk) drow[key + 1] = T(g1);
            }
          }
        }
      }
    }
    uint32_t da[4][4];
    acc_to_a<T>(ds, da);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) wgmma_rs<T>(dq, da[kk], tile_desc<128>(sKt, D, 0, 32 * kk), 1);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(dq);
  }

  T* base = reinterpret_cast<T*>(p.dq) + b * p.q_sb + h * p.q_sh + sq.q_off * p.q_ss;
  store_rows<T, D>(dq, base + int64_t(q_row[0]) * p.q_ss, base + int64_t(q_row[1]) * p.q_ss, q_row[0] < sq.q_len,
                   q_row[1] < sq.q_len, t, p.sm_scale);
}

template <int D, bool kKT, typename T>
__global__ void __launch_bounds__(kBwdThreads, 1) bwd_dq_kernel(const __grid_constant__ BwdParams p) {
  if (p.a.cu_q != nullptr) bwd_dq_tile<D, kKT, T, true>(p);
  else bwd_dq_tile<D, kKT, T, false>(p);
}

// the varlen form with a per-sequence K mean (sab_qk_int8_attn_bwd_varlen_seq)
template <int D, bool kKT, typename T>
__global__ void __launch_bounds__(kBwdThreads, 1) bwd_dq_varlen_seq_kernel(const __grid_constant__ BwdParams p) {
  bwd_dq_tile<D, kKT, T, true, 0, false, false, true>(p);
}

// the masked form: dense, non-causal, per-block / per-warp K scales (those of the masked forward)
template <int D, typename T>
__global__ void __launch_bounds__(kBwdThreads, 1) bwd_dq_masked_kernel(const __grid_constant__ BwdParams p, void* dbias) {
  if (p.a.mask_kind == SAB_MASK_BOOL) bwd_dq_tile<D, false, T, false, SAB_MASK_BOOL>(p);
  else bwd_dq_tile<D, false, T, false, SAB_MASK_BIAS>(p, dbias);
}

// the block-sparse form: dense, non-varlen; its dynamic shared memory adds kv_list_bytes(ceil(Skv/64))
template <int D, bool kKT, typename T>
__global__ void __launch_bounds__(kBwdThreads, 1) bwd_dq_blocksparse_kernel(const __grid_constant__ BwdParams p,
                                                                             const __grid_constant__ BlockMask bm) {
  bwd_dq_tile<D, kKT, T, false, 0, true>(p, nullptr, &bm);
}

// the sliding-window form: dense, non-varlen
template <int D, bool kKT, typename T>
__global__ void __launch_bounds__(kBwdThreads, 1) bwd_dq_window_kernel(const __grid_constant__ BwdParams p,
                                                                        const __grid_constant__ Window win) {
  bwd_dq_tile<D, kKT, T, false, 0, false, true>(p, nullptr, nullptr, &win);
}

// the packed sliding-window form with a per-sequence K mean: sequence blockIdx.z sees the window clamped at its own lengths, as
// the forward does (seq_window)
template <int D, bool kKT, typename T>
__global__ void __launch_bounds__(kBwdThreads, 1) bwd_dq_varlen_window_kernel(const __grid_constant__ BwdParams p,
                                                                               const __grid_constant__ Window win) {
  const int b = blockIdx.z;
  const Window w = seq_window(win, p.a.cu_q[b + 1] - p.a.cu_q[b], p.a.cu_k[b + 1] - p.a.cu_k[b]);
  bwd_dq_tile<D, kKT, T, true, 0, false, true, true>(p, nullptr, nullptr, &w);
}

// the packed block-sparse form with a per-sequence K mean: sequence blockIdx.z compacts row (sequence, h, its own Q tile) of the
// [nseq,Hq,.,.] mask, as the forward does; its dynamic shared memory adds kv_list_bytes(ceil(max_seqlen_k/64))
template <int D, bool kKT, typename T>
__global__ void __launch_bounds__(kBwdThreads, 1) bwd_dq_varlen_blocksparse_kernel(const __grid_constant__ BwdParams p,
                                                                                    const __grid_constant__ BlockMask bm) {
  bwd_dq_tile<D, kKT, T, true, 0, true, false, true>(p, nullptr, &bm);
}

// ------------------------------------------------------------------------------------------------ dK, dV
template <int D>
constexpr size_t bwd_dkdv_smem_bytes() {
  return size_t(128) * D + size_t(128) * D * 2 + size_t(64) * D + size_t(64) * D * 2 + 2 * size_t(D) * 64 * 2 + 3 * 64 * 4 + 1024;
}

// kSparse: the block-sparse form.  Warpgroup wg's 64 keys are one block of *bm, and a 64-row Q tile lies in one 128-row block, so
// each (Q head, Q tile) step has two mask bits: a step with neither set is skipped (no loads, no barriers; the bits are uniform
// across the CTA), and with one set the other warpgroup takes part in the loads and barriers but adds nothing.
// kWindow: the sliding-window form.  The loop runs only over the 64-row Q tiles that meet rows [k0 - right, k0 + 127 + left] (the
// rows that see a key of the tile under *win), clipped to the causal start, and every element outside the window gets P = 0.
template <int D, bool kKT, typename T, bool kVarlen, int kMask = 0, bool kSparse = false, bool kWindow = false>
__device__ __forceinline__ void bwd_dkdv_tile(const BwdParams& p, const BlockMask* bm = nullptr, const Window* win = nullptr) {
  constexpr int KB = 128, QB = 64;
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* sK8 = smem;                       // [128 x D] int8        A of S^T = K Q^T
  uint8_t* sV = sK8 + KB * D;                // [128 x D] 16-bit      A of dP^T = V dO^T
  uint8_t* sQ8 = sV + KB * D * 2;            // [64 x D] int8         B of S^T
  uint8_t* sdO = sQ8 + QB * D;               // [64 x D] 16-bit       B of dP^T
  uint8_t* sdOt = sdO + QB * D * 2;          // [D x 64] 16-bit       B of dV += P^T dO
  uint8_t* sQt = sdOt + D * QB * 2;          // [D x 64] 16-bit       B of dK += dS^T Q
  float* s_qss = reinterpret_cast<float*>(sQt + D * QB * 2);   // per Q row of the tile: q dequant scale, -lse, delta
  float* s_nlse = s_qss + QB;
  float* s_dlt = s_nlse + QB;
  [[maybe_unused]] uint8_t* s_mask = reinterpret_cast<uint8_t*>(s_dlt + QB);   // masked: [64 Q rows x 128 keys] (load_mask_tile)
  const AttnParams& a = p.a;

  const int k0 = blockIdx.x * KB, hk = blockIdx.y, b = blockIdx.z;
  const SeqSpan sq = seq_span<kVarlen>(a, b);
  if (k0 >= sq.kv_len) return;               // varlen: a sequence shorter than the longest (keys with no queries still store zeros)
  const int G = a.Hq / a.Hkv;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2, t = lane & 3;
  const int kr = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // keys k0 + kr, k0 + kr + 8 (accumulator rows)

  if ((smem_u32(smem) & 1023u) != 0) __trap();
  load_tile<KB, D, 1>(sK8, p.k8 + b * p.k8_sb + hk * p.k8_sh + sq.k_off * p.k8_ss, p.k8_ss, k0, sq.kv_len);
  load_tile<KB, D, 2>(sV, p.v + b * p.v_sb + hk * p.v_sh + sq.k_off * p.v_ss, p.v_ss, k0, sq.kv_len);

  const float* ks_base = a.k_scale + (int64_t(sq.tb) * a.Hkv + hk) * a.ks_stride_bh;
  int key[2];
  float ksr[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    key[i] = k0 + kr + 8 * i;
    // per-thread K scales: key % 8 == lane / 4, so its scale group is lane / 8
    ksr[i] = key[i] < sq.kv_len ? k_dequant<kKT>(a, ks_base, sq.k_blk0 + key[i] / 64, lane >> 3) : 0.f;
  }
  float dk[D / 2], dv[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) dk[i] = dv[i] = 0.f;

  int n_qt = (sq.q_len + QB - 1) / QB;
  int qt0 = a.causal ? k0 / QB : 0;          // causal (top-left): rows before the first key see none of this tile
  if constexpr (kWindow) {
    if (win->right >= 0) qt0 = max(qt0, max(0, k0 - win->right) / QB);
    if (win->left >= 0) n_qt = min(n_qt, (k0 + KB - 1 + win->left) / QB + 1);
  }
  // block-sparse: the raw mask bytes of warpgroup 0's and 1's key blocks for step (hh, qt), loaded one step ahead
  [[maybe_unused]] const int kb0 = 2 * blockIdx.x, n_kb = (sq.kv_len + 63) / 64;
  [[maybe_unused]] uint32_t nxt[2] = {0u, 0u};
  [[maybe_unused]] auto load_bits = [&](int hh, int qt) {
    const uint8_t* r = bm->ptr + int64_t(b) * bm->sb + int64_t(hk * G + hh) * bm->sh + int64_t(qt / 2) * bm->sqb;
    nxt[0] = __ldg(r + int64_t(kb0) * bm->skb);
    nxt[1] = kb0 + 1 < n_kb ? __ldg(r + int64_t(kb0 + 1) * bm->skb) : 0u;
  };
  if constexpr (kSparse) {
    if (qt0 < n_qt) load_bits(0, qt0);
  }
  for (int hh = 0; hh < G; ++hh) {
    const int h = hk * G + hh;
    const float* qs_base = a.q_scale + (int64_t(sq.tb) * a.Hq + h) * a.qs_stride_bh;
    for (int qt = qt0; qt < n_qt; ++qt) {
      const int q0 = qt * QB;
      bool visible = true;   // this warpgroup's keys are visible to Q tile qt of head h
      if constexpr (kSparse) {
        const bool v0 = nxt[0] != 0u, v1 = nxt[1] != 0u;
        if (qt + 1 < n_qt) load_bits(hh, qt + 1);
        else if (hh + 1 < G) load_bits(hh + 1, qt0);
        if (!v0 && !v1) continue;
        visible = wg == 0 ? v0 : v1;
      }
      __syncthreads();   // the previous tile's operands are consumed
      load_tile<QB, D, 1>(sQ8, p.q8 + b * p.q8_sb + h * p.q8_sh + sq.q_off * p.q8_ss, p.q8_ss, q0, sq.q_len);
      load_tile<QB, D, 2>(sdO, p.dout + b * p.do_sb + h * p.do_sh + sq.q_off * p.do_ss, p.do_ss, q0, sq.q_len);
      load_tile_t<D, T>(sdOt, p.dout + b * p.do_sb + h * p.do_sh + sq.q_off * p.do_ss, p.do_ss, q0, sq.q_len);
      load_tile_t<D, T>(sQt, p.q + b * p.q_sb + h * p.q_sh + sq.q_off * p.q_ss, p.q_ss, q0, sq.q_len);
      if constexpr (kMask != 0) load_mask_tile<kMask, T>(s_mask, a, b, h, q0, k0, sq.q_len, sq.kv_len);   // Q head h, not hk
      if (threadIdx.x < QB) {
        const int r = q0 + threadIdx.x;
        const bool ok = r < sq.q_len;
        const int64_t li = (int64_t(sq.tb) * a.Hq + h) * a.Sq + sq.q_off + r;
        int q_blk0 = sq.q_blk0;
        if constexpr (kVarlen && kSparse) q_blk0 = *reinterpret_cast<const volatile int32_t*>(a.cu_qs + b);   // as k_off below
        s_qss[threadIdx.x] = ok ? q_dequant_log2(a, qs_base, q_blk0 + r / 128, r % 128) : 0.f;
        if constexpr (kMask != 0 || kSparse || kWindow) s_nlse[threadIdx.x] = ok ? masked_nlse(p.lse[li]) : -INFINITY;
        else s_nlse[threadIdx.x] = ok ? -p.lse[li] : 0.f;
        s_dlt[threadIdx.x] = ok ? p.delta[li] : 0.f;
      }
      fence_proxy_async_smem();
      __syncthreads();
      if (!visible) continue;   // warpgroup-uniform; the next step starts with a barrier both warpgroups reach

      uint32_t s[32];
      float dp[32];
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < D / 32; ++k) wgmma_qk_i8(s, tile_desc<D>(sK8, KB, wg * 64, 32 * k), tile_desc<D>(sQ8, QB, 0, 32 * k), k > 0);
#pragma unroll
      for (int k = 0; k < D / 16; ++k) wgmma_ss<T>(dp, tile_desc<2 * D>(sV, KB, wg * 64, 32 * k), tile_desc<2 * D>(sdO, QB, 0, 32 * k), k > 0);
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs(s);
      fence_regs(dp);

      // P^T and dS^T: accumulator row = key, column c = Q row q0 + c
      float pt[32], dst[32];
#pragma unroll
      for (int c = 0; c < 16; ++c) {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int idx = 4 * (c >> 1) + 2 * i + (c & 1);
          const int col = 8 * (c >> 1) + 2 * t + (c & 1);
          const int q = q0 + col;
          bool ok = key[i] < sq.kv_len && q < sq.q_len && (!a.causal || key[i] <= q);
          if constexpr (kWindow) ok = ok && (win->left < 0 || q - key[i] <= win->left) && (win->right < 0 || key[i] - q <= win->right);
          float pe;
          if constexpr (kMask != 0)
            pe = ok ? masked_p<kMask, T>(s[idx], ksr[i] * s_qss[col], s_nlse[col],
                                         reinterpret_cast<const MaskElem<kMask>*>(s_mask)[col * kMaskTileRow<kMask> + kr + 8 * i])
                    : 0.f;
          else
            pe = ok ? ex2_approx(logit_log2(s[idx], ksr[i] * s_qss[col], s_nlse[col])) : 0.f;
          pt[idx] = pe;
          dst[idx] = pe * (dp[idx] - s_dlt[col]);
        }
      }
      uint32_t pa[4][4], da[4][4];
      acc_to_a<T>(pt, pa);
      acc_to_a<T>(dst, da);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) wgmma_rs<T>(dv, pa[kk], tile_desc<128>(sdOt, D, 0, 32 * kk), 1);
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) wgmma_rs<T>(dk, da[kk], tile_desc<128>(sQt, D, 0, 32 * kk), 1);
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs(dv);
      fence_regs(dk);
    }
  }

  // the packed block-sparse form reads its sequence's first key (and, per step, its first Q scale block) again instead of
  // holding them through the loop: at D = 128 those registers keep the kernel within 255 without a spill
  int k_off = sq.k_off;
  if constexpr (kVarlen && kSparse) k_off = *reinterpret_cast<const volatile int32_t*>(a.cu_k + b);
  T* kb = reinterpret_cast<T*>(p.dk) + b * p.k_sb + hk * p.k_sh + k_off * p.k_ss;
  T* vb = reinterpret_cast<T*>(p.dv) + b * p.v_sb + hk * p.v_sh + k_off * p.v_ss;
  const bool ok0 = key[0] < sq.kv_len, ok1 = key[1] < sq.kv_len;
  store_rows<T, D>(dk, kb + int64_t(key[0]) * p.k_ss, kb + int64_t(key[1]) * p.k_ss, ok0, ok1, t, p.sm_scale);
  store_rows<T, D>(dv, vb + int64_t(key[0]) * p.v_ss, vb + int64_t(key[1]) * p.v_ss, ok0, ok1, t, 1.0f);
}

template <int D, bool kKT, typename T>
__global__ void __launch_bounds__(kBwdThreads, 1) bwd_dkdv_kernel(const __grid_constant__ BwdParams p) {
  if (p.a.cu_q != nullptr) bwd_dkdv_tile<D, kKT, T, true>(p);
  else bwd_dkdv_tile<D, kKT, T, false>(p);
}

template <int D, typename T>
__global__ void __launch_bounds__(kBwdThreads, 1) bwd_dkdv_masked_kernel(const __grid_constant__ BwdParams p) {
  if (p.a.mask_kind == SAB_MASK_BOOL) bwd_dkdv_tile<D, false, T, false, SAB_MASK_BOOL>(p);
  else bwd_dkdv_tile<D, false, T, false, SAB_MASK_BIAS>(p);
}

template <int D, bool kKT, typename T>
__global__ void __launch_bounds__(kBwdThreads, 1) bwd_dkdv_blocksparse_kernel(const __grid_constant__ BwdParams p,
                                                                               const __grid_constant__ BlockMask bm) {
  bwd_dkdv_tile<D, kKT, T, false, 0, true>(p, &bm);
}

template <int D, bool kKT, typename T>
__global__ void __launch_bounds__(kBwdThreads, 1) bwd_dkdv_window_kernel(const __grid_constant__ BwdParams p,
                                                                          const __grid_constant__ Window win) {
  bwd_dkdv_tile<D, kKT, T, false, 0, false, true>(p, nullptr, &win);
}

template <int D, bool kKT, typename T>
__global__ void __launch_bounds__(kBwdThreads, 1) bwd_dkdv_varlen_window_kernel(const __grid_constant__ BwdParams p,
                                                                                 const __grid_constant__ Window win) {
  const int b = blockIdx.z;
  const Window w = seq_window(win, p.a.cu_q[b + 1] - p.a.cu_q[b], p.a.cu_k[b + 1] - p.a.cu_k[b]);
  bwd_dkdv_tile<D, kKT, T, true, 0, false, true>(p, nullptr, &w);
}

// the packed block-sparse form: the mask bits of (sequence blockIdx.z, Q head, its own Q tile, its own key blocks)
template <int D, bool kKT, typename T>
__global__ void __launch_bounds__(kBwdThreads, 1) bwd_dkdv_varlen_blocksparse_kernel(const __grid_constant__ BwdParams p,
                                                                                      const __grid_constant__ BlockMask bm) {
  bwd_dkdv_tile<D, kKT, T, true, 0, true>(p, &bm);
}

// delta, then the dQ kernel kq (smem_q bytes, arguments p, q_args...) and the dK/dV kernel kkv (smem_kv bytes); cfg_*: their
// per-device smem opt-in
template <typename T>
static int launch_bwd_delta(const BwdParams& p, int D, cudaStream_t stream) {
  BwdParams pd = p;
  if (p.a.cu_q != nullptr) pd.a.B = 1;   // varlen: every packed row, [Hq,Tq] like the LSE
  const int64_t rows = int64_t(pd.a.B) * pd.a.Hq * pd.a.Sq;
  bwd_delta_kernel<T><<<unsigned((rows + 7) / 8), 256, 0, stream>>>(pd, D);
  SAB_CUDA_OK(cudaGetLastError());
  return SAB_OK;
}

template <typename T, typename KQ, typename KKV, typename... QArgs>
static int launch_bwd_kernels(const BwdParams& p, int D, KQ kq, size_t smem_q, bool (&cfg_q)[64], KKV kkv, size_t smem_kv,
                              bool (&cfg_kv)[64], cudaStream_t stream, QArgs... q_args) {
  if (int st = launch_bwd_delta<T>(p, D, stream)) return st;
  if (int st = ensure_dynamic_smem(kq, smem_q, cfg_q)) return st;
  kq<<<dim3(p.a.n_q_tiles, p.a.Hq, p.a.B), kBwdThreads, smem_q, stream>>>(p, q_args...);
  SAB_CUDA_OK(cudaGetLastError());
  if (int st = ensure_dynamic_smem(kkv, smem_kv, cfg_kv)) return st;
  kkv<<<dim3(p.n_k_tiles, p.a.Hkv, p.a.B), kBwdThreads, smem_kv, stream>>>(p);
  SAB_CUDA_OK(cudaGetLastError());
  return SAB_OK;
}

template <int D, bool kKT, typename T>
static int launch_bwd(const BwdParams& p, cudaStream_t stream) {
  static bool cfg_q[64] = {}, cfg_kv[64] = {};
  return launch_bwd_kernels<T>(p, D, bwd_dq_kernel<D, kKT, T>, bwd_dq_smem_bytes<D>(), cfg_q, bwd_dkdv_kernel<D, kKT, T>,
                               bwd_dkdv_smem_bytes<D>(), cfg_kv, stream);
}

// varlen with a per-sequence K mean: its own dQ kernel; the dK/dV kernel does not read the mean
template <int D, bool kKT, typename T>
static int launch_bwd_varlen_seq(const BwdParams& p, cudaStream_t stream) {
  static bool cfg_q[64] = {}, cfg_kv[64] = {};
  return launch_bwd_kernels<T>(p, D, bwd_dq_varlen_seq_kernel<D, kKT, T>, bwd_dq_smem_bytes<D>(), cfg_q, bwd_dkdv_kernel<D, kKT, T>,
                               bwd_dkdv_smem_bytes<D>(), cfg_kv, stream);
}

template <int D, typename T>
static int launch_bwd_masked(const BwdParams& p, void* dbias, cudaStream_t stream) {
  static bool cfg_q[64] = {}, cfg_kv[64] = {};
  return launch_bwd_kernels<T>(p, D, bwd_dq_masked_kernel<D, T>, bwd_dq_smem_bytes<D>(), cfg_q, bwd_dkdv_masked_kernel<D, T>,
                               bwd_dkdv_smem_bytes<D>() + kMaskTileBytes, cfg_kv, stream, dbias);
}

// kVarlen: the packed form (grids sized from the longest sequence by the caller).  max_k: the longest key range a dQ CTA compacts
// (Skv dense, max_seqlen_k packed).
template <int D, bool kKT, typename T, bool kVarlen = false>
static int launch_bwd_blocksparse(const BwdParams& p, const BlockMask& bm, int max_k, cudaStream_t stream) {
  static bool cfg_q[64] = {}, cfg_kv[64] = {};
  if (int st = launch_bwd_delta<T>(p, D, stream)) return st;
  auto kq = kVarlen ? bwd_dq_varlen_blocksparse_kernel<D, kKT, T> : bwd_dq_blocksparse_kernel<D, kKT, T>;
  const size_t smem_q = bwd_dq_smem_bytes<D>() + kv_list_bytes((max_k + BN - 1) / BN);
  if (int st = ensure_dynamic_smem(kq, bwd_dq_smem_bytes<D>() + kv_list_bytes(kMaxKvBlocks), cfg_q)) return st;
  kq<<<dim3(p.a.n_q_tiles, p.a.Hq, p.a.B), kBwdThreads, smem_q, stream>>>(p, bm);
  SAB_CUDA_OK(cudaGetLastError());
  auto kkv = kVarlen ? bwd_dkdv_varlen_blocksparse_kernel<D, kKT, T> : bwd_dkdv_blocksparse_kernel<D, kKT, T>;
  if (int st = ensure_dynamic_smem(kkv, bwd_dkdv_smem_bytes<D>(), cfg_kv)) return st;
  kkv<<<dim3(p.n_k_tiles, p.a.Hkv, p.a.B), kBwdThreads, bwd_dkdv_smem_bytes<D>(), stream>>>(p, bm);
  SAB_CUDA_OK(cudaGetLastError());
  return SAB_OK;
}

// kVarlen: the packed form (grids sized from the longest sequence by the caller, as for sab_qk_int8_attn_bwd_varlen_seq)
template <int D, bool kKT, typename T, bool kVarlen = false>
static int launch_bwd_window(const BwdParams& p, const Window& w, cudaStream_t stream) {
  static bool cfg_q[64] = {}, cfg_kv[64] = {};
  if (int st = launch_bwd_delta<T>(p, D, stream)) return st;
  auto kq = kVarlen ? bwd_dq_varlen_window_kernel<D, kKT, T> : bwd_dq_window_kernel<D, kKT, T>;
  if (int st = ensure_dynamic_smem(kq, bwd_dq_smem_bytes<D>(), cfg_q)) return st;
  kq<<<dim3(p.a.n_q_tiles, p.a.Hq, p.a.B), kBwdThreads, bwd_dq_smem_bytes<D>(), stream>>>(p, w);
  SAB_CUDA_OK(cudaGetLastError());
  auto kkv = kVarlen ? bwd_dkdv_varlen_window_kernel<D, kKT, T> : bwd_dkdv_window_kernel<D, kKT, T>;
  if (int st = ensure_dynamic_smem(kkv, bwd_dkdv_smem_bytes<D>(), cfg_kv)) return st;
  kkv<<<dim3(p.n_k_tiles, p.a.Hkv, p.a.B), kBwdThreads, bwd_dkdv_smem_bytes<D>(), stream>>>(p, w);
  SAB_CUDA_OK(cudaGetLastError());
  return SAB_OK;
}

// The first checks of every entry, after its window / block-mask checks: the forward's codes and messages (attn.cu).  B / Sq / Skv
// are nseq / Tq / Tk for the packed entries.
static int check_bwd_args(const int8_t* q_int8, const int8_t* k_int8, const float* q_scale, const float* k_scale, const void* q,
                          const void* k, const void* v, const void* o, const void* dout, const float* lse, const void* dq,
                          const void* dk, const void* dv, const void* workspace, int dtype, int B, int Hq, int Hkv, int Sq, int Skv,
                          int D) {
  SAB_REQUIRE(q_int8 && k_int8 && q_scale && k_scale && q && k && v && o && dout && lse && dq && dk && dv && workspace,
              SAB_ERR_INVALID, "null tensor pointer");
  SAB_REQUIRE(D == 64 || D == 128, SAB_ERR_UNSUPPORTED, "Unsupported head dim: %d (64 or 128 after padding)", D);
  SAB_REQUIRE(dtype == SAB_DTYPE_FP16 || dtype == SAB_DTYPE_BF16, SAB_ERR_UNSUPPORTED, "dtype must be fp16 or bf16");
  SAB_REQUIRE(B > 0 && Hq > 0 && Hkv > 0 && Sq > 0 && Skv > 0, SAB_ERR_INVALID, "bad sizes B=%d Hq=%d Hkv=%d Sq=%d Skv=%d", B, Hq, Hkv, Sq, Skv);
  SAB_REQUIRE(Hq % Hkv == 0, SAB_ERR_INVALID, "num_qo_heads (%d) must be divisible by num_kv_heads (%d)", Hq, Hkv);
  return SAB_OK;
}

// The last checks of every entry, then the device check.  st: (b, h, s) element strides of q8, k8, q, k, v, o, dout.
static int check_bwd_layout(const int8_t* q_int8, const int8_t* k_int8, const void* q, const void* k, const void* v,
                            const void* o, const void* dout, void* dq, void* dk, void* dv, const int64_t (&st)[21]) {
  bool ok16 = aligned16(q) && aligned16(k) && aligned16(v) && aligned16(o) && aligned16(dout) && aligned16(dq) && aligned16(dk) && aligned16(dv);
  for (int i = 6; i < 21; ++i) ok16 = ok16 && st[i] % 8 == 0;
  SAB_REQUIRE(ok16, SAB_ERR_INVALID, "16-bit tensors must be 16-byte aligned with strides multiple of 8 elements");
  bool ok8 = aligned16(q_int8) && aligned16(k_int8);
  for (int i = 0; i < 6; ++i) ok8 = ok8 && st[i] % 16 == 0;
  SAB_REQUIRE(ok8, SAB_ERR_INVALID, "int8 tensors must be 16-byte aligned with strides multiple of 16");
  return sab_check_device();
}

// The parameters every entry fills; the packed entries then add their sequence tables
static BwdParams bwd_params(const int8_t* q_int8, const int8_t* k_int8, const float* q_scale, const float* k_scale, const void* q,
                            const void* k, const void* v, const void* o, const void* dout, const float* lse, const void* k_mean,
                            void* dq, void* dk, void* dv, void* workspace, int B, int Hq, int Hkv, int Sq, int Skv,
                            const int64_t (&st)[21], int is_causal, int q_gran, int k_gran, float sm_scale, int fold_sm_scale) {
  BwdParams p{};
  AttnParams& a = p.a;
  a.q_scale = q_scale; a.k_scale = k_scale;
  a.B = B; a.Hq = Hq; a.Hkv = Hkv; a.Sq = Sq; a.Sk = Skv;
  a.n_q_tiles = (Sq + BM - 1) / BM;
  p.n_k_tiles = (Skv + 127) / 128;
  a.causal = is_causal ? 1 : 0;
  a.sm_scale_log2 = fold_sm_scale ? 1.0f : sm_scale * 1.44269504088896340736f;   // as the forward (attn.cu)
  a.q_gran = q_gran;
  a.q_mult = q_gran == SAB_GRAN_PER_BLOCK ? 1 : (q_gran == SAB_GRAN_PER_WARP ? 4 : 32);
  a.k_mult = k_gran == SAB_GRAN_PER_THREAD ? 4 : 1;
  a.qs_stride_bh = int64_t((Sq + BM - 1) / BM) * a.q_mult;
  a.ks_stride_bh = int64_t((Skv + 63) / 64) * a.k_mult;
  a.qs_stride_idx = 1;
  a.ks_stride_idx = 1;
  p.q8 = q_int8; p.k8 = k_int8;
  p.q8_sb = st[0]; p.q8_sh = st[1]; p.q8_ss = st[2];
  p.k8_sb = st[3]; p.k8_sh = st[4]; p.k8_ss = st[5];
  p.q = static_cast<const uint16_t*>(q); p.k = static_cast<const uint16_t*>(k); p.v = static_cast<const uint16_t*>(v);
  p.o = static_cast<const uint16_t*>(o); p.dout = static_cast<const uint16_t*>(dout);
  p.kmean = static_cast<const uint16_t*>(k_mean);
  p.q_sb = st[6]; p.q_sh = st[7]; p.q_ss = st[8];
  p.k_sb = st[9]; p.k_sh = st[10]; p.k_ss = st[11];
  p.v_sb = st[12]; p.v_sh = st[13]; p.v_ss = st[14];
  p.o_sb = st[15]; p.o_sh = st[16]; p.o_ss = st[17];
  p.do_sb = st[18]; p.do_sh = st[19]; p.do_ss = st[20];
  p.lse = lse;
  p.delta = static_cast<float*>(workspace);
  p.dq = dq; p.dk = dk; p.dv = dv;
  p.sm_scale = sm_scale;
  return p;
}

static int dispatch_bwd(const BwdParams& p, int D, int dtype, int k_gran, void* stream) {
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const bool kt = k_gran == SAB_GRAN_PER_THREAD;
  const bool bf = dtype == SAB_DTYPE_BF16;
  if (D == 128) {
    if (kt) { if (bf) return launch_bwd<128, true, __nv_bfloat16>(p, s); return launch_bwd<128, true, __half>(p, s); }
    if (bf) return launch_bwd<128, false, __nv_bfloat16>(p, s);
    return launch_bwd<128, false, __half>(p, s);
  }
  if (kt) { if (bf) return launch_bwd<64, true, __nv_bfloat16>(p, s); return launch_bwd<64, true, __half>(p, s); }
  if (bf) return launch_bwd<64, false, __nv_bfloat16>(p, s);
  return launch_bwd<64, false, __half>(p, s);
}

}  // namespace sab

extern "C" int64_t sab_attn_bwd_workspace_bytes(int B, int Hq, int Sq) {
  if (B <= 0 || Hq <= 0 || Sq <= 0) return 0;
  return (int64_t(B) * Hq * Sq * 4 + 255) / 256 * 256;
}

// sab_qk_int8_attn_bwd and, with a window w or a block mask bm (already checked) or an attention mask m and its nullable dbias,
// sab_qk_int8_attn_bwd_window / sab_qk_int8_attn_bwd_blocksparse / sab_qk_int8_attn_bwd_masked
static int bwd_dense(const int8_t* q_int8, const int8_t* k_int8, const float* q_scale, const float* k_scale, const void* q,
                     const void* k, const void* v, const void* o, const void* dout, const float* lse, const void* k_mean, void* dq,
                     void* dk, void* dv, void* workspace, int dtype, int B, int Hq, int Hkv, int Sq, int Skv, int D,
                     int64_t q8_stride_b, int64_t q8_stride_h, int64_t q8_stride_s, int64_t k8_stride_b, int64_t k8_stride_h,
                     int64_t k8_stride_s, int64_t q_stride_b, int64_t q_stride_h, int64_t q_stride_s, int64_t k_stride_b,
                     int64_t k_stride_h, int64_t k_stride_s, int64_t v_stride_b, int64_t v_stride_h, int64_t v_stride_s,
                     int64_t o_stride_b, int64_t o_stride_h, int64_t o_stride_s, int64_t do_stride_b, int64_t do_stride_h,
                     int64_t do_stride_s, int is_causal, int q_gran, int k_gran, float sm_scale, int fold_sm_scale,
                     const sab::Window* w, const sab::BlockMask* bm, const sab::MaskArgs* m, void* dbias, void* stream) {
  using namespace sab;
  if (int e = check_bwd_args(q_int8, k_int8, q_scale, k_scale, q, k, v, o, dout, lse, dq, dk, dv, workspace, dtype, B, Hq, Hkv, Sq, Skv, D))
    return e;
  SAB_REQUIRE(q_gran >= 1 && q_gran <= 3 && k_gran >= 1 && k_gran <= 3, SAB_ERR_INVALID, "unknown quant granularity q=%d k=%d", q_gran, k_gran);
  SAB_REQUIRE(!is_causal || Sq == Skv, SAB_ERR_INVALID, "qo_len and kv_len must be equal for causal attention.");
  if (m != nullptr) {
    // the masked forward's checks (attn.cu), then the gradient's own
    SAB_REQUIRE(k_gran != SAB_GRAN_PER_THREAD, SAB_ERR_UNSUPPORTED,
                "attn_mask is supported by the dense non-causal fp16-PV path with per-block / per-warp K scales only");
    SAB_REQUIRE(m->ptr != nullptr && (m->kind == SAB_MASK_BOOL || m->kind == SAB_MASK_BIAS), SAB_ERR_INVALID,
                "attn_mask: null pointer or unknown kind %d", m->kind);
    SAB_REQUIRE(dbias == nullptr || m->kind == SAB_MASK_BIAS, SAB_ERR_INVALID, "dbias needs an additive bias mask (SAB_MASK_BIAS)");
    SAB_REQUIRE(aligned16(dbias), SAB_ERR_INVALID, "dbias must be 16-byte aligned");
  }
  const int64_t st[21] = {q8_stride_b, q8_stride_h, q8_stride_s, k8_stride_b, k8_stride_h, k8_stride_s, q_stride_b, q_stride_h, q_stride_s,
                          k_stride_b, k_stride_h, k_stride_s, v_stride_b, v_stride_h, v_stride_s, o_stride_b, o_stride_h, o_stride_s,
                          do_stride_b, do_stride_h, do_stride_s};
  if (int e = check_bwd_layout(q_int8, k_int8, q, k, v, o, dout, dq, dk, dv, st)) return e;
  BwdParams p = bwd_params(q_int8, k_int8, q_scale, k_scale, q, k, v, o, dout, lse, k_mean, dq, dk, dv, workspace, B, Hq, Hkv, Sq, Skv,
                           st, is_causal, q_gran, k_gran, sm_scale, fold_sm_scale);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const bool kt = k_gran == SAB_GRAN_PER_THREAD;
  const bool bf = dtype == SAB_DTYPE_BF16;
  if (m != nullptr) {
    p.a.mask = m->ptr; p.a.mask_kind = m->kind;
    p.a.mask_sb = m->sb; p.a.mask_sh = m->sh; p.a.mask_sm = m->sm; p.a.mask_sn = m->sn;
    if (D == 128) return bf ? launch_bwd_masked<128, __nv_bfloat16>(p, dbias, s) : launch_bwd_masked<128, __half>(p, dbias, s);
    return bf ? launch_bwd_masked<64, __nv_bfloat16>(p, dbias, s) : launch_bwd_masked<64, __half>(p, dbias, s);
  }
  if (w != nullptr) {
    if (D == 128) {
      if (kt) return bf ? launch_bwd_window<128, true, __nv_bfloat16>(p, *w, s) : launch_bwd_window<128, true, __half>(p, *w, s);
      return bf ? launch_bwd_window<128, false, __nv_bfloat16>(p, *w, s) : launch_bwd_window<128, false, __half>(p, *w, s);
    }
    if (kt) return bf ? launch_bwd_window<64, true, __nv_bfloat16>(p, *w, s) : launch_bwd_window<64, true, __half>(p, *w, s);
    return bf ? launch_bwd_window<64, false, __nv_bfloat16>(p, *w, s) : launch_bwd_window<64, false, __half>(p, *w, s);
  }
  if (bm != nullptr) {
    if (D == 128) {
      if (kt) return bf ? launch_bwd_blocksparse<128, true, __nv_bfloat16>(p, *bm, Skv, s) : launch_bwd_blocksparse<128, true, __half>(p, *bm, Skv, s);
      return bf ? launch_bwd_blocksparse<128, false, __nv_bfloat16>(p, *bm, Skv, s) : launch_bwd_blocksparse<128, false, __half>(p, *bm, Skv, s);
    }
    if (kt) return bf ? launch_bwd_blocksparse<64, true, __nv_bfloat16>(p, *bm, Skv, s) : launch_bwd_blocksparse<64, true, __half>(p, *bm, Skv, s);
    return bf ? launch_bwd_blocksparse<64, false, __nv_bfloat16>(p, *bm, Skv, s) : launch_bwd_blocksparse<64, false, __half>(p, *bm, Skv, s);
  }
  return dispatch_bwd(p, D, dtype, k_gran, stream);
}

extern "C" int sab_qk_int8_attn_bwd(const int8_t* q_int8, const int8_t* k_int8, const float* q_scale, const float* k_scale,
                                    const void* q, const void* k, const void* v, const void* o, const void* dout, const float* lse,
                                    const void* k_mean, void* dq, void* dk, void* dv, void* workspace, int dtype, int B, int Hq, int Hkv, int Sq,
                                    int Skv, int D, int64_t q8_stride_b, int64_t q8_stride_h, int64_t q8_stride_s,
                                    int64_t k8_stride_b, int64_t k8_stride_h, int64_t k8_stride_s, int64_t q_stride_b,
                                    int64_t q_stride_h, int64_t q_stride_s, int64_t k_stride_b, int64_t k_stride_h,
                                    int64_t k_stride_s, int64_t v_stride_b, int64_t v_stride_h, int64_t v_stride_s,
                                    int64_t o_stride_b, int64_t o_stride_h, int64_t o_stride_s, int64_t do_stride_b,
                                    int64_t do_stride_h, int64_t do_stride_s, int is_causal, int q_gran, int k_gran,
                                    float sm_scale, int fold_sm_scale, void* stream) {
  return bwd_dense(q_int8, k_int8, q_scale, k_scale, q, k, v, o, dout, lse, k_mean, dq, dk, dv, workspace, dtype, B, Hq, Hkv, Sq, Skv, D,
                   q8_stride_b, q8_stride_h, q8_stride_s, k8_stride_b, k8_stride_h, k8_stride_s, q_stride_b, q_stride_h, q_stride_s,
                   k_stride_b, k_stride_h, k_stride_s, v_stride_b, v_stride_h, v_stride_s, o_stride_b, o_stride_h, o_stride_s,
                   do_stride_b, do_stride_h, do_stride_s, is_causal, q_gran, k_gran, sm_scale, fold_sm_scale, nullptr, nullptr, nullptr,
                   nullptr, stream);
}

extern "C" int sab_qk_int8_attn_bwd_varlen(const int8_t* q_int8, const int8_t* k_int8, const float* q_scale, const float* k_scale,
                                           const void* q, const void* k, const void* v, const void* o, const void* dout,
                                           const float* lse, const void* k_mean, void* dq, void* dk, void* dv, void* workspace,
                                           int dtype, int nseq, int Hq, int Hkv, int Tq, int Tk, int D, int64_t q8_stride_t,
                                           int64_t q8_stride_h, int64_t k8_stride_t, int64_t k8_stride_h, int64_t q_stride_t,
                                           int64_t q_stride_h, int64_t k_stride_t, int64_t k_stride_h, int64_t v_stride_t,
                                           int64_t v_stride_h, int64_t o_stride_t, int64_t o_stride_h, int64_t do_stride_t,
                                           int64_t do_stride_h, const int32_t* cu_seqlens_q, const int32_t* cu_seqlens_k,
                                           const int32_t* cu_q_scale, const int32_t* cu_k_scale, int max_seqlen_q,
                                           int max_seqlen_k, int is_causal, float sm_scale, int fold_sm_scale, void* stream) {
  using namespace sab;
  if (int e = check_bwd_args(q_int8, k_int8, q_scale, k_scale, q, k, v, o, dout, lse, dq, dk, dv, workspace, dtype, nseq, Hq, Hkv, Tq, Tk, D))
    return e;
  SAB_REQUIRE(cu_seqlens_q && cu_seqlens_k && cu_q_scale && cu_k_scale && max_seqlen_q > 0 && max_seqlen_k > 0, SAB_ERR_INVALID,
              "varlen needs cu_seqlens_q, cu_seqlens_k, cu_q_scale, cu_k_scale, max_seqlen_q and max_seqlen_k");
  // packed [T,H,D]: no batch stride
  const int64_t st[21] = {0, q8_stride_h, q8_stride_t, 0, k8_stride_h, k8_stride_t, 0, q_stride_h, q_stride_t, 0, k_stride_h, k_stride_t,
                          0, v_stride_h, v_stride_t, 0, o_stride_h, o_stride_t, 0, do_stride_h, do_stride_t};
  if (int e = check_bwd_layout(q_int8, k_int8, q, k, v, o, dout, dq, dk, dv, st)) return e;
  BwdParams p = bwd_params(q_int8, k_int8, q_scale, k_scale, q, k, v, o, dout, lse, k_mean, dq, dk, dv, workspace, nseq, Hq, Hkv, Tq, Tk,
                           st, is_causal, SAB_GRAN_PER_BLOCK, SAB_GRAN_PER_BLOCK, sm_scale, fold_sm_scale);
  AttnParams& a = p.a;
  a.n_q_tiles = (max_seqlen_q + BM - 1) / BM;
  p.n_k_tiles = (max_seqlen_k + 127) / 128;
  a.qs_stride_bh = a.ks_stride_bh = 1;   // scale bases h / hk (batch index 0), blocks [nblocks,H]: the forward's varlen indexing
  a.qs_stride_idx = Hq;
  a.ks_stride_idx = Hkv;
  a.cu_q = cu_seqlens_q; a.cu_k = cu_seqlens_k; a.cu_qs = cu_q_scale; a.cu_ks = cu_k_scale;
  return dispatch_bwd(p, D, dtype, SAB_GRAN_PER_BLOCK, stream);
}

extern "C" int sab_qk_int8_attn_bwd_masked(const int8_t* q_int8, const int8_t* k_int8, const float* q_scale, const float* k_scale,
                                           const void* q, const void* k, const void* v, const void* o, const void* dout,
                                           const float* lse, const void* k_mean, void* dq, void* dk, void* dv, void* workspace,
                                           int dtype, int B, int Hq, int Hkv, int Sq, int Skv, int D, int64_t q8_stride_b,
                                           int64_t q8_stride_h, int64_t q8_stride_s, int64_t k8_stride_b, int64_t k8_stride_h,
                                           int64_t k8_stride_s, int64_t q_stride_b, int64_t q_stride_h, int64_t q_stride_s,
                                           int64_t k_stride_b, int64_t k_stride_h, int64_t k_stride_s, int64_t v_stride_b,
                                           int64_t v_stride_h, int64_t v_stride_s, int64_t o_stride_b, int64_t o_stride_h,
                                           int64_t o_stride_s, int64_t do_stride_b, int64_t do_stride_h, int64_t do_stride_s,
                                           int q_gran, int k_gran, float sm_scale, int fold_sm_scale, const void* attn_mask,
                                           int mask_kind, int64_t mask_stride_b, int64_t mask_stride_h, int64_t mask_stride_m,
                                           int64_t mask_stride_n, void* dbias, void* stream) {
  const sab::MaskArgs m{attn_mask, mask_kind, mask_stride_b, mask_stride_h, mask_stride_m, mask_stride_n};
  return bwd_dense(q_int8, k_int8, q_scale, k_scale, q, k, v, o, dout, lse, k_mean, dq, dk, dv, workspace, dtype, B, Hq, Hkv, Sq, Skv, D,
                   q8_stride_b, q8_stride_h, q8_stride_s, k8_stride_b, k8_stride_h, k8_stride_s, q_stride_b, q_stride_h, q_stride_s,
                   k_stride_b, k_stride_h, k_stride_s, v_stride_b, v_stride_h, v_stride_s, o_stride_b, o_stride_h, o_stride_s,
                   do_stride_b, do_stride_h, do_stride_s, 0, q_gran, k_gran, sm_scale, fold_sm_scale, nullptr, nullptr, &m, dbias,
                   stream);
}

extern "C" int sab_qk_int8_attn_bwd_blocksparse(const int8_t* q_int8, const int8_t* k_int8, const float* q_scale,
                                                const float* k_scale, const void* q, const void* k, const void* v, const void* o,
                                                const void* dout, const float* lse, const void* k_mean, void* dq, void* dk, void* dv,
                                                void* workspace, int dtype, int B, int Hq, int Hkv, int Sq, int Skv, int D,
                                                int64_t q8_stride_b, int64_t q8_stride_h, int64_t q8_stride_s, int64_t k8_stride_b,
                                                int64_t k8_stride_h, int64_t k8_stride_s, int64_t q_stride_b, int64_t q_stride_h,
                                                int64_t q_stride_s, int64_t k_stride_b, int64_t k_stride_h, int64_t k_stride_s,
                                                int64_t v_stride_b, int64_t v_stride_h, int64_t v_stride_s, int64_t o_stride_b,
                                                int64_t o_stride_h, int64_t o_stride_s, int64_t do_stride_b, int64_t do_stride_h,
                                                int64_t do_stride_s, int is_causal, int q_gran, int k_gran, float sm_scale,
                                                int fold_sm_scale, const uint8_t* block_mask, int64_t mask_stride_b,
                                                int64_t mask_stride_h, int64_t mask_stride_qb, int64_t mask_stride_kb, void* stream) {
  if (int e = sab::check_block_mask(block_mask, mask_stride_b, mask_stride_h, mask_stride_qb, mask_stride_kb, q_gran, is_causal, Sq, Skv))
    return e;
  const sab::BlockMask bm{block_mask, mask_stride_b, mask_stride_h, mask_stride_qb, mask_stride_kb};
  return bwd_dense(q_int8, k_int8, q_scale, k_scale, q, k, v, o, dout, lse, k_mean, dq, dk, dv, workspace, dtype, B, Hq, Hkv, Sq, Skv, D,
                   q8_stride_b, q8_stride_h, q8_stride_s, k8_stride_b, k8_stride_h, k8_stride_s, q_stride_b, q_stride_h, q_stride_s,
                   k_stride_b, k_stride_h, k_stride_s, v_stride_b, v_stride_h, v_stride_s, o_stride_b, o_stride_h, o_stride_s,
                   do_stride_b, do_stride_h, do_stride_s, is_causal, q_gran, k_gran, sm_scale, fold_sm_scale, nullptr, &bm, nullptr,
                   nullptr, stream);
}

extern "C" int sab_qk_int8_attn_bwd_window(const int8_t* q_int8, const int8_t* k_int8, const float* q_scale, const float* k_scale,
                                           const void* q, const void* k, const void* v, const void* o, const void* dout,
                                           const float* lse, const void* k_mean, void* dq, void* dk, void* dv, void* workspace,
                                           int dtype, int B, int Hq, int Hkv, int Sq, int Skv, int D, int64_t q8_stride_b,
                                           int64_t q8_stride_h, int64_t q8_stride_s, int64_t k8_stride_b, int64_t k8_stride_h,
                                           int64_t k8_stride_s, int64_t q_stride_b, int64_t q_stride_h, int64_t q_stride_s,
                                           int64_t k_stride_b, int64_t k_stride_h, int64_t k_stride_s, int64_t v_stride_b,
                                           int64_t v_stride_h, int64_t v_stride_s, int64_t o_stride_b, int64_t o_stride_h,
                                           int64_t o_stride_s, int64_t do_stride_b, int64_t do_stride_h, int64_t do_stride_s,
                                           int is_causal, int q_gran, int k_gran, float sm_scale, int fold_sm_scale,
                                           int window_left, int window_right, void* stream) {
  if (int e = sab::check_window(window_left, window_right, is_causal, Sq, Skv)) return e;
  const sab::Window w{window_left, window_right};
  return bwd_dense(q_int8, k_int8, q_scale, k_scale, q, k, v, o, dout, lse, k_mean, dq, dk, dv, workspace, dtype, B, Hq, Hkv, Sq, Skv, D,
                   q8_stride_b, q8_stride_h, q8_stride_s, k8_stride_b, k8_stride_h, k8_stride_s, q_stride_b, q_stride_h, q_stride_s,
                   k_stride_b, k_stride_h, k_stride_s, v_stride_b, v_stride_h, v_stride_s, o_stride_b, o_stride_h, o_stride_s,
                   do_stride_b, do_stride_h, do_stride_s, is_causal, q_gran, k_gran, sm_scale, fold_sm_scale, &w, nullptr, nullptr,
                   nullptr, stream);
}

// sab_qk_int8_attn_bwd_varlen_seq and, with a window w or a block mask bm (already checked), sab_qk_int8_attn_bwd_varlen_window /
// sab_qk_int8_attn_bwd_varlen_blocksparse
static int bwd_varlen_seq(const int8_t* q_int8, const int8_t* k_int8, const float* q_scale, const float* k_scale, const void* q,
                          const void* k, const void* v, const void* o, const void* dout, const float* lse, const void* k_mean, void* dq,
                          void* dk, void* dv, void* workspace, int dtype, int nseq, int Hq, int Hkv, int Tq, int Tk, int D,
                          int64_t q8_stride_t, int64_t q8_stride_h, int64_t k8_stride_t, int64_t k8_stride_h, int64_t q_stride_t,
                          int64_t q_stride_h, int64_t k_stride_t, int64_t k_stride_h, int64_t v_stride_t, int64_t v_stride_h,
                          int64_t o_stride_t, int64_t o_stride_h, int64_t do_stride_t, int64_t do_stride_h,
                          const int32_t* cu_seqlens_q, const int32_t* cu_seqlens_k, const int32_t* cu_q_scale,
                          const int32_t* cu_k_scale, int max_seqlen_q, int max_seqlen_k, int is_causal, int q_gran, int k_gran,
                          float sm_scale, const sab::Window* w, const sab::BlockMask* bm, void* stream) {
  using namespace sab;
  if (int e = check_bwd_args(q_int8, k_int8, q_scale, k_scale, q, k, v, o, dout, lse, dq, dk, dv, workspace, dtype, nseq, Hq, Hkv, Tq, Tk, D))
    return e;
  SAB_REQUIRE((q_gran == SAB_GRAN_PER_WARP || q_gran == SAB_GRAN_PER_THREAD) && (k_gran == SAB_GRAN_PER_WARP || k_gran == SAB_GRAN_PER_THREAD),
              SAB_ERR_INVALID, "q_gran / k_gran must be SAB_GRAN_PER_WARP or SAB_GRAN_PER_THREAD (got %d, %d)", q_gran, k_gran);
  SAB_REQUIRE(cu_seqlens_q && cu_seqlens_k && cu_q_scale && cu_k_scale && max_seqlen_q > 0 && max_seqlen_k > 0, SAB_ERR_INVALID,
              "varlen needs cu_seqlens_q, cu_seqlens_k, cu_q_scale, cu_k_scale, max_seqlen_q and max_seqlen_k");
  // packed [T,H,D]: no batch stride
  const int64_t st[21] = {0, q8_stride_h, q8_stride_t, 0, k8_stride_h, k8_stride_t, 0, q_stride_h, q_stride_t, 0, k_stride_h, k_stride_t,
                          0, v_stride_h, v_stride_t, 0, o_stride_h, o_stride_t, 0, do_stride_h, do_stride_t};
  if (int e = check_bwd_layout(q_int8, k_int8, q, k, v, o, dout, dq, dk, dv, st)) return e;
  BwdParams p = bwd_params(q_int8, k_int8, q_scale, k_scale, q, k, v, o, dout, lse, k_mean, dq, dk, dv, workspace, nseq, Hq, Hkv, Tq, Tk,
                           st, is_causal, q_gran, k_gran, sm_scale, 0);
  AttnParams& a = p.a;
  a.n_q_tiles = (max_seqlen_q + BM - 1) / BM;
  p.n_k_tiles = (max_seqlen_k + 127) / 128;
  a.qs_stride_bh = a.ks_stride_bh = 1;   // as sab_qk_int8_attn_bwd_varlen: scale bases h / hk, rows [blocks * mult, H]
  a.qs_stride_idx = Hq;
  a.ks_stride_idx = Hkv;
  a.cu_q = cu_seqlens_q; a.cu_k = cu_seqlens_k; a.cu_qs = cu_q_scale; a.cu_ks = cu_k_scale;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const bool kt = k_gran == SAB_GRAN_PER_THREAD;
  const bool bf = dtype == SAB_DTYPE_BF16;
  if (w != nullptr) {
    if (D == 128) {
      if (kt) return bf ? launch_bwd_window<128, true, __nv_bfloat16, true>(p, *w, s) : launch_bwd_window<128, true, __half, true>(p, *w, s);
      return bf ? launch_bwd_window<128, false, __nv_bfloat16, true>(p, *w, s) : launch_bwd_window<128, false, __half, true>(p, *w, s);
    }
    if (kt) return bf ? launch_bwd_window<64, true, __nv_bfloat16, true>(p, *w, s) : launch_bwd_window<64, true, __half, true>(p, *w, s);
    return bf ? launch_bwd_window<64, false, __nv_bfloat16, true>(p, *w, s) : launch_bwd_window<64, false, __half, true>(p, *w, s);
  }
  if (bm != nullptr) {
    const int mk = max_seqlen_k;
    if (D == 128) {
      if (kt) return bf ? launch_bwd_blocksparse<128, true, __nv_bfloat16, true>(p, *bm, mk, s)
                        : launch_bwd_blocksparse<128, true, __half, true>(p, *bm, mk, s);
      return bf ? launch_bwd_blocksparse<128, false, __nv_bfloat16, true>(p, *bm, mk, s)
                : launch_bwd_blocksparse<128, false, __half, true>(p, *bm, mk, s);
    }
    if (kt) return bf ? launch_bwd_blocksparse<64, true, __nv_bfloat16, true>(p, *bm, mk, s)
                      : launch_bwd_blocksparse<64, true, __half, true>(p, *bm, mk, s);
    return bf ? launch_bwd_blocksparse<64, false, __nv_bfloat16, true>(p, *bm, mk, s)
              : launch_bwd_blocksparse<64, false, __half, true>(p, *bm, mk, s);
  }
  if (D == 128) {
    if (kt) return bf ? launch_bwd_varlen_seq<128, true, __nv_bfloat16>(p, s) : launch_bwd_varlen_seq<128, true, __half>(p, s);
    return bf ? launch_bwd_varlen_seq<128, false, __nv_bfloat16>(p, s) : launch_bwd_varlen_seq<128, false, __half>(p, s);
  }
  if (kt) return bf ? launch_bwd_varlen_seq<64, true, __nv_bfloat16>(p, s) : launch_bwd_varlen_seq<64, true, __half>(p, s);
  return bf ? launch_bwd_varlen_seq<64, false, __nv_bfloat16>(p, s) : launch_bwd_varlen_seq<64, false, __half>(p, s);
}

extern "C" int sab_qk_int8_attn_bwd_varlen_seq(const int8_t* q_int8, const int8_t* k_int8, const float* q_scale, const float* k_scale,
                                               const void* q, const void* k, const void* v, const void* o, const void* dout,
                                               const float* lse, const void* k_mean, void* dq, void* dk, void* dv, void* workspace,
                                               int dtype, int nseq, int Hq, int Hkv, int Tq, int Tk, int D, int64_t q8_stride_t,
                                               int64_t q8_stride_h, int64_t k8_stride_t, int64_t k8_stride_h, int64_t q_stride_t,
                                               int64_t q_stride_h, int64_t k_stride_t, int64_t k_stride_h, int64_t v_stride_t,
                                               int64_t v_stride_h, int64_t o_stride_t, int64_t o_stride_h, int64_t do_stride_t,
                                               int64_t do_stride_h, const int32_t* cu_seqlens_q, const int32_t* cu_seqlens_k,
                                               const int32_t* cu_q_scale, const int32_t* cu_k_scale, int max_seqlen_q,
                                               int max_seqlen_k, int is_causal, int q_gran, int k_gran, float sm_scale, void* stream) {
  return bwd_varlen_seq(q_int8, k_int8, q_scale, k_scale, q, k, v, o, dout, lse, k_mean, dq, dk, dv, workspace, dtype, nseq, Hq, Hkv, Tq,
                        Tk, D, q8_stride_t, q8_stride_h, k8_stride_t, k8_stride_h, q_stride_t, q_stride_h, k_stride_t, k_stride_h,
                        v_stride_t, v_stride_h, o_stride_t, o_stride_h, do_stride_t, do_stride_h, cu_seqlens_q, cu_seqlens_k,
                        cu_q_scale, cu_k_scale, max_seqlen_q, max_seqlen_k, is_causal, q_gran, k_gran, sm_scale, nullptr, nullptr,
                        stream);
}

extern "C" int sab_qk_int8_attn_bwd_varlen_window(const int8_t* q_int8, const int8_t* k_int8, const float* q_scale,
                                                  const float* k_scale, const void* q, const void* k, const void* v, const void* o,
                                                  const void* dout, const float* lse, const void* k_mean, void* dq, void* dk, void* dv,
                                                  void* workspace, int dtype, int nseq, int Hq, int Hkv, int Tq, int Tk, int D,
                                                  int64_t q8_stride_t, int64_t q8_stride_h, int64_t k8_stride_t, int64_t k8_stride_h,
                                                  int64_t q_stride_t, int64_t q_stride_h, int64_t k_stride_t, int64_t k_stride_h,
                                                  int64_t v_stride_t, int64_t v_stride_h, int64_t o_stride_t, int64_t o_stride_h,
                                                  int64_t do_stride_t, int64_t do_stride_h, const int32_t* cu_seqlens_q,
                                                  const int32_t* cu_seqlens_k, const int32_t* cu_q_scale, const int32_t* cu_k_scale,
                                                  int max_seqlen_q, int max_seqlen_k, int is_causal, int q_gran, int k_gran,
                                                  float sm_scale, int window_left, int window_right, void* stream) {
  if (int e = sab::check_window_varlen(window_left, window_right, max_seqlen_q, max_seqlen_k)) return e;
  const sab::Window w{window_left, window_right};
  return bwd_varlen_seq(q_int8, k_int8, q_scale, k_scale, q, k, v, o, dout, lse, k_mean, dq, dk, dv, workspace, dtype, nseq, Hq, Hkv, Tq,
                        Tk, D, q8_stride_t, q8_stride_h, k8_stride_t, k8_stride_h, q_stride_t, q_stride_h, k_stride_t, k_stride_h,
                        v_stride_t, v_stride_h, o_stride_t, o_stride_h, do_stride_t, do_stride_h, cu_seqlens_q, cu_seqlens_k,
                        cu_q_scale, cu_k_scale, max_seqlen_q, max_seqlen_k, is_causal, q_gran, k_gran, sm_scale, &w, nullptr, stream);
}

extern "C" int sab_qk_int8_attn_bwd_varlen_blocksparse(const int8_t* q_int8, const int8_t* k_int8, const float* q_scale,
                                                       const float* k_scale, const void* q, const void* k, const void* v, const void* o,
                                                       const void* dout, const float* lse, const void* k_mean, void* dq, void* dk,
                                                       void* dv, void* workspace, int dtype, int nseq, int Hq, int Hkv, int Tq, int Tk,
                                                       int D, int64_t q8_stride_t, int64_t q8_stride_h, int64_t k8_stride_t,
                                                       int64_t k8_stride_h, int64_t q_stride_t, int64_t q_stride_h, int64_t k_stride_t,
                                                       int64_t k_stride_h, int64_t v_stride_t, int64_t v_stride_h, int64_t o_stride_t,
                                                       int64_t o_stride_h, int64_t do_stride_t, int64_t do_stride_h,
                                                       const int32_t* cu_seqlens_q, const int32_t* cu_seqlens_k,
                                                       const int32_t* cu_q_scale, const int32_t* cu_k_scale, int max_seqlen_q,
                                                       int max_seqlen_k, int is_causal, int q_gran, int k_gran, float sm_scale,
                                                       const uint8_t* block_mask, int64_t mask_stride_b, int64_t mask_stride_h,
                                                       int64_t mask_stride_qb, int64_t mask_stride_kb, void* stream) {
  if (int e = sab::check_block_mask_varlen(block_mask, mask_stride_b, mask_stride_h, mask_stride_qb, mask_stride_kb, q_gran,
                                           max_seqlen_q, max_seqlen_k))
    return e;
  const sab::BlockMask bm{block_mask, mask_stride_b, mask_stride_h, mask_stride_qb, mask_stride_kb};
  return bwd_varlen_seq(q_int8, k_int8, q_scale, k_scale, q, k, v, o, dout, lse, k_mean, dq, dk, dv, workspace, dtype, nseq, Hq, Hkv, Tq,
                        Tk, D, q8_stride_t, q8_stride_h, k8_stride_t, k8_stride_h, q_stride_t, q_stride_h, k_stride_t, k_stride_h,
                        v_stride_t, v_stride_h, o_stride_t, o_stride_h, do_stride_t, do_stride_h, cu_seqlens_q, cu_seqlens_k,
                        cu_q_scale, cu_k_scale, max_seqlen_q, max_seqlen_k, is_causal, q_gran, k_gran, sm_scale, nullptr, &bm, stream);
}
