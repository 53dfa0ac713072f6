// Quantisation front-end for sm_90a (H100): K-smoothing mean, INT8 quantisation of Q/K (per-block / per-warp /
// per-thread granularity, CUDA or Triton rounding semantics), per-channel FP8 quantisation of V into the
// token-contiguous V^T layout the wgmma PV product consumes.  All kernels are HBM-streaming: 128-bit loads,
// one read of the input (+ one statistics pre-pass where the algorithm needs a full-sequence reduction),
// 64/128-bit stores.  Semantics follow csrc/fused/fused.cu and sageattention/triton/quant_per_*.py of the
// reference (see include/sageattn_b200.h for the per-entry citations).
#include <cstdlib>
#include <type_traits>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include "common.cuh"
#include "quant_common.cuh"

namespace sab {

template <typename T>
__device__ __forceinline__ void load8(const T* p, float (&f)[8]) {
  uint4 raw = *reinterpret_cast<const uint4*>(p);
  const T* e = reinterpret_cast<const T*>(&raw);
#pragma unroll
  for (int i = 0; i < 8; ++i) f[i] = to_f<T>(e[i]);
}

__device__ __forceinline__ uint64_t pack2f(float lo, float hi) {
  uint64_t r;
  asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi));
  return r;
}
__device__ __forceinline__ void unpack2f(uint64_t v, float& lo, float& hi) {
  asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v));
}
// Pairs of IEEE round-to-nearest fp32 operations on packed operands.  The _rn intrinsics are never contracted into an
// FMA by the compiler, so each operation rounds on its own exactly as the reference's scalar code does.
__device__ __forceinline__ uint64_t fmul2q(uint64_t a, uint64_t b) {
  float a0, a1, b0, b1;
  unpack2f(a, a0, a1);
  unpack2f(b, b0, b1);
  return pack2f(__fmul_rn(a0, b0), __fmul_rn(a1, b1));
}
__device__ __forceinline__ uint64_t fadd2q(uint64_t a, uint64_t b) {
  float a0, a1, b0, b1;
  unpack2f(a, a0, a1);
  unpack2f(b, b0, b1);
  return pack2f(__fadd_rn(a0, b0), __fadd_rn(a1, b1));
}
__device__ __forceinline__ uint64_t ffma2q(uint64_t a, uint64_t b, uint64_t c) {
  float a0, a1, b0, b1, c0, c1;
  unpack2f(a, a0, a1);
  unpack2f(b, b0, b1);
  unpack2f(c, c0, c1);
  return pack2f(__fmaf_rn(a0, b0, c0), __fmaf_rn(a1, b1, c1));
}
// How the per-sequence kernels address input row r (r < L_b) of sequence b, relative to the base of its head: `first` is the
// offset of the sequence's first row, `row` the offset of row r from there (ss: the row stride of the input).
// PackedRows: packed [T,H,D] (or one dense batch entry), row r at token t0 + r.  The contiguous kernels use it, and it spells the
// same index arithmetic they had, so their code is unchanged.
struct PackedRows {
  __device__ __forceinline__ int64_t first(int t0, int64_t ss) const { return int64_t(t0) * ss; }
  __device__ __forceinline__ int64_t row(int r, int64_t ss) const { return int64_t(r) * ss; }
};
// A paged cache [num_pages, page_size, H, D] (page stride page_stride, slot stride ss) with a block table: row r of sequence b
// is slot r % page_size of page table[b][r / page_size].  Indexed in int64: a cache can hold more than 2^31 elements.
struct PageTable {
  const int32_t* table; int64_t table_stride;   // [nseq, max_pages] int32, row stride table_stride
  int page_size; int64_t page_stride;
};
struct PagedRows {
  const int32_t* table;   // this sequence's row of the block table
  int page_size; int64_t page_stride;
  __device__ __forceinline__ PagedRows(const PageTable& pt, int b)
      : table(pt.table + int64_t(b) * pt.table_stride), page_size(pt.page_size), page_stride(pt.page_stride) {}
  __device__ __forceinline__ int64_t first(int, int64_t) const { return 0; }
  __device__ __forceinline__ int64_t row(int r, int64_t ss) const {
    return int64_t(__ldg(table + r / page_size)) * page_stride + int64_t(r % page_size) * ss;
  }
};

// =====================================================================================================
// Channel statistics over the token dimension: per (b,h,d) sum / max / min.  Two deterministic stages
// (no atomics): stage 1 reduces 1024-token chunks, stage 2 folds the chunk partials in order.
// =====================================================================================================
constexpr int kStatChunk = 1024;

// kSeq: packed [T,H,D] input, blockIdx.z = sequence b = tokens [cu[b], cu[b+1]); its chunks start at the sequence's first token, so
// the partials of a sequence are those of the dense call on that sequence alone.
// Rows: how a row of sequence b is addressed (kSeq only; channel_stats_stage1_paged reads a paged cache).
template <typename T, int D, bool kSeq, typename Rows = PackedRows>
__device__ __forceinline__ void channel_stats_chunk(const T* __restrict__ x, float* __restrict__ part, int S, int64_t sb, int64_t sh,
                                                    int64_t ss, int nchunk, const int32_t* __restrict__ cu, const Rows rows = Rows{}) {
  constexpr int TPR = D / 8;        // threads per token row
  constexpr int RPP = 256 / TPR;    // rows per pass
  const int chunk = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int tr = threadIdx.x / TPR, tc = threadIdx.x % TPR;
  const T* base = x + b * sb + h * sh + tc * 8;
  if constexpr (kSeq) {
    const int t0 = cu[b];
    S = cu[b + 1] - t0;
    if (chunk * kStatChunk >= S) return;
    base += rows.first(t0, ss);
  }
  float sum[8], mx[8], mn[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) { sum[i] = 0.f; mx[i] = -INFINITY; mn[i] = INFINITY; }
  const int r0 = chunk * kStatChunk;
  const int r1 = min(S, r0 + kStatChunk);
  for (int r = r0 + tr; r < r1; r += RPP) {
    float f[8];
    load8<T>(base + rows.row(r, ss), f);
#pragma unroll
    for (int i = 0; i < 8; ++i) { sum[i] += f[i]; mx[i] = fmaxf(mx[i], f[i]); mn[i] = fminf(mn[i], f[i]); }
  }
  __shared__ float s_sum[RPP][D + 1], s_mx[RPP][D + 1], s_mn[RPP][D + 1];
#pragma unroll
  for (int i = 0; i < 8; ++i) { s_sum[tr][tc * 8 + i] = sum[i]; s_mx[tr][tc * 8 + i] = mx[i]; s_mn[tr][tc * 8 + i] = mn[i]; }
  __syncthreads();
  if (threadIdx.x < D) {
    float a = 0.f, m1 = -INFINITY, m2 = INFINITY;
    for (int r = 0; r < RPP; ++r) { a += s_sum[r][threadIdx.x]; m1 = fmaxf(m1, s_mx[r][threadIdx.x]); m2 = fminf(m2, s_mn[r][threadIdx.x]); }
    float* o = part + ((int64_t(b) * gridDim.y + h) * nchunk + chunk) * 3 * D;
    o[threadIdx.x] = a; o[D + threadIdx.x] = m1; o[2 * D + threadIdx.x] = m2;
  }
}

template <typename T, int D, bool kSeq = false>
__global__ void __launch_bounds__(256) channel_stats_stage1(const T* __restrict__ x, float* __restrict__ part, int S,
                                                             int64_t sb, int64_t sh, int64_t ss, int nchunk,
                                                             const int32_t* __restrict__ cu = nullptr) {
  channel_stats_chunk<T, D, kSeq>(x, part, S, sb, sh, ss, nchunk, cu);
}
// the kSeq form on a paged cache: sequence b's rows through its block-table row; cu: the packed offsets, i.e. the lengths
template <typename T, int D>
__global__ void __launch_bounds__(256) channel_stats_stage1_paged(const T* __restrict__ x, float* __restrict__ part, int64_t sh,
                                                                   int64_t ss, int nchunk, const int32_t* __restrict__ cu,
                                                                   const PageTable pt) {
  channel_stats_chunk<T, D, true>(x, part, 0, 0, sh, ss, nchunk, cu, PagedRows(pt, blockIdx.z));
}

// mode 0: K mean -> T [B,H,D].  mode 1: V scale (+ mean) -> fp32.  mode 2: raw sum / max / min -> fp32.
// kSeq (modes 0 and 1): grid (H, nseq), sequence b = blockIdx.y of length cu[b+1] - cu[b] folds its own chunks; an empty sequence
// gets mean 0, scale 0 and reciprocal 0.
template <typename T, bool kSeq = false>
__global__ void channel_stats_stage2(const float* __restrict__ part, int nchunk, int D, int S, int mode, T* mean_out,
                                     float* scale_out, float* vmean_out, float scale_max, float* recp_out,
                                     const int32_t* __restrict__ cu = nullptr) {
  const int bh = kSeq ? blockIdx.y * gridDim.x + blockIdx.x : blockIdx.x, d = threadIdx.x;
  if (d >= D) return;
  const float* p = part + int64_t(bh) * nchunk * 3 * D;
  int nc = nchunk;
  if constexpr (kSeq) {
    S = cu[blockIdx.y + 1] - cu[blockIdx.y];
    nc = (S + kStatChunk - 1) / kStatChunk;
    if (S == 0) {
      if (mode == 0) {
        mean_out[int64_t(bh) * D + d] = from_f<T>(0.f);
      } else {
        scale_out[int64_t(bh) * D + d] = 0.f;
        recp_out[int64_t(bh) * D + d] = 0.f;
        if (vmean_out) vmean_out[int64_t(bh) * D + d] = 0.f;
      }
      return;
    }
  }
  float a = 0.f, m1 = -INFINITY, m2 = INFINITY;
  for (int c = 0; c < nc; ++c) { a += p[c * 3 * D + d]; m1 = fmaxf(m1, p[c * 3 * D + D + d]); m2 = fminf(m2, p[c * 3 * D + 2 * D + d]); }
  if (mode == 2) {
    scale_out[int64_t(bh) * D + d] = a;
    vmean_out[int64_t(bh) * D + d] = m1;
    recp_out[int64_t(bh) * D + d] = m2;
  } else if (mode == 0) {
    mean_out[int64_t(bh) * D + d] = from_f<T>(__fdiv_rn(a, float(S)));  // torch.mean: fp32 sum / N, cast
  } else {
    float amax;
    if (vmean_out) {  // smooth_v: fused.cu:375-386 (mean over the 16-padded length)
      const float mean = __fdiv_rn(a, float((S + 15) / 16 * 16));
      vmean_out[int64_t(bh) * D + d] = mean;
      amax = fmaxf(fabsf(m1 - mean), fabsf(m2 - mean));
    } else {
      amax = fmaxf(fabsf(m1), fabsf(m2));
    }
    scale_out[int64_t(bh) * D + d] = __fdividef(amax, scale_max);             // fused.cu:389
    recp_out[int64_t(bh) * D + d] = amax > 0.f ? __fdividef(scale_max, amax) : 0.f;  // fused.cu:392 (guarded)
  }
}

// =====================================================================================================
// INT8 quantisation of a 128-row tile of one (b,h): per-row amax -> per-group amax -> scale -> int8.
// =====================================================================================================
enum GroupMode { kGroupBlock = 0, kGroupThreadQ = 1, kGroupThreadK = 2 };

struct QuantParams {
  const void* x; const void* mean; int8_t* out; float* scale;
  int H, S, scale_cols;
  int64_t xsb, xsh, xss, osb, osh, oss;
  int blk;            // rows per scale group (kGroupBlock)
  int semantics;      // SAB_SEM_*
  int has_sm_scale; float sm_scale;
  int eps_after;      // Triton per-thread: scale = amax/127 + 1e-7
  // varlen (nullable): packed [T,H,D]
  const int32_t* cu; const int32_t* cu_scale;
};

// Two 16-bit elements of one 32-bit word -> two floats (exact).
template <typename T>
__device__ __forceinline__ void cvt_pair(uint32_t w, float& lo, float& hi);
template <>
__device__ __forceinline__ void cvt_pair<__nv_bfloat16>(uint32_t w, float& lo, float& hi) {
  lo = __uint_as_float(w << 16);
  hi = __uint_as_float(w & 0xffff0000u);
}
template <>
__device__ __forceinline__ void cvt_pair<__half>(uint32_t w, float& lo, float& hi) {
  const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&w));
  lo = f.x;
  hi = f.y;
}
// Two floats -> one word of two T (round to nearest even).
template <typename T>
__device__ __forceinline__ uint32_t round_pair(float lo, float hi);
template <>
__device__ __forceinline__ uint32_t round_pair<__nv_bfloat16>(float lo, float hi) {
  const __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<const uint32_t*>(&v);
}
template <>
__device__ __forceinline__ uint32_t round_pair<__half>(float lo, float hi) {
  const __half2 v = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<const uint32_t*>(&v);
}

constexpr int kQfTriton = 1, kQfMean = 2, kQfSmScale = 4;   // FLAGS bits of quant_int8_kernel
// FLAGS bit of the per-sequence varlen form (sab_quant_int8_varlen): the mean is [nseq,H,D], and the scales of sequence b are the
// rows [cu_scale[b] * mult, (cu_scale[b] + nblk) * mult) of a [rows,H] table, cu_scale counting 128-row Q / 64-key K blocks.  Every
// group of those blocks is written, as the dense call writes every column of its ceil(S/128)*4 / *32 or ceil(S/64) / *4 scales.
constexpr int kQfSeq = 8;

// Scale-table geometry of the per-sequence form: rows per scale block (128 Q rows, or 64 keys) and scales per block
template <int MODE>
__device__ __forceinline__ int seq_scale_unit(int blk) { return (MODE == kGroupThreadK || (MODE == kGroupBlock && blk == 64)) ? 64 : 128; }
template <int MODE>
__device__ __forceinline__ int seq_scale_mult(int blk) {
  return MODE == kGroupThreadQ ? 32 : (MODE == kGroupThreadK ? 4 : seq_scale_unit<MODE>(blk) / blk);
}

// FLAGS (compile time): rounding semantics, fused mean subtraction, fused sm_scale multiply — no per-element
// runtime conditionals.  The tile stays in registers as raw 16-bit words (NP x 16 B per thread).
//   amax pass : |x| after the transform; the sm_scale multiply is applied once to the ROW maximum, which is exact:
//               rounding and multiplication by a positive constant are monotone, so max_i RN(|x_i| s) = RN(max_i |x_i| s).
//   int8 pass : y = x * (1/scale or 127/amax); t = y + 1.5*2^23 rounds y to the nearest-even integer n, and the low
//               byte of t's bit pattern IS the two's-complement int8 — no F2I, bytes gathered with PRMT.
//               CUDA semantics (cvt.rni.sat.s8 of x*mult, |y| <= 127 by construction): that is already the result.
//               Triton semantics need trunc(RN(x/scale) + 0.5 sign): equal to n unless y is within 1e-4 of a
//               half-integer (ties, or the 2.4e-5 error of x*RN(1/scale) against the IEEE quotient could matter);
//               one |y - n| maximum per 8 elements decides, and those rare rows redo the exact reference sequence.
// One 128-row tile of one (b,h).  `mean_bh`: the D per-channel means of this (b,h) (global or shared memory), or nullptr.
// Rows: how a row of sequence b is addressed (varlen only; quant_int8_paged_kernel reads a paged cache).
template <typename T, int D, int MODE, int FLAGS, typename Rows = PackedRows>
__device__ __forceinline__ void quant_int8_tile(const QuantParams& p, const int tile, const int h, const int b, const T* mean_bh,
                                                const Rows rows = Rows{}) {
  constexpr bool kTriton = (FLAGS & kQfTriton) != 0, kMean = (FLAGS & kQfMean) != 0, kSms = (FLAGS & kQfSmScale) != 0;
  constexpr int TPR = D / 8;
  constexpr int RPP = 256 / TPR;     // 16 (D=128) / 32 (D=64)
  constexpr int NP = 128 / RPP;      // passes: 8 / 4
  const int tr = threadIdx.x / TPR, tc = threadIdx.x % TPR;
  int S = p.S;
  int64_t x_off, o_off;
  int scale_row0 = 0;
  const bool varlen = p.cu != nullptr;
  if (varlen) {
    const int t0 = p.cu[b];
    S = p.cu[b + 1] - t0;
    if (tile * 128 >= S) return;
    x_off = rows.first(t0, p.xss) + int64_t(h) * p.xsh;
    o_off = int64_t(t0) * p.oss + int64_t(h) * p.osh;
    scale_row0 = p.cu_scale[b];
    if constexpr ((FLAGS & kQfSeq) != 0) scale_row0 *= seq_scale_mult<MODE>(p.blk);
  } else {
    x_off = int64_t(b) * p.xsb + int64_t(h) * p.xsh;
    o_off = int64_t(b) * p.osb + int64_t(h) * p.osh;
  }
  const T* xb = reinterpret_cast<const T*>(p.x) + x_off + tc * 8;
  int8_t* ob = p.out + o_off + tc * 8;

  uint64_t nmean2[4];   // (-mean[2w], -mean[2w+1])
  if constexpr (kMean) {
    float mean[8];
    load8<T>(mean_bh + tc * 8, mean);
#pragma unroll
    for (int w = 0; w < 4; ++w) nmean2[w] = pack2f(-mean[2 * w], -mean[2 * w + 1]);
  }

  __shared__ float s_row_amax[128];
  __shared__ float s_scale[32];
  __shared__ float s_inv[32];   // RN(1/scale): fast path of the Triton-semantics division

  uint4 raw[NP];
#pragma unroll
  for (int ps = 0; ps < NP; ++ps) {
    const int row = tile * 128 + ps * RPP + tr;
    raw[ps] = make_uint4(0, 0, 0, 0);
    if (row < S) raw[ps] = *reinterpret_cast<const uint4*>(xb + rows.row(row, p.xss));
  }
  // transform of one word before the sm_scale multiply: x - mean (Triton: `k - km` rounds to the input dtype)
  auto centred = [&](uint32_t w, int wi, float& lo, float& hi) {
    cvt_pair<T>(w, lo, hi);
    if constexpr (kMean) {
      unpack2f(fadd2q(pack2f(lo, hi), nmean2[wi]), lo, hi);
      if constexpr (kTriton) cvt_pair<T>(round_pair<T>(lo, hi), lo, hi);
    }
  };
#pragma unroll
  for (int ps = 0; ps < NP; ++ps) {
    const int r = ps * RPP + tr;
    const int row = tile * 128 + r;
    float amax = 0.f;
    uint32_t* wv = reinterpret_cast<uint32_t*>(&raw[ps]);
#pragma unroll
    for (int w = 0; w < 4; ++w) {
      float lo, hi;
      if constexpr (kMean && kTriton) {
        // the centred value is a T again: keep it in place of the input so the int8 pass does not redo the subtraction
        cvt_pair<T>(wv[w], lo, hi);
        unpack2f(fadd2q(pack2f(lo, hi), nmean2[w]), lo, hi);
        wv[w] = round_pair<T>(lo, hi);
        cvt_pair<T>(wv[w], lo, hi);
      } else {
        centred(wv[w], w, lo, hi);
      }
      amax = fmaxf(fmaxf(amax, fabsf(lo)), fabsf(hi));
    }
    if (row >= S) amax = 0.f;   // (rows past the end were loaded as zeros; with a mean they would read |0 - mean|)
    if constexpr (kSms) amax *= p.sm_scale;
#pragma unroll
    for (int o = TPR / 2; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    if (tc == 0) s_row_amax[r] = amax;
  }
  __syncthreads();

  // ---- group amax -> scale
  int ngroups;
  if (MODE == kGroupBlock) ngroups = 128 / p.blk;
  else if (MODE == kGroupThreadQ) ngroups = 32;
  else ngroups = 8;
  if (threadIdx.x < ngroups) {
    const int g = threadIdx.x;
    float amax = 0.f;
    if (MODE == kGroupBlock) {
      for (int r = g * p.blk; r < (g + 1) * p.blk; ++r) amax = fmaxf(amax, s_row_amax[r]);
    } else if (MODE == kGroupThreadQ) {  // rows {g%8 + 8i} of 32-row block g/8
      for (int i = 0; i < 4; ++i) amax = fmaxf(amax, s_row_amax[(g / 8) * 32 + i * 8 + (g % 8)]);
    } else {                             // keys {8j + 2t, 8j + 2t + 1} of 64-key block g/4
      for (int j8 = 0; j8 < 8; ++j8) {
        amax = fmaxf(amax, s_row_amax[(g / 4) * 64 + j8 * 8 + (g % 4) * 2]);
        amax = fmaxf(amax, s_row_amax[(g / 4) * 64 + j8 * 8 + (g % 4) * 2 + 1]);
      }
    }
    float scale, mult;
    if constexpr (!kTriton) {   // fused.cu:147-184 (compiled with --use_fast_math there)
      amax = fmaxf(amax, 0.0000001f);
      scale = __fdividef(amax, 127.0f);
      mult = __fdividef(127.0f, amax);
    } else {
      scale = __fdiv_rn(amax, 127.0f);
      if (p.eps_after) scale += 0.0000001f;
      mult = scale;
    }
    s_scale[g] = mult;
    s_inv[g] = mult > 0.f ? __fdiv_rn(1.0f, mult) : 0.f;   // all-zero block (scale 0): reference 0/0 -> NaN -> int8 0
    const int gcol = tile * ngroups + g;
    if constexpr ((FLAGS & kQfSeq) != 0) {
      const int unit = seq_scale_unit<MODE>(p.blk);
      if (gcol < (S + unit - 1) / unit * seq_scale_mult<MODE>(p.blk)) p.scale[int64_t(scale_row0 + gcol) * p.H + h] = scale;
    } else if (varlen) {
      const int nblk = (S + p.blk - 1) / p.blk;
      if (gcol < nblk) p.scale[int64_t(scale_row0 + gcol) * p.H + h] = scale;
    } else if (gcol < p.scale_cols) {
      p.scale[(int64_t(b) * p.H + h) * p.scale_cols + gcol] = scale;
    }
  }
  __syncthreads();

  // ---- quantise + store
  const uint64_t magic2 = pack2f(12582912.0f, 12582912.0f);
  const uint64_t nmagic2 = pack2f(-12582912.0f, -12582912.0f);
  const uint64_t mone2 = pack2f(-1.0f, -1.0f);
  const uint64_t sms2 = pack2f(p.sm_scale, p.sm_scale);
#pragma unroll
  for (int ps = 0; ps < NP; ++ps) {
    const int r = ps * RPP + tr;
    const int row = tile * 128 + r;
    if (row >= S) continue;
    int g;
    if (MODE == kGroupBlock) g = r / p.blk;
    else if (MODE == kGroupThreadQ) g = (r / 32) * 8 + (r % 8);
    else g = (r / 64) * 4 + (r % 8) / 2;
    const float mult = s_scale[g];
    const float fac = kTriton ? s_inv[g] : mult;
    const uint64_t fac2 = pack2f(fac, fac);
    const uint32_t* wv = reinterpret_cast<const uint32_t*>(&raw[ps]);
    uint32_t tb[8];     // bit patterns of y + 1.5*2^23: low byte = int8
    // A denormal scale (bf16 block with amax < 127 * 2^-128) has RN(1/scale) = inf: y and y - n are inf / NaN, which fmaxf
    // drops, so the residual starts above the threshold and the row takes the exact sequence (IEEE x / scale is finite).
    float dmax = (kTriton && !(fac <= 3.402823466e+38f)) ? 1.f : 0.f;
#pragma unroll
    for (int w = 0; w < 4; ++w) {
      float lo, hi;
      if constexpr (kMean && kTriton) cvt_pair<T>(wv[w], lo, hi);   // already centred and rounded in place
      else centred(wv[w], w, lo, hi);
      uint64_t x2 = pack2f(lo, hi);
      if constexpr (kSms) x2 = fmul2q(x2, sms2);
      // y must be rounded on its own (the reference rounds x*mult, then converts): a multiply-add contracted into one FMA
      // would flip x.5 ties (63 vs 64).  fmul2q / fadd2q use the non-contractible _rn intrinsics.
      const uint64_t y2 = fmul2q(x2, fac2);
      const uint64_t t2 = fadd2q(y2, magic2);
      if constexpr (kTriton) {
        float d0, d1;
        unpack2f(ffma2q(fadd2q(t2, nmagic2), mone2, y2), d0, d1);   // y - n, exact
        dmax = fmaxf(fmaxf(dmax, fabsf(d0)), fabsf(d1));
      } else {
        float y0, y1;
        unpack2f(y2, y0, y1);
        dmax = fmaxf(fmaxf(dmax, fabsf(y0)), fabsf(y1));   // cvt.rni.sat.s8 saturates; the byte trick wraps
      }
      float t0, t1;
      unpack2f(t2, t0, t1);
      tb[2 * w] = __float_as_uint(t0);
      tb[2 * w + 1] = __float_as_uint(t1);
    }
    if constexpr (!kTriton) {
      if (dmax > 127.49f) {   // never for finite data (|x| <= amax by construction): saturate like cvt.rni.sat.s8
#pragma unroll
        for (int w = 0; w < 4; ++w) {
          float xs[2];
          centred(wv[w], w, xs[0], xs[1]);
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            float x = xs[i];
            if constexpr (kSms) x = __fmul_rn(x, p.sm_scale);
            tb[2 * w + i] = uint32_t(int(cvt_rni_sat_s8(__fmul_rn(x, mult))));
          }
        }
      }
    }
    if constexpr (kTriton) {
      if (dmax > 0.4999f) {   // rare (~1e-3 of the rows): redo the reference sequence with the exact IEEE quotient
#pragma unroll
        for (int w = 0; w < 4; ++w) {
          float xs[2];
          if constexpr (kMean) cvt_pair<T>(wv[w], xs[0], xs[1]);
          else centred(wv[w], w, xs[0], xs[1]);
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            float x = xs[i];
            if constexpr (kSms) x = __fmul_rn(x, p.sm_scale);
            const float y = __fdiv_rn(x, mult);
            const float z = __fadd_rn(y, y >= 0.f ? 0.5f : -0.5f);   // quant_per_block.py:43-45
            tb[2 * w + i] = uint32_t(__float2int_rz(z));              // NaN (0/0, all-zero block) -> 0
          }
        }
      }
    }
    uint2 q;
    q.x = __byte_perm(__byte_perm(tb[0], tb[1], 0x0040), __byte_perm(tb[2], tb[3], 0x0040), 0x5410);
    q.y = __byte_perm(__byte_perm(tb[4], tb[5], 0x0040), __byte_perm(tb[6], tb[7], 0x0040), 0x5410);
    *reinterpret_cast<uint2*>(ob + int64_t(row) * p.oss) = q;
  }
}

template <typename T, int D, int MODE, int FLAGS>
__global__ void __launch_bounds__(256, 3) quant_int8_kernel(const QuantParams p) {
  const int h = blockIdx.y, b = blockIdx.z;
  const T* mean_bh = nullptr;
  if constexpr ((FLAGS & kQfMean) != 0)
    mean_bh = reinterpret_cast<const T*>(p.mean) + (int64_t((FLAGS & kQfSeq) == 0 && p.cu != nullptr ? 0 : b) * p.H + h) * D;
  quant_int8_tile<T, D, MODE, FLAGS>(p, blockIdx.x, h, b, mean_bh);
}
// the per-sequence form (kQfSeq) on a paged cache: sequence b's input rows through its block-table row; the output, the scales and
// p.cu (the packed offsets) are those of the packed form
template <typename T, int D, int MODE, int FLAGS>
__global__ void __launch_bounds__(256, 3) quant_int8_paged_kernel(const QuantParams p, const PageTable pt) {
  static_assert((FLAGS & kQfSeq) != 0, "the paged input exists for the per-sequence form only");
  const int h = blockIdx.y, b = blockIdx.z;
  const T* mean_bh = nullptr;
  if constexpr ((FLAGS & kQfMean) != 0) mean_bh = reinterpret_cast<const T*>(p.mean) + (int64_t(b) * p.H + h) * D;
  quant_int8_tile<T, D, MODE, FLAGS>(p, blockIdx.x, h, b, mean_bh, PagedRows(pt, b));
}

// =====================================================================================================
// Single-pass K path: K smoothing mean + INT8 quantisation in ONE launch.  A thread-block cluster of
// kKCluster CTAs owns one (b,h) slice; CTA r takes the 128-row tiles r, r+C, ...  Phase 1: per-channel fp32 sums of its tiles
// -> shared memory; cluster barrier; every CTA folds the C partial sums in rank order through distributed shared memory
// (identical result in every CTA), rounds the mean to T like `k.mean` (core.py:773) and rank 0 writes it out.  Phase 2: the
// tiles are quantised with that mean — their second read comes from L2 (the slice was just streamed by this cluster), so
// HBM sees K once instead of twice (stats pass + quant pass) and two launches disappear.
// =====================================================================================================
constexpr int kKCluster = 8;
constexpr int kFusedDynSmem = 0;   // default dynamic shared-memory request of the fused kernels (see launch_cluster)

__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ float ld_dsmem_f32(const float* local_smem_ptr, uint32_t rank) {
  uint32_t a = static_cast<uint32_t>(__cvta_generic_to_shared(local_smem_ptr)), ra;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(a), "r"(rank));
  float v;
  asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(v) : "r"(ra));
  return v;
}

// per-channel sums of the 128-row tiles r, r+C, ... of one (b,h): thread (tr, tc) accumulates rows tr, tr+RPP, ... of 8 channels
template <typename T, int D>
__device__ __forceinline__ void cluster_channel_sums(const T* base, int64_t ss, int S, int rank, float* s_part /* [D] */) {
  constexpr int TPR = D / 8, RPP = 256 / TPR;
  const int tr = threadIdx.x / TPR, tc = threadIdx.x % TPR;
  __shared__ float s_red[RPP][D + 1];
  float sum[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) sum[i] = 0.f;
  const int ntiles = (S + 127) / 128;
  for (int t = rank; t < ntiles; t += kKCluster) {
    const int r1 = min(S, (t + 1) * 128);
#pragma unroll 4
    for (int r = t * 128 + tr; r < r1; r += RPP) {
      float f[8];
      load8<T>(base + int64_t(r) * ss + tc * 8, f);
#pragma unroll
      for (int i = 0; i < 8; ++i) sum[i] += f[i];
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) s_red[tr][tc * 8 + i] = sum[i];
  __syncthreads();
  if (threadIdx.x < D) {
    float a = 0.f;
    for (int r = 0; r < RPP; ++r) a += s_red[r][threadIdx.x];
    s_part[threadIdx.x] = a;
  }
}

template <typename T, int D, int MODE, int FLAGS>
__global__ void __launch_bounds__(256, 3) k_smooth_quant_kernel(const QuantParams p, T* __restrict__ mean_out) {
  static_assert((FLAGS & kQfMean) != 0, "the fused K path always subtracts the mean");
  const int h = blockIdx.y, b = blockIdx.z;
  const int rank = int(cluster_ctarank());
  __shared__ float s_part[D];
  __shared__ __align__(16) T s_mean[D];
  const T* xb = reinterpret_cast<const T*>(p.x) + int64_t(b) * p.xsb + int64_t(h) * p.xsh;
  cluster_channel_sums<T, D>(xb, p.xss, p.S, rank, s_part);
  cluster_sync_all();                      // every CTA's partial sums are visible cluster-wide
  if (threadIdx.x < D) {
    float a = 0.f;
#pragma unroll
    for (int r = 0; r < kKCluster; ++r) a += ld_dsmem_f32(&s_part[threadIdx.x], uint32_t(r));
    const T m = from_f<T>(__fdiv_rn(a, float(p.S)));     // torch.mean: fp32 sum / N, cast
    s_mean[threadIdx.x] = m;
    if (rank == 0) mean_out[(int64_t(b) * p.H + h) * D + threadIdx.x] = m;
  }
  cluster_sync_all();                      // nobody leaves (or reuses s_part) while a peer still reads it; s_mean is complete
  const int ntiles = (p.S + 127) / 128;
  for (int t = rank; t < ntiles; t += kKCluster) {
    quant_int8_tile<T, D, MODE, FLAGS>(p, t, h, b, s_mean);
    __syncthreads();                       // the tile function's shared scratch is reused by the next tile
  }
}

// =====================================================================================================
// V: per-channel scale, e4m3, transpose to [.., D, S_pad] (token-contiguous).  One CTA = 128 tokens.
// =====================================================================================================
struct VQuantParams {
  const void* v; uint8_t* out; const float* recp; const float* vmean;
  int H, S; int64_t sb, sh, ss; int64_t s_pad; float scale_max;
  const int32_t* cu; const int32_t* cu_pad;
};

// One 128-token tile.  recp_bh / vmean_bh: the D per-channel values of this (b,h) (global or shared memory; vmean may be null).
// Rows: how a row of sequence b is addressed (varlen only; v_quant_transpose_paged_kernel reads a paged cache).
template <typename T, int D, typename Rows = PackedRows>
__device__ __forceinline__ void v_quant_transpose_tile(const VQuantParams& p, const int tile, const int h, const int b,
                                                       const float* recp_bh, const float* vmean_bh, const Rows rows = Rows{}) {
  constexpr int TPR = D / 8;
  constexpr int RPP = 256 / TPR;
  int S = p.S, tok0 = 0;
  int64_t col0 = int64_t(tile) * 128;
  const bool varlen = p.cu != nullptr;
  if (varlen) {
    tok0 = p.cu[b];
    S = p.cu[b + 1] - tok0;
    if (tile * 128 >= S) return;
    col0 += p.cu_pad[b];
  }
  __shared__ __align__(16) T s_in[128][D + 8];  // +8 elements: conflict-free column reads
  const int tr = threadIdx.x / TPR, tc = threadIdx.x % TPR;
  // packed rows keep the plain conditional: with the call in it, the compiler schedules the dense caller v_scale_quant_kernel anew
  int64_t seq0;
  if constexpr (std::is_same_v<Rows, PackedRows>) seq0 = varlen ? int64_t(tok0) * p.ss : int64_t(b) * p.sb;
  else seq0 = rows.first(tok0, p.ss);
  const T* vb = reinterpret_cast<const T*>(p.v) + seq0 + int64_t(h) * p.sh + tc * 8;
#pragma unroll
  for (int r = tr; r < 128; r += RPP) {
    const int row = tile * 128 + r;
    uint4 raw = make_uint4(0, 0, 0, 0);
    if (row < S) raw = *reinterpret_cast<const uint4*>(vb + rows.row(row, p.ss));
    *reinterpret_cast<uint4*>(&s_in[r][tc * 8]) = raw;
  }
  __syncthreads();
  // thread -> (channel d, 32-token segment): 32 bytes = one full sector per thread
  const int bh = (varlen ? 0 : b) * p.H + h;
  for (int task = threadIdx.x; task < D * 4; task += 256) {
    const int d = task % D, seg = task / D;
    const float recp = recp_bh[d];      // scale_max / amax
    const float mean = vmean_bh ? vmean_bh[d] : 0.f;
    uint32_t w[8];
#pragma unroll
    for (int q4 = 0; q4 < 8; ++q4) {
      float f[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int t = seg * 32 + q4 * 4 + i;
        float x = to_f<T>(s_in[t][d]);
        x = (tile * 128 + t < S) ? (x - mean) * recp : 0.f;
        f[i] = x;
      }
      w[q4] = pack_e4m3x4_q(f[0], f[1], f[2], f[3]);
    }
    uint8_t* dst = p.out + (int64_t(bh) * D + d) * p.s_pad + col0 + seg * 32;
    reinterpret_cast<uint4*>(dst)[0] = make_uint4(w[0], w[1], w[2], w[3]);
    reinterpret_cast<uint4*>(dst)[1] = make_uint4(w[4], w[5], w[6], w[7]);
  }
}

// kSeq: varlen with per-sequence statistics, recp / vmean [nseq,H,D]
template <typename T, int D, bool kSeq = false>
__global__ void __launch_bounds__(256) v_quant_transpose_kernel(const VQuantParams p) {
  const int h = blockIdx.y, b = blockIdx.z;
  const int64_t bh = int64_t(!kSeq && p.cu != nullptr ? 0 : b) * p.H + h;
  v_quant_transpose_tile<T, D>(p, blockIdx.x, h, b, p.recp + bh * D, p.vmean ? p.vmean + bh * D : nullptr);
}
// the kSeq form on a paged cache: sequence b's input rows through its block-table row; v_fp8, p.cu and p.cu_pad as in the packed form
template <typename T, int D>
__global__ void __launch_bounds__(256) v_quant_transpose_paged_kernel(const VQuantParams p, const PageTable pt) {
  const int h = blockIdx.y, b = blockIdx.z;
  const int64_t bh = int64_t(b) * p.H + h;
  v_quant_transpose_tile<T, D>(p, blockIdx.x, h, b, p.recp + bh * D, p.vmean ? p.vmean + bh * D : nullptr, PagedRows(pt, b));
}

// Single-pass V path: per-channel |max| (+ mean for smooth_v) and the e4m3 quantisation + transpose in ONE launch, same cluster
// scheme as k_smooth_quant_kernel (max / min are order-independent, so the scales are bit-identical to the two-launch path).
template <typename T, int D>
__global__ void __launch_bounds__(256) v_scale_quant_kernel(const VQuantParams p, float* __restrict__ scale_out, float* __restrict__ vmean_out) {
  constexpr int TPR = D / 8, RPP = 256 / TPR;
  const int h = blockIdx.y, b = blockIdx.z;
  const int rank = int(cluster_ctarank());
  const int tr = threadIdx.x / TPR, tc = threadIdx.x % TPR;
  __shared__ float s_red[RPP][D + 1];     // one reduction at a time (the tile function needs 35 KB of the 48 KB static limit)
  __shared__ float s_part[3][D];          // sum / max / min of this CTA's tiles
  __shared__ float s_recp[D], s_vmean[D];
  const T* vb = reinterpret_cast<const T*>(p.v) + int64_t(b) * p.sb + int64_t(h) * p.sh;
  float sum[8], mx[8], mn[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) { sum[i] = 0.f; mx[i] = -INFINITY; mn[i] = INFINITY; }
  const int ntiles = int(p.s_pad / 128);
  for (int t = rank; t < ntiles; t += kKCluster) {
    const int r1 = min(p.S, (t + 1) * 128);
#pragma unroll 4
    for (int r = t * 128 + tr; r < r1; r += RPP) {
      float f[8];
      load8<T>(vb + int64_t(r) * p.ss + tc * 8, f);
#pragma unroll
      for (int i = 0; i < 8; ++i) { sum[i] += f[i]; mx[i] = fmaxf(mx[i], f[i]); mn[i] = fminf(mn[i], f[i]); }
    }
  }
#pragma unroll
  for (int q3 = 0; q3 < 3; ++q3) {
#pragma unroll
    for (int i = 0; i < 8; ++i) s_red[tr][tc * 8 + i] = q3 == 0 ? sum[i] : (q3 == 1 ? mx[i] : mn[i]);
    __syncthreads();
    if (threadIdx.x < D) {
      float a = q3 == 0 ? 0.f : (q3 == 1 ? -INFINITY : INFINITY);
      for (int r = 0; r < RPP; ++r) {
        const float x = s_red[r][threadIdx.x];
        a = q3 == 0 ? a + x : (q3 == 1 ? fmaxf(a, x) : fminf(a, x));
      }
      s_part[q3][threadIdx.x] = a;
    }
    __syncthreads();
  }
  cluster_sync_all();
  if (threadIdx.x < D) {
    float a = 0.f, m1 = -INFINITY, m2 = INFINITY;
#pragma unroll
    for (int r = 0; r < kKCluster; ++r) {
      a += ld_dsmem_f32(&s_part[0][threadIdx.x], uint32_t(r));
      m1 = fmaxf(m1, ld_dsmem_f32(&s_part[1][threadIdx.x], uint32_t(r)));
      m2 = fminf(m2, ld_dsmem_f32(&s_part[2][threadIdx.x], uint32_t(r)));
    }
    float amax, mean = 0.f;
    if (vmean_out) {  // smooth_v: fused.cu:375-386 (mean over the 16-padded length)
      mean = __fdiv_rn(a, float((p.S + 15) / 16 * 16));
      amax = fmaxf(fabsf(m1 - mean), fabsf(m2 - mean));
    } else {
      amax = fmaxf(fabsf(m1), fabsf(m2));
    }
    s_vmean[threadIdx.x] = mean;
    s_recp[threadIdx.x] = amax > 0.f ? __fdividef(p.scale_max, amax) : 0.f;   // fused.cu:392 (guarded)
    if (rank == 0) {
      const int64_t o = (int64_t(b) * p.H + h) * D + threadIdx.x;
      scale_out[o] = __fdividef(amax, p.scale_max);                          // fused.cu:389
      if (vmean_out) vmean_out[o] = mean;
    }
  }
  cluster_sync_all();
  for (int t = rank; t < ntiles; t += kKCluster) {
    v_quant_transpose_tile<T, D>(p, t, h, b, s_recp, vmean_out ? s_vmean : nullptr);
    __syncthreads();
  }
}

// V -> fp16, transposed to [.., D, S_pad] (token-contiguous), zero padded: the B operand of the kind::f16 PV MMA
// (`v.to(torch.float16)`, sageattention/core.py:297-298, + the K-major layout the wgmma B operand wants).
template <typename T, int D>
__global__ void __launch_bounds__(256) v_transpose_f16_kernel(const VQuantParams p) {
  constexpr int TPR = D / 8;
  constexpr int RPP = 256 / TPR;
  const int tile = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  int S = p.S, tok0 = 0;
  int64_t col0 = int64_t(tile) * 128;
  const bool varlen = p.cu != nullptr;
  if (varlen) {
    tok0 = p.cu[b];
    S = p.cu[b + 1] - tok0;
    if (tile * 128 >= S) return;
    col0 += p.cu_pad[b];
  }
  __shared__ __align__(16) T s_in[128][D + 8];
  const int tr = threadIdx.x / TPR, tc = threadIdx.x % TPR;
  const T* vb = reinterpret_cast<const T*>(p.v) + (varlen ? int64_t(tok0) * p.ss : int64_t(b) * p.sb) + int64_t(h) * p.sh + tc * 8;
#pragma unroll
  for (int r = tr; r < 128; r += RPP) {
    const int row = tile * 128 + r;
    uint4 raw = make_uint4(0, 0, 0, 0);
    if (row < S) raw = *reinterpret_cast<const uint4*>(vb + int64_t(row) * p.ss);
    *reinterpret_cast<uint4*>(&s_in[r][tc * 8]) = raw;
  }
  __syncthreads();
  const int bh = (varlen ? 0 : b) * p.H + h;
  __half* out = reinterpret_cast<__half*>(p.out);
  for (int task = threadIdx.x; task < D * 8; task += 256) {   // (channel d, 16-token segment): 32 bytes per thread
    const int d = task % D, seg = task / D;
    __half hv[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) hv[i] = __float2half_rn(to_f<T>(s_in[seg * 16 + i][d]));
    uint4* dst = reinterpret_cast<uint4*>(out + (int64_t(bh) * D + d) * p.s_pad + col0 + seg * 16);
    dst[0] = reinterpret_cast<uint4*>(hv)[0];
    dst[1] = reinterpret_cast<uint4*>(hv)[1];
  }
}

static int check_common(const void* x, int dtype, int D, int64_t s0, int64_t s1, int64_t s2) {
  SAB_REQUIRE(x != nullptr, SAB_ERR_INVALID, "null input pointer");
  SAB_REQUIRE(dtype == SAB_DTYPE_FP16 || dtype == SAB_DTYPE_BF16, SAB_ERR_UNSUPPORTED, "Only half and bfloat16 are supported");
  SAB_REQUIRE(D == 64 || D == 128, SAB_ERR_UNSUPPORTED, "Unsupported head dim: %d", D);
  SAB_REQUIRE(aligned16(x) && s0 % 8 == 0 && s1 % 8 == 0 && s2 % 8 == 0, SAB_ERR_INVALID,
              "input must be 16-byte aligned with strides multiple of 8 elements");
  return SAB_OK;
}

template <typename T, int D>
static int launch_stats(const void* x, float* part, int B, int H, int S, int64_t sb, int64_t sh, int64_t ss, cudaStream_t st) {
  const int nchunk = (S + kStatChunk - 1) / kStatChunk;
  channel_stats_stage1<T, D><<<dim3(nchunk, H, B), 256, 0, st>>>(reinterpret_cast<const T*>(x), part, S, sb, sh, ss, nchunk);
  SAB_CUDA_OK(cudaGetLastError());
  return SAB_OK;
}

static int run_stats(const void* x, int dtype, float* part, int B, int H, int S, int D, int64_t sb, int64_t sh, int64_t ss, cudaStream_t st) {
  if (dtype == SAB_DTYPE_FP16) return D == 128 ? launch_stats<__half, 128>(x, part, B, H, S, sb, sh, ss, st) : launch_stats<__half, 64>(x, part, B, H, S, sb, sh, ss, st);
  return D == 128 ? launch_stats<__nv_bfloat16, 128>(x, part, B, H, S, sb, sh, ss, st) : launch_stats<__nv_bfloat16, 64>(x, part, B, H, S, sb, sh, ss, st);
}

template <typename T, int D, int FLAGS>
static int launch_quant_f(const QuantParams& p, int mode, dim3 grid, cudaStream_t st) {
  if (mode == kGroupBlock) quant_int8_kernel<T, D, kGroupBlock, FLAGS><<<grid, 256, 0, st>>>(p);
  else if (mode == kGroupThreadQ) quant_int8_kernel<T, D, kGroupThreadQ, FLAGS><<<grid, 256, 0, st>>>(p);
  else quant_int8_kernel<T, D, kGroupThreadK, FLAGS><<<grid, 256, 0, st>>>(p);
  SAB_CUDA_OK(cudaGetLastError());
  return SAB_OK;
}
template <typename T, int D>
static int launch_quant_t(const QuantParams& p, int mode, dim3 grid, cudaStream_t st) {
  const int flags = (p.semantics == SAB_SEM_TRITON ? kQfTriton : 0) | (p.mean != nullptr ? kQfMean : 0) |
                    (p.has_sm_scale ? kQfSmScale : 0);
  switch (flags) {
    case 0: return launch_quant_f<T, D, 0>(p, mode, grid, st);
    case 1: return launch_quant_f<T, D, 1>(p, mode, grid, st);
    case 2: return launch_quant_f<T, D, 2>(p, mode, grid, st);
    case 3: return launch_quant_f<T, D, 3>(p, mode, grid, st);
    case 4: return launch_quant_f<T, D, 4>(p, mode, grid, st);
    case 5: return launch_quant_f<T, D, 5>(p, mode, grid, st);
    case 6: return launch_quant_f<T, D, 6>(p, mode, grid, st);
    default: return launch_quant_f<T, D, 7>(p, mode, grid, st);
  }
}
// the per-sequence varlen form: per-thread Q / K (Triton semantics) and per-warp Q / K (CUDA semantics); a mean on K only.
// pg: K read from a paged cache (nullptr: packed input).
template <typename T, int D>
static int launch_quant_seq_t(const QuantParams& p, int mode, dim3 grid, cudaStream_t st, const PageTable* pg) {
  const bool mean = p.mean != nullptr;
  if (pg != nullptr) {
    if (mode == kGroupThreadK && mean) quant_int8_paged_kernel<T, D, kGroupThreadK, kQfTriton | kQfMean | kQfSeq><<<grid, 256, 0, st>>>(p, *pg);
    else if (mode == kGroupThreadK) quant_int8_paged_kernel<T, D, kGroupThreadK, kQfTriton | kQfSeq><<<grid, 256, 0, st>>>(p, *pg);
    else if (mean) quant_int8_paged_kernel<T, D, kGroupBlock, kQfMean | kQfSeq><<<grid, 256, 0, st>>>(p, *pg);
    else quant_int8_paged_kernel<T, D, kGroupBlock, kQfSeq><<<grid, 256, 0, st>>>(p, *pg);
  } else if (mode == kGroupThreadQ) quant_int8_kernel<T, D, kGroupThreadQ, kQfTriton | kQfSeq><<<grid, 256, 0, st>>>(p);
  else if (mode == kGroupThreadK && mean) quant_int8_kernel<T, D, kGroupThreadK, kQfTriton | kQfMean | kQfSeq><<<grid, 256, 0, st>>>(p);
  else if (mode == kGroupThreadK) quant_int8_kernel<T, D, kGroupThreadK, kQfTriton | kQfSeq><<<grid, 256, 0, st>>>(p);
  else if (mean) quant_int8_kernel<T, D, kGroupBlock, kQfMean | kQfSeq><<<grid, 256, 0, st>>>(p);
  else quant_int8_kernel<T, D, kGroupBlock, kQfSeq><<<grid, 256, 0, st>>>(p);
  SAB_CUDA_OK(cudaGetLastError());
  return SAB_OK;
}
static int launch_quant_seq(const QuantParams& p, int dtype, int D, int mode, dim3 grid, cudaStream_t st, const PageTable* pg) {
  if (dtype == SAB_DTYPE_FP16) return D == 128 ? launch_quant_seq_t<__half, 128>(p, mode, grid, st, pg) : launch_quant_seq_t<__half, 64>(p, mode, grid, st, pg);
  return D == 128 ? launch_quant_seq_t<__nv_bfloat16, 128>(p, mode, grid, st, pg) : launch_quant_seq_t<__nv_bfloat16, 64>(p, mode, grid, st, pg);
}

static int launch_quant(const QuantParams& p, int dtype, int D, int mode, dim3 grid, cudaStream_t st) {
  if (dtype == SAB_DTYPE_FP16) return D == 128 ? launch_quant_t<__half, 128>(p, mode, grid, st) : launch_quant_t<__half, 64>(p, mode, grid, st);
  return D == 128 ? launch_quant_t<__nv_bfloat16, 128>(p, mode, grid, st) : launch_quant_t<__nv_bfloat16, 64>(p, mode, grid, st);
}

}  // namespace sab

using namespace sab;

// ---------------------------------------------------------------------------------------------- fused single-pass front-end
template <typename Kern, typename... Args>
static int launch_cluster(Kern kern, dim3 grid, cudaStream_t st, Args... args) {
  // Occupancy knob: every resident cluster keeps one (b,h) slice in flight between its two phases and the second read should hit
  // L2, so the number of co-resident clusters is bounded through a dynamic shared-memory request (unused by the kernels).
  static int dyn = -1;
  if (dyn < 0) {
    const char* e = getenv("SAB_FUSED_DYNSMEM");
    dyn = e ? atoi(e) : kFusedDynSmem;
  }
  if (dyn > 0) SAB_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, dyn));
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = dim3(256); cfg.dynamicSmemBytes = size_t(dyn); cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = kKCluster; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr; cfg.numAttrs = 1;
  SAB_CUDA_OK(cudaLaunchKernelEx(&cfg, kern, args...));
  return SAB_OK;
}

extern "C" int64_t sab_k_mean_workspace_bytes(int B, int H, int S, int D) {
  const int64_t nchunk = (S + kStatChunk - 1) / kStatChunk;
  return int64_t(B) * H * nchunk * 3 * D * sizeof(float);
}
extern "C" int64_t sab_per_channel_fp8_workspace_bytes(int B, int H, int S, int D) {
  return sab_k_mean_workspace_bytes(B, H, S, D) + int64_t(B) * H * D * sizeof(float);
}

extern "C" int sab_k_mean(const void* k, int dtype, void* mean, int B, int H, int S, int D, int64_t stride_b,
                          int64_t stride_h, int64_t stride_s, void* workspace, void* stream) {
  int st = check_common(k, dtype, D, stride_b, stride_h, stride_s);
  if (st) return st;
  SAB_REQUIRE(mean && workspace && B > 0 && H > 0 && S > 0, SAB_ERR_INVALID, "bad arguments to sab_k_mean");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if ((st = run_stats(k, dtype, reinterpret_cast<float*>(workspace), B, H, S, D, stride_b, stride_h, stride_s, s))) return st;
  const int nchunk = (S + kStatChunk - 1) / kStatChunk;
  if (dtype == SAB_DTYPE_FP16)
    channel_stats_stage2<__half><<<B * H, 128, 0, s>>>(reinterpret_cast<float*>(workspace), nchunk, D, S, 0, reinterpret_cast<__half*>(mean), nullptr, nullptr, 0.f, nullptr);
  else
    channel_stats_stage2<__nv_bfloat16><<<B * H, 128, 0, s>>>(reinterpret_cast<float*>(workspace), nchunk, D, S, 0, reinterpret_cast<__nv_bfloat16*>(mean), nullptr, nullptr, 0.f, nullptr);
  SAB_CUDA_OK(cudaGetLastError());
  return SAB_OK;
}

extern "C" int sab_quant_per_block_int8(const void* x, int dtype, const void* mean, int8_t* out, float* scale, int B,
                                        int H, int S, int D, int64_t x_stride_b, int64_t x_stride_h, int64_t x_stride_s,
                                        int64_t o_stride_b, int64_t o_stride_h, int64_t o_stride_s, int scale_cols,
                                        int blk, int semantics, int has_sm_scale, float sm_scale, void* stream) {
  int st = check_common(x, dtype, D, x_stride_b, x_stride_h, x_stride_s);
  if (st) return st;
  SAB_REQUIRE(out && scale && B > 0 && H > 0 && S > 0, SAB_ERR_INVALID, "bad arguments to sab_quant_per_block_int8");
  SAB_REQUIRE(blk == 16 || blk == 32 || blk == 64 || blk == 128, SAB_ERR_UNSUPPORTED, "Unsupported block size: %d", blk);
  SAB_REQUIRE(semantics == SAB_SEM_CUDA || semantics == SAB_SEM_TRITON, SAB_ERR_INVALID, "unknown semantics %d", semantics);
  SAB_REQUIRE(scale_cols >= (S + blk - 1) / blk, SAB_ERR_INVALID, "scale_cols %d < ceil(S/blk)", scale_cols);
  SAB_REQUIRE((reinterpret_cast<uintptr_t>(out) & 7) == 0 && o_stride_s % 8 == 0 && o_stride_h % 8 == 0 && o_stride_b % 8 == 0, SAB_ERR_INVALID, "int8 output must be 8-byte aligned");
  QuantParams p{};
  p.x = x; p.mean = mean; p.out = out; p.scale = scale; p.H = H; p.S = S; p.scale_cols = scale_cols;
  p.xsb = x_stride_b; p.xsh = x_stride_h; p.xss = x_stride_s; p.osb = o_stride_b; p.osh = o_stride_h; p.oss = o_stride_s;
  p.blk = blk; p.semantics = semantics; p.has_sm_scale = has_sm_scale; p.sm_scale = sm_scale; p.eps_after = 0;
  // scale columns beyond the last 128-row tile (possible only when the caller over-allocates) are left untouched;
  // the reference per_warp layout ceil(S/128)*4 is fully covered by the tiles.
  return launch_quant(p, dtype, D, kGroupBlock, dim3((S + 127) / 128, H, B), reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int sab_quant_per_thread_int8(const void* x, int dtype, const void* mean, int8_t* out, float* scale, int B,
                                         int H, int S, int D, int64_t x_stride_b, int64_t x_stride_h, int64_t x_stride_s,
                                         int64_t o_stride_b, int64_t o_stride_h, int64_t o_stride_s, int scale_cols,
                                         int is_key, void* stream) {
  int st = check_common(x, dtype, D, x_stride_b, x_stride_h, x_stride_s);
  if (st) return st;
  SAB_REQUIRE(out && scale && B > 0 && H > 0 && S > 0, SAB_ERR_INVALID, "bad arguments to sab_quant_per_thread_int8");
  const int need = is_key ? (S + 63) / 64 * 4 : (S + 127) / 128 * 32;
  SAB_REQUIRE(scale_cols >= need, SAB_ERR_INVALID, "scale_cols %d < %d", scale_cols, need);
  QuantParams p{};
  p.x = x; p.mean = mean; p.out = out; p.scale = scale; p.H = H; p.S = S; p.scale_cols = scale_cols;
  p.xsb = x_stride_b; p.xsh = x_stride_h; p.xss = x_stride_s; p.osb = o_stride_b; p.osh = o_stride_h; p.oss = o_stride_s;
  p.blk = is_key ? 64 : 32; p.semantics = SAB_SEM_TRITON; p.has_sm_scale = 0; p.sm_scale = 1.f; p.eps_after = 1;
  return launch_quant(p, dtype, D, is_key ? kGroupThreadK : kGroupThreadQ, dim3((S + 127) / 128, H, B), reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int sab_quant_per_block_int8_varlen(const void* x, int dtype, const void* mean, int8_t* out, float* scale,
                                               const int32_t* cu_seqlens, const int32_t* cu_scale, int nseq,
                                               int max_seqlen, int H, int D, int64_t x_stride_t, int64_t x_stride_h,
                                               int64_t o_stride_t, int64_t o_stride_h, int blk, int has_sm_scale,
                                               float sm_scale, void* stream) {
  int st = check_common(x, dtype, D, 0, x_stride_h, x_stride_t);
  if (st) return st;
  SAB_REQUIRE(out && scale && cu_seqlens && cu_scale && nseq > 0 && max_seqlen > 0 && H > 0, SAB_ERR_INVALID, "bad arguments to sab_quant_per_block_int8_varlen");
  SAB_REQUIRE(blk == 64 || blk == 128, SAB_ERR_UNSUPPORTED, "Unsupported block size: %d", blk);
  QuantParams p{};
  p.x = x; p.mean = mean; p.out = out; p.scale = scale; p.H = H; p.S = 0; p.scale_cols = 0;
  p.xsh = x_stride_h; p.xss = x_stride_t; p.osh = o_stride_h; p.oss = o_stride_t;
  p.blk = blk; p.semantics = SAB_SEM_TRITON; p.has_sm_scale = has_sm_scale; p.sm_scale = sm_scale; p.eps_after = 0;
  p.cu = cu_seqlens; p.cu_scale = cu_scale;
  return launch_quant(p, dtype, D, kGroupBlock, dim3((max_seqlen + 127) / 128, H, nseq), reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int sab_per_channel_fp8(const void* v, int dtype, uint8_t* v_fp8, float* v_scale, float* v_mean, int B, int H,
                                   int S, int D, int64_t stride_b, int64_t stride_h, int64_t stride_s, int64_t s_pad,
                                   float scale_max, const int32_t* cu_seqlens, const int32_t* cu_pad, int nseq,
                                   int max_seqlen, void* workspace, void* stream) {
  int st = check_common(v, dtype, D, cu_seqlens ? 0 : stride_b, stride_h, stride_s);
  if (st) return st;
  SAB_REQUIRE(v_fp8 && v_scale && workspace && H > 0 && S > 0, SAB_ERR_INVALID, "bad arguments to sab_per_channel_fp8");
  SAB_REQUIRE(s_pad % 128 == 0 && aligned16(v_fp8), SAB_ERR_INVALID, "s_pad must be a multiple of 128 and v_fp8 16-byte aligned");
  const bool varlen = cu_seqlens != nullptr;
  if (varlen) SAB_REQUIRE(cu_pad && nseq > 0 && max_seqlen > 0, SAB_ERR_INVALID, "varlen needs cu_pad, nseq, max_seqlen");
  else SAB_REQUIRE(s_pad >= S && B > 0, SAB_ERR_INVALID, "s_pad < S");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const int Bs = varlen ? 1 : B;  // statistics over all tokens of the packed batch
  if ((st = run_stats(v, dtype, reinterpret_cast<float*>(workspace), Bs, H, S, D, varlen ? 0 : stride_b, stride_h, stride_s, s))) return st;
  const int nchunk = (S + kStatChunk - 1) / kStatChunk;
  float* recp = reinterpret_cast<float*>(workspace) + int64_t(Bs) * H * nchunk * 3 * D;
  channel_stats_stage2<__half><<<Bs * H, 128, 0, s>>>(reinterpret_cast<float*>(workspace), nchunk, D, S, 1, nullptr, v_scale, v_mean, scale_max, recp);
  SAB_CUDA_OK(cudaGetLastError());
  VQuantParams p{};
  p.v = v; p.out = v_fp8; p.recp = recp; p.vmean = v_mean; p.H = H; p.S = S;
  p.sb = stride_b; p.sh = stride_h; p.ss = stride_s; p.s_pad = s_pad; p.scale_max = scale_max; p.cu = cu_seqlens; p.cu_pad = cu_pad;
  dim3 grid(varlen ? (max_seqlen + 127) / 128 : int(s_pad / 128), H, varlen ? nseq : B);
#define SAB_VQ(T, DD) v_quant_transpose_kernel<T, DD><<<grid, 256, 0, s>>>(p)
  if (dtype == SAB_DTYPE_FP16) { if (D == 128) SAB_VQ(__half, 128); else SAB_VQ(__half, 64); }
  else { if (D == 128) SAB_VQ(__nv_bfloat16, 128); else SAB_VQ(__nv_bfloat16, 64); }
#undef SAB_VQ
  SAB_CUDA_OK(cudaGetLastError());
  return SAB_OK;
}

__global__ void amax_to_scale_kernel(const float* __restrict__ amax, float* __restrict__ scale, float* __restrict__ recp,
                                     int n, float scale_max) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    const float a = amax[i];
    scale[i] = __fdividef(a, scale_max);
    recp[i] = a > 0.f ? __fdividef(scale_max, a) : 0.f;
  }
}

extern "C" int sab_channel_stats(const void* x, int dtype, float* sum_out, float* max_out, float* min_out, int B, int H,
                                 int S, int D, int64_t stride_b, int64_t stride_h, int64_t stride_s, void* workspace,
                                 void* stream) {
  int st = check_common(x, dtype, D, stride_b, stride_h, stride_s);
  if (st) return st;
  SAB_REQUIRE(sum_out && max_out && min_out && workspace && B > 0 && H > 0 && S > 0, SAB_ERR_INVALID, "bad arguments to sab_channel_stats");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if ((st = run_stats(x, dtype, reinterpret_cast<float*>(workspace), B, H, S, D, stride_b, stride_h, stride_s, s))) return st;
  const int nchunk = (S + kStatChunk - 1) / kStatChunk;
  channel_stats_stage2<__half><<<B * H, 128, 0, s>>>(reinterpret_cast<float*>(workspace), nchunk, D, S, 2, nullptr, sum_out, max_out, 0.f, min_out);
  SAB_CUDA_OK(cudaGetLastError());
  return SAB_OK;
}

extern "C" int sab_v_quant_with_amax(const void* v, int dtype, uint8_t* v_fp8, const float* amax, float* v_scale, int B,
                                     int H, int S, int D, int64_t stride_b, int64_t stride_h, int64_t stride_s,
                                     int64_t s_pad, float scale_max, void* workspace, void* stream) {
  int st = check_common(v, dtype, D, stride_b, stride_h, stride_s);
  if (st) return st;
  SAB_REQUIRE(v_fp8 && amax && v_scale && workspace && B > 0 && H > 0 && S > 0, SAB_ERR_INVALID, "bad arguments to sab_v_quant_with_amax");
  SAB_REQUIRE(s_pad % 128 == 0 && s_pad >= S && aligned16(v_fp8), SAB_ERR_INVALID, "s_pad must be a multiple of 128, >= S, v_fp8 16-byte aligned");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  float* recp = reinterpret_cast<float*>(workspace);   // B*H*D floats
  const int n = B * H * D;
  amax_to_scale_kernel<<<(n + 255) / 256, 256, 0, s>>>(amax, v_scale, recp, n, scale_max);
  SAB_CUDA_OK(cudaGetLastError());
  VQuantParams p{};
  p.v = v; p.out = v_fp8; p.recp = recp; p.vmean = nullptr; p.H = H; p.S = S;
  p.sb = stride_b; p.sh = stride_h; p.ss = stride_s; p.s_pad = s_pad; p.scale_max = scale_max; p.cu = nullptr; p.cu_pad = nullptr;
  dim3 grid(int(s_pad / 128), H, B);
#define SAB_VQ(T, DD) v_quant_transpose_kernel<T, DD><<<grid, 256, 0, s>>>(p)
  if (dtype == SAB_DTYPE_FP16) { if (D == 128) SAB_VQ(__half, 128); else SAB_VQ(__half, 64); }
  else { if (D == 128) SAB_VQ(__nv_bfloat16, 128); else SAB_VQ(__nv_bfloat16, 64); }
#undef SAB_VQ
  SAB_CUDA_OK(cudaGetLastError());
  return SAB_OK;
}

extern "C" int sab_v_transpose_f16(const void* v, int dtype, void* v_f16t, int B, int H, int S, int D, int64_t stride_b,
                                   int64_t stride_h, int64_t stride_s, int64_t s_pad, const int32_t* cu_seqlens,
                                   const int32_t* cu_pad, int nseq, int max_seqlen, void* stream) {
  int st = check_common(v, dtype, D, cu_seqlens ? 0 : stride_b, stride_h, stride_s);
  if (st) return st;
  SAB_REQUIRE(v_f16t && H > 0 && S > 0, SAB_ERR_INVALID, "bad arguments to sab_v_transpose_f16");
  SAB_REQUIRE(s_pad % 128 == 0 && aligned16(v_f16t), SAB_ERR_INVALID, "s_pad must be a multiple of 128 and the output 16-byte aligned");
  const bool varlen = cu_seqlens != nullptr;
  if (varlen) SAB_REQUIRE(cu_pad && nseq > 0 && max_seqlen > 0, SAB_ERR_INVALID, "varlen needs cu_pad, nseq, max_seqlen");
  else SAB_REQUIRE(s_pad >= S && B > 0, SAB_ERR_INVALID, "s_pad < S");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  VQuantParams p{};
  p.v = v; p.out = reinterpret_cast<uint8_t*>(v_f16t); p.H = H; p.S = S;
  p.sb = stride_b; p.sh = stride_h; p.ss = stride_s; p.s_pad = s_pad; p.cu = cu_seqlens; p.cu_pad = cu_pad;
  dim3 grid(varlen ? (max_seqlen + 127) / 128 : int(s_pad / 128), H, varlen ? nseq : B);
#define SAB_VT(T, DD) v_transpose_f16_kernel<T, DD><<<grid, 256, 0, s>>>(p)
  if (dtype == SAB_DTYPE_FP16) { if (D == 128) SAB_VT(__half, 128); else SAB_VT(__half, 64); }
  else { if (D == 128) SAB_VT(__nv_bfloat16, 128); else SAB_VT(__nv_bfloat16, 64); }
#undef SAB_VT
  SAB_CUDA_OK(cudaGetLastError());
  return SAB_OK;
}

extern "C" int sab_k_smooth_quant_int8(const void* k, int dtype, void* mean_out, int8_t* out, float* scale, int B, int H, int S,
                                       int D, int64_t x_stride_b, int64_t x_stride_h, int64_t x_stride_s, int64_t o_stride_b,
                                       int64_t o_stride_h, int64_t o_stride_s, int scale_cols, int granularity, void* stream) {
  int st = check_common(k, dtype, D, x_stride_b, x_stride_h, x_stride_s);
  if (st) return st;
  SAB_REQUIRE(mean_out && out && scale && B > 0 && H > 0 && S > 0, SAB_ERR_INVALID, "bad arguments to sab_k_smooth_quant_int8");
  SAB_REQUIRE(granularity == SAB_GRAN_PER_WARP || granularity == SAB_GRAN_PER_THREAD || granularity == SAB_GRAN_PER_BLOCK, SAB_ERR_INVALID,
              "unknown granularity %d", granularity);
  const bool pt = granularity == SAB_GRAN_PER_THREAD;
  const int need = pt ? (S + 63) / 64 * 4 : (S + 63) / 64;
  SAB_REQUIRE(scale_cols >= need, SAB_ERR_INVALID, "scale_cols %d < %d", scale_cols, need);
  SAB_REQUIRE((reinterpret_cast<uintptr_t>(out) & 7) == 0 && o_stride_s % 8 == 0 && o_stride_h % 8 == 0 && o_stride_b % 8 == 0, SAB_ERR_INVALID, "int8 output must be 8-byte aligned");
  QuantParams p{};
  p.x = k; p.mean = mean_out; p.out = out; p.scale = scale; p.H = H; p.S = S; p.scale_cols = scale_cols;
  p.xsb = x_stride_b; p.xsh = x_stride_h; p.xss = x_stride_s; p.osb = o_stride_b; p.osh = o_stride_h; p.oss = o_stride_s;
  p.blk = 64; p.has_sm_scale = 0; p.sm_scale = 1.f;
  p.semantics = pt ? SAB_SEM_TRITON : SAB_SEM_CUDA;   // per-thread: quant_per_thread.py semantics; per-warp: csrc/fused/fused.cu
  p.eps_after = pt ? 1 : 0;
  const dim3 grid(kKCluster, H, B);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
#define SAB_KF(T, DD)                                                                                                             \
  do {                                                                                                                            \
    if (pt) return launch_cluster(k_smooth_quant_kernel<T, DD, kGroupThreadK, kQfTriton | kQfMean>, grid, s, p, reinterpret_cast<T*>(mean_out)); \
    return launch_cluster(k_smooth_quant_kernel<T, DD, kGroupBlock, kQfMean>, grid, s, p, reinterpret_cast<T*>(mean_out));       \
  } while (0)
  if (dtype == SAB_DTYPE_FP16) { if (D == 128) SAB_KF(__half, 128); else SAB_KF(__half, 64); }
  else { if (D == 128) SAB_KF(__nv_bfloat16, 128); else SAB_KF(__nv_bfloat16, 64); }
#undef SAB_KF
}

extern "C" int sab_per_channel_fp8_fused(const void* v, int dtype, uint8_t* v_fp8, float* v_scale, float* v_mean, int B, int H,
                                         int S, int D, int64_t stride_b, int64_t stride_h, int64_t stride_s, int64_t s_pad,
                                         float scale_max, void* stream) {
  int st = check_common(v, dtype, D, stride_b, stride_h, stride_s);
  if (st) return st;
  SAB_REQUIRE(v_fp8 && v_scale && B > 0 && H > 0 && S > 0, SAB_ERR_INVALID, "bad arguments to sab_per_channel_fp8_fused");
  SAB_REQUIRE(s_pad % 128 == 0 && s_pad >= S && aligned16(v_fp8), SAB_ERR_INVALID, "s_pad must be a multiple of 128, >= S, v_fp8 16-byte aligned");
  VQuantParams p{};
  p.v = v; p.out = v_fp8; p.recp = nullptr; p.vmean = nullptr; p.H = H; p.S = S;
  p.sb = stride_b; p.sh = stride_h; p.ss = stride_s; p.s_pad = s_pad; p.scale_max = scale_max; p.cu = nullptr; p.cu_pad = nullptr;
  const dim3 grid(kKCluster, H, B);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (dtype == SAB_DTYPE_FP16) {
    if (D == 128) return launch_cluster(v_scale_quant_kernel<__half, 128>, grid, s, p, v_scale, v_mean);
    return launch_cluster(v_scale_quant_kernel<__half, 64>, grid, s, p, v_scale, v_mean);
  }
  if (D == 128) return launch_cluster(v_scale_quant_kernel<__nv_bfloat16, 128>, grid, s, p, v_scale, v_mean);
  return launch_cluster(v_scale_quant_kernel<__nv_bfloat16, 64>, grid, s, p, v_scale, v_mean);
}

// ---------------------------------------------------------------------------------------------- per-sequence varlen front-end
// Packed [T,H,D] inputs, every statistic and scale block taken per sequence: sequence b gives the bits of the dense call on
// tokens [cu_seqlens[b], cu_seqlens[b+1]) alone.
extern "C" int64_t sab_k_mean_varlen_workspace_bytes(int nseq, int H, int max_seqlen, int D) {
  return sab_k_mean_workspace_bytes(nseq, H, max_seqlen, D);
}
extern "C" int64_t sab_per_channel_fp8_varlen_workspace_bytes(int nseq, int H, int max_seqlen, int D) {
  return sab_per_channel_fp8_workspace_bytes(nseq, H, max_seqlen, D);
}

template <typename T, int D>
static void launch_stats_seq(const void* x, float* part, const int32_t* cu, int nseq, int H, int nchunk, int64_t sh, int64_t ss,
                             cudaStream_t st, const PageTable* pg) {
  const dim3 grid(nchunk, H, nseq);
  if (pg != nullptr) channel_stats_stage1_paged<T, D><<<grid, 256, 0, st>>>(reinterpret_cast<const T*>(x), part, sh, ss, nchunk, cu, *pg);
  else channel_stats_stage1<T, D, true><<<grid, 256, 0, st>>>(reinterpret_cast<const T*>(x), part, 0, 0, sh, ss, nchunk, cu);
}
static int run_stats_seq(const void* x, int dtype, float* part, const int32_t* cu, int nseq, int H, int nchunk, int D, int64_t sh,
                         int64_t ss, cudaStream_t st, const PageTable* pg) {
  if (dtype == SAB_DTYPE_FP16) {
    if (D == 128) launch_stats_seq<__half, 128>(x, part, cu, nseq, H, nchunk, sh, ss, st, pg);
    else launch_stats_seq<__half, 64>(x, part, cu, nseq, H, nchunk, sh, ss, st, pg);
  } else {
    if (D == 128) launch_stats_seq<__nv_bfloat16, 128>(x, part, cu, nseq, H, nchunk, sh, ss, st, pg);
    else launch_stats_seq<__nv_bfloat16, 64>(x, part, cu, nseq, H, nchunk, sh, ss, st, pg);
  }
  SAB_CUDA_OK(cudaGetLastError());
  return SAB_OK;
}

// The per-sequence front-end on packed input (pg == nullptr) or on a paged cache (pg: block table and page geometry).  The
// sequences, their lengths and every output layout come from cu_seqlens in both cases; only the input rows are addressed differently.
static int k_mean_seq(const void* k, int dtype, void* mean, const int32_t* cu_seqlens, int nseq, int max_seqlen, int H, int D,
                      int64_t stride_t, int64_t stride_h, void* workspace, void* stream, const PageTable* pg) {
  SAB_REQUIRE(mean && workspace && cu_seqlens && nseq > 0 && max_seqlen > 0 && H > 0, SAB_ERR_INVALID, "bad arguments to sab_k_mean_varlen");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const int nchunk = (max_seqlen + kStatChunk - 1) / kStatChunk;
  float* part = reinterpret_cast<float*>(workspace);
  if (int st = run_stats_seq(k, dtype, part, cu_seqlens, nseq, H, nchunk, D, stride_h, stride_t, s, pg)) return st;
  if (dtype == SAB_DTYPE_FP16)
    channel_stats_stage2<__half, true><<<dim3(H, nseq), 128, 0, s>>>(part, nchunk, D, 0, 0, reinterpret_cast<__half*>(mean), nullptr,
                                                                     nullptr, 0.f, nullptr, cu_seqlens);
  else
    channel_stats_stage2<__nv_bfloat16, true><<<dim3(H, nseq), 128, 0, s>>>(part, nchunk, D, 0, 0, reinterpret_cast<__nv_bfloat16*>(mean),
                                                                            nullptr, nullptr, 0.f, nullptr, cu_seqlens);
  SAB_CUDA_OK(cudaGetLastError());
  return SAB_OK;
}

static int quant_int8_seq(const void* x, int dtype, const void* mean, int8_t* out, float* scale, const int32_t* cu_seqlens,
                          const int32_t* cu_scale, int nseq, int max_seqlen, int H, int D, int64_t x_stride_t, int64_t x_stride_h,
                          int64_t o_stride_t, int64_t o_stride_h, int granularity, int is_key, void* stream, const PageTable* pg) {
  SAB_REQUIRE(out && scale && cu_seqlens && cu_scale && nseq > 0 && max_seqlen > 0 && H > 0, SAB_ERR_INVALID,
              "bad arguments to sab_quant_int8_varlen");
  SAB_REQUIRE(granularity == SAB_GRAN_PER_WARP || granularity == SAB_GRAN_PER_THREAD, SAB_ERR_INVALID,
              "granularity must be SAB_GRAN_PER_WARP or SAB_GRAN_PER_THREAD (got %d)", granularity);
  SAB_REQUIRE(mean == nullptr || is_key, SAB_ERR_INVALID, "the mean is subtracted from K only (is_key == 0)");
  SAB_REQUIRE((reinterpret_cast<uintptr_t>(out) & 7) == 0 && o_stride_t % 8 == 0 && o_stride_h % 8 == 0, SAB_ERR_INVALID,
              "int8 output must be 8-byte aligned");
  const bool pt = granularity == SAB_GRAN_PER_THREAD;
  QuantParams p{};
  p.x = x; p.mean = mean; p.out = out; p.scale = scale; p.H = H; p.S = 0; p.scale_cols = 0;
  p.xsh = x_stride_h; p.xss = x_stride_t; p.osh = o_stride_h; p.oss = o_stride_t;
  // per-thread: quant_per_thread.py semantics (sab_quant_per_thread_int8); per-warp: csrc/fused/fused.cu (blk 32 Q, 64 K)
  p.blk = is_key ? 64 : 32;
  p.semantics = pt ? SAB_SEM_TRITON : SAB_SEM_CUDA;
  p.eps_after = pt ? 1 : 0;
  p.has_sm_scale = 0; p.sm_scale = 1.f;
  p.cu = cu_seqlens; p.cu_scale = cu_scale;
  const int mode = pt ? (is_key ? kGroupThreadK : kGroupThreadQ) : kGroupBlock;
  return launch_quant_seq(p, dtype, D, mode, dim3((max_seqlen + 127) / 128, H, nseq), reinterpret_cast<cudaStream_t>(stream), pg);
}

static int per_channel_fp8_seq(const void* v, int dtype, uint8_t* v_fp8, float* v_scale, float* v_mean, const int32_t* cu_seqlens,
                               const int32_t* cu_pad, int nseq, int max_seqlen, int H, int D, int64_t stride_t, int64_t stride_h,
                               int64_t t_pad, float scale_max, void* workspace, void* stream, const PageTable* pg) {
  SAB_REQUIRE(v_fp8 && v_scale && workspace && cu_seqlens && cu_pad && nseq > 0 && max_seqlen > 0 && H > 0, SAB_ERR_INVALID,
              "bad arguments to sab_per_channel_fp8_varlen");
  SAB_REQUIRE(t_pad % 128 == 0 && aligned16(v_fp8), SAB_ERR_INVALID, "t_pad must be a multiple of 128 and v_fp8 16-byte aligned");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const int nchunk = (max_seqlen + kStatChunk - 1) / kStatChunk;
  float* part = reinterpret_cast<float*>(workspace);
  float* recp = part + int64_t(nseq) * H * nchunk * 3 * D;
  if (int st = run_stats_seq(v, dtype, part, cu_seqlens, nseq, H, nchunk, D, stride_h, stride_t, s, pg)) return st;
  channel_stats_stage2<__half, true><<<dim3(H, nseq), 128, 0, s>>>(part, nchunk, D, 0, 1, nullptr, v_scale, v_mean, scale_max, recp,
                                                                   cu_seqlens);
  SAB_CUDA_OK(cudaGetLastError());
  VQuantParams p{};
  p.v = v; p.out = v_fp8; p.recp = recp; p.vmean = v_mean; p.H = H; p.S = 0;
  p.sb = 0; p.sh = stride_h; p.ss = stride_t; p.s_pad = t_pad; p.scale_max = scale_max; p.cu = cu_seqlens; p.cu_pad = cu_pad;
  const dim3 grid((max_seqlen + 127) / 128, H, nseq);
#define SAB_VQ(T, DD)                                                                                  \
  do {                                                                                                 \
    if (pg != nullptr) v_quant_transpose_paged_kernel<T, DD><<<grid, 256, 0, s>>>(p, *pg);             \
    else v_quant_transpose_kernel<T, DD, true><<<grid, 256, 0, s>>>(p);                                \
  } while (0)
  if (dtype == SAB_DTYPE_FP16) { if (D == 128) SAB_VQ(__half, 128); else SAB_VQ(__half, 64); }
  else { if (D == 128) SAB_VQ(__nv_bfloat16, 128); else SAB_VQ(__nv_bfloat16, 64); }
#undef SAB_VQ
  SAB_CUDA_OK(cudaGetLastError());
  return SAB_OK;
}

extern "C" int sab_k_mean_varlen(const void* k, int dtype, void* mean, const int32_t* cu_seqlens, int nseq, int max_seqlen, int H,
                                 int D, int64_t stride_t, int64_t stride_h, void* workspace, void* stream) {
  if (int st = check_common(k, dtype, D, 0, stride_h, stride_t)) return st;
  return k_mean_seq(k, dtype, mean, cu_seqlens, nseq, max_seqlen, H, D, stride_t, stride_h, workspace, stream, nullptr);
}

extern "C" int sab_quant_int8_varlen(const void* x, int dtype, const void* mean, int8_t* out, float* scale, const int32_t* cu_seqlens,
                                     const int32_t* cu_scale, int nseq, int max_seqlen, int H, int D, int64_t x_stride_t,
                                     int64_t x_stride_h, int64_t o_stride_t, int64_t o_stride_h, int granularity, int is_key,
                                     void* stream) {
  if (int st = check_common(x, dtype, D, 0, x_stride_h, x_stride_t)) return st;
  return quant_int8_seq(x, dtype, mean, out, scale, cu_seqlens, cu_scale, nseq, max_seqlen, H, D, x_stride_t, x_stride_h, o_stride_t,
                        o_stride_h, granularity, is_key, stream, nullptr);
}

extern "C" int sab_per_channel_fp8_varlen(const void* v, int dtype, uint8_t* v_fp8, float* v_scale, float* v_mean,
                                          const int32_t* cu_seqlens, const int32_t* cu_pad, int nseq, int max_seqlen, int H, int D,
                                          int64_t stride_t, int64_t stride_h, int64_t t_pad, float scale_max, void* workspace,
                                          void* stream) {
  if (int st = check_common(v, dtype, D, 0, stride_h, stride_t)) return st;
  return per_channel_fp8_seq(v, dtype, v_fp8, v_scale, v_mean, cu_seqlens, cu_pad, nseq, max_seqlen, H, D, stride_t, stride_h, t_pad,
                             scale_max, workspace, stream, nullptr);
}

// ---------------------------------------------------------------------------------------------- per-sequence front-end, paged input
// The per-sequence varlen front-end reading a paged cache [num_pages, page_size, H, D] through a block table: the outputs are the
// packed form's, bit for bit those of the varlen entries on the gathered packed tensor.
static int check_paged(const void* x, int dtype, int D, const int32_t* block_table, int64_t table_stride, int page_size,
                       int64_t page_stride, int64_t stride_t, int64_t stride_h, PageTable& pg) {
  if (int st = check_common(x, dtype, D, page_stride, stride_h, stride_t)) return st;
  SAB_REQUIRE(block_table != nullptr && table_stride >= 0 && page_size > 0 && page_stride >= 0, SAB_ERR_INVALID,
              "the paged form needs a block table, table_stride >= 0, page_size > 0 and page_stride >= 0");
  pg = PageTable{block_table, table_stride, page_size, page_stride};
  return SAB_OK;
}

extern "C" int sab_k_mean_paged(const void* k_cache, int dtype, void* mean, const int32_t* cu_seqlens, const int32_t* block_table,
                                int64_t table_stride, int page_size, int nseq, int max_seqlen, int H, int D, int64_t page_stride,
                                int64_t stride_t, int64_t stride_h, void* workspace, void* stream) {
  PageTable pg;
  if (int st = check_paged(k_cache, dtype, D, block_table, table_stride, page_size, page_stride, stride_t, stride_h, pg)) return st;
  return k_mean_seq(k_cache, dtype, mean, cu_seqlens, nseq, max_seqlen, H, D, stride_t, stride_h, workspace, stream, &pg);
}

extern "C" int sab_quant_int8_paged(const void* k_cache, int dtype, const void* mean, int8_t* out, float* scale,
                                    const int32_t* cu_seqlens, const int32_t* cu_scale, const int32_t* block_table, int64_t table_stride,
                                    int page_size, int nseq, int max_seqlen, int H, int D, int64_t page_stride, int64_t stride_t,
                                    int64_t stride_h, int64_t o_stride_t, int64_t o_stride_h, int granularity, void* stream) {
  PageTable pg;
  if (int st = check_paged(k_cache, dtype, D, block_table, table_stride, page_size, page_stride, stride_t, stride_h, pg)) return st;
  return quant_int8_seq(k_cache, dtype, mean, out, scale, cu_seqlens, cu_scale, nseq, max_seqlen, H, D, stride_t, stride_h, o_stride_t,
                        o_stride_h, granularity, 1, stream, &pg);
}

extern "C" int sab_per_channel_fp8_paged(const void* v_cache, int dtype, uint8_t* v_fp8, float* v_scale, float* v_mean,
                                         const int32_t* cu_seqlens, const int32_t* cu_pad, const int32_t* block_table,
                                         int64_t table_stride, int page_size, int nseq, int max_seqlen, int H, int D, int64_t page_stride,
                                         int64_t stride_t, int64_t stride_h, int64_t t_pad, float scale_max, void* workspace,
                                         void* stream) {
  PageTable pg;
  if (int st = check_paged(v_cache, dtype, D, block_table, table_stride, page_size, page_stride, stride_t, stride_h, pg)) return st;
  return per_channel_fp8_seq(v_cache, dtype, v_fp8, v_scale, v_mean, cu_seqlens, cu_pad, nseq, max_seqlen, H, D, stride_t, stride_h,
                             t_pad, scale_max, workspace, stream, &pg);
}
