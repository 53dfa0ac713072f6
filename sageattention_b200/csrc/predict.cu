// Block-mask prediction from pooled Q/K statistics (predict_block_mask): the block_mask of sab_qk_int8_sv_f8_attn_blocksparse
// chosen from per-block means and self-similarities (SpargeAttn's first stage, training-free).
//   predict_stats_kernel  : one read of q or k; per block of `blk` rows the fp32 mean m and the self-similarity
//                        s = |sum of unit rows|^2 / n^2 (the mean of the block's cosine-similarity matrix).
//   predict_select_kernel : per 128-row Q block, the softmax over the candidate key blocks of sm_scale * (m_q . m_k), the smallest
//                        prefix of them in descending order whose mass reaches cdf_threshold, plus the forced rows / columns and
//                        the causal diagonal; writes the mask bytes.
// The definition every layer follows is in include/sageattn_b200.h.  Deterministic: fixed summation orders, no atomics.
#include <cmath>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include "attn_common.cuh"

namespace sab {

constexpr int kStatsThreads = 128;
constexpr int kSelThreads = 256;
constexpr int kSelWarps = kSelThreads / 32;
constexpr int kSelChunk = 32;          // key-block means staged in shared memory per pass
constexpr int kSelMaxRows = 16;        // Q blocks per select CTA (fewer when nk is large)
constexpr int kMaxKeyBlocks = 16384;   // Skv <= 1048576, the limit of the block-sparse attention
constexpr int kSelSmemMax = 226 * 1024;  // dynamic shared memory: 227 KB per CTA less the static part

template <typename T>
__device__ __forceinline__ float to_float(T v);
template <>
__device__ __forceinline__ float to_float<__half>(__half v) { return __half2float(v); }
template <>
__device__ __forceinline__ float to_float<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }

// Grid (nblk, H, B); DP = D rounded up to 64 or 128, each row read by DP/8 threads with one 16-byte load (lanes past D read 0).
// kSeq: the packed form (sab_block_stats_varlen).  x is [T,H,D] (sb unused), b is the sequence, and its blocks restart at its first
// token cu[b]: block nb of sequence b is the dense kernel's block nb of that sequence alone.  The grid is sized by the longest
// sequence (nblk = ceil(max_seqlen/blk)); a block past the end of its sequence writes mean 0 and sim 0.
template <typename T, int DP, bool kSeq = false>
__global__ void __launch_bounds__(kStatsThreads) predict_stats_kernel(const T* __restrict__ x, float* __restrict__ mean,
                                                                     float* __restrict__ sim, int S, int D, int blk, int64_t sb,
                                                                     int64_t sh, int64_t ss, const int32_t* __restrict__ cu = nullptr) {
  constexpr int TPR = DP / 8;                 // threads per row (8 or 16: a power of two inside one warp)
  constexpr int RPP = kStatsThreads / TPR;    // rows per pass
  const int nb = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int tr = threadIdx.x / TPR, tc = threadIdx.x % TPR;
  const int r0 = nb * blk;
  [[maybe_unused]] int64_t tok0 = 0;   // packed form: the sequence's first token
  if constexpr (kSeq) {
    tok0 = cu[b];
    S = cu[b + 1] - cu[b];
    if (r0 >= S) {
      const int64_t blk_idx = (int64_t(b) * gridDim.y + h) * gridDim.x + nb;
      for (int d = threadIdx.x; d < D; d += kStatsThreads) mean[blk_idx * D + d] = 0.f;
      if (threadIdx.x == 0) sim[blk_idx] = 0.f;
      return;
    }
  }
  const int n = min(blk, S - r0);
  const bool live = tc * 8 < D;
  const T* base = kSeq ? x + h * sh + (tok0 + r0) * ss + tc * 8 : x + b * sb + h * sh + int64_t(r0) * ss + tc * 8;
  float sx[8], su[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) { sx[e] = 0.f; su[e] = 0.f; }
  const int passes = (n + RPP - 1) / RPP;     // the same count in every thread: the row norm is a warp shuffle
#pragma unroll 4
  for (int it = 0; it < passes; ++it) {
    const int r = tr + it * RPP;
    float f[8];
    if (live && r < n) {
      const uint4 raw = *reinterpret_cast<const uint4*>(base + int64_t(r) * ss);
      const T* e = reinterpret_cast<const T*>(&raw);
#pragma unroll
      for (int i = 0; i < 8; ++i) f[i] = to_float<T>(e[i]);
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) f[i] = 0.f;
    }
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) q = fmaf(f[i], f[i], q);
#pragma unroll
    for (int o = TPR / 2; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
    const float inv = q > 0.f ? 1.f / sqrtf(q) : 0.f;   // a zero row has unit vector 0
#pragma unroll
    for (int i = 0; i < 8; ++i) { sx[i] += f[i]; su[i] = fmaf(f[i], inv, su[i]); }
  }
  __shared__ float s_x[RPP][DP], s_u[RPP][DP];
  __shared__ float s_red[kStatsThreads / 32];
#pragma unroll
  for (int i = 0; i < 8; ++i) { s_x[tr][tc * 8 + i] = sx[i]; s_u[tr][tc * 8 + i] = su[i]; }
  __syncthreads();
  const int d = threadIdx.x;
  float ax = 0.f, au = 0.f;
  if (d < DP) {
    for (int r = 0; r < RPP; ++r) { ax += s_x[r][d]; au += s_u[r][d]; }
  }
  const int64_t blk_idx = (int64_t(b) * gridDim.y + h) * gridDim.x + nb;
  if (d < D) mean[blk_idx * D + d] = ax / float(n);
  float t = au * au;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = t;
  __syncthreads();
  if (threadIdx.x == 0) {
    float tot = 0.f;
    for (int w = 0; w < kStatsThreads / 32; ++w) tot += s_red[w];
    sim[blk_idx] = tot / (float(n) * float(n));
  }
}

struct SelectParams {
  const float* qm;   // [B,Hq,nq,D]
  const float* qs;   // [B,Hq,nq]
  const float* km;   // [B,Hkv,nk,D]
  const float* ks;   // [B,Hkv,nk]
  uint8_t* mask;     // [B,Hq,nq,nk]
  int Hq, Hkv, nq, nk, D, npow, rows, causal;
  float scale_log2, cdf, sim;
  // packed form (predict_select_kernel<true>): B = nseq, nq / nk / npow are the bounds of the longest sequences (the tensors'
  // extents), and sequence b's own are read from the sequence tables on the device
  const int32_t* cu_q;
  const int32_t* cu_k;
};

// Every thread gets the reduction of v over the CTA, in a fixed order.  red: kSelWarps floats, free on entry.
template <bool kMax>
__device__ __forceinline__ float block_reduce(float v, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float w = __shfl_xor_sync(0xffffffffu, v, o);
    v = kMax ? fmaxf(v, w) : v + w;
  }
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = red[0];
  for (int w = 1; w < kSelWarps; ++w) r = kMax ? fmaxf(r, red[w]) : r + red[w];
  __syncthreads();
  return r;
}

__device__ __forceinline__ float key_p(uint64_t key) { return __uint_as_float(uint32_t(key >> 32)); }

// Grid (ceil(nq/rows), Hq, B).  Shared memory: npow sort keys, the rows' Q means, one chunk of K means, the rows' logits.
// kSeq: the packed form (sab_predict_block_mask_varlen).  b is the sequence; its rows run the dense kernel's steps on its own
// nq_b = ceil(Lq_b/128) rows and nk_b = ceil(Lk_b/64) key blocks, with its own sort length npow_b (the bitonic network and the
// scan's per-thread chunks depend on it, and so does the fp32 order of the prefix mass), so slice [b, :, :nq_b, :nk_b] is the
// dense kernel's mask of that sequence alone.  Every other byte of the sequence's [Hq, nq, nk] slab is written 0.
template <bool kSeq = false>
__global__ void __launch_bounds__(kSelThreads) predict_select_kernel(const SelectParams p) {
  extern __shared__ __align__(16) unsigned char smem[];
  uint64_t* keys = reinterpret_cast<uint64_t*>(smem);
  float* qmean = reinterpret_cast<float*>(keys + p.npow);
  float* kstage = qmean + p.rows * p.D;             // kSelChunk rows of D + 1 floats: conflict-free column reads
  float* logit = kstage + kSelChunk * (p.D + 1);    // rows x nk, log2 units
  __shared__ float red[kSelWarps];
  __shared__ float scan[kSelWarps];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int h = blockIdx.y, b = blockIdx.z, hk = h / (p.Hq / p.Hkv);
  const int D = p.D;
  int nk = p.nk, npow = p.npow;   // packed form: this sequence's; the tensors keep the strides p.nq, p.nk
  const int i0 = blockIdx.x * p.rows;
  int nr = min(p.rows, p.nq - i0);
  const int64_t qrow0 = (int64_t(b) * p.Hq + h) * p.nq + i0;
  const float* km = p.km + (int64_t(b) * p.Hkv + hk) * nk * D;
  const float* ks = p.ks + (int64_t(b) * p.Hkv + hk) * nk;
  if constexpr (kSeq) {
    const int lq = p.cu_q[b + 1] - p.cu_q[b], lk = p.cu_k[b + 1] - p.cu_k[b];
    const int nq = lk > 0 ? (lq + 127) / 128 : 0;   // a sequence without keys has no visible block
    nk = (lk + 63) / 64;
    npow = 1;
    while (npow < nk) npow <<= 1;
    // the bytes outside the sequence's blocks: whole rows past nq_b, columns past nk_b
    for (int r = 0; r < nr; ++r) {
      uint8_t* out = p.mask + (qrow0 + r) * p.nk;
      for (int j = (i0 + r < nq ? nk : 0) + tid; j < p.nk; j += kSelThreads) out[j] = 0;
    }
    if (i0 >= nq) return;
    nr = min(nr, nq - i0);
  }
  for (int t = tid; t < nr * D; t += kSelThreads) qmean[t] = p.qm[qrow0 * D + t];

  // 1. logits of every (row, key block) the CTA's rows can see, the K means staged once for all rows
  const int jlim = p.causal ? min(nk, 2 * (i0 + nr - 1) + 2) : nk;
  for (int j0 = 0; j0 < jlim; j0 += kSelChunk) {
    const int nj = min(kSelChunk, jlim - j0);
    __syncthreads();
    for (int t = tid; t < nj * D; t += kSelThreads) kstage[(t / D) * (D + 1) + t % D] = km[int64_t(j0) * D + t];
    __syncthreads();
    for (int t = tid; t < nr * kSelChunk; t += kSelThreads) {
      const int r = t / kSelChunk, jj = t % kSelChunk;
      if (jj < nj) {
        const float* a = qmean + r * D;
        const float* c = kstage + jj * (D + 1);
        float acc = 0.f;
#pragma unroll 8
        for (int d = 0; d < D; ++d) acc = fmaf(a[d], c[d], acc);
        logit[r * nk + j0 + jj] = acc * p.scale_log2;
      }
    }
  }
  __syncthreads();

  // 2. per row: softmax over the candidates, descending order (ties: ascending j), prefix mass, forced blocks, mask bytes
  const int per = (npow + kSelThreads - 1) / kSelThreads;   // sorted positions scanned by each thread, contiguous
  for (int r = 0; r < nr; ++r) {
    const int i = i0 + r;
    const bool row_forced = p.qs[qrow0 + r] < p.sim;
    const int jmax = p.causal ? min(nk - 1, 2 * i + 1) : nk - 1;   // causal horizon: 64 j <= 128 i + 127
    float* lg = logit + r * nk;
    uint8_t* kept = reinterpret_cast<uint8_t*>(lg);                // reuses the row's logits once the keys are built
    const bool select = !row_forced && p.cdf < 1.f;                // cdf >= 1 keeps every candidate by rule
    if (select) {
      float mx = -INFINITY;
      for (int j = tid; j <= jmax; j += kSelThreads)
        if (ks[j] >= p.sim) mx = fmaxf(mx, lg[j]);
      mx = block_reduce<true>(mx, red);
      float sum = 0.f;
      for (int j = tid; j <= jmax; j += kSelThreads)
        if (ks[j] >= p.sim) sum += exp2f(lg[j] - mx);
      sum = block_reduce<false>(sum, red);
      // key = (p bits, ~j): p >= 0, so descending keys are descending p with ties in ascending j; non-candidates are 0
      for (int t = tid; t < npow; t += kSelThreads) {
        uint64_t key = 0;
        if (t <= jmax && ks[t] >= p.sim)
          key = (uint64_t(__float_as_uint(__fdiv_rn(exp2f(lg[t] - mx), sum))) << 32) | uint32_t(~uint32_t(t));
        keys[t] = key;
      }
      __syncthreads();
      for (int k = 2; k <= npow; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
          for (int t = tid; t < (npow >> 1); t += kSelThreads) {
            const int lo = ((t & ~(j - 1)) << 1) | (t & (j - 1));
            const int hi = lo + j;
            const uint64_t a = keys[lo], c = keys[hi];
            if (((lo & k) == 0) ? a < c : a > c) { keys[lo] = c; keys[hi] = a; }
          }
          __syncthreads();
        }
      }
      for (int j = tid; j < nk; j += kSelThreads) kept[j] = 0;
      // exclusive prefix sum of p over the sorted positions: per-thread chunk, then warp and CTA offsets (fixed order)
      const int t0 = tid * per;
      float local = 0.f;
      for (int u = 0; u < per; ++u)
        if (t0 + u < npow) local += key_p(keys[t0 + u]);
      float inc = local;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const float w = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += w;
      }
      if (lane == 31) scan[warp] = inc;
      __syncthreads();
      float run = inc - local;
      for (int w = 0; w < warp; ++w) run += scan[w];
      for (int u = 0; u < per; ++u) {
        const int t = t0 + u;
        if (t >= npow) break;
        const uint64_t key = keys[t];
        if (key != 0 && run < p.cdf) kept[~uint32_t(key)] = 1;
        run += key_p(key);
      }
      __syncthreads();
    }
    uint8_t* out = p.mask + (qrow0 + r) * p.nk;
    for (int j = tid; j < nk; j += kSelThreads) {
      bool v = false;
      if (j <= jmax) {
        const bool col_forced = ks[j] < p.sim;
        const bool diag = p.causal && j >= 2 * i;                  // 128 i <= 64 j + 63 and j <= jmax
        v = !select || col_forced || diag || kept[j] != 0;
      }
      out[j] = v ? 1 : 0;
    }
    __syncthreads();   // the next row's reductions reuse red / scan and its keys overwrite these
  }
}

template <typename T, int DP, bool kSeq = false>
int launch_stats(const void* x, float* mean, float* sim, int B, int H, int S, int D, int64_t sb, int64_t sh, int64_t ss, int blk,
                 const int32_t* cu, cudaStream_t stream) {
  const dim3 grid((S + blk - 1) / blk, H, B);
  predict_stats_kernel<T, DP, kSeq><<<grid, kStatsThreads, 0, stream>>>(reinterpret_cast<const T*>(x), mean, sim, S, D, blk, sb, sh,
                                                                        ss, cu);
  SAB_CUDA_OK(cudaGetLastError());
  return SAB_OK;
}

// The statistics entries' checks and launch.  Packed form (cu != nullptr): B = nseq, S = max_seqlen, no batch stride.
static int block_stats(const void* x, int dtype, float* mean, float* sim, int B, int H, int S, int D, int64_t stride_b,
                       int64_t stride_h, int64_t stride_s, int blk, const int32_t* cu, void* stream) {
  SAB_REQUIRE(x && mean && sim, SAB_ERR_INVALID, "null tensor pointer");
  SAB_REQUIRE(dtype == SAB_DTYPE_FP16 || dtype == SAB_DTYPE_BF16, SAB_ERR_UNSUPPORTED, "Only half and bfloat16 are supported");
  SAB_REQUIRE(D > 0 && D <= 128 && D % 8 == 0, SAB_ERR_UNSUPPORTED, "Unsupported head dim: %d (a multiple of 8, at most 128)", D);
  SAB_REQUIRE(B > 0 && H > 0 && S > 0, SAB_ERR_INVALID, "bad sizes B=%d H=%d S=%d", B, H, S);
  SAB_REQUIRE(stride_b >= 0 && stride_h >= 0 && stride_s >= 0, SAB_ERR_INVALID, "strides must be >= 0");
  SAB_REQUIRE(aligned16(x) && stride_b % 8 == 0 && stride_h % 8 == 0 && stride_s % 8 == 0, SAB_ERR_INVALID,
              "input must be 16-byte aligned with strides multiple of 8 elements");
  SAB_REQUIRE(blk == 64 || blk == 128, SAB_ERR_INVALID, "block size must be 64 or 128, got %d", blk);
  if (int st = sab_check_device()) return st;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const bool bf = dtype == SAB_DTYPE_BF16;
  if (cu != nullptr) {
    if (D <= 64)
      return bf ? launch_stats<__nv_bfloat16, 64, true>(x, mean, sim, B, H, S, D, 0, stride_h, stride_s, blk, cu, s)
                : launch_stats<__half, 64, true>(x, mean, sim, B, H, S, D, 0, stride_h, stride_s, blk, cu, s);
    return bf ? launch_stats<__nv_bfloat16, 128, true>(x, mean, sim, B, H, S, D, 0, stride_h, stride_s, blk, cu, s)
              : launch_stats<__half, 128, true>(x, mean, sim, B, H, S, D, 0, stride_h, stride_s, blk, cu, s);
  }
  if (D <= 64)
    return bf ? launch_stats<__nv_bfloat16, 64>(x, mean, sim, B, H, S, D, stride_b, stride_h, stride_s, blk, nullptr, s)
              : launch_stats<__half, 64>(x, mean, sim, B, H, S, D, stride_b, stride_h, stride_s, blk, nullptr, s);
  return bf ? launch_stats<__nv_bfloat16, 128>(x, mean, sim, B, H, S, D, stride_b, stride_h, stride_s, blk, nullptr, s)
            : launch_stats<__half, 128>(x, mean, sim, B, H, S, D, stride_b, stride_h, stride_s, blk, nullptr, s);
}

// The selection entries' checks and launch.  Packed form (cu_q != nullptr): B = nseq, Sq / Skv = max_seqlen_q / max_seqlen_k, and
// causal needs no Sq == Skv (top-left inside each sequence).
static int predict_mask(const float* q_mean, const float* q_sim, const float* k_mean, const float* k_sim, uint8_t* block_mask, int B,
                        int Hq, int Hkv, int Sq, int Skv, int D, int is_causal, float sm_scale, float cdf_threshold,
                        float sim_threshold, const int32_t* cu_q, const int32_t* cu_k, void* stream) {
  SAB_REQUIRE(q_mean && q_sim && k_mean && k_sim && block_mask, SAB_ERR_INVALID, "null tensor pointer");
  SAB_REQUIRE(D > 0 && D <= 128 && D % 8 == 0, SAB_ERR_UNSUPPORTED, "Unsupported head dim: %d (a multiple of 8, at most 128)", D);
  SAB_REQUIRE(B > 0 && Hq > 0 && Hkv > 0 && Sq > 0 && Skv > 0, SAB_ERR_INVALID, "bad sizes B=%d Hq=%d Hkv=%d Sq=%d Skv=%d", B, Hq,
              Hkv, Sq, Skv);
  SAB_REQUIRE(Hq % Hkv == 0, SAB_ERR_INVALID, "num_qo_heads (%d) must be divisible by num_kv_heads (%d)", Hq, Hkv);
  SAB_REQUIRE(Skv <= 64 * kMaxKeyBlocks, SAB_ERR_UNSUPPORTED, "block mask prediction supports kv_len <= %d, got %d",
              64 * kMaxKeyBlocks, Skv);
  SAB_REQUIRE(!is_causal || Sq == Skv || cu_q != nullptr, SAB_ERR_INVALID,
              "qo_len (%d) and kv_len (%d) must be equal for causal attention", Sq, Skv);
  SAB_REQUIRE(cdf_threshold > 0.f, SAB_ERR_INVALID, "cdf_threshold must be > 0, got %g", double(cdf_threshold));
  SAB_REQUIRE(!std::isnan(sim_threshold), SAB_ERR_INVALID, "sim_threshold must not be NaN");
  SAB_REQUIRE(std::isfinite(sm_scale), SAB_ERR_INVALID, "sm_scale must be finite, got %g", double(sm_scale));
  if (int st = sab_check_device()) return st;
  SelectParams p{};
  p.qm = q_mean; p.qs = q_sim; p.km = k_mean; p.ks = k_sim; p.mask = block_mask;
  p.Hq = Hq; p.Hkv = Hkv; p.nq = (Sq + 127) / 128; p.nk = (Skv + 63) / 64; p.D = D;
  p.causal = is_causal ? 1 : 0;
  p.scale_log2 = sm_scale * 1.44269504088896340736f;
  p.cdf = cdf_threshold; p.sim = sim_threshold;
  p.cu_q = cu_q; p.cu_k = cu_k;
  p.npow = 1;
  while (p.npow < p.nk) p.npow <<= 1;
  const size_t fixed = size_t(p.npow) * 8 + size_t(kSelChunk) * (D + 1) * 4;
  const size_t per_row = size_t(D) * 4 + size_t(p.nk) * 4;
  p.rows = int(std::min<size_t>(kSelMaxRows, (kSelSmemMax - fixed) / per_row));
  p.rows = std::max(1, std::min(p.rows, p.nq));
  const size_t smem = fixed + per_row * p.rows;
  static bool configured[64] = {}, configured_seq[64] = {};
  auto kern = cu_q != nullptr ? predict_select_kernel<true> : predict_select_kernel<false>;
  if (int st = ensure_dynamic_smem(kern, kSelSmemMax, cu_q != nullptr ? configured_seq : configured)) return st;
  const dim3 grid((p.nq + p.rows - 1) / p.rows, Hq, B);
  kern<<<grid, kSelThreads, smem, reinterpret_cast<cudaStream_t>(stream)>>>(p);
  SAB_CUDA_OK(cudaGetLastError());
  return SAB_OK;
}

}  // namespace sab

extern "C" int sab_block_stats(const void* x, int dtype, float* mean, float* sim, int B, int H, int S, int D, int64_t stride_b,
                               int64_t stride_h, int64_t stride_s, int blk, void* stream) {
  return sab::block_stats(x, dtype, mean, sim, B, H, S, D, stride_b, stride_h, stride_s, blk, nullptr, stream);
}

extern "C" int sab_predict_block_mask(const float* q_mean, const float* q_sim, const float* k_mean, const float* k_sim,
                                      uint8_t* block_mask, int B, int Hq, int Hkv, int Sq, int Skv, int D, int is_causal,
                                      float sm_scale, float cdf_threshold, float sim_threshold, void* stream) {
  return sab::predict_mask(q_mean, q_sim, k_mean, k_sim, block_mask, B, Hq, Hkv, Sq, Skv, D, is_causal, sm_scale, cdf_threshold,
                           sim_threshold, nullptr, nullptr, stream);
}

extern "C" int sab_block_stats_varlen(const void* x, int dtype, float* mean, float* sim, const int32_t* cu_seqlens, int nseq,
                                      int max_seqlen, int H, int D, int64_t stride_t, int64_t stride_h, int blk, void* stream) {
  SAB_REQUIRE(cu_seqlens != nullptr, SAB_ERR_INVALID, "the packed statistics need cu_seqlens");
  return sab::block_stats(x, dtype, mean, sim, nseq, H, max_seqlen, D, 0, stride_h, stride_t, blk, cu_seqlens, stream);
}

extern "C" int sab_predict_block_mask_varlen(const float* q_mean, const float* q_sim, const float* k_mean, const float* k_sim,
                                             uint8_t* block_mask, const int32_t* cu_seqlens_q, const int32_t* cu_seqlens_k, int nseq,
                                             int Hq, int Hkv, int max_seqlen_q, int max_seqlen_k, int D, int is_causal,
                                             float sm_scale, float cdf_threshold, float sim_threshold, void* stream) {
  SAB_REQUIRE(cu_seqlens_q != nullptr && cu_seqlens_k != nullptr, SAB_ERR_INVALID,
              "the packed prediction needs cu_seqlens_q and cu_seqlens_k");
  return sab::predict_mask(q_mean, q_sim, k_mean, k_sim, block_mask, nseq, Hq, Hkv, max_seqlen_q, max_seqlen_k, D, is_causal, sm_scale,
                           cdf_threshold, sim_threshold, cu_seqlens_q, cu_seqlens_k, stream);
}
