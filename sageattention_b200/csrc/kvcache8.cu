// 8-bit paged KV cache for decoding on sm_90a (H100): the write kernel that quantises each token once, per (token, head), into
// INT8 K / e4m3 V pages, and split-KV attention that reads those pages directly.
//   kv8_write_kernel   one warp per (token, head): K - k_smooth -> INT8 with an fp32 scale, V -> e4m3 with an fp32 scale.
//   kv8_attn_kernel    one CTA per (sequence, KV head, chunk of kChunk keys) holding every query row of that KV head (GQA head
//                      packing, <= 64 rows): Q quantised in the prologue, 64-key tiles loaded through the block table with 16-byte
//                      cp.async (double-buffered), QK^T on mma.sync s8, an exact running max, P = bf16(p * v_scale) times
//                      bf16(v8) on mma.sync bf16 with fp32 accumulators.  Writes the chunk's unnormalised O, max and sum.
//   kv8_combine_kernel one CTA per (query row, Q head): folds the row's chunks in ascending order, O / L and the natural-log lse.
// Decode is bound by the bytes of the cache, so the kernels aim at one read of each K / V byte per chunk, not at tensor-core rate.
//   kv8_prefill_kernel one CTA per (sequence, 128-row Q tile, Q head) for query chunks of any length (chunked prefill): the decode
//                      numerics without chunks, on the warpgroup tensor cores (see its section below).
#include <algorithm>
#include <atomic>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include "common.cuh"
#include "ptx.cuh"
#include "quant_common.cuh"

#ifndef SAB_KV8_CHUNK
#define SAB_KV8_CHUNK 1024
#endif

namespace sab {
namespace {

constexpr int kChunk = SAB_KV8_CHUNK;   // keys per split-KV chunk: a multiple of 64, fixed so a row's bits depend on its own keys
static_assert(kChunk % 64 == 0, "the chunk is a whole number of 64-key tiles");
constexpr int kRows = 64;               // query rows per CTA: max_seqlen_q * Hq / Hkv
constexpr int kTile = 64;               // keys per tile
constexpr int kThreads = 128;
constexpr float kLog2e = 1.4426950408889634f;

// Per-row quantisation to [-qmax, qmax]: scale = amax / qmax, x * RN(qmax / amax) rounded by the caller's instruction.  amax == 0
// gives scale 0 and zeros; a denormal amax, whose RN(qmax / amax) overflows, takes the IEEE quotient x / scale instead.
struct RowQuant {
  float scale, mult;
  bool exact;
  __device__ __forceinline__ RowQuant(float amax, float qmax) {
    scale = amax > 0.f ? __fdiv_rn(amax, qmax) : 0.f;
    mult = amax > 0.f ? __fdiv_rn(qmax, amax) : 0.f;
    exact = !(mult <= 3.402823466e+38f);
  }
  __device__ __forceinline__ float operator()(float x) const { return exact ? __fdiv_rn(x, scale) : __fmul_rn(x, mult); }
};

template <typename T, int E>
__device__ __forceinline__ void load_row(const T* p, float (&f)[E]) {
  static_assert(E == 2 || E == 4, "2 or 4 elements per lane");
  if constexpr (E == 4) {
    const uint2 raw = *reinterpret_cast<const uint2*>(p);
    const T* e = reinterpret_cast<const T*>(&raw);
#pragma unroll
    for (int i = 0; i < 4; ++i) f[i] = to_f<T>(e[i]);
  } else {
    const uint32_t raw = *reinterpret_cast<const uint32_t*>(p);
    const T* e = reinterpret_cast<const T*>(&raw);
    f[0] = to_f<T>(e[0]);
    f[1] = to_f<T>(e[1]);
  }
}

template <int E>
__device__ __forceinline__ float warp_amax(const float (&x)[E]) {
  float a = 0.f;
#pragma unroll
  for (int i = 0; i < E; ++i) a = fmaxf(a, fabsf(x[i]));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) a = fmaxf(a, __shfl_xor_sync(0xffffffffu, a, o));
  return a;
}

template <int E>
__device__ __forceinline__ uint32_t pack_s8(const float (&x)[E], const RowQuant& rq) {
  uint32_t r = 0;
#pragma unroll
  for (int i = 0; i < E; ++i) r |= uint32_t(uint8_t(cvt_rni_sat_s8(rq(x[i])))) << (8 * i);
  return r;
}

// ------------------------------------------------------------------------------------------------ write
template <typename T, int D>
__global__ void __launch_bounds__(256) kv8_write_kernel(const T* __restrict__ k, const T* __restrict__ v,
                                                        const float* __restrict__ k_smooth, const int64_t* __restrict__ slot_mapping,
                                                        int T_, int Hkv, int64_t kst, int64_t ksh, int64_t vst, int64_t vsh,
                                                        int8_t* __restrict__ k_pages, float* __restrict__ k_scale,
                                                        uint8_t* __restrict__ v_pages, float* __restrict__ v_scale, int64_t num_slots) {
  constexpr int E = D / 32;
  const int lane = threadIdx.x % 32;
  const int64_t item = int64_t(blockIdx.x) * 8 + threadIdx.x / 32;
  if (item >= int64_t(T_) * Hkv) return;
  const int t = int(item / Hkv), h = int(item % Hkv);
  const int64_t slot = slot_mapping[t];
  if (slot < 0 || slot >= num_slots) return;
  const int64_t row = slot * Hkv + h;   // [num_slots, Hkv] rows of the cache
  float x[E];
  load_row<T, E>(k + int64_t(t) * kst + int64_t(h) * ksh + lane * E, x);
#pragma unroll
  for (int i = 0; i < E; ++i) x[i] = __fsub_rn(x[i], k_smooth[h * D + lane * E + i]);
  const RowQuant kq(warp_amax<E>(x), 127.f);
  const uint32_t k8 = pack_s8<E>(x, kq);
  load_row<T, E>(v + int64_t(t) * vst + int64_t(h) * vsh + lane * E, x);
  const RowQuant vq(warp_amax<E>(x), 448.f);
  uint32_t v8;
  if constexpr (E == 4) v8 = pack_e4m3x4_q(vq(x[0]), vq(x[1]), vq(x[2]), vq(x[3]));
  else v8 = pack_e4m3x4_q(vq(x[0]), vq(x[1]), 0.f, 0.f);
  if constexpr (E == 4) {
    reinterpret_cast<uint32_t*>(k_pages + row * D)[lane] = k8;
    reinterpret_cast<uint32_t*>(v_pages + row * D)[lane] = v8;
  } else {
    reinterpret_cast<uint16_t*>(k_pages + row * D)[lane] = uint16_t(k8);
    reinterpret_cast<uint16_t*>(v_pages + row * D)[lane] = uint16_t(v8);
  }
  if (lane == 0) {
    k_scale[row] = kq.scale;
    v_scale[row] = vq.scale;
  }
}

// ------------------------------------------------------------------------------------------------ attention
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool valid) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(valid ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async4(uint32_t dst, const void* src, bool valid) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(dst), "l"(src), "r"(valid ? 4 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
// D[16 x 8] += A[16 x 32 s8] * B[32 x 8 s8], int32
__device__ __forceinline__ void mma_s8(int (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.s8.s8.s32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// D[16 x 8] += A[16 x 16 bf16] * B[16 x 8 bf16], fp32
__device__ __forceinline__ void mma_bf16(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// two e4m3 bytes (lo, hi) -> bf16x2, exactly (every e4m3 value is an f16 and a bf16)
__device__ __forceinline__ uint32_t e4m3x2_to_bf16x2(uint32_t lo, uint32_t hi) {
  const uint16_t pair = uint16_t(lo | (hi << 8));
  uint32_t h2;
  asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(h2) : "h"(pair));
  const __half2 hv = *reinterpret_cast<const __half2*>(&h2);
  const __nv_bfloat162 b = __floats2bfloat162_rn(__low2float(hv), __high2float(hv));
  return *reinterpret_cast<const uint32_t*>(&b);
}

struct Kv8Params {
  const void* q; const int8_t* k_pages; const float* k_scale; const uint8_t* v_pages; const float* v_scale;
  const int32_t* cu_q; const int32_t* seqused_k; const int32_t* table; int64_t table_stride;
  int max_pages, page_size, Hq, Hkv, max_chunks, max_seqlen_q;
  int64_t q_st, q_sh;
  float scale_log2;     // sm_scale * log2(e)
  float* o_part;        // [Tq, Hq, max_chunks, D]
  float2* ml_part;      // [Tq, Hq, max_chunks]: (running max in log2 units, sum of p)
  int window_left, window_right;   // kWindow: query i sees keys [i + off - left, i + off + right], off = Lk - Lq_b (-1: unbounded)
  int nseq, shared_chunks, shared_seqs;   // kShared: chunks c < shared_chunks are shared; shared_seqs sequences per shared CTA
};

// kShared: chunk c of sequence b goes to a shared CTA iff every held row of b sees every key of the chunk (so no row has a masked
// key in it): b has a query, and the chunk ends at or before Lk_b (non-causal) or the first row's diagonal key + 1 (causal).
template <bool kCausal>
__device__ __forceinline__ bool kv8_takes_shared(int Lqb, int Lk, int c) {
  return Lqb >= 1 && int64_t(c + 1) * kChunk <= (kCausal ? int64_t(Lk) - Lqb + 1 : int64_t(Lk));
}

template <int D>
struct Kv8Smem {
  static constexpr int kRowB = D + 16;                   // int8 / e4m3 row pitch in bytes: conflict-free ldmatrix and byte reads
  static constexpr int kPB = kTile * 2 + 16;             // bf16 P row pitch in bytes
  alignas(128) int8_t q8[kRows * kRowB];
  alignas(128) int8_t k8[2][kTile * kRowB];
  alignas(128) uint8_t v8[2][kTile * kRowB];
  alignas(128) uint8_t p[kRows * kPB];
  float ks[2][kTile], vs[2][kTile];
  float qc[kRows];                                       // q_scale * sm_scale * log2(e)
  float red_max[4][kRows], red_sum[4][kRows];            // per-warp partial row max / sum of the tile
};

// kWindow: the sliding-window form.  The causal rule arrives folded into window_right (0), so kCausal is false.  Tiles left of the
// CTA's first visible key are skipped (a tile in which a row sees nothing is an exact identity on its m, l and O), and keys left of
// it are zero-filled without reading their table entry.  Three CTAs per SM (168 registers, no spill) as the D = 128 forms; the
// D = 64 forms' 128 registers would spill here.  The minimum of 0 leaves the other forms as they were.
//
// kShared: the shared-prefix form.  Grid x is nseq * max_chunks per-sequence CTAs, then ceil(nseq / shared_seqs) * shared_chunks
// shared CTAs.  A per-sequence CTA runs as above, and exits at once when kv8_takes_shared gives its chunk to a shared CTA.  Shared
// CTA (slice s, chunk c) holds the rows of sequences s * shared_seqs + m, member m's at rows m * G * max_seqlen_q + i * G + g, and
// reads chunk c once, through table row 0, for all of them.  Every row it writes runs the per-row arithmetic above on the same
// keys, unmasked as in its own sequence's CTA, so it writes the partial that CTA would have written.  The token of each query slot
// r / G (-1: the row is not computed here) lives in shared memory past Kv8Smem.
template <typename T, int D, bool kCausal, bool kWindow = false, bool kShared = false>
__global__ void __launch_bounds__(kThreads, kWindow ? 3 : 0) kv8_attn_kernel(const Kv8Params p) {
  using S = Kv8Smem<D>;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  S& sm = *reinterpret_cast<S*>(smem_raw);
  int* const slot_tok = reinterpret_cast<int*>(smem_raw + sizeof(S));   // kShared: [kRows]
  const int nper = p.nseq * p.max_chunks;                                 // kShared: the per-sequence CTAs
  const bool shared_cta = kShared && int(blockIdx.x) >= nper;
  const int slice = shared_cta ? (int(blockIdx.x) - nper) / p.shared_chunks : 0;
  const int b = shared_cta ? 0 : blockIdx.x / p.max_chunks, h = blockIdx.y;   // a shared CTA reads table row 0
  const int chunk = shared_cta ? (int(blockIdx.x) - nper) % p.shared_chunks : blockIdx.x % p.max_chunks;
  const int G = p.Hq / p.Hkv;
  const int q0 = p.cu_q[b];
  const int Lqb = p.cu_q[b + 1] - q0;   // the sequence's queries: the causal and window offsets are taken from it
  const int Lq = min(Lqb, p.max_seqlen_q);   // the rows held and written
  const int Lk = min(p.seqused_k[b], p.max_pages * p.page_size);
  const int off = Lk - Lqb;             // query i's diagonal key is i + off
  const int kbeg = chunk * kChunk;
  if constexpr (kShared) {
    if (!shared_cta && chunk < p.shared_chunks && kv8_takes_shared<kCausal>(Lqb, Lk, chunk)) return;
  }
  if (!shared_cta && (Lq <= 0 || kbeg >= Lk)) return;
  const int kend = shared_cta ? kbeg + kChunk : min(Lk, kbeg + kChunk);
  // rows r = i * G + g: query i, Q head h * G + g (shared CTA: query slot i of its members, max_seqlen_q per member)
  const int R = shared_cta ? min(p.shared_seqs, p.nseq - slice * p.shared_seqs) * p.max_seqlen_q * G : Lq * G;
  if constexpr (kShared) {
    bool live = false;
    if (threadIdx.x < kRows) {
      const int u = threadIdx.x;
      int tok = -1;
      if (!shared_cta) {
        if (u < Lq) tok = q0 + u;
      } else if (u * G < R) {
        const int bm = slice * p.shared_seqs + u / p.max_seqlen_q, i = u % p.max_seqlen_q;
        const int qm = p.cu_q[bm], Lqm = p.cu_q[bm + 1] - qm;
        if (i < min(Lqm, p.max_seqlen_q) && kv8_takes_shared<kCausal>(Lqm, min(p.seqused_k[bm], p.max_pages * p.page_size), chunk))
          tok = qm + i;
      }
      slot_tok[u] = tok;
      live = tok >= 0;
    }
    if (!__syncthreads_or(live)) return;   // a shared CTA none of whose members takes the chunk
  }
  const int nM = (R + 15) / 16;
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32, g8 = lane / 4, c4 = lane % 4;
  const int32_t* table = p.table + int64_t(b) * p.table_stride;
  const int64_t hD = int64_t(h) * D;
  // keys [klo, kend) hold every key a row of the CTA sees: klo is row 0's first key (the lower bounds rise with the row), and no
  // row sees a key at or past Lk.  Keys of [klo, kend) that no row sees (past the last held row's upper bound) are masked.  The
  // tiles visited start at kb, the 64-key tile (of the grid from key 0) holding klo.
  int klo = kbeg, kb = kbeg;
  if constexpr (kWindow) {
    if (p.window_left >= 0) klo = int(max(int64_t(kbeg), int64_t(off) - p.window_left));
    if (klo >= kend) {
      // nothing to read: the empty partials (m = -inf, l = 0, O = 0) the combine folds with weight 0
      for (int e = threadIdx.x; e < R * D; e += kThreads) {
        const int r = e / D;
        p.o_part[((int64_t(q0 + r / G) * p.Hq + h * G + r % G) * p.max_chunks + chunk) * D + e % D] = 0.f;
      }
      for (int r = threadIdx.x; r < R; r += kThreads)
        p.ml_part[(int64_t(q0 + r / G) * p.Hq + h * G + r % G) * p.max_chunks + chunk] = make_float2(-INFINITY, 0.f);
      return;
    }
    kb = klo - (klo - kbeg) % kTile;
  }

  // ---- tile loader: keys kb + 64 t .. of this KV head, zero-filled outside [klo, kend); only the first tile (first) holds keys
  // below klo
  auto load_tile = [&](int t, int buf, bool first) {
    constexpr int CPR = D / 16;   // 16-byte chunks per row
    for (int i = threadIdx.x; i < kTile * CPR; i += kThreads) {
      const int r = i / CPR, cc = i % CPR;
      const int key = kb + t * kTile + r;
      const bool ok = key < kend && (!kWindow || !first || key >= klo);
      const int64_t slot = ok ? int64_t(__ldg(table + key / p.page_size)) * p.page_size + key % p.page_size : 0;
      const int64_t off = (slot * p.Hkv) * D + hD + cc * 16;
      cp_async16(smem_u32(&sm.k8[buf][r * S::kRowB + cc * 16]), p.k_pages + off, ok);
      cp_async16(smem_u32(&sm.v8[buf][r * S::kRowB + cc * 16]), p.v_pages + off, ok);
    }
    if (threadIdx.x < kTile) {
      const int key = kb + t * kTile + threadIdx.x;
      const bool ok = key < kend && (!kWindow || !first || key >= klo);
      const int64_t slot = ok ? int64_t(__ldg(table + key / p.page_size)) * p.page_size + key % p.page_size : 0;
      cp_async4(smem_u32(&sm.ks[buf][threadIdx.x]), p.k_scale + slot * p.Hkv + h, ok);
      cp_async4(smem_u32(&sm.vs[buf][threadIdx.x]), p.v_scale + slot * p.Hkv + h, ok);
    }
  };
  const int ntiles = (kend - kb + kTile - 1) / kTile;
  load_tile(0, 0, true);
  cp_async_commit();

  // ---- Q prologue: per (token, head) INT8, one warp per row
  {
    constexpr int E = D / 32;
    const T* q = reinterpret_cast<const T*>(p.q);
    for (int r = warp; r < nM * 16; r += 4) {
      uint32_t q8 = 0;
      float qc = 0.f;
      if (kShared ? slot_tok[r / G] >= 0 : r < R) {
        const int i = r / G, hq = h * G + r % G;
        float x[E];
        load_row<T, E>(q + int64_t(kShared ? slot_tok[i] : q0 + i) * p.q_st + int64_t(hq) * p.q_sh + lane * E, x);
        const RowQuant rq(warp_amax<E>(x), 127.f);
        q8 = pack_s8<E>(x, rq);
        qc = __fmul_rn(rq.scale, p.scale_log2);
      }
      if constexpr (E == 4) *reinterpret_cast<uint32_t*>(&sm.q8[r * S::kRowB + lane * 4]) = q8;
      else *reinterpret_cast<uint16_t*>(&sm.q8[r * S::kRowB + lane * 2]) = uint16_t(q8);
      if (lane == 0) sm.qc[r] = qc;
    }
  }

  // per thread: rows 16 mt + g8 (+8); QK keys 16 warp + 8 nt + 2 c4 (+1); PV columns (D / 4) warp + 8 nt + 2 c4 (+1)
  constexpr int NO = D / 32;            // PV n-tiles per warp
  float o[4][NO][4];
  float m_run[4][2], l_run[4][2];
#pragma unroll
  for (int mt = 0; mt < 4; ++mt) {
#pragma unroll
    for (int j = 0; j < 2; ++j) { m_run[mt][j] = -INFINITY; l_run[mt][j] = 0.f; }
#pragma unroll
    for (int nt = 0; nt < NO; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) o[mt][nt][e] = 0.f;
  }
  // the last key row r may see: causal is bottom-right inside the sequence.  kWindow, in one register per row as lim: row r sees
  // key < kend iff unsigned(key - lo) <= span, with lo = i + off - left and span = left + right.  A side past what the sequence
  // can reach (left > Lk, right > Lq_b: rows are i < Lq_b) sees as much as -1 and is clamped to it, so 0 <= wl <= Lk and
  // 0 <= wr <= Lq_b.  For every key in [0, kend) and row i < Lq_b, key - lo = key - i + Lq_b - Lk + wl then lies in
  // [wl - Lk + 1, Lq_b + wl - 1]: a key left of lo maps to an unsigned value of at least 2^32 + wl - Lk + 1, above
  // span <= wl + Lq_b because Lk + Lq_b < 2^32, so the unsigned test is exact.  Rows r >= R take lo = kend and see nothing.
  int lim[4][2];
  const int wl = p.window_left < 0 || p.window_left > Lk ? Lk : p.window_left;
  const int wr = p.window_right < 0 || p.window_right > Lqb ? Lqb : p.window_right;
  const unsigned span = unsigned(wl) + unsigned(wr);
#pragma unroll
  for (int mt = 0; mt < 4; ++mt)
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int r = mt * 16 + g8 + 8 * j;
      if constexpr (kWindow) lim[mt][j] = r >= R ? kend : r / G + off - wl;
      else if constexpr (kShared) lim[mt][j] = slot_tok[r / G] < 0 ? -1 : (kCausal && !shared_cta ? min(kend - 1, r / G + off) : kend - 1);
      else lim[mt][j] = r >= R ? -1 : (kCausal ? min(kend - 1, r / G + off) : kend - 1);
    }

  for (int t = 0; t < ntiles; ++t) {
    const int buf = t & 1;
    // Tile t is the only group in flight.  Past the barrier it is visible to every warp, and every warp has finished the P V of
    // tile t - 1, the last reader of buffer buf ^ 1, so only now may the loads of tile t + 1 overwrite that buffer.
    cp_async_wait<0>();
    __syncthreads();
    if (t + 1 < ntiles) load_tile(t + 1, buf ^ 1, false);
    cp_async_commit();

    // ---- S = Q K^T for this warp's 16 keys, in log2 units
    const int key0 = kb + t * kTile + warp * 16;
    float s[4][2][4];
    {
      int acc[4][2][4];
#pragma unroll
      for (int mt = 0; mt < 4; ++mt)
#pragma unroll
        for (int nt = 0; nt < 2; ++nt)
#pragma unroll
          for (int e = 0; e < 4; ++e) acc[mt][nt][e] = 0;
#pragma unroll
      for (int ks = 0; ks < D / 32; ++ks) {
        uint32_t bk[4];
        ldsm_x4(smem_u32(&sm.k8[buf][(warp * 16 + (lane / 16) * 8 + lane % 8) * S::kRowB + ks * 32 + ((lane / 8) & 1) * 16]), bk);
#pragma unroll
        for (int mt = 0; mt < 4; ++mt) {
          if (mt < nM) {
            uint32_t a[4];
            ldsm_x4(smem_u32(&sm.q8[(mt * 16 + lane % 8 + ((lane / 8) & 1) * 8) * S::kRowB + ks * 32 + (lane / 16) * 16]), a);
            mma_s8(acc[mt][0], a, bk[0], bk[1]);
            mma_s8(acc[mt][1], a, bk[2], bk[3]);
          }
        }
      }
#pragma unroll
      for (int mt = 0; mt < 4; ++mt) {
        float rmax[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const float qc = sm.qc[mt * 16 + g8 + 8 * j];
#pragma unroll
          for (int nt = 0; nt < 2; ++nt)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int kl = warp * 16 + nt * 8 + 2 * c4 + e;
              float x = __fmul_rn(__fmul_rn(float(acc[mt][nt][2 * j + e]), qc), sm.ks[buf][kl]);
              const int key = key0 + nt * 8 + 2 * c4 + e;
              if (kWindow ? key >= kend || unsigned(key - lim[mt][j]) > span : key > lim[mt][j]) x = -INFINITY;
              s[mt][nt][2 * j + e] = x;
              rmax[j] = fmaxf(rmax[j], x);
            }
        }
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          rmax[j] = fmaxf(rmax[j], __shfl_xor_sync(0xffffffffu, rmax[j], 1));
          rmax[j] = fmaxf(rmax[j], __shfl_xor_sync(0xffffffffu, rmax[j], 2));
          if (c4 == 0) sm.red_max[warp][mt * 16 + g8 + 8 * j] = rmax[j];
        }
      }
    }
    __syncthreads();

    // ---- exact running max, p = 2^(s - m), P = bf16(p * v_scale) to shared memory, partial row sums
    float alpha[4][2];
#pragma unroll
    for (int mt = 0; mt < 4; ++mt) {
      float rsum[2] = {0.f, 0.f};
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int r = mt * 16 + g8 + 8 * j;
        const float m_new = fmaxf(fmaxf(m_run[mt][j], fmaxf(sm.red_max[0][r], sm.red_max[1][r])),
                                  fmaxf(sm.red_max[2][r], sm.red_max[3][r]));
        alpha[mt][j] = m_run[mt][j] == -INFINITY ? 0.f : ex2_approx(__fsub_rn(m_run[mt][j], m_new));
        m_run[mt][j] = m_new;
#pragma unroll
        for (int nt = 0; nt < 2; ++nt) {
          float pe[2];
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const float x = s[mt][nt][2 * j + e];
            pe[e] = x == -INFINITY ? 0.f : ex2_approx(__fsub_rn(x, m_new));
            rsum[j] += pe[e];
          }
          const int kl = warp * 16 + nt * 8 + 2 * c4;
          const __nv_bfloat162 pv = __floats2bfloat162_rn(__fmul_rn(pe[0], sm.vs[buf][kl]), __fmul_rn(pe[1], sm.vs[buf][kl + 1]));
          if (mt < nM) *reinterpret_cast<__nv_bfloat162*>(&sm.p[r * S::kPB + kl * 2]) = pv;
        }
      }
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        rsum[j] += __shfl_xor_sync(0xffffffffu, rsum[j], 1);
        rsum[j] += __shfl_xor_sync(0xffffffffu, rsum[j], 2);
        if (c4 == 0) sm.red_sum[warp][mt * 16 + g8 + 8 * j] = rsum[j];
      }
    }
    __syncthreads();

    // ---- l = alpha l + sum p;  O = alpha O + P V for this warp's D / 4 columns
#pragma unroll
    for (int mt = 0; mt < 4; ++mt)
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int r = mt * 16 + g8 + 8 * j;
        l_run[mt][j] = __fmaf_rn(alpha[mt][j], l_run[mt][j],
                                 __fadd_rn(__fadd_rn(sm.red_sum[0][r], sm.red_sum[1][r]), __fadd_rn(sm.red_sum[2][r], sm.red_sum[3][r])));
#pragma unroll
        for (int nt = 0; nt < NO; ++nt) {
          o[mt][nt][2 * j] *= alpha[mt][j];
          o[mt][nt][2 * j + 1] *= alpha[mt][j];
        }
      }
    const uint8_t* vt = sm.v8[buf];
#pragma unroll
    for (int kk = 0; kk < kTile / 16; ++kk) {
      uint32_t bv[NO][2];
#pragma unroll
      for (int nt = 0; nt < NO; ++nt) {
        const int col = warp * (D / 4) + nt * 8 + g8;
        const int k0 = kk * 16 + 2 * c4;
        bv[nt][0] = e4m3x2_to_bf16x2(vt[k0 * S::kRowB + col], vt[(k0 + 1) * S::kRowB + col]);
        bv[nt][1] = e4m3x2_to_bf16x2(vt[(k0 + 8) * S::kRowB + col], vt[(k0 + 9) * S::kRowB + col]);
      }
#pragma unroll
      for (int mt = 0; mt < 4; ++mt) {
        if (mt < nM) {
          uint32_t a[4];
          ldsm_x4(smem_u32(&sm.p[(mt * 16 + lane % 8 + ((lane / 8) & 1) * 8) * S::kPB + (kk * 16 + (lane / 16) * 8) * 2]), a);
#pragma unroll
          for (int nt = 0; nt < NO; ++nt) mma_bf16(o[mt][nt], a, bv[nt][0], bv[nt][1]);
        }
      }
    }
  }

  // ---- the chunk's partials of rows r < R
#pragma unroll
  for (int mt = 0; mt < 4; ++mt)
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int r = mt * 16 + g8 + 8 * j;
      if (kShared ? slot_tok[r / G] < 0 : r >= R) continue;
      const int64_t idx = (int64_t(kShared ? slot_tok[r / G] : q0 + r / G) * p.Hq + h * G + r % G) * p.max_chunks + chunk;
#pragma unroll
      for (int nt = 0; nt < NO; ++nt)
        *reinterpret_cast<float2*>(p.o_part + idx * D + warp * (D / 4) + nt * 8 + 2 * c4) = make_float2(o[mt][nt][2 * j], o[mt][nt][2 * j + 1]);
      if (warp == 0 && c4 == 0) p.ml_part[idx] = make_float2(m_run[mt][j], l_run[mt][j]);
    }
}

// ------------------------------------------------------------------------------------------------ combine
struct Kv8CombineParams {
  const void* q; const float* k_smooth; const int32_t* cu_q; const int32_t* seqused_k;
  const float* o_part; const float2* ml_part;
  void* out; float* lse;
  int Tq, Hq, Hkv, max_chunks, max_seqlen_q, max_keys;
  int64_t q_st, q_sh, o_st, o_sh;
  float sm_scale;
};

template <typename T, int D>
__global__ void __launch_bounds__(D) kv8_combine_kernel(const Kv8CombineParams p) {
  const int b = blockIdx.x / p.max_seqlen_q, i = blockIdx.x % p.max_seqlen_q, hq = blockIdx.y, d = threadIdx.x;
  const int q0 = p.cu_q[b];
  if (i >= p.cu_q[b + 1] - q0) return;
  const int t = q0 + i;
  const int nc = (min(p.seqused_k[b], p.max_keys) + kChunk - 1) / kChunk;
  const int64_t base = (int64_t(t) * p.Hq + hq) * p.max_chunks;
  float M = -INFINITY;
  for (int c = 0; c < nc; ++c) M = fmaxf(M, p.ml_part[base + c].x);
  float L = 0.f, acc = 0.f;
  if (M != -INFINITY) {
    for (int c = 0; c < nc; ++c) {
      const float2 ml = p.ml_part[base + c];
      const float w = ml.x == -INFINITY ? 0.f : ex2_approx(__fsub_rn(ml.x, M));
      L = __fmaf_rn(w, ml.y, L);
      acc = __fmaf_rn(w, p.o_part[(base + c) * D + d], acc);
    }
  }
  T* out = reinterpret_cast<T*>(p.out) + int64_t(t) * p.o_st + int64_t(hq) * p.o_sh;
  out[d] = from_f<T>(M == -INFINITY ? 0.f : __fdiv_rn(acc, L));
  if (p.lse == nullptr) return;
  // lse = (M + log2 L) / log2(e) + (q . k_smooth) * sm_scale: the softmax ran on q . (k - k_smooth)
  __shared__ float red[D / 32];
  const T* q = reinterpret_cast<const T*>(p.q) + int64_t(t) * p.q_st + int64_t(hq) * p.q_sh;
  float dot = to_f<T>(q[d]) * p.k_smooth[(hq / (p.Hq / p.Hkv)) * D + d];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
  if (d % 32 == 0) red[d / 32] = dot;
  __syncthreads();
  if (d == 0) {
    float qk = 0.f;
#pragma unroll
    for (int w = 0; w < D / 32; ++w) qk += red[w];
    p.lse[int64_t(hq) * p.Tq + t] = M == -INFINITY ? -INFINITY : (M + log2f(L)) / kLog2e + qk * p.sm_scale;
  }
}

// ------------------------------------------------------------------------------------------------ chunked prefill
// kv8_prefill_kernel: one CTA per (sequence, 128-row Q tile, Q head), three warpgroups.
//   warpgroups 0-1  consumers, 64 query rows each.  Q is quantised per (token, head) into a swizzled s8 tile; per 64-key tile, S =
//                   Q K^T on wgmma m64n64k32 s8, the decode kernel's exact running max, P = bf16(p * v_scale) as the register A
//                   operand of wgmma bf16 against V^T, O in fp32 registers.  A row folds all its keys: no chunks, no combine.
//   warpgroup 2     producer.  16-byte cp.async of each tile's K (int8) and V (e4m3) rows through the block table into a
//                   kPfStages-deep ring, zero-filled past Lk_b (no slot past the sequence is read), with the tile's 64 k / v scales;
//                   kPfLag tiles behind its loads it converts V exactly to bf16 into the swizzled V^T tile the PV wgmma reads, so
//                   the consumers' serial path holds no conversion.
// Every row runs over the same tile grid from key 0, and a tile past a row's horizon adds p = 0 with alpha = 1, so a row's bits do
// not depend on which other rows share its CTA: prefilling a prompt in chunks of any size gives the same bits.
constexpr int kPfRows = 128;       // query rows per CTA
constexpr int kPfStages = 4;       // K / V ring depth (64-key tiles)
constexpr int kPfLag = 2;          // tiles the producer's loads run ahead of its V conversion
constexpr int kPfThreads = 384;

template <int D>
struct PfSmem {
  alignas(1024) int8_t q8[kPfRows * D];              // s8 Q, K-major, swizzled (span D bytes)
  alignas(1024) int8_t k8[kPfStages][kTile * D];     // s8 K rows, K-major, swizzled (span D bytes)
  alignas(1024) uint16_t vt[kPfStages][D * kTile];   // bf16 V^T [D][64 keys], 128-B swizzle
  alignas(16) uint8_t v8[kPfStages][kTile * D];      // e4m3 V rows as loaded
  float ks[kPfStages][kTile], vs[kPfStages][kTile];
  float qc[kPfRows];                                 // q_scale * sm_scale * log2(e)
  float qk[kPfRows];                                 // q . k_smooth (lse only)
  uint64_t full[kPfStages], empty[kPfStages];
};

// 16-byte chunk c of row r of a K-major tile of D-byte rows under the D-byte hardware swizzle (128 B: c ^ r % 8; 64 B: c ^ r / 2 % 4)
template <int D>
__device__ __forceinline__ int pf_swz(int r, int c) { return c ^ ((r * D >> 7) & (D / 16 - 1)); }

struct PfParams {
  const void* q; const int8_t* k_pages; const float* k_scale; const uint8_t* v_pages; const float* v_scale; const float* k_smooth;
  const int32_t* cu_q; const int32_t* seqused_k; const int32_t* table; int64_t table_stride;
  void* out; float* lse;
  int max_pages, page_size, Hq, Hkv, n_qt, max_seqlen_q, Tq;
  int64_t q_st, q_sh, o_st, o_sh;
  float sm_scale, scale_log2;   // scale_log2 = sm_scale * log2(e)
  int window_left, window_right;   // kWindow: as Kv8Params
};

// kWindow: the sliding-window form, the causal rule folded into window_right (0) as in kv8_attn_kernel.  The CTA visits the tiles
// from the one holding its first row's first key; loop index t counts visited tiles, tile tf + t of the grid from key 0.
template <typename T, int D, bool kCausal, bool kWindow = false>
__global__ void __launch_bounds__(kPfThreads, 1) kv8_prefill_kernel(const PfParams p) {
  using S = PfSmem<D>;
  extern __shared__ __align__(1024) unsigned char pf_smem[];
  S& sm = *reinterpret_cast<S*>(pf_smem + ((1024u - (smem_u32(pf_smem) & 1023u)) & 1023u));   // 1 KB-aligned swizzled tiles
  const int b = blockIdx.x / p.n_qt, qt = p.n_qt - 1 - blockIdx.x % p.n_qt, hq = blockIdx.y;   // longest rows first
  const int hk = hq / (p.Hq / p.Hkv);
  const int q0 = p.cu_q[b];
  const int Lqb = p.cu_q[b + 1] - q0;   // the sequence's queries: the causal and window offsets are taken from it
  const int Lq = min(Lqb, p.max_seqlen_q);   // the rows held and written
  const int Lk = max(0, min(p.seqused_k[b], p.max_pages * p.page_size));
  const int off = Lk - Lqb;             // query i's diagonal key is i + off
  const int r0 = qt * kPfRows;          // the CTA's first row inside the sequence
  if (r0 >= Lq) return;
  // keys [klo, kmax) hold every key a row of the CTA sees; tiles past `first_h` (the first row's last key), and kWindow: tiles
  // starting before `lo_last` (the last row's first key), take the masked path
  const int last = min(r0 + kPfRows, Lq) - 1;
  int kmax = kCausal ? max(0, min(Lk, last + off + 1)) : Lk;
  int first_h = kCausal ? min(Lk - 1, r0 + off) : Lk - 1;
  int klo = 0, lo_last = 0, tf = 0;
  if constexpr (kWindow) {
    if (p.window_right >= 0) {
      kmax = int(max(int64_t(0), min(int64_t(Lk), last + int64_t(off) + p.window_right + 1)));
      first_h = int(min(int64_t(Lk - 1), r0 + int64_t(off) + p.window_right));
    }
    if (p.window_left >= 0) {
      klo = int(max(int64_t(0), min(int64_t(Lk), r0 + int64_t(off) - p.window_left)));
      lo_last = int(max(int64_t(0), min(int64_t(Lk), last + int64_t(off) - p.window_left)));
    }
    tf = klo / kTile;
  }
  const int n = kWindow ? max(0, (kmax + kTile - 1) / kTile - tf) : (kmax + kTile - 1) / kTile;
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;

  if (threadIdx.x == 0) {
    for (int i = 0; i < kPfStages; ++i) {
      mbar_init(&sm.full[i], 128);      // every producer thread, after its copies and its part of V^T
      mbar_init(&sm.empty[i], 2);       // one thread per consumer warpgroup, after its P V of the tile
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >= 8) {
    // =============================== producer ===============================
    const int pt = threadIdx.x - 256;
    const int32_t* table = p.table + int64_t(b) * p.table_stride;
    auto slot_of = [&](int key) { return int64_t(__ldg(table + key / p.page_size)) * p.page_size + key % p.page_size; };
    auto load_tile = [&](int t) {
      const int s = t % kPfStages;
      constexpr int CPR = D / 16;       // 16-byte chunks per row; two threads per row
      const int r = pt >> 1, key = (tf + t) * kTile + r;
      const bool ok = kWindow ? key >= klo && key < kmax : key < Lk;
      const int64_t off = ((ok ? slot_of(key) : 0) * p.Hkv + hk) * D;
#pragma unroll
      for (int i = 0; i < CPR / 2; ++i) {
        const int c = (pt & 1) * (CPR / 2) + i;
        cp_async16(smem_u32(&sm.k8[s][r * D + pf_swz<D>(r, c) * 16]), p.k_pages + off + c * 16, ok);
        cp_async16(smem_u32(&sm.v8[s][r * D + c * 16]), p.v_pages + off + c * 16, ok);
      }
      const int sk = (tf + t) * kTile + (pt & (kTile - 1));
      const bool sok = kWindow ? sk >= klo && sk < kmax : sk < Lk;
      const int64_t si = (sok ? slot_of(sk) : 0) * p.Hkv + hk;
      if (pt < kTile) cp_async4(smem_u32(&sm.ks[s][pt]), p.k_scale + si, sok);
      else cp_async4(smem_u32(&sm.vs[s][pt - kTile]), p.v_scale + si, sok);
    };
    // V^T element (d, key) of a tile: 16-byte chunk key / 8 of row d, swizzled.  Item (key octet ko, column quad dg) reads 8 words
    // of V8 and writes 4 chunks; the column order is rotated by dg to spread the stores over the banks.
    auto convert = [&](int t) {
      const int s = t % kPfStages;
      constexpr int NQ = D / 4;
#pragma unroll
      for (int it = 0; it < (8 * NQ) / 128; ++it) {
        const int w = it * 128 + pt, ko = w / NQ, dg = w % NQ;
        uint32_t x[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) x[j] = *reinterpret_cast<const uint32_t*>(&sm.v8[s][(8 * ko + j) * D + 4 * dg]);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int e = (i + dg) & 3, d = 4 * dg + e, sh = 8 * e;
          uint32_t y[4];
#pragma unroll
          for (int j = 0; j < 4; ++j) y[j] = e4m3x2_to_bf16x2((x[2 * j] >> sh) & 0xffu, (x[2 * j + 1] >> sh) & 0xffu);
          st_shared_v4(smem_u32(&sm.vt[s][d * kTile]) + ((ko ^ (d & 7)) * 16), y[0], y[1], y[2], y[3]);
        }
      }
    };
    for (int t = 0; t < n + kPfLag; ++t) {
      if (t < n) {
        mbar_wait(&sm.empty[t % kPfStages], ((t / kPfStages) & 1) ^ 1);
        load_tile(t);
      }
      cp_async_commit();
      const int c = t - kPfLag;
      if (c >= 0) {
        cp_async_wait<kPfLag>();          // this thread's copies of tile c have landed
        named_bar_sync(2, 128);           // ... and every producer thread's
        convert(c);
        fence_proxy_async_smem();         // the cp.async and V^T writes, before the consumers' wgmma reads them
        mbar_arrive(&sm.full[c % kPfStages]);
      }
    }
    return;
  }

  // =============================== consumers ===============================
  // ---- Q prologue: one warp per row, per (token, head) INT8 as the decode kernel's
  {
    constexpr int E = D / 32;
    const T* q = reinterpret_cast<const T*>(p.q);
    for (int r = warp; r < kPfRows; r += 8) {
      uint32_t q8 = 0;
      float qc = 0.f, qk = 0.f;
      if (r0 + r < Lq) {
        const int64_t tok = q0 + r0 + r;
        float x[E];
        load_row<T, E>(q + tok * p.q_st + int64_t(hq) * p.q_sh + lane * E, x);
        const RowQuant rq(warp_amax<E>(x), 127.f);
        q8 = pack_s8<E>(x, rq);
        qc = __fmul_rn(rq.scale, p.scale_log2);
        if (p.lse != nullptr) {
#pragma unroll
          for (int i = 0; i < E; ++i) qk += x[i] * p.k_smooth[hk * D + lane * E + i];
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) qk += __shfl_xor_sync(0xffffffffu, qk, o);
        }
      }
      int8_t* dst = &sm.q8[r * D + pf_swz<D>(r, lane * E / 16) * 16 + (lane * E) % 16];
      if constexpr (E == 4) *reinterpret_cast<uint32_t*>(dst) = q8;
      else *reinterpret_cast<uint16_t*>(dst) = uint16_t(q8);
      if (lane == 0) {
        sm.qc[r] = qc;
        sm.qk[r] = qk;
      }
    }
    fence_proxy_async_smem();
    named_bar_sync(1, 256);
  }

  // wgmma accumulator layout (m64nN): warp w of the warpgroup owns rows 16w..16w+15; lane = 4 g + t4 holds rows 16w+g (registers
  // 4i, 4i+1) and 16w+g+8 (4i+2, 4i+3) at columns 8i+2t4, 8i+2t4+1.  A row is spread over the 4 lanes of a quad.
  const int wg = warp / 4, t4 = lane % 4;
  const int row0 = wg * 64 + (warp % 4) * 16 + lane / 4;   // rows row0 and row0 + 8 of the CTA
  float qcr[2];
  int lim[2], lo[2];                    // the last key each row sees (-1: a row past Lq); kWindow: the first
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int i = r0 + row0 + 8 * r;
    qcr[r] = sm.qc[row0 + 8 * r];
    lim[r] = i >= Lq ? -1 : (kCausal ? min(Lk - 1, i + off) : Lk - 1);
    if constexpr (kWindow) {
      const int64_t diag = int64_t(i) + off;
      if (i < Lq && p.window_right >= 0) lim[r] = int(max(int64_t(-1), min(int64_t(Lk - 1), diag + p.window_right)));
      lo[r] = p.window_left < 0 ? 0 : int(max(int64_t(0), min(int64_t(Lk), diag - p.window_left)));
    }
  }
  constexpr int NO = D / 2;
  float o[NO];
#pragma unroll
  for (int i = 0; i < NO; ++i) o[i] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};   // l: this thread's part of the row sum
  uint32_t acc[32];
  uint32_t a[4][4];                     // P of the tile, as the A operand of four k16 steps
  const uint64_t dQ = make_wgmma_desc<D>(smem_u32(sm.q8 + wg * 64 * D));
  const uint64_t dK0 = make_wgmma_desc<D>(smem_u32(sm.k8[0]));
  const uint64_t dV0 = make_wgmma_desc<128>(smem_u32(sm.vt[0]));
  auto issue_qk = [&](int t) {
    const uint64_t dK = dK0 + uint64_t(t % kPfStages) * ((kTile * D) >> 4);
#pragma unroll
    for (int k = 0; k < D / 32; ++k) wgmma_qk_i8(acc, dQ + 2 * k, dK + 2 * k, k > 0);
  };
  auto issue_pv = [&](int t) {
    const uint64_t dV = dV0 + uint64_t(t % kPfStages) * ((D * kTile * 2) >> 4);
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) wgmma_rs_bf16(o, a[kk], dV + 2 * kk, 1);
  };

  // Each step: S = Q K(t)^T, softmax, O += P V(t), each product waited for before the next (QK(t + 1) queued behind PV(t) makes
  // ptxas serialise every wgmma of the loop).  The two consumer warpgroups overlap each other's softmax and products.  Slot t - 1
  // is released once PV(t - 1) has completed.
  for (int t = 0; t < n; ++t) {
    const int s = t % kPfStages;
    mbar_wait(&sm.full[s], (t / kPfStages) & 1);
    wgmma_fence();
    issue_qk(t);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(acc);
    fence_regs(o);
    if (t > 0 && (threadIdx.x & 127) == 0) mbar_arrive(&sm.empty[(t - 1) % kPfStages]);
    // ---- logits in log2 units, the exact running max, p = 2^(s - m), P = bf16(p * v_scale)
    const int kt = (tf + t) * kTile;    // the tile's first key
    const bool masked = kt + kTile - 1 > first_h || (kWindow && kt < lo_last);
    float2 ksv[8], vsv[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      ksv[i] = *reinterpret_cast<const float2*>(&sm.ks[s][8 * i + 2 * t4]);
      vsv[i] = *reinterpret_cast<const float2*>(&sm.vs[s][8 * i + 2 * t4]);
    }
    float e[32];
    float alpha[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      float x[16];
      float mx = -INFINITY;
#pragma unroll
      for (int c = 0; c < 16; ++c) {
        const int idx = 4 * (c >> 1) + 2 * r + (c & 1);
        const float kscale = (c & 1) ? ksv[c >> 1].y : ksv[c >> 1].x;
        float v = __fmul_rn(__fmul_rn(float(int(acc[idx])), qcr[r]), kscale);
        const int key = kt + 8 * (c >> 1) + 2 * t4 + (c & 1);
        if (masked && (key > lim[r] || (kWindow && key < lo[r]))) v = -INFINITY;
        x[c] = v;
        mx = fmaxf(mx, v);
      }
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m[r], mx);
      alpha[r] = m[r] == -INFINITY ? 0.f : ex2_approx(__fsub_rn(m[r], m_new));
      m[r] = m_new;
      float sum = 0.f;
#pragma unroll
      for (int c = 0; c < 16; ++c) {
        const int idx = 4 * (c >> 1) + 2 * r + (c & 1);
        const float pe = x[c] == -INFINITY ? 0.f : ex2_approx(__fsub_rn(x[c], m_new));
        sum += pe;
        e[idx] = __fmul_rn(pe, (c & 1) ? vsv[c >> 1].y : vsv[c >> 1].x);
      }
      l[r] = __fmaf_rn(alpha[r], l[r], sum);
    }
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const __nv_bfloat162 pv = __floats2bfloat162_rn(e[8 * kk + 2 * j], e[8 * kk + 2 * j + 1]);
        a[kk][j] = *reinterpret_cast<const uint32_t*>(&pv);
      }
#pragma unroll
    for (int i = 0; i < NO; i += 4) {
      o[i] *= alpha[0];
      o[i + 1] *= alpha[0];
      o[i + 2] *= alpha[1];
      o[i + 3] *= alpha[1];
    }
    // ---- O += P V(t)
    fence_regs(o);
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) fence_regs(a[kk]);
    wgmma_fence();
    issue_pv(t);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(o);
  }
  if (n > 0) {
    wgmma_wait<0>();
    fence_regs(o);
  }

  // ---- epilogue: O / l in the output type; lse = (m + log2 l) / log2(e) + (q . k_smooth) * sm_scale
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    float L = l[r];
    L += __shfl_xor_sync(0xffffffffu, L, 1);
    L += __shfl_xor_sync(0xffffffffu, L, 2);
    const int row = row0 + 8 * r, i = r0 + row;
    if (i >= Lq) continue;
    const bool seen = m[r] != -INFINITY;
    T* orow = reinterpret_cast<T*>(p.out) + int64_t(q0 + i) * p.o_st + int64_t(hq) * p.o_sh;
#pragma unroll
    for (int nb = 0; nb < D / 8; ++nb) {
      T pair[2];
      pair[0] = from_f<T>(seen ? __fdiv_rn(o[4 * nb + 2 * r], L) : 0.f);
      pair[1] = from_f<T>(seen ? __fdiv_rn(o[4 * nb + 2 * r + 1], L) : 0.f);
      *reinterpret_cast<uint32_t*>(orow + 8 * nb + 2 * t4) = *reinterpret_cast<const uint32_t*>(pair);
    }
    if (p.lse != nullptr && t4 == 0)
      p.lse[int64_t(hq) * p.Tq + q0 + i] = seen ? (m[r] + log2f(L)) / kLog2e + sm.qk[row] * p.sm_scale : -INFINITY;
  }
}

// ------------------------------------------------------------------------------------------------ host
int check_dtype_dim(int dtype, int D) {
  SAB_REQUIRE(dtype == SAB_DTYPE_FP16 || dtype == SAB_DTYPE_BF16, SAB_ERR_UNSUPPORTED, "Only half and bfloat16 are supported");
  SAB_REQUIRE(D == 64 || D == 128, SAB_ERR_UNSUPPORTED, "Unsupported head dim: %d", D);
  return SAB_OK;
}

template <typename T, int D>
int launch_write(const void* k, const void* v, const float* k_smooth, const int64_t* slots, int T_, int Hkv, int64_t kst, int64_t ksh,
                 int64_t vst, int64_t vsh, int8_t* kp, float* ksc, uint8_t* vp, float* vsc, int64_t num_slots, cudaStream_t st) {
  const int64_t blocks = (int64_t(T_) * Hkv + 7) / 8;
  kv8_write_kernel<T, D><<<dim3(unsigned(blocks)), 256, 0, st>>>(reinterpret_cast<const T*>(k), reinterpret_cast<const T*>(v), k_smooth,
                                                                slots, T_, Hkv, kst, ksh, vst, vsh, kp, ksc, vp, vsc, num_slots);
  SAB_CUDA_OK(cudaGetLastError());
  return SAB_OK;
}

// kShared: the per-sequence CTAs, then ceil(nseq / shared_seqs) slices x shared_chunks shared CTAs
template <typename T, int D, bool kCausal, bool kWindow = false, bool kShared = false>
int launch_attn_t(const Kv8Params& p, int nseq, cudaStream_t st) {
  auto kern = kv8_attn_kernel<T, D, kCausal, kWindow, kShared>;
  const int bytes = int(sizeof(Kv8Smem<D>)) + (kShared ? kRows * int(sizeof(int)) : 0);
  const int64_t grid_x = int64_t(nseq) * p.max_chunks +
                         (kShared ? int64_t(nseq + p.shared_seqs - 1) / p.shared_seqs * p.shared_chunks : 0);
  // once per device, so a launch inside CUDA-graph capture makes no attribute call
  static std::atomic<uint64_t> configured{0};
  int dev = 0;
  SAB_CUDA_OK(cudaGetDevice(&dev));
  const uint64_t bit = uint64_t(1) << (dev & 63);
  if (!(configured.load() & bit)) {
    SAB_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    configured.fetch_or(bit);
  }
  kern<<<dim3(unsigned(grid_x), unsigned(p.Hkv)), kThreads, bytes, st>>>(p);
  SAB_CUDA_OK(cudaGetLastError());
  return SAB_OK;
}

// window: the kWindow kernel, with the causal rule already folded into p.window_right; p.shared_chunks > 0: the kShared kernel
template <typename T, int D>
int launch_attn(const Kv8Params& p, const Kv8CombineParams& c, int nseq, bool causal, bool window, cudaStream_t st) {
  const bool shared = p.shared_chunks > 0;
  if (int r = window ? launch_attn_t<T, D, false, true>(p, nseq, st)
              : shared ? (causal ? launch_attn_t<T, D, true, false, true>(p, nseq, st) : launch_attn_t<T, D, false, false, true>(p, nseq, st))
                       : causal ? launch_attn_t<T, D, true>(p, nseq, st) : launch_attn_t<T, D, false>(p, nseq, st))
    return r;
  kv8_combine_kernel<T, D><<<dim3(unsigned(nseq * c.max_seqlen_q), unsigned(c.Hq)), D, 0, st>>>(c);
  SAB_CUDA_OK(cudaGetLastError());
  return SAB_OK;
}

template <typename T, int D, bool kCausal, bool kWindow = false>
int launch_prefill_t(const PfParams& p, int nseq, cudaStream_t st) {
  auto kern = kv8_prefill_kernel<T, D, kCausal, kWindow>;
  const int bytes = int(sizeof(PfSmem<D>)) + 1024;   // + the alignment of the swizzled tiles
  // once per device, so a launch inside CUDA-graph capture makes no attribute call
  static std::atomic<uint64_t> configured{0};
  int dev = 0;
  SAB_CUDA_OK(cudaGetDevice(&dev));
  const uint64_t bit = uint64_t(1) << (dev & 63);
  if (!(configured.load() & bit)) {
    SAB_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    configured.fetch_or(bit);
  }
  kern<<<dim3(unsigned(int64_t(nseq) * p.n_qt), unsigned(p.Hq)), kPfThreads, bytes, st>>>(p);
  SAB_CUDA_OK(cudaGetLastError());
  return SAB_OK;
}

template <typename T, int D>
int launch_prefill(const PfParams& p, int nseq, bool causal, bool window, cudaStream_t st) {
  if (window) return launch_prefill_t<T, D, false, true>(p, nseq, st);
  return causal ? launch_prefill_t<T, D, true>(p, nseq, st) : launch_prefill_t<T, D, false>(p, nseq, st);
}

// The window rule the kernels take: < -1 is refused; causal makes the right side 0 (j <= i + off whatever right is).
int window_args(int window_left, int window_right, int is_causal, int& right) {
  SAB_REQUIRE(window_left >= -1 && window_right >= -1, SAB_ERR_INVALID, "window_left and window_right must be >= -1 (-1: unbounded)");
  right = is_causal ? 0 : window_right;
  return SAB_OK;
}

}  // namespace
}  // namespace sab

using namespace sab;

extern "C" int sab_kvcache8_chunk_keys(void) { return kChunk; }

extern "C" int64_t sab_kvcache8_workspace_bytes(int Tq, int Hq, int D, int64_t max_keys) {
  const int64_t chunks = (max_keys + kChunk - 1) / kChunk;
  return int64_t(Tq) * Hq * chunks * (int64_t(D) + 2) * 4;
}

extern "C" int sab_kvcache8_write(const void* k, const void* v, int dtype, const float* k_smooth, const int64_t* slot_mapping, int T,
                                  int Hkv, int D, int64_t k_stride_t, int64_t k_stride_h, int64_t v_stride_t, int64_t v_stride_h,
                                  int8_t* k_pages, float* k_scale, uint8_t* v_pages, float* v_scale, int64_t num_pages, int page_size,
                                  void* stream) {
  SAB_REQUIRE(k && v && k_smooth && slot_mapping && k_pages && k_scale && v_pages && v_scale, SAB_ERR_INVALID, "null pointer argument");
  if (int r = check_dtype_dim(dtype, D)) return r;
  SAB_REQUIRE(T >= 0 && Hkv > 0 && num_pages > 0 && page_size > 0 && page_size % 16 == 0, SAB_ERR_INVALID,
              "need T >= 0, Hkv > 0, num_pages > 0 and page_size a positive multiple of 16");
  SAB_REQUIRE(k_stride_t >= 0 && k_stride_h >= 0 && v_stride_t >= 0 && v_stride_h >= 0 && (k_stride_t | k_stride_h | v_stride_t | v_stride_h) % 4 == 0 &&
                  (reinterpret_cast<uintptr_t>(k) | reinterpret_cast<uintptr_t>(v)) % 8 == 0,
              SAB_ERR_INVALID, "k and v need 8-byte aligned rows (non-negative strides, multiples of 4 elements)");
  SAB_REQUIRE(int64_t(T) * Hkv < (int64_t(1) << 33), SAB_ERR_INVALID, "too many tokens in one write");
  if (T == 0) return SAB_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int64_t ns = num_pages * page_size;
  if (dtype == SAB_DTYPE_FP16)
    return D == 128 ? launch_write<__half, 128>(k, v, k_smooth, slot_mapping, T, Hkv, k_stride_t, k_stride_h, v_stride_t, v_stride_h, k_pages, k_scale, v_pages, v_scale, ns, st)
                    : launch_write<__half, 64>(k, v, k_smooth, slot_mapping, T, Hkv, k_stride_t, k_stride_h, v_stride_t, v_stride_h, k_pages, k_scale, v_pages, v_scale, ns, st);
  return D == 128 ? launch_write<__nv_bfloat16, 128>(k, v, k_smooth, slot_mapping, T, Hkv, k_stride_t, k_stride_h, v_stride_t, v_stride_h, k_pages, k_scale, v_pages, v_scale, ns, st)
                  : launch_write<__nv_bfloat16, 64>(k, v, k_smooth, slot_mapping, T, Hkv, k_stride_t, k_stride_h, v_stride_t, v_stride_h, k_pages, k_scale, v_pages, v_scale, ns, st);
}

// sab_kvcache8_attn and, with window, sab_kvcache8_attn_window (window_right with the causal rule folded in); with
// shared_prefix_len >= one chunk, sab_kvcache8_attn_shared
static int kvcache8_attn(const void* q, int dtype, const int8_t* k_pages, const float* k_scale, const uint8_t* v_pages,
                         const float* v_scale, const float* k_smooth, void* out, float* lse, const int32_t* cu_seqlens_q,
                         const int32_t* seqused_k, const int32_t* block_table, int64_t table_stride, int max_pages, int nseq,
                         int Tq, int Hq, int Hkv, int D, int page_size, int64_t q_stride_t, int64_t q_stride_h,
                         int64_t o_stride_t, int64_t o_stride_h, int max_seqlen_q, int is_causal, float sm_scale,
                         void* workspace, bool window, int window_left, int window_right, int shared_prefix_len,
                         void* stream) {
  SAB_REQUIRE(q && k_pages && k_scale && v_pages && v_scale && k_smooth && out && cu_seqlens_q && seqused_k && block_table && workspace,
              SAB_ERR_INVALID, "null pointer argument");
  if (int r = check_dtype_dim(dtype, D)) return r;
  SAB_REQUIRE(Hkv > 0 && Hq > 0 && Hq % Hkv == 0, SAB_ERR_INVALID, "num_qo_heads (%d) must be divisible by num_kv_heads (%d)", Hq, Hkv);
  SAB_REQUIRE(nseq > 0 && Tq > 0 && max_seqlen_q > 0 && max_pages > 0 && page_size > 0 && page_size % 16 == 0 && table_stride >= max_pages,
              SAB_ERR_INVALID, "need nseq, Tq, max_seqlen_q, max_pages > 0, page_size a positive multiple of 16 and table_stride >= max_pages");
  SAB_REQUIRE(int64_t(max_seqlen_q) * (Hq / Hkv) <= kRows, SAB_ERR_INVALID,
              "max_seqlen_q * Hq / Hkv = %lld exceeds %d query rows per KV head", (long long)max_seqlen_q * (Hq / Hkv), kRows);
  SAB_REQUIRE(q_stride_t >= 0 && q_stride_h >= 0 && (q_stride_t | q_stride_h) % 4 == 0 && reinterpret_cast<uintptr_t>(q) % 8 == 0,
              SAB_ERR_INVALID, "q needs 8-byte aligned rows (non-negative strides, multiples of 4 elements)");
  const int64_t max_keys = int64_t(max_pages) * page_size;
  const int64_t chunks = (max_keys + kChunk - 1) / kChunk;
  // grid y is Hkv (attention) and Hq (combine); grid x is nseq * chunks and nseq * max_seqlen_q; key indices are int
  SAB_REQUIRE(Hq <= 65535 && chunks * nseq < (int64_t(1) << 31) && int64_t(nseq) * max_seqlen_q < (int64_t(1) << 31),
              SAB_ERR_INVALID, "launch grid too large: need Hq <= 65535, nseq * chunks < 2^31 and nseq * max_seqlen_q < 2^31");
  SAB_REQUIRE(max_keys < (int64_t(1) << 31), SAB_ERR_INVALID, "max_pages * page_size must be < 2^31 keys");
  // shared prefix: whole chunks only, at most the table's keys; shared_seqs sequences' rows fill one CTA's kRows
  const int64_t shared_chunks = std::min(int64_t(shared_prefix_len), max_keys) / kChunk;
  const int shared_seqs = kRows / (max_seqlen_q * (Hq / Hkv));
  SAB_REQUIRE(chunks * nseq + (nseq + shared_seqs - 1) / shared_seqs * shared_chunks < (int64_t(1) << 31), SAB_ERR_INVALID,
              "launch grid too large: need nseq * chunks + ceil(nseq / shared sequences per CTA) * shared chunks < 2^31");
  Kv8Params p{q, k_pages, k_scale, v_pages, v_scale, cu_seqlens_q, seqused_k, block_table, table_stride, max_pages, page_size, Hq, Hkv,
              int(chunks), max_seqlen_q, q_stride_t, q_stride_h, float(double(sm_scale) * 1.4426950408889634),
              static_cast<float*>(workspace), nullptr, window_left, window_right, nseq, int(shared_chunks), shared_seqs};
  p.ml_part = reinterpret_cast<float2*>(p.o_part + int64_t(Tq) * Hq * chunks * D);
  Kv8CombineParams c{q, k_smooth, cu_seqlens_q, seqused_k, p.o_part, p.ml_part, out, lse, Tq, Hq, Hkv, int(chunks), max_seqlen_q,
                     int(max_keys), q_stride_t, q_stride_h, o_stride_t, o_stride_h, sm_scale};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const bool causal = is_causal != 0;
  if (dtype == SAB_DTYPE_FP16)
    return D == 128 ? launch_attn<__half, 128>(p, c, nseq, causal, window, st) : launch_attn<__half, 64>(p, c, nseq, causal, window, st);
  return D == 128 ? launch_attn<__nv_bfloat16, 128>(p, c, nseq, causal, window, st)
                  : launch_attn<__nv_bfloat16, 64>(p, c, nseq, causal, window, st);
}

extern "C" int sab_kvcache8_attn(const void* q, int dtype, const int8_t* k_pages, const float* k_scale, const uint8_t* v_pages,
                                 const float* v_scale, const float* k_smooth, void* out, float* lse, const int32_t* cu_seqlens_q,
                                 const int32_t* seqused_k, const int32_t* block_table, int64_t table_stride, int max_pages, int nseq,
                                 int Tq, int Hq, int Hkv, int D, int page_size, int64_t q_stride_t, int64_t q_stride_h,
                                 int64_t o_stride_t, int64_t o_stride_h, int max_seqlen_q, int is_causal, float sm_scale,
                                 void* workspace, void* stream) {
  return kvcache8_attn(q, dtype, k_pages, k_scale, v_pages, v_scale, k_smooth, out, lse, cu_seqlens_q, seqused_k, block_table,
                       table_stride, max_pages, nseq, Tq, Hq, Hkv, D, page_size, q_stride_t, q_stride_h, o_stride_t, o_stride_h,
                       max_seqlen_q, is_causal, sm_scale, workspace, false, -1, -1, 0, stream);
}

extern "C" int sab_kvcache8_attn_window(const void* q, int dtype, const int8_t* k_pages, const float* k_scale, const uint8_t* v_pages,
                                        const float* v_scale, const float* k_smooth, void* out, float* lse, const int32_t* cu_seqlens_q,
                                        const int32_t* seqused_k, const int32_t* block_table, int64_t table_stride, int max_pages,
                                        int nseq, int Tq, int Hq, int Hkv, int D, int page_size, int64_t q_stride_t,
                                        int64_t q_stride_h, int64_t o_stride_t, int64_t o_stride_h, int max_seqlen_q, int is_causal,
                                        float sm_scale, void* workspace, int window_left, int window_right, void* stream) {
  int right = -1;
  if (int r = window_args(window_left, window_right, is_causal, right)) return r;
  return kvcache8_attn(q, dtype, k_pages, k_scale, v_pages, v_scale, k_smooth, out, lse, cu_seqlens_q, seqused_k, block_table,
                       table_stride, max_pages, nseq, Tq, Hq, Hkv, D, page_size, q_stride_t, q_stride_h, o_stride_t, o_stride_h,
                       max_seqlen_q, is_causal, sm_scale, workspace, true, window_left, right, 0, stream);
}

extern "C" int sab_kvcache8_attn_shared(const void* q, int dtype, const int8_t* k_pages, const float* k_scale, const uint8_t* v_pages,
                                        const float* v_scale, const float* k_smooth, void* out, float* lse, const int32_t* cu_seqlens_q,
                                        const int32_t* seqused_k, const int32_t* block_table, int64_t table_stride, int max_pages,
                                        int nseq, int Tq, int Hq, int Hkv, int D, int page_size, int64_t q_stride_t,
                                        int64_t q_stride_h, int64_t o_stride_t, int64_t o_stride_h, int max_seqlen_q, int is_causal,
                                        float sm_scale, void* workspace, int shared_prefix_len, void* stream) {
  SAB_REQUIRE(shared_prefix_len >= 0, SAB_ERR_INVALID, "shared_prefix_len must be >= 0");
  return kvcache8_attn(q, dtype, k_pages, k_scale, v_pages, v_scale, k_smooth, out, lse, cu_seqlens_q, seqused_k, block_table,
                       table_stride, max_pages, nseq, Tq, Hq, Hkv, D, page_size, q_stride_t, q_stride_h, o_stride_t, o_stride_h,
                       max_seqlen_q, is_causal, sm_scale, workspace, false, -1, -1, shared_prefix_len, stream);
}

// sab_kvcache8_prefill and, with window, sab_kvcache8_prefill_window (window_right with the causal rule folded in)
static int kvcache8_prefill(const void* q, int dtype, const int8_t* k_pages, const float* k_scale, const uint8_t* v_pages,
                            const float* v_scale, const float* k_smooth, void* out, float* lse, const int32_t* cu_seqlens_q,
                            const int32_t* seqused_k, const int32_t* block_table, int64_t table_stride, int max_pages, int nseq,
                            int Tq, int Hq, int Hkv, int D, int page_size, int64_t q_stride_t, int64_t q_stride_h,
                            int64_t o_stride_t, int64_t o_stride_h, int max_seqlen_q, int is_causal, float sm_scale,
                            bool window, int window_left, int window_right, void* stream) {
  SAB_REQUIRE(q && k_pages && k_scale && v_pages && v_scale && k_smooth && out && cu_seqlens_q && seqused_k && block_table,
              SAB_ERR_INVALID, "null pointer argument");
  if (int r = check_dtype_dim(dtype, D)) return r;
  SAB_REQUIRE(Hkv > 0 && Hq > 0 && Hq % Hkv == 0, SAB_ERR_INVALID, "num_qo_heads (%d) must be divisible by num_kv_heads (%d)", Hq, Hkv);
  SAB_REQUIRE(nseq > 0 && Tq > 0 && max_seqlen_q > 0 && max_pages > 0 && page_size > 0 && page_size % 16 == 0 && table_stride >= max_pages,
              SAB_ERR_INVALID, "need nseq, Tq, max_seqlen_q, max_pages > 0, page_size a positive multiple of 16 and table_stride >= max_pages");
  SAB_REQUIRE(q_stride_t >= 0 && q_stride_h >= 0 && (q_stride_t | q_stride_h) % 4 == 0 && reinterpret_cast<uintptr_t>(q) % 8 == 0,
              SAB_ERR_INVALID, "q needs 8-byte aligned rows (non-negative strides, multiples of 4 elements)");
  SAB_REQUIRE(o_stride_t >= 0 && o_stride_h >= 0 && (o_stride_t | o_stride_h) % 2 == 0 && reinterpret_cast<uintptr_t>(out) % 4 == 0,
              SAB_ERR_INVALID, "out needs 4-byte aligned element pairs (non-negative, even strides)");
  const int64_t n_qt = (int64_t(max_seqlen_q) + kPfRows - 1) / kPfRows;
  // grid y is Hq, grid x is nseq * ceil(max_seqlen_q / 128); key indices are int
  SAB_REQUIRE(Hq <= 65535 && n_qt * nseq < (int64_t(1) << 31), SAB_ERR_INVALID,
              "launch grid too large: need Hq <= 65535 and nseq * ceil(max_seqlen_q / 128) < 2^31");
  SAB_REQUIRE(int64_t(max_pages) * page_size < (int64_t(1) << 31), SAB_ERR_INVALID, "max_pages * page_size must be < 2^31 keys");
  PfParams p{q, k_pages, k_scale, v_pages, v_scale, k_smooth, cu_seqlens_q, seqused_k, block_table, table_stride, out, lse,
             max_pages, page_size, Hq, Hkv, int(n_qt), max_seqlen_q, Tq, q_stride_t, q_stride_h, o_stride_t, o_stride_h,
             sm_scale, float(double(sm_scale) * 1.4426950408889634), window_left, window_right};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const bool causal = is_causal != 0;
  if (dtype == SAB_DTYPE_FP16)
    return D == 128 ? launch_prefill<__half, 128>(p, nseq, causal, window, st) : launch_prefill<__half, 64>(p, nseq, causal, window, st);
  return D == 128 ? launch_prefill<__nv_bfloat16, 128>(p, nseq, causal, window, st)
                  : launch_prefill<__nv_bfloat16, 64>(p, nseq, causal, window, st);
}

extern "C" int sab_kvcache8_prefill(const void* q, int dtype, const int8_t* k_pages, const float* k_scale, const uint8_t* v_pages,
                                    const float* v_scale, const float* k_smooth, void* out, float* lse, const int32_t* cu_seqlens_q,
                                    const int32_t* seqused_k, const int32_t* block_table, int64_t table_stride, int max_pages, int nseq,
                                    int Tq, int Hq, int Hkv, int D, int page_size, int64_t q_stride_t, int64_t q_stride_h,
                                    int64_t o_stride_t, int64_t o_stride_h, int max_seqlen_q, int is_causal, float sm_scale,
                                    void* stream) {
  return kvcache8_prefill(q, dtype, k_pages, k_scale, v_pages, v_scale, k_smooth, out, lse, cu_seqlens_q, seqused_k, block_table,
                          table_stride, max_pages, nseq, Tq, Hq, Hkv, D, page_size, q_stride_t, q_stride_h, o_stride_t, o_stride_h,
                          max_seqlen_q, is_causal, sm_scale, false, -1, -1, stream);
}

extern "C" int sab_kvcache8_prefill_window(const void* q, int dtype, const int8_t* k_pages, const float* k_scale,
                                           const uint8_t* v_pages, const float* v_scale, const float* k_smooth, void* out, float* lse,
                                           const int32_t* cu_seqlens_q, const int32_t* seqused_k, const int32_t* block_table,
                                           int64_t table_stride, int max_pages, int nseq, int Tq, int Hq, int Hkv, int D, int page_size,
                                           int64_t q_stride_t, int64_t q_stride_h, int64_t o_stride_t, int64_t o_stride_h,
                                           int max_seqlen_q, int is_causal, float sm_scale, int window_left, int window_right,
                                           void* stream) {
  int right = -1;
  if (int r = window_args(window_left, window_right, is_causal, right)) return r;
  return kvcache8_prefill(q, dtype, k_pages, k_scale, v_pages, v_scale, k_smooth, out, lse, cu_seqlens_q, seqused_k, block_table,
                          table_stride, max_pages, nseq, Tq, Hq, Hkv, D, page_size, q_stride_t, q_stride_h, o_stride_t, o_stride_h,
                          max_seqlen_q, is_causal, sm_scale, true, window_left, right, stream);
}
