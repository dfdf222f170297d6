// K1 / K3: expanded-form metrics on Hopper tensor cores (sm_90a, wgmma).
//
// Replaces the pair loop of raft::distance::pairwise_distance for L2Expanded / L2SqrtExpanded /
// CosineExpanded / CorrelationExpanded / InnerProduct (+ Hellinger, RusselRao) and of
// raft::distance::fusedL2NN / fusedDistanceNN (SURVEY.md 8(a2),(a3),(a5),(f1); the reference's last
// implementation was a CUTLASS 3xTF32 mma.sync kernel, CHANGELOG.md:1443,1140 -- this is not a
// port of it).
//
// Numerics: fp32 inputs are pre-split (prep.cuh) into fp16 hi/lo with one power-of-two scale per
// matrix; acc = hi*hi + hi*lo + lo*hi accumulates in fp32 (products of fp16 pairs are exact in
// fp32), i.e. ~22 significant bits per operand -- fp32-grade, same idea as the reference's 3xTF32
// but at the 2x higher fp16 rate and with 4 B/element staged instead of 8.  The tensor core aligns
// every product to the accumulator's exponent and truncates, so the error grows with the number of
// MMAs that touch a LARGE accumulator: the 2^-11-sized cross terms are kept in an accumulator of
// their own and added to the hi*hi sum in the epilogue with one round-to-nearest fp32 add.
// Operands that are exact in fp16 (fp16 inputs, small integers) skip the cross terms altogether.
//
// Structure (one persistent CTA per SM, 384 threads = 3 warpgroups):
//   warpgroup 0     TMA producer: one elected lane per feeding warp issues cp.async.bulk.tensor 2-D loads
//                   (SWIZZLE_128B, mbarrier complete_tx); the other warps only hand their registers over
//   warpgroups 1-2  consumers: warpgroup c owns rows [64c, 64c+64) of every x tile; it issues the
//                   wgmma.m64n128k16 of its rows and runs the epilogue on the accumulator fragments
// Work item = (256-row block of y, run of 128-row tiles of x); every x tile is worked through as two
// 128 x 128 halves (one per 128-row half of the y block): main (hi*hi) + cross accumulators of a
// 64 x 128 warpgroup tile are 128 fp32 registers per thread.
//
//  kResident (k <= 128): the y block (all of K, <= 128 KB) stays in shared memory for the whole run;
//    each consumer warpgroup has an x ring of its own (64-row k-blocks of its slab, fed by producer warp c), loaded once
//    per tile: both halves read them, the last half releases them (a ring holds a whole tile, so it wraps across tiles
//    when nkb < stages).  The two warpgroups take turns issuing their MMAs (named barriers 4 and 5), so one
//    warpgroup's epilogue runs while the other's MMAs do.
//  !kResident (k > 128): both operands stream per k-block (stages of 16 KB of x + 16 KB of the y half).
//
// Epilogues (straight from the registers; d = acc * c + (t_x[i] + t_y[j]), c one scalar):
//   EPI_STORE         the finished 64 x 128 fragment goes to the warpgroup's own staging boxes in shared
//                     memory (SWIZZLE_128B, a ring of 32-row x 64-column boxes) and leaves by TMA stores that
//                     drain while the warpgroup runs the next half's MMAs (tc_stage_store).  Where TMA cannot
//                     address dist (unaligned base or pitch) and in the read-modify-write path of K-chunked
//                     accumulation (k > 320), each thread stores its 2 adjacent columns of 2 rows per
//                     8-column group straight from the registers (8-byte streaming stores).  The kernel Gram
//                     matrices (POST_RBF / POST_POLY / POST_TANH) transform the final value in registers first
//                     (gram_post), so the transformed matrix is the only one written.
//   EPI_MINLOC       per row the minimum of the thread's 16 values of a 64-column chunk is compared with
//                     the row's current global best (read from keys at tile start: an upper bound, keys
//                     only decrease); only a candidate that can change the result takes the slow path
//                     (smallest-column scan + packed 64-bit atomicMin).
//   EPI_MINLOC_MASKED EPI_MINLOC under a row x group adjacency mask (masked_nn.cuh): tiles the mask rules out are not
//                     loaded or multiplied, partly adjacent ones set the non-adjacent values to +inf first.
//   EPI_TOPK          fused brute-force kNN: the same minimum and vote against the row's current k-th best;
//                     every pair at or below it is appended to the row's candidate list (see the kNN
//                     kernels in knn.cuh).
//   EPI_EPS           epsilon neighbourhood: the EPI_STORE / POST_CLAMP distance, compared with eps; the 0/1 bytes go to
//                     the EPI_STORE staging ring (one 64 x 128-byte box per tile), leave from there by TMA or a copy, and
//                     are counted per column into shared memory (tc_eps_tile).
//   EPI_RADIUS        radius neighbours: the EPI_STORE distance of kPost, compared with eps as a 32-bit hit mask per
//                     row and half tile in registers; count mode adds the row's hits to its degree, fill mode appends
//                     them as packed keys to the row's CSR segment (radius_row32).
//
// Diagnostic builds (DESIGN.md section 5, scripts/tc_breakdown.py; never the library's own build): B2D_TC_DIAG = 1 keeps
// the MMAs only (no epilogue, no staging; one sum of the accumulators keeps them live), 2 computes and stages every value
// but issues no TMA store, 3 skips the MMAs (stages zeros, TMA stores on).  The results are wrong by design.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cstdint>
#include <type_traits>
#include "nn_key.cuh"
#include "ptx.cuh"
#include "tc_params.cuh"

namespace b2d {

// max(v, 0) that keeps a NaN (fmaxf(NaN, 0) = 0 would turn a poisoned distance into a perfect match)
__device__ __forceinline__ float clamp0(float v)
{
  float r;
  asm("max.NaN.f32 %0, %1, 0f00000000;" : "=f"(r) : "f"(v));
  return r;
}

// Gram-matrix transform of one finished value u (RBF: the clamped squared distance; POLY / TANH: the inner product), in
// full-precision fp32: one rounding for gamma u (+ coef0), then expf / tanhf, or the power by binary exponentiation
// (degree 0 gives 1 for every u, NaN included)
template <int kPost>
__device__ __forceinline__ float gram_post(float u, float gamma, float coef0, int degree)
{
  if constexpr (kPost == POST_RBF) return expf(-(gamma * u));
  const float t = fmaf(gamma, u, coef0);
  if constexpr (kPost == POST_TANH) return tanhf(t);
  float r = 1.f, b = t;
  for (unsigned e = static_cast<unsigned>(degree); e != 0u; e >>= 1) {
    if (e & 1u) r *= b;
    if (e > 1u) b *= b;
  }
  return r;
}

// ratio metrics on the tensor path: a = acc * c (the inner product), s = t_x + t_y (the squared norms)
template <int kPost>
__device__ __forceinline__ float post_ratio(float a, float s)
{
  const float den = kPost == POST_JACCARD ? s - a : s;
  const float num = kPost == POST_JACCARD ? a : 2.f * a;
  return !(den <= 0.f) ? clamp0(1.f - __fdividef(num, den)) : 0.f;   // (NaN inputs give NaN, 0/0 gives 0)
}

__device__ __forceinline__ float min3(float a, float b, float c) { return fminf(fminf(a, b), c); }
__device__ __forceinline__ float max3(float a, float b, float c) { return fmaxf(fmaxf(a, b), c); }

// EPI_TOPK slow path (one row of one 64-column chunk: 16 values, columns col0 + 8 i + e): every value at or below the
// row's k-th best so far takes a slot of the row's list; a full list keeps the smallest dropped key (knn_merge_kernel
// decides from it whether the row must be repaired).  Deliberately NOT inlined: one copy instead of one per call site
// keeps the kNN instantiation inside the instruction cache.
__device__ __noinline__ void knn_append16(unsigned* cnt, long long* cand, unsigned cap, long long* dropmin, int64_t row,
                                          long long col0, float xn, float thr, float a0, float a1, float a2, float a3,
                                          float a4, float a5, float a6, float a7, float a8, float a9, float a10, float a11,
                                          float a12, float a13, float a14, float a15)
{
  const float a[16] = {a0, a1, a2, a3, a4, a5, a6, a7, a8, a9, a10, a11, a12, a13, a14, a15};
#pragma unroll
  for (int t = 0; t < 16; ++t) {
    const float lv = a[t];
    const float dv = lv + xn;
    if (dv <= thr && lv < __int_as_float(0x7f800000)) {
      const long long key = key_pack(dv, col0 + 8 * (t >> 1) + (t & 1));
      const unsigned slot = atomicAdd(&cnt[row], 1u);
      if (slot < cap) cand[row * cap + slot] = key;
      else atomicMin(&dropmin[row], key);   // list full (ordered / adversarial data): remember the best key that was dropped
    }
  }
}

// EPI_MINLOC_MASKED, PARTIAL tiles: bit 4i + 2j + e of the result is set when row row0 + 8j of x is adjacent to the group
// of column cl0 + 8i + e of the y block (col_grp: the block's column groups in shared memory).  Not inlined, for the
// same reason as knn_append16.
__device__ __noinline__ unsigned long long masked_keep64(const int* col_grp, int cl0, const unsigned* bits, int64_t groups,
                                                         int64_t row0, int64_t m)
{
  unsigned long long keep = 0ull;
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const int64_t r = row0 + 8 * j;
    if (r >= m) continue;
    const unsigned* word = bits + (r >> 5) * groups;
    const int sh         = static_cast<int>(r & 31);
#pragma unroll
    for (int i = 0; i < 16; ++i)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int g = col_grp[cl0 + 8 * i + e];
        if (g >= 0 && ((__ldg(&word[g]) >> sh) & 1u)) keep |= 1ull << (4 * i + 2 * j + e);
      }
  }
  return keep;
}

// EPI_RADIUS, one row of a 64 x 128 warpgroup tile: a0..a31 are the thread's distances of the row (a[2 i + e] at column
// col0 + 8 i + e) and bit t of `hits` is set when a[t] is within the radius.  The 4 lanes of a quad hold the row's 128
// columns; the whole warp calls (the quad shuffles), a lane of a row outside the matrix with hits == 0.
//   count: the quad's hits are added to cnt[row] (one atomic when there are any).
//   fill:  one atomic on the row's fill counter cnt[row] reserves the quad's slots; each lane writes its hits, in column
//          order after those of the lanes below it, as key_pack(d, j) to out[indptr[row] + slot].  A slot at or past
//          min(indptr[row + 1], nnz) is dropped (the degrees no longer match the data): nothing is written outside out.
// Not inlined, for the reason given at knn_append16.
__device__ __noinline__ void radius_row32(unsigned* cnt, long long* out, const long long* indptr, long long nnz, int64_t row,
                                          long long col0, unsigned hits, int fill, float a0, float a1, float a2, float a3,
                                          float a4, float a5, float a6, float a7, float a8, float a9, float a10, float a11,
                                          float a12, float a13, float a14, float a15, float a16, float a17, float a18,
                                          float a19, float a20, float a21, float a22, float a23, float a24, float a25,
                                          float a26, float a27, float a28, float a29, float a30, float a31)
{
  const unsigned tq = threadIdx.x & 3u;
  const unsigned c  = __popc(hits);
  if (!fill) {
    unsigned t = c + __shfl_xor_sync(0xffffffffu, c, 1);
    t += __shfl_xor_sync(0xffffffffu, t, 2);
    if (tq == 0u && t != 0u) atomicAdd(&cnt[row], t);
    return;
  }
  // exclusive prefix of the quad's counts, the quad's total from its last lane
  unsigned incl = c, u = __shfl_up_sync(0xffffffffu, incl, 1, 4);
  if (tq >= 1u) incl += u;
  u = __shfl_up_sync(0xffffffffu, incl, 2, 4);
  if (tq >= 2u) incl += u;
  const unsigned total = __shfl_sync(0xffffffffu, incl, 3, 4);
  unsigned base = 0u;
  if (tq == 0u && total != 0u) base = atomicAdd(&cnt[row], total);
  base = __shfl_sync(0xffffffffu, base, 0, 4);
  if (c == 0u) return;
  const long long start = indptr[row];
  const long long lim   = min(indptr[row + 1], nnz);
  long long pos         = start + base + (incl - c);
  const float a[32] = {a0,  a1,  a2,  a3,  a4,  a5,  a6,  a7,  a8,  a9,  a10, a11, a12, a13, a14, a15,
                       a16, a17, a18, a19, a20, a21, a22, a23, a24, a25, a26, a27, a28, a29, a30, a31};
#pragma unroll
  for (int t = 0; t < 32; ++t) {
    if ((hits >> t) & 1u) {
      if (pos < lim) out[pos] = key_pack(a[t], col0 + 8 * (t >> 1) + (t & 1));
      ++pos;
    }
  }
}

// The finished distance of a clamping post (tc_post_clamps) in the fragment layout of tc_epilogue: clamped at 0, 0 where
// row i of x is row i - diag_off of y, then the sqrt of POST_CLAMP_SQRT.  kGuardN: only columns below n are zeroed.  EPI_EPS
// needs that, since it counts every column of a row window; EPI_STORE and EPI_RADIUS set diag_off = 0 only with m == n, so
// a column at or past n pairs with a row at or past m, which they never store or count.
template <int kPost, bool kGuardN>
__device__ __forceinline__ void tc_finish(float (&v)[64], const TcParams& p, int64_t row0, int64_t gc0)
{
#pragma unroll
  for (int c = 0; c < 64; ++c) v[c] = clamp0(v[c]);
  if (p.diag_off != TC_NO_DIAG) {
    // row0 + 8 j - diag_off == gc0 + 8 i + e  <=>  dd == 8 (i - j) + e, which lies in [-8, 121]
    const int64_t dd = row0 - p.diag_off - gc0;
    if (dd >= -8 && dd < 128) {
      const int d = static_cast<int>(dd);
#pragma unroll
      for (int i = 0; i < 16; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j)
#pragma unroll
          for (int e = 0; e < 2; ++e)
            if (d == 8 * (i - j) + e && (!kGuardN || gc0 + 8 * i + e < p.n)) v[4 * i + 2 * j + e] = 0.f;
    }
  }
  if (kPost == POST_CLAMP_SQRT) {
#pragma unroll
    for (int c = 0; c < 64; ++c) asm("sqrt.approx.f32 %0, %1;" : "=f"(v[c]) : "f"(v[c]));
  }
}

// Epilogue of one 64 x 128 warpgroup tile.  v[4i + 2j + e] holds row row0 + 8j, column gc0 + 8i + e of the accumulator
// (main + cross already summed); on return (EPI_STORE) v holds the finished distances, and they have been written
// unless p.tma_store (then tc_stage_store writes them).  EPI_MINLOC_MASKED: the values whose bit in `keep` is clear
// become +inf (never a candidate) before the minimum.
template <int kEpi, int kPost>
__device__ __forceinline__ void tc_epilogue(float (&v)[64], const TcParams& p, const float* col_tb, int cl0, int64_t gc0,
                                            int64_t row0, const float (&ta)[2], const float (&cfr)[2], float (&thr)[2],
                                            const float (&xnr)[2], bool ynu, unsigned long long keep = ~0ull)
{
  // d = acc * c_row (* column factor) + (t_x + t_y); the arg-min modes leave the row-constant t_x out (added on the
  // slow path only)
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    const float2 tb = *reinterpret_cast<const float2*>(&col_tb[cl0 + 8 * i]);
    float sb0 = 1.f, sb1 = 1.f;
    if (ynu) {  // rows of y with their own exponent: per-column factors straight from global memory (rare)
      const int64_t gc = gc0 + 8 * i;
      sb0 = gc < p.n ? __ldg(&p.ysc[gc]) : 1.f;
      sb1 = gc + 1 < p.n ? __ldg(&p.ysc[gc + 1]) : 1.f;
    }
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      float a0 = v[4 * i + 2 * j], a1 = v[4 * i + 2 * j + 1];
      if (ynu) { a0 *= sb0; a1 *= sb1; }
      if (kEpi == EPI_STORE && tc_post_ratio(kPost)) {
        v[4 * i + 2 * j]     = post_ratio<kPost>(a0 * cfr[j], ta[j] + tb.x);
        v[4 * i + 2 * j + 1] = post_ratio<kPost>(a1 * cfr[j], ta[j] + tb.y);
      } else if (kEpi == EPI_STORE || kEpi == EPI_EPS || kEpi == EPI_RADIUS) {
        v[4 * i + 2 * j]     = fmaf(a0, cfr[j], ta[j] + tb.x);
        v[4 * i + 2 * j + 1] = fmaf(a1, cfr[j], ta[j] + tb.y);
      } else {
        v[4 * i + 2 * j]     = fmaf(a0, cfr[j], tb.x);
        v[4 * i + 2 * j + 1] = fmaf(a1, cfr[j], tb.y);
      }
    }
  }
  if constexpr (kEpi == EPI_EPS) {
    // the POST_CLAMP distance of EPI_STORE.  (Columns beyond n hold NaN from t_y and stay unmatched; the row window check
    // keeps them out.)
    tc_finish<POST_CLAMP, true>(v, p, row0, gc0);
    return;
  }
  if constexpr (kEpi == EPI_RADIUS) {
    // the EPI_STORE values of acc_mode 0, then one hit mask per row instead of the stores.  Columns beyond n hold NaN (from
    // t_y), rows beyond m are left out here.
    if (tc_post_clamps(kPost)) tc_finish<kPost, false>(v, p, row0, gc0);
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      unsigned hits = 0u;
#pragma unroll
      for (int t = 0; t < 32; ++t)
        if (v[4 * (t >> 1) + 2 * j + (t & 1)] <= p.eps) hits |= 1u << t;
      if (row0 + 8 * j >= p.m) hits = 0u;
      if (__any_sync(0xffffffffu, hits != 0u))
        radius_row32(p.knn_cnt, p.knn_cand, p.rad_indptr, p.rad_nnz, row0 + 8 * j, gc0, hits, p.rad_fill, v[2 * j],
                     v[2 * j + 1], v[4 + 2 * j], v[5 + 2 * j], v[8 + 2 * j], v[9 + 2 * j], v[12 + 2 * j], v[13 + 2 * j],
                     v[16 + 2 * j], v[17 + 2 * j], v[20 + 2 * j], v[21 + 2 * j], v[24 + 2 * j], v[25 + 2 * j],
                     v[28 + 2 * j], v[29 + 2 * j], v[32 + 2 * j], v[33 + 2 * j], v[36 + 2 * j], v[37 + 2 * j],
                     v[40 + 2 * j], v[41 + 2 * j], v[44 + 2 * j], v[45 + 2 * j], v[48 + 2 * j], v[49 + 2 * j],
                     v[52 + 2 * j], v[53 + 2 * j], v[56 + 2 * j], v[57 + 2 * j], v[60 + 2 * j], v[61 + 2 * j]);
    }
    return;
  }
  if (kEpi == EPI_STORE) {
    // (the manual stores: 8-byte vectors when dist and its pitch allow them)
    const bool fast = row0 + 8 < p.m && gc0 + 127 < p.n && tc_dist_vec2(reinterpret_cast<uintptr_t>(p.dist), p.ldd);
    if (p.acc_mode >= 2) {
      // K-chunked accumulation (k > 320): add this chunk's contribution to what the earlier chunks left in dist -- a
      // round-to-nearest fp32 add per chunk instead of ever longer truncating MMA chains on one accumulator
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int64_t gi = row0 + 8 * j;
        const float* q   = p.dist + gi * p.ldd + gc0;
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          if (fast) {
            const float2 o = __ldcs(reinterpret_cast<const float2*>(q + 8 * i));
            v[4 * i + 2 * j] += o.x;
            v[4 * i + 2 * j + 1] += o.y;
          } else if (gi < p.m) {
            if (gc0 + 8 * i < p.n) v[4 * i + 2 * j] += __ldcs(q + 8 * i);
            if (gc0 + 8 * i + 1 < p.n) v[4 * i + 2 * j + 1] += __ldcs(q + 8 * i + 1);
          }
        }
      }
    }
    if (tc_post_clamps(kPost) && (p.acc_mode == 0 || p.acc_mode == 3)) tc_finish<kPost, false>(v, p, row0, gc0);
    if constexpr (tc_post_gram(kPost)) {
      if (p.acc_mode == 0 || p.acc_mode == 3) {   // (K-chunked: the earlier chunks store the partial sum untransformed)
#pragma unroll
        for (int c = 0; c < 64; ++c) v[c] = gram_post<kPost>(v[c], p.gamma, p.coef0, p.degree);
      }
    }
    if (p.tma_store) return;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int64_t gi = row0 + 8 * j;
      float* q         = p.dist + gi * p.ldd + gc0;
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        if (fast) {
          ptx::st_global_cs_v2(q + 8 * i, v[4 * i + 2 * j], v[4 * i + 2 * j + 1]);
        } else if (gi < p.m) {
          if (gc0 + 8 * i < p.n) ptx::st_global_cs(q + 8 * i, v[4 * i + 2 * j]);
          if (gc0 + 8 * i + 1 < p.n) ptx::st_global_cs(q + 8 * i + 1, v[4 * i + 2 * j + 1]);
        }
      }
    }
    return;
  }
  // Arg-min modes, per 64-column chunk and row: the minimum of this thread's 16 values is compared with the row's
  // current global best.  Only a candidate that can change the result (value <= best: '<=' so that an equal value with
  // a smaller index still gets through) takes the slow path: locate the smallest column holding the minimum (ascending
  // scan) and let the packed 64-bit atomicMin decide -- (value, index) order == raft::argmin_op
  // (cpp/include/raft/core/operators.hpp:187-194).  After the first few y blocks this is rare.
  const float inf = __int_as_float(0x7f800000);
  if (kEpi == EPI_MINLOC_MASKED && keep != ~0ull) {
#pragma unroll
    for (int c = 0; c < 64; ++c)
      if (!((keep >> c) & 1ull)) v[c] = inf;
  }
#pragma unroll
  for (int cc = 0; cc < 2; ++cc) {
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int b = 32 * cc + 2 * j;   // v[b + 4i + e], i in [0, 8)
      float m0 = min3(v[b], v[b + 1], v[b + 4]);
      float m1 = min3(v[b + 5], v[b + 8], v[b + 9]);
      float m2 = min3(v[b + 12], v[b + 13], v[b + 16]);
      float m3 = min3(v[b + 17], v[b + 20], v[b + 21]);
      m0       = min3(m0, v[b + 24], v[b + 25]);
      m1       = min3(m1, v[b + 28], v[b + 29]);
      const float mn = fminf(min3(m0, m1, m2), m3);
      // (+inf marks columns beyond n: never a candidate).  Keys hold the full distance |x|^2 + v, so the row term is
      // added for the comparison -- one FADD per row here instead of one per element
      const bool cand = (mn + xnr[j]) <= thr[j] && mn < inf;
      if (__any_sync(0xffffffffu, cand) && cand) {
        const int64_t gcc = gc0 + 64 * cc;   // global column of v[b]
        if (kEpi != EPI_TOPK) {
          int cbest = 0;
#pragma unroll
          for (int i = 7; i >= 0; --i) {
            if (v[b + 4 * i + 1] == mn) cbest = 8 * i + 1;
            if (v[b + 4 * i] == mn) cbest = 8 * i;
          }
          const float dv = mn + xnr[j];
          long long gj   = gcc + cbest;
          if (p.col_map != nullptr) {  // permuted columns: the smallest SOURCE index among the equal minima
            int best = 0x7fffffff;
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
              for (int e = 0; e < 2; ++e)
                if (v[b + 4 * i + e] == mn) best = min(best, __ldg(&p.col_map[gcc + 8 * i + e]));
            gj = best;
          }
          atomicMin(&p.keys[row0 + 8 * j], key_pack(dv, gj + p.idx_offset));
          thr[j] = dv;
        } else {
          knn_append16(p.knn_cnt, p.knn_cand, p.knn_cap, p.knn_dropmin, row0 + 8 * j, gcc + p.idx_offset, xnr[j], thr[j],
                       v[b], v[b + 1], v[b + 4], v[b + 5], v[b + 8], v[b + 9], v[b + 12], v[b + 13], v[b + 16], v[b + 17],
                       v[b + 20], v[b + 21], v[b + 24], v[b + 25], v[b + 28], v[b + 29]);
        }
      }
    }
  }
}

// EPI_STORE through TMA, the common case (one warp-uniform test in the kernel: p.tma_store, p.acc_mode == 0, no self pairs,
// no per-column scales): tc_epilogue's arithmetic for it, without the branches of the other cases.  Ragged tiles take it
// too: TMA clips what lies outside the matrix.  The kernel keeps the Gram matrices off it (kFastPost): a second inlined
// copy of their expf / tanhf made the tanh instantiation spill.
template <int kPost>
__device__ __forceinline__ void tc_epilogue_store_fast(float (&v)[64], const TcParams& p, const float* col_tb, int cl0,
                                                       const float (&ta)[2], const float (&cfr)[2])
{
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    const float2 tb = *reinterpret_cast<const float2*>(&col_tb[cl0 + 8 * i]);
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        float& d      = v[4 * i + 2 * j + e];
        const float s = ta[j] + (e ? tb.y : tb.x);
        if constexpr (tc_post_ratio(kPost)) d = post_ratio<kPost>(d * cfr[j], s);
        else d = fmaf(d, cfr[j], s);
        if constexpr (tc_post_clamps(kPost)) d = clamp0(d);
        if constexpr (kPost == POST_CLAMP_SQRT) asm("sqrt.approx.f32 %0, %1;" : "=f"(d) : "f"(d));
        if constexpr (tc_post_gram(kPost)) d = gram_post<kPost>(d, p.gamma, p.coef0, p.degree);
      }
  }
}

// EPI_STORE through TMA: the warpgroup's finished 64 x 128 tile v (fragment layout as in tc_epilogue) is written into
// its ring of two staging boxes and stored with one cp.async.bulk.tensor per 32-row x 64-column box (L2 evict-first: the
// result is not read again here).  The box goes through a 3-D view of dist, {32 columns, column group, row} with box
// {32, 2, 32}, so each store writes 256 contiguous bytes of each of its 32 rows; 64 x 32 boxes of 128-byte row pieces
// made the kernel measurably slower (DESIGN.md section 5).  The tile's 4 boxes go out as two pairs: pair q holds columns
// [64 q, 64 q + 64), rows [32 s, 32 s + 32) in slot s, written by warps 2 s and 2 s + 1.  The lead thread (`issuer`)
// waits until the previous pair's stores have finished reading both slots, the warpgroup meets at its named barrier,
// writes the pair, fences it for the TMA unit once and meets again, and the lead issues both stores as one bulk group.
// One fence (MEMBAR + FENCE.VIEW.ASYNC in the SASS) and two barriers per pair measured faster than a fence per box or a
// per-slot mbarrier hand-off (DESIGN.md section 5).  Only this warpgroup writes its boxes and only its lead issues and
// waits for their stores.  Boxes outside the matrix are skipped; TMA clips the ragged ones at row m and at the last whole
// column group of tmap_d ({32, n / 32, m}).  When n % 32 != 0, the box holding the last, partial group ng = n / 32 also
// goes out through tmap_dt, a view of the groups from the box's first one, gb = ng rounded down to even (boxes start at
// even groups), to ng: {n % 32, ng - gb + 1, m}, same box, at coordinates (0, 0, row).  TMA clips every column at or past
// n there, so nothing lands in the caller's padding; when ng is odd it also writes the first n % 32 columns of group
// ng - 1 again, with the values tmap_d wrote there.  (The view starts at the box, not at the partial group, so that no
// coordinate is negative: a store at group coordinate -1 ended in a device fault on an H100.)  After the CTA's last
// tile (`last`) the issuer waits for all its stores, so the CTA's shared memory outlives them.
//   box element (r, g, c) (row, column group, column of the group) sits in 128-byte line L = 2 r + g, at byte
//   L * 128 + ((c / 4) ^ (L % 8)) * 16 + (c % 4) * 4 (SWIZZLE_128B).  L % 8 = (2 quad + g) % 8 for the warp's rows, so
//   rows quad and quad + 4 share a phase, but the warp's 8-byte writes (8 rows x 2 adjacent 16-byte chunks) still cover
//   every bank exactly twice -- no conflicts.
__device__ __forceinline__ void tc_stage_store(const float (&v)[64], const CUtensorMap* tmap_d, const CUtensorMap* tmap_dt,
                                               uint32_t stg, bool issuer, bool last, int wg, int64_t row_w, int64_t col_w,
                                               const TcParams& p)
{
  static_assert(TC_STG_BOXES == 2, "a pair of boxes fills the ring: wait_group.read 0 frees it");
  static_assert(TC_D_BOX_GROUPS == 2 && TC_D_BOX_ROWS == 32, "the addressing below is written for 32 x 64 boxes");
  const int lane = threadIdx.x & 31, w = (threadIdx.x >> 5) & 3;
  const int quad = lane >> 2, tq = lane & 3;
  // this thread's rows 16 (w % 2) + quad (+8) of the box in slot w / 2 and the swizzled 16-byte chunk of its column pair
  const uint32_t t_off = stg + (w >> 1) * TC_D_BOX_BYTES + (16 * (w & 1) + quad) * 256 + 8 * (tq & 1);
  const uint32_t t_xor = static_cast<uint32_t>((tq >> 1) ^ (2 * (quad & 3))) * 16;
#pragma unroll
  for (int q = 0; q < 2; ++q) {
    // the previous pair's stores have read both slots
    if (issuer) ptx::tma_store_wait_read<0>();
    ptx::bar_sync(2 + wg, 128);
#pragma unroll
    for (int ii = 0; ii < 8; ++ii) {
      const int i = 8 * q + ii, g = ii >> 2;   // 8-column group of the tile, column group of the box
#pragma unroll
      for (int j = 0; j < 2; ++j)
        ptx::st_shared_v2(t_off + j * 8 * 256 + g * 128 + ((32 * (ii & 3) + 16 * g) ^ t_xor), v[4 * i + 2 * j],
                          v[4 * i + 2 * j + 1]);
    }
    ptx::fence_proxy_async_smem();   // the generic-proxy writes become visible to the TMA unit
    ptx::bar_sync(2 + wg, 128);
    if (issuer) {
      // (32-bit coordinates: the TMA path is only taken with m and n below 2^31, tc_store_plan)
      const int n = static_cast<int>(p.n), ng = n >> 5;                          // whole column groups of dist
      const int gc = static_cast<int>(col_w) + TC_D_BOX_COLS * q, gg = gc >> 5;   // the pair's first column and group
#pragma unroll
      for (int s = 0; s < 2; ++s) {
        const int gr = static_cast<int>(row_w) + TC_D_BOX_ROWS * s;
#if !defined(B2D_TC_DIAG) || B2D_TC_DIAG != 2
        if (gc < n && gr < static_cast<int>(p.m)) {
          const uint32_t box = stg + s * TC_D_BOX_BYTES;
          if (gg < ng) ptx::tma_store_3d(tmap_d, box, 0, gg, gr, ptx::policy_evict_first());
          if ((n & 31) != 0 && gg == (ng & ~1))   // the box holds the partial group ng
            ptx::tma_store_3d(tmap_dt, box, 0, 0, gr, ptx::policy_evict_first());
        }
#endif
      }
      ptx::tma_store_commit();   // one group per pair (possibly empty): the wait above counts pairs
    }
  }
  if (issuer && last) ptx::tma_store_wait_all();   // the CTA's last tile: its shared memory outlives every store
}

// EPI_EPS after tc_epilogue: the warpgroup's finished 64 x 128 tile v becomes 0 / 1 bytes in one 64-row x 128-byte box of
// its EPI_STORE staging ring (slot = parity of the warpgroup's tile count box_it), byte (r, c) at
// r * 128 + ((c / 16) ^ (r % 8)) * 16 + c % 16 (SWIZZLE_128B).  Rows beyond m never match (d is >= 0 or NaN), columns
// beyond n hold NaN.  Each thread writes its flags as 2-byte shared stores (conflict-free: the 8 rows of a warp's store
// hit 8 different 16-byte chunks).  Everything after reads the box, in every output mode:
//   adjacency: TMA (p.tma_store) as in tc_stage_store, or else each warp copies 16 rows out, one row per step with 4 bytes
//     per lane (2- or 1-byte stores where the base or pitch is not 4- or 2-byte aligned, and at the end of a row);
//     count-only stores nothing.
//   counts: thread t sums 4 rows of the 16-byte chunk t % 8 (bytes <= 4), the warp's 4 threads of a chunk add theirs by
//     a reduce-scatter (3 shuffles; bytes <= 16), and each adds 4 column counts to the item's col_cnt in shared memory.
// (The fragment's own registers are not an option for either: acc and crs keep 128 registers live through the epilogue.)
__device__ __forceinline__ void tc_eps_tile(const float (&v)[64], const TcParams& p, uint32_t* col_cnt, int hcol, int64_t row0,
                                            const CUtensorMap* tmap_d, uint32_t stg, bool issuer, bool last, int wg,
                                            int64_t row_w, int64_t col_w, uint32_t& box_it)
{
  const int lane = threadIdx.x & 31;
  const int quad = lane >> 2, tq = lane & 3;
  const uint32_t box = stg + (box_it & 1u) * TC_D_BOX_BYTES;
  ++box_it;
  // TMA: the store issued two tiles ago read this slot, it must be done (the latest store may still be reading)
  if (issuer && p.tma_store) ptx::tma_store_wait_read<1>();
  ptx::bar_sync(2 + wg, 128);
  const uint32_t t_off = box + (16 * ((threadIdx.x >> 5) & 3) + quad) * 128 + 2 * tq;
#pragma unroll
  for (int w = 0; w < 8; ++w) {   // the thread's columns 8 i + {0, 1}, i = 2 w, 2 w + 1 -> bytes 2 (i & 1) + {0, 1}
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      uint32_t word = 0u;
#pragma unroll
      for (int b = 0; b < 4; ++b)
        if (v[4 * (2 * w + (b >> 1)) + 2 * j + (b & 1)] <= p.eps) word |= 1u << (8 * b);
      if (row0 + 8 * j >= p.m) word = 0u;
      const uint32_t o = t_off + 8 * j * 128 + ((16 * w) ^ (16 * quad));
      ptx::st_shared_u16(o, word);
      ptx::st_shared_u16(o + 8, word >> 16);
    }
  }
  if (p.tma_store) ptx::fence_proxy_async_smem();   // the generic-proxy writes become visible to the TMA unit
  ptx::bar_sync(2 + wg, 128);
  if (p.tma_store) {
    if (issuer) {
      if (col_w < p.n && row_w < p.m)
        ptx::tma_store_2d(tmap_d, box, static_cast<int32_t>(col_w), static_cast<int32_t>(row_w), ptx::policy_evict_first());
      ptx::tma_store_commit();
      if (last) ptx::tma_store_wait_all();   // the CTA's last tile: its shared memory outlives every store
    }
  } else if (p.adj != nullptr) {
    // warp w copies rows [16 w, 16 w + 16) of the box, one row per step: lane l the 4 bytes at column 4 l, so every store
    // instruction writes 128 contiguous bytes of one row
    const int c       = 4 * lane;
    const int64_t nc  = p.n - col_w - c;   // columns of this lane's 4 inside the matrix
    const int al      = static_cast<int>((reinterpret_cast<uintptr_t>(p.adj) | static_cast<uintptr_t>(p.ld_adj)) & 3u);
    const int w16     = 16 * ((threadIdx.x >> 5) & 3);
#pragma unroll 4
    for (int rr = 0; rr < 16; ++rr) {
      const int r = w16 + rr;
      if (row_w + r >= p.m || nc <= 0) continue;
      uint32_t wd;
      asm volatile("ld.shared.u32 %0, [%1];" : "=r"(wd) : "r"(box + r * 128 + (((lane >> 2) ^ (r & 7)) * 16) + 4 * (lane & 3)));
      uint8_t* q = p.adj + (row_w + r) * p.ld_adj + col_w + c;
      if (al == 0 && nc >= 4) {
        __stcs(reinterpret_cast<unsigned*>(q), wd);
      } else if ((al & 1) == 0) {
        if (nc >= 2) __stcs(reinterpret_cast<unsigned short*>(q), static_cast<unsigned short>(wd & 0xffffu));
        else __stcs(q, static_cast<unsigned char>(wd & 0xffu));
        if (nc >= 4) __stcs(reinterpret_cast<unsigned short*>(q + 2), static_cast<unsigned short>(wd >> 16));
        else if (nc == 3) __stcs(q + 2, static_cast<unsigned char>((wd >> 16) & 0xffu));
      } else {
#pragma unroll
        for (int b = 0; b < 4; ++b)
          if (b < nc) __stcs(q + b, static_cast<unsigned char>((wd >> (8 * b)) & 0xffu));
      }
    }
  }
  if (p.vd == nullptr) return;
  const int cc = threadIdx.x & 7, rg = (threadIdx.x & 127) >> 3;   // chunk cc of rows [4 rg, 4 rg + 4)
  uint4 s = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const int r   = 4 * rg + u;
    const uint4 d = ptx::ld_shared_v4(box + r * 128 + ((cc ^ (r & 7)) * 16));
    s.x += d.x; s.y += d.y; s.z += d.z; s.w += d.w;
  }
  // lanes cc, cc + 8, cc + 16, cc + 24 of the warp hold the same chunk: lane bit 4 keeps words {z, w} or {x, y}, bit 3 one
  // of those, so lane (lane >> 3) ends with word lane >> 3 of the chunk: columns 16 cc + 4 (lane >> 3) + {0..3}
  const bool b4 = (lane & 16) != 0, b3 = (lane & 8) != 0;
  const uint32_t k0 = (b4 ? s.z : s.x) + __shfl_xor_sync(0xffffffffu, b4 ? s.x : s.z, 16);
  const uint32_t k1 = (b4 ? s.w : s.y) + __shfl_xor_sync(0xffffffffu, b4 ? s.y : s.w, 16);
  const uint32_t c4 = (b3 ? k1 : k0) + __shfl_xor_sync(0xffffffffu, b3 ? k0 : k1, 8);
  if (c4 != 0u) {
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      const uint32_t c = (c4 >> (8 * b)) & 0xffu;
      if (c != 0u) atomicAdd(&col_cnt[hcol + 16 * cc + 4 * (lane >> 3) + b], c);
    }
  }
}

// EPI_EPS: the counts of y block n_blk go to vd, one atomic per column (ct: the consumer thread's column) and one per warp
// for the total vd[n]
__device__ __forceinline__ void tc_eps_flush(const TcParams& p, const uint32_t* col_cnt, int n_blk, int ct)
{
  const uint32_t c   = col_cnt[ct];
  const int64_t gj   = static_cast<int64_t>(n_blk) * TC_BN + ct;
  const uint32_t tot = __reduce_add_sync(0xffffffffu, c);
  if (p.vd64) {
    if (c != 0u) atomicAdd(static_cast<unsigned long long*>(p.vd) + gj, static_cast<unsigned long long>(c));
    if ((threadIdx.x & 31) == 0 && tot != 0u) atomicAdd(static_cast<unsigned long long*>(p.vd) + p.n, static_cast<unsigned long long>(tot));
  } else {
    if (c != 0u) atomicAdd(static_cast<unsigned*>(p.vd) + gj, c);
    if ((threadIdx.x & 31) == 0 && tot != 0u) atomicAdd(static_cast<unsigned*>(p.vd) + p.n, tot);
  }
}

template <bool kResident, int kEpi, int kPost>
__global__ void __launch_bounds__(TC_THREADS, 1)
expanded_tc_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                   const __grid_constant__ CUtensorMap tmap_d, const __grid_constant__ CUtensorMap tmap_dt, const TcParams p)
{
  using Carve                    = TcCarve<kResident, kEpi>;
  constexpr int kStages          = Carve::stages;
  constexpr uint32_t kStageBytes = Carve::stage_bytes;
  constexpr bool kMasked         = kEpi == EPI_MINLOC_MASKED;
  constexpr bool kMinloc         = kEpi == EPI_MINLOC || kMasked;
  if (p.run_flag != nullptr && __ldg(p.run_flag) == 0u) return;  // conditional launch (no host round trip)
  extern __shared__ __align__(1024) uint8_t smem[];
  // SWIZZLE_128B atoms need 1024-byte alignment; the dynamic window starts 1024-aligned (no static
  // shared memory in this kernel).  Checked, not assumed: a misaligned base traps.
  if ((ptx::smem_u32(smem) & 1023u) != 0u) __trap();
  uint8_t* b_base = smem;  // resident: [nkb] k-blocks of the y block
  uint8_t* a_base = smem + Carve::a_off;  // stages: x k-block (+ y half k-block)
  float* col_tb   = reinterpret_cast<float*>(smem + Carve::tb_off);  // [256] t_y of this y block
  int* col_grp    = reinterpret_cast<int*>(smem + Carve::grp_off);  // masked: [256] group of every column of the y block
  uint64_t* bars  = reinterpret_cast<uint64_t*>(col_tb + TC_BN);
  constexpr int kRings = Carve::rings;
  uint64_t* afull  = bars;                               // [kRings * TC_MAX_STAGES]: slot s of ring w at kRings * s + w
  uint64_t* aempty = bars + kRings * TC_MAX_STAGES;      // [kRings * TC_MAX_STAGES]
  uint64_t* bfull  = bars + 2 * kRings * TC_MAX_STAGES;  // [TC_MAX_RES_KB]
  uint64_t* bempty = bfull + TC_MAX_RES_KB;              // [TC_MAX_RES_KB]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    // empty barriers: one arrival per consumer warpgroup that reads the ring (resident: its own ring; streaming: both)
    for (int i = 0; i < kRings * TC_MAX_STAGES; ++i) { ptx::mbar_init(&afull[i], 1); ptx::mbar_init(&aempty[i], kResident ? 1 : 2); }
    for (int i = 0; i < TC_MAX_RES_KB; ++i) { ptx::mbar_init(&bfull[i], 1); ptx::mbar_init(&bempty[i], 2); }
    ptx::fence_mbar_init();
    ptx::prefetch_tmap(&tmap_a);
    ptx::prefetch_tmap(&tmap_b);
    if ((kEpi == EPI_STORE || kEpi == EPI_EPS) && p.tma_store) ptx::prefetch_tmap(&tmap_d);
    if (kEpi == EPI_STORE && p.tma_store && p.n % 32 != 0) ptx::prefetch_tmap(&tmap_dt);
  }
  __syncthreads();

  const int nkb = p.nkb;

  if (warp < 4) {
    // ================================ TMA producer =================================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    // resident: warp w feeds ring w with the 64-row slab w of every x tile (both walk the same load order), and warp 0
    // alone loads the y block; streaming: warp 0 feeds the one ring
    if (warp >= kRings) return;
    // The whole warp runs the loop with warp-uniform values and one elected lane issues (inside a divergent
    // `if (lane == 0)` the compiler cannot keep descriptors / barrier addresses in uniform registers).
    const uint64_t pol = ptx::policy_evict_last();
    const int ring     = kResident ? warp : 0;
    tc_producer_walk<kResident, kMasked>(
        p, nkb, blockIdx.x, gridDim.x,
        [&](int kb, uint32_t it_local, const TcItem& t) {
          if (warp != 0) return;
          ptx::mbar_wait(&bempty[kb], (it_local & 1) ^ 1);
          if (ptx::elect_one()) {
            ptx::mbar_expect_tx(&bfull[kb], TC_B_BYTES);
            ptx::tma_load_2d(b_base + kb * TC_B_BYTES, &tmap_b, &bfull[kb], kb * 64, t.n_blk * TC_BN, pol);
          }
        },
        [&](uint32_t a_it, const TcItem& t, int mt, int h, int kb) {
          const uint32_t s = a_it % kStages, ph = (a_it / kStages) & 1;
          ptx::mbar_wait(&aempty[kRings * s + ring], ph ^ 1);
          if (ptx::elect_one()) {
            // resident: the ring's 64-row slab of the tile (the x tensor map has 64-row boxes then)
            ptx::mbar_expect_tx(&afull[kRings * s + ring], kResident ? TC_A_BYTES / 2 : kStageBytes);
            ptx::tma_load_2d(a_base + s * kStageBytes + ring * (TC_A_BYTES / 2), &tmap_a, &afull[kRings * s + ring], kb * 64,
                             mt * TC_BM + 64 * ring, pol);
            if (!kResident)
              ptx::tma_load_2d(a_base + s * kStageBytes + TC_A_BYTES, &tmap_b, &afull[s], kb * 64,
                               t.n_blk * TC_BN + h * TC_HN, pol);
          }
          __syncwarp();
        });
    return;
  }

  // ================================ consumer warpgroups ================================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  const int wg     = (threadIdx.x >> 7) - 1;  // rows [64 wg, 64 wg + 64) of every x tile
  const int ct     = threadIdx.x - 128;       // 0..255 (fills the per-column terms)
  const bool lead  = (threadIdx.x & 127) == 0;  // arrives on the empty barriers for its warpgroup
  const int quad   = lane >> 2;               // fragment row inside a 16-row group (and +8)
  const int tq     = lane & 3;                // fragment column pair inside an 8-column group
  const bool has_lo = __ldg(p.has_lo) != 0u;
  const float cf    = __ldg(p.coef);
  // rows with their own exponent (prep.cuh): per-row factor on x (one multiply per row and tile), per-column factor on y
  // only when some row of y has one (rare; read straight from global memory then)
  const bool xnu = __ldg(&p.nonuni[0]) != 0u, ynu = __ldg(&p.nonuni[1]) != 0u;
  // EPI_STORE through TMA in one pass, without the diagonal or per-column scales: tc_epilogue_store_fast
  constexpr bool kFastPost = !tc_post_gram(kPost);
  const bool fast_store    = kEpi == EPI_STORE && kFastPost && p.tma_store && p.acc_mode == 0 && p.diag_off == TC_NO_DIAG && !ynu;
  // the x ring this warpgroup reads: resident, its own (its rows of every stage); streaming, the one both read
  const int ring = kResident ? wg : 0;
  // Resident: ordered MMA turns.  Both warpgroups walk the same (item, tile, half) units; warpgroup w takes its turn at
  // named barrier 4 + w before a unit's first wgmma and passes it (bar.arrive on the other's barrier) after the unit's
  // last commit, so one warpgroup's epilogue runs under the other's MMAs.  Warpgroup 0 takes the first turn; a unit
  // without MMAs (a masked NONE half) still takes and passes it, so the counts always match.  After its last item,
  // warpgroup 0 takes the turn warpgroup 1 passed last, so every arrival is matched (every CTA has an item: grid <=
  // n_items).  (Constant barrier ids: no register holds them.)
  auto take_turn = [&] { if (wg == 0) ptx::bar_sync(4, 256); else ptx::bar_sync(5, 256); };
  auto pass_turn = [&] { if (wg == 0) ptx::bar_arrive(5, 256); else ptx::bar_arrive(4, 256); };
  if (kResident && wg == 1) ptx::bar_arrive(4, 256);
  uint32_t a_it = 0, it_local = 0;
  float acc[64], crs[64];
  // EPI_EPS: the item's column counts (flushed at the next item's t_y fill and after the last item) and the warpgroup's
  // adjacency box count (tc_eps_tile)
  uint32_t* col_cnt = reinterpret_cast<uint32_t*>(smem + Carve::grp_off);
  uint32_t eps_box = 0u;
  for (int64_t item = blockIdx.x; item < p.n_items; item += gridDim.x, ++it_local) {
    const TcItem t  = tc_item(p, item);
    const int n_blk = t.n_blk, mt0 = t.mt0, mt1 = t.mt1, nh = t.nh;
    // masked: the item's last loaded tile (its y block is handed back after it); no loaded tile: the producer skipped
    // the item, and it does not count in it_local
    int mt_last = mt1 - 1;
    const uint8_t* cls = nullptr;
    if constexpr (kMasked) {
      cls     = p.mask_cls + static_cast<int64_t>(n_blk) * p.tiles_m;
      mt_last = mask_mt_last(cls, mt0, mt1);
      if (mt_last < 0) {
        if (kResident && wg == 0 && item + gridDim.x >= p.n_items) take_turn();   // warpgroup 1's last pass
        --it_local;
        continue;
      }
    }
    bool b_first = true;   // masked: this warpgroup has not waited for the item's y block yet
    // per-column epilogue terms of this y block (shared by every tile of the item)
    ptx::bar_sync(1, 256);
    if constexpr (kEpi == EPI_EPS) {
      if (p.vd != nullptr) {
        if (item != blockIdx.x) tc_eps_flush(p, col_cnt, tc_item(p, item - gridDim.x).n_blk, ct);   // the previous item's
        col_cnt[ct] = 0u;
      }
    }
    {
      const int64_t gj = static_cast<int64_t>(n_blk) * TC_BN + ct;
      // +inf: never the arg-min; NaN: never within eps
      float tv = (kEpi == EPI_EPS || kEpi == EPI_RADIUS) ? __int_as_float(0x7fffffff)
               : kEpi != EPI_STORE                     ? __int_as_float(0x7f800000) : 0.f;
      if (gj < p.n) tv = __ldg(&p.yt[gj]);
      if (kEpi == EPI_STORE && p.acc_mode >= 2) tv = 0.f;  // the t terms entered with the first K chunk
      col_tb[ct] = tv;
      if (kMasked) col_grp[ct] = gj < p.n ? __ldg(&p.mask_grp[gj]) : -1;
    }
    ptx::bar_sync(1, 256);

    for (int mt = mt0; mt < mt1; ++mt) {
      unsigned tcls = 0u;
      if constexpr (kMasked) {
        tcls = mask_cls_at(cls, mt);
        if (tcls == 0u) continue;   // not loaded
      }
      // the two tile rows this thread owns: row0 and row0 + 8
      const int64_t row0 = static_cast<int64_t>(mt) * TC_BM + 64 * wg + 16 * (warp & 3) + quad;
      float ta[2], cfr[2], thr[2], xnr[2];
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int64_t gi = row0 + 8 * j;
        float rv = 0.f, cr = cf;
        thr[j] = __int_as_float(0xff800000);  // -inf: rows outside the matrix never trigger
        if (gi < p.m) {
          if (xnu) cr *= __ldg(&p.xsc[gi]);
          if (kEpi != EPI_STORE || p.acc_mode < 2) rv = __ldg(&p.xt[gi]);
          if (kEpi == EPI_TOPK) thr[j] = __ldg(&p.knn_thr[gi]);
          if (kMinloc)  // the row's current best (an upper bound: keys only decrease)
            thr[j] = key_bound(*reinterpret_cast<volatile long long*>(&p.keys[gi]));
        }
        ta[j]  = rv;
        xnr[j] = rv;
        cfr[j] = cr;
      }
      for (int h = 0; h < nh; ++h) {
        int hcls = MASK_ALL;
        if constexpr (kMasked) {
          hcls = mask_class_of(tcls, h, wg);
          if (hcls == MASK_NONE) {
            // nothing of this warpgroup's slab is adjacent: no MMAs, no epilogue.  Stages the producer loaded (the
            // tile's, resident; the half's when the other slab needs it, streaming) are still waited for and handed
            // back by this warpgroup, and so is the y block after the item's last loaded tile.  Stage by stage, every
            // thread waits, as in a live half, and the warpgroup meets at its named barrier before the lead hands the
            // stage back.  Both matter: a warp that skipped the waits could run ahead to a later live tile and find a
            // stage's barrier a whole phase behind (try_wait.parity would pass at once, on an old tile), and a warp
            // still waiting when the lead handed the stage back could find it refilled, its barrier two phases on, and
            // wait forever.  One stage at a time: a streamed half has more k-blocks (k > 192) than the ring has stages,
            // so holding them all before handing any back would starve the producer.  (Barrier 2 + wg is free here:
            // only EPI_STORE uses it.)  Resident, the half still takes and passes its MMA turn.
            if (kResident) {
              take_turn();
              pass_turn();
            }
            if (!mask_half_loaded(kResident, tcls, h)) continue;
            if (tc_half_releases(kResident, h, nh)) {
              for (int kb = 0; kb < nkb; ++kb) {
                const uint32_t it = a_it + kb;
                ptx::mbar_wait(&afull[kRings * (it % kStages) + ring], (it / kStages) & 1);
                ptx::bar_sync(2 + wg, 128);
                if (lead) ptx::mbar_arrive(&aempty[kRings * (it % kStages) + ring]);
              }
              if (kResident && lead && mt == mt_last)
                for (int kb = 0; kb < nkb; ++kb) ptx::mbar_arrive(&bempty[kb]);
              a_it += nkb;
            }
            continue;
          }
        }
        if (!has_lo) {
#pragma unroll
          for (int c = 0; c < 64; ++c) crs[c] = 0.f;
        }
#if defined(B2D_TC_DIAG) && B2D_TC_DIAG == 3
#pragma unroll
        for (int c = 0; c < 64; ++c) acc[c] = crs[c] = 0.f;
#endif
        // Resident: both halves read the tile's nkb x stages (a_it counts (tile, kb)), and only the last half hands
        // them back.  In an earlier half the stage's phase cannot advance, so waiting on it again returns at once.
        // (the rule of tc_half_releases, written out: through the call the resident instantiations schedule differently)
        const bool release = !kResident || h == nh - 1;
        const uint32_t it0 = a_it;
        if (kResident) take_turn();   // this unit's MMA turn
        // descriptor start-address units are 16 B; inside the 128-B swizzled row of a k-block:
        //   hi k[0,16) +0, hi k[16,32) +2, lo k[0,16) +4, lo k[16,32) +6
        // One copy of the k-block loop with the cross terms and one without: a k-block's MMAs are one straight batch
        // (one wgmma group, as the release waits below count them), with no branch for the compiler to split it at.
        auto mma_unit = [&](auto with_lo) {
          constexpr bool kLo = decltype(with_lo)::value;
          for (int kb = 0; kb < nkb; ++kb) {
            const uint32_t it = it0 + kb;
            const uint32_t s = it % kStages, ph = (it / kStages) & 1;
            // (the first MMAs of the item on the resident y block wait for it; the other warpgroup has passed the turn,
            // so its hand-back of the previous y block does not wait on this one)
            if (kResident && (kMasked ? b_first : (mt == mt0 && h == 0))) ptx::mbar_wait(&bfull[kb], it_local & 1);
            ptx::mbar_wait(&afull[kRings * s + ring], ph);
            const uint64_t da = ptx::gmma_desc_sw128(ptx::smem_u32(a_base + s * kStageBytes) + wg * 64 * 128);
            const uint64_t db = ptx::gmma_desc_sw128(kResident ? ptx::smem_u32(b_base + kb * TC_B_BYTES) + h * TC_BH_BYTES
                                                               : ptx::smem_u32(a_base + s * kStageBytes + TC_A_BYTES));
            const uint32_t accum = kb > 0 ? 1u : 0u;
            ptx::fence_regs(acc);
            if (kLo) ptx::fence_regs(crs);
            ptx::wgmma_fence();
#if !defined(B2D_TC_DIAG) || B2D_TC_DIAG != 3
            if constexpr (kLo) {
              ptx::wgmma_m64n128k16_f16(crs, da + 4, db + 0, accum);  // lo0 * hi0
              ptx::wgmma_m64n128k16_f16(crs, da + 6, db + 2, 1u);     // lo1 * hi1
              ptx::wgmma_m64n128k16_f16(crs, da + 0, db + 4, 1u);     // hi0 * lo0
              ptx::wgmma_m64n128k16_f16(crs, da + 2, db + 6, 1u);     // hi1 * lo1
            }
            ptx::wgmma_m64n128k16_f16(acc, da + 0, db + 0, accum);    // hi0 * hi0
            ptx::wgmma_m64n128k16_f16(acc, da + 2, db + 2, 1u);       // hi1 * hi1
#endif
            ptx::wgmma_commit();
            ptx::fence_regs(acc);
            if (kLo) ptx::fence_regs(crs);
            if (!kResident && release && kb > 0) {  // the previous k-block's MMAs have finished reading their stage: hand it back
              ptx::wgmma_wait<1>();
              if (lead) ptx::mbar_arrive(&aempty[kRings * ((it - 1) % kStages) + ring]);
            }
          }
        };
        if (has_lo) mma_unit(std::true_type{});
        else mma_unit(std::false_type{});
        if (kResident) {
          // Every MMA of the unit is issued without waiting on any of them: the other warpgroup's turn.  Then the
          // stages go back as the MMAs that read them finish (k-block kb's group is done once at most nkb - 1 - kb
          // groups are pending; the last one after the wait for all).
          pass_turn();
          if (release)
            for (int kb = 0; kb + 1 < nkb; ++kb) {
              const int pending = nkb - 1 - kb;
              if (pending >= 3) ptx::wgmma_wait<3>();
              else if (pending == 2) ptx::wgmma_wait<2>();
              else ptx::wgmma_wait<1>();
              if (lead) ptx::mbar_arrive(&aempty[kRings * ((it0 + kb) % kStages) + ring]);
            }
        }
        ptx::wgmma_wait<0>();
        ptx::fence_regs(acc);
        ptx::fence_regs(crs);
        if (kMasked) b_first = false;
        if (release) {
          a_it = it0 + nkb;
          if (lead) {
            ptx::mbar_arrive(&aempty[kRings * ((a_it - 1) % kStages) + ring]);
            if (kResident && mt == (kMasked ? mt_last : mt1 - 1) && h == nh - 1)   // the item's last MMAs on the y block are done
              for (int kb = 0; kb < nkb; ++kb) ptx::mbar_arrive(&bempty[kb]);
          }
        }
#if defined(B2D_TC_DIAG) && B2D_TC_DIAG == 1
        {   // the accumulators must have a use, or ptxas drops the MMAs that write them: a sum stored under a condition
            // that never holds at run time (empty asm fences are not a use)
          float sum = 0.f;
#pragma unroll
          for (int c = 0; c < 64; ++c) sum += acc[c] + crs[c];
          if (p.m < 0) p.dist[threadIdx.x] = sum;
          continue;
        }
#endif
#pragma unroll
        for (int c = 0; c < 64; ++c) acc[c] += crs[c];
        const int cl0 = h * TC_HN + 2 * tq;  // this thread's first column inside the tile
        unsigned long long keep = ~0ull;
        if (kMasked && hcls == MASK_PARTIAL) keep = masked_keep64(col_grp, cl0, p.mask_bits, p.mask_groups, row0, p.m);
        if (kEpi == EPI_STORE && fast_store)
          tc_epilogue_store_fast<kPost>(acc, p, col_tb, cl0, ta, cfr);
        else
          tc_epilogue<kEpi, kPost>(acc, p, col_tb, cl0, static_cast<int64_t>(n_blk) * TC_BN + cl0, row0, ta, cfr, thr, xnr,
                                   ynu, keep);
        if (kEpi == EPI_STORE && p.tma_store)   // (this warpgroup's staging boxes: computed here, not kept live)
          tc_stage_store(acc, &tmap_d, &tmap_dt,
                         ptx::smem_u32(smem + Carve::stg_off) + wg * TC_STG_BOXES * TC_D_BOX_BYTES, lead,
                         item + gridDim.x >= p.n_items && mt == mt1 - 1 && h == nh - 1, wg,
                         static_cast<int64_t>(mt) * TC_BM + 64 * wg, static_cast<int64_t>(n_blk) * TC_BN + h * TC_HN, p);
        if constexpr (kEpi == EPI_EPS)
          tc_eps_tile(acc, p, col_cnt, h * TC_HN, row0, &tmap_d,
                      ptx::smem_u32(smem + Carve::stg_off) + wg * TC_STG_BOXES * TC_D_BOX_BYTES, lead,
                      item + gridDim.x >= p.n_items && mt == mt1 - 1 && h == nh - 1, wg,
                      static_cast<int64_t>(mt) * TC_BM + 64 * wg, static_cast<int64_t>(n_blk) * TC_BN + h * TC_HN, eps_box);
      }
    }
    if (kResident && wg == 0 && item + gridDim.x >= p.n_items) take_turn();   // warpgroup 1's last pass
  }
  if constexpr (kEpi == EPI_EPS) {
    if (p.vd != nullptr) {   // the last item's counts
      ptx::bar_sync(1, 256);
      const int64_t last_item = blockIdx.x + (p.n_items - 1 - blockIdx.x) / gridDim.x * gridDim.x;   // (grid <= n_items)
      tc_eps_flush(p, col_cnt, tc_item(p, last_item).n_blk, ct);
    }
  }
}

}  // namespace b2d
