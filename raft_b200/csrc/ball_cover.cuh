// Kernels of the random ball cover (ball_cover.cu): exact kNN and epsilon queries for 2-D and 3-D points, SIMT, and the
// one ball walk (bc_walk) they, DBSCAN's ball-cover fit (dbscan.cuh) and the EMST (single_linkage_rbc.cuh) run on.  The
// build's kernels are in ball_cover_build.cuh.
//
// A pair's value is fixed bit for bit: s = ((q0-p0)^2 + (q1-p1)^2) + (q2-p2)^2, every operation rounded separately
// (bc_s), and the distance f = s (L2Unexpanded) or sqrt(s) (L2SqrtUnexpanded).  The queries prune whole balls and ball
// members by the triangle inequality on the TRUE distances of the fp32 points, bounded from the rounded s values with the
// margin below (DESIGN.md K19 derives it); every bound is formed with directed rounding, so a pruned row provably has
// f(q, p) above the current k-th value (or above eps) and can never order before it.
//
//   D^2 (1 - 6u) - A  <=  s  <=  D^2 (1 + 6u) + A,   u = 2^-24, A = 2^-148 >= 3 squares' underflow (3 * 2^-150),
//   s = inf only if D^2 >= 2^127 (an overflowing difference, square or sum).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

#include "ball_cover_types.cuh"
#include "nn_key.cuh"

namespace b2d {

constexpr float BC_INF = __builtin_huge_valf();
constexpr float BC_A   = 0x1p-148f;         // absolute slack of s
constexpr float BC_UP  = 1.f + 0x1p-21f;    // >= 1 + 6u, >= 1 / (1 - 6u) and >= 1 / (1 - u)^2
constexpr float BC_DN  = 1.f - 0x1p-21f;    // <= 1 / (1 + 6u)
constexpr float BC_CAP = 0x1p126f;          // a threshold above this cannot be compared with an s of inf

template <int D>
__device__ __forceinline__ float bc_s(const float* q, const float* p)
{
  const float t0 = __fsub_rn(q[0], p[0]), t1 = __fsub_rn(q[1], p[1]);
  float s = __fadd_rn(__fmul_rn(t0, t0), __fmul_rn(t1, t1));
  if (D == 3) {
    const float t2 = __fsub_rn(q[2], p[2]);
    s = __fadd_rn(s, __fmul_rn(t2, t2));
  }
  return s;
}

// lower / upper bound of the true distance of a pair whose s is s
__device__ __forceinline__ float bc_dlo(float s)
{
  if (s == BC_INF) return 0x1p63f;
  return __fsqrt_rd(__fmul_rd(fmaxf(__fsub_rd(s, BC_A), 0.f), BC_DN));
}
__device__ __forceinline__ float bc_dhi(float s) { return __fsqrt_ru(__fmul_ru(__fadd_ru(s, BC_A), BC_UP)); }
// an s above bc_above(t) proves the true distance above t
__device__ __forceinline__ float bc_above(float t)
{
  const float v = __fadd_ru(__fmul_ru(__fmul_ru(t, t), BC_UP), BC_A);
  return v <= BC_CAP ? v : BC_INF;
}
// an s below bc_below(g) proves the true distance below g
__device__ __forceinline__ float bc_below(float g) { return g > 0.f ? __fsub_rd(__fmul_rd(__fmul_rd(g, g), BC_DN), BC_A) : -1.f; }
// the largest true distance of a pair whose distance f is at most v
__device__ __forceinline__ float bc_dmax(float v, int root) { return bc_dhi(root ? __fmul_ru(__fmul_ru(v, v), BC_UP) : v); }

// The member window of a ball for a query at s = sq from its landmark and a distance bound dmax: members with s outside
// [*lo, *hi] are farther than dmax from the query (|D(q, L) - D(L, p)| > dmax).
__device__ __forceinline__ void bc_window(float sq, float dmax, float* lo, float* hi)
{
  *lo = bc_below(__fsub_rd(bc_dlo(sq), dmax));
  *hi = bc_above(__fadd_ru(bc_dhi(sq), dmax));
}

// the ball lies farther than dmax from a query at s = sq from its landmark
__device__ __forceinline__ bool bc_ball_out(float sq, float rhi, float dmax) { return sq > bc_above(__fadd_ru(rhi, dmax)); }

// first position in [lo, hi) whose rl is not below t (upper: above t)
__device__ __forceinline__ int bc_search(const float* rl, int lo, int hi, float t, bool upper)
{
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    const float r = rl[mid];
    if (upper ? !(r > t) : r < t) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// ------------------------------------------------------------------------------------------
// queries

// The landmarks and their rhi in shared memory when they fit (smem), else read where they are.
template <int D>
__device__ __forceinline__ void bc_stage(const BcIndex& ix, int nl, bool smem, const float** lm, const float** rhi)
{
  extern __shared__ float bc_sm[];
  *lm  = ix.lm;
  *rhi = ix.rhi;
  if (!smem) return;
  for (int e = threadIdx.x; e < nl * D; e += blockDim.x) bc_sm[e] = ix.lm[e];
  for (int e = threadIdx.x; e < nl; e += blockDim.x) bc_sm[nl * D + e] = ix.rhi[e];
  __syncthreads();
  *lm  = bc_sm;
  *rhi = bc_sm + nl * D;
}

// the query point at p; false: a NaN coordinate (the query has no neighbour)
template <int D>
__device__ __forceinline__ bool bc_query(const float* p, float (&q)[D])
{
  bool nan = false;
  for (int c = 0; c < D; ++c) {
    q[c] = p[c];
    nan  = nan || isnan(q[c]);
  }
  return !nan;
}

// The ball loop of every walk, for one query q (not NaN) of a warp: the balls in index order, every admitted non-empty
// ball that bc_ball_out does not rule out at the bound of the moment it is reached, then the non-finite rows [off[nl], n)
// with sq = 0 (nothing is pruned there).  The walker v gives admit(j) (the ball filter), dmax (the distance bound) and
// scan(lo, hi, sq), which visits the positions [lo, hi) of a ball at s = sq from the query and returns true (the same on
// every lane) to end the walk.  Shrinking: v's bound decreases as it scans (kNN, EMST), so the nearest admitted ball goes
// first to tighten it early, and each ball is tested again when it is reached; a fixed bound (epsilon) needs neither.
// The kNN, epsilon, DBSCAN (dbscan.cuh) and EMST (single_linkage_rbc.cuh) walks all run on it, so the ball pruning has
// one definition.
template <int D, bool Shrinking, typename Walker>
__device__ __forceinline__ void bc_walk(const BcIndex& ix, int n, int nl, const float* lm, const float* rhi, const float* q,
                                        int lane, Walker& v)
{
  int b0 = -1;
  if (Shrinking) {
    long long near = KEY_EMPTY;
    for (int j = lane; j < nl; j += 32)
      if (rhi[j] >= 0.f && v.admit(j)) near = min(near, key_pack(bc_s<D>(q, lm + j * D), j));
    for (int o = 16; o > 0; o >>= 1) near = min(near, __shfl_xor_sync(0xffffffffu, near, o));
    b0 = near == KEY_EMPTY ? -1 : static_cast<int>(key_index(near));
    if (b0 >= 0 && v.scan(ix.off[b0], ix.off[b0 + 1], key_dist(near))) return;
  }
  for (int base = 0; base < nl; base += 32) {
    const int j = base + lane;
    float s     = 0.f;
    bool want   = false;
    if (j < nl && j != b0 && rhi[j] >= 0.f && v.admit(j)) {
      s    = bc_s<D>(q, lm + j * D);
      want = !bc_ball_out(s, rhi[j], v.dmax);
    }
    unsigned mask = __ballot_sync(0xffffffffu, want);
    while (mask) {
      const int src  = __ffs(mask) - 1;
      mask          &= mask - 1;
      const float sj = __shfl_sync(0xffffffffu, s, src);
      const int b    = base + src;
      if ((!Shrinking || !bc_ball_out(sj, rhi[b], v.dmax)) && v.scan(ix.off[b], ix.off[b + 1], sj)) return;
    }
  }
  v.scan(ix.off[nl], n, 0.f);
}

// A warp's sorted list of the 64 best keys so far: lane l holds slots l (a0) and l + 32 (a1).
struct BcTopK {
  long long a0 = KEY_EMPTY, a1 = KEY_EMPTY;

  __device__ __forceinline__ long long slot(int j) const
  {
    return j < 32 ? __shfl_sync(0xffffffffu, a0, j) : __shfl_sync(0xffffffffu, a1, j - 32);
  }
  // insert c (warp-uniform, not in the list): every slot at or after c's place takes its predecessor
  __device__ __forceinline__ void insert(long long c, int lane)
  {
    long long u0       = __shfl_up_sync(0xffffffffu, a0, 1);
    long long u1       = __shfl_up_sync(0xffffffffu, a1, 1);
    const long long l0 = __shfl_sync(0xffffffffu, a0, 31);
    if (lane == 0) { u0 = KEY_EMPTY; u1 = l0; }
    const bool first0 = lane == 0 || u0 < c;
    a0 = a0 < c ? a0 : (first0 ? c : u0);
    a1 = a1 < c ? a1 : (u1 < c ? c : u1);
  }
};

// The kNN walker of one query of a warp: the list, its k-th key and the distance bound that k-th key gives.
template <int D>
struct BcKnn {
  const BcIndex& ix;
  const float* q;
  int k, root, lane;
  BcTopK list;
  long long kth = KEY_EMPTY;
  float dmax    = BC_INF;

  __device__ __forceinline__ bool admit(int) const { return true; }

  // the members [lo, hi) of one ball at s = sq from the query into the list, in a window that shrinks with the k-th key
  __device__ __forceinline__ bool scan(int lo, int hi, float sq)
  {
    float wlo, whi;
    bc_window(sq, dmax, &wlo, &whi);
    for (int p = bc_search(ix.rl, lo, hi, wlo, false); p < hi; p += 32) {
      const int i    = p + lane;
      const float r  = i < hi ? ix.rl[i] : BC_INF;
      const bool out = i < hi && r > whi;
      long long key  = KEY_EMPTY;
      if (i < hi && !out && r >= wlo) {
        const float s = bc_s<D>(q, ix.pts + static_cast<int64_t>(i) * D);
        const float f = root ? __fsqrt_rn(s) : s;
        if (f == f) key = key_pack(f, ix.ids[i]);
      }
      unsigned mask = __ballot_sync(0xffffffffu, key < kth);
      if (mask) {
        do {
          const int src     = __ffs(mask) - 1;
          mask             &= mask - 1;
          const long long c = __shfl_sync(0xffffffffu, key, src);
          if (c < kth) {
            list.insert(c, lane);
            kth = list.slot(k - 1);
          }
        } while (mask);
        if (kth != KEY_EMPTY) {
          dmax = bc_dmax(key_dist(kth), root);
          bc_window(sq, dmax, &wlo, &whi);
        }
      }
      if (__any_sync(0xffffffffu, out)) break;
    }
    return false;
  }
};

// One warp per query: bc_walk with the nearest ball first, which seeds the list.
template <int D>
__global__ void __launch_bounds__(kBcWarps * 32) bc_knn_kernel(BcIndex ix, int n, int nl, int root, const float* qs,
                                                               int64_t ldq, int m, int k, int64_t* out_idx,
                                                               float* out_dist, int smem)
{
  const float *lm, *rhi;
  bc_stage<D>(ix, nl, smem, &lm, &rhi);
  const int lane = threadIdx.x & 31;
  const int qi   = blockIdx.x * kBcWarps + (threadIdx.x >> 5);
  if (qi >= m) return;
  float q[D];
  BcKnn<D> st{ix, q, k, root, lane};
  if (bc_query<D>(qs + static_cast<int64_t>(qi) * ldq, q)) bc_walk<D, true>(ix, n, nl, lm, rhi, q, lane, st);
  for (int j = lane; j < k; j += 32) {
    const long long key = j < 32 ? st.list.a0 : st.list.a1;
    const int64_t o     = static_cast<int64_t>(qi) * k + j;
    out_idx[o]          = key == KEY_EMPTY ? -1 : key_index(key);
    out_dist[o]         = key == KEY_EMPTY ? BC_INF : key_dist(key);
  }
}

// The epsilon walker: the fixed bound of eps, and in each ball the member window by two binary searches, every position
// of which is measured.
template <int D, typename Act>
struct BcEpsWalk {
  const BcIndex& ix;
  const float* q;
  int root;
  float eps;
  int lane;
  float dmax;
  Act& act;

  __device__ __forceinline__ bool admit(int) const { return true; }

  __device__ __forceinline__ bool scan(int lo, int hi, float sq)
  {
    float wlo, whi;
    bc_window(sq, dmax, &wlo, &whi);
    lo = bc_search(ix.rl, lo, hi, wlo, false);
    hi = bc_search(ix.rl, lo, hi, whi, true);
    for (int p = lo; p < hi; p += 32) {
      const int i = p + lane;
      float f     = BC_INF;
      bool hit    = false;
      if (i < hi) {
        const float s = bc_s<D>(q, ix.pts + static_cast<int64_t>(i) * D);
        f             = root ? __fsqrt_rn(s) : s;
        hit           = f <= eps;
      }
      if (act(i, f, hit)) return true;
    }
    return false;
  }
};

// The epsilon walk of one query q (not NaN) of a warp, bc_walk with the fixed bound of eps.  Every step of 32 positions calls
// act(i, f, hit) on all lanes: i = the lane's position, f = its distance and hit = (f <= eps) for a position inside the
// window, else hit = false.  act returns true (the same on every lane) to end the walk there.  The epsilon queries and
// DBSCAN's walks (dbscan.cuh) share it.
template <int D, typename Act>
__device__ __forceinline__ void bc_eps_walk(const BcIndex& ix, int n, int nl, const float* lm, const float* rhi,
                                            const float* q, int root, float eps, int lane, Act&& act)
{
  BcEpsWalk<D, Act> w{ix, q, root, eps, lane, bc_dmax(eps, root), act};
  bc_walk<D, false>(ix, n, nl, lm, rhi, q, lane, w);
}

// Epsilon queries, one warp per query, by bc_eps_walk.  Count (keys == nullptr): indptr[qi + 1] = the query's pairs
// (indptr[0] = 0).  Fill: the pairs as packed keys into keys[indptr[qi], min(indptr[qi + 1], nnz)).
template <int D>
__global__ void __launch_bounds__(kBcWarps * 32) bc_eps_kernel(BcIndex ix, int n, int nl, int root, const float* qs,
                                                               int64_t ldq, int m, float eps, int64_t* indptr,
                                                               long long* keys, int64_t nnz, int smem)
{
  const float *lm, *rhi;
  bc_stage<D>(ix, nl, smem, &lm, &rhi);
  const int lane = threadIdx.x & 31;
  const int qi   = blockIdx.x * kBcWarps + (threadIdx.x >> 5);
  if (qi >= m) return;
  float q[D];
  const bool ok = bc_query<D>(qs + static_cast<int64_t>(qi) * ldq, q);
  int64_t at = 0, end = 0;
  if (keys) {
    at  = indptr[qi];
    end = min(indptr[qi + 1], nnz);
  }
  int64_t cnt = 0;
  if (ok)
    bc_eps_walk<D>(ix, n, nl, lm, rhi, q, root, eps, lane, [&](int i, float f, bool hit) {
      const unsigned mask = __ballot_sync(0xffffffffu, hit);
      if (keys) {
        const int64_t e = at + cnt + __popc(mask & ((1u << lane) - 1u));
        if (hit && e < end) keys[e] = key_pack(f, ix.ids[i]);
      }
      cnt += __popc(mask);
      return false;
    });
  if (!keys && lane == 0) {
    indptr[qi + 1] = cnt;
    if (qi == 0) indptr[0] = 0;
  }
}

}  // namespace b2d
