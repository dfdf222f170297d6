// raft::cluster::kmeans_balanced: hierarchical balanced k-means (kmeans_balanced.cu; DESIGN.md section 2, K16).
//
// A stage runs balanced EM on a set of problems at once.  Problem p owns the rows [rend[p-1], rend[p]) of a row order
// (a list of operand rows, or the operand rows themselves) and the centroids [cend[p-1], cend[p]) (rend[-1] = cend[-1]
// = 0); one problem with all centroids when cend is null.  The assignment and the update are k-means' own (kmeans.cuh,
// and the EPI_MINLOC_MASKED arg-min for the fine stage); this file holds the rest:
//   kb_valid_kernel   label 0 for a row whose elements are all finite, -1 otherwise, and the count of finite rows
//   kb_init_kernel    centroid t of a problem with R rows and C centroids <- its row floor(t R / C) (zeros when R = 0)
//   kb_adjust_kernel  a centroid of size s < a / 4 (a = R / C) moves towards a uniformly drawn donor row of its problem
//                     whose cluster has size >= a: c <- (w c + x_d) / (w + 1), w = min(s, 7)
//   kb_alloc_kernel   n_clusters split over the mesoclusters by largest remainders, at least one per non-empty one
//   kb_gather_kernel  the rows sorted by mesocluster, copied into the workspace (zero rows past the finite ones)
//   kb_bits_kernel    the adjacency bits of the masked arg-min straight from the mesoclusters' sorted row ranges
//   kb_sizes_kernel   cluster sizes from the counting sort's cursors
// Random numbers: one Philox4x32-10 block per (seed, stage, iteration, centroid); integer atomics only.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <curand_kernel.h>

#include "kmeans_types.cuh"
#include "tc_params.cuh"   // masked_group_of

namespace b2d {

constexpr int kKbMaxWeight = 7;   // the adjust step's weight cap of the old centroid

// The problems of one stage (see the top of the file)
struct KbProblems {
  const float* x;     // operand rows
  int64_t ldx;
  const int* rows;    // position in the row order -> operand row (null: the identity)
  const int* rend;    // [P] ends of the problems' rows in the row order
  const int* cend;    // [P] ends of their centroids (null: one problem holding all nc centroids)
  int P;
  int nc;
};

// problem of centroid j, and its row range [r0, r1) and centroid range [c0, c1)
__device__ __forceinline__ int kb_problem(const KbProblems& q, int j, int64_t& r0, int64_t& r1, int64_t& c0, int64_t& c1)
{
  const int p = q.cend ? masked_group_of(q.cend, q.P, j) : 0;
  r0 = p > 0 ? q.rend[p - 1] : 0;
  r1 = q.rend[p];
  c0 = q.cend ? (p > 0 ? q.cend[p - 1] : 0) : 0;
  c1 = q.cend ? q.cend[p] : q.nc;
  return p;
}

__device__ __forceinline__ int64_t kb_row(const KbProblems& q, int64_t pos) { return q.rows ? q.rows[pos] : pos; }

// one warp per row: lab[i] = 0 when every element of row i is finite, else -1; *count += the finite rows
__global__ void __launch_bounds__(256) kb_valid_kernel(const float* x, int64_t ldx, int k, int64_t m, int* lab, int* count)
{
  const int lane = threadIdx.x & 31;
  const int64_t i = static_cast<int64_t>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  bool ok = true;
  if (i < m)
    for (int t = lane; t < k; t += 32) ok &= isfinite(__ldg(&x[i * ldx + t]));
  ok = __all_sync(0xffffffffu, ok);
  if (i < m && lane == 0) {
    lab[i] = ok ? 0 : -1;
    if (ok) atomicAdd(count, 1);
  }
}

// one 128-thread block per centroid
__global__ void kb_init_kernel(KbProblems q, float* c, int k)
{
  const int j = blockIdx.x;
  int64_t r0, r1, c0, c1;
  kb_problem(q, j, r0, r1, c0, c1);
  float* out = c + static_cast<int64_t>(j) * k;
  if (r1 <= r0) {
    for (int col = threadIdx.x; col < k; col += blockDim.x) out[col] = 0.f;
    return;
  }
  const int64_t row = kb_row(q, r0 + (j - c0) * (r1 - r0) / (c1 - c0));
  for (int col = threadIdx.x; col < k; col += blockDim.x) out[col] = q.x[row * q.ldx + col];
}

// The donor position of centroid j: uniform in [0, R) from the first two words of Philox4x32-10 with counter
// (j, iteration, stage, 0) and key (seed low, seed high): floor(((w0 << 32) | w1) * R / 2^64)
__device__ __forceinline__ int64_t kb_draw(unsigned long long seed, int stage, int it, int j, int64_t R)
{
  const uint4 r = curand_Philox4x32_10(make_uint4(static_cast<unsigned>(j), static_cast<unsigned>(it),
                                                  static_cast<unsigned>(stage), 0u),
                                       make_uint2(static_cast<unsigned>(seed), static_cast<unsigned>(seed >> 32)));
  const unsigned long long u = (static_cast<unsigned long long>(r.x) << 32) | r.y;
  return static_cast<int64_t>(__umul64hi(u, static_cast<unsigned long long>(R)));
}

// One 128-thread block per centroid, after the update of iteration `it`: labels are in operand-row order, the sizes are
// the counting sort's cluster ranges (cur, nblk: km_cluster_range).  Sizes are compared with a = R / C in integers.
__global__ void kb_adjust_kernel(KbProblems q, const int* labels, const unsigned* cur, int64_t nblk, float* c, int k,
                                 unsigned long long seed, int stage, int it)
{
  const int j = blockIdx.x;
  int64_t r0, r1, c0, c1;
  kb_problem(q, j, r0, r1, c0, c1);
  const int64_t R = r1 - r0, C = c1 - c0;
  int64_t cs, ce;
  km_cluster_range(cur, nblk, j, cs, ce);
  const int64_t s = ce - cs;
  if (R <= 0 || s > (R - 1) / (4 * C)) return;   // s < a / 4, i.e. 4 s C < R
  const int64_t d = kb_row(q, r0 + kb_draw(seed, stage, it, j, R));
  const int ld = labels[d];
  if (ld < 0) return;
  km_cluster_range(cur, nblk, ld, cs, ce);
  if (ce - cs < (R + C - 1) / C) return;          // the donor's cluster has size >= a
  const double w = static_cast<double>(s < kKbMaxWeight ? s : kKbMaxWeight);
  float* out = c + static_cast<int64_t>(j) * k;
  for (int col = threadIdx.x; col < k; col += blockDim.x)
    out[col] = static_cast<float>((w * static_cast<double>(out[col]) + static_cast<double>(q.x[d * q.ldx + col])) / (w + 1.0));
}

// One CTA of kKbAllocThreads.  Mesocluster g holds S_g rows (the counting sort's ranges, R = sum S_g rows in all);
// it gets a_g of the nc fine clusters: floor(nc S_g / R), plus one for the nc - sum floor(...) largest remainders
// nc S_g mod R (ties: the lower g); then every non-empty mesocluster left with none takes one from the mesocluster of
// the largest a / S holding at least two (ties: the lower g).  Writes the row ends E [G] and the centroid ends F [G].
constexpr int kKbAllocThreads = 1024;
__global__ void __launch_bounds__(kKbAllocThreads) kb_alloc_kernel(const unsigned* cur, int64_t nblk, int G, int64_t nc,
                                                                   int* a, int* E, int* F)
{
  __shared__ long long s_left;
  int64_t R = 0;   // every thread sums the sizes in the same order
  for (int g = 0; g < G; ++g) {
    int64_t cs, ce;
    km_cluster_range(cur, nblk, g, cs, ce);
    R += ce - cs;
  }
  auto size = [&](int g) { int64_t cs, ce; km_cluster_range(cur, nblk, g, cs, ce); return ce - cs; };
  if (threadIdx.x == 0) s_left = nc;
  __syncthreads();
  for (int g = threadIdx.x; g < G; g += kKbAllocThreads) {
    const int64_t f = R > 0 ? nc * size(g) / R : (g == 0 ? nc : 0);
    a[g] = static_cast<int>(f);
    atomicAdd(reinterpret_cast<unsigned long long*>(&s_left), static_cast<unsigned long long>(-f));
  }
  __syncthreads();
  const int64_t left = s_left;
  if (R > 0)
    for (int g = threadIdx.x; g < G; g += kKbAllocThreads) {
      const int64_t rg = nc * size(g) % R;
      int64_t rank = 0;
      for (int h = 0; h < G && rank < left; ++h) {
        const int64_t rh = nc * size(h) % R;
        rank += (rh > rg || (rh == rg && h < g)) ? 1 : 0;
      }
      if (rank < left) a[g] += 1;
    }
  __syncthreads();
  if (threadIdx.x != 0) return;
  for (int g = 0; g < G; ++g) {
    if (a[g] > 0 || size(g) == 0) continue;
    int best = -1;
    for (int h = 0; h < G; ++h)
      if (a[h] >= 2 && (best < 0 || static_cast<int64_t>(a[h]) * size(best) > static_cast<int64_t>(a[best]) * size(h)))
        best = h;
    if (best < 0) break;   // (cannot happen: G <= nc)
    a[best] -= 1;
    a[g] = 1;
  }
  int64_t e = 0, f = 0;
  for (int g = 0; g < G; ++g) {
    e += size(g);
    f += a[g];
    E[g] = static_cast<int>(e);
    F[g] = static_cast<int>(f);
  }
}

// One 128-thread block per sorted position p: xs[p] = x[perm[p]] for the first E[G-1] positions, zeros after them.
// km_gather_rows_kernel would read perm past the finite rows, where the counting sort wrote nothing; the zero rows keep
// the operand preparation of xs from reading stale workspace.  (At small k most of the block idles; the gather runs
// once per fit.)
__global__ void kb_gather_kernel(const float* x, int64_t ldx, int k, const int* perm, const int* E, int G, float* xs)
{
  const int64_t p = blockIdx.x;
  float* out = xs + p * k;
  if (p >= E[G - 1]) {
    for (int col = threadIdx.x; col < k; col += blockDim.x) out[col] = 0.f;
    return;
  }
  const int64_t r = perm[p];
  for (int col = threadIdx.x; col < k; col += blockDim.x) out[col] = x[r * ldx + col];
}

// bits[w][g] (w < ceil(m / 32)): bit r set when the sorted row 32 w + r lies in [E[g-1], E[g]).  Grid-stride over the
// ceil(m / 32) G words, so any grid writes them all.
__global__ void kb_bits_kernel(unsigned* bits, const int* E, int64_t G, int64_t m)
{
  const int64_t nw = (m + 31) / 32 * G;
  for (int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; t < nw;
       t += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t w = t / G, g = t % G;
    const int64_t lo = max(g > 0 ? static_cast<int64_t>(E[g - 1]) : 0, 32 * w), hi = min(static_cast<int64_t>(E[g]), 32 * w + 32);
    unsigned word = 0u;
    if (hi > lo) {
      const int a = static_cast<int>(lo - 32 * w), n = static_cast<int>(hi - lo);
      word = (n >= 32 ? ~0u : ((1u << n) - 1u)) << a;
    }
    bits[t] = word;
  }
}

__global__ void kb_sizes_kernel(const unsigned* cur, int64_t nblk, int nc, int* sizes)
{
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= nc) return;
  int64_t cs, ce;
  km_cluster_range(cur, nblk, j, cs, ce);
  sizes[j] = static_cast<int>(ce - cs);
}

}  // namespace b2d
