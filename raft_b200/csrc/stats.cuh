// Callers of the distance path (SURVEY.md 8(f3)): silhouette and trustworthiness scores on top of the
// pairwise / kNN engine.
//
// Semantics follow raft::stats::silhouette_score (cpp/include/raft/stats/detail/silhouette_score.cuh:
// 186-328): a(i) = mean distance to the other members of i's cluster (-1 marks a singleton cluster ->
// score 0), b(i) = min over the other non-empty clusters of the mean distance to that cluster,
// s(i) = 0 if a == b, (b - a) / max(a, b) otherwise; result = mean of s.  The reference materialises
// the n x n matrix (its batched variant, detail/batched/silhouette_score.cuh:213-243, works in chunks);
// here the database side is a copy of X with rows grouped by label, so the per-cluster sums of a row
// are sums over contiguous column segments of a [chunk x n] slab that is produced by the engine and
// consumed straight away.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

namespace b2d {

__global__ void sil_count_kernel(const int* labels, int* counts, int64_t n, int n_labels, unsigned* bad)
{
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int l = labels[i];
  if (l < 0 || l >= n_labels) { *bad = 1u; return; }
  atomicAdd(&counts[l], 1);
}

// exclusive scan of the label counts (n_labels is small next to n: one block)
__global__ void sil_scan_kernel(const int* counts, int* offsets, int* cursor, int n_labels)
{
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    int run = 0;
    for (int l = 0; l < n_labels; ++l) { offsets[l] = run; cursor[l] = run; run += counts[l]; }
    offsets[n_labels] = run;
  }
}

// y_sorted[pos] = x[i] with pos inside the segment of labels[i] (order inside a segment is irrelevant)
__global__ void sil_gather_kernel(const float* x, int64_t ldx, const int* labels, int* cursor, float* ys, int* where,
                                  int64_t n, int k, int n_labels)
{
  const int lane    = threadIdx.x & 31;
  const int64_t row = static_cast<int64_t>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= n) return;
  const int l = labels[row];
  if (l < 0 || l >= n_labels) return;
  int pos = 0;
  if (lane == 0) pos = atomicAdd(&cursor[l], 1);
  pos = __shfl_sync(0xffffffffu, pos, 0);
  if (lane == 0) where[row] = pos;
  for (int t = lane; t < k; t += 32) ys[static_cast<int64_t>(pos) * k + t] = x[row * ldx + t];
}

// one block per row of the slab: per-cluster sums over the column segments, then a, b, s
__global__ void __launch_bounds__(256) sil_row_kernel(const float* slab, int64_t ld, int64_t row0, int64_t rows,
                                                      const int* labels, const int* counts, const int* offsets,
                                                      const int* where, int n_labels, float* per_sample, double* total)
{
  extern __shared__ float sums[];  // [n_labels]
  const int64_t r = blockIdx.x;
  if (r >= rows) return;
  const float* d = slab + r * ld;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  for (int l = threadIdx.x; l < n_labels; l += blockDim.x) sums[l] = 0.f;
  __syncthreads();
  for (int l = 0; l < n_labels; ++l) {
    // every warp takes an equal slice of every segment: balanced for 2 clusters as for 2000
    const int64_t a = offsets[l], b = offsets[l + 1], len = b - a;
    const int64_t lo = a + len * warp / nw, hi = a + len * (warp + 1) / nw;
    float acc = 0.f;
    for (int64_t j = lo + lane; j < hi; j += 32) acc += d[j];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0 && hi > lo) atomicAdd(&sums[l], acc);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    const int own = labels[row0 + r];
    float s = 0.f;
    if (own < 0 || own >= n_labels) {
      s = __int_as_float(0x7fc00000);  // invalid label: NaN (see sil_finish_kernel)
    } else if (counts[own] > 1) {
      // the sample's distance to itself is 0 by definition (the reference gets that from x == y aliasing;
      // here the column side is a permuted copy, so whatever rounding left in d(i, i) is taken out)
      const float av = (sums[own] - d[where[row0 + r]]) / static_cast<float>(counts[own] - 1);
      float bv       = 3.402823466e38f;
      for (int l = 0; l < n_labels; ++l)
        if (l != own && counts[l] > 0) bv = fminf(bv, sums[l] / static_cast<float>(counts[l]));
      if (!((av == 0.f && bv == 0.f) || av == bv)) s = av > bv ? (bv - av) / av : (bv - av) / bv;
    }
    if (per_sample) per_sample[row0 + r] = s;
    atomicAdd(total, static_cast<double>(s));
  }
}

// labels outside [0, n_labels) were flagged by sil_count_kernel: the score is NaN then (device-side validation,
// the call never synchronises).  So it is when fewer than two clusters are non-empty: every b is FLT_MAX there and
// s ~ 1 would score a clustering that is not one.
__global__ void sil_finish_kernel(const double* total, float* score, int64_t n, const unsigned* bad, const int* counts,
                                  int n_labels)
{
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    int present = 0;
    for (int l = 0; l < n_labels; ++l) present += counts[l] > 0;
    *score = *bad || present < 2 ? __int_as_float(0x7fc00000) : static_cast<float>(*total / static_cast<double>(n));
  }
}

// ---------------------------------------------------------------------------------------------
// Trustworthiness (raft::stats::trustworthiness_score, cpp/include/raft/stats/detail/
// trustworthiness_score.cuh:113-211): for every sample i and each of its n_neighbors nearest
// neighbours j != i in the EMBEDDED space (from a kNN list of n_neighbors + 1 that normally holds i itself),
// r(i, j) = position of j when the samples are ordered by their
// ORIGINAL-space distance from i (i itself first), penalty max(0, r - n_neighbors);
// score = 1 - 2 / (n k (2n - 3k - 1)) * sum of the penalties.  The reference sorts every row of the
// original-space distance matrix (sort_cols_per_row + a lookup table); only k + 1 ranks per row are
// needed, so here a rank is a COUNT: the entries of the row that precede d(i, j) -- one block per row
// of the slab, ballots over 32 columns at a time, batches that cannot precede any of the row's
// thresholds skipped.
__global__ void __launch_bounds__(256) trust_rank_kernel(const float* slab, int64_t ld, int64_t row0, int64_t n,
                                                         const int64_t* emb_idx, int kk1, int n_neighbors,
                                                         unsigned long long* penalty)
{
  __shared__ float thr[64];
  __shared__ int nbr[64];
  __shared__ unsigned cnt[64];
  __shared__ float tmax_s;
  const int64_t row = row0 + blockIdx.x;
  const float* d    = slab + static_cast<int64_t>(blockIdx.x) * ld;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  if (threadIdx.x < 64) {
    float t = __int_as_float(0xff800000);  // -inf: nothing precedes (self entries, padding)
    int j   = -1;
    if (threadIdx.x < kk1) {
      const int64_t e = emb_idx[row * kk1 + threadIdx.x];
      if (e >= 0 && e < n && e != row) { j = static_cast<int>(e); t = d[e]; }
    }
    thr[threadIdx.x] = t;
    nbr[threadIdx.x] = j;
    cnt[threadIdx.x] = 0u;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    // exactly n_neighbors neighbours per sample: the list is ascending by (distance, index) (knn_finalize_kernel), so a
    // sample missing from its own list (n_neighbors + 1 coincident rows of smaller index, or a rounded d(i, i) > 0
    // above a neighbour's distance) drops the last entry, the farthest
    bool self = false;
    for (int q = 0; q < kk1; ++q) self |= emb_idx[row * kk1 + q] == row;
    if (!self) { thr[kk1 - 1] = __int_as_float(0xff800000); nbr[kk1 - 1] = -1; }
    float tm = __int_as_float(0xff800000);
    for (int q = 0; q < kk1; ++q) tm = fmaxf(tm, thr[q]);
    tmax_s = tm;
  }
  __syncthreads();
  const float tmax = tmax_s;
  unsigned c0 = 0, c1 = 0;  // lane q & 31 counts for neighbour q (q < 32 -> c0, else c1)
  for (int64_t l0 = static_cast<int64_t>(warp) * 32; l0 < n; l0 += static_cast<int64_t>(nw) * 32) {
    const int64_t l  = l0 + lane;
    const bool valid = l < n && l != row;
    const float v    = valid ? d[l] : 0.f;
    if (!__any_sync(0xffffffffu, valid && v <= tmax)) continue;
    for (int q = 0; q < kk1; ++q) {
      const float t = thr[q];
      const int j   = nbr[q];
      const bool before = valid && l != j && (v < t || (v == t && l < j));
      const unsigned b  = __ballot_sync(0xffffffffu, before);
      if (lane == (q & 31)) { if (q < 32) c0 += __popc(b); else c1 += __popc(b); }
    }
  }
  if (lane < kk1 && c0) atomicAdd(&cnt[lane], c0);
  if (lane + 32 < kk1 && c1) atomicAdd(&cnt[lane + 32], c1);
  __syncthreads();
  if (threadIdx.x < kk1 && nbr[threadIdx.x] >= 0) {
    const long long r = static_cast<long long>(cnt[threadIdx.x]) + 1;  // the sample itself comes first
    if (r > n_neighbors) atomicAdd(penalty, static_cast<unsigned long long>(r - n_neighbors));
  }
}

// score = 1 - 2 / (n k (2n - 3k - 1)) * sum of the penalties, written to DEVICE memory
__global__ void trust_finish_kernel(const unsigned long long* penalty, double* score, int64_t n, int n_neighbors)
{
  const double nn = static_cast<double>(n), kk = static_cast<double>(n_neighbors);
  *score = 1.0 - (2.0 / ((nn * kk) * ((2.0 * nn) - (3.0 * kk) - 1.0))) * static_cast<double>(*penalty);
}

}  // namespace b2d
