// DBSCAN (DESIGN.md K14) on the epsilon neighbourhood of the tensor kernel (EPI_EPS).  The adjacency A of one batch of
// columns [s, s + w) arrives as bytes adj [m][ld] (row i, column s + c at adj[i * ld + c]); the degrees come from the
// count-only pass.  Core points are joined by a lock-free union-find over the set bytes whose two ends are core, border
// points take the smallest root among the core columns of their row.
//   db_core_kernel      degrees -> core flags, parent[i] = i (core) or -1, border[i] = INT_MAX
//   db_link_kernel      per batch: every set byte (i, s + c) with both ends core unites their trees
//   db_compress_kernel  parent[i] = root of i (a find that only reads), root flags
//   db_border_kernel    per batch: every non-core row i, atomicMin of the smallest root among its core columns
//   db_label_kernel     labels, core_sample_indices and n_clusters from the two scanned flag arrays
// The union hooks the larger root under the smaller (CAS on parent), so the root of a component is its smallest core
// row whatever the interleaving; every atomic is an integer CAS or atomicMin, and the results do not depend on order.
// The ball-cover fit's three walks (db_rbc_*) take the place of the EPI_EPS batches for 2-D and 3-D points.
#pragma once
#include <cuda_runtime.h>
#include <climits>
#include <cstdint>

#include "ball_cover.cuh"

namespace b2d {

constexpr int kDbThreads = 256;

// row i's core flag from its degree: column j of batch t = j / b was counted at deg[j + t] (each batch's total follows
// its columns)
__global__ void db_core_kernel(const unsigned* deg, int64_t m, int64_t b, unsigned min_samples, int* parent, int* border,
                               unsigned* core)
{
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= m) return;
  const bool c = deg[i + i / b] >= min_samples;
  parent[i]    = c ? static_cast<int>(i) : -1;
  border[i]    = INT_MAX;
  core[i]      = c ? 1u : 0u;
}

// Root of v with path halving.  Every write replaces a parent by one of its ancestors, and hooks only change roots, so
// concurrent finds and unions never make a pointer wrong.
__device__ __forceinline__ int db_find(int* parent, int v)
{
  volatile int* p = parent;
  while (true) {
    const int pv = p[v];
    if (pv == v) return v;
    const int gv = p[pv];
    if (gv == pv) return pv;
    p[v] = gv;
    v    = gv;
  }
}

// unites the trees of roots a and b: the larger root is hooked under the smaller
__device__ __forceinline__ void db_union(int* parent, int a, int b)
{
  while (a != b) {
    if (a > b) { const int t = a; a = b; b = t; }
    const int old = atomicCAS(&parent[b], b, a);
    if (old == b) return;
    b = db_find(parent, old);
    a = db_find(parent, a);
  }
}

// One warp per row of the batch, 16 bytes per lane and step.  Non-core rows are skipped without reading; the root of the
// row is kept between bytes, and a column already in the same tree costs one find and no atomic.
__global__ void __launch_bounds__(kDbThreads) db_link_kernel(const uint8_t* adj, int64_t ld, int64_t m, int64_t s, int64_t w,
                                                             const unsigned* core, int* parent)
{
  const int lane = threadIdx.x & 31;
  const int64_t warps = static_cast<int64_t>(gridDim.x) * (kDbThreads / 32);
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * (kDbThreads / 32) + (threadIdx.x >> 5); i < m; i += warps) {
    if (__ldg(&core[i]) == 0u) continue;
    const uint8_t* row = adj + i * ld;
    int ri = -1;
    for (int64_t c0 = 16 * lane; c0 < w; c0 += 512) {
      const uint4 v = __ldcs(reinterpret_cast<const uint4*>(row + c0));
      const unsigned wd[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        unsigned bits = wd[q];
        while (bits != 0u) {
          const int byte = (__ffs(bits) - 1) >> 3;
          bits &= ~(0xffu << (8 * byte));
          const int64_t c = c0 + 4 * q + byte;
          if (c >= w) continue;
          const int64_t j = s + c;
          if (j == i || __ldg(&core[j]) == 0u) continue;
          if (ri < 0) ri = db_find(parent, static_cast<int>(i));
          const int rj = db_find(parent, static_cast<int>(j));
          if (rj == ri) continue;
          ri = db_find(parent, ri);
          db_union(parent, ri, rj);
          ri = db_find(parent, ri);
        }
      }
    }
  }
}

// parent[i] <- root of i for core rows; root[i] = 1 for the roots (i == its root), else 0.  The find only reads: a
// path-halving find (db_find) stores parent[v] = grandparent while walking, and can so overwrite the root another thread
// just stored at v with a non-root ancestor, which the labels would then read.  Every value this find can see at a node
// (the parent the links left, or the root stored here) is an ancestor, so it ends at the root, and its one store is
// parent[i] = root.
__global__ void db_compress_kernel(int* parent, int64_t m, unsigned* root)
{
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= m) return;
  const volatile int* p = parent;
  int r = p[i];
  if (r >= 0) {
    for (int v = p[r]; v != r; v = p[r]) r = v;
    parent[i] = r;
  }
  root[i] = r == static_cast<int>(i) ? 1u : 0u;
}

// One warp per non-core row: the smallest root (parent, compressed) among the row's core columns of the batch, one
// atomicMin per row.
__global__ void __launch_bounds__(kDbThreads) db_border_kernel(const uint8_t* adj, int64_t ld, int64_t m, int64_t s, int64_t w,
                                                               const int* parent, int* border)
{
  const int lane = threadIdx.x & 31;
  const int64_t warps = static_cast<int64_t>(gridDim.x) * (kDbThreads / 32);
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * (kDbThreads / 32) + (threadIdx.x >> 5); i < m; i += warps) {
    if (__ldg(&parent[i]) >= 0) continue;
    const uint8_t* row = adj + i * ld;
    int best = INT_MAX;
    for (int64_t c0 = 16 * lane; c0 < w; c0 += 512) {
      const uint4 v = __ldcs(reinterpret_cast<const uint4*>(row + c0));
      const unsigned wd[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        unsigned bits = wd[q];
        while (bits != 0u) {
          const int byte = (__ffs(bits) - 1) >> 3;
          bits &= ~(0xffu << (8 * byte));
          const int64_t c = c0 + 4 * q + byte;
          if (c >= w) continue;
          const int r = __ldg(&parent[s + c]);   // -1: not core
          if (r >= 0) best = min(best, r);
        }
      }
    }
    best = __reduce_min_sync(0xffffffffu, best);
    if (lane == 0 && best != INT_MAX) atomicMin(&border[i], best);
  }
}

// ------------------------------------------------------------------------------------------
// The ball-cover fit (b2d_dbscan_rbc_fit, DESIGN.md K20): A from the ball cover's epsilon walk (bc_eps_walk) over the
// index of x itself.  One warp per position t of the index, whose point is ix.pts[t] and caller row ix.ids[t]: warps next
// to each other walk the same balls, and x is not read again.  A is symmetric bit for bit, so a row's hits are its
// column's too.
//   db_rbc_degree_kernel    deg[i] = the hits of row i, the walk ending once min_samples is reached
//   db_rbc_link_kernel      core rows: every core hit j < i unites the trees of i and j
//   db_rbc_border_kernel    non-core rows: border[i] = the smallest root (parent, compressed) among the core hits
// The core flags, the compression and the labels are db_core_kernel (b = m), db_compress_kernel and db_label_kernel.
// A NaN query point (bc_query) is nobody's neighbour.

template <int D>
__global__ void __launch_bounds__(kBcWarps * 32) db_rbc_degree_kernel(BcIndex ix, int n, int nl, int root, float eps,
                                                                      unsigned min_samples, unsigned* deg, int smem)
{
  const float *lm, *rhi;
  bc_stage<D>(ix, nl, smem, &lm, &rhi);
  const int lane = threadIdx.x & 31;
  const int t    = blockIdx.x * kBcWarps + (threadIdx.x >> 5);
  if (t >= n) return;
  float q[D];
  const bool ok = bc_query<D>(ix.pts + static_cast<int64_t>(t) * D, q);
  const int row = ix.ids[t];
  unsigned cnt  = 0;
  if (ok)
    bc_eps_walk<D>(ix, n, nl, lm, rhi, q, root, eps, lane, [&](int, float, bool hit) {
      cnt += __popc(__ballot_sync(0xffffffffu, hit));
      return cnt >= min_samples;   // only the core test reads the degree
    });
  if (lane == 0) deg[row] = cnt;
}

// One find per hit, and no atomic for a hit already in the row's tree; each lane keeps the row's root between its hits,
// as db_link_kernel does.  Only hits below the row: A is symmetric, so the larger end of every core pair takes it.
template <int D>
__global__ void __launch_bounds__(kBcWarps * 32) db_rbc_link_kernel(BcIndex ix, int n, int nl, int root, float eps,
                                                                    const unsigned* core, int* parent, int smem)
{
  const float *lm, *rhi;
  bc_stage<D>(ix, nl, smem, &lm, &rhi);
  const int lane = threadIdx.x & 31;
  const int t    = blockIdx.x * kBcWarps + (threadIdx.x >> 5);
  if (t >= n) return;
  float q[D];
  const bool ok = bc_query<D>(ix.pts + static_cast<int64_t>(t) * D, q);
  const int row = ix.ids[t];
  if (!ok || __ldg(&core[row]) == 0u) return;
  int ri = -1;
  bc_eps_walk<D>(ix, n, nl, lm, rhi, q, root, eps, lane, [&](int i, float, bool hit) {
    if (hit) {
      const int j = __ldg(&ix.ids[i]);
      if (j < row && __ldg(&core[j]) != 0u) {
        if (ri < 0) ri = db_find(parent, row);
        const int rj = db_find(parent, j);
        if (rj != ri) {
          ri = db_find(parent, ri);
          db_union(parent, ri, rj);
          ri = db_find(parent, ri);
        }
      }
    }
    return false;
  });
}

// One warp owns each non-core row, so its smallest root is a plain store.
template <int D>
__global__ void __launch_bounds__(kBcWarps * 32) db_rbc_border_kernel(BcIndex ix, int n, int nl, int root, float eps,
                                                                      const int* parent, int* border, int smem)
{
  const float *lm, *rhi;
  bc_stage<D>(ix, nl, smem, &lm, &rhi);
  const int lane = threadIdx.x & 31;
  const int t    = blockIdx.x * kBcWarps + (threadIdx.x >> 5);
  if (t >= n) return;
  float q[D];
  const bool ok = bc_query<D>(ix.pts + static_cast<int64_t>(t) * D, q);
  const int row = ix.ids[t];
  if (!ok || __ldg(&parent[row]) >= 0) return;
  int best = INT_MAX;
  bc_eps_walk<D>(ix, n, nl, lm, rhi, q, root, eps, lane, [&](int i, float, bool hit) {
    if (hit) {
      const int r = __ldg(&parent[__ldg(&ix.ids[i])]);   // -1: not core
      if (r >= 0) best = min(best, r);
    }
    return false;
  });
  best = __reduce_min_sync(0xffffffffu, best);
  if (lane == 0) border[row] = best;
}

// ------------------------------------------------------------------------------------------

// rank: the root flags scanned (cluster number of root r = rank[r]); crank: the core flags scanned, ctrl_c->total core rows
__global__ void db_label_kernel(const int* parent, const int* border, const unsigned* rank, const unsigned* crank, int64_t m,
                                const unsigned* n_roots, const unsigned* n_core, int* labels, int* core_idx, int* n_clusters)
{
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i == 0 && n_clusters) *n_clusters = static_cast<int>(*n_roots);
  if (i >= m) return;
  const int r = parent[i];
  if (r >= 0) {
    labels[i] = static_cast<int>(rank[r]);
    if (core_idx) core_idx[crank[i]] = static_cast<int>(i);
  } else {
    const int b = border[i];
    labels[i]   = b == INT_MAX ? -1 : static_cast<int>(rank[b]);
  }
  if (core_idx && i >= static_cast<int64_t>(*n_core)) core_idx[i] = -1;
}

}  // namespace b2d
