// raft::cluster::kmeans: Lloyd's k-means on the exact fused L2 arg-min (DESIGN.md section 2, K12).
//
// The assignment is the EPI_MINLOC launch of expanded_tc_kernel; this file holds everything around it:
//   km_begin_kernel      keys <- KEY_EMPTY, the centroid side's exponent and scale flag <- 0 (before the centroids are
//                        prepared again), label histogram <- 0
//   km_assign_kernel     label of every row from its key (or the caller's labels), the fp64 inertia partial of the row
//                        block, and the integer histogram of the labels per (cluster, row block)
//   km_scan_tiles_kernel / km_scan_kernel   exclusive integer scan of the histogram in (cluster, row block) order
//   km_scatter_kernel    stable counting sort of the row ids by label (cub::BlockRadixSort inside each row block)
//   km_sum_kernel        fp64 sums of w_i x_i in row order over fixed chunks of the sorted rows
//   km_finalize_kernel   per cluster: chunk partials in chunk order, divide, round once to fp32; zero weight keeps the
//                        previous centroid; the fp64 squared shift of the cluster
//   km_converge_kernel   one CTA: fixed-order sums of the shifts and the inertia partials, the stopping rules
// Determinism: every floating-point sum has an order fixed by m, k and n_clusters alone (rows in row order inside a
// chunk, chunks in chunk order, block partials by cub::BlockReduce over a fixed block shape).  Atomics are integer only.
// The loop runs on the device: every kernel above (and the operand preparation and arg-min launches) returns at once when
// the run word is 0, so a fit enqueues max_iter iterations and never waits for the host.
//
// k-means++ (km_pp_*): greedy k-means++ with 2 + floor(ln n_clusters) trials per round ([RECALLED] RAFT init_plus_plus).
// D^2 is the fp32 difference form, so a duplicate of a chosen row gets exactly 0 and is never drawn.  Sampling: fp64 sums
// per block of kKmPpBlock rows in a fixed order, a one-CTA scan of those sums, and a search in row order inside the chosen
// block.  Random numbers: Philox4x32-10 keyed by (seed, round, trial) -- curand's header-only device functions.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <curand_kernel.h>
#include <cub/block/block_radix_sort.cuh>
#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>

#include "nn_key.cuh"
#include "kmeans_types.cuh"

namespace b2d {

__device__ __forceinline__ bool km_running(const unsigned* run) { return run == nullptr || *reinterpret_cast<const volatile unsigned*>(run) != 0u; }

// sum of a[0..n) in a fixed order: thread t sums t, t + blockDim, ... sequentially, then a fixed reduction tree
template <int kThreads>
__device__ double km_block_sum_fixed(const double* a, int64_t n)
{
  using R = cub::BlockReduce<double, kThreads>;
  __shared__ typename R::TempStorage tmp;
  double s = 0.0;
  for (int64_t i = threadIdx.x; i < n; i += kThreads) s += a[i];
  const double r = R(tmp).Sum(s);
  __syncthreads();
  return r;  // valid in thread 0
}

__global__ void km_begin_kernel(const unsigned* run, long long* keys, int64_t m, unsigned* gmax, unsigned* nonuni,
                                unsigned* hist, int64_t nhist)
{
  if (!km_running(run)) return;
  const int64_t i0 = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i0 == 0 && gmax) { gmax[1] = 0u; nonuni[1] = 0u; }
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  if (keys)
    for (int64_t i = i0; i < m; i += stride) keys[i] = KEY_EMPTY;
  if (hist)
    for (int64_t i = i0; i < nhist; i += stride) hist[i] = 0u;
}

// One CTA per row block of rb rows.  keys != null: label = arg-min of the row (-1 when the row has none: a NaN distance),
// written to labels, and the block's fp64 inertia partial sum w_i d_i (NaN for a row without arg-min).  keys == null:
// labels are read.  hist != null: hist[label * nblk + block] counts the rows with a label in [0, nc).
__global__ void __launch_bounds__(kKmThreads) km_assign_kernel(const unsigned* run, const long long* keys, int* labels,
                                                               const float* w, int64_t m, int nc, int64_t rb, int64_t nblk,
                                                               unsigned* hist, double* ipart)
{
  if (!km_running(run)) return;
  const int64_t b  = blockIdx.x;
  const int64_t r0 = b * rb, r1 = min(m, r0 + rb);
  double acc = 0.0;
  for (int64_t i = r0 + threadIdx.x; i < r1; i += kKmThreads) {
    int lab;
    if (keys) {
      const long long key = keys[i];
      lab = key == KEY_EMPTY ? -1 : static_cast<int>(key_index(key));
      labels[i] = lab;
      const float d  = key == KEY_EMPTY ? __int_as_float(0x7fffffff) : fmaxf(key_dist(key), 0.f);
      const float wi = w ? w[i] : 1.f;
      acc += static_cast<double>(wi) * static_cast<double>(d);
    } else {
      lab = labels[i];
    }
    if (hist && lab >= 0 && lab < nc) atomicAdd(&hist[static_cast<int64_t>(lab) * nblk + b], 1u);
  }
  if (ipart) {
    using R = cub::BlockReduce<double, kKmThreads>;
    __shared__ typename R::TempStorage tmp;
    const double s = R(tmp).Sum(acc);
    if (threadIdx.x == 0) ipart[b] = s;
  }
}

// The reported inertia: sum_i w_i ||x_i - c_{label_i}||^2 in fp64 in the difference form (a row equal to its centroid
// adds exactly 0; a row without a label adds NaN), one warp per row, the block's partial in warp order into ipart.
__global__ void __launch_bounds__(kKmThreads) km_cost_kernel(const float* x, int64_t ldx, int k, const float* c,
                                                             const int* labels, const float* w, int64_t m, int64_t rb,
                                                             double* ipart)
{
  __shared__ double wsum[kKmThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t r0 = static_cast<int64_t>(blockIdx.x) * rb, r1 = min(m, r0 + rb);
  double acc = 0.0;
  for (int64_t i = r0 + warp; i < r1; i += kKmThreads / 32) {
    const int lab = labels[i];
    double d = 0.0;
    if (lab >= 0) {
      for (int t = lane; t < k; t += 32) {
        const double e = static_cast<double>(x[i * ldx + t]) - static_cast<double>(c[static_cast<int64_t>(lab) * k + t]);
        d += e * e;
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
    } else {
      d = __longlong_as_double(0x7ff8000000000000ll);
    }
    acc += static_cast<double>(w ? w[i] : 1.f) * d;
  }
  if (lane == 0) wsum[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int v = 0; v < kKmThreads / 32; ++v) s += wsum[v];
    ipart[blockIdx.x] = s;
  }
}

__global__ void __launch_bounds__(kKmThreads) km_scan_tiles_kernel(const unsigned* run, const unsigned* hist, int64_t n,
                                                                   unsigned* tile_sum)
{
  if (!km_running(run)) return;
  using R = cub::BlockReduce<unsigned, kKmThreads>;
  __shared__ typename R::TempStorage tmp;
  const int64_t base = static_cast<int64_t>(blockIdx.x) * kKmScanTile;
  unsigned s = 0;
  for (int j = threadIdx.x; j < kKmScanTile; j += kKmThreads)
    if (base + j < n) s += hist[base + j];
  s = R(tmp).Sum(s);
  if (threadIdx.x == 0) tile_sum[blockIdx.x] = s;
}

// offs = exclusive scan of hist (in place); the last tile also stores the total in ctrl->total
__global__ void __launch_bounds__(kKmThreads) km_scan_kernel(const unsigned* run, unsigned* hist, int64_t n,
                                                             const unsigned* tile_sum, KmCtrl* ctrl)
{
  if (!km_running(run)) return;
  using R = cub::BlockReduce<unsigned, kKmThreads>;
  using S = cub::BlockScan<unsigned, kKmThreads>;
  __shared__ union { typename R::TempStorage r; typename S::TempStorage s; } tmp;
  __shared__ unsigned carry;
  unsigned pre = 0;
  for (unsigned t = threadIdx.x; t < blockIdx.x; t += kKmThreads) pre += tile_sum[t];
  pre = R(tmp.r).Sum(pre);
  if (threadIdx.x == 0) carry = pre;
  __syncthreads();
  const int64_t base = static_cast<int64_t>(blockIdx.x) * kKmScanTile;
  constexpr int kItems = kKmScanTile / kKmThreads;
  unsigned v[kItems];
#pragma unroll
  for (int j = 0; j < kItems; ++j) {
    const int64_t at = base + threadIdx.x * kItems + j;
    v[j] = at < n ? hist[at] : 0u;
  }
  unsigned agg;
  S(tmp.s).ExclusiveSum(v, v, agg);
#pragma unroll
  for (int j = 0; j < kItems; ++j) {
    const int64_t at = base + threadIdx.x * kItems + j;
    if (at < n) hist[at] = v[j] + carry;
  }
  if (threadIdx.x == 0 && blockIdx.x == gridDim.x - 1) ctrl->total = carry + agg;
}

// Stable counting sort: row i goes to position cur[label * nblk + block] + (rank of i among the rows of its label in
// the block).  One CTA per row block, sub-blocks of kKmSub rows in order; cub::BlockRadixSort is stable, so a run of
// equal labels in the sorted sub-block is in row order.  After the kernel cur[c * nblk + b] holds the end of (c, b):
// cluster c occupies [cur[c * nblk - 1], cur[c * nblk + nblk - 1]) (start 0 for c = 0).
__global__ void __launch_bounds__(kKmThreads) km_scatter_kernel(const unsigned* run, const int* labels, int64_t m, int nc,
                                                                int end_bit, int64_t rb, int64_t nblk, unsigned* cur,
                                                                int* perm, int* slab)
{
  if (!km_running(run)) return;
  using Sort = cub::BlockRadixSort<unsigned, kKmThreads, kKmSortItems, int>;
  using Scan = cub::BlockScan<int, kKmThreads>;
  __shared__ union { typename Sort::TempStorage sort; typename Scan::TempStorage scan; } tmp;
  __shared__ unsigned skey[kKmSub + 1];
  const int64_t b  = blockIdx.x;
  const int64_t r1 = min(m, (b + 1) * rb);
  for (int64_t s0 = b * rb; s0 < r1; s0 += kKmSub) {
    unsigned key[kKmSortItems];
    int row[kKmSortItems];
#pragma unroll
    for (int j = 0; j < kKmSortItems; ++j) {
      const int64_t i = s0 + threadIdx.x * kKmSortItems + j;   // blocked arrangement: sub-block order is row order
      int lab = i < r1 ? labels[i] : -1;
      key[j]  = (lab >= 0 && lab < nc) ? static_cast<unsigned>(lab) : static_cast<unsigned>(nc);
      row[j]  = static_cast<int>(i);
    }
    Sort(tmp.sort).Sort(key, row, 0, end_bit);
    __syncthreads();
#pragma unroll
    for (int j = 0; j < kKmSortItems; ++j) skey[threadIdx.x * kKmSortItems + j] = key[j];
    if (threadIdx.x == 0) skey[kKmSub] = 0xffffffffu;
    __syncthreads();
    int start[kKmSortItems];
#pragma unroll
    for (int j = 0; j < kKmSortItems; ++j) {
      const int s = threadIdx.x * kKmSortItems + j;
      start[j]    = (s == 0 || skey[s - 1] != key[j]) ? s : 0;
    }
    Scan(tmp.scan).InclusiveScan(start, start, cub::Max());
    unsigned pos[kKmSortItems];
#pragma unroll
    for (int j = 0; j < kKmSortItems; ++j) {
      const int s = threadIdx.x * kKmSortItems + j;
      pos[j] = key[j] < static_cast<unsigned>(nc) ? cur[static_cast<int64_t>(key[j]) * nblk + b] + (s - start[j]) : 0u;
    }
    __syncthreads();   // every thread has read the cursors of this sub-block
#pragma unroll
    for (int j = 0; j < kKmSortItems; ++j) {
      const int s = threadIdx.x * kKmSortItems + j;
      if (key[j] >= static_cast<unsigned>(nc)) continue;
      perm[pos[j]] = row[j];
      slab[pos[j]] = static_cast<int>(key[j]);
      if (skey[s + 1] != key[j]) cur[static_cast<int64_t>(key[j]) * nblk + b] += static_cast<unsigned>(s - start[j] + 1);
    }
    __syncthreads();   // cursor updates visible before the next sub-block
  }
}

__device__ __forceinline__ void km_cluster_range(const unsigned* cur, int64_t nblk, int c, int64_t& cs, int64_t& ce)
{
  cs = c > 0 ? cur[static_cast<int64_t>(c) * nblk - 1] : 0;
  ce = cur[static_cast<int64_t>(c) * nblk + nblk - 1];
}

// Chunk q = sorted positions [q * kKmChunk, (q + 1) * kKmChunk), columns [kKmCols * blockIdx.y, ...).  Each run of one
// label is summed in fp64 in row order.  A run that is a whole cluster goes to sums / wsums; a run cut by the chunk
// boundary goes to part / wpart slot 2q (it starts the chunk) or 2q + 1 (it ends the chunk).
__global__ void __launch_bounds__(kKmCols) km_sum_kernel(const unsigned* run, const float* x, int64_t ldx, int k,
                                                         const float* w, const int* perm, const int* slab,
                                                         const unsigned* cur, int64_t nblk, const KmCtrl* ctrl,
                                                         double* sums, double* wsums, double* part, double* wpart)
{
  if (!km_running(run)) return;
  __shared__ int srow[kKmChunk + 1], slb[kKmChunk + 1];
  __shared__ float sw[kKmChunk];
  const int64_t total = ctrl->total;
  const int64_t p0 = static_cast<int64_t>(blockIdx.x) * kKmChunk;
  if (p0 >= total) return;
  const int len = static_cast<int>(min(static_cast<int64_t>(kKmChunk), total - p0));
  for (int j = threadIdx.x; j < len; j += kKmCols) {
    srow[j] = perm[p0 + j];
    slb[j]  = slab[p0 + j];
    sw[j]   = w ? w[srow[j]] : 1.f;
  }
  if (threadIdx.x == 0) slb[len] = -1;
  __syncthreads();
  // (grid.y is capped at the launch limit: a CTA takes every gridDim.y-th strip of kKmCols columns)
  for (int64_t col0 = static_cast<int64_t>(blockIdx.y) * kKmCols; col0 < k; col0 += static_cast<int64_t>(gridDim.y) * kKmCols) {
  const int col    = static_cast<int>(col0) + threadIdx.x;
  const bool on    = col < k;
  const bool wlead = col0 == 0 && threadIdx.x == 0;
  double acc = 0.0, wacc = 0.0;
  int a = 0;
  for (int j = 0; j < len; ++j) {
    const float xv = on ? __ldg(&x[static_cast<int64_t>(srow[j]) * ldx + col]) : 0.f;
    acc += static_cast<double>(sw[j]) * static_cast<double>(xv);
    wacc += static_cast<double>(sw[j]);
    if (slb[j + 1] != slb[j]) {   // the run [a, j] ends
      const int c = slb[j];
      int64_t cs, ce;
      km_cluster_range(cur, nblk, c, cs, ce);
      const int64_t ra = p0 + a, re = p0 + j + 1;
      if (ra == cs && re == ce) {
        if (on) sums[static_cast<int64_t>(c) * k + col] = acc;
        if (wlead) wsums[c] = wacc;
      } else {
        const int64_t slot = 2 * static_cast<int64_t>(blockIdx.x) + (a == 0 ? 0 : 1);
        if (on) part[slot * k + col] = acc;
        if (wlead) wpart[slot] = wacc;
      }
      acc = 0.0; wacc = 0.0; a = j + 1;
    }
  }
  }
}

// One CTA per cluster.  new = round(sum / W) unless W == 0 (empty or zero-weight cluster: the old bits stay).
// old and out may be the same array.  shift[c] = sum over columns of (new - old)^2 in fp64; wpc[c] = W as fp32.
__global__ void __launch_bounds__(kKmCols) km_finalize_kernel(const unsigned* run, int k, const unsigned* cur, int64_t nblk,
                                                              const double* sums, const double* wsums, const double* part,
                                                              const double* wpart, const float* old_c, float* out_c,
                                                              double* shift, float* wpc)
{
  if (!km_running(run)) return;
  const int c = blockIdx.x;
  int64_t cs, ce;
  km_cluster_range(cur, nblk, c, cs, ce);
  const int64_t q0 = cs / kKmChunk, q1 = ce > cs ? (ce - 1) / kKmChunk : q0;
  const bool whole = ce > cs && q0 == q1;
  double W = 0.0;
  if (ce > cs) {
    if (whole) W = wsums[c];
    else
      for (int64_t q = q0; q <= q1; ++q) W += wpart[2 * q + ((q == q0 && cs != q0 * kKmChunk) ? 1 : 0)];
  }
  const bool keep = !(W != 0.0);
  double sh = 0.0;
  for (int col = threadIdx.x; col < k; col += kKmCols) {
    const float o = old_c[static_cast<int64_t>(c) * k + col];
    float v       = o;
    if (!keep) {
      double s = 0.0;
      if (whole) s = sums[static_cast<int64_t>(c) * k + col];
      else
        for (int64_t q = q0; q <= q1; ++q) s += part[(2 * q + ((q == q0 && cs != q0 * kKmChunk) ? 1 : 0)) * k + col];
      v = static_cast<float>(s / W);
    }
    out_c[static_cast<int64_t>(c) * k + col] = v;
    const double d = static_cast<double>(v) - static_cast<double>(o);
    sh += d * d;
  }
  using R = cub::BlockReduce<double, kKmCols>;
  __shared__ typename R::TempStorage tmp;
  sh = R(tmp).Sum(sh);
  if (threadIdx.x == 0) {
    if (shift) shift[c] = sh;
    if (wpc) wpc[c] = static_cast<float>(W);
  }
}

// End of iteration ([RECALLED] kmeans_fit_main): stop when the summed squared shift is below tol or, with inertia_check
// after the first iteration, when inertia_t / inertia_{t-1} > 1 - tol.
__global__ void __launch_bounds__(kKmThreads) km_converge_kernel(unsigned* run, KmCtrl* ctrl, const double* shift, int nc,
                                                                 const double* ipart, int64_t nipart, double tol,
                                                                 int inertia_check)
{
  if (!km_running(run)) return;
  const double sh = km_block_sum_fixed<kKmThreads>(shift, nc);
  const double in = km_block_sum_fixed<kKmThreads>(ipart, nipart);
  if (threadIdx.x != 0) return;
  const double inertia = ctrl->bad ? __longlong_as_double(0x7ff8000000000000ll) : in;
  const int it         = ++ctrl->iter;
  bool done            = sh < tol;
  if (inertia_check && it > 1 && inertia / ctrl->prior > 1.0 - tol) done = true;
  ctrl->prior = inertia;
  if (done) *run = 0u;
}

// inertia of the last assignment -> ctrl->inertia (and the caller's outputs when given)
__global__ void __launch_bounds__(kKmThreads) km_finish_kernel(KmCtrl* ctrl, const double* ipart, int64_t nipart,
                                                               double* inertia_out, int* n_iter_out)
{
  const double in = km_block_sum_fixed<kKmThreads>(ipart, nipart);
  if (threadIdx.x != 0) return;
  const double inertia = ctrl->bad ? __longlong_as_double(0x7ff8000000000000ll) : in;
  ctrl->inertia = inertia;
  if (inertia_out) *inertia_out = inertia;
  if (n_iter_out) *n_iter_out = ctrl->iter;
}

__global__ void km_fit_begin_kernel(KmCtrl* ctrl)
{
  ctrl->run   = 1u;
  ctrl->iter  = 0;
  ctrl->prior = 0.0;
}

// ---- weights: fp64 block sums (fixed order), then one CTA forms the scale m / sum; negative or NaN weights mark bad
__global__ void __launch_bounds__(kKmThreads) km_wsum_kernel(const float* w, int64_t m, double* bs, KmCtrl* ctrl)
{
  using R = cub::BlockReduce<double, kKmThreads>;
  __shared__ typename R::TempStorage tmp;
  const int64_t r0 = static_cast<int64_t>(blockIdx.x) * kKmPpBlock;
  double s = 0.0;
  bool bad = false;
  for (int j = threadIdx.x; j < kKmPpBlock; j += kKmThreads) {
    if (r0 + j >= m) break;
    const float v = w[r0 + j];
    bad |= !(v >= 0.f);
    s += static_cast<double>(v);
  }
  if (__syncthreads_or(bad) && threadIdx.x == 0) ctrl->bad = 1u;
  s = R(tmp).Sum(s);
  if (threadIdx.x == 0) bs[blockIdx.x] = s;
}

__global__ void __launch_bounds__(kKmThreads) km_wscale_kernel(const double* bs, int64_t nb, int64_t m, KmCtrl* ctrl)
{
  const double t = km_block_sum_fixed<kKmThreads>(bs, nb);
  if (threadIdx.x != 0) return;
  if (!(t > 0.0)) ctrl->bad = 1u;
  ctrl->wscale = t > 0.0 ? static_cast<double>(m) / t : 1.0;
}

// w_out = w * (float)(m / sum)  ([RECALLED] checkWeight: the weights are scaled to sum to m)
__global__ void km_wapply_kernel(const float* w, float* wout, int64_t m, const KmCtrl* ctrl)
{
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < m) wout[i] = w[i] * static_cast<float>(ctrl->wscale);
}

__global__ void km_ctrl_init_kernel(KmCtrl* ctrl)
{
  ctrl->bad       = 0u;
  ctrl->run       = 1u;
  ctrl->iter      = 0;
  ctrl->take      = 0u;
  ctrl->best_iter = 0;
  ctrl->best_inertia = 0.0;
}

// ---- n_init: keep the first run with the strictly lowest inertia
__global__ void km_best_decide_kernel(KmCtrl* ctrl, int first)
{
  const bool take = first || ctrl->inertia < ctrl->best_inertia;
  ctrl->take      = take ? 1u : 0u;
  if (take) {
    ctrl->best_inertia = ctrl->inertia;
    ctrl->best_iter    = ctrl->iter;
  }
}

__global__ void km_copy_kernel(const KmCtrl* ctrl, int only_if_take, const float* src, float* dst, int64_t n)
{
  if (only_if_take && ctrl->take == 0u) return;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x)
    dst[i] = src[i];
}

__global__ void km_best_out_kernel(const KmCtrl* ctrl, double* inertia, int* n_iter)
{
  *inertia = ctrl->best_inertia;
  *n_iter  = ctrl->best_iter;
}

// ---- Random init: one seeded uniform per row (select_k of the n_clusters smallest picks distinct rows)
__device__ __forceinline__ double km_uniform(unsigned long long seed, unsigned long long stream_id)
{
  curandStatePhilox4_32_10_t st;
  curand_init(seed, stream_id, 0, &st);
  return 1.0 - curand_uniform_double(&st);   // [0, 1)
}

__global__ void km_uniforms_kernel(float* u, int64_t m, unsigned long long seed)
{
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= m) return;
  curandStatePhilox4_32_10_t st;
  curand_init(seed, static_cast<unsigned long long>(i), 0, &st);
  u[i] = curand_uniform(&st);
}

// centroid c = row idx[c] of x (int64 or int32 indices)
template <typename I>
__global__ void km_gather_rows_kernel(const float* x, int64_t ldx, int k, const I* idx, int nc, float* out)
{
  const int c = blockIdx.x;
  if (c >= nc) return;
  const int64_t r = static_cast<int64_t>(idx[c]);
  for (int col = threadIdx.x; col < k; col += blockDim.x) out[static_cast<int64_t>(c) * k + col] = x[r * ldx + col];
}

// ---- k-means++
// squared distance of rows a and b of x, difference form in fp32, summed by a warp in a fixed order
__device__ __forceinline__ float km_row_d2(const float* x, int64_t ldx, int k, int64_t a, int64_t b, int lane)
{
  float s = 0.f;
  for (int t = lane; t < k; t += 32) {
    const float d = __ldg(&x[a * ldx + t]) - __ldg(&x[b * ldx + t]);
    s             = fmaf(d, d, s);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  return s;
}

// D2 <- +inf, bs[b * kKmPpMaxTrials] = the block's sum of w (the weights of the first draw)
__global__ void __launch_bounds__(kKmThreads) km_pp_init_kernel(const float* w, int64_t m, float* d2, double* bs,
                                                                KmCtrl* ctrl)
{
  using R = cub::BlockReduce<double, kKmThreads>;
  __shared__ typename R::TempStorage tmp;
  const int64_t r0 = static_cast<int64_t>(blockIdx.x) * kKmPpBlock;
  double s = 0.0;
  for (int j = threadIdx.x; j < kKmPpBlock; j += kKmThreads) {
    if (r0 + j >= m) break;
    d2[r0 + j] = __int_as_float(0x7f800000);
    s += w ? static_cast<double>(fmaxf(w[r0 + j], 0.f)) : 1.0;
  }
  s = R(tmp).Sum(s);
  if (threadIdx.x == 0) bs[blockIdx.x * static_cast<int64_t>(kKmPpMaxTrials)] = s;
  if (blockIdx.x == 0 && threadIdx.x == 0) ctrl->pp_last = -1;
}

// One pass over x per round: D2 <- min(D2, d(x_i, last chosen)); for every trial t, bs[b][t] = sum over the block of
// w_i min(D2_i, d(x_i, cand_t)) -- the potential of trial t, and, if t wins, the block sums of the next round's draw.
// One warp per row; the partial of every warp is kept per trial, then summed over the warps in warp order.
__global__ void __launch_bounds__(kKmThreads) km_pp_pass_kernel(const float* x, int64_t ldx, int k, const float* w,
                                                                int64_t m, float* d2, double* bs, const KmCtrl* ctrl)
{
  __shared__ double wsum[kKmThreads / 32][kKmPpMaxTrials];
  __shared__ int cand[kKmPpMaxTrials];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int T    = ctrl->pp_trials;
  const int last = ctrl->pp_last;
  if (threadIdx.x < T) cand[threadIdx.x] = ctrl->pp_cand[threadIdx.x];
  __syncthreads();
  double acc[kKmPpMaxTrials];
#pragma unroll
  for (int t = 0; t < kKmPpMaxTrials; ++t) acc[t] = 0.0;
  const int64_t r0 = static_cast<int64_t>(blockIdx.x) * kKmPpBlock;
  for (int j = warp; j < kKmPpBlock; j += kKmThreads / 32) {
    const int64_t i = r0 + j;
    if (i >= m) break;
    float D = d2[i];
    if (last >= 0) {
      D = fminf(D, km_row_d2(x, ldx, k, i, last, lane));
      if (lane == 0) d2[i] = D;
    }
    const double wi = w ? static_cast<double>(fmaxf(w[i], 0.f)) : 1.0;
#pragma unroll
    for (int t = 0; t < kKmPpMaxTrials; ++t)
      if (t < T) acc[t] += wi * static_cast<double>(fminf(D, km_row_d2(x, ldx, k, i, cand[t], lane)));
  }
  if (lane == 0)
#pragma unroll
    for (int t = 0; t < kKmPpMaxTrials; ++t) wsum[warp][t] = acc[t];
  __syncthreads();
  if (threadIdx.x < T) {
    double s = 0.0;
    for (int v = 0; v < kKmThreads / 32; ++v) s += wsum[v][threadIdx.x];
    bs[blockIdx.x * static_cast<int64_t>(kKmPpMaxTrials) + threadIdx.x] = s;
  }
}

// Draw one row with probability p_i / sum p, where p_i = w_i * f_i and f_i = min(D2_i, d(x_i, x_last)) (f = 1 while no
// centroid is chosen).  The block sums bs[b * kKmPpMaxTrials + t] of p are given.  u in [0, 1).  Runs in one CTA.
__device__ int km_pp_draw(const float* x, int64_t ldx, int k, const float* w, int64_t m, const float* d2, int last,
                          const double* bs, int t, int64_t nb, double u)
{
  using S = cub::BlockScan<double, kKmThreads>;
  __shared__ typename S::TempStorage tmp;
  __shared__ double pv[kKmPpBlock];
  __shared__ double s_carry, s_target;
  __shared__ int64_t s_blk;
  __shared__ int s_pick;
  // total and the block holding u * total: chunks of kKmThreads block sums, scanned in order
  if (threadIdx.x == 0) { s_carry = 0.0; s_blk = -1; }
  __syncthreads();
  double total = 0.0;
  for (int64_t b0 = 0; b0 < nb; b0 += kKmThreads) {
    const int64_t b = b0 + threadIdx.x;
    const double v  = b < nb ? bs[b * kKmPpMaxTrials + t] : 0.0;
    double inc, agg;
    S(tmp).InclusiveSum(v, inc, agg);
    __syncthreads();
    if (threadIdx.x == 0) s_carry += agg;
    __syncthreads();
  }
  total = s_carry;
  const double target = u * total;
  __syncthreads();   // every thread has read the total before thread 0 clears the carry
  if (threadIdx.x == 0) s_carry = 0.0;
  __syncthreads();
  if (total > 0.0) {
    __shared__ double sinc[kKmThreads];
    for (int64_t b0 = 0; b0 < nb && s_blk < 0; b0 += kKmThreads) {
      const int64_t b = b0 + threadIdx.x;
      const double v  = b < nb ? bs[b * kKmPpMaxTrials + t] : 0.0;
      double inc, agg;
      S(tmp).InclusiveSum(v, inc, agg);
      inc += s_carry;
      sinc[threadIdx.x] = inc;
      __syncthreads();
      // the first block whose inclusive prefix exceeds the target (so it holds positive mass)
      const double prev = threadIdx.x ? sinc[threadIdx.x - 1] : s_carry;
      if (b < nb && inc > target && prev <= target) { s_blk = b; s_target = target - prev; }
      __syncthreads();
      if (threadIdx.x == 0) s_carry += agg;
      __syncthreads();
    }
    const int64_t found = s_blk;   // (read by every thread after the loop's last barrier, before thread 0 may write it)
    if (found < 0) {   // rounding put the target past the last block: the last block with mass
      if (threadIdx.x == 0)
        for (int64_t b = nb - 1; b >= 0; --b)
          if (bs[b * kKmPpMaxTrials + t] > 0.0) { s_blk = b; s_target = bs[b * kKmPpMaxTrials + t]; break; }
      __syncthreads();
    }
  }
  if (s_blk < 0) {   // no mass at all (every row coincides with a chosen centroid): a uniform row
    const int64_t r = min(m - 1, static_cast<int64_t>(u * static_cast<double>(m)));
    __syncthreads();
    return static_cast<int>(r);
  }
  // p of every row of the chosen block, then a sequential search in row order
  const int64_t r0 = s_blk * kKmPpBlock;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int j = warp; j < kKmPpBlock; j += kKmThreads / 32) {
    const int64_t i = r0 + j;
    double p = 0.0;
    if (i < m) {
      float f = 1.f;
      if (last >= 0) f = fminf(d2[i], km_row_d2(x, ldx, k, i, last, lane));
      p = (w ? static_cast<double>(fmaxf(w[i], 0.f)) : 1.0) * static_cast<double>(f);
    }
    if (lane == 0) pv[j] = p;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double c = 0.0;
    int pick = -1, lastpos = -1;
    for (int j = 0; j < kKmPpBlock && r0 + j < m; ++j) {
      if (pv[j] > 0.0) lastpos = j;
      c += pv[j];
      if (pv[j] > 0.0 && c > s_target) { pick = j; break; }
    }
    s_pick = static_cast<int>(r0) + (pick >= 0 ? pick : lastpos);
  }
  __syncthreads();
  return s_pick;
}

// Round `round`: choose the trial with the smallest potential (ties: the earlier trial), make it centroid `round`, and
// draw the candidates of the next round.  round < 0: only the first draw (probability ~ w).
__global__ void __launch_bounds__(kKmThreads) km_pp_choose_kernel(const float* x, int64_t ldx, int k, const float* w,
                                                                  int64_t m, const float* d2, double* bs, int64_t nb,
                                                                  KmCtrl* ctrl, float* centroids, int round, int nc,
                                                                  int trials, unsigned long long seed)
{
  __shared__ int s_win, s_row;
  int tw = 0;
  if (round >= 0) {
    const int T = ctrl->pp_trials;
    if (threadIdx.x == 0) { s_win = 0; }
    __syncthreads();
    double best = 0.0;
    for (int t = 0; t < T; ++t) {
      double s = 0.0;
      // fixed order over the blocks: thread j sums j, j + kKmThreads, ...; then a fixed tree
      using R = cub::BlockReduce<double, kKmThreads>;
      __shared__ typename R::TempStorage tmp;
      for (int64_t b = threadIdx.x; b < nb; b += kKmThreads) s += bs[b * kKmPpMaxTrials + t];
      s = R(tmp).Sum(s);
      if (threadIdx.x == 0 && (t == 0 || s < best)) { best = s; s_win = t; }
      __syncthreads();
    }
    tw = s_win;
    if (threadIdx.x == 0) s_row = ctrl->pp_cand[tw];
    __syncthreads();
    const int64_t r = s_row;
    for (int col = threadIdx.x; col < k; col += kKmThreads)
      centroids[static_cast<int64_t>(round) * k + col] = x[r * ldx + col];
    if (round + 1 >= nc) return;
  }
  // the draws of the next round, from the block sums of the winner (round < 0: of the weights)
  const int last  = round >= 0 ? s_row : -1;
  const int T     = round >= 0 ? trials : 1;
  for (int t = 0; t < T; ++t) {
    const double u = km_uniform(seed, (static_cast<unsigned long long>(round + 1) << 8) | static_cast<unsigned>(t));
    const int row  = km_pp_draw(x, ldx, k, w, m, d2, last, bs, tw, nb, u);
    if (threadIdx.x == 0) ctrl->pp_cand[t] = row;
  }
  if (threadIdx.x == 0) {
    ctrl->pp_trials = T;
    ctrl->pp_last   = last;
  }
}

}  // namespace b2d
