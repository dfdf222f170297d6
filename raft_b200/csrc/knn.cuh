// Kernels of the fused brute-force kNN around the EPI_TOPK launches of expanded_tc.cuh.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include "nn_key.cuh"
#include "tc_params.cuh"

namespace b2d {

// ---------------------------------------------------------------------------------------------
// Fused brute-force kNN (SURVEY.md 8(f2)): the distance tiles are never written.  The database is
// swept in passes of doubling width; EPI_TOPK appends every pair at or below the row's current k-th
// best to the row's list (~k per row and pass on unordered data), knn_merge_kernel folds the list
// into the row's sorted top-k and publishes the new k-th best.

__global__ void knn_init_kernel(long long* topk, float* thr, unsigned* cnt, long long* dropmin, unsigned* dirty_cnt,
                                unsigned* repaired, int64_t m, int kk)
{
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < 65) dirty_cnt[i] = 0u;   // one counter per pass, then the counter of the repaired-row list
  if (i < m) { thr[i] = __int_as_float(0x7f800000); cnt[i] = 0u; dropmin[i] = KEY_EMPTY; repaired[i] = 0u; }
  if (i < m * kk) topk[i] = KEY_EMPTY;
}

// one warp per row: sort (top-k so far) + (this pass's list) by (distance, index), keep the first kk.  A row whose list
// was full lost entries; that only matters if the best dropped key could still enter the new top-k -- such rows go
// to the pass's dirty list and knn_fix_kernel redoes them over the pass's columns (no host round trip anywhere).  A row
// dirty for the first time also goes to the repaired-row list (rep_list / rep_cnt, flag repaired[row]), which is measured
// again over all columns after the last pass.
__global__ void __launch_bounds__(256) knn_merge_kernel(long long* topk, const long long* cand, unsigned* cnt, float* thr,
                                                        long long* dropmin, int* dirty, unsigned* dirty_cnt, unsigned* repaired,
                                                        int* rep_list, unsigned* rep_cnt, int64_t m, int kk)
{
  __shared__ long long buf[8][KNN_SORT];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int64_t row = static_cast<int64_t>(blockIdx.x) * 8 + wid;
  if (row >= m) return;
  const unsigned craw = cnt[row];
  const unsigned nc   = min(craw, static_cast<unsigned>(KNN_CAP));
  if (nc == 0u) return;  // nothing new for this row (the common case in the late passes)
  long long* b = buf[wid];
  // sort only as much as there is (warp-uniform): with k = 16 and ~16 new entries per pass that is 32 or 64 keys,
  // not KNN_SORT = 256 -- the merge launches were a third of a 100000 x 100000 kNN
  int ssz = 32;
  while (ssz < kk + static_cast<int>(nc)) ssz <<= 1;
  for (int t = lane; t < ssz; t += 32) {
    long long key = KEY_EMPTY;
    if (t < kk) key = topk[row * kk + t];
    else if (t - kk < static_cast<int>(nc)) key = cand[row * KNN_CAP + (t - kk)];
    b[t] = key;
  }
  __syncwarp();
  for (int size = 2; size <= ssz; size <<= 1)
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int t = lane; t < ssz / 2; t += 32) {
        const int i = 2 * t - (t & (stride - 1)), j = i + stride;
        const bool up = (i & size) == 0;
        const long long a = b[i], c = b[j];
        if ((a > c) == up) { b[i] = c; b[j] = a; }
      }
      __syncwarp();
    }
  for (int t = lane; t < kk; t += 32) topk[row * kk + t] = b[t];
  if (lane == 0) {
    cnt[row]            = 0u;
    const long long kth = b[kk - 1];
    if (kth != KEY_EMPTY) thr[row] = key_dist(kth);
    if (craw > static_cast<unsigned>(KNN_CAP)) {
      if (dropmin[row] <= kth) {
        dirty[atomicAdd(dirty_cnt, 1u)] = static_cast<int>(row);
        if (!repaired[row]) {   // (one warp owns the row, and the merges of the passes run one after another)
          repaired[row]                    = 1u;
          rep_list[atomicAdd(rep_cnt, 1u)] = static_cast<int>(row);
        }
      }
      dropmin[row] = KEY_EMPTY;
    }
  }
}

// Rows whose candidate list overflowed in a way that matters (database ordered by decreasing distance, duplicates of one
// near point, ...): one block per dirty row re-evaluates the pass's columns [off, off + width) straight from the fp32
// inputs -- family 0: sum (x - y)^2, family 1: 1 - <x', y'> / (|x'||y'|) with x' centred for correlation -- one column per
// thread, and folds them into the row's top-k (entries this pass had already contributed are taken out first, so no
// column can appear twice).  Exact for any input order; costs O(width * k) per dirty row, nothing when the list is empty.
// After the last pass the same kernel measures every repaired row again over all columns (off = 0, width = n): the
// entries of a repaired row would otherwise come from two arithmetics (tensor and direct), and exact duplicates could
// then be ranked out of index order.
__global__ void __launch_bounds__(256) knn_fix_kernel(long long* topk, float* thr, const int* dirty, const unsigned* dirty_cnt,
                                                      const float* x, int64_t ldx, const float* y, int64_t ldy, int k, int kk,
                                                      int64_t off, int64_t width, int family, int center)
{
  __shared__ float xs[320];
  __shared__ long long keys[512];
  __shared__ unsigned ncand;
  __shared__ float xstat[2];
  const int tid = threadIdx.x;
  const unsigned total = *dirty_cnt;
  for (unsigned d = blockIdx.x; d < total; d += gridDim.x) {
    const int64_t row = dirty[d];
    __syncthreads();
    if (tid == 0) {
      float mean = 0.f;
      if (family == 1 && center) {
        for (int t = 0; t < k; ++t) mean += x[row * ldx + t];
        mean /= static_cast<float>(k);
      }
      float nx = 0.f;
      for (int t = 0; t < k; ++t) { const float v = x[row * ldx + t] - mean; nx = fmaf(v, v, nx); }
      xstat[0] = mean; xstat[1] = nx;
    }
    __syncthreads();
    for (int t = tid; t < k; t += 256) xs[t] = x[row * ldx + t] - xstat[0];
    // the row's top-k without what this pass had put in
    for (int t = tid; t < 512; t += 256) {
      long long key = KEY_EMPTY;
      if (t < kk) {
        key = topk[row * kk + t];
        const long long j = key_index(key);
        if (key != KEY_EMPTY && j >= off && j < off + width) key = KEY_EMPTY;
      }
      keys[t] = key;
    }
    if (tid == 0) ncand = 0u;
    __syncthreads();
    for (int64_t j0 = 0; j0 < width; j0 += 256) {
      // (the k-th best of what is in keys[0, kk) bounds what can still enter; unsorted holes are +max)
      long long kth = 0;
      for (int t = 0; t < kk; ++t) kth = max(kth, keys[t]);
      const int64_t j = j0 + tid;
      bool appended   = false;
      if (j < width) {
        const float* yr = y + (off + j) * ldy;
        float val;
        if (family == 0) {
          float acc = 0.f;
          for (int t = 0; t < k; ++t) { const float df = xs[t] - __ldg(yr + t); acc = fmaf(df, df, acc); }
          val = acc;
        } else {
          float my = 0.f;
          if (center) {
            for (int t = 0; t < k; ++t) my += __ldg(yr + t);
            my /= static_cast<float>(k);
          }
          float dot = 0.f, ny = 0.f;
          for (int t = 0; t < k; ++t) { const float b = __ldg(yr + t) - my; dot = fmaf(xs[t], b, dot); ny = fmaf(b, b, ny); }
          val = 1.f - dot / sqrtf(xstat[1] * ny);
        }
        const long long key = key_pack(val, off + j);
        if (key < kth && val == val) {   // (kk + 256 <= 320 < 512)
          keys[kk + atomicAdd(&ncand, 1u)] = key;
          appended = true;
        }
      }
      // the branch must be block-uniform: a thread that read ncand after a barrier could see the next iteration's
      // atomicAdd of a faster warp, so the decision comes from the barrier itself
      if (__syncthreads_or(appended)) {   // block-wide bitonic sort of the 512 slots, smallest first
        for (int size = 2; size <= 512; size <<= 1)
          for (int stride = size >> 1; stride > 0; stride >>= 1) {
            const int t = tid;
            const int i = 2 * t - (t & (stride - 1)), jj = i + stride;
            const bool up = (i & size) == 0;
            const long long a = keys[i], c = keys[jj];
            if ((a > c) == up) { keys[i] = c; keys[jj] = a; }
            __syncthreads();
          }
        for (int t = kk + tid; t < 512; t += 256) keys[t] = KEY_EMPTY;
        if (tid == 0) ncand = 0u;
        __syncthreads();
      }
    }
    // final order (holes from the removed entries may have left the first kk slots unsorted)
    for (int size = 2; size <= 512; size <<= 1)
      for (int stride = size >> 1; stride > 0; stride >>= 1) {
        const int t = tid;
        const int i = 2 * t - (t & (stride - 1)), jj = i + stride;
        const bool up = (i & size) == 0;
        const long long a = keys[i], c = keys[jj];
        if ((a > c) == up) { keys[i] = c; keys[jj] = a; }
        __syncthreads();
      }
    for (int t = tid; t < kk; t += 256) topk[row * kk + t] = keys[t];
    if (tid == 0) thr[row] = key_bound(keys[kk - 1]);
  }
}

// sorted packed keys -> (index, distance) arrays: clamp at 0, optional sqrt
__global__ void knn_finalize_kernel(int64_t* out_idx, float* out_dist, const long long* topk, int64_t total, int do_sqrt)
{
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const long long key = topk[i];
  float d             = key_dist(key);
  d                   = d < 0.f ? 0.f : d;  // NaN propagates
  if (do_sqrt) d = sqrtf(d);
  out_idx[i]  = key == KEY_EMPTY ? -1 : static_cast<int64_t>(key_index(key));
  out_dist[i] = key == KEY_EMPTY ? __int_as_float(0x7f800000) : d;
}

}  // namespace b2d
