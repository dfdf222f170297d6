// HDBSCAN for 2-D and 3-D points (single_linkage.cu, the one file that includes this header): core distances by the
// ball cover's kNN walk, then the mutual-reachability minimum spanning tree by the EMST's Borůvka rounds
// (single_linkage_rbc.cuh) with the walker's Mr weight (DESIGN.md K22).  Everything is in the s domain: core[p] is the
// min_samples-th smallest s of the row at position p (the row itself included), and pair (i, j) weighs
// w = max(core_i, core_j, s(i, j)).  The tree stages run on the host (hdbscan_tree.cuh).
#pragma once
#include "single_linkage_rbc.cuh"

namespace b2d {

// One warp per position t: core[t] = the k-th smallest s from the row at t (bc_knn_kernel's walk, root = 0), none of the
// list written out
template <int D>
__global__ void __launch_bounds__(kBcWarps * 32) hdb_core_kernel(BcIndex ix, int n, int nl, int k, float* core, int smem)
{
  const float *lm, *rhi;
  bc_stage<D>(ix, nl, smem, &lm, &rhi);
  const int lane = threadIdx.x & 31;
  const int t    = blockIdx.x * kBcWarps + (threadIdx.x >> 5);
  if (t >= n) return;
  float q[D];
  BcKnn<D> st{ix, q, k, 0, lane};
  if (bc_query<D>(ix.pts + static_cast<int64_t>(t) * D, q)) bc_walk<D, true>(ix, n, nl, lm, rhi, q, lane, st);
  if (lane == 0) core[t] = key_bound(st.kth);
}

// cmin[b] = the smallest core distance of ball b's members (+inf for an empty ball); one warp per ball
__global__ void hdb_cmin_kernel(const int* off, const float* core, int nl, float* cmin)
{
  const int lane = threadIdx.x & 31;
  const int b    = blockIdx.x * kBcWarps + (threadIdx.x >> 5);
  if (b >= nl) return;
  float mn = BC_INF;
  for (int p = off[b] + lane; p < off[b + 1]; p += 32) mn = fminf(mn, core[p]);
  for (int o = 16; o > 0; o >>= 1) mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
  if (lane == 0) cmin[b] = mn;
}

// slr_walk_kernel with the mutual-reachability weight: the first edge in the order (w, min row, max row) from t's row to
// a row of another colour.  Besides the K19 margin (valid at bc_dhi(bound) since w >= s), three prunes, each strict
// against the bound: the whole row when its core exceeds it, a ball when max(core, the ball's cmin) does, a member when
// its core does, before its s is formed.
template <int D>
__global__ void __launch_bounds__(kBcWarps * 32) hdb_walk_kernel(const SlCtrl* ctrl, BcIndex ix, int n, int nl,
                                                                 const int* colour, const int* bcol, const float* core,
                                                                 const float* cmin, long long* best1, int* best2,
                                                                 long long* cand1, int* cand2, int smem)
{
  if (!sl_running(ctrl)) return;
  const float *lm, *rhi;
  bc_stage<D>(ix, nl, smem, &lm, &rhi);
  const int t = blockIdx.x * kBcWarps + (threadIdx.x >> 5);
  if (t >= n) return;
  const int col = colour[t];
  SlrWalk<D, true> w(ix, colour, bcol, best1 + col);
  w.lane = threadIdx.x & 31;
  w.row  = ix.ids[t];
  w.col  = col;
  w.core = core;
  w.cmin = cmin;
  w.cq   = core[t];
  if (bc_query<D>(ix.pts + static_cast<int64_t>(t) * D, w.q)) bc_walk<D, true>(ix, n, nl, lm, rhi, w.q, w.lane, w);
  if (w.lane == 0) {
    cand1[t] = w.b1;
    cand2[t] = w.b2;
    best2[t] = INT_MAX;
  }
}

}  // namespace b2d
