// HDBSCAN for 2-D and 3-D points (single_linkage.cu, the one file that includes this header): core distances by the
// ball cover's kNN walk, then the mutual-reachability minimum spanning tree by the EMST's Borůvka rounds
// (single_linkage_rbc.cuh) with the walker's Mr weight (DESIGN.md K22).  Everything is in the s domain: core[p] is the
// min_samples-th smallest s of the row at position p (the row itself included), and pair (i, j) weighs
// w = max(core_i, core_j, s(i, j)).  The tree stages run on the host (hdbscan_tree.cuh).  approximate_predict places new
// points in a fitted model (hdb_predict_kernel, DESIGN.md K23).
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

// A fitted model as the predict kernel reads it (its regions: hdb_model_layout in single_linkage.cu): the fit's index,
// core by position, cmin by ball, pos by row, and the condensed tree of HdbTreeExport (rows by caller row, clusters by
// id).
struct HdbModelHead {
  double thr;
  int single_root;
  int n_clusters;
};
struct HdbModel {
  BcIndex ix;
  float* core;          // [m] by position
  float* cmin;          // [nl]
  int* pos;             // [m] the position of every caller row
  int* row_parent;      // [m]
  double* row_lambda;   // [m]
  int *parent, *owner, *label;   // [m] (clusters: at most m)
  double *birth, *death;         // [m]
  HdbModelHead* head;
};

// One warp per query qi: approximate_predict's contract (include/raft_b200.h).  The core walk is hdb_core_kernel's (the
// list kept); the MR walk is SlrWalk's Pred mode, its bound seeded by the best (w, s, row) of that list, so it starts at
// a real candidate.  Lane 0 then walks the condensed tree up from the neighbour's parent cluster and applies the fit's
// label rule.  A query with a non-finite coordinate is noise with no neighbour.
template <int D>
__global__ void __launch_bounds__(kBcWarps * 32) hdb_predict_kernel(HdbModel M, int n, int nl, int k, int root,
                                                                    const float* qs, int64_t ldq, int mq, int* labels,
                                                                    float* prob, int* nn_rows, float* nn_w, int smem)
{
  const float *lm, *rhi;
  bc_stage<D>(M.ix, nl, smem, &lm, &rhi);
  const int lane = threadIdx.x & 31;
  const int qi   = blockIdx.x * kBcWarps + (threadIdx.x >> 5);
  if (qi >= mq) return;
  SlrWalk<D, true, true> w(M.ix, nullptr, nullptr, nullptr);
  bool ok = bc_query<D>(qs + static_cast<int64_t>(qi) * ldq, w.q);
  for (int c = 0; c < D; ++c) ok = ok && isfinite(w.q[c]);
  if (!ok) {
    if (lane == 0) {
      labels[qi] = -1;
      prob[qi]   = 0.f;
      if (nn_rows) nn_rows[qi] = -1;
      if (nn_w) nn_w[qi] = BC_INF;
    }
    return;
  }
  BcKnn<D> kn{M.ix, w.q, k, 0, lane};
  bc_walk<D, true>(M.ix, n, nl, lm, rhi, w.q, lane, kn);
  w.lane = lane;
  w.core = M.core;
  w.cmin = M.cmin;
  w.cq   = key_bound(kn.kth);
  // the seed: the best of the list's k rows, lane l holding slots l and l + 32
  for (int h = 0; h < 2; ++h) {
    const long long e = h ? kn.list.a1 : kn.list.a0;
    if (lane + 32 * h < k && e != KEY_EMPTY) {
      const int j    = static_cast<int>(key_index(e));
      const float s  = key_dist(e);
      const long long k1 = key_pack(fmaxf(fmaxf(w.cq, M.core[M.pos[j]]), s), __float_as_int(s));
      if (slr_before(k1, j, w.b1, w.b2)) { w.b1 = k1; w.b2 = j; }
    }
  }
  for (int o = 16; o > 0; o >>= 1) {
    const long long o1 = __shfl_xor_sync(0xffffffffu, w.b1, o);
    const int o2       = __shfl_xor_sync(0xffffffffu, w.b2, o);
    if (slr_before(o1, o2, w.b1, w.b2)) { w.b1 = o1; w.b2 = o2; }
  }
  w.bound();
  bc_walk<D, true>(M.ix, n, nl, lm, rhi, w.q, lane, w);
  if (lane != 0) return;
  const int j   = w.b2;
  const float ws = key_dist(w.b1);
  const float W  = root ? __fsqrt_rn(ws) : ws;
  const double wd = W;
  double lam      = wd > 0.0 ? 1.0 / wd : static_cast<double>(BC_INF);
  lam             = fmin(lam, M.row_lambda[j]);
  int p = M.row_parent[j];
  while (p != 0 && M.birth[p] > lam) p = M.parent[p];
  const int o = M.owner[p];
  int lab     = M.label[o];
  if (o == 0 && !(M.head->single_root && lam >= M.head->thr)) lab = -1;
  float pr = 0.f;
  if (lab >= 0) {
    const double md = M.death[o];
    pr = static_cast<float>(md == 0.0 || isinf(lam) ? 1.0 : fmin(lam, md) / md);
  }
  labels[qi] = lab;
  prob[qi]   = pr;
  if (nn_rows) nn_rows[qi] = j;
  if (nn_w) nn_w[qi] = W;
}

}  // namespace b2d
