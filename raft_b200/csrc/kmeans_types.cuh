// Constants, control words and the sorted cluster ranges of k-means (kmeans.cuh), without kernels: the label sort and scan of the host code
// serve single linkage and DBSCAN too.
#pragma once
#include <cstdint>

namespace b2d {

constexpr int kKmThreads   = 256;
constexpr int kKmSortItems = 8;                            // rows per thread of one radix-sorted sub-block
constexpr int kKmSub       = kKmThreads * kKmSortItems;    // 2048 rows
constexpr int kKmScanTile  = kKmThreads * 16;              // histogram words per scan tile
constexpr int kKmChunk     = 256;                          // sorted rows per fp64 summation chunk
constexpr int kKmCols      = 128;                          // columns per summation / finalize CTA
constexpr int kKmPpBlock   = 1024;                         // rows per sampling block of k-means++
constexpr int kKmPpMaxTrials = 32;

// control words of a fit (one copy in the workspace)
struct KmCtrl {
  unsigned run;         // 1 while the fit is running (the run word of every conditional launch)
  unsigned bad;         // a negative weight, a NaN weight or a zero weight sum: the inertia is NaN
  int iter;             // iterations that ran
  unsigned total;       // rows with a label in [0, n_clusters)
  double prior;         // inertia of the previous iteration
  double inertia;       // result of km_finish_kernel
  double wscale;        // m / sum of the weights
  unsigned take;        // n_init: this run is the best so far
  int best_iter;
  double best_inertia;
  int pp_last;          // k-means++: row of the centroid chosen last (-1: none yet)
  int pp_trials;        // k-means++: trials of the current round
  int pp_cand[kKmPpMaxTrials];
};

#ifdef __CUDACC__
// rows [cs, ce) of cluster c in the sorted order, from the cursors the stable counting sort leaves (km_scatter_kernel)
__device__ __forceinline__ void km_cluster_range(const unsigned* cur, int64_t nblk, int c, int64_t& cs, int64_t& ce)
{
  cs = c > 0 ? cur[static_cast<int64_t>(c) * nblk - 1] : 0;
  ce = cur[static_cast<int64_t>(c) * nblk + nblk - 1];
}
#endif

}  // namespace b2d
