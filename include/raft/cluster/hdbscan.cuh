// raft::cluster::hdbscan -- header-only HDBSCAN of 2-D and 3-D points on the random ball cover, in the shape of cuML's
// ML::HDBSCAN::fit, dispatching through b2d_hdbscan_rbc_fit (include/raft_b200.h).  float data, int labels.
//   X [m, 2] or [m, 3] row-major (any row pitch), labels [m] and probabilities [m] (any 1-d views with data_handle() /
//   extent(0)); metric L2SqrtUnexpanded (the default) or L2Unexpanded, L2SqrtExpanded and L2Expanded taken as those.
// Labels are numbered 0, 1, ... in order of each cluster's smallest row, -1 is noise.  The result is
// sklearn.cluster.HDBSCAN's on the ball cover's pair distances with the mutual-reachability tree merged in the order
// (weight, min row, max row); it does not depend on n_landmarks (0: ceil(sqrt(m))) or seed.  Temporaries come from the
// handle's workspace (raft/core/b200_workspace.hpp); the call synchronises the handle's stream.
#pragma once
#include <cstddef>
#include <cstdint>

#include "../../raft_b200.h"
#include "../core/b200_workspace.hpp"
#include "../distance/distance.cuh"

namespace raft {
namespace cluster {
namespace hdbscan {

enum class cluster_selection_method { EOM = B2D_HDBSCAN_EOM, LEAF = B2D_HDBSCAN_LEAF };

/** cuML's HDBSCANParams without alpha and max_cluster_size.  min_samples = 0 means min_cluster_size. */
struct params {
  int min_cluster_size                    = 5;
  int min_samples                         = 0;
  double cluster_selection_epsilon        = 0.0;
  cluster_selection_method method         = cluster_selection_method::EOM;
  bool allow_single_cluster               = false;
  int64_t n_landmarks                     = 0;
  uint64_t seed                           = 0;
};

namespace detail {
inline int fit_call(raft::resources const& handle, const float* x, int64_t ldx, int64_t m, int64_t d, const params& p,
                    raft::distance::DistanceType metric, int* labels, float* probabilities)
{
  using raft::distance::DistanceType;
  if (metric == DistanceType::L2SqrtExpanded) metric = DistanceType::L2SqrtUnexpanded;
  if (metric == DistanceType::L2Expanded) metric = DistanceType::L2Unexpanded;
  const size_t need = b2d_hdbscan_rbc_workspace_bytes(m, d, p.n_landmarks);
  const size_t ws   = need != SIZE_MAX ? need : 0;   // invalid extents: the fit says which
  const size_t tree = m > 1 ? (static_cast<size_t>(m - 1) * 4 + 255) / 256 * 256 : 0;
  raft::b200::scoped_workspace buf(handle, ws + 3 * tree);   // the workspace, then the tree's three arrays
  char* base = static_cast<char*>(buf.data());
  int32_t n_clusters = 0;
  raft::distance::detail::b2d_check(b2d_hdbscan_rbc_fit(
    raft::resource::get_cuda_stream(handle), static_cast<int>(metric), x, ldx, m, d,
    p.min_samples > 0 ? p.min_samples : p.min_cluster_size, p.min_cluster_size, p.cluster_selection_epsilon,
    static_cast<int>(p.method), p.allow_single_cluster ? 1 : 0, p.n_landmarks, p.seed, labels, probabilities,
    m > 1 ? reinterpret_cast<int32_t*>(base + ws) : nullptr, m > 1 ? reinterpret_cast<int32_t*>(base + ws + tree) : nullptr,
    m > 1 ? reinterpret_cast<float*>(base + ws + 2 * tree) : nullptr, &n_clusters, base, ws));
  return n_clusters;
}
}  // namespace detail

/** HDBSCAN of the rows of X: labels [m] (-1: noise) and probabilities [m]; returns the number of clusters. */
template <typename LabelsView, typename ProbView>
int fit(raft::resources const& handle, raft::device_matrix_view<const float, int, raft::row_major> X, LabelsView labels,
        ProbView probabilities, const params& p = params{},
        raft::distance::DistanceType metric = raft::distance::DistanceType::L2SqrtUnexpanded)
{
  const int64_t m = X.extent(0), d = X.extent(1);
  RAFT_EXPECTS(static_cast<int64_t>(labels.extent(0)) == m, "hdbscan: labels must have m entries");
  RAFT_EXPECTS(static_cast<int64_t>(probabilities.extent(0)) == m, "hdbscan: probabilities must have m entries");
  const int64_t ldx = m > 1 ? static_cast<int64_t>(X.stride(0)) : d;
  return detail::fit_call(handle, X.data_handle(), ldx, m, d, p, metric, labels.data_handle(),
                          probabilities.data_handle());
}

/** Pointer form in cuML's argument order: x [n_rows, n_cols] row-major contiguous, labels [n_rows], probabilities
 * [n_rows]; returns the number of clusters. */
inline int fit(raft::resources const& handle, const float* x, int n_rows, int n_cols, raft::distance::DistanceType metric,
               const params& p, int* labels, float* probabilities)
{
  return detail::fit_call(handle, x, n_cols, n_rows, n_cols, p, metric, labels, probabilities);
}

}  // namespace hdbscan
}  // namespace cluster
}  // namespace raft
