// raft::cluster::dbscan -- header-only DBSCAN in the shape of cuML's ML::Dbscan::fit, dispatching through b2d_dbscan_fit
// and, for EpsNnMethod::RBC (2-D and 3-D points on the random ball cover), b2d_dbscan_rbc_fit (include/raft_b200.h).
// float data, int labels.
//   mdspan form    X [m, d] row-major, labels [m] and optional core_sample_indices [m]
//                  (any 1-d views with data_handle() / extent(0))
//   pointer form   x [n_rows, n_cols] contiguous, cuML's argument order
// Labels are numbered 0, 1, ... in order of each cluster's smallest row, -1 is noise; core_sample_indices lists the core
// rows ascending, padded with -1.  The result does not depend on max_bytes_per_batch (0: 2^30 bytes of adjacency per
// batch).  Temporaries come from the handle's workspace (raft/core/b200_workspace.hpp); the call only enqueues work.
#pragma once
#include <cstddef>
#include <cstdint>
#include <optional>
#include <type_traits>

#include "../../raft_b200.h"
#include "../core/b200_workspace.hpp"
#include "../distance/distance.cuh"

namespace raft {
namespace cluster {
namespace dbscan {

/** How the epsilon neighbourhoods are found (cuML's ML::Dbscan::EpsNnMethod): every pair on the tensor path, or the
 * random ball cover (d = 2 or 3, the unexpanded metrics L2SqrtUnexpanded and L2Unexpanded). */
enum class EpsNnMethod { BRUTE_FORCE, RBC };

namespace detail {
inline void fit_call(raft::resources const& handle, const float* x, int64_t ldx, int64_t m, int64_t d, float eps,
                     int min_samples, raft::distance::DistanceType metric, int* labels, int* core_sample_indices,
                     int64_t max_bytes_per_batch)
{
  RAFT_EXPECTS(max_bytes_per_batch >= 0, "dbscan: max_bytes_per_batch must be >= 0");
  const size_t need = b2d_dbscan_workspace_bytes(m, d, max_bytes_per_batch);
  RAFT_EXPECTS(need != SIZE_MAX, "dbscan: negative extents");
  raft::b200::scoped_workspace ws(handle, need);
  raft::distance::detail::b2d_check(b2d_dbscan_fit(raft::resource::get_cuda_stream(handle), static_cast<int>(metric), x,
                                                   ldx, m, d, static_cast<double>(eps), min_samples, max_bytes_per_batch,
                                                   labels, core_sample_indices, nullptr, ws.data(), need));
}

inline void rbc_fit_call(raft::resources const& handle, const float* x, int64_t ldx, int64_t m, int64_t d, float eps,
                         int min_samples, raft::distance::DistanceType metric, int* labels, int* core_sample_indices,
                         int64_t n_landmarks, uint64_t seed)
{
  const size_t need = b2d_dbscan_rbc_workspace_bytes(m, d, n_landmarks);
  raft::b200::scoped_workspace ws(handle, need != SIZE_MAX ? need : 0);   // invalid extents: the fit says which
  raft::distance::detail::b2d_check(b2d_dbscan_rbc_fit(raft::resource::get_cuda_stream(handle), static_cast<int>(metric),
                                                       x, ldx, m, d, static_cast<double>(eps), min_samples, n_landmarks,
                                                       seed, labels, core_sample_indices, nullptr, ws.data(),
                                                       need != SIZE_MAX ? need : 0));
}
}  // namespace detail

/** DBSCAN of the rows of X: labels [m] (-1: noise) and, optionally, core_sample_indices [m].  metric: L2SqrtExpanded
 * (distance <= eps, the default), L2Expanded (squared distance <= eps) or CosineExpanded. */
template <typename LabelsView, typename CoreView = LabelsView>
void fit(raft::resources const& handle, raft::device_matrix_view<const float, int, raft::row_major> X, LabelsView labels,
         float eps, int min_samples,
         raft::distance::DistanceType metric = raft::distance::DistanceType::L2SqrtExpanded,
         std::optional<CoreView> core_sample_indices = std::nullopt, int64_t max_bytes_per_batch = 0)
{
  const int64_t m = X.extent(0), d = X.extent(1);
  RAFT_EXPECTS(static_cast<int64_t>(labels.extent(0)) == m, "dbscan: labels must have m entries");
  RAFT_EXPECTS(!core_sample_indices || static_cast<int64_t>(core_sample_indices->extent(0)) == m,
               "dbscan: core_sample_indices must have m entries");
  const int64_t ldx = m > 1 ? static_cast<int64_t>(X.stride(0)) : d;
  detail::fit_call(handle, X.data_handle(), ldx, m, d, eps, min_samples, metric, labels.data_handle(),
                   core_sample_indices ? core_sample_indices->data_handle() : nullptr, max_bytes_per_batch);
}

/** Pointer form in cuML's argument order: x [n_rows, n_cols] row-major contiguous, labels [n_rows], optional
 * core_sample_indices [n_rows]. */
inline void fit(raft::resources const& handle, const float* x, int n_rows, int n_cols, float eps, int min_pts,
                raft::distance::DistanceType metric, int* labels, int* core_sample_indices = nullptr,
                size_t max_bytes_per_batch = 0)
{
  detail::fit_call(handle, x, n_cols, n_rows, n_cols, eps, min_pts, metric, labels, core_sample_indices,
                   static_cast<int64_t>(max_bytes_per_batch));
}

/** DBSCAN of the rows of X by `method`.  RBC: X is [m, 2] or [m, 3], metric L2SqrtUnexpanded (distance <= eps, the
 * default) or L2Unexpanded (squared distance <= eps), on a ball cover of n_landmarks landmarks (0: ceil(sqrt(m))) drawn
 * from seed; the result depends on neither.  BRUTE_FORCE: the form above, with its metrics. */
template <typename LabelsView, typename CoreView = LabelsView>
void fit(raft::resources const& handle, raft::device_matrix_view<const float, int, raft::row_major> X, LabelsView labels,
         float eps, int min_samples, EpsNnMethod method,
         raft::distance::DistanceType metric = raft::distance::DistanceType::L2SqrtUnexpanded,
         std::optional<CoreView> core_sample_indices = std::nullopt, int64_t n_landmarks = 0, uint64_t seed = 0)
{
  if (method == EpsNnMethod::BRUTE_FORCE) {
    fit(handle, X, labels, eps, min_samples, metric, core_sample_indices);
    return;
  }
  const int64_t m = X.extent(0), d = X.extent(1);
  RAFT_EXPECTS(static_cast<int64_t>(labels.extent(0)) == m, "dbscan: labels must have m entries");
  RAFT_EXPECTS(!core_sample_indices || static_cast<int64_t>(core_sample_indices->extent(0)) == m,
               "dbscan: core_sample_indices must have m entries");
  const int64_t ldx = m > 1 ? static_cast<int64_t>(X.stride(0)) : d;
  detail::rbc_fit_call(handle, X.data_handle(), ldx, m, d, eps, min_samples, metric, labels.data_handle(),
                       core_sample_indices ? core_sample_indices->data_handle() : nullptr, n_landmarks, seed);
}

/** Pointer form in cuML's argument order with the method trailing.  RBC has no batches: max_bytes_per_batch must be 0. */
inline void fit(raft::resources const& handle, const float* x, int n_rows, int n_cols, float eps, int min_pts,
                raft::distance::DistanceType metric, int* labels, int* core_sample_indices, size_t max_bytes_per_batch,
                EpsNnMethod method, int64_t n_landmarks = 0, uint64_t seed = 0)
{
  if (method == EpsNnMethod::BRUTE_FORCE) {
    fit(handle, x, n_rows, n_cols, eps, min_pts, metric, labels, core_sample_indices, max_bytes_per_batch);
    return;
  }
  RAFT_EXPECTS(max_bytes_per_batch == 0, "dbscan: EpsNnMethod::RBC has no batches (max_bytes_per_batch must be 0)");
  detail::rbc_fit_call(handle, x, n_cols, n_rows, n_cols, eps, min_pts, metric, labels, core_sample_indices, n_landmarks,
                       seed);
}

}  // namespace dbscan
}  // namespace cluster
}  // namespace raft
