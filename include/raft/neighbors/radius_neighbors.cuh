// raft::neighbors::radius_neighbors_count / radius_neighbors_fill -- shim over b2d_radius_neighbors_count / _fill
// (include/raft_b200.h).  A project API: RAFT has no radius-neighbours entry point, so no upstream signature is claimed.
// For every row i of queries [m, d] the rows j of dataset [n, d] with d(i, j) <= radius, as CSR: indptr int64 [m + 1],
// indices int64 [nnz], distances float [nnz], each row in ascending (distance, index) order.  d(i, j) is exactly the value
// pairwise_distance(queries, dataset, metric) returns, metric L2Expanded (radius squared), L2SqrtExpanded, CosineExpanded
// or CorrelationExpanded; a NaN distance never matches, nor does anything for a NaN or negative radius.
// Two calls: count writes indptr; the caller reads nnz = indptr[m] (a copy to the host), sizes indices / distances to nnz
// and calls fill with the same inputs.  Both run on the handle's stream with scratch from its workspace, and neither
// synchronises.  d <= 320 and nnz <= 2^31 - 1 (else raft::logic_error: split the queries).
#pragma once
#include "../distance/distance.cuh"

namespace raft {
namespace neighbors {

template <typename matrix_idx_t>
void radius_neighbors_count(raft::resources const& handle,
                            raft::device_matrix_view<const float, matrix_idx_t, raft::row_major> queries,
                            raft::device_matrix_view<const float, matrix_idx_t, raft::row_major> dataset,
                            raft::device_vector_view<int64_t, matrix_idx_t> indptr, float radius,
                            raft::distance::DistanceType metric)
{
  const int64_t m = queries.extent(0), n = dataset.extent(0), d = queries.extent(1);
  RAFT_EXPECTS(dataset.extent(1) == queries.extent(1), "queries and dataset must have the same number of columns");
  RAFT_EXPECTS(static_cast<int64_t>(indptr.extent(0)) == m + 1, "indptr must have m + 1 entries");
  const size_t need = b2d_radius_neighbors_workspace_bytes(m, n, d, 0);
  RAFT_EXPECTS(need != SIZE_MAX, "negative extent");
  raft::b200::scoped_workspace ws(handle, need);
  raft::distance::detail::b2d_check(b2d_radius_neighbors_count(raft::resource::get_cuda_stream(handle),
                                                               indptr.data_handle(), static_cast<int>(metric),
                                                               queries.data_handle(), d, dataset.data_handle(), d, m,
                                                               n, d, radius, ws.data(), need));
}

template <typename matrix_idx_t>
void radius_neighbors_fill(raft::resources const& handle,
                           raft::device_matrix_view<const float, matrix_idx_t, raft::row_major> queries,
                           raft::device_matrix_view<const float, matrix_idx_t, raft::row_major> dataset,
                           raft::device_vector_view<const int64_t, matrix_idx_t> indptr,
                           raft::device_vector_view<int64_t, matrix_idx_t> indices,
                           raft::device_vector_view<float, matrix_idx_t> distances, float radius,
                           raft::distance::DistanceType metric)
{
  const int64_t m = queries.extent(0), n = dataset.extent(0), d = queries.extent(1);
  const int64_t nnz = indices.extent(0);
  RAFT_EXPECTS(dataset.extent(1) == queries.extent(1), "queries and dataset must have the same number of columns");
  RAFT_EXPECTS(static_cast<int64_t>(indptr.extent(0)) == m + 1, "indptr must have m + 1 entries");
  RAFT_EXPECTS(static_cast<int64_t>(distances.extent(0)) == nnz, "indices and distances must have nnz entries");
  const size_t need = b2d_radius_neighbors_workspace_bytes(m, n, d, nnz);
  RAFT_EXPECTS(need != SIZE_MAX, "negative extent");
  raft::b200::scoped_workspace ws(handle, need);
  raft::distance::detail::b2d_check(b2d_radius_neighbors_fill(raft::resource::get_cuda_stream(handle),
                                                              indptr.data_handle(), nnz, indices.data_handle(),
                                                              distances.data_handle(), static_cast<int>(metric),
                                                              queries.data_handle(), d, dataset.data_handle(), d, m, n,
                                                              d, radius, ws.data(), need));
}

}  // namespace neighbors
}  // namespace raft
