// raft::cluster::single_linkage -- header-only shim of the removed raft/cluster/single_linkage.cuh ([RECALLED], <= 25.12):
// single-linkage clustering on the kNN graph (LinkageDistance::KNN_GRAPH, b2d_single_linkage) or, for d = 2 and 3,
// exactly over all pairs (LinkageDistance::PAIRWISE, b2d_single_linkage_rbc; include/raft_b200.h).  float data, int
// indices.
//   mdspan form    X [m, d] row-major, dendrogram [m - 1, 2], labels [m] (any 1-d view with data_handle() / extent(0))
//   pointer form   X [m, n] contiguous, out->children / out->labels, optional deltas / sizes
// PAIRWISE at d > 3 throws raft::logic_error.  Temporaries come from the handle's workspace
// (raft/core/b200_workspace.hpp).  The call synchronises the handle's stream (the dendrogram is built on the host).
#pragma once
#include <cstddef>
#include <cstdint>
#include <optional>
#include <type_traits>

#include "../../raft_b200.h"
#include "../core/b200_workspace.hpp"
#include "../distance/distance.cuh"
#include "single_linkage_types.hpp"

namespace raft {
namespace cluster {

constexpr int DEFAULT_CONST_C = 15;   // n_nb = min(m, max(2, floor(log2 m) + c))

namespace detail {
// device scratch of one call: the C-ABI workspace, then deltas and sizes when the caller does not want them
inline void single_linkage_call(raft::resources const& handle, const float* x, int64_t ldx, int64_t m, int64_t d,
                                raft::distance::DistanceType metric, int c, int n_clusters, int* children,
                                float* deltas, int* sizes, int* labels, int* n_components)
{
  const size_t need = b2d_single_linkage_workspace_bytes(m, d, c);
  RAFT_EXPECTS(need != SIZE_MAX, "single_linkage: unsupported extents or c (n_nb must be at most 64)");
  const size_t tail = static_cast<size_t>(m > 1 ? m - 1 : 0) * 8 + 256;
  raft::b200::scoped_workspace ws(handle, need + tail);
  char* extra = static_cast<char*>(ws.data()) + (need + 255) / 256 * 256;
  if (!deltas) deltas = reinterpret_cast<float*>(extra);
  if (!sizes) sizes = reinterpret_cast<int*>(extra + static_cast<size_t>(m > 1 ? m - 1 : 0) * 4);
  int32_t nc_host = 0;
  raft::distance::detail::b2d_check(b2d_single_linkage(raft::resource::get_cuda_stream(handle), static_cast<int>(metric),
                                                       x, ldx, m, d, c, n_clusters, children, deltas, sizes, labels,
                                                       &nc_host, ws.data(), need));
  if (n_components) *n_components = nc_host;
}

// PAIRWISE: the ball cover's unexpanded distances, L2SqrtExpanded / L2Expanded mapped to them as Python's
// dbscan(algorithm="rbc") maps "euclidean" / "sqeuclidean"; c is not used
inline void single_linkage_pairwise_call(raft::resources const& handle, const float* x, int64_t ldx, int64_t m, int64_t d,
                                         raft::distance::DistanceType metric, int n_clusters, int* children,
                                         float* deltas, int* sizes, int* labels)
{
  using raft::distance::DistanceType;
  RAFT_EXPECTS(d == 2 || d == 3,
               "single_linkage: LinkageDistance::PAIRWISE is exact on the random ball cover, which supports d = 2 and "
               "d = 3; use LinkageDistance::KNN_GRAPH for d > 3");
  DistanceType um = metric;
  if (metric == DistanceType::L2SqrtExpanded) um = DistanceType::L2SqrtUnexpanded;
  if (metric == DistanceType::L2Expanded) um = DistanceType::L2Unexpanded;
  RAFT_EXPECTS(um == DistanceType::L2SqrtUnexpanded || um == DistanceType::L2Unexpanded,
               "single_linkage: LinkageDistance::PAIRWISE supports the L2 metrics");
  const size_t need = b2d_single_linkage_rbc_workspace_bytes(m, d, 0);
  RAFT_EXPECTS(need != SIZE_MAX, "single_linkage: unsupported extents (m must be in [1, 2^30))");
  const size_t tail = static_cast<size_t>(m > 1 ? m - 1 : 0) * 8 + 256;
  raft::b200::scoped_workspace ws(handle, need + tail);
  char* extra = static_cast<char*>(ws.data()) + (need + 255) / 256 * 256;
  if (!deltas) deltas = reinterpret_cast<float*>(extra);
  if (!sizes) sizes = reinterpret_cast<int*>(extra + static_cast<size_t>(m > 1 ? m - 1 : 0) * 4);
  raft::distance::detail::b2d_check(b2d_single_linkage_rbc(raft::resource::get_cuda_stream(handle), static_cast<int>(um),
                                                           x, ldx, m, d, 0, 0, n_clusters, children, deltas, sizes,
                                                           labels, ws.data(), need));
}
}  // namespace detail

/** Single-linkage clustering of the rows of X: dendrogram [m - 1, 2] (merge t creates cluster m + t; smaller child
 * first) and the labels of n_clusters flat clusters, numbered in order of each cluster's smallest row.
 * KNN_GRAPH: c sets the kNN graph's n_nb = min(m, max(2, floor(log2 m) + c)) (default 15); metric L2Expanded or
 * L2SqrtExpanded.  PAIRWISE (d = 2 or 3): the exact single linkage over all pairs; c is ignored; metric
 * L2SqrtUnexpanded or L2Unexpanded (L2SqrtExpanded / L2Expanded are taken as those: the distances are always the
 * unexpanded ones). */
template <typename value_idx, typename value_t, LinkageDistance dist_type = LinkageDistance::KNN_GRAPH, typename LabelsView>
void single_linkage(raft::resources const& handle, raft::device_matrix_view<const value_t, value_idx, raft::row_major> X,
                    raft::device_matrix_view<value_idx, value_idx, raft::row_major> dendrogram, LabelsView labels,
                    raft::distance::DistanceType metric, size_t n_clusters,
                    std::optional<int> c = std::make_optional<int>(DEFAULT_CONST_C))
{
  static_assert(std::is_same<value_t, float>::value && std::is_same<value_idx, int>::value,
                "raft_b200 single_linkage: float data, int indices");
  const int64_t m = X.extent(0), d = X.extent(1);
  RAFT_EXPECTS(dendrogram.extent(0) == (m > 1 ? m - 1 : 0) && dendrogram.extent(1) == 2,
               "single_linkage: dendrogram must be [m - 1, 2]");
  RAFT_EXPECTS(static_cast<int64_t>(labels.extent(0)) == m, "single_linkage: labels must have m entries");
  if (dist_type == LinkageDistance::PAIRWISE) {
    detail::single_linkage_pairwise_call(handle, X.data_handle(), d, m, d, metric, static_cast<int>(n_clusters),
                                         dendrogram.data_handle(), nullptr, nullptr, labels.data_handle());
    return;
  }
  detail::single_linkage_call(handle, X.data_handle(), d, m, d, metric, c.value_or(DEFAULT_CONST_C),
                              static_cast<int>(n_clusters), dendrogram.data_handle(), nullptr, nullptr,
                              labels.data_handle(), nullptr);
}

/** Pointer form: X [m, n] row-major contiguous; fills out->children, out->labels, out->n_connected_components (1 for
 * PAIRWISE) and out's extents.  deltas / sizes [m - 1]: optional device outputs of the merge distances and cluster
 * sizes. */
template <typename value_idx, typename value_t, LinkageDistance dist_type = LinkageDistance::KNN_GRAPH>
void single_linkage(raft::resources const& handle, const value_t* X, size_t m, size_t n,
                    raft::distance::DistanceType metric, linkage_output<value_idx>* out, int c, size_t n_clusters,
                    value_t* deltas = nullptr, value_idx* sizes = nullptr)
{
  static_assert(std::is_same<value_t, float>::value && std::is_same<value_idx, int>::value,
                "raft_b200 single_linkage: float data, int indices");
  RAFT_EXPECTS(out != nullptr, "single_linkage: null output");
  int ncomp = 1;
  if (dist_type == LinkageDistance::PAIRWISE)
    detail::single_linkage_pairwise_call(handle, X, static_cast<int64_t>(n), static_cast<int64_t>(m),
                                         static_cast<int64_t>(n), metric, static_cast<int>(n_clusters), out->children,
                                         deltas, sizes, out->labels);
  else
    detail::single_linkage_call(handle, X, static_cast<int64_t>(n), static_cast<int64_t>(m), static_cast<int64_t>(n), metric,
                              c, static_cast<int>(n_clusters), out->children, deltas, sizes, out->labels, &ncomp);
  out->m                      = static_cast<value_idx>(m);
  out->n_leaves               = static_cast<value_idx>(m);
  out->n_clusters             = static_cast<value_idx>(n_clusters);
  out->n_connected_components = ncomp;
}

}  // namespace cluster
}  // namespace raft
