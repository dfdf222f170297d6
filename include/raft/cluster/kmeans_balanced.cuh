// raft::cluster::kmeans_balanced -- header-only shim of the removed raft/cluster/kmeans_balanced.cuh ([RECALLED],
// <= 25.12): hierarchical balanced k-means under L2Expanded, dispatching through b2d_kmeans_balanced_fit and
// b2d_kmeans_predict (include/raft_b200.h).  float data only.
//   fit          centroids [n_clusters, k] out (n_clusters = centroids.extent(0))
//   predict      labels [m] on the device: the nearest centroid (ties to the smaller index, -1 for a row with NaN)
//   fit_predict  both; the labels are the assignment the fit's last update used (predict on the returned centroids
//                can move the rows near a boundary)
// Labels are a device vector view of int32_t or uint32_t (the same bits).  Any metric but L2Expanded throws raft::logic_error.  Departures from
// the recalled signatures: no mapping_op (the input is float; MathT is float), and kmeans_balanced_params carries a seed.
// Temporaries come from the handle's workspace (raft/core/b200_workspace.hpp).
#pragma once
#include <cstdint>
#include <type_traits>

#include "../../raft_b200.h"
#include "../core/b200_workspace.hpp"
#include "../distance/distance.cuh"
#include "kmeans_balanced_types.hpp"

namespace raft {
namespace cluster {
namespace kmeans_balanced {

namespace detail {
template <typename IndexT, typename Layout>
int64_t row_pitch(raft::device_matrix_view<const float, IndexT, Layout> v)
{
  bool row_major;
  int64_t ld;
  raft::distance::detail::view_layout(v, row_major, ld);
  RAFT_EXPECTS(row_major, "kmeans_balanced: X must be row-major");
  return ld;
}
inline void check_params(const kmeans_balanced_params& p)
{
  RAFT_EXPECTS(p.metric == raft::distance::DistanceType::L2Expanded,
               "kmeans_balanced: only the L2Expanded metric is supported");
  RAFT_EXPECTS(p.n_iters >= 1 && p.n_iters <= 0x7fffffffu, "kmeans_balanced: n_iters must be in [1, 2^31)");
}
// labels: any 1-d device mdspan of int32_t or uint32_t (raft::device_vector_view<LabelT, IndexT>)
template <typename LabelsView>
void check_label_view()
{
  using LabelT = typename std::remove_cv<typename LabelsView::element_type>::type;
  static_assert(LabelsView::rank() == 1, "raft_b200 kmeans_balanced: labels must be a vector view");
  static_assert(std::is_same<LabelT, int32_t>::value || std::is_same<LabelT, uint32_t>::value,
                "raft_b200 kmeans_balanced: int32_t or uint32_t labels");
}

template <typename IndexT, typename Layout>
void fit_impl(raft::resources const& handle, const kmeans_balanced_params& params,
              raft::device_matrix_view<const float, IndexT, Layout> X, raft::device_matrix_view<float, IndexT> centroids,
              int32_t* labels)
{
  check_params(params);
  const int64_t m = X.extent(0), k = X.extent(1), nc = centroids.extent(0);
  RAFT_EXPECTS(centroids.extent(1) == k, "kmeans_balanced: centroids must have n_features columns");
  const int64_t ldx = row_pitch(X);
  const size_t need = b2d_kmeans_balanced_workspace_bytes(m, k, nc);
  RAFT_EXPECTS(need != SIZE_MAX, "kmeans_balanced: invalid extents");
  raft::b200::scoped_workspace ws(handle, need);
  raft::distance::detail::b2d_check(b2d_kmeans_balanced_fit(
    raft::resource::get_cuda_stream(handle), static_cast<int>(nc), static_cast<int>(params.n_iters), params.seed,
    X.data_handle(), ldx, m, k, centroids.data_handle(), labels, nullptr, ws.data(), need));
}
}  // namespace detail

template <typename DataT, typename MathT, typename IndexT, typename Layout>
void fit(raft::resources const& handle, const kmeans_balanced_params& params,
         raft::device_matrix_view<const DataT, IndexT, Layout> X, raft::device_matrix_view<MathT, IndexT> centroids)
{
  static_assert(std::is_same<DataT, float>::value && std::is_same<MathT, float>::value,
                "raft_b200 kmeans_balanced: float data");
  detail::fit_impl(handle, params, X, centroids, nullptr);
}

template <typename DataT, typename MathT, typename IndexT, typename Layout, typename LabelsView>
void predict(raft::resources const& handle, const kmeans_balanced_params& params,
             raft::device_matrix_view<const DataT, IndexT, Layout> X, raft::device_matrix_view<const MathT, IndexT> centroids,
             LabelsView labels)
{
  static_assert(std::is_same<DataT, float>::value && std::is_same<MathT, float>::value,
                "raft_b200 kmeans_balanced: float data");
  detail::check_label_view<LabelsView>();
  detail::check_params(params);
  const int64_t m = X.extent(0), k = X.extent(1), nc = centroids.extent(0);
  RAFT_EXPECTS(centroids.extent(1) == k, "kmeans_balanced: centroids must have n_features columns");
  RAFT_EXPECTS(labels.extent(0) == m, "kmeans_balanced: labels must have n_samples entries");
  const int64_t ldx = detail::row_pitch(X);
  const size_t need = b2d_kmeans_workspace_bytes(m, k, nc);
  RAFT_EXPECTS(need != SIZE_MAX, "kmeans_balanced: invalid extents");
  raft::b200::scoped_workspace ws(handle, need + 256);   // (the first 256 bytes take the inertia)
  raft::distance::detail::b2d_check(b2d_kmeans_predict(
    raft::resource::get_cuda_stream(handle), X.data_handle(), ldx, nullptr, m, k, centroids.data_handle(),
    static_cast<int>(nc), reinterpret_cast<int32_t*>(labels.data_handle()), static_cast<double*>(ws.data()), 1,
    static_cast<char*>(ws.data()) + 256, need));
}

template <typename DataT, typename MathT, typename IndexT, typename Layout, typename LabelsView>
void fit_predict(raft::resources const& handle, const kmeans_balanced_params& params,
                 raft::device_matrix_view<const DataT, IndexT, Layout> X, raft::device_matrix_view<MathT, IndexT> centroids,
                 LabelsView labels)
{
  static_assert(std::is_same<DataT, float>::value && std::is_same<MathT, float>::value,
                "raft_b200 kmeans_balanced: float data");
  detail::check_label_view<LabelsView>();
  RAFT_EXPECTS(labels.extent(0) == X.extent(0), "kmeans_balanced: labels must have n_samples entries");
  detail::fit_impl(handle, params, X, centroids, reinterpret_cast<int32_t*>(labels.data_handle()));
}

}  // namespace kmeans_balanced
}  // namespace cluster
}  // namespace raft
