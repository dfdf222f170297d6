// raft::cluster::kmeans -- header-only shim of the removed raft/cluster/kmeans.cuh ([RECALLED], <= 25.12): Lloyd's
// k-means under L2Expanded, dispatching through b2d_kmeans_* (include/raft_b200.h).  float data only.
//   fit            centroids [n_clusters, k] in/out (read for InitMethod::Array), inertia and n_iter to the host
//   predict        labels [m] on the device, inertia to the host
//   cluster_cost   sum_i min_j ||x_i - c_j||^2 to the host
// InitMethod::KMeansPlusPlus with oversampling_factor > 0 seeds with k-means|| (b2d_kmeans_fit_scalable).  Departure:
// the reference's default oversampling_factor is 2.0, which selects k-means||; here the default is 0.0 (greedy
// k-means++), so k-means|| must be asked for explicitly.
// Temporaries come from the handle's workspace (raft/core/b200_workspace.hpp).  The host outputs are read after a sync of
// the handle's stream, as the reference's host_scalar_view outputs were.  Departures from the recalled signatures: the
// optional sample weights are a nullable device pointer and the host scalars are plain pointers (the 1-d and scalar
// views are not part of the mdspan subset this shim depends on).
#pragma once
#include <cstdint>
#include <type_traits>

#include "../../raft_b200.h"
#include "../core/b200_workspace.hpp"
#include "../distance/distance.cuh"

namespace raft {
namespace cluster {
namespace kmeans {

enum class InitMethod { KMeansPlusPlus = 0, Random = 1, Array = 2 };

struct KMeansParams {
  int n_clusters = 8;
  InitMethod init = InitMethod::KMeansPlusPlus;
  int max_iter = 300;
  double tol = 1e-4;
  int verbosity = 0;                                   // accepted, no effect
  struct { uint64_t seed = 0; } rng_state;
  raft::distance::DistanceType metric = raft::distance::DistanceType::L2Expanded;
  int n_init = 1;
  double oversampling_factor = 0.0;                    // > 0 with KMeansPlusPlus: k-means|| seeding (reference: 2.0)
  int batch_samples = 1 << 15;                         // accepted, no effect (the assignment is never batched)
  int batch_centroids = 0;                             // accepted, no effect
  bool inertia_check = false;
};

namespace detail {
// device scratch of one call: the C-ABI workspace plus a double and an int for the device-side results
struct km_scratch {
  raft::b200::scoped_workspace ws;
  size_t bytes;
  km_scratch(raft::resources const& handle, size_t need) : ws(handle, need + 256), bytes(need) {}
  void* base() { return static_cast<char*>(ws.data()) + 256; }
  double* d() { return static_cast<double*>(ws.data()); }
  int32_t* i() { return reinterpret_cast<int32_t*>(static_cast<char*>(ws.data()) + 8); }
};
template <typename IndexT, typename Layout>
int64_t row_pitch(raft::device_matrix_view<const float, IndexT, Layout> v)
{
  bool row_major;
  int64_t ld;
  raft::distance::detail::view_layout(v, row_major, ld);
  RAFT_EXPECTS(row_major, "kmeans: X must be row-major");
  return ld;
}
inline void cuda_check(cudaError_t e)
{
  if (e != cudaSuccess) throw raft::cuda_error(std::string("raft_b200 kmeans: ") + cudaGetErrorString(e));
}
inline void check_metric(const KMeansParams& p)
{
  RAFT_EXPECTS(p.metric == raft::distance::DistanceType::L2Expanded, "kmeans: only the L2Expanded metric is supported");
}
}  // namespace detail

template <typename DataT, typename IndexT, typename Layout>
void fit(raft::resources const& handle, const KMeansParams& params, raft::device_matrix_view<const DataT, IndexT, Layout> X,
         const DataT* sample_weight, raft::device_matrix_view<DataT, IndexT> centroids, DataT* inertia, IndexT* n_iter)
{
  static_assert(std::is_same<DataT, float>::value, "raft_b200 kmeans: float data");
  detail::check_metric(params);
  const int64_t m = X.extent(0), k = X.extent(1);
  RAFT_EXPECTS(centroids.extent(0) == params.n_clusters && centroids.extent(1) == k,
               "kmeans: centroids must be [n_clusters, n_features]");
  const int64_t ldx = detail::row_pitch(X);
  const bool scalable = params.init == InitMethod::KMeansPlusPlus && params.oversampling_factor > 0;
  const size_t need = scalable ? b2d_kmeans_scalable_workspace_bytes(m, k, params.n_clusters, params.oversampling_factor)
                               : b2d_kmeans_workspace_bytes(m, k, params.n_clusters);
  RAFT_EXPECTS(need != SIZE_MAX, "kmeans: invalid extents or oversampling_factor");
  detail::km_scratch s(handle, need);
  cudaStream_t st = raft::resource::get_cuda_stream(handle);
  if (scalable)
    raft::distance::detail::b2d_check(b2d_kmeans_fit_scalable(
      st, params.n_clusters, params.max_iter, params.tol, params.oversampling_factor, params.n_init, params.rng_state.seed,
      params.inertia_check ? 1 : 0, X.data_handle(), ldx, sample_weight, m, k, centroids.data_handle(), s.d(), s.i(),
      s.base(), need));
  else
    raft::distance::detail::b2d_check(b2d_kmeans_fit(
      st, params.n_clusters, params.max_iter, params.tol, static_cast<int>(params.init), params.n_init, params.rng_state.seed,
      params.inertia_check ? 1 : 0, X.data_handle(), ldx, sample_weight, m, k, centroids.data_handle(), s.d(), s.i(),
      s.base(), need));
  double hi = 0.0;
  int32_t hn = 0;
  if (m > 0) {
    detail::cuda_check(cudaMemcpyAsync(&hi, s.d(), sizeof hi, cudaMemcpyDeviceToHost, st));
    detail::cuda_check(cudaMemcpyAsync(&hn, s.i(), sizeof hn, cudaMemcpyDeviceToHost, st));
  }
  raft::resource::sync_stream(handle);
  if (inertia) *inertia = static_cast<DataT>(hi);
  if (n_iter) *n_iter = static_cast<IndexT>(hn);
}

template <typename DataT, typename IndexT, typename Layout>
void predict(raft::resources const& handle, const KMeansParams& params, raft::device_matrix_view<const DataT, IndexT, Layout> X,
             const DataT* sample_weight, raft::device_matrix_view<const DataT, IndexT> centroids, int32_t* labels,
             bool normalize_weight, DataT* inertia)
{
  static_assert(std::is_same<DataT, float>::value, "raft_b200 kmeans: float data");
  detail::check_metric(params);
  const int64_t m = X.extent(0), k = X.extent(1), nc = centroids.extent(0);
  RAFT_EXPECTS(centroids.extent(1) == k, "kmeans: centroids must have n_features columns");
  const int64_t ldx = detail::row_pitch(X);
  const size_t need = b2d_kmeans_workspace_bytes(m, k, nc);
  RAFT_EXPECTS(need != SIZE_MAX, "kmeans: invalid extents");
  detail::km_scratch s(handle, need);
  cudaStream_t st = raft::resource::get_cuda_stream(handle);
  raft::distance::detail::b2d_check(b2d_kmeans_predict(st, X.data_handle(), ldx, sample_weight, m, k,
                                                       centroids.data_handle(), static_cast<int>(nc), labels, s.d(),
                                                       normalize_weight ? 1 : 0, s.base(), need));
  if (inertia) {
    double hi = 0.0;
    if (m > 0) detail::cuda_check(cudaMemcpyAsync(&hi, s.d(), sizeof hi, cudaMemcpyDeviceToHost, st));
    raft::resource::sync_stream(handle);
    *inertia = static_cast<DataT>(hi);
  }
}

template <typename DataT, typename IndexT, typename Layout>
void cluster_cost(raft::resources const& handle, raft::device_matrix_view<const DataT, IndexT, Layout> X,
                  raft::device_matrix_view<const DataT, IndexT> centroids, DataT* cost)
{
  KMeansParams p;
  p.n_clusters = static_cast<int>(centroids.extent(0));
  predict(handle, p, X, static_cast<const DataT*>(nullptr), centroids, nullptr, true, cost);
}

}  // namespace kmeans
}  // namespace cluster
}  // namespace raft
