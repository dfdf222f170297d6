// raft::neighbors::kernel_density::score_samples -- shim over b2d_kde_score_samples (include/raft_b200.h).  A project API:
// RAFT has no kernel-density entry point, so no upstream signature is claimed.  out[i] (double) is the log density of
// row i of queries [m, d] under the kernel density estimate of dataset [n, d] with the given weights (std::nullopt: all
// 1), the answer of sklearn.neighbors.KernelDensity(kernel, bandwidth, atol = 0, rtol = 0).fit(dataset, sample_weight)
// .score_samples(queries) (with the exact normalisation of the cosine kernel).  The squared distance is exactly the one
// pairwise_distance(L2Expanded) returns, including its self-pair rule when queries and dataset are the same matrix.
// A negative, non-finite or all-zero weight makes every output NaN (checked on the device: no synchronisation).  Runs on
// the handle's stream with scratch from its workspace and never synchronises.  d <= 320.
#pragma once
#include <cstdint>
#include <optional>

#include "../distance/distance.cuh"

namespace raft {
namespace neighbors {
namespace kernel_density {

// B2D_KDE_* (sklearn's kernel names, in their order)
enum class KernelType { Gaussian = 0, Tophat = 1, Epanechnikov = 2, Exponential = 3, Linear = 4, Cosine = 5 };

struct KdeParams {
  KernelType kernel = KernelType::Gaussian;
  double bandwidth  = 1.0;
  int64_t batch_cols = 0;   // dataset columns per pass, rounded up to 256; 0: the partials at about 1 GiB
};

template <typename matrix_idx_t>
void score_samples(raft::resources const& handle,
                   raft::device_matrix_view<const float, matrix_idx_t, raft::row_major> dataset,
                   raft::device_matrix_view<const float, matrix_idx_t, raft::row_major> queries,
                   std::optional<raft::device_vector_view<const float, matrix_idx_t>> sample_weight,
                   raft::device_vector_view<double, matrix_idx_t> out, const KdeParams& params)
{
  const int64_t m = queries.extent(0), n = dataset.extent(0), d = queries.extent(1);
  RAFT_EXPECTS(dataset.extent(1) == queries.extent(1), "queries and dataset must have the same number of columns");
  RAFT_EXPECTS(static_cast<int64_t>(out.extent(0)) == m, "out must have one entry per query row");
  RAFT_EXPECTS(!sample_weight || static_cast<int64_t>(sample_weight->extent(0)) == n,
               "sample_weight must have one entry per dataset row");
  const size_t need = b2d_kde_workspace_bytes(m, n, d, params.batch_cols);
  RAFT_EXPECTS(need != SIZE_MAX, "negative extent or batch_cols");
  raft::b200::scoped_workspace ws(handle, need);
  raft::distance::detail::b2d_check(b2d_kde_score_samples(
      raft::resource::get_cuda_stream(handle), static_cast<int>(params.kernel), params.bandwidth, dataset.data_handle(), d,
      sample_weight ? sample_weight->data_handle() : nullptr, queries.data_handle(), d, m, n, d, params.batch_cols,
      out.data_handle(), ws.data(), need));
}

}  // namespace kernel_density
}  // namespace neighbors
}  // namespace raft
