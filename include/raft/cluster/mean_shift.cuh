// raft::cluster::mean_shift::fit -- shim over b2d_mean_shift_fit (include/raft_b200.h).  A project API: RAFT has no
// mean-shift entry point, so no upstream signature is claimed.  The fit of sklearn.cluster.MeanShift(bandwidth, seeds,
// bin_seeding, min_bin_freq, cluster_all, max_iter).fit(X) with the neighbourhood test decided by the engine's squared
// distance against fp32(bandwidth^2), as dbscan decides it.  centers [s or m, d] receives the kept centres first;
// n_centers and n_iter are written on the host (the call synchronises the handle's stream, see raft_b200.h).  Scratch
// comes from the handle's workspace.  d <= 320.
#pragma once
#include <cstdint>
#include <optional>

#include "../../raft_b200.h"
#include "../core/b200_workspace.hpp"
#include "../distance/distance.cuh"

namespace raft {
namespace cluster {
namespace mean_shift {

struct MeanShiftParams {
  double bandwidth        = 1.0;
  bool bin_seeding        = false;
  int64_t min_bin_freq    = 1;
  bool cluster_all        = true;
  int max_iter            = 300;
  int64_t max_bytes_per_batch = 0;   // adjacency bytes formed at once; 0: 2^30.  The result does not depend on it.
};

/** Mean shift of the rows of X [m, d] (row-major, any row pitch).  seeds [s, d] (std::nullopt: bin seeding or the rows
 * of X); centers must hold s (or m) rows, labels m entries. */
template <typename LabelsView>
void fit(raft::resources const& handle, const MeanShiftParams& params,
         raft::device_matrix_view<const float, int64_t, raft::row_major> X,
         std::optional<raft::device_matrix_view<const float, int64_t, raft::row_major>> seeds,
         raft::device_matrix_view<float, int64_t, raft::row_major> centers, LabelsView labels, int& n_centers, int& n_iter)
{
  const int64_t m = X.extent(0), d = X.extent(1), s = seeds ? seeds->extent(0) : 0;
  RAFT_EXPECTS(!seeds || seeds->extent(1) == d, "mean_shift: seeds must have d columns");
  RAFT_EXPECTS(static_cast<int64_t>(centers.extent(0)) >= (seeds ? s : m) && centers.extent(1) == d,
               "mean_shift: centers must hold one row per seed (or per row of X) of d columns");
  RAFT_EXPECTS(static_cast<int64_t>(labels.extent(0)) == m, "mean_shift: labels must have m entries");
  const int64_t ldx = m > 1 ? static_cast<int64_t>(X.stride(0)) : d;
  const int64_t lds = seeds && s > 1 ? static_cast<int64_t>(seeds->stride(0)) : d;
  const size_t need = b2d_mean_shift_fit_workspace_bytes(m, d, s, params.max_bytes_per_batch);
  RAFT_EXPECTS(need != SIZE_MAX, "mean_shift: negative extents or max_bytes_per_batch");
  raft::b200::scoped_workspace ws(handle, need + 8);
  int32_t* out = reinterpret_cast<int32_t*>(static_cast<char*>(ws.data()) + need);   // n_centers, n_iter
  raft::distance::detail::b2d_check(b2d_mean_shift_fit(
      raft::resource::get_cuda_stream(handle), X.data_handle(), ldx, m, d, params.bandwidth,
      seeds ? seeds->data_handle() : nullptr, lds, s, params.bin_seeding ? 1 : 0, params.min_bin_freq,
      params.cluster_all ? 1 : 0, params.max_iter, params.max_bytes_per_batch, centers.data_handle(), out,
      labels.data_handle(), out + 1, ws.data(), need));
  int32_t host[2];
  if (cudaMemcpyAsync(host, out, sizeof(host), cudaMemcpyDeviceToHost, raft::resource::get_cuda_stream(handle)) != cudaSuccess)
    throw raft::cuda_error("mean_shift: reading n_centers / n_iter failed");
  raft::resource::sync_stream(handle);
  n_centers = host[0];
  n_iter    = host[1];
}

}  // namespace mean_shift
}  // namespace cluster
}  // namespace raft
