// raft::neighbors::epsilon_neighborhood -- shim over b2d_eps_neighbors_l2sq (include/raft_b200.h).  Signatures of the
// removed raft/neighbors/epsilon_neighborhood.cuh ([RECALLED], <= 25.12).  eps is the SQUARED radius; adj[i, j] = d(i, j)
// <= eps with d exactly pairwise_distance's L2Expanded value; vd[j] += the number of rows of x adjacent to row j of y and
// vd[n] += the total: PER-COLUMN degrees, length n + 1 (the reference's doc comment said m + 1; its kernel summed per
// column).  Both forms add to vd without clearing it, like the reference: zero it first.  When y is x or a window of its
// rows (same memory, same pitch), a row's pair with itself is adjacent for every eps >= 0.  k <= 320 (else
// raft::logic_error).
#pragma once
#include "../distance/distance.cuh"

namespace raft {
namespace neighbors {
namespace epsilon_neighborhood {

namespace detail {
template <typename idx_t>
void eps_l2sq(cudaStream_t stream, bool* adj, idx_t* vd, const float* x, const float* y, int64_t m, int64_t n, int64_t k,
              float eps, void* ws, size_t ws_bytes)
{
  static_assert(std::is_same<idx_t, int>::value || std::is_same<idx_t, int64_t>::value,
                "raft_b200: the vertex degrees are int or int64_t");
  raft::distance::detail::b2d_check(b2d_eps_neighbors_l2sq(stream, reinterpret_cast<uint8_t*>(adj), n, vd,
                                                           sizeof(idx_t) == 8 ? 1 : 0, 0, x, k, y, k, m, n, k, eps, ws,
                                                           ws_bytes));
}
}  // namespace detail

/**
 * Pointer form: adj [m, n] row-major and vd [n + 1] (added to) for x [m, k] and y [n, k], row-major.  It takes no handle,
 * so its scratch is allocated stream-ordered on `stream` (raft::b200::scoped_workspace).
 */
template <typename value_t, typename idx_t>
void epsUnexpL2SqNeighborhood(bool* adj, idx_t* vd, const value_t* x, const value_t* y, idx_t m, idx_t n, idx_t k,
                              value_t eps, cudaStream_t stream)
{
  static_assert(std::is_same<value_t, float>::value, "raft_b200: the epsilon neighbourhood is provided for float");
  const size_t need = b2d_eps_neighbors_l2sq_workspace_bytes(m, n, k);
  RAFT_EXPECTS(need != SIZE_MAX, "negative extent");
  raft::b200::scoped_workspace ws(stream, need);
  detail::eps_l2sq<idx_t>(stream, adj, vd, x, y, m, n, k, eps, ws.data(), need);
}

/**
 * mdspan form: x [m, k], y [n, k], adj [m, n], vd [n + 1] (added to), on the handle's stream with its workspace.
 */
template <typename value_t, typename idx_t, typename matrix_idx_t>
void eps_neighbors_l2sq(raft::resources const& handle,
                        raft::device_matrix_view<const value_t, matrix_idx_t, raft::row_major> x,
                        raft::device_matrix_view<const value_t, matrix_idx_t, raft::row_major> y,
                        raft::device_matrix_view<bool, matrix_idx_t, raft::row_major> adj,
                        raft::device_vector_view<idx_t, matrix_idx_t> vd, value_t eps)
{
  static_assert(std::is_same<value_t, float>::value, "raft_b200: the epsilon neighbourhood is provided for float");
  const int64_t m = x.extent(0), n = y.extent(0), k = x.extent(1);
  RAFT_EXPECTS(y.extent(1) == x.extent(1), "x and y must have the same number of columns");
  RAFT_EXPECTS(adj.extent(0) == x.extent(0) && adj.extent(1) == y.extent(0), "adj must be [rows of x, rows of y]");
  RAFT_EXPECTS(static_cast<int64_t>(vd.extent(0)) == n + 1, "vd must have n + 1 entries");
  const size_t need = b2d_eps_neighbors_l2sq_workspace_bytes(m, n, k);
  raft::b200::scoped_workspace ws(handle, need);
  detail::eps_l2sq<idx_t>(raft::resource::get_cuda_stream(handle), adj.data_handle(), vd.data_handle(), x.data_handle(),
                          y.data_handle(), m, n, k, eps, ws.data(), need);
}

}  // namespace epsilon_neighborhood
}  // namespace neighbors
}  // namespace raft
