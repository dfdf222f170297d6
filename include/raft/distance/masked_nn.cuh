// raft::distance::masked_l2_nn -- shim over b2d_masked_l2_nn (include/raft_b200.h): fusedL2NN restricted by a row x
// group adjacency mask (the nearest-neighbour step of connect_components).  Signature of the removed
// raft/distance/masked_nn.cuh ([RECALLED], <= 25.12): group_idxs holds the END of every group of rows of y (the inclusive
// scan of the group sizes); adj[i, g] admits the rows of group g as candidates for row i of x.  x_norm / y_norm are the
// SQUARED row norms.  As in the generic fusedL2NN, the engine finds the per-row {arg-min, min} (ties -> smaller index)
// and params.redOp is applied once per row to that winner; rows without any adjacent candidate are left to redOp.init
// (initOutBuffer) or keep the caller's value.  group_idxs must be non-decreasing and inside [0, n]: the engine checks
// it on the device (this call never synchronises) and, when it fails, reports every row as without a candidate.
#pragma once
#include "fused_l2_nn.cuh"

namespace raft {
namespace distance {

template <typename ReduceOpT, typename KVPReduceOpT>
struct masked_l2_nn_params {
  ReduceOpT redOp;
  KVPReduceOpT pairRedOp;   // (accepted for compatibility; must be a minimum, as in fusedL2NN)
  bool sqrt;
  bool initOutBuffer;
};

#ifdef __CUDACC__
template <typename DataT, typename OutT, typename IdxT, typename ReduceOpT, typename KVPReduceOpT>
void masked_l2_nn(raft::resources const& handle, raft::distance::masked_l2_nn_params<ReduceOpT, KVPReduceOpT> params,
                  raft::device_matrix_view<const DataT, IdxT, raft::layout_c_contiguous> x,
                  raft::device_matrix_view<const DataT, IdxT, raft::layout_c_contiguous> y,
                  raft::device_vector_view<const DataT, IdxT, raft::layout_c_contiguous> x_norm,
                  raft::device_vector_view<const DataT, IdxT, raft::layout_c_contiguous> y_norm,
                  raft::device_matrix_view<const bool, IdxT, raft::layout_c_contiguous> adj,
                  raft::device_vector_view<const IdxT, IdxT, raft::layout_c_contiguous> group_idxs,
                  raft::device_vector_view<OutT, IdxT, raft::layout_c_contiguous> out)
{
  static_assert(std::is_same<DataT, float>::value && sizeof(IdxT) == 4,
                "raft_b200: masked_l2_nn is provided for DataT = float, 32-bit IdxT");
  const IdxT m = x.extent(0), n = y.extent(0), k = x.extent(1), G = group_idxs.extent(0);
  RAFT_EXPECTS(y.extent(1) == k, "x and y must have the same number of columns");
  RAFT_EXPECTS(x_norm.extent(0) == m && y_norm.extent(0) == n, "x_norm / y_norm must have one entry per row");
  RAFT_EXPECTS(adj.extent(0) == m && adj.extent(1) == G, "adj must be [rows of x, number of groups]");
  RAFT_EXPECTS(out.extent(0) == m, "out must have one entry per row of x");
  if (m == 0) return;
  const size_t need = b2d_masked_l2_nn_workspace_bytes(m, n, k, G);
  const size_t kvpb = (static_cast<size_t>(m) * sizeof(b2d_kvp_if) + 255) / 256 * 256;
  raft::b200::scoped_workspace ws(handle, kvpb + need);
  char* base           = static_cast<char*>(ws.data());
  b2d_kvp_if* nn       = reinterpret_cast<b2d_kvp_if*>(base);
  cudaStream_t stream  = raft::resource::get_cuda_stream(handle);
  detail::b2d_check(b2d_masked_l2_nn(stream, nn, x.data_handle(), k, y.data_handle(), k, x_norm.data_handle(),
                                     y_norm.data_handle(), reinterpret_cast<const uint8_t*>(adj.data_handle()), G,
                                     reinterpret_cast<const int32_t*>(group_idxs.data_handle()), G, m, n, k,
                                     params.sqrt ? 1 : 0, 1, base + kvpb, need));
  detail::b2d_apply_reduce_kernel<OutT, IdxT, DataT, ReduceOpT><<<static_cast<unsigned>((m + 255) / 256), 256, 0, stream>>>(
    out.data_handle(), nn, m, params.redOp, params.initOutBuffer, 3.402823466e+38f);
  if (cudaGetLastError() != cudaSuccess) throw raft::cuda_error("masked_l2_nn: reduction launch failed");
}
#endif  // __CUDACC__

}  // namespace distance
}  // namespace raft
