// raft::matrix::select_k -- shim over b2d_select_k (include/raft_b200.h); signature of
// cpp/include/raft/matrix/select_k.cuh:72-106.
#pragma once
#include <optional>

#include "../distance/distance.cuh"
#include "select_k_types.hpp"

namespace raft {
namespace matrix {

/**
 * Select the k smallest (select_min) or largest values of every row of in_val, with their payloads.
 *
 * @param[in] handle    its stream receives the work; scratch comes from raft::b200::scoped_workspace
 * @param[in] in_val    [batch_size, len] row-major values
 * @param[in] in_idx    optional [batch_size, len] payloads; without it the payload is the column
 * @param[out] out_val  [batch_size, k] selected values, the input bits unchanged
 * @param[out] out_idx  [batch_size, k] their payloads
 * @param[in] select_min  smallest (true) or largest (false) values
 * @param[in] sorted    accepted for compatibility: every row is always written sorted, best first, equal values in
 *                      ascending column order (-0.0 == +0.0, every NaN above +inf)
 * @param[in] algo      accepted for compatibility and ignored: there is one selection path
 */
template <typename T, typename IdxT>
void select_k(raft::resources const& handle, raft::device_matrix_view<const T, int64_t, raft::row_major> in_val,
              std::optional<raft::device_matrix_view<const IdxT, int64_t, raft::row_major>> in_idx,
              raft::device_matrix_view<T, int64_t, raft::row_major> out_val,
              raft::device_matrix_view<IdxT, int64_t, raft::row_major> out_idx, bool select_min, bool sorted = false,
              SelectAlgo algo = SelectAlgo::kAuto)
{
  static_assert(std::is_same<T, float>::value && std::is_same<IdxT, int64_t>::value,
                "raft_b200: select_k is provided for <float, int64_t>");
  (void)sorted;
  (void)algo;
  const int64_t rows = in_val.extent(0), len = in_val.extent(1), k = out_val.extent(1);
  RAFT_EXPECTS(rows == out_val.extent(0) && rows == out_idx.extent(0), "batch sizes must be equal");
  RAFT_EXPECTS(k == out_idx.extent(1), "value and index output lengths must be equal");
  if (in_idx.has_value())
    RAFT_EXPECTS(in_idx->extent(0) == rows && in_idx->extent(1) == len, "in_idx must have the shape of in_val");
  const size_t need = b2d_select_k_workspace_bytes(rows, len, k);
  RAFT_EXPECTS(need != SIZE_MAX, "k must be in [1, len] and len below 2^31");
  raft::b200::scoped_workspace ws(handle, need);
  raft::distance::detail::b2d_check(b2d_select_k(raft::resource::get_cuda_stream(handle), in_val.data_handle(), len,
                                                 in_idx.has_value() ? in_idx->data_handle() : nullptr, rows, len, k,
                                                 select_min ? 1 : 0, out_val.data_handle(), out_idx.data_handle(),
                                                 need ? ws.data() : nullptr, need));
}

}  // namespace matrix
}  // namespace raft
