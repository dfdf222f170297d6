// raft::distance::pairwise_distance -- header-only shim with the signatures of the removed
// raft/distance/distance.cuh, dispatching through the C ABI (include/raft_b200.h) into the sm_90a
// kernels.  Call shapes kept (verbatim from the surviving callers):
//   pairwise_distance(handle, x, y, dist, m, n, k, metric)             cpp/include/raft/stats/detail/silhouette_score.cuh:205-206
//   pairwise_distance(handle, x, y, dist, m, n, k, metric, isRowMajor, metric_arg)
//                                                                      cpp/include/raft/stats/detail/trustworthiness_score.cuh:152-153
//   pairwise_distance(handle, x_view, y_view, dist_view, metric, metric_arg)   (mdspan form, README.md:115-127 analogue)
// Semantics kept: asynchronous on raft::resource::get_cuda_stream(handle), never synchronises,
// temporaries from the handle's workspace, errors as raft::logic_error / raft::cuda_error.
#pragma once
#include <type_traits>

#include "../../raft_b200.h"
#include "../core/b200_workspace.hpp"
#include "distance_types.hpp"

namespace raft {
namespace distance {
namespace detail {
inline void b2d_check(int status)
{
  if (status == B2D_OK) return;
  std::string msg = b2d_last_error();
  if (status == B2D_ERR_CUDA) throw raft::cuda_error(msg);
  throw raft::logic_error(msg);
}
template <typename T>
constexpr int b2d_dtype()
{
  static_assert(std::is_same<T, float>::value || std::is_same<T, double>::value,
                "raft_b200: float or double (fp16 inputs through the C ABI)");
  return std::is_same<T, double>::value ? B2D_F64 : B2D_F32;
}
}  // namespace detail

template <typename DataT, typename IdxT = int>
void pairwise_distance(raft::resources const& handle, const DataT* x, const DataT* y, DataT* dist, IdxT m, IdxT n,
                       IdxT k, raft::distance::DistanceType metric, bool isRowMajor = true, DataT metric_arg = 2.0f)
{
  const int dt      = detail::b2d_dtype<DataT>();
  const size_t need = b2d_pairwise_workspace_bytes(static_cast<int>(metric), dt, m, n, k);
  RAFT_EXPECTS(need != static_cast<size_t>(-1), "pairwise_distance: metric not supported by raft_b200");
  raft::b200::scoped_workspace ws(handle, need);  // the handle's workspace resource (b200_workspace.hpp)
  const int64_t ldx = isRowMajor ? k : m, ldy = isRowMajor ? k : n, ldd = isRowMajor ? n : m;
  detail::b2d_check(b2d_pairwise_distance(raft::resource::get_cuda_stream(handle), static_cast<int>(metric), dt, x, ldx,
                                          y, ldy, dist, ldd, m, n, k, isRowMajor ? 1 : 0,
                                          static_cast<float>(metric_arg), need ? ws.data() : nullptr, need));
}

// overload with a caller-supplied workspace (the reference took an rmm::device_uvector<char>&;
// here: any device buffer of at least b2d_pairwise_workspace_bytes() bytes)
template <typename DataT, typename IdxT = int>
void pairwise_distance(raft::resources const& handle, const DataT* x, const DataT* y, DataT* dist, IdxT m, IdxT n,
                       IdxT k, void* workspace, size_t workspace_bytes, raft::distance::DistanceType metric,
                       bool isRowMajor = true, DataT metric_arg = 2.0f)
{
  const int64_t ldx = isRowMajor ? k : m, ldy = isRowMajor ? k : n, ldd = isRowMajor ? n : m;
  detail::b2d_check(b2d_pairwise_distance(raft::resource::get_cuda_stream(handle), static_cast<int>(metric),
                                          detail::b2d_dtype<DataT>(), x, ldx, y, ldy, dist, ldd, m, n, k,
                                          isRowMajor ? 1 : 0, static_cast<float>(metric_arg), workspace,
                                          workspace_bytes));
}

namespace detail {
// (row_major?, leading dimension) of a 2-d view: layout_right / layout_left are dense; a layout_stride view must
// have unit stride along one dimension (what make_device_strided_matrix_view builds, device_mdspan.hpp:178-199)
template <typename View>
inline void view_layout(const View& v, bool& row_major, int64_t& ld)
{
  const int64_t s0 = static_cast<int64_t>(v.stride(0)), s1 = static_cast<int64_t>(v.stride(1));
  if (s1 == 1 || v.extent(1) <= 1) { row_major = true; ld = s0 > 0 ? s0 : v.extent(1); }
  else {
    RAFT_EXPECTS(s0 == 1 || v.extent(0) <= 1, "pairwise_distance: views need unit stride along one dimension");
    row_major = false;
    ld        = s1;
  }
  if (row_major && ld < static_cast<int64_t>(v.extent(1))) ld = v.extent(1);
  if (!row_major && ld < static_cast<int64_t>(v.extent(0))) ld = v.extent(0);
}
}  // namespace detail

// mdspan form: x [m,k], y [n,k], dist [m,n]; row_major / col_major / strided views (leading dimensions honoured)
template <typename DataT, typename IdxT, typename LayoutX, typename LayoutY, typename LayoutD>
void pairwise_distance(raft::resources const& handle, raft::device_matrix_view<const DataT, IdxT, LayoutX> x,
                       raft::device_matrix_view<const DataT, IdxT, LayoutY> y,
                       raft::device_matrix_view<DataT, IdxT, LayoutD> dist, raft::distance::DistanceType metric,
                       DataT metric_arg = 2.0f)
{
  RAFT_EXPECTS(x.extent(1) == y.extent(1), "Number of columns must be equal.");
  RAFT_EXPECTS(dist.extent(0) == x.extent(0), "Number of rows in output must be equal to number of rows in X");
  RAFT_EXPECTS(dist.extent(1) == y.extent(0), "Number of columns in output must be equal to number of rows in Y");
  bool rx, ry, rd;
  int64_t ldx, ldy, ldd;
  detail::view_layout(x, rx, ldx);
  detail::view_layout(y, ry, ldy);
  detail::view_layout(dist, rd, ldd);
  RAFT_EXPECTS(rx == ry && rx == rd, "pairwise_distance: x, y and dist must share one layout (all row- or all column-major)");
  const int64_t m = x.extent(0), n = y.extent(0), k = x.extent(1);
  const int dt      = detail::b2d_dtype<DataT>();
  const size_t need = b2d_pairwise_workspace_bytes(static_cast<int>(metric), dt, m, n, k);
  RAFT_EXPECTS(need != static_cast<size_t>(-1), "pairwise_distance: metric not supported by raft_b200");
  raft::b200::scoped_workspace ws(handle, need);
  detail::b2d_check(b2d_pairwise_distance(raft::resource::get_cuda_stream(handle), static_cast<int>(metric), dt,
                                          x.data_handle(), ldx, y.data_handle(), ldy, dist.data_handle(), ldd, m, n, k,
                                          rx ? 1 : 0, static_cast<float>(metric_arg), need ? ws.data() : nullptr, need));
}

}  // namespace distance
}  // namespace raft
