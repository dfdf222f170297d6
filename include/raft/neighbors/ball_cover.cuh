// raft::neighbors::ball_cover -- shim over b2d_ball_cover_* (include/raft_b200.h), shaped after RAFT's random ball cover
// from before the move to cuVS: BallCoverIndex, build_index, knn_query, all_knn_query and eps_nn in its CSR form.
// Exact only: there is no weight < 1 and no switch that turns the post-filtering off.  2-D and 3-D float points under
// L2Unexpanded or L2SqrtUnexpanded; the distance of a pair is fixed bit for bit (see raft_b200.h), and neighbours come in
// ascending (distance, index) order.  Every call runs on the handle's stream and none synchronises; the index buffer and
// the scratch come from the handle's workspace (b200_workspace.hpp).
#pragma once
#include <memory>

#include "../distance/distance.cuh"

namespace raft {
namespace neighbors {
namespace ball_cover {

template <typename idx_t, typename value_t, typename int_t = std::uint32_t, typename matrix_idx_t = std::int64_t>
class BallCoverIndex {
  static_assert(std::is_same<idx_t, std::int64_t>::value && std::is_same<value_t, float>::value,
                "raft_b200: ball_cover takes float points and int64 neighbour indices");

 public:
  // n_landmarks = 0: ceil(sqrt(n)).  X must stay valid for all_knn_query (the queries are its rows); the index itself
  // holds its own copy of the points once built.
  BallCoverIndex(raft::resources const& handle, raft::device_matrix_view<const value_t, matrix_idx_t, raft::row_major> X,
                 raft::distance::DistanceType metric, std::int64_t n_landmarks = 0, std::uint64_t seed = 0)
    : X_(X), metric_(metric), n_landmarks_(n_landmarks), seed_(seed)
  {
    const size_t need = b2d_ball_cover_index_bytes(X.extent(0), X.extent(1), n_landmarks);
    RAFT_EXPECTS(need != SIZE_MAX, "ball_cover: n >= 1, d in {2, 3} and n_landmarks in [0, n]");
    buf_ = std::make_unique<raft::b200::scoped_workspace>(handle, need);
  }
  raft::device_matrix_view<const value_t, matrix_idx_t, raft::row_major> get_X() const { return X_; }
  raft::distance::DistanceType get_metric() const { return metric_; }
  std::int64_t get_n_landmarks() const { return n_landmarks_; }
  bool is_index_trained() const { return trained_; }

  void* data() const { return buf_->data(); }
  std::uint64_t seed() const { return seed_; }
  void set_index_trained() { trained_ = true; }

 private:
  raft::device_matrix_view<const value_t, matrix_idx_t, raft::row_major> X_;
  raft::distance::DistanceType metric_;
  std::int64_t n_landmarks_;
  std::uint64_t seed_;
  bool trained_ = false;
  std::unique_ptr<raft::b200::scoped_workspace> buf_;
};

template <typename idx_t, typename value_t, typename int_t, typename matrix_idx_t>
void build_index(raft::resources const& handle, BallCoverIndex<idx_t, value_t, int_t, matrix_idx_t>& index)
{
  const auto X      = index.get_X();
  const int64_t n   = X.extent(0), d = X.extent(1);
  const size_t need = b2d_ball_cover_build_workspace_bytes(n, d, index.get_n_landmarks());
  raft::b200::scoped_workspace ws(handle, need);
  raft::distance::detail::b2d_check(b2d_ball_cover_build(raft::resource::get_cuda_stream(handle), index.data(),
                                                         X.data_handle(), d, n, d, static_cast<int>(index.get_metric()),
                                                         index.get_n_landmarks(), index.seed(), ws.data(), need));
  index.set_index_trained();
}

// inds / dists [m, k]: the k nearest rows of X for every row of query [m, d]
template <typename idx_t, typename value_t, typename int_t, typename matrix_idx_t>
void knn_query(raft::resources const& handle, const BallCoverIndex<idx_t, value_t, int_t, matrix_idx_t>& index,
               raft::device_matrix_view<const value_t, matrix_idx_t, raft::row_major> query,
               raft::device_matrix_view<idx_t, matrix_idx_t, raft::row_major> inds,
               raft::device_matrix_view<value_t, matrix_idx_t, raft::row_major> dists)
{
  RAFT_EXPECTS(index.is_index_trained(), "ball_cover: build_index first");
  const auto X    = index.get_X();
  const int64_t m = query.extent(0), k = inds.extent(1);
  RAFT_EXPECTS(query.extent(1) == X.extent(1), "query and index must have the same number of columns");
  RAFT_EXPECTS(inds.extent(0) == m && dists.extent(0) == m && dists.extent(1) == k, "inds and dists must be [m, k]");
  raft::distance::detail::b2d_check(b2d_ball_cover_knn(raft::resource::get_cuda_stream(handle), inds.data_handle(),
                                                       dists.data_handle(), index.data(), X.extent(0), X.extent(1),
                                                       static_cast<int>(index.get_metric()), index.get_n_landmarks(),
                                                       query.data_handle(), query.extent(1), m, k));
}

// knn_query of the index's own points: every row finds itself at distance 0 (ties by index)
template <typename idx_t, typename value_t, typename int_t, typename matrix_idx_t>
void all_knn_query(raft::resources const& handle, const BallCoverIndex<idx_t, value_t, int_t, matrix_idx_t>& index,
                   raft::device_matrix_view<idx_t, matrix_idx_t, raft::row_major> inds,
                   raft::device_matrix_view<value_t, matrix_idx_t, raft::row_major> dists)
{
  knn_query(handle, index, index.get_X(), inds, dists);
}

// The epsilon neighbourhood in CSR form, in two calls: eps_nn_count writes adj_ia [m + 1]; the caller reads
// nnz = adj_ia[m], sizes adj_ja / dists to nnz and calls eps_nn with the same query and eps.  Under L2Unexpanded eps is a
// squared distance.
template <typename idx_t, typename value_t, typename int_t, typename matrix_idx_t>
void eps_nn_count(raft::resources const& handle, const BallCoverIndex<idx_t, value_t, int_t, matrix_idx_t>& index,
                  raft::device_matrix_view<const value_t, matrix_idx_t, raft::row_major> query,
                  raft::device_vector_view<idx_t, matrix_idx_t> adj_ia, value_t eps)
{
  RAFT_EXPECTS(index.is_index_trained(), "ball_cover: build_index first");
  const auto X    = index.get_X();
  const int64_t m = query.extent(0);
  RAFT_EXPECTS(query.extent(1) == X.extent(1), "query and index must have the same number of columns");
  RAFT_EXPECTS(static_cast<int64_t>(adj_ia.extent(0)) == m + 1, "adj_ia must have m + 1 entries");
  const size_t need = b2d_ball_cover_eps_workspace_bytes(m, 0);
  raft::b200::scoped_workspace ws(handle, need);
  raft::distance::detail::b2d_check(b2d_ball_cover_eps_count(raft::resource::get_cuda_stream(handle), adj_ia.data_handle(),
                                                             index.data(), X.extent(0), X.extent(1),
                                                             static_cast<int>(index.get_metric()), index.get_n_landmarks(),
                                                             query.data_handle(), query.extent(1), m, eps, ws.data(),
                                                             need));
}

template <typename idx_t, typename value_t, typename int_t, typename matrix_idx_t>
void eps_nn(raft::resources const& handle, const BallCoverIndex<idx_t, value_t, int_t, matrix_idx_t>& index,
            raft::device_matrix_view<const value_t, matrix_idx_t, raft::row_major> query,
            raft::device_vector_view<const idx_t, matrix_idx_t> adj_ia, raft::device_vector_view<idx_t, matrix_idx_t> adj_ja,
            raft::device_vector_view<value_t, matrix_idx_t> dists, value_t eps)
{
  RAFT_EXPECTS(index.is_index_trained(), "ball_cover: build_index first");
  const auto X      = index.get_X();
  const int64_t m   = query.extent(0);
  const int64_t nnz = adj_ja.extent(0);
  RAFT_EXPECTS(query.extent(1) == X.extent(1), "query and index must have the same number of columns");
  RAFT_EXPECTS(static_cast<int64_t>(adj_ia.extent(0)) == m + 1, "adj_ia must have m + 1 entries");
  RAFT_EXPECTS(static_cast<int64_t>(dists.extent(0)) == nnz, "adj_ja and dists must have nnz entries");
  const size_t need = b2d_ball_cover_eps_workspace_bytes(m, nnz);
  RAFT_EXPECTS(need != SIZE_MAX, "negative extent");
  raft::b200::scoped_workspace ws(handle, need);
  raft::distance::detail::b2d_check(b2d_ball_cover_eps_fill(raft::resource::get_cuda_stream(handle), adj_ia.data_handle(),
                                                            nnz, adj_ja.data_handle(), dists.data_handle(), index.data(),
                                                            X.extent(0), X.extent(1), static_cast<int>(index.get_metric()),
                                                            index.get_n_landmarks(), query.data_handle(), query.extent(1),
                                                            m, eps, ws.data(), need));
}

}  // namespace ball_cover
}  // namespace neighbors
}  // namespace raft
