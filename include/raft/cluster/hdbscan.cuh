// raft::cluster::hdbscan -- header-only HDBSCAN of 2-D and 3-D points on the random ball cover, in the shape of cuML's
// ML::HDBSCAN::fit, dispatching through b2d_hdbscan_rbc_fit (include/raft_b200.h).  float data, int labels.
//   X [m, 2] or [m, 3] row-major (any row pitch), labels [m] and probabilities [m] (any 1-d views with data_handle() /
//   extent(0)); metric L2SqrtUnexpanded (the default) or L2Unexpanded, L2SqrtExpanded and L2Expanded taken as those.
// Labels are numbered 0, 1, ... in order of each cluster's smallest row, -1 is noise.  The result is
// sklearn.cluster.HDBSCAN's on the ball cover's pair distances with the mutual-reachability tree merged in the order
// (weight, min row, max row); it does not depend on n_landmarks (0: ceil(sqrt(m))) or seed.  Temporaries come from the
// handle's workspace (raft/core/b200_workspace.hpp); the call synchronises the handle's stream.
// With a prediction_model, fit also keeps the fitted model, and approximate_predict places new points in it
// (b2d_hdbscan_rbc_approximate_predict states the contract: an exact mutual-reachability neighbour over every fitted row).
#pragma once
#include <cstddef>
#include <cstdint>
#include <memory>

#include "../../raft_b200.h"
#include "../core/b200_workspace.hpp"
#include "../distance/distance.cuh"

namespace raft {
namespace cluster {
namespace hdbscan {

enum class cluster_selection_method { EOM = B2D_HDBSCAN_EOM, LEAF = B2D_HDBSCAN_LEAF };

/** cuML's HDBSCANParams without alpha and max_cluster_size.  min_samples = 0 means min_cluster_size. */
struct params {
  int min_cluster_size                    = 5;
  int min_samples                         = 0;
  double cluster_selection_epsilon        = 0.0;
  cluster_selection_method method         = cluster_selection_method::EOM;
  bool allow_single_cluster               = false;
  int64_t n_landmarks                     = 0;
  uint64_t seed                           = 0;
};

/** A fitted HDBSCAN for approximate_predict: one device buffer (the fit's ball cover with its own copy of the points,
 * the core distances and the condensed tree) and the extents it was fitted with.  Filled by the fit overload below. */
class prediction_model {
 public:
  int64_t n_rows() const { return m_; }
  int64_t n_cols() const { return d_; }
  bool is_fitted() const { return buf_ != nullptr; }
  const void* data() const { return buf_ ? buf_->data() : nullptr; }

 private:
  friend struct model_access;
  std::unique_ptr<raft::b200::scoped_workspace> buf_;
  int64_t m_ = 0, d_ = 0, n_landmarks_ = 0;
  int metric_ = 0, min_samples_ = 0;
};

namespace detail {
inline raft::distance::DistanceType unexpanded(raft::distance::DistanceType metric)
{
  using raft::distance::DistanceType;
  if (metric == DistanceType::L2SqrtExpanded) return DistanceType::L2SqrtUnexpanded;
  if (metric == DistanceType::L2Expanded) return DistanceType::L2Unexpanded;
  return metric;
}
}  // namespace detail

struct model_access {
  static void set(prediction_model& pm, raft::resources const& handle, size_t bytes, int64_t m, int64_t d,
                  int64_t n_landmarks, int metric, int min_samples)
  {
    pm.buf_ = std::make_unique<raft::b200::scoped_workspace>(handle, bytes);
    pm.m_ = m, pm.d_ = d, pm.n_landmarks_ = n_landmarks, pm.metric_ = metric, pm.min_samples_ = min_samples;
  }
  static void* data(prediction_model& pm) { return pm.buf_ ? pm.buf_->data() : nullptr; }
  static int metric(const prediction_model& pm) { return pm.metric_; }
  static int min_samples(const prediction_model& pm) { return pm.min_samples_; }
  static int64_t n_landmarks(const prediction_model& pm) { return pm.n_landmarks_; }
};

namespace detail {
inline int fit_call(raft::resources const& handle, const float* x, int64_t ldx, int64_t m, int64_t d, const params& p,
                    raft::distance::DistanceType metric, int* labels, float* probabilities,
                    prediction_model* model = nullptr)
{
  metric = unexpanded(metric);
  const size_t need = b2d_hdbscan_rbc_workspace_bytes(m, d, p.n_landmarks);
  const size_t ws   = need != SIZE_MAX ? need : 0;   // invalid extents: the fit says which
  const size_t tree = m > 1 ? (static_cast<size_t>(m - 1) * 4 + 255) / 256 * 256 : 0;
  raft::b200::scoped_workspace buf(handle, ws + 3 * tree);   // the workspace, then the tree's three arrays
  char* base = static_cast<char*>(buf.data());
  int32_t n_clusters = 0;
  const int ms       = p.min_samples > 0 ? p.min_samples : p.min_cluster_size;
  int32_t* src       = m > 1 ? reinterpret_cast<int32_t*>(base + ws) : nullptr;
  int32_t* dst       = m > 1 ? reinterpret_cast<int32_t*>(base + ws + tree) : nullptr;
  float* w           = m > 1 ? reinterpret_cast<float*>(base + ws + 2 * tree) : nullptr;
  cudaStream_t s     = raft::resource::get_cuda_stream(handle);
  if (!model) {
    raft::distance::detail::b2d_check(b2d_hdbscan_rbc_fit(
      s, static_cast<int>(metric), x, ldx, m, d, ms, p.min_cluster_size, p.cluster_selection_epsilon,
      static_cast<int>(p.method), p.allow_single_cluster ? 1 : 0, p.n_landmarks, p.seed, labels, probabilities, src, dst,
      w, &n_clusters, base, ws));
    return n_clusters;
  }
  const size_t mb = b2d_hdbscan_rbc_model_bytes(m, d, p.n_landmarks);
  model_access::set(*model, handle, mb != SIZE_MAX ? mb : 0, m, d, p.n_landmarks, static_cast<int>(metric), ms);
  raft::distance::detail::b2d_check(b2d_hdbscan_rbc_fit_model(
    s, static_cast<int>(metric), x, ldx, m, d, ms, p.min_cluster_size, p.cluster_selection_epsilon,
    static_cast<int>(p.method), p.allow_single_cluster ? 1 : 0, p.n_landmarks, p.seed, labels, probabilities, src, dst, w,
    &n_clusters, base, ws, model_access::data(*model)));
  return n_clusters;
}
}  // namespace detail

/** HDBSCAN of the rows of X: labels [m] (-1: noise) and probabilities [m]; returns the number of clusters. */
template <typename LabelsView, typename ProbView>
int fit(raft::resources const& handle, raft::device_matrix_view<const float, int, raft::row_major> X, LabelsView labels,
        ProbView probabilities, const params& p = params{},
        raft::distance::DistanceType metric = raft::distance::DistanceType::L2SqrtUnexpanded)
{
  const int64_t m = X.extent(0), d = X.extent(1);
  RAFT_EXPECTS(static_cast<int64_t>(labels.extent(0)) == m, "hdbscan: labels must have m entries");
  RAFT_EXPECTS(static_cast<int64_t>(probabilities.extent(0)) == m, "hdbscan: probabilities must have m entries");
  const int64_t ldx = m > 1 ? static_cast<int64_t>(X.stride(0)) : d;
  return detail::fit_call(handle, X.data_handle(), ldx, m, d, p, metric, labels.data_handle(),
                          probabilities.data_handle());
}

/** Pointer form in cuML's argument order: x [n_rows, n_cols] row-major contiguous, labels [n_rows], probabilities
 * [n_rows]; returns the number of clusters. */
inline int fit(raft::resources const& handle, const float* x, int n_rows, int n_cols, raft::distance::DistanceType metric,
               const params& p, int* labels, float* probabilities)
{
  return detail::fit_call(handle, x, n_cols, n_rows, n_cols, p, metric, labels, probabilities);
}

/** fit, keeping the fitted model in `model` for approximate_predict (labels, probabilities and the count as fit's). */
template <typename LabelsView, typename ProbView>
int fit(raft::resources const& handle, raft::device_matrix_view<const float, int, raft::row_major> X, LabelsView labels,
        ProbView probabilities, prediction_model& model, const params& p = params{},
        raft::distance::DistanceType metric = raft::distance::DistanceType::L2SqrtUnexpanded)
{
  const int64_t m = X.extent(0), d = X.extent(1);
  RAFT_EXPECTS(static_cast<int64_t>(labels.extent(0)) == m, "hdbscan: labels must have m entries");
  RAFT_EXPECTS(static_cast<int64_t>(probabilities.extent(0)) == m, "hdbscan: probabilities must have m entries");
  const int64_t ldx = m > 1 ? static_cast<int64_t>(X.stride(0)) : d;
  return detail::fit_call(handle, X.data_handle(), ldx, m, d, p, metric, labels.data_handle(),
                          probabilities.data_handle(), &model);
}

/** Places the rows of queries [q, d] (d the model's, any row pitch) in a fitted model: labels [q] (-1: noise) and
 * probabilities [q], in the fit's numbering.  Only enqueues work on the handle's stream. */
template <typename LabelsView, typename ProbView>
void approximate_predict(raft::resources const& handle, const prediction_model& model,
                         raft::device_matrix_view<const float, int, raft::row_major> queries, LabelsView labels,
                         ProbView probabilities)
{
  const int64_t q = queries.extent(0);
  RAFT_EXPECTS(model.is_fitted(), "hdbscan: approximate_predict needs a model filled by fit");
  RAFT_EXPECTS(queries.extent(1) == model.n_cols(), "hdbscan: queries must have the model's number of columns");
  RAFT_EXPECTS(static_cast<int64_t>(labels.extent(0)) == q, "hdbscan: labels must have one entry per query");
  RAFT_EXPECTS(static_cast<int64_t>(probabilities.extent(0)) == q, "hdbscan: probabilities must have one entry per query");
  const int64_t ldq = q > 1 ? static_cast<int64_t>(queries.stride(0)) : model.n_cols();
  raft::distance::detail::b2d_check(b2d_hdbscan_rbc_approximate_predict(
    raft::resource::get_cuda_stream(handle), model.data(), model.n_rows(), model.n_cols(), model_access::metric(model),
    model_access::n_landmarks(model), model_access::min_samples(model), queries.data_handle(), ldq, q,
    labels.data_handle(), probabilities.data_handle(), nullptr, nullptr));
}

}  // namespace hdbscan
}  // namespace cluster
}  // namespace raft
