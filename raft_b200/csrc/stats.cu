// silhouette_score and trustworthiness_score (stats.cuh) on the pairwise distance and the fused kNN.
#include <cuda_runtime.h>
#include <algorithm>
#include <string>

#include "host.cuh"
#include "stats.cuh"

using namespace b2d;

// ------------------------------------------------------------------------------------------
// raft::stats::silhouette_score on the distance engine (SURVEY.md 8(f3); stats.cuh)

namespace {
// silhouette and trustworthiness work through the n x n distances in [chunk x n] fp32 slabs, row pitch ld: chunk is the
// caller's row count or about 1 GiB, a multiple of 128 and at most max(n, 1)
struct Slab {
  int64_t chunk, ld;
};
Slab slab_shape(int64_t n, int64_t chunk_rows)
{
  Slab sl;
  sl.ld     = (n + 3) / 4 * 4;
  int64_t c = chunk_rows > 0 ? chunk_rows : (int64_t(1) << 30) / (4 * std::max<int64_t>(sl.ld, 1));
  c         = std::max<int64_t>(128, c / 128 * 128);
  sl.chunk  = std::min<int64_t>(c, std::max<int64_t>(n, 1));
  return sl;
}

struct SilLayout {
  Slab sl;
  int *counts, *offsets, *cursor;  // zeroed together with bad and total: everything in front of where
  unsigned* bad;
  double* total;
  int* where;
  float *ys, *slab;
  void* pw;                        // b2d_pairwise_distance's workspace
  size_t pw_bytes, bytes;
};
SilLayout sil_layout(void* base, int64_t n, int64_t k, int n_labels, int metric, int64_t chunk_rows)
{
  Carve c(base, 1024);
  SilLayout L;
  L.sl       = slab_shape(n, chunk_rows);
  L.counts   = c.take<int>(n_labels);
  L.offsets  = c.take<int>(n_labels + 1);
  L.cursor   = c.take<int>(n_labels);
  L.bad      = c.take<unsigned>(1);
  L.total    = c.take<double>(1);
  L.where    = c.take<int>(n);
  L.ys       = c.take<float>(static_cast<size_t>(n) * k);
  L.slab     = c.take<float>(static_cast<size_t>(L.sl.chunk) * L.sl.ld);
  L.pw_bytes = b2d_pairwise_workspace_bytes(metric, B2D_F32, L.sl.chunk, n, k);
  L.pw       = c.take<char>(L.pw_bytes == static_cast<size_t>(-1) ? 0 : L.pw_bytes);
  L.bytes    = c.bytes;
  return L;
}
}  // namespace

size_t b2d_silhouette_score_workspace_bytes(int64_t n, int64_t k, int n_labels, int metric, int64_t chunk_rows)
{
  if (n < 0 || k < 0 || n_labels < 1 || chunk_rows < 0) return static_cast<size_t>(-1);
  if (b2d_pairwise_workspace_bytes(metric, B2D_F32, 1, 1, k) == static_cast<size_t>(-1)) return static_cast<size_t>(-1);
  return sil_layout(nullptr, n, k, n_labels, metric, chunk_rows).bytes;
}

int b2d_silhouette_score(void* stream, float* score, float* per_sample, const float* x, int64_t ldx, const int* labels,
                         int64_t n, int64_t k, int n_labels, int metric, float metric_arg, int64_t chunk_rows,
                         void* workspace, size_t workspace_bytes)
{
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (n < 0 || k <= 0 || chunk_rows < 0) return fail(B2D_ERR_INVALID_ARG, "bad extent");
  if (!score || !x || !labels) return fail(B2D_ERR_INVALID_ARG, "null score / x / labels");
  if (n_labels < 2 || n_labels > n - 1)
    return fail(B2D_ERR_INVALID_ARG, "silhouette score is not defined for this number of labels (need 2 <= n_labels <= n - 1)");
  if (n_labels > 12000) return fail(B2D_ERR_UNSUPPORTED, "n_labels > 12000");
  if (ldx < k) return fail(B2D_ERR_INVALID_ARG, "leading dimension smaller than k");
  const size_t need = b2d_silhouette_score_workspace_bytes(n, k, n_labels, metric, chunk_rows);
  if (need == static_cast<size_t>(-1)) return fail(B2D_ERR_UNSUPPORTED, "metric " + std::to_string(metric) + " is not on the tensor-core / SIMT distance path");
  int rc = check_workspace(workspace, workspace_bytes, need);
  if (rc) return rc;
  const SilLayout L = sil_layout(workspace, n, k, n_labels, metric, chunk_rows);
  B2D_CUDA(cudaMemsetAsync(workspace, 0, reinterpret_cast<char*>(L.where) - static_cast<char*>(workspace), s));
  const unsigned nb = static_cast<unsigned>((n + 255) / 256);
  sil_count_kernel<<<nb, 256, 0, s>>>(labels, L.counts, n, n_labels, L.bad);
  sil_scan_kernel<<<1, 32, 0, s>>>(L.counts, L.offsets, L.cursor, n_labels);
  sil_gather_kernel<<<static_cast<unsigned>((n + 7) / 8), 256, 0, s>>>(x, ldx, labels, L.cursor, L.ys, L.where, n, static_cast<int>(k), n_labels);
  B2D_CUDA(cudaGetLastError());
  // labels outside [0, n_labels) are detected on the device (no host round trip: the call stays asynchronous);
  // they poison the result: *score and the per-sample values of the offending rows become NaN
  for (int64_t r0 = 0; r0 < n; r0 += L.sl.chunk) {
    const int64_t rows = std::min<int64_t>(L.sl.chunk, n - r0);
    rc = b2d_pairwise_distance(stream, metric, B2D_F32, x + r0 * ldx, ldx, L.ys, k, L.slab, L.sl.ld, rows, n, k, 1,
                               metric_arg, L.pw, L.pw_bytes);
    if (rc) return rc;
    sil_row_kernel<<<static_cast<unsigned>(rows), 256, static_cast<size_t>(n_labels) * 4, s>>>(
      L.slab, L.sl.ld, r0, rows, labels, L.counts, L.offsets, L.where, n_labels, per_sample, L.total);
    B2D_CUDA(cudaGetLastError());
  }
  sil_finish_kernel<<<1, 32, 0, s>>>(L.total, score, n, L.bad, L.counts, n_labels);
  B2D_CUDA(cudaGetLastError());
  return B2D_OK;
}

// raft::stats::trustworthiness_score on the kNN + distance engine (stats.cuh)
namespace {
struct TrustLayout {
  Slab sl;
  unsigned long long* penalty;
  int64_t* emb_idx;
  float *emb_dist, *slab;
  void* scratch;    // the kNN's workspace, then b2d_pairwise_distance's
  size_t knn_bytes, pw_bytes, bytes;
};
TrustLayout trust_layout(void* base, int64_t n, int64_t m, int64_t d, int n_neighbors, int metric, int64_t batch_rows)
{
  Carve c(base, 1024);
  TrustLayout L;
  L.sl        = slab_shape(n, batch_rows);
  L.penalty   = c.take<unsigned long long>(1);
  L.emb_idx   = c.take<int64_t>(static_cast<size_t>(n) * (n_neighbors + 1));
  L.emb_dist  = c.take<float>(static_cast<size_t>(n) * (n_neighbors + 1));
  L.slab      = c.take<float>(static_cast<size_t>(L.sl.chunk) * L.sl.ld);
  L.knn_bytes = b2d_knn_l2_workspace_bytes(n, n, d, n_neighbors + 1);
  L.pw_bytes  = b2d_pairwise_workspace_bytes(metric, B2D_F32, L.sl.chunk, n, m);
  const size_t a = L.knn_bytes == static_cast<size_t>(-1) ? 0 : L.knn_bytes;
  const size_t b = L.pw_bytes == static_cast<size_t>(-1) ? 0 : L.pw_bytes;
  L.scratch   = c.take<char>(std::max(a, b));
  L.bytes     = c.bytes;
  return L;
}
}  // namespace

size_t b2d_trustworthiness_score_workspace_bytes(int64_t n, int64_t m, int64_t d, int n_neighbors, int metric,
                                                 int64_t batch_rows)
{
  if (n < 0 || m < 0 || d < 0 || n_neighbors < 1 || n_neighbors + 1 > KNN_MAX_K || batch_rows < 0) return static_cast<size_t>(-1);
  if (b2d_pairwise_workspace_bytes(metric, B2D_F32, 1, 1, m) == static_cast<size_t>(-1)) return static_cast<size_t>(-1);
  return trust_layout(nullptr, n, m, d, n_neighbors, metric, batch_rows).bytes;
}

int b2d_trustworthiness_score(void* stream, double* score, const float* x, int64_t ldx, const float* x_embedded,
                              int64_t lde, int64_t n, int64_t m, int64_t d, int n_neighbors, int metric,
                              int64_t batch_rows, void* workspace, size_t workspace_bytes)
{
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (n < 0 || m <= 0 || d <= 0 || batch_rows < 0) return fail(B2D_ERR_INVALID_ARG, "bad extent");
  if (!score || !x || !x_embedded) return fail(B2D_ERR_INVALID_ARG, "null score / x / x_embedded");
  // the reference uses distance_type for BOTH spaces (trustworthiness_score<math_t, distance_type>,
  // cpp/include/raft/stats/detail/trustworthiness_score.cuh:113-211): the embedded-space neighbours come from
  // the fused kNN, which covers the L2 and the cosine families
  int knn_metric = metric;
  if (metric == B2D_L2Unexpanded) knn_metric = B2D_L2Expanded;
  if (metric == B2D_L2SqrtUnexpanded) knn_metric = B2D_L2SqrtExpanded;
  if (knn_metric != B2D_L2Expanded && knn_metric != B2D_L2SqrtExpanded && knn_metric != B2D_CosineExpanded &&
      knn_metric != B2D_CorrelationExpanded)
    return fail(B2D_ERR_UNSUPPORTED, "trustworthiness_score supports the L2 metrics, CosineExpanded and CorrelationExpanded");
  if (n_neighbors < 1 || n_neighbors + 1 > KNN_MAX_K) return fail(B2D_ERR_UNSUPPORTED, "n_neighbors must be in [1, 63]");
  if (2 * n - 3 * static_cast<int64_t>(n_neighbors) - 1 <= 0 || n_neighbors + 1 > n)
    return fail(B2D_ERR_INVALID_ARG, "n_neighbors must be smaller than n / 2");
  if (ldx < m || lde < d) return fail(B2D_ERR_INVALID_ARG, "leading dimension smaller than the row length");
  const size_t need = b2d_trustworthiness_score_workspace_bytes(n, m, d, n_neighbors, metric, batch_rows);
  if (need == static_cast<size_t>(-1)) return fail(B2D_ERR_UNSUPPORTED, "metric " + std::to_string(metric) + " is not on the tensor-core / SIMT distance path");
  int rc = check_workspace(workspace, workspace_bytes, need);
  if (rc) return rc;
  const TrustLayout L = trust_layout(workspace, n, m, d, n_neighbors, metric, batch_rows);
  const int kk1       = n_neighbors + 1;
  B2D_CUDA(cudaMemsetAsync(L.penalty, 0, 8, s));
  // neighbours in the embedded space (the sample itself included, as in the reference)
  rc = b2d_knn(stream, L.emb_idx, L.emb_dist, knn_metric, x_embedded, lde, x_embedded, lde, n, n, d, kk1, L.scratch,
               L.knn_bytes);
  if (rc) return rc;
  for (int64_t r0 = 0; r0 < n; r0 += L.sl.chunk) {
    const int64_t rows = std::min<int64_t>(L.sl.chunk, n - r0);
    rc = b2d_pairwise_distance(stream, metric, B2D_F32, x + r0 * ldx, ldx, x, ldx, L.slab, L.sl.ld, rows, n, m, 1, 2.0f,
                               L.scratch, L.pw_bytes);
    if (rc) return rc;
    trust_rank_kernel<<<static_cast<unsigned>(rows), 256, 0, s>>>(L.slab, L.sl.ld, r0, n, L.emb_idx, kk1, n_neighbors, L.penalty);
    B2D_CUDA(cudaGetLastError());
  }
  trust_finish_kernel<<<1, 1, 0, s>>>(L.penalty, score, n, n_neighbors);
  B2D_CUDA(cudaGetLastError());
  return B2D_OK;
}
