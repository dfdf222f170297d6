// k-means|| seeding (scalable k-means++, Bahmani et al. 2012) and the fit that starts from it (DESIGN.md section 2, K12).
// Every launch size is known on the host: the candidate set has exactly C = 1 + 8L rows, so no call synchronises.
#include <cuda_runtime.h>
#include <algorithm>
#include <cmath>

#include "host.cuh"

using namespace b2d;

namespace {
constexpr int kParRounds = 8;   // oversampling rounds after the first draw

// L = min(m, max(ceil(f nc), ceil((nc - 1) / 8))) rows per oversampling round; C = 1 + 8L >= nc
struct KmParSizes {
  int64_t L, C;
};

KmParSizes km_par_sizes(int64_t m, int64_t nc, double f)
{
  const double want = std::max(std::ceil(f * static_cast<double>(nc)),
                               std::ceil(static_cast<double>(nc - 1) / kParRounds));
  KmParSizes z;
  z.L = static_cast<int64_t>(std::max(0.0, std::min(static_cast<double>(m), want)));
  z.C = 1 + kParRounds * z.L;
  return z;
}

// The fit's own layout, the candidate set, then two phases that share their bytes: the rounds and the weights pass (x
// against at most C rows), and the recluster on the C candidates.
struct KmParLayout {
  KmLayout fit;     // (m, k, nc): b2d_kmeans_fit_scalable's Lloyd loop
  KmParSizes z;
  float* cand;      // [C, k] candidate rows: round 0 at 0, round r >= 1 at 1 + (r - 1) L
  int* ids;         // [C] their row ids
  float* W;         // [C] candidate weights
  // phase 1: the rounds and the weights pass
  float* d2;        // [m] D^2
  float* key;       // [m] sampling keys
  float* sk_val;    // select_k (1, m, L) outputs and scratch
  int64_t* sk_idx;
  void* sk_ws;
  size_t sk_bytes;
  KmLayout x_c;     // (m, k, C): x prepared once, the arg-min against a round's rows or all C, the weight sums
  // phase 2
  KmLayout rec;     // (C, k, nc): greedy k-means++ and Lloyd on the weighted candidates
  size_t bytes;
};

char* at(void* base, size_t off) { return base ? static_cast<char*>(base) + off : nullptr; }

KmParLayout km_par_layout(void* base, int64_t m, int64_t k, int64_t nc, const KmParSizes& z)
{
  KmParLayout P{};
  P.z = z;
  Carve c(base, 1024);
  P.fit = km_layout(base, m, k, nc);
  c.take<char>(P.fit.bytes);
  P.cand = c.take<float>(static_cast<size_t>(z.C) * k);
  P.ids  = c.take<int>(z.C);
  P.W    = c.take<float>(z.C);
  Carve a(at(base, c.bytes), 1024);
  P.d2       = a.take<float>(m);
  P.key      = a.take<float>(m);
  P.sk_val   = a.take<float>(std::max<int64_t>(z.L, 1));
  P.sk_idx   = a.take<int64_t>(std::max<int64_t>(z.L, 1));
  P.sk_bytes = (m >= 1 && z.L >= 1) ? std::max(b2d_select_k_workspace_bytes(1, m, 1), b2d_select_k_workspace_bytes(1, m, z.L))
                                    : 0;
  P.sk_ws    = a.take<char>(P.sk_bytes);
  P.x_c      = km_layout(at(base, c.bytes + a.bytes), m, k, z.C);
  P.rec      = km_layout(at(base, c.bytes), z.C, k, nc);
  P.bytes    = c.bytes + std::max(a.bytes + P.x_c.bytes, P.rec.bytes);
  return P;
}

int km_par_args(double f, int64_t m, int64_t nc)
{
  if (!std::isfinite(f) || !(f > 0.0)) return fail(B2D_ERR_INVALID_ARG, "oversampling_factor must be finite and > 0");
  if (km_par_sizes(m, nc, f).C > 0x7fffffffll)
    return fail(B2D_ERR_UNSUPPORTED, "k-means|| candidate set of 1 + 8 L rows must stay below 2^31");
  return B2D_OK;
}

// The seeding: round 0 draws one row with probability ~ w, rounds 1..8 draw L rows without replacement with
// probability ~ w D^2, D^2 folded after each round by the arg-min against that round's rows; the candidates are weighted
// by the w of the rows nearest to them, then reclustered (greedy k-means++ and Lloyd) into centroids [nc, k].
// ids / W: where the candidate ids and weights go (P.ids / P.W, or the caller's outputs).
int km_scalable(cudaStream_t s, const KmParLayout& P, const float* x, int64_t ldx, const float* w, int64_t m, int64_t k,
                int64_t nc, uint64_t seed, float* centroids, int* ids, float* W)
{
  const KmLayout& X = P.x_c;
  const int64_t L = P.z.L, C = P.z.C;
  km_par_keys(s, nullptr, P.d2, w, m, seed, 0, P.key);
  B2D_CUDA(cudaGetLastError());
  for (int r = 0; r <= kParRounds; ++r) {
    const int64_t n    = r == 0 ? 1 : L;
    const int64_t off  = r == 0 ? 0 : 1 + (r - 1) * L;
    float* rows        = P.cand + off * k;
    int rc = b2d_select_k(s, P.key, m, nullptr, 1, m, n, 1, P.sk_val, P.sk_idx, P.sk_ws, P.sk_bytes);
    if (rc) return rc;
    km_par_take(s, x, ldx, static_cast<int>(k), P.sk_idx, static_cast<int>(n), rows, ids + off, P.d2);
    B2D_CUDA(cudaGetLastError());
    if (r == kParRounds) break;
    if (r == 0) {   // x is prepared once, with the first candidate
      rc = launch_prep<float>(s, X.tc, x, ldx, 1, m, rows, k, 1, n, k, nullptr, nullptr, TC_L2);
      if (rc) return rc;
    }
    rc = km_assign(s, X, m, k, n, rows, nullptr, X.labels, nullptr, r > 0, false);
    if (rc) return rc;
    km_par_keys(s, X.tc.keys, P.d2, w, m, seed, r + 1, P.key);
    B2D_CUDA(cudaGetLastError());
  }
  // W_c = sum of w over the rows whose nearest candidate is c (b2d_kmeans_update_centroids' weight_per_cluster)
  int rc = km_assign(s, X, m, k, C, P.cand, nullptr, X.labels, nullptr, true, true);
  if (rc) return rc;
  rc = km_update(s, X, x, ldx, m, k, C, w, X.labels, P.cand, X.best, W, nullptr);
  if (rc) return rc;
  // the recluster: b2d_kmeans_fit's loop on the candidates with weights W, greedy k-means++, max_iter 300, tol 1e-4
  const KmLayout& R = P.rec;
  km_ctrl_init(s, R.ctrl);
  const float* wr = km_weights(s, R, W, C, true);
  B2D_CUDA(cudaGetLastError());
  return km_fit_runs(s, R, P.cand, k, wr, C, k, nc, 300, 1e-4, 0, 1, centroids, nullptr, nullptr,
                     [&](int) { return km_plus_plus(s, R, P.cand, k, wr, C, k, nc, seed, centroids); });
}
}  // namespace

size_t b2d_kmeans_scalable_workspace_bytes(int64_t m, int64_t k, int64_t n_clusters, double oversampling_factor)
{
  if (m < 0 || k < 0 || n_clusters < 0) return static_cast<size_t>(-1);
  if (!std::isfinite(oversampling_factor) || !(oversampling_factor > 0.0)) return static_cast<size_t>(-1);
  const KmParSizes z = km_par_sizes(m, n_clusters, oversampling_factor);
  if (z.C > 0x7fffffffll) return static_cast<size_t>(-1);
  return km_par_layout(nullptr, m, k, n_clusters, z).bytes;
}

int b2d_kmeans_init_scalable(void* stream, const float* x, int64_t ldx, const float* sample_weight, int64_t m, int64_t k,
                             int n_clusters, double oversampling_factor, uint64_t seed, float* centroids,
                             int32_t* candidates, float* candidate_weights, void* workspace, size_t workspace_bytes)
{
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (m == 0) return B2D_OK;
  int rc = km_args(x, ldx, m, k, n_clusters, centroids);
  if (rc) return rc;
  rc = km_par_args(oversampling_factor, m, n_clusters);
  if (rc) return rc;
  const int64_t nc = n_clusters;
  const KmParSizes z = km_par_sizes(m, nc, oversampling_factor);
  rc = check_workspace(workspace, workspace_bytes, km_par_layout(nullptr, m, k, nc, z).bytes);
  if (rc) return rc;
  const KmParLayout P = km_par_layout(workspace, m, k, nc, z);
  return km_scalable(s, P, x, ldx, sample_weight, m, k, nc, seed, centroids, candidates ? candidates : P.ids,
                     candidate_weights ? candidate_weights : P.W);
}

int b2d_kmeans_fit_scalable(void* stream, int n_clusters, int max_iter, double tol, double oversampling_factor, int n_init,
                            uint64_t seed, int inertia_check, const float* x, int64_t ldx, const float* sample_weight,
                            int64_t m, int64_t k, float* centroids, double* inertia, int32_t* n_iter, void* workspace,
                            size_t workspace_bytes)
{
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (m == 0) return B2D_OK;
  int rc = km_args(x, ldx, m, k, n_clusters, centroids);
  if (rc) return rc;
  rc = km_fit_args(inertia, n_iter, max_iter, tol, B2D_KMEANS_INIT_PLUS_PLUS, n_init);
  if (rc) return rc;
  rc = km_par_args(oversampling_factor, m, n_clusters);
  if (rc) return rc;
  const int64_t nc = n_clusters;
  const KmParSizes z = km_par_sizes(m, nc, oversampling_factor);
  rc = check_workspace(workspace, workspace_bytes, km_par_layout(nullptr, m, k, nc, z).bytes);
  if (rc) return rc;
  const KmParLayout P = km_par_layout(workspace, m, k, nc, z);
  const KmLayout& L  = P.fit;
  km_ctrl_init(s, L.ctrl);
  const float* w = km_weights(s, L, sample_weight, m, true);
  B2D_CUDA(cudaGetLastError());
  return km_fit_runs(s, L, x, ldx, w, m, k, nc, max_iter, tol, inertia_check, n_init, centroids, inertia, n_iter,
                     [&](int r) { return km_scalable(s, P, x, ldx, w, m, k, nc, seed + r, centroids, P.ids, P.W); });
}
